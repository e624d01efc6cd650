"""Encoding into a fixed-size destination: test infrastructure for k4lz4_encode_dest_size(_batch).

* ``Upstream`` calls upstream lz4's ``LZ4_compress_default``, ``LZ4_compress_destSize`` and
  ``LZ4_decompress_safe`` through ctypes on the reference engine the oracle builds (``oracle/_ref/libk4ref.so``).
* ``model(seqs, n, target)`` is the sequence-level model of upstream's fillOutput directive
  (lz4.c:1028-1032, 1057-1062, 1097-1117, 1206-1218).  Its input is upstream's plain encoding of the same n bytes,
  parsed with ``tests.lz4_blocks.parse``.  The search never reads the output limit, so the fill encoder emits
  the plain encoder's sequences up to a cut, and four rules decide where the cut falls:

  1. literal rule: the sequence's token, literal-length bytes, literals, offset and MFLIMIT - MINMATCH would
     pass the target; the sequence is dropped and the rest goes to last literals;
  2. next-match rule: the same test for a zero-literal sequence (the match right after a match);
  3. match-length rule: the match-length bytes would pass the target; the match is shortened to
     14 + (target - op - 6) * 255 and no later sequence can fit;
  4. last-literal rule: the last run is cut to room - 1 - (room - 1 + 241) // 256.

  Rules 1 and 2 are one test (the run header's extra bytes are (lit + 240) // 255), so a sequence whose literal
  run the catch-up shrank to nothing is reported as rule 2 too: upstream tests it in rule 1's place, with the
  same result.  ``rule`` is the first rule that fired, or None where the whole input fits.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from tests.lz4_blocks import parse

MINMATCH, MFLIMIT, LASTLITERALS, RUN_MASK = 4, 12, 5, 15
MAX_INPUT_SIZE = 0x7E000000
LIMIT_64K = 65536 + 11


def bound(n: int) -> int:
    """LZ4_compressBound: 0 beyond LZ4_MAX_INPUT_SIZE (and for negative sizes)."""
    return 0 if n < 0 or n > MAX_INPUT_SIZE else n + n // 255 + 16


def _hdr(run: int) -> int:
    return 1 + ((run - 15) // 255 + 1 if run >= 15 else 0)


def _ext(mc: int) -> int:
    """match-length bytes after the token for a match code (match length - MINMATCH)"""
    return (mc - 15) // 255 + 1 if mc >= 15 else 0


def last_cut(room: int) -> int:
    """Rule 4 (lz4.c:1212-1213): the longest last run that fits `room` bytes, token and length bytes included."""
    run = room - 1
    return run - (run + 256 - RUN_MASK) // 256


def last_cut_1_9_2(room: int) -> int:
    """lz4 1.9.2's rule 4, (run + 240) // 255 length bytes (the reference's unreachable branch).  It differs from
    upstream on incompressible input, and model() takes it only to show that."""
    run = room - 1
    return run - (run + 240) // 255


def model(seqs, n: int, target: int, cut=last_cut):
    """-> (result, consumed, rule) of LZ4_compress_destSize on n bytes whose plain encoding parses to `seqs`.
    Where nothing is written, consumed is 0 (k4lz4_encode_dest_size's convention)."""
    if target < 1 or n < 0 or n > MAX_INPUT_SIZE:
        return 0, 0, None
    if target >= bound(n):                              # lz4.c:1387-1388: the plain encoder, everything consumed
        return (sum(s.next - s.tp for s in seqs) if n else 1), n, None
    op, anchor, rule = 0, 0, None
    for k, s in enumerate(seqs):
        if s.ml == 0:                                   # the terminal literal run
            break
        after_off = op + _hdr(s.lit) + s.lit + 2
        if after_off + 1 + (MFLIMIT - MINMATCH) > target:   # rules 1 and 2
            rule = 2 if s.lit == 0 and k > 0 else 1
            break
        mc = s.ml - MINMATCH
        if after_off + 1 + LASTLITERALS + (mc + 240) // 255 > target:   # rule 3
            mc = 14 + (target - after_off - 1 - LASTLITERALS) * 255
            op, anchor, rule = after_off + _ext(mc), anchor + s.lit + mc + MINMATCH, 3
            break
        op, anchor = after_off + _ext(mc), anchor + s.lit + s.ml
    run = n - anchor
    if op + run + 1 + (run + 255 - RUN_MASK) // 255 > target:         # rule 4
        run = cut(target - op)
        rule = rule or 4
    return op + _hdr(run) + run, anchor + run, rule


def rule_targets(seqs, n: int, first: int = 400) -> dict:
    """{rule: the smallest target at which model() reports it} over the targets that sit at the thresholds of the
    first `first` sequences (the largest target each of rules 1-3 still cuts at) and one byte below the whole block."""
    cand, op = set(), 0
    for s in seqs[:first]:
        if s.ml == 0:
            break
        after_off = op + _hdr(s.lit) + s.lit + 2
        mc = s.ml - MINMATCH
        cand |= {after_off + MFLIMIT - MINMATCH, after_off + LASTLITERALS + (mc + 240) // 255}
        op = after_off + _ext(mc)
    cand.add(sum(s.next - s.tp for s in seqs) - 1)
    found: dict = {}
    for t in sorted(x for x in cand if x >= 1):
        rule = model(seqs, n, t)[2]
        if rule is not None and rule not in found:
            found[rule] = t
    return found


class Upstream:
    """Upstream lz4's block calls on the oracle's reference engine."""

    def __init__(self):
        import oracle
        self._lib = lib = C.CDLL(oracle.REF_SO)
        lib.LZ4_compress_default.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        lib.LZ4_compress_destSize.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int]
        lib.LZ4_decompress_safe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]

    def plain(self, src: bytes) -> bytes:
        s = np.frombuffer(src, dtype=np.uint8) if src else np.zeros(1, dtype=np.uint8)
        d = np.zeros(bound(len(src)) + 1, dtype=np.uint8)
        r = self._lib.LZ4_compress_default(s.ctypes.data, d.ctypes.data, len(src), bound(len(src)))
        assert r > 0
        return d[:r].tobytes()

    def dest_size(self, src: bytes, target: int):
        """-> (result, consumed, bytes) of LZ4_compress_destSize; consumed is what upstream leaves in its size
        argument, which it does not touch where it writes nothing."""
        s = np.frombuffer(src, dtype=np.uint8) if src else np.zeros(1, dtype=np.uint8)
        d = np.full(max(target, 0) + 64, 0xCD, dtype=np.uint8)
        n = C.c_int(len(src))
        r = self._lib.LZ4_compress_destSize(s.ctypes.data, d.ctypes.data, C.byref(n), target)
        assert (d[max(r, 0):] == 0xCD).all(), "upstream wrote past its result"
        return r, n.value, d[:max(r, 0)].tobytes()

    def decode(self, block: bytes, cap: int) -> bytes:
        s = np.frombuffer(block, dtype=np.uint8)
        d = np.zeros(max(cap, 1), dtype=np.uint8)
        r = self._lib.LZ4_decompress_safe(s.ctypes.data, d.ctypes.data, len(block), cap)
        assert r >= 0, r
        return d[:r].tobytes()

    def model(self, src: bytes, target: int, cut=last_cut):
        """model() on upstream's plain encoding of src."""
        return model(parse(self.plain(src)) if src else [], len(src), target, cut)


# ---- inputs and targets of the test grid ----------------------------------------------------------------------

SIZES = [0, 1, 12, 13, 14, 4096, 65535, 65546, 65547, 65548, 300000, 1 << 20]
KINDS = ["datagen", "random", "runs"]


def content(kind: str, n: int, seed: int) -> bytes:
    """datagen 0.63 (the reference's generator), random bytes, or long single-byte runs."""
    if n == 0:
        return b""
    if kind == "datagen":
        import oracle
        return oracle.Port().datagen(n, 0.63, 0.0, seed)[:n].tobytes()
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    out = bytearray()
    while len(out) < n:                                 # runs of 1 to 20 000 bytes of one value
        out += bytes([int(rng.integers(0, 256))]) * int(rng.integers(1, 20000))
    return bytes(out[:n])


def targets(n: int, seed: int, extra: int = 6) -> list[int]:
    """0-20, 255, 256, 270-272, n/4, n/2, bound - 1, bound and `extra` seeded random targets below the bound."""
    b = bound(n)
    t = set(range(0, 21)) | {255, 256, 270, 271, 272, n // 4, n // 2, b - 1, b}
    rng = np.random.default_rng(seed)
    t |= {int(x) for x in rng.integers(1, b + 1, extra)}
    return sorted(x for x in t if x >= 0)
