"""Upstream's LZ4F_compressFrame, and a restatement of it over upstream's block calls: test infrastructure for
k4lz4_lz4f_compress_batch.

* ``Lz4fUpstream.frame`` is upstream's own call (oracle/_ref/libk4ref.so, lz4frame.c) at level 0 into a buffer of
  LZ4F_compressFrameBound bytes.
* ``Lz4fUpstream.assemble`` writes the same frame by hand, as the GPU call does: the block size shrinks to the
  smallest of 64 KiB, 256 KiB, 1 MiB that holds the content (LZ4F_optimalBSID), a one-block frame is independent, the
  content size is written when asked for and the content is not empty; then every block is
  LZ4_compress_fast (independent) or LZ4_compress_fast_continue on one fresh stream (linked) with capacity n - 1,
  stored raw with bit 31 when that fails, then the end mark and the content checksum.
* ``grid`` is the seeded case grid both are compared on, on the CPU and on the GPU.
"""
from __future__ import annotations

import ctypes as C
import functools
import struct

import numpy as np

from tests import chain_ref as CR

MAGIC = 0x184D2204
BLOCK_SIZES = [1 << 16, 1 << 18, 1 << 20, 1 << 22]
SIZE_ID = {1 << 16: 4, 1 << 18: 5, 1 << 20: 6, 1 << 22: 7}
INDEPENDENT, BLOCK_CHECKSUM, CONTENT_CHECKSUM, CONTENT_SIZE = 1, 2, 4, 8
SMALL_SIZES = [0, 1, 12, 13, 4095, 4096] + list(range(65535, 65548))
CHECKSUMS = [(False, False), (True, False), (False, True), (True, True)]


def flags_of(linked: bool, bc: bool, cc: bool, cs: bool) -> int:
    return ((0 if linked else INDEPENDENT) | (BLOCK_CHECKSUM if bc else 0) | (CONTENT_CHECKSUM if cc else 0) |
            (CONTENT_SIZE if cs else 0))


def optimal_block_size(bs: int, n: int) -> int:
    """LZ4F_optimalBSID (lz4frame.c:304-316), as a block size."""
    size = 1 << 16
    while size < bs and n > size:
        size <<= 2
    return size


class Lz4fUpstream:
    def __init__(self):
        import oracle
        self.ref = oracle.Ref()
        self.lib = L = C.CDLL(oracle.REF_SO)
        vp, i32, sz = C.c_void_p, C.c_int, C.c_size_t
        L.LZ4F_compressFrameBound.argtypes = [sz, C.POINTER(CR._Prefs)]
        L.LZ4F_compressFrameBound.restype = sz
        L.LZ4F_compressFrame.argtypes = [vp, sz, vp, sz, C.POINTER(CR._Prefs)]
        L.LZ4F_compressFrame.restype = sz
        L.LZ4_compress_fast.argtypes = [vp, vp, i32, i32, i32]
        L.LZ4_compress_fast.restype = i32
        L.LZ4_createStream.restype = vp
        L.LZ4_freeStream.argtypes = [vp]
        L.LZ4_compress_fast_continue.argtypes = [vp, vp, vp, i32, i32, i32]
        L.LZ4_compress_fast_continue.restype = i32

    @staticmethod
    def prefs(bs: int, flags: int, n: int) -> CR._Prefs:
        pr = CR._Prefs()
        pr.frameInfo.blockSizeID = SIZE_ID[bs]
        pr.frameInfo.blockMode = 1 if flags & INDEPENDENT else 0
        pr.frameInfo.blockChecksumFlag = int(bool(flags & BLOCK_CHECKSUM))
        pr.frameInfo.contentChecksumFlag = int(bool(flags & CONTENT_CHECKSUM))
        pr.frameInfo.contentSize = max(n, 1) if flags & CONTENT_SIZE else 0
        return pr

    def bound(self, n: int, bs: int, flags: int) -> int:
        """LZ4F_compressFrameBound(n, prefs)."""
        return int(self.lib.LZ4F_compressFrameBound(n, C.byref(self.prefs(bs, flags, n))))

    def frame(self, data: bytes, bs: int, flags: int) -> bytes:
        pr = self.prefs(bs, flags, len(data))
        cap = self.bound(len(data), bs, flags)
        s = np.frombuffer(bytes(data) + b"\0", dtype=np.uint8)
        d = np.zeros(cap, dtype=np.uint8)
        r = int(self.lib.LZ4F_compressFrame(d.ctypes.data, cap, s.ctypes.data, len(data), C.byref(pr)))
        assert 0 < r <= cap, r
        return d[:r].tobytes()

    def header(self, n: int, bs: int, flags: int) -> bytes:
        size = optimal_block_size(bs, n)
        indep = bool(flags & INDEPENDENT) or n <= size
        cs = bool(flags & CONTENT_SIZE) and n > 0
        flg = (0x40 | (0x20 if indep else 0) | (0x10 if flags & BLOCK_CHECKSUM else 0) | (0x08 if cs else 0) |
               (0x04 if flags & CONTENT_CHECKSUM else 0))
        desc = bytes([flg, SIZE_ID[size] << 4]) + (struct.pack("<Q", n) if cs else b"")
        return struct.pack("<I", MAGIC) + desc + bytes([(self.ref.xxh32(desc) >> 8) & 0xFF])

    def blocks(self, data: bytes, bs: int, flags: int) -> list:
        """(stored bytes, raw) per block, as the assembly encodes them."""
        n = len(data)
        size = optimal_block_size(bs, n)
        linked = not (flags & INDEPENDENT) and n > size
        s = np.frombuffer(bytes(data) + b"\0", dtype=np.uint8)
        d = np.zeros(size + 16, dtype=np.uint8)
        st = self.lib.LZ4_createStream() if linked else None
        out = []
        try:
            for o in range(0, n, size):
                k = min(size, n - o)
                if linked:
                    r = int(self.lib.LZ4_compress_fast_continue(st, s.ctypes.data + o, d.ctypes.data, k, k - 1, 1))
                else:
                    r = int(self.lib.LZ4_compress_fast(s.ctypes.data + o, d.ctypes.data, k, k - 1, 1))
                out.append((data[o:o + k], True) if r <= 0 else (d[:r].tobytes(), False))
        finally:
            if st is not None:
                self.lib.LZ4_freeStream(st)
        return out

    def assemble(self, data: bytes, bs: int, flags: int) -> bytes:
        parts = [self.header(len(data), bs, flags)]
        for body, raw in self.blocks(data, bs, flags):
            parts.append(struct.pack("<I", len(body) | (0x80000000 if raw else 0)) + body)
            if flags & BLOCK_CHECKSUM:
                parts.append(struct.pack("<I", self.ref.xxh32(body)))
        parts.append(b"\0\0\0\0")
        if flags & CONTENT_CHECKSUM:
            parts.append(struct.pack("<I", self.ref.xxh32(data)))
        return b"".join(parts)


@functools.lru_cache(maxsize=1)
def pools(seed: int = 5):
    """Compressible (datagen 0.63) and random byte pools of 10 MiB."""
    import oracle
    rng = np.random.default_rng(seed)
    text = oracle.Port().datagen(10 << 20, 0.63, 0.0, seed).tobytes()
    noise = rng.integers(0, 256, 10 << 20, dtype=np.uint8).tobytes()
    return text, noise


def content(kind: str, n: int, at: int, bs: int = 1 << 16) -> bytes:
    """n bytes of `kind`: "text" (datagen 0.63), "random", "zeros" (highly compressible) or "mixed" (text, random
    and text again in bs-byte stretches, so that a linked frame stores a block raw mid-stream)."""
    text, noise = pools()
    at %= 1 << 20
    if kind == "text":
        return text[at:at + n]
    if kind == "random":
        return noise[at:at + n]
    if kind == "zeros":
        return bytes(n)
    out = bytearray()
    while len(out) < n:
        src = noise if (len(out) // bs) % 3 == 1 else text
        out += src[at + len(out):at + len(out) + min(bs, n - len(out))]
    return bytes(out)


@functools.lru_cache(maxsize=1)
def grid():
    """The seeded case grid: (content, block size, flags, kind).

    * every block size x mode x content size on/off x the four checksum pairs, at SMALL_SIZES;
    * every block size x mode x content size on/off at every block size <= it, - 1, + 1 (and the block size itself),
      the checksum pair rotating;
    * every block size x mode: a frame of two blocks and a third, whose middle block is random, so that a linked
      frame stores it raw between compressed blocks."""
    cases = []
    kinds = ["text", "random", "zeros"]
    j = 0
    for bs in BLOCK_SIZES:
        for linked in (True, False):
            for cs in (False, True):
                for bc, cc in CHECKSUMS:
                    fl = flags_of(linked, bc, cc, cs)
                    for n in SMALL_SIZES:
                        kind = kinds[j % 3]
                        cases.append((content(kind, n, j * 4099), bs, fl, kind))
                        j += 1
                edges = sorted({s + d for s in BLOCK_SIZES if s <= bs for d in (-1, 1)} | {bs})
                for e, n in enumerate(edges):
                    bc, cc = CHECKSUMS[(j + e) % 4]
                    kind = "text" if e % 2 else "random"
                    cases.append((content(kind, n, j * 7919), bs, flags_of(linked, bc, cc, cs), kind))
                j += 1
            bc, cc = CHECKSUMS[j % 4]
            n = 2 * bs + bs // 3
            cases.append((content("mixed", n, j * 131, bs), bs, flags_of(linked, bc, cc, j % 2 == 0), "mixed"))
            j += 1
    return cases


def groups():
    """The grid by (block size, flags): one batched call each -> {(bs, flags): [content, ...]}."""
    out = {}
    for data, bs, fl, _ in grid():
        out.setdefault((bs, fl), []).append(data)
    return out
