"""How upstream's `lz4 -d` reads a whole .lz4 input, restated in Python over upstream's own calls: test infrastructure
for k4lz4_lz4f_decompress_batch.

* ``CliModel.run`` is selectDecoder / LZ4IO_decompressLZ4F / LZ4IO_decodeLegacyStream (programs/lz4io.c) on one input,
  over LZ4F_decompress_usingDict and LZ4_decompress_safe from oracle/_ref/libk4ref.so, fed as the CLI feeds them: the
  4 magic bytes first, then what LZ4F asks for, at most 64 KiB at a time, into a 64 KiB output buffer.  That makes a
  failed block report ERROR_GENERIC or ERROR_decompressionFailed as the CLI's does.  -> (content, cliError, lz4fCode,
  end): cliError is the CLI's exit code (0 on success), lz4fCode the LZ4F_errorCodes value for error 66, end the
  offset of the undecodable data reading stopped at, else the input's length.
* ``grid`` is the seeded case grid the model, the CLI and the GPU are compared on: (name, input, dictionary).
"""
from __future__ import annotations

import ctypes as C
import functools
import struct

import numpy as np

from tests import lz4f_ref as LR
from tests.frame_dict_ref import FrameDictUpstream

FRAME_MAGIC, LEGACY_MAGIC, SKIP_MAGIC = 0x184D2204, 0x184C2102, 0x184D2A50
LEGACY_BLOCK, LEGACY_BOUND = 8 << 20, 8421520
BUF = 64 << 10

# LZ4F_errorCodes the reader raises
GENERIC, MAX_BLOCK, VERSION, BLOCK_SUM, RESERVED = 1, 2, 6, 7, 8
FRAME_SIZE, DECOMPRESS, HEADER_SUM, CONTENT_SUM = 14, 16, 17, 18
CLI_ERRORS = {40, 42, 44, 52, 53, 66, 68}
LZ4F_ERRORS = {GENERIC, MAX_BLOCK, VERSION, BLOCK_SUM, RESERVED, FRAME_SIZE, DECOMPRESS, HEADER_SUM, CONTENT_SUM}


class CliModel:
    def __init__(self):
        self.up = FrameDictUpstream()
        L = self.lib = self.up.lib
        L.LZ4_decompress_safe.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.LZ4_decompress_safe.restype = C.c_int
        self.dst = np.zeros(BUF, dtype=np.uint8)
        self.legacy = np.zeros(LEGACY_BLOCK, dtype=np.uint8)

    def run(self, data: bytes, dictionary: bytes | None = None):
        L, data = self.lib, bytes(data)
        d = np.frombuffer((dictionary[-BUF:] if dictionary else b"") + b"\0", dtype=np.uint8)
        dptr, dlen = (d.ctypes.data, len(dictionary[-BUF:])) if dictionary else (None, 0)
        out, pos, first, magic_read = bytearray(), 0, True, None
        end = len(data)

        def read(k):
            nonlocal pos
            chunk = data[pos:pos + k] if pos < len(data) else b""
            pos += len(chunk)
            return chunk

        dctx = C.c_void_p()
        assert L.LZ4F_createDecompressionContext(C.byref(dctx), 100) == 0
        try:
            while True:
                if magic_read is not None:
                    magic, magic_read = magic_read, None
                else:
                    m = read(4)
                    if not m:
                        break
                    if len(m) != 4:
                        return bytes(out), 40, 0, end
                    magic = struct.unpack("<I", m)[0]
                if (magic & 0xFFFFFFF0) == SKIP_MAGIC:
                    s = read(4)
                    if len(s) != 4:
                        return bytes(out), 42, 0, end
                    pos += struct.unpack("<I", s)[0]          # fseek past the end succeeds
                elif magic == FRAME_MAGIC:
                    e = self._frame(dctx, read, out, dptr, dlen)
                    if e:
                        return bytes(out), e[0], e[1], end
                elif magic == LEGACY_MAGIC:
                    while True:
                        h = read(4)
                        if not h:
                            break
                        if len(h) != 4:
                            return bytes(out), 52, 0, end
                        n = struct.unpack("<I", h)[0]
                        if n > LEGACY_BOUND:
                            magic_read = n
                            break
                        blk = read(n)
                        if len(blk) != n:
                            return bytes(out), 52, 0, end
                        src = np.frombuffer(blk + b"\0", dtype=np.uint8)
                        r = L.LZ4_decompress_safe(src.ctypes.data, self.legacy.ctypes.data, n, LEGACY_BLOCK)
                        if r < 0:
                            return bytes(out), 53, 0, end
                        out += self.legacy[:r].tobytes()
                else:
                    if first:
                        return bytes(out), 44, 0, end
                    return bytes(out), 0, 0, min(pos, len(data)) - 4
                first = False
        finally:
            L.LZ4F_freeDecompressionContext(dctx)
        return bytes(out), 0, 0, end

    def _frame(self, dctx, read, out, dptr, dlen):
        L, sz = self.lib, C.c_size_t
        buf = np.zeros(BUF, dtype=np.uint8)
        buf[:4] = np.frombuffer(struct.pack("<I", FRAME_MAGIC), dtype=np.uint8)
        ins, outs = sz(4), sz(0)
        nxt = L.LZ4F_decompress_usingDict(dctx, self.dst.ctypes.data, C.byref(outs), buf.ctypes.data, C.byref(ins),
                                          dptr, dlen, None)
        assert nxt < (1 << 63)                                   # error 62 is unreachable
        while nxt:
            chunk = read(min(nxt, BUF))
            if not chunk:
                break
            buf[:len(chunk)] = np.frombuffer(chunk, dtype=np.uint8)
            p, decoded = 0, BUF
            while p < len(chunk) or decoded == BUF:
                rem, dec = sz(len(chunk) - p), sz(BUF)
                nxt = L.LZ4F_decompress_usingDict(dctx, self.dst.ctypes.data, C.byref(dec), buf.ctypes.data + p,
                                                  C.byref(rem), dptr, dlen, None)
                if nxt > (1 << 63):
                    return 66, (1 << 64) - nxt
                p, decoded = p + rem.value, dec.value
                out += self.dst[:decoded].tobytes()
                if not nxt:
                    break
        return (68, 0) if nxt else None


# ---- the grid ---------------------------------------------------------------------------------------------------

def _hc(desc: bytes) -> int:
    import oracle
    return (oracle.Ref().xxh32(desc) >> 8) & 0xFF


def layout(frame: bytes):
    """(header length, [(length-code offset, stored length, raw)], end-mark offset) of a well-formed frame."""
    flg = frame[4]
    p = 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)
    bc = 4 if flg & 0x10 else 0
    blocks = []
    while True:
        c = struct.unpack_from("<I", frame, p)[0]
        if c == 0:
            return 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0), blocks, p
        blocks.append((p, c & 0x7FFFFFFF, bool(c >> 31)))
        p += 4 + (c & 0x7FFFFFFF) + bc


def reheader(frame: bytes, flg=None, bd=None, size=None) -> bytes:
    """The frame with its FLG, BD or content-size field replaced and the header checksum recomputed."""
    h, _, _ = layout(frame)
    f = bytearray(frame)
    if flg is not None:
        f[4] = flg
    if bd is not None:
        f[5] = bd
    if size is not None:
        struct.pack_into("<Q", f, 6, size)
    f[h - 1] = _hc(bytes(f[4:h - 1]))
    return bytes(f)


def frame_of(blocks, bd_id=4, linked=False, bc=False, cc_of=None, size=None) -> bytes:
    """A frame built by hand from (stored bytes, raw) blocks."""
    import oracle
    ref = oracle.Ref()
    flg = 0x40 | (0 if linked else 0x20) | (0x10 if bc else 0) | (0x08 if size is not None else 0) | \
        (0x04 if cc_of is not None else 0)
    desc = bytes([flg, bd_id << 4]) + (struct.pack("<Q", size) if size is not None else b"")
    parts = [struct.pack("<I", FRAME_MAGIC), desc, bytes([_hc(desc)])]
    for body, raw in blocks:
        parts.append(struct.pack("<I", len(body) | (0x80000000 if raw else 0)) + body)
        if bc:
            parts.append(struct.pack("<I", ref.xxh32(body)))
    parts.append(b"\0\0\0\0")
    if cc_of is not None:
        parts.append(struct.pack("<I", ref.xxh32(cc_of)))
    return b"".join(parts)


def literal_block(data: bytes) -> bytes:
    """An LZ4 block of literals only."""
    n = len(data)
    if n < 15:
        return bytes([n << 4]) + data
    k, ext = n - 15, bytearray()
    while k >= 255:
        ext.append(255)
        k -= 255
    ext.append(k)
    return bytes([0xF0]) + bytes(ext) + data


def run_block(total: int) -> bytes:
    """An LZ4 block of 8 literals, one match of offset 1 and 5 last literals: `total` bytes out of a few dozen."""
    m = total - 13
    k, ext = m - 4 - 15, bytearray()
    while k >= 255:
        ext.append(255)
        k -= 255
    ext.append(k)
    return bytes([0x8F]) + b"abcdefgh" + struct.pack("<H", 1) + bytes(ext) + bytes([0x50]) + b"vwxyz"


def legacy(up, data: bytes) -> bytes:
    """What lz4 -l writes: the legacy magic, then each 8 MiB of content as a length and an LZ4 block."""
    parts = [struct.pack("<I", LEGACY_MAGIC)]
    for o in range(0, len(data), LEGACY_BLOCK):
        chunk = data[o:o + LEGACY_BLOCK]
        s = np.frombuffer(chunk + b"\0", dtype=np.uint8)
        d = np.zeros(len(chunk) + len(chunk) // 255 + 64, dtype=np.uint8)
        r = int(up.lib.LZ4_compress_fast(s.ctypes.data, d.ctypes.data, len(chunk), len(d), 1))
        assert r > 0
        parts.append(struct.pack("<I", r) + d[:r].tobytes())
    return b"".join(parts)


def skippable(k: int, size: int, payload: bytes | None = None) -> bytes:
    body = payload if payload is not None else bytes((i * 7) & 0xFF for i in range(size))
    return struct.pack("<II", SKIP_MAGIC + k, size) + body


@functools.lru_cache(maxsize=1)
def grid():
    """The seeded grid: (name, input, dictionary or None).

    * LZ4F_compressFrame frames: every block size x mode x checksum pair x content size (the two largest block sizes
      with the no- and both-checksum pairs), 1 or 2 blocks;
    * CDict frames with and without a dictID, read with and without a dictionary, and frames whose blocks are smaller
      than BD declares (as the reference's writer and autoFlush write them);
    * legacy members (one with a full 8 MiB block), skippable frames of 0, 1 and 65 536 bytes and one reaching past
      the end, the empty input;
    * concatenations of those kinds in every order, trailing garbage of 1-3 and of >= 4 bytes, garbage first;
    * mutants of every header field, of block lengths at and past maxBlockSize, of blocks, checksums and content
      sizes, truncations inside every field, and a linked frame whose match reaches into the member before it."""
    up = LR.Lz4fUpstream()
    fd = FrameDictUpstream()
    rng = np.random.default_rng(31)
    text = lambda n, at=0: LR.content("text", n, at)                                  # noqa: E731
    cases = []
    add = lambda name, data, d=None: cases.append((name, bytes(data), d))             # noqa: E731

    # LZ4F_compressFrame frames
    for bs in LR.BLOCK_SIZES:
        pairs = LR.CHECKSUMS if bs <= (1 << 18) else [(False, False), (True, True)]
        for linked in (True, False):
            for bc, cc in pairs:
                for cs in (False, True):
                    n = bs + 5000 if bs <= (1 << 20) or linked else 70000
                    fl = LR.flags_of(linked, bc, cc, cs)
                    add(f"lz4f/{bs}/{'L' if linked else 'I'}/{int(bc)}{int(cc)}/{int(cs)}",
                        up.frame(text(n, bs + n), bs, fl))
    # dictionaries, small blocks
    dic = LR.content("text", 70000, 777)
    for linked in (True, False):
        body = text(150000, 4321)
        with_id = fd.cdict_frame(body, dic, 65536, linked, True, True, dict_id=7)
        no_id = fd.cdict_frame(body, dic, 65536, linked, False, True, dict_id=0)
        add(f"dict/id/{linked}", with_id, dic)
        add(f"dict/id-nodict/{linked}", with_id)
        add(f"dict/noflag/{linked}", no_id, dic)
        add(f"dict/plain-with-dict/{linked}", up.frame(body, 1 << 16, LR.flags_of(linked, False, True, True)), dic)
        small = fd.cdict_frame(text(30000, 99), b"", 65536, linked, True, True, chunks=[1024] * 29 + [304])
        add(f"small-blocks/{linked}", small)
        add(f"small-blocks-dict/{linked}", fd.cdict_frame(text(30000, 99), dic, 262144, linked, False, True,
                                                          chunks=[4096] * 7 + [1328]), dic)
    # legacy, skippable, empty
    leg_small = legacy(up, text(5000, 5))
    leg_full = legacy(up, text(LEGACY_BLOCK, 11) + text(1000, 3))
    add("legacy/small", leg_small)
    add("legacy/full", leg_full)
    for size in (0, 1, 65536):
        add(f"skip/{size}", skippable(size % 16, size))
    add("skip/past-end", skippable(3, 1000, b"0123456789"))
    add("empty", b"")

    # concatenations
    fsmall = up.frame(text(3000, 17), 1 << 16, LR.flags_of(False, True, True, True))
    flinked = up.frame(text(200000, 23), 1 << 16, LR.flags_of(True, False, True, False))
    kinds = {"frame": fsmall, "linked": flinked, "legacy": leg_small, "skip0": skippable(0, 0),
             "skip1": skippable(5, 1)}
    for a, x in kinds.items():
        for b, y in kinds.items():
            add(f"cat/{a}+{b}", x + y)
    add("cat/legacy+legacy+frame", leg_small + leg_small + fsmall)
    add("cat/frame+skip+garbage", fsmall + skippable(1, 16) + b"garbage!garbage!")
    for g in (1, 2, 3):
        add(f"cat/frame+garbage{g}", fsmall + b"xyz"[:g])
        add(f"cat/legacy+garbage{g}", leg_small + b"xyz"[:g])
    add("cat/frame+garbage4", fsmall + b"\x01\x02\x03\x04\x05")
    add("cat/legacy+garbage4", leg_small + struct.pack("<I", LEGACY_BOUND + 1) + b"tail")
    add("cat/skip+garbage4", skippable(2, 3) + b"\xff\xff\xff\xff")
    add("cat/garbage-first", b"\x00\x01\x02\x03" + fsmall)
    add("cat/garbage-first-short", b"\x04\x22")
    add("cat/50-frames", b"".join(up.frame(text(2000 + 97 * i, i), 1 << 16, LR.flags_of(i % 2 == 0, i % 3 == 0,
                                                                                        i % 5 == 0, i % 7 == 0))
                                 for i in range(50)))

    # header mutants
    base = up.frame(text(150000, 41), 1 << 16, LR.flags_of(True, True, True, True))
    bi = up.frame(text(150000, 43), 1 << 16, LR.flags_of(False, True, True, True))
    for v in (0, 2, 3):
        add(f"mut/version{v}", reheader(base, flg=(base[4] & 0x3F) | (v << 6)))
    add("mut/flg-reserved", reheader(base, flg=base[4] | 2))
    add("mut/bd-reserved7", reheader(base, bd=base[5] | 0x80))
    add("mut/bd-low", reheader(base, bd=base[5] | 0x03))
    for i in range(4):
        add(f"mut/bd-id{i}", reheader(base, bd=i << 4))
    hc = bytearray(base)
    hc[layout(base)[0] - 1] ^= 0x5A
    add("mut/hc", hc)
    # block lengths at and past the maximum
    add("mut/stored-max", frame_of([(text(65536, 3), True)]))
    add("mut/stored-max+1", frame_of([(text(65537, 3), True)]))
    lit = literal_block(text(65536 - 260, 7))
    lit = literal_block(text(65536 - 260 - (len(lit) - 65536), 7))
    assert len(lit) == 65536, len(lit)
    add("mut/compressed-max", frame_of([(lit, False)]))
    add("mut/compressed-max+1", frame_of([(lit + b"\0", False)]))
    for j in range(0, 9):
        add(f"mut/indep-decodes-to-max+{j}", frame_of([(run_block(65536 + j), False)]))
        add(f"mut/linked-decodes-to-max+{j}", frame_of([(run_block(65536 + j), False)], linked=True))
    add("mut/indep-256k-to-max+3", frame_of([(run_block((1 << 18) + 3), False)], bd_id=5))
    # content sizes
    n = 150000
    for name, sz in (("small", n - 1), ("large", n + 1), ("zero", 0), ("huge", 1 << 40)):
        add(f"mut/content-size-{name}", reheader(base, size=sz))
        add(f"mut/content-size-{name}-indep", reheader(bi, size=sz))
    # flipped bytes and checksums
    for fr_, tag in ((base, "L"), (bi, "I"), (up.frame(text(300000, 45), 1 << 18, LR.flags_of(False, False, False,
                                                                                              False)), "I256")):
        h, blocks, endp = layout(fr_)
        bc = 4 if fr_[4] & 0x10 else 0
        for k, (p, ln, raw) in enumerate(blocks):
            for at in (p + 4 + 1, p + 4 + ln // 2, p + 4 + ln - 1):
                f = bytearray(fr_)
                f[at] ^= 0xA5
                add(f"mut/{tag}/flip-block{k}@{at - p}", f)
            if bc:
                f = bytearray(fr_)
                f[p + 4 + ln] ^= 1
                add(f"mut/{tag}/flip-bsum{k}", f)
        if fr_[4] & 0x04:
            f = bytearray(fr_)
            f[endp + 4] ^= 1
            add(f"mut/{tag}/flip-csum", f)
    # GENERIC / decompressionFailed on blocks that fail without checksums, at every block size
    for bs in LR.BLOCK_SIZES:
        fr_ = frame_of([(run_block(5000)[:-3], False)], bd_id=LR.SIZE_ID[bs])
        add(f"mut/bad-block-{bs}", fr_)
    # truncations inside every field
    h, blocks, endp = layout(base)
    p0, ln0, _ = blocks[0]
    cuts = {"magic": 2, "header": 6, "header-cs": h - 3, "blen": h + 2, "body": p0 + 4 + ln0 // 2,
            "bsum": p0 + 4 + ln0 + 2, "endmark": endp + 2, "csum": endp + 4 + 2}
    for name, at in cuts.items():
        add(f"trunc/{name}", base[:at])
        add(f"trunc/{name}-after-frame", fsmall + base[:at])
    add("trunc/legacy-length", leg_small[:4 + 2])
    add("trunc/legacy-body", leg_small[:-10])
    add("trunc/legacy-length-second", leg_small + struct.pack("<I", 100)[:3])
    add("trunc/skip-size", skippable(0, 4)[:6])
    add("trunc/skip-size-after-frame", fsmall + skippable(0, 4)[:7])
    add("mut/legacy-zero-block", leg_small + struct.pack("<I", 0))
    lb = bytearray(leg_small)
    lb[20] ^= 0xFF
    lb[len(lb) // 2] ^= 0xFF
    add("mut/legacy-flip", lb)
    # a linked frame whose first block needs the member before it
    both = text(65536 * 2, 3)
    two = up.frame(both, 1 << 16, LR.flags_of(True, False, False, False))
    _, blocks2, _ = layout(two)
    p1, l1, r1 = blocks2[1]
    cross = frame_of([(two[p1 + 4:p1 + 4 + l1], r1)], linked=True)
    add("mut/cross-member", up.frame(both[:65536], 1 << 16, LR.flags_of(True, False, False, False)) + cross)
    # random tails and cuts over multi-member inputs
    cat = fsmall + leg_small + skippable(1, 7) + flinked
    for i in range(12):
        at = int(rng.integers(1, len(cat)))
        add(f"trunc/random{i}", cat[:at])
    return cases
