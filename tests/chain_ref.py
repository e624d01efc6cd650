"""Chained (linked) LZ4 blocks: test infrastructure for prefix-mode decoding.

* ``decompress_prefix(src, cap, history)`` restates LZ4_decompress_generic in the prefix mode that
  LZ4_decompress_safe_continue reaches from LZ4ChainDecoder (LL64.dec.cs:124-467 with lowPrefix = dst - P,
  dictSize = 0; :479-498 for the three entry points, :558-592 for the dispatch).  It is the authority on
  malformed input, like the C restatement is for independent blocks.  Returns (engine result, bytes).
* ``Upstream`` drives the reference's own C engine (orig/lib/lz4.c, built into oracle/_ref/) through its
  public streaming API: LZ4_decompress_safe_continue, LZ4_compress_fast_continue, LZ4F_compressFrame with
  linked blocks.
* ``RingModel`` is LZ4ChainDecoder.cs restated over upstream's LZ4_streamDecode_t, for the bookkeeping tests.
* ``build_prefix_block`` / ``tile_route_p`` extend tests/lz4_blocks.py's builder and routing model by the
  history length P (decode_tile.cuh: accept test ``off > op + lit + P``).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from tests import lz4_blocks as LB

MINMATCH, MFLIMIT, LASTLITERALS = 4, 12, 5


# ---- restatement ---------------------------------------------------------------------------------------

def decompress_prefix(src: bytes, cap: int, history: bytes = b"") -> tuple[int, bytes]:
    """LZ4_decompress_safe (P = 0), _withSmallPrefix (P < 65535) or _withPrefix64k (P >= 65535), as
    LZ4_decompress_safe_continue picks them; `history` are the P bytes in front of dst.  -> (r, decoded);
    r < 0 is an error (the engine's own negative position is reported as -1)."""
    P = len(history)
    p64 = P >= 65535
    low = -65536 if p64 else -P                              # lowPrefix relative to dst
    n = len(src)
    if cap == 0:                                             # :162-168
        return (0 if n == 1 and src[0] == 0 else -1), b""
    if n == 0:                                               # :172
        return -1, b""
    buf = bytearray(history)                                 # buf[P + op] is output byte op
    ip, op = 0, 0
    iend, oend = n, cap
    shortiend, shortoend = iend - 16, oend - 32              # :152-153

    def copy_match(match: int, length: int) -> None:
        if match == op:                                      # offset 0: accepted, content unspecified (zeros)
            buf.extend(bytes(length))
            return
        for k in range(length):                              # overlapping copies are byte-serial
            buf.append(buf[P + match + k])

    while True:
        token = src[ip]; ip += 1
        length = token >> 4
        if length != 15 and ip < shortiend and op <= shortoend:      # :191-193
            buf += src[ip:ip + length]; op += length; ip += length
            length = token & 15
            offset = src[ip] | (src[ip + 1] << 8); ip += 2
            match = op - offset
            if length != 15 and offset >= 8 and (p64 or match >= low):   # :211-220
                copy_match(match, length + MINMATCH)
                op += length + MINMATCH
                continue
        else:
            if length == 15:                                 # LZ4_readVLE, LL.tools.cs:165-193
                if ip >= iend - 15:
                    return -1, b""
                while True:
                    s = src[ip]; ip += 1; length += s
                    if ip >= iend - 15 or s != 255:
                        break
            cpy = op + length
            if cpy > oend - MFLIMIT or ip + length > iend - (2 + 1 + LASTLITERALS):   # :247
                if ip + length != iend or cpy > oend:        # :291-294
                    return -1, b""
                buf += src[ip:ip + length]
                return op + length, bytes(buf[P:])
            buf += src[ip:ip + length]; ip += length; op = cpy
            offset = src[ip] | (src[ip + 1] << 8); ip += 2
            match = op - offset
            length = token & 15
        if length == 15:                                     # :326-334
            while True:
                s = src[ip]; ip += 1; length += s
                if ip >= iend - LASTLITERALS + 1:
                    return -1, b""
                if s != 255:
                    break
        length += MINMATCH
        if match < low:                                      # :338 (checkOffset, dictSize = 0)
            return -1, b""
        if op + length > oend - LASTLITERALS:                # :427-433
            return -1, b""
        copy_match(match, length)
        op += length


# ---- upstream ---------------------------------------------------------------------------------------------

class _FrameInfo(C.Structure):
    _fields_ = [("blockSizeID", C.c_int), ("blockMode", C.c_int), ("contentChecksumFlag", C.c_int),
                ("frameType", C.c_int), ("contentSize", C.c_ulonglong), ("dictID", C.c_uint),
                ("blockChecksumFlag", C.c_int)]


class _Prefs(C.Structure):
    _fields_ = [("frameInfo", _FrameInfo), ("compressionLevel", C.c_int), ("autoFlush", C.c_uint),
                ("favorDecSpeed", C.c_uint), ("reserved", C.c_uint * 3)]


class _StreamDecode(C.Structure):            # LZ4_streamDecode_t_internal (orig/lib/lz4.h)
    _fields_ = [("externalDict", C.c_void_p), ("extDictSize", C.c_size_t), ("prefixEnd", C.c_void_p),
                ("prefixSize", C.c_size_t)]


class Upstream:
    def __init__(self):
        import oracle
        self.lib = L = C.CDLL(oracle.REF_SO)
        vp, i32 = C.c_void_p, C.c_int
        L.LZ4_createStream.restype = vp
        L.LZ4_freeStream.argtypes = [vp]
        L.LZ4_compress_fast_continue.argtypes = [vp, vp, vp, i32, i32, i32]
        L.LZ4_compress_fast_continue.restype = i32
        L.LZ4_createStreamDecode.restype = vp
        L.LZ4_freeStreamDecode.argtypes = [vp]
        L.LZ4_setStreamDecode.argtypes = [vp, vp, i32]
        L.LZ4_setStreamDecode.restype = i32
        L.LZ4_decompress_safe_continue.argtypes = [vp, vp, vp, i32, i32]
        L.LZ4_decompress_safe_continue.restype = i32
        L.LZ4_decompress_safe_usingDict.argtypes = [vp, vp, i32, i32, vp, i32]
        L.LZ4_decompress_safe_usingDict.restype = i32
        L.LZ4F_compressFrameBound.argtypes = [C.c_size_t, C.POINTER(_Prefs)]
        L.LZ4F_compressFrameBound.restype = C.c_size_t
        L.LZ4F_compressFrame.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.POINTER(_Prefs)]
        L.LZ4F_compressFrame.restype = C.c_size_t

    def decode_prefix(self, src: bytes, cap: int, history: bytes = b"") -> tuple[int, bytes]:
        """The prefix branches of LZ4_decompress_safe_continue: usingDict with the dictionary directly in
        front of dst dispatches to exactly the same three functions (lz4.c)."""
        P = len(history)
        buf = np.zeros(P + max(cap, 1), dtype=np.uint8)
        buf[:P] = np.frombuffer(history, dtype=np.uint8)
        s = np.frombuffer(bytes(src) or b"\0", dtype=np.uint8)
        r = int(self.lib.LZ4_decompress_safe_usingDict(s.ctypes.data, buf.ctypes.data + P, len(src), cap,
                                                       buf.ctypes.data, P))
        return (r, buf[P:P + r].tobytes()) if r >= 0 else (-1, b"")

    def encode_chain(self, data: bytes, block: int = 65536) -> list[bytes]:
        """One stream of linked blocks: LZ4_compress_fast_continue over consecutive blocks of one buffer
        (the encoder keeps the previous 64 KiB as its window), acceleration 1."""
        src = np.frombuffer(data, dtype=np.uint8)
        st = self.lib.LZ4_createStream()
        out = []
        cap = block + block // 255 + 16
        dst = np.zeros(cap, dtype=np.uint8)
        try:
            for o in range(0, len(data), block):
                k = min(block, len(data) - o)
                r = int(self.lib.LZ4_compress_fast_continue(st, src.ctypes.data + o, dst.ctypes.data, k, cap, 1))
                assert r > 0
                out.append(dst[:r].tobytes())
        finally:
            self.lib.LZ4_freeStream(st)
        return out

    def frame_linked(self, data: bytes, size_id: int = 4, block_checksum: bool = False,
                     content_checksum: bool = False) -> bytes:
        """LZ4F_compressFrame with LZ4F_blockLinked (orig/lib/lz4frame.c); size_id 4..7 = 64 KiB..4 MiB."""
        pr = _Prefs()
        pr.frameInfo.blockSizeID = size_id
        pr.frameInfo.blockMode = 0                          # LZ4F_blockLinked
        pr.frameInfo.contentChecksumFlag = int(content_checksum)
        pr.frameInfo.blockChecksumFlag = int(block_checksum)
        s = np.frombuffer(data, dtype=np.uint8)
        cap = int(self.lib.LZ4F_compressFrameBound(len(data), C.byref(pr)))
        d = np.zeros(cap, dtype=np.uint8)
        r = int(self.lib.LZ4F_compressFrame(d.ctypes.data, cap, s.ctypes.data if len(data) else None, len(data),
                                            C.byref(pr)))
        assert 0 < r <= cap
        return d[:r].tobytes()


class RingModel:
    """LZ4ChainDecoder.cs:26-143 over upstream: the same ring buffer and CopyDict / ApplyDict calls, blocks
    decoded by upstream's LZ4_decompress_safe_continue into the ring."""
    K64 = 65536

    def __init__(self, up: Upstream, block_size: int, extra: int = 0):
        self.up = up
        self.block = (max(block_size, 1024) + 1023) // 1024 * 1024
        self.out_len = self.K64 + (1 + max(extra, 0)) * self.block + 32
        self.buf = np.zeros(self.out_len + 8, dtype=np.uint8)
        self.index = 0
        self.ctx = up.lib.LZ4_createStreamDecode()

    def close(self):
        self.up.lib.LZ4_freeStreamDecode(self.ctx)

    @property
    def prefix_size(self) -> int:
        return int(_StreamDecode.from_address(self.ctx).prefixSize)

    def _set(self, start: int, size: int):
        self.up.lib.LZ4_setStreamDecode(self.ctx, self.buf.ctypes.data + start, size)

    def decode(self, src: bytes, block_size: int = 0) -> int:
        bs = block_size if block_size > 0 else self.block
        if self.index + bs > self.out_len:                   # Prepare -> CopyDict
            start = max(self.index - self.K64, 0)
            size = self.index - start
            self.buf[:size] = self.buf[start:self.index].copy()
            self._set(0, size)
            self.index = size
        s = np.frombuffer(bytes(src) or b"\0", dtype=np.uint8)
        r = int(self.up.lib.LZ4_decompress_safe_continue(self.ctx, s.ctypes.data, self.buf.ctypes.data + self.index,
                                                         len(src), bs))
        if r < 0:
            raise RuntimeError("InvalidOperationException")
        self.index += r
        return r

    def _apply(self, index: int) -> int:
        start = max(index - self.K64, 0)
        self._set(start, index - start)
        return index

    def inject(self, src: bytes) -> int:
        n = len(src)
        if n <= 0:
            return 0
        if n > max(self.block, self.K64):
            raise RuntimeError("InvalidOperationException")
        a = np.frombuffer(src, dtype=np.uint8)
        if self.index + n < self.out_len:
            self.buf[self.index:self.index + n] = a
            self.index = self._apply(self.index + n)
        elif n >= self.K64:
            self.buf[:n] = a
            self.index = self._apply(n)
        else:
            tail = min(self.K64 - n, self.index)
            self.buf[:tail] = self.buf[self.index - tail:self.index].copy()
            self.buf[tail:tail + n] = a
            self.index = self._apply(tail + n)
        return n

    def peek(self, offset: int) -> bytes:
        o = self.index + offset
        if o < 0 or o > self.index:
            raise RuntimeError("InvalidOperationException")
        return self.buf[o:self.index].tobytes()


# ---- builder and routing model with a history ---------------------------------------------------------------

def build_prefix_block(history: bytes, seqs, last: bytes = b"") -> tuple[bytes, bytes]:
    """Like lz4_blocks.build_block, but matches may reach `len(history)` bytes in front of the block.
    -> (stream, decoded block bytes)."""
    out, dec = bytearray(), bytearray(history)
    P = len(history)
    for lits, off, ml in seqs:
        L, M = len(lits), ml - MINMATCH
        if M < 0 or not 1 <= off <= 65535:
            raise ValueError((off, ml))
        out.append((min(L, 15) << 4) | min(M, 15))
        if L >= 15:
            out += LB._ext(L - 15)
        out += lits
        dec += lits
        if off > len(dec):
            raise ValueError(f"offset {off} reaches before the history at {len(dec) - P}")
        out += bytes([off & 0xFF, off >> 8])
        if M >= 15:
            out += LB._ext(M - 15)
        LB._append_match(dec, off, ml)
    L = len(last)
    out.append(min(L, 15) << 4)
    if L >= 15:
        out += LB._ext(L - 15)
    out += last
    dec += last
    return bytes(out), bytes(dec[P:])


def tile_route_p(stream: bytes, cap: int, P: int, src_phase: int = 0) -> str:
    """lz4_blocks.tile_route with the history: the offset accept test of decode_tile.cuh becomes
    off > op + lit + P (P clamped to 65535); every other test is unchanged.  Returns the engine."""
    P = min(P, 65535)
    r = LB.tile_route(stream, cap, src_phase)
    if r.engine != "generic" or P == 0 or not r.why.startswith("sequence"):
        return r.engine                                      # a looser offset test cannot decline a block
    n, seqs = len(stream), LB.parse(stream)
    op, N = 0, len(seqs)
    for i, s in enumerate(seqs):
        bad = bool(s.flags & (LB.SQ_EDGE | LB.SQ_BAD))
        if i == N - 1:
            bad |= not (s.flags & LB.SQ_LAST) or op + s.lit > cap
        else:
            bad |= bool(s.flags & LB.SQ_LAST) or s.lit_pos + s.lit > n - 8 or op + s.lit > cap - MFLIMIT
            bad |= s.off == 0 or s.off > op + s.lit + P or op + s.lit + s.ml > cap - LASTLITERALS
        if bad:
            return "generic"
        op += s.lit + s.ml
    return "tile" if r.stage == "small" else "tile_big"
