"""Chained (linked) LZ4 block ENCODING: test infrastructure.

* ``EncUpstream`` extends tests/chain_ref.Upstream by LZ4_saveDict and a ctypes view of LZ4_stream_t_internal
  (orig/lib/lz4.h:596-603), so that a test can read upstream's state after a call and plant any state before
  one.  ``step`` is the oracle of k4lz4_encode_chain_batch for one block: upstream's
  LZ4_compress_fast_continue on a planted state whose dictionary is the min(state.dictSize, prefixLen) bytes
  directly in front of the source (what LZ4_saveDict leaves behind).
* ``RingModel`` is LZ4EncoderBase.cs:27-97 + LZ4FastChainEncoder.cs restated over upstream on a real ring
  buffer: Topup / Encode / Commit with CopyDict = LZ4_saveDict.
* ``frame_linked_ref`` restates the reference's frame writer (LZ4FrameWriter.cs:57-189) with linked blocks over
  upstream's chained encoder.
"""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np

from tests import chain_ref as CR

STATE_BYTES = 16400
K64 = 65536


class _StreamInternal(C.Structure):          # LZ4_stream_t_internal (orig/lib/lz4.h:596-603)
    _fields_ = [("hashTable", C.c_uint32 * 4096), ("currentOffset", C.c_uint32), ("tableType", C.c_uint32),
                ("dictionary", C.c_void_p), ("dictCtx", C.c_void_p), ("dictSize", C.c_uint32)]


def make_state(table=None, current_offset: int = 0, dict_size: int = 0) -> np.ndarray:
    """A K4LZ4_CHAIN_STATE_BYTES record."""
    s = np.zeros(STATE_BYTES // 4, dtype=np.uint32)
    if table is not None:
        s[:4096] = table
    s[4096], s[4097] = current_offset, dict_size
    return s.view(np.uint8)


class EncUpstream(CR.Upstream):
    def __init__(self):
        super().__init__()
        L = self.lib
        L.LZ4_saveDict.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.LZ4_saveDict.restype = C.c_int

    def view(self, st) -> _StreamInternal:
        return _StreamInternal.from_address(st)

    def state_of(self, st) -> np.ndarray:
        """Upstream's stream as a K4LZ4_CHAIN_STATE_BYTES record."""
        v = self.view(st)
        return make_state(np.ctypeslib.as_array(v.hashTable), v.currentOffset, v.dictSize)

    def compress(self, st, ptr: int, n: int, cap: int) -> tuple[int, bytes]:
        d = np.zeros(max(cap, 1) + 16, dtype=np.uint8)
        r = int(self.lib.LZ4_compress_fast_continue(st, ptr, d.ctypes.data, n, cap, 1))
        return r, d[:max(r, 0)].tobytes()

    def step(self, state: np.ndarray, history: bytes, src: bytes, cap: int):
        """-> (engine result, bytes, state after) of one chained block: `state` planted, its dictionary the
        min(dictSize, len(history)) bytes in front of `src`."""
        P, n = len(history), len(src)
        buf = np.zeros(P + n + 16, dtype=np.uint8)
        buf[:P] = np.frombuffer(history, dtype=np.uint8)
        buf[P:P + n] = np.frombuffer(src, dtype=np.uint8)
        s32 = state.view(np.uint32)
        st = self.lib.LZ4_createStream()
        try:
            v = self.view(st)
            np.ctypeslib.as_array(v.hashTable)[:] = s32[:4096]
            v.currentOffset = int(s32[4096])
            v.tableType = 2                                # byU32
            d = min(int(s32[4097]), P)
            v.dictSize = d
            v.dictionary = buf.ctypes.data + P - d
            v.dictCtx = None
            r, out = self.compress(st, buf.ctypes.data + P, n, cap)
            after = self.state_of(st)
        finally:
            self.lib.LZ4_freeStream(st)
        after.view(np.uint32)[4098:] = s32[4098:]
        return r, out, after


class RingModel:
    """LZ4FastChainEncoder over upstream on a real ring buffer (LZ4EncoderBase.cs:27-97).  `prefix` is what the
    GPU call is given: the bytes in front of the block in the ring (_inputIndex)."""

    def __init__(self, up: EncUpstream, block_size: int, extra: int = 0):
        self.up = up
        self.block = (max(block_size, 1024) + 1023) // 1024 * 1024
        self.in_len = K64 + (1 + max(extra, 0)) * self.block + 32
        self.buf = np.zeros(self.in_len + 8, dtype=np.uint8)
        self.index = self.pointer = 0
        self.st = up.lib.LZ4_createStream()

    def close(self):
        self.up.lib.LZ4_freeStream(self.st)

    def topup(self, src: bytes) -> int:
        left = self.index + self.block - self.pointer
        if not src or left <= 0:
            return 0
        k = min(left, len(src))
        self.buf[self.pointer:self.pointer + k] = np.frombuffer(src[:k], dtype=np.uint8)
        self.pointer += k
        return k

    def encode(self, cap: int, allow_copy: bool):
        """-> (Encode's result, stored bytes, prefix passed, upstream's state before and right after the call)."""
        n = self.pointer - self.index
        if n <= 0:
            return 0, b"", 0, None, None
        before = self.up.state_of(self.st)
        P = self.index
        r, out = self.up.compress(self.st, self.buf.ctypes.data + self.index, n, cap)
        after = self.up.state_of(self.st)
        if r <= 0:
            raise RuntimeError("Failed to encode chunk. Target buffer too small.")
        if allow_copy and r >= n:
            out, r = self.buf[self.index:self.pointer].tobytes(), -n
        self.index = self.pointer                          # Commit
        if self.index + self.block > self.in_len:
            k = int(self.up.lib.LZ4_saveDict(self.st, self.buf.ctypes.data, self.pointer))
            self.index = self.pointer = k
        return r, out, P, before, after


def frame_linked_ref(up: EncUpstream, data: bytes, block_size: int, block_checksum: bool,
                     content_checksum: bool) -> bytes:
    """LZ4FrameWriter with Chaining = true (FLG bit 5 clear), its encoder's blocks from upstream's
    LZ4_compress_fast_continue over the contiguous content with capacity MaximumOutputSize(blockSize); a block
    that does not shrink is stored raw (bit 31 of the length code)."""
    import oracle
    ref = oracle.Ref()
    code = {1 << 16: 4, 1 << 18: 5, 1 << 20: 6, 1 << 22: 7}[block_size]
    flg = (1 << 6) | (int(block_checksum) << 4) | (int(content_checksum) << 2)
    head = struct.pack("<IBB", 0x184D2204, flg, code << 4)
    out = [head, bytes([(ref.xxh32(head[4:6]) >> 8) & 0xFF])]
    src = np.frombuffer(data, dtype=np.uint8) if data else np.zeros(1, dtype=np.uint8)
    cap = block_size + block_size // 255 + 16
    st = up.lib.LZ4_createStream()
    try:
        for o in range(0, len(data), block_size):
            n = min(block_size, len(data) - o)
            r, enc = up.compress(st, src.ctypes.data + o, n, cap)
            assert r > 0
            body = data[o:o + n] if r >= n else enc
            out.append(struct.pack("<I", len(body) | (0x80000000 if r >= n else 0)))
            out.append(body)
            if block_checksum:
                out.append(struct.pack("<I", ref.xxh32(body)))
    finally:
        up.lib.LZ4_freeStream(st)
    out.append(struct.pack("<I", 0))
    if content_checksum:
        out.append(struct.pack("<I", ref.xxh32(data)))
    return b"".join(out)
