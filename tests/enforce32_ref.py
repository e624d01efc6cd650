"""The 32-bit engine (LZ4Codec.Enforce32, LL32): test infrastructure.

* ``REF32_SO`` is oracle/_ref/libk4ref32.so: upstream's orig/lib/lz4.c with the hash5 branch of
  LZ4_hashPosition turned off (oracle/ref32.mk), so its u32 table hashes 4 bytes as LL32.tools.cs:143-150
  does.  Apart from that hash LL32's text is LL64's, so this build is the reference's 32-bit engine.
* ``EncUpstream32`` is tests/chain_enc_ref.EncUpstream over that build: ``step`` is the oracle of
  k4lz4_encode_chain_batch_x32 for one block on a planted state.
* ``pickle`` / ``pickle_writer`` restate LZ4Pickler.Pickle and Pickle<TBufferWriter>
  (LZ4Pickler.pickle.cs:51-148) over the C restatement's LZ4Codec.Encode with enforce32, as the oracle's
  k4o_pickle / k4o_pickle_writer do with it off.
* ``frame_ref`` restates LZ4FrameWriter (LZ4FrameWriter.cs:57-189) for both block modes over the 32-bit engine:
  linked blocks from EncUpstream32, independent blocks from the restatement's LZ4Codec.Encode with enforce32.
"""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np

from tests import chain_enc_ref as ER

REF32_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                        "libk4ref32.so")
LIMIT_64K = 65547                      # LZ4_64Klimit: the first length the u32 table (and so the hash) decides


def have_ref32() -> bool:
    return os.path.exists(REF32_SO)


class EncUpstream32(ER.EncUpstream):
    """EncUpstream with upstream's streaming encoder as the 32-bit engine."""

    def __init__(self):
        self.lib = L = C.CDLL(REF32_SO)
        vp, i32 = C.c_void_p, C.c_int
        L.LZ4_createStream.restype = vp
        L.LZ4_freeStream.argtypes = [vp]
        L.LZ4_compress_fast_continue.argtypes = [vp, vp, vp, i32, i32, i32]
        L.LZ4_compress_fast_continue.restype = i32
        L.LZ4_saveDict.argtypes = [vp, vp, i32]
        L.LZ4_saveDict.restype = i32
        L.LZ4_compress_fast.argtypes = [vp, vp, i32, i32, i32]
        L.LZ4_compress_fast.restype = i32

    def compress_fast(self, src: bytes, cap: int) -> tuple[int, bytes]:
        """LZ4_compress_fast(src, dst, n, cap, 1): the engine's value and bytes."""
        s = np.frombuffer(src or b"\0", dtype=np.uint8)
        d = np.zeros(max(cap, 1) + 16, dtype=np.uint8)
        r = int(self.lib.LZ4_compress_fast(s.ctypes.data, d.ctypes.data, len(src), cap, 1))
        return r, d[:max(r, 0)].tobytes()


def _diff_width(v: int) -> int:                               # EffectiveSizeOf, LZ4Pickler.pickle.cs:224-225
    return 4 if (v > 0xFFFF or v < 0) else (2 if v > 0xFF else 1)


def _header(k: int, diff: int) -> bytes:                      # :221-228
    return bytes([((3 if k == 4 else k) & 3) << 6]) + diff.to_bytes(4, "little")[:k]


def pickle(port, src: bytes) -> bytes:
    """LZ4Pickler.Pickle under Enforce32 (pickle.cs:51-106): scratch capacity 1024 if n <= 1024 else n."""
    n = len(src)
    if n == 0:
        return b""
    enc, body = port.encode(src, 1024 if n <= 1024 else n, 0, enforce32=True)
    if enc <= 0 or enc >= n:
        return b"\0" + src
    k = _diff_width(n - enc)
    return _header(k, n - enc) + body


def pickle_writer(port, src: bytes) -> bytes:
    """LZ4Pickler.Pickle<TBufferWriter> under Enforce32 (pickle.cs:113-148): header width from n, capacity n."""
    n = len(src)
    if n == 0:
        return b""
    enc, body = port.encode(src, n, 0, enforce32=True)
    if enc <= 0 or enc >= n:
        return b"\0" + src
    return _header(_diff_width(n), n - enc) + body


def frame_ref(up32: EncUpstream32, port, xxh32, data: bytes, block_size: int, linked: bool, block_checksum: bool,
              content_checksum: bool) -> bytes:
    """LZ4FrameWriter under Enforce32: header (BD of block_size), blocks of B = block_size rounded as
    LZ4EncoderBase.cs:29 does, each encoded with capacity MaximumOutputSize(B) and stored raw when it does not
    shrink, the end mark and the checksums."""
    B = max(1024, (block_size + 1023) // 1024 * 1024)
    code = 4 if block_size <= 1 << 16 else 5 if block_size <= 1 << 18 else 6 if block_size <= 1 << 20 else 7
    flg = (1 << 6) | (0 if linked else 1 << 5) | (int(block_checksum) << 4) | (int(content_checksum) << 2)
    head = struct.pack("<IBB", 0x184D2204, flg, code << 4)
    out = [head, bytes([(xxh32(head[4:6]) >> 8) & 0xFF])]
    src = np.frombuffer(data or b"\0", dtype=np.uint8)
    cap = B + B // 255 + 16
    st = up32.lib.LZ4_createStream()
    try:
        for o in range(0, len(data), B):
            n = min(B, len(data) - o)
            if linked:
                r, enc = up32.compress(st, src.ctypes.data + o, n, cap)
            else:
                r, enc = port.encode(data[o:o + n], cap, 0, enforce32=True)
            assert r > 0
            body = data[o:o + n] if r >= n else enc
            out.append(struct.pack("<I", len(body) | (0x80000000 if r >= n else 0)))
            out.append(body)
            if block_checksum:
                out.append(struct.pack("<I", xxh32(body)))
    finally:
        up32.lib.LZ4_freeStream(st)
    out.append(struct.pack("<I", 0))
    if content_checksum:
        out.append(struct.pack("<I", xxh32(data)))
    return b"".join(out)


def hash4(b4: bytes) -> int:
    """hash4 at 12 bits (LL.tools.cs:46-58 with the u32 table's log)."""
    return ((int.from_bytes(b4[:4], "little") * 2654435761) & 0xFFFFFFFF) >> 20
