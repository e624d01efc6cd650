"""LZ4 frames against a dictionary: test infrastructure for k4lz4_frame_encode_dict_batch / _decode_dict_batch /
k4lz4_frame_info_batch.

* ``FrameDictUpstream.cdict_frame`` is upstream's own writer (oracle/_ref/libk4ref.so, lz4frame.c):
  LZ4F_createCDict(dictionary), LZ4F_compressBegin_usingCDict, LZ4F_compressUpdate of the content (in one update, or
  in the given chunks with autoFlush, which gives short non-final blocks), LZ4F_compressEnd.
* ``FrameDictUpstream.assemble`` writes the same frame by hand over upstream's block calls: LZ4_loadDict of the
  dictionary's last 64 KiB, then LZ4_compress_fast_continue per block with capacity n - 1, stored raw when that
  fails; independent blocks load the dictionary afresh, linked blocks share one stream.
* ``decode`` is LZ4F_decompress_usingDict, ``frame_info`` LZ4F_getFrameInfo, ``attach_encode`` one block through
  LZ4_attach_dictionary (the dictCtx mode upstream's CDict frames use for blocks of <= 4 KiB).
"""
from __future__ import annotations

import ctypes as C
import functools
import struct

import numpy as np

from tests import chain_ref as CR
from tests import dict_enc_ref as DR

MAGIC = 0x184D2204
SIZES = {1 << 16: 4, 1 << 18: 5, 1 << 20: 6, 1 << 22: 7}


def _err(r: int) -> bool:
    return r > (1 << 63)                      # LZ4F_isError: (size_t)-code


class FrameDictUpstream(DR.DictUpstream):
    def __init__(self):
        super().__init__()
        import oracle
        self.ref = oracle.Ref()
        L, vp, sz = self.lib, C.c_void_p, C.c_size_t
        L.LZ4F_createCDict.argtypes = [vp, sz]
        L.LZ4F_createCDict.restype = vp
        L.LZ4F_freeCDict.argtypes = [vp]
        L.LZ4F_createCompressionContext.argtypes = [C.POINTER(vp), C.c_uint]
        L.LZ4F_freeCompressionContext.argtypes = [vp]
        L.LZ4F_compressBegin_usingCDict.argtypes = [vp, vp, sz, vp, C.POINTER(CR._Prefs)]
        L.LZ4F_compressBegin_usingCDict.restype = sz
        L.LZ4F_compressUpdate.argtypes = [vp, vp, sz, vp, sz, vp]
        L.LZ4F_compressUpdate.restype = sz
        L.LZ4F_compressEnd.argtypes = [vp, vp, sz, vp]
        L.LZ4F_compressEnd.restype = sz
        L.LZ4F_createDecompressionContext.argtypes = [C.POINTER(vp), C.c_uint]
        L.LZ4F_freeDecompressionContext.argtypes = [vp]
        L.LZ4F_decompress_usingDict.argtypes = [vp, vp, C.POINTER(sz), vp, C.POINTER(sz), vp, sz, vp]
        L.LZ4F_decompress_usingDict.restype = sz
        L.LZ4F_getFrameInfo.argtypes = [vp, C.POINTER(CR._FrameInfo), vp, C.POINTER(sz)]
        L.LZ4F_getFrameInfo.restype = sz
        L.LZ4_attach_dictionary.argtypes = [vp, vp]
        L.LZ4_resetStream_fast.argtypes = [vp]

    def cdict_frame(self, data: bytes, dictionary: bytes, block_size: int = 65536, linked: bool = True,
                    block_checksum: bool = False, content_checksum: bool = False, dict_id: int = 0,
                    chunks=None, content_size: bool = False) -> bytes:
        """Upstream's CDict frame at level 0; `chunks` (sizes): one compressUpdate each, with autoFlush."""
        pr = CR._Prefs()
        pr.frameInfo.blockSizeID = SIZES[block_size]
        pr.frameInfo.blockMode = 0 if linked else 1
        pr.frameInfo.contentChecksumFlag = int(content_checksum)
        pr.frameInfo.blockChecksumFlag = int(block_checksum)
        pr.frameInfo.dictID = dict_id
        pr.frameInfo.contentSize = len(data) if content_size else 0
        pr.autoFlush = 1 if chunks is not None else 0
        L = self.lib
        dic = np.frombuffer(bytes(dictionary) + b"\0", dtype=np.uint8)
        src = np.frombuffer(bytes(data) + b"\0", dtype=np.uint8)
        cap = len(data) + (len(data) // 1024 + 8) * 64 + (4 << 20)
        dst = np.zeros(cap, dtype=np.uint8)
        cd = L.LZ4F_createCDict(dic.ctypes.data, len(dictionary))
        cx = C.c_void_p()
        assert L.LZ4F_createCompressionContext(C.byref(cx), 100) == 0
        try:
            q = L.LZ4F_compressBegin_usingCDict(cx, dst.ctypes.data, cap, cd, C.byref(pr))
            assert not _err(q)
            at = 0
            for k in (chunks if chunks is not None else [len(data)]):
                r = L.LZ4F_compressUpdate(cx, dst.ctypes.data + q, cap - q, src.ctypes.data + at, k, None)
                assert not _err(r)
                q, at = q + r, at + k
            assert at == len(data)
            r = L.LZ4F_compressEnd(cx, dst.ctypes.data + q, cap - q, None)
            assert not _err(r)
            return dst[:q + r].tobytes()
        finally:
            L.LZ4F_freeCompressionContext(cx)
            L.LZ4F_freeCDict(cd)

    def assemble(self, data: bytes, dictionary: bytes, block_size: int = 65536, linked: bool = True,
                 block_checksum: bool = False, content_checksum: bool = False, dict_id: int = 0) -> bytes:
        """The per-block assembly of a CDict frame over upstream's block calls."""
        L = self.lib
        flg = 0x40 | (0 if linked else 0x20) | (int(block_checksum) << 4) | (int(content_checksum) << 2)
        desc = struct.pack("<BB", flg | (1 if dict_id else 0), SIZES[block_size] << 4)
        if dict_id:
            desc += struct.pack("<I", dict_id)
        out = [struct.pack("<I", MAGIC), desc, bytes([(self.ref.xxh32(desc) >> 8) & 0xFF])]
        tail = bytes(dictionary[-65536:])
        dic = np.frombuffer(tail + b"\0", dtype=np.uint8)
        src = np.frombuffer(bytes(data) + b"\0" * 8, dtype=np.uint8)
        st = L.LZ4_createStream()
        try:
            L.LZ4_loadDict(st, dic.ctypes.data, len(tail))
            for o in range(0, len(data), block_size):
                n = min(block_size, len(data) - o)
                if not linked and o:
                    L.LZ4_loadDict(st, dic.ctypes.data, len(tail))
                r, enc = self.compress(st, src.ctypes.data + o, n, n - 1)
                body = enc if r > 0 else bytes(data[o:o + n])
                out.append(struct.pack("<I", len(body) | (0 if r > 0 else 0x80000000)))
                out.append(body)
                if block_checksum:
                    out.append(struct.pack("<I", self.ref.xxh32(body)))
        finally:
            L.LZ4_freeStream(st)
        out.append(struct.pack("<I", 0))
        if content_checksum:
            out.append(struct.pack("<I", self.ref.xxh32(bytes(data))))
        return b"".join(out)

    def decode_frame(self, frame: bytes, dictionary: bytes, n: int):
        """LZ4F_decompress_usingDict over a whole frame -> content, or None on an error."""
        L = self.lib
        dx = C.c_void_p()
        assert L.LZ4F_createDecompressionContext(C.byref(dx), 100) == 0
        dic = np.frombuffer(bytes(dictionary) + b"\0", dtype=np.uint8)
        src = np.frombuffer(bytes(frame) + b"\0", dtype=np.uint8)
        dst = np.zeros(n + 16, dtype=np.uint8)
        ip = op = 0
        try:
            while True:
                ds, ss = C.c_size_t(n + 16 - op), C.c_size_t(len(frame) - ip)
                r = L.LZ4F_decompress_usingDict(dx, dst.ctypes.data + op, C.byref(ds), src.ctypes.data + ip,
                                                C.byref(ss), dic.ctypes.data, len(dictionary), None)
                if _err(r):
                    return None
                ip, op = ip + ss.value, op + ds.value
                if r == 0:
                    return dst[:op].tobytes()
                if ss.value == 0 and ds.value == 0:
                    return None
        finally:
            L.LZ4F_freeDecompressionContext(dx)

    def frame_info(self, frame: bytes):
        """LZ4F_getFrameInfo -> (dictID, contentSize), or None on an error."""
        L = self.lib
        dx = C.c_void_p()
        assert L.LZ4F_createDecompressionContext(C.byref(dx), 100) == 0
        src = np.frombuffer(bytes(frame) + b"\0", dtype=np.uint8)
        fi = CR._FrameInfo()
        ss = C.c_size_t(len(frame))
        try:
            r = L.LZ4F_getFrameInfo(dx, C.byref(fi), src.ctypes.data, C.byref(ss))
            return None if _err(r) else (int(fi.dictID), int(fi.contentSize))
        finally:
            L.LZ4F_freeDecompressionContext(dx)

    def attach_encode(self, src: bytes, dictionary: bytes, cap: int, working=None) -> tuple[int, bytes]:
        """One block through LZ4_attach_dictionary (dictCtx) of a stream LZ4_loadDict filled; `working` may be a
        reused stream (LZ4_resetStream_fast first, as lz4frame does)."""
        L = self.lib
        dic = np.frombuffer(bytes(dictionary) + b"\0", dtype=np.uint8)
        s = np.frombuffer(bytes(src) + b"\0" * 8, dtype=np.uint8)
        ds = L.LZ4_createStream()
        ws = working if working is not None else L.LZ4_createStream()
        try:
            L.LZ4_loadDict(ds, dic.ctypes.data, len(dictionary))
            L.LZ4_resetStream_fast(ws)
            L.LZ4_attach_dictionary(ws, ds)
            return self.compress(ws, s.ctypes.data, len(src), cap)
        finally:
            if working is None:
                L.LZ4_freeStream(ws)
            L.LZ4_freeStream(ds)


@functools.lru_cache(maxsize=1)
def _pool() -> bytes:
    return DR.records(4 << 20, 4242)


def content(rng, n: int, dictionary: bytes, noise: int = 0) -> bytes:
    """Seeded records (random slices of one pool of them) with slices of the dictionary; `noise` incompressible
    stretches of up to 70 000 bytes (they become raw blocks)."""
    pool, parts, got = _pool(), [], 0
    while got < n:
        k = min(n - got, int(rng.integers(4096, 65537)))
        at = int(rng.integers(0, len(pool) - k))
        parts.append(pool[at:at + k])
        got += k
    base = bytearray(b"".join(parts))
    if len(dictionary) >= 64:
        for _ in range(n // 400):
            k = int(rng.integers(8, 64))
            at, fr = int(rng.integers(0, max(n - k, 1))), int(rng.integers(0, len(dictionary) - k))
            base[at:at + k] = dictionary[fr:fr + k]
    for _ in range(noise if n > 1000 else 0):
        k = min(n, int(rng.integers(1000, 70001)))
        at = int(rng.integers(0, n - k + 1))
        base[at:at + k] = rng.integers(0, 256, k, dtype=np.uint8).tobytes()
    return bytes(base[:n])


def dictionary(rng, n: int) -> bytes:
    return DR.records(n, int(rng.integers(1, 1 << 30)))


DICT_SIZES = [0, 1, 7, 8, 65535, 65536, 100000]
BLOCK_SIZES = [1 << 16, 1 << 18, 1 << 20, 1 << 22]
CONTENT_SIZES = [0, 1, 4096, 4097, 65536, 3 << 20]


@functools.lru_cache(maxsize=1)
def grid(seed: int = 11):
    """The seeded case grid: (content, dictionary, block size, linked, block checksum, content checksum, ID).

    * every dictionary size x block size x mode, the content size from CONTENT_SIZES by (dictionary, block size), the
      same for both modes (several MiB become 300 000 bytes at 64 KiB blocks);
    * every dictionary size x block size: a linked frame of 2 blocks and a part, so that block 0's state goes on to
      the chained steps;
    * linked frames whose block 0 is incompressible (stored raw: its table stops where the search did) followed by
      compressible blocks, at every block size."""
    rng = np.random.default_rng(seed)
    dicts = {d: dictionary(rng, d) for d in DICT_SIZES}
    cases, j = [], 0
    ids = [0, 7, 0xDEADBEEF]
    for k, (d, bs) in enumerate((d, bs) for d in DICT_SIZES for bs in BLOCK_SIZES):
        n = CONTENT_SIZES[k % len(CONTENT_SIZES)]
        if n == 3 << 20 and bs == 1 << 16:
            n = 300000
        data = content(rng, n, dicts[d], noise=2 if k % 3 == 0 else 0)
        for linked in (True, False):
            cases.append((data, dicts[d], bs, linked, j % 2 == 0, j % 4 < 2, ids[j % 3]))
            j += 1
        more = 2 * bs + min(bs // 3, 300000)
        cases.append((content(rng, more, dicts[d], noise=1 if k % 2 else 0), dicts[d], bs, True, j % 2 == 0,
                      j % 4 < 2, ids[j % 3]))
        j += 1
    for d, bs in ((65536, 1 << 16), (7, 1 << 16), (100000, 1 << 18), (8, 1 << 20), (65535, 1 << 22)):
        data = rng.integers(0, 256, bs, dtype=np.uint8).tobytes() + content(rng, bs + 70000, dicts[d])
        cases.append((data, dicts[d], bs, True, j % 2 == 0, True, ids[j % 3]))
        j += 1
    return cases


R_CORRUPT = -1000
_TRUNC, _SUM, _RAW, _BLOCK = 0, 1, 2, 3


def frame_verdicts(up, f: bytes, dictionary: bytes):
    """What k4lz4_frame_info_batch and k4lz4_frame_decode_dict_batch give for frame f against `dictionary`, restated
    over upstream's block decoder: -> (info result, decode result with dstCap >= the sum of the block sizes, content
    or None, that sum).  The first
    problem in stream order decides (key = block index, then kind: cut off, checksum, stored block too large, block
    rejected); a header problem decides before any block."""
    from tests.test_frame_model import walk
    L = len(f)
    if L < 7 or struct.unpack_from("<I", f, 0)[0] != MAGIC or ((f[4] >> 6) & 0x11) != 1:
        return R_CORRUPT, R_CORRUPT, None, 0
    flg, bd = f[4], f[5]
    p = 6 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)
    if L < p + 1 or ((up.ref.xxh32(f[4:p]) >> 8) & 0xFF) != f[p]:
        return R_CORRUPT, R_CORRUPT, None, 0
    p += 1
    maxb = {4: 1 << 16, 5: 1 << 18, 6: 1 << 20, 7: 1 << 22}.get((bd >> 4) & 7, 1 << 16)
    linked, bc, cc = not (flg >> 5) & 1, bool((flg >> 4) & 1), bool((flg >> 2) & 1)
    blocks, done, expect = [], False, None
    while p + 4 <= L:
        code = struct.unpack_from("<I", f, p)[0]
        p += 4
        if code == 0:
            done = True
            break
        n = code & 0x7FFFFFFF
        if p + n + (4 if bc else 0) > L:
            break
        blocks.append((f[p:p + n], bool(code >> 31), struct.unpack_from("<I", f, p + n)[0] if bc else None))
        p += n + (4 if bc else 0)
    if done and cc:
        if p + 4 > L:
            done = False
        else:
            expect = struct.unpack_from("<I", f, p)[0]
    cap = maxb if linked else maxb + 8
    raw_limit = max(maxb, 65536) if linked else maxb + 8
    info_keys, keys = [], []
    if not done:
        info_keys.append((len(blocks), _TRUNC))
    total, out = 0, b""
    for k, (body, raw, s) in enumerate(blocks):
        if raw:
            if len(body) > raw_limit:
                info_keys.append((k, _RAW))
            total += len(body)
            out += body
            continue
        lb = (len(body) - 2) * 255 // 256 if len(body) > 2 else 0     # frame.cuh frame_lb: a size never below it
        w = walk(body)
        if w < 0:
            info_keys.append((k, _BLOCK))
            total += lb
            out += b"\0" * lb
            continue
        w = max(w, lb)
        total += w
        hist = (bytes(dictionary) + out)[-65536:] if linked else bytes(dictionary)[-65536:]
        r, got = up.decode(body, cap, hist)
        if r != w:
            keys.append((k, _BLOCK))
        out += got if r == w else b"\0" * w
    keys += info_keys
    keys += [(k, _SUM) for k, (body, _, s) in enumerate(blocks) if bc and up.ref.xxh32(body) != s]
    if done and cc and not keys and up.ref.xxh32(out) != expect:
        keys.append((len(blocks), _SUM))
    info = total if not info_keys else (-1 if min(info_keys)[1] == _BLOCK else R_CORRUPT)
    dec = total if not keys else (-1 if min(keys)[1] == _BLOCK else R_CORRUPT)
    return info, dec, (out if not keys else None), total
