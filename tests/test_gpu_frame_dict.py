"""LZ4 frames against a dictionary on the GPU (k4lz4_frame_encode_dict_batch / _decode_dict_batch /
k4lz4_frame_info_batch, LZ4Frame.*WithDictionary / Info).

Encoded frames are compared byte for byte with upstream's CDict frames (tests/frame_dict_ref.py, whose per-block
assembly test_frame_dict_model.py pins); decoded frames come from upstream's writer (with and without an ID, with
autoFlush and short non-final blocks, with a content size) and ours.  Destinations are surrounded by 0xCD
canaries.  Needs the reference engine that __graft_entry__.build() compiles into oracle/_ref/."""
import struct

import numpy as np
import pytest

from tests import dict_enc_ref as DR
from tests import frame_dict_ref as FD
from tests.test_gpu_frames import CD, GAP, layout

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return FD.FrameDictUpstream()


def _flags(linked, bc, cc):
    return (0 if linked else 1) | (2 if bc else 0) | (4 if cc else 0)


def _dicts(dictionaries):
    dic, off, at = [], [], 0
    for d in dictionaries:
        off.append(at)
        dic.append(bytes(d) + b"\xAB" * 5)            # odd phases
        at += len(d) + 5
    base = np.frombuffer(b"".join(dic) + b"\0" * 16, dtype=np.uint8).copy()
    return base, np.array(off, dtype=np.int64), np.array([len(d) for d in dictionaries], dtype=np.int32)


def run(k4, what, items, dictionaries, caps=None, ids=None, mem="device", bs=65536, flags=0, level=0, nodict=False):
    """One dictionary frame call -> (results, dst, dstOff, dstCap) or, for "info", (sizes, ids)."""
    import torch
    N = k4._native
    L = N.lib()
    src, so, sl, dst, do, dc = layout(items, caps if caps is not None else [0] * len(items))
    db, doff, dl = _dicts(dictionaries)
    n = len(items)
    idv = None if ids is None else np.array(ids, dtype=np.uint32)
    out = np.full(n, 12345, dtype=np.int32)
    oid = np.full(n, 777, dtype=np.int64)
    if mem == "host":
        if what == "encode":
            rc = L.k4lz4_frame_encode_dict_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                 do.ctypes.data, dc.ctypes.data, db.ctypes.data, doff.ctypes.data,
                                                 dl.ctypes.data, None if idv is None else idv.ctypes.data,
                                                 out.ctypes.data, n, bs, flags, level, N.MEM_HOST, None, 0)
        elif what == "decode":
            rc = L.k4lz4_frame_decode_dict_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                 do.ctypes.data, dc.ctypes.data, None if nodict else db.ctypes.data,
                                                 doff.ctypes.data, dl.ctypes.data, out.ctypes.data, n, N.MEM_HOST,
                                                 None, 0)
        else:
            rc = L.k4lz4_frame_info_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, out.ctypes.data,
                                          oid.ctypes.data, n, N.MEM_HOST, None, 0)
        N.check(rc)
        return (out, oid) if what == "info" else (out, dst, do, dc)
    dev = torch.device("cuda", 0)
    arrs = dict(src=src, so=so, sl=sl, dst=dst, do=do, dc=dc, db=db, doff=doff, dl=dl)
    t = {k: torch.from_numpy(v.copy()).to(dev) for k, v in arrs.items()}
    o = torch.from_numpy(out).to(dev)
    F = k4.LZ4Frame
    st = torch.cuda.current_stream().cuda_stream
    if what == "encode":
        ti = None if idv is None else torch.from_numpy(idv.view(np.int32).copy()).to(dev)
        F.encode_many_with_dictionary_device(t["src"], t["so"], t["sl"], t["dst"], t["do"], t["dc"], t["db"],
                                             t["doff"], t["dl"], ti, o, bs, not (flags & 1), bool(flags & 2),
                                             bool(flags & 4), level, st)
    elif what == "decode":
        F.decode_many_with_dictionary_device(t["src"], t["so"], t["sl"], t["dst"], t["do"], t["dc"],
                                             None if nodict else t["db"], t["doff"], t["dl"], o, st)
    else:
        ti = torch.from_numpy(oid).to(dev)
        F.info_device(t["src"], t["so"], t["sl"], o, ti, st)
        torch.cuda.synchronize()
        return o.cpu().numpy(), ti.cpu().numpy()
    torch.cuda.synchronize()
    return o.cpu().numpy(), t["dst"].cpu().numpy(), do, dc


def frames_of(out, dst, do, dc):
    res = []
    for i in range(len(out)):
        r = int(out[i])
        a, c = int(do[i]), int(dc[i])
        assert (dst[a - GAP:a] == CD).all() and (dst[a + c:a + c + GAP] == CD).all(), f"canary of frame {i}"
        res.append(dst[a:a + r].tobytes() if r >= 0 else None)
    return res


def bound(k4, n, bs, flags, did):
    return int(k4._native.lib().k4lz4_frame_bound(n, bs, flags)) + (4 if did else 0)


@pytest.mark.parametrize("mem", ["device", "host"])
def test_encode_equals_upstream_cdict_frames(k4, up, mem):
    cases = FD.grid()
    for bs in FD.BLOCK_SIZES:
        for linked in (True, False):
            for bc, cc in ((False, False), (True, True)):
                sub = [c for c in cases if c[2] == bs and c[3] == linked]
                if not sub:
                    continue
                fl = _flags(linked, bc, cc)
                items = [c[0] for c in sub]
                dics = [c[1] for c in sub]
                ids = [c[6] for c in sub]
                caps = [bound(k4, len(x), bs, fl, d) for x, d in zip(items, ids)]
                out, dst, do, dc = run(k4, "encode", items, dics, caps, ids, mem, bs, fl)
                got = frames_of(out, dst, do, dc)
                for g, x, d, i in zip(got, items, dics, ids):
                    assert g == up.cdict_frame(x, d, bs, linked, bc, cc, i), (len(x), len(d), bs, linked, bc, cc)


def test_many_small_frames_few_dictionaries(k4, up):
    rng = np.random.default_rng(21)
    dics = [DR.records(65536, s) for s in (1, 2, 3)] + [b"", b"abc"]
    items, ds, ids = [], [], []
    for i in range(3000):
        n = int(rng.integers(0, 4097))
        d = dics[i % len(dics)]
        items.append(FD.content(rng, n, d))
        ds.append(d)
        ids.append(i % 3)
    for linked in (True, False):
        fl = _flags(linked, False, True)
        caps = [bound(k4, len(x), 65536, fl, d) for x, d in zip(items, ids)]
        out, dst, do, dc = run(k4, "encode", items, ds, caps, ids, "host", 65536, fl)
        got = frames_of(out, dst, do, dc)
        for j in range(0, len(items), 7):
            assert got[j] == up.cdict_frame(items[j], ds[j], 65536, linked, False, True, ids[j]), j
        back, r = k4.LZ4Frame.DecodeManyWithDictionary(got, ds)
        assert back == items and (r == [len(x) for x in items]).all()


def test_more_dictionaries_than_records(k4, up):
    rng = np.random.default_rng(22)
    n = 1300                                        # > DICT_RECORDS (1 024) distinct dictionaries in one launch
    ds = [DR.records(int(rng.integers(8, 3000)), 100 + i) for i in range(n)]
    items = [FD.content(rng, int(rng.integers(1, 3000)), d) for d in ds]
    caps = [bound(k4, len(x), 65536, 1, 0) for x in items]
    out, dst, do, dc = run(k4, "encode", items, ds, caps, None, "device", 65536, 1)
    got = frames_of(out, dst, do, dc)
    for j in range(0, n, 11):
        assert got[j] == up.cdict_frame(items[j], ds[j], 65536, False), j


@pytest.mark.parametrize("linked", [True, False])
def test_dst_one_byte_short(k4, up, linked):
    rng = np.random.default_rng(23)
    d = DR.records(20000, 9)
    items = [FD.content(rng, 150000, d), FD.content(rng, 3000, d)]
    fl = _flags(linked, True, True)
    want = [up.cdict_frame(x, d, 65536, linked, True, True, 4) for x in items]
    out, dst, do, dc = run(k4, "encode", items, [d, d], [len(w) - 1 for w in want], [4, 4], "device", 65536, fl)
    assert (out == -1).all()
    frames_of(out, dst, do, dc)                        # canaries: nothing at or beyond dstCap
    out, dst, do, dc = run(k4, "encode", items, [d, d], [len(w) for w in want], [4, 4], "host", 65536, fl)
    assert frames_of(out, dst, do, dc) == want


def test_level3_delegates_and_arguments(k4):
    N = k4._native
    L = N.lib()
    out, dst, do, dc = run(k4, "encode", [b"x" * 100], [b"d" * 100], [1000], None, "host", 65536, 0, level=3)
    assert out[0] == N.R_DELEGATE and (dst == CD).all()
    out, _, _, _ = run(k4, "encode", [b"x" * 100], [b"d" * 100], [1000], None, "device", 65536, 0, level=3)
    assert out[0] == N.R_DELEGATE
    src = np.zeros(16, dtype=np.uint8)
    off = np.zeros(1, dtype=np.int64)
    ln = np.ones(1, dtype=np.int32)
    o = np.zeros(1, dtype=np.int32)
    p = src.ctypes.data
    for bs in (65535, 65537, 1024, 2 << 20, 8 << 20):
        assert L.k4lz4_frame_encode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                               p, off.ctypes.data, ln.ctypes.data, None, o.ctypes.data, 1, bs, 0, 0,
                                               N.MEM_HOST, None, 0) == N.E_ARG
    assert L.k4lz4_frame_encode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                           p, off.ctypes.data, ln.ctypes.data, None, o.ctypes.data, 1, 65536, 8, 0,
                                           N.MEM_HOST, None, 0) == N.E_ARG
    # the dictionary arrays are required for encode
    assert L.k4lz4_frame_encode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                           None, None, None, None, o.ctypes.data, 1, 65536, 0, 0,
                                           N.MEM_HOST, None, 0) == N.E_ARG
    assert L.k4lz4_frame_encode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                           p, None, ln.ctypes.data, None, o.ctypes.data, 1, 65536, 0, 0,
                                           N.MEM_HOST, None, 0) == N.E_ARG
    assert L.k4lz4_frame_encode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                           None, None, None, None, o.ctypes.data, 0, 65536, 0, 0,
                                           N.MEM_HOST, None, 0) == N.OK
    # decode: dictBase may be null, but then not half the arrays
    assert L.k4lz4_frame_decode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                           p, off.ctypes.data, None, o.ctypes.data, 1, N.MEM_HOST, None, 0) == N.E_ARG
    assert L.k4lz4_frame_decode_dict_batch(p, off.ctypes.data, ln.ctypes.data, p, off.ctypes.data, ln.ctypes.data,
                                           p, off.ctypes.data, ln.ctypes.data, o.ctypes.data, 1, 7, None, 0) == N.E_ARG
    assert L.k4lz4_frame_info_batch(p, off.ctypes.data, ln.ctypes.data, o.ctypes.data, None, 1, N.MEM_HOST, None,
                                    0) == N.E_ARG


def _upstream_corpus(up, rng):
    """Upstream frames against dictionaries: with and without an ID, autoFlush with short non-final blocks (their
    windows reach into both the dictionary and the output), a content-size field, every block size."""
    out = []
    for j, (dl, bs) in enumerate([(65536, 1 << 16), (100000, 1 << 18), (3000, 1 << 16), (0, 1 << 16), (7, 1 << 20),
                                  (65535, 1 << 22), (8, 1 << 16)]):
        d = FD.dictionary(rng, dl)
        for linked in (True, False):
            n = [0, 1, 5000, 70000, 300000, 1 << 20][j % 6]
            x = FD.content(rng, n, d, noise=1)
            out.append((up.cdict_frame(x, d, bs, linked, j % 2 == 0, True, j * 3), x, d))
            out.append((up.cdict_frame(x, d, bs, linked, False, False, 0, content_size=True), x, d))
            if n > 10:
                cuts, at = [], 0
                while at < n:
                    k = min(n - at, int(rng.integers(1, 20000)))
                    cuts.append(k)
                    at += k
                out.append((up.cdict_frame(x, d, bs, linked, True, False, 0, chunks=cuts), x, d))
    return out


@pytest.mark.parametrize("mem", ["device", "host"])
def test_decode_upstream_and_own_frames(k4, up, mem):
    rng = np.random.default_rng(31)
    corpus = _upstream_corpus(up, rng)
    for data, dic, bs, linked, bc, cc, did in FD.grid()[::3]:
        corpus.append((up.cdict_frame(data, dic, bs, linked, bc, cc, did), data, dic))
    frames = [c[0] for c in corpus]
    want = [c[1] for c in corpus]
    dics = [c[2] for c in corpus]
    sizes, ids = run(k4, "info", frames, dics, mem=mem)
    assert list(sizes) == [len(w) for w in want]
    for f, i in zip(frames, ids):
        did = up.frame_info(f)[0]
        assert i == (did if f[4] & 1 else -1)
    out, dst, do, dc = run(k4, "decode", frames, dics, [len(w) for w in want], mem=mem)
    assert list(out) == [len(w) for w in want]
    assert frames_of(out, dst, do, dc) == want


def test_info_id_field_holding_zero(k4, up):
    d = b"dictionary bytes" * 10
    f = up.assemble(b"hello hello hello", d)
    desc = bytes([f[4] | 1, f[5]]) + b"\0\0\0\0"
    hc = (up.ref.xxh32(desc) >> 8) & 0xFF
    g = f[:4] + desc + bytes([hc]) + f[7:]
    sizes, ids = k4.LZ4Frame.Info([f, g])
    assert list(sizes) == [17, 17] and list(ids) == [-1, 0]
    assert k4.LZ4Frame.DecodeWithDictionary(g, d) == b"hello hello hello"
    # the frame calls without dictionaries still delegate the flag
    assert k4.LZ4Frame.ContentSizes([g])[0] == k4._native.R_DELEGATE


def _edge_block(lit, off):
    """`lit` literals, a match of 18 at `off`, 12 last literals."""
    return bytes([(lit << 4) | 14]) + b"ABCDEFGH"[:lit] + struct.pack("<H", off) + bytes([0xC0]) + b"0123456789ab"


def _frame(blocks, linked):
    desc = bytes([0x40 | (0 if linked else 0x20), 0x40])
    import oracle
    hc = (oracle.Ref().xxh32(desc) >> 8) & 0xFF
    body = b"".join(struct.pack("<I", len(b)) + b for b in blocks)
    return struct.pack("<I", FD.MAGIC) + desc + bytes([hc]) + body + b"\0\0\0\0"


@pytest.mark.parametrize("dl", [1000, 65527, 65535, 100000])
def test_offset_reaching_dictionary_start(k4, up, dl):
    """A match reaching exactly the dictionary's first byte the decoder keeps is accepted, one byte further is -1;
    from 65 535 bytes of dictionary on, every offset reaches inside it (the tile kernel's P = 65 535 clamp)."""
    d = FD.dictionary(np.random.default_rng(dl), dl)
    lit = 8 if dl <= 65527 else 0
    n = lit + 30
    ok = _edge_block(lit, lit + min(dl, 65535 - lit))
    r, want = up.decode(ok, n, d)
    first = max(dl - 65535, 0) if lit == 0 else 0
    assert r == n and want[lit:lit + 18] == d[first:first + 18]
    assert k4.LZ4Codec.Decode(ok, bytearray(n), d) == n
    frames, caps = [_frame([ok, ok], False), _frame([ok], True)], [2 * n, n]
    bad = _edge_block(lit, lit + dl + 1) if lit + dl + 1 <= 65535 else None
    if bad is not None:
        assert up.decode(bad, n, d)[0] < 0
        assert k4.LZ4Codec.Decode(bad, bytearray(n), d) < 0
        frames += [_frame([ok, bad], False), _frame([bad], True)]
        caps += [2 * n, n]
    B = k4.batch
    B.decode_stats(0, reset=True)
    contents, out = k4.LZ4Frame.DecodeManyWithDictionary(frames, [d] * len(frames), caps)
    stats = B.decode_stats(0, reset=True)
    assert out[0] == 2 * n and contents[0] == want * 2
    assert out[1] == n and contents[1] == want
    if bad is not None:
        assert list(out[2:]) == [-1, -1]
    else:                                               # the accepted blocks stayed on the tile kernel
        assert stats["tile"] == 3 and stats["generic"] == 0, stats


def test_empty_dictionary_matches_frame_decode(k4, up):
    from tests.test_gpu_frames import content as fcontent
    rng = np.random.default_rng(41)
    from tests import chain_ref as CR
    U = CR.Upstream()
    frames = []
    for n in (0, 1, 5000, 70000, 300000):
        x = fcontent(rng, n)
        frames.append(U.frame_linked(x, 4, True, True))
        frames.append(k4.LZ4Frame.Encode(x, 65536, chaining=False, block_checksum=True))
        frames.append(k4.LZ4Frame.Encode(x, 1 << 18, chaining=True, content_checksum=True))
    # mutations: truncations, flipped bytes in headers and blocks
    muts = []
    for f in frames:
        for _ in range(6):
            g = bytearray(f)
            at = int(rng.integers(0, len(g)))
            g[at] ^= 1 << int(rng.integers(0, 8))
            muts.append(bytes(g))
        muts.append(f[:int(rng.integers(0, len(f)))])
    allf = frames + muts
    caps = [max(int(s), 0) + 64 for s in k4.LZ4Frame.ContentSizes(allf)]
    a = run(k4, "decode", allf, [b""] * len(allf), caps, nodict=True)
    b = run(k4, "decode", allf, [b""] * len(allf), caps)
    sizes = k4.LZ4Frame.ContentSizes(allf)
    N = k4._native
    L = N.lib()
    src, so, sl, dst, do, dc = layout(allf, caps)
    ref = np.zeros(len(allf), dtype=np.int32)
    N.check(L.k4lz4_frame_decode_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                       do.ctypes.data, dc.ctypes.data, ref.ctypes.data, len(allf), N.MEM_HOST, None, 0))
    for out, d2, _, _ in (a, b):
        for i in range(len(allf)):
            if ref[i] == N.R_DELEGATE:                 # a flipped dictionary flag: the dictionary call reads the ID
                assert out[i] != N.R_DELEGATE
                continue
            assert out[i] == ref[i], i
            if ref[i] >= 0:
                assert d2[do[i]:do[i] + ref[i]].tobytes() == dst[do[i]:do[i] + ref[i]].tobytes()
    info, ids = run(k4, "info", allf, [b""] * len(allf))
    for i in range(len(allf)):
        if sizes[i] != N.R_DELEGATE:
            assert info[i] == sizes[i] and ids[i] == -1, i


def test_mutated_dict_frames_follow_restatement(k4, up):
    """Every header bit, block length codes, block bodies and truncations of dictionary frames: the info call's
    sizes and the decode's verdicts and contents equal frame_dict_ref.frame_verdicts exactly."""
    rng = np.random.default_rng(43)
    d = FD.dictionary(rng, 5000)
    base = [up.cdict_frame(FD.content(rng, n, d), d, 65536, linked, True, True, 1234)
            for n in (3000, 100000) for linked in (True, False)]
    base.append(up.cdict_frame(FD.content(rng, 100000, d), d, 65536, True, False, False, 0, content_size=True))
    muts = list(base)
    for f in base:
        head = 11 + (8 if f[4] & 8 else 0) - (0 if f[4] & 1 else 4)
        for at in range(4, head + 4):                   # FLG, BD, [size], [ID], HC, the first length code
            for bit in range(8):
                g = bytearray(f)
                g[at] ^= 1 << bit
                muts.append(bytes(g))
        for _ in range(24):                             # block bodies and checksums
            g = bytearray(f)
            g[int(rng.integers(head, len(f)))] ^= 1 << int(rng.integers(0, 8))
            muts.append(bytes(g))
        muts += [f[:k] for k in (5, 8, 11, 12, 20, len(f) // 2, len(f) - 5, len(f) - 1)]
    want = [FD.frame_verdicts(up, g, d) for g in muts]
    sizes, _ = run(k4, "info", muts, [d] * len(muts))
    assert list(sizes) == [w[0] for w in want]
    out, dst, do, dc = run(k4, "decode", muts, [d] * len(muts), [w[3] + 64 for w in want])
    assert list(out) == [w[1] for w in want]
    got = frames_of(out, dst, do, dc)
    for i, w in enumerate(want):
        if w[2] is not None:
            assert got[i] == w[2], i
    assert sum(w[1] >= 0 for w in want) > len(base) and sum(w[1] == -1 for w in want) > 0


def test_tile_kernel_decodes_clean_dictionary_blocks(k4, up):
    B = k4.batch
    rng = np.random.default_rng(47)
    d = DR.records(65536, 77)
    items = [FD.content(rng, int(rng.integers(200, 4096)), d) for _ in range(200)]
    frames = [up.cdict_frame(x, d, 65536, linked, False, False, 9) for x in items for linked in (False, True)]
    want = [x for x in items for _ in range(2)]
    B.decode_stats(0, reset=True)
    contents, out = k4.LZ4Frame.DecodeManyWithDictionary(frames, [d] * len(frames))
    stats = B.decode_stats(0, reset=True)
    assert contents == want
    compressed = sum(1 for f in frames if not any(_raws(f)))
    assert stats["generic"] == 0 and stats["tile"] >= compressed, stats


def _raws(f):
    from k4os.compression.lz4_b200.frame import _Frame
    return _Frame(f, dictionary=True).raws
