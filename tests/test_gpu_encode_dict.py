"""Encoding against an external dictionary on the GPU (k4lz4_encode_dict_batch), compared byte for byte with
upstream's LZ4_loadDict + LZ4_compress_fast_continue on the dictionary in a buffer of its own, and decoded back
through k4lz4_decode_dict_batch and upstream's LZ4_decompress_safe_usingDict."""
import ctypes as C

import numpy as np
import pytest

from tests import dict_enc_ref as DR

pytestmark = pytest.mark.gpu

DICT_LENGTHS = [0, 1, 7, 8, 9, 3000, 65535, 65536, 65537, 200000]
MSG_LENGTHS = [1, 4, 12, 13, 14, 100, 256, 1024, 4096, 65535, 65536, 65547, 1 << 20]


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
    return DR.DictUpstream()


def _datagen(n, seed):
    import oracle
    return oracle.Port().datagen(max(n, 1), 0.55, 0.0, seed)[:n].tobytes()


def _content(kind, n, seed):
    if kind == "records":
        return DR.records(n, seed)
    if kind == "datagen":
        return _datagen(n, seed)
    if kind == "random":
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()
    return bytes(n)


def _check(k4, up, blocks, dicts, res, out):
    for i, (s, d) in enumerate(zip(blocks, dicts)):
        r, want = up.encode(s, d)
        assert out[i] == r and res[i] == want, (i, len(s), len(d), out[i], r)


@pytest.mark.parametrize("kind", ["records", "datagen", "random", "zeros"])
def test_matrix_equals_upstream_and_round_trips(k4, up, kind):
    from k4os.compression.lz4_b200 import batch
    dicts_by_len = {n: _content(kind, n, 1000 + n) for n in DICT_LENGTHS}
    blocks, dicts = [], []
    for dn in DICT_LENGTHS:
        for mn in MSG_LENGTHS:
            blocks.append(_content(kind, mn, 7 * dn + mn))
            dicts.append(dicts_by_len[dn])
    res, out = batch.encode_dict_batch_host(blocks, dicts)
    _check(k4, up, blocks, dicts, res, out)
    dec, dout = batch.decode_dict_batch_host(res, [len(b) for b in blocks], dicts)
    assert list(dout) == [len(b) for b in blocks] and dec == blocks
    for i in range(0, len(blocks), 7):
        assert up.decode(res[i], len(blocks[i]), dicts[i]) == (len(blocks[i]), blocks[i])


def test_catchup_stops_at_the_source_start(k4, up):
    from k4os.compression.lz4_b200 import batch
    src, d = DR.catchup_input()
    res, out = batch.encode_dict_batch_host([src], [d])
    assert (out[0], res[0]) == up.encode(src, d)
    assert res[0] != up.encode_prefix(src, d)[1]


def _flat(blocks, dicts, caps):
    from k4os.compression.lz4_b200 import batch
    src, so, sl = batch._pack(blocks)
    dic, do, dl = batch._pack(dicts)
    dst, doff, dc = batch._slots(caps)
    return src, so, sl, dic, do, dl, dst, doff, dc


def test_capacities_and_untouched_tail(k4, up, native):
    from k4os.compression.lz4_b200 import _native as N
    d = DR.records(65536, 21)
    blocks, dicts, caps = [], [], []
    for n in (13, 300, 4096, 70000):
        s = DR.records(n, 22 + n)
        r, _ = up.encode(s, d)
        for c in (n + n // 255 + 16, r, r - 1, 1):
            blocks.append(s); dicts.append(d); caps.append(c)
    src, so, sl, dic, do, dl, dst, doff, dc = _flat(blocks, dicts, caps)
    out = np.full(len(blocks), -7, dtype=np.int32)
    N.check(native.k4lz4_encode_dict_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                           doff.ctypes.data, dc.ctypes.data, dic.ctypes.data, do.ctypes.data,
                                           dl.ctypes.data, out.ctypes.data, len(blocks), N.MEM_HOST, None, 0))
    for i, (s, c) in enumerate(zip(blocks, caps)):
        r, want = up.encode(s, d, c)
        assert out[i] == (r if r > 0 else -1), (i, c, r, out[i])
        slot = dst[doff[i]:doff[i] + c]
        if r > 0:
            assert slot[:r].tobytes() == want
        assert np.all(slot[max(r, 0):] == 0xCD)
    single = np.full(len(blocks[0]) + 64, 0xCD, dtype=np.uint8)
    s0 = np.frombuffer(blocks[0], dtype=np.uint8)
    dd = np.frombuffer(d, dtype=np.uint8)
    assert native.k4lz4_encode_dict(s0.ctypes.data, len(s0), single.ctypes.data, caps[0], dd.ctypes.data,
                                    len(d)) == out[0]
    assert single[:out[0]].tobytes() == up.encode(blocks[0], d)[1]
    assert native.k4lz4_encode_dict(s0.ctypes.data, len(s0), single.ctypes.data, 0, dd.ctypes.data, len(d)) == -1
    assert native.k4lz4_encode_dict(s0.ctypes.data, 0, single.ctypes.data, 10, dd.ctypes.data, len(d)) == 0
    assert native.k4lz4_encode_dict(s0.ctypes.data, len(s0), single.ctypes.data, caps[0], None, 0) == \
        up.encode(blocks[0], b"")[0]


def _mix(n, seed):
    """The pickler benchmark's message lengths: 256 B .. 4 KiB."""
    return np.random.default_rng(seed).integers(256, 4097, n)


def test_more_blocks_than_resident_warps(k4, up):
    from k4os.compression.lz4_b200 import batch
    d = DR.records(65536, 31)
    lens = _mix(6000, 32)
    body = DR.records(int(lens.sum()), 33)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    blocks = [body[o:o + n] for o, n in zip(offs, lens)]
    before = batch.encode_stats(0)["chain"]
    res, out = batch.encode_dict_batch_host(blocks, [d] * len(blocks))
    assert batch.encode_stats(0)["chain"] - before == len(blocks)
    _check(k4, up, blocks, [d] * len(blocks), res, out)


def _device_run(torch, blocks, dicts_idx, dict_bytes, caps, stream=None):
    """The batch in device memory: dictionary i of block b is dict_bytes[dicts_idx[b]]; -> (dst, doff, out)."""
    from k4os.compression.lz4_b200 import batch
    src, so, sl = batch._pack(blocks)
    dic, uo, ul = batch._pack(dict_bytes)
    do, dl = uo[np.asarray(dicts_idx)], ul[np.asarray(dicts_idx)]
    dst_h, doff, dc = batch._slots(caps)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    g = [t(src), t(so), t(sl), t(dst_h), t(doff), t(dc), t(dic), t(do.astype(np.int64)), t(dl.astype(np.int32)),
         torch.full((len(blocks),), -7, dtype=torch.int32, device="cuda")]
    return g, doff


def _call_device(g, n, stream):
    from k4os.compression.lz4_b200 import batch
    batch.encode_dict_batch_device(*[x.data_ptr() for x in g], n, stream=stream, device=0)


def test_messages_over_three_dictionaries_host_and_device(k4, up):
    torch = pytest.importorskip("torch")
    from k4os.compression.lz4_b200 import batch
    n = 100000
    dict_bytes = [DR.records(65536, 41), DR.records(20000, 42), _datagen(65536, 43)]
    which = np.random.default_rng(44).integers(0, 3, n)
    lens = _mix(n, 45)
    body = DR.records(int(lens.sum()), 46)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    blocks = [body[o:o + k] for o, k in zip(offs, lens)]
    dicts = [dict_bytes[w] for w in which]
    res, out = batch.encode_dict_batch_host(blocks, dicts)
    caps = [k + k // 255 + 16 for k in lens]
    g, doff = _device_run(torch, blocks, which, dict_bytes, caps)
    _call_device(g, n, 0)
    torch.cuda.synchronize()
    dout, ddst = g[9].cpu().numpy(), g[3].cpu().numpy()
    assert np.array_equal(dout, out)
    assert all(ddst[doff[i]:doff[i] + out[i]].tobytes() == res[i] for i in range(n))
    for i in range(0, n, 97):
        assert (out[i], res[i]) == up.encode(blocks[i], dicts[i]), i


def test_more_dictionaries_than_loaded_records(k4, up):
    """Every block with a dictionary of its own: beyond the launch's loaded records, warps load their own tables."""
    torch = pytest.importorskip("torch")
    from k4os.compression.lz4_b200 import batch
    n = 1500
    pool = DR.records(n * 64 + 4096, 51)
    dict_bytes = [pool[64 * i:64 * i + 3000] for i in range(n)]
    blocks = [DR.records(int(k), 52 + i) for i, k in enumerate(_mix(n, 53))]
    res, out = batch.encode_dict_batch_host(blocks, dict_bytes)
    _check(k4, up, blocks, dict_bytes, res, out)
    g, doff = _device_run(torch, blocks, np.arange(n), dict_bytes, [len(b) + len(b) // 255 + 16 for b in blocks])
    _call_device(g, n, 0)
    torch.cuda.synchronize()
    assert np.array_equal(g[9].cpu().numpy(), out)


def test_device_call_in_a_cuda_graph(k4, up):
    torch = pytest.importorskip("torch")
    d = DR.records(65536, 61)
    blocks = [DR.records(int(k), 62 + i) for i, k in enumerate(_mix(5000, 63))]
    caps = [len(b) + len(b) // 255 + 16 for b in blocks]
    g, doff = _device_run(torch, blocks, [0] * len(blocks), [d], caps)
    s = torch.cuda.Stream()
    _call_device(g, len(blocks), s.cuda_stream)         # warm-up outside the capture
    torch.cuda.synchronize()
    g[9].fill_(-7)
    g[3].fill_(0xCD)
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph, stream=s):
        _call_device(g, len(blocks), s.cuda_stream)
    assert np.all(g[9].cpu().numpy() == -7)            # captured, not run
    graph.replay()
    torch.cuda.synchronize()
    out, dst = g[9].cpu().numpy(), g[3].cpu().numpy()
    for i in range(len(blocks)):
        r, want = up.encode(blocks[i], d)
        assert out[i] == r and dst[doff[i]:doff[i] + r].tobytes() == want, i


def test_argument_codes_follow_decode_dict(k4, native):
    from k4os.compression.lz4_b200 import _native as N
    keep = [np.zeros(16, dtype=np.int64) for _ in range(10)]
    real = [a.ctypes.data for a in keep]
    ndev = native.k4lz4_device_count()
    fns = [native.k4lz4_encode_dict_batch, native.k4lz4_decode_dict_batch]
    for ptrs, n, mk, dev in [([None] * 10, 1, N.MEM_HOST, 0), ([None] * 10, -1, N.MEM_HOST, 0),
                             ([None] * 10, 0, N.MEM_HOST, 0), ([None] * 10, 0, N.MEM_DEVICE, 0),
                             (real, 1, 7, 0), (real, 1, N.MEM_HOST, ndev), (real, 1, N.MEM_DEVICE, ndev)]:
        codes = [f(*ptrs[:6], *ptrs[6:9], ptrs[9], n, mk, None, dev) for f in fns]
        assert codes[0] == codes[1], (n, mk, dev, codes)
    no_dict = real[:6] + [None, None, None] + real[9:]
    assert native.k4lz4_encode_dict_batch(*no_dict, 1, N.MEM_HOST, None, 0) == N.E_ARG
    assert native.k4lz4_encode_dict_batch(*no_dict, 0, N.MEM_HOST, None, 0) == N.OK
    assert native.k4lz4_encode_dict(None, 10, None, 10, None, 0) == N.E_ARG
