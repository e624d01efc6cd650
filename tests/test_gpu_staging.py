"""GPU tests of the synchronous host-memory calls (dictionary, partial and chained decode, XXH32).

Each batch goes through the same export twice, once with host memory (staged in chunks of at most 256 MiB)
and once with device memory, and the two must agree: the same results, and the same bytes in every
[dstOff, dstOff + outLen).  Each batch stages more than 256 MiB, so the host call runs in at least two
chunks.  The host call must leave every other destination byte as it was: the 0xCD sentinels after each
outLen and the history bytes in front of each chained slot."""
import numpy as np
import pytest

from tests import inputs
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
GOLD = ROOT + "/tests/golden/"
BS = 65536


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def data(k4):
    raw = k4.batch.synth_host(64, BS, 525, seed=5)
    plain = [raw[i * BS:(i + 1) * BS].tobytes() for i in range(64)]
    enc, _ = k4.batch.encode_batch_host(plain)
    rng = np.random.default_rng(3)
    bad = [inputs.mutate(enc[i], rng) for i in range(24)]
    gold = {k: open(GOLD + f"issue64_{k}", "rb").read() for k in ("block0.bin", "block1.lz4", "block1.bin")}
    return plain, enc, bad, gold


def _layout(items):
    """items: (source, capacity, history).  Distinct sources are stored once; slot i is [history | capacity]
    with 32 sentinel bytes after it."""
    at, parts, pos, soff = {}, [], 0, []
    for s, _, _ in items:
        if s not in at:
            at[s] = pos
            parts.append(s)
            pos += len(s)
        soff.append(at[s])
    src = np.frombuffer(b"".join(parts) + b"\0" * 16, dtype=np.uint8)
    doff, pos = [], 0
    for _, cap, h in items:
        pos = (pos + len(h) + 15) // 16 * 16
        doff.append(pos)
        pos += max(cap, 0) + 32
    dst = np.full(pos + 16, 0xCD, dtype=np.uint8)
    for o, (_, _, h) in zip(doff, items):
        if h:
            dst[o - len(h):o] = np.frombuffer(h, dtype=np.uint8)
    return (src, np.array(soff, dtype=np.int64), np.array([len(s) for s, _, _ in items], dtype=np.int32),
            dst, np.array(doff, dtype=np.int64), np.array([c for _, c, _ in items], dtype=np.int32))


def _both(native, call, arrays, out_dtype=np.int32):
    """call(pointers, out pointer, memKind, stream) with the arrays in host memory, then with copies of them
    on the device.  -> (host results, device results, host arrays after, device arrays after)."""
    import torch
    from k4os.compression.lz4_b200 import _native as N
    n = len(arrays[1])
    host = [a.copy() for a in arrays]
    out_h = np.full(n, -7, dtype=np.int32).view(out_dtype)
    N.check(call([a.ctypes.data for a in host], out_h.ctypes.data, N.MEM_HOST, None))
    dev = [torch.from_numpy(a.copy()).cuda() for a in arrays]
    out_d = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    N.check(call([t.data_ptr() for t in dev], out_d.data_ptr(), N.MEM_DEVICE,
                 torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out_h, out_d.cpu().numpy().view(out_dtype), host, [t.cpu().numpy() for t in dev]


def _check_dst(before, dst_h, dst_d, doff, out):
    written = np.zeros(before.shape, dtype=bool)
    for o, r in zip(doff, out):
        if r > 0:
            written[o:o + r] = True
    assert np.array_equal(dst_h[written], dst_d[written])
    assert np.array_equal(dst_h[~written], before[~written]), "the host call wrote outside [dstOff, dstOff + outLen)"


def _staged_bytes(items, dict_len=0):
    return sum(len(s) + max(c, 0) + len(h) + dict_len for s, c, h in items)


def test_dict_decode_host_equals_device(native, k4, data):
    plain, enc, bad, gold = data
    d0 = gold["block0.bin"]
    items = [(gold["block1.lz4"], BS, b""), (enc[0], BS - 1, b""), (b"", 10, b"")]
    items += [(b, BS, b"") for b in bad]
    items += [(enc[i % 64], BS, b"") for i in range(1800)]
    assert _staged_bytes(items, len(d0)) > 256 << 20
    src, so, sl, dst, do, dc = _layout(items)
    dic = np.frombuffer(d0, dtype=np.uint8).copy()
    dio = np.zeros(len(items), dtype=np.int64)
    dil = np.full(len(items), len(d0), dtype=np.int32)
    dil[1::2] = 0                                      # every other block without a dictionary
    call = lambda p, out, mk, st: native.k4lz4_decode_dict_batch(*p, out, len(items), mk, st, 0)
    oh, od, h, d = _both(native, call, [src, so, sl, dst, do, dc, dic, dio, dil])
    assert np.array_equal(oh, od)
    assert oh[0] == len(gold["block1.bin"]) and oh[1] == -1 and oh[2] == 0
    assert (oh[3 + len(bad):] == BS).all()
    _check_dst(dst, h[3], d[3], do, oh)
    assert h[3][do[0]:do[0] + oh[0]].tobytes() == gold["block1.bin"]


def test_partial_decode_host_equals_device(native, k4, data):
    plain, enc, bad, _ = data
    items = [(enc[i % 64], t, b"") for i, t in enumerate([0, 1, 5, 17, 1000, BS - 1, BS, BS + 100, -3])]
    items += [(b, 3000, b"") for b in bad]
    items += [(enc[i % 64], BS - (i % 7) * 4099, b"") for i in range(3200)]
    assert _staged_bytes(items) > 256 << 20
    src, so, sl, dst, do, dc = _layout(items)
    call = lambda p, out, mk, st: native.k4lz4_partial_decode_batch(*p, out, len(items), mk, st, 0)
    oh, od, h, d = _both(native, call, [src, so, sl, dst, do, dc])
    assert np.array_equal(oh, od)
    _check_dst(dst, h[3], d[3], do, oh)
    for i, (s, t, _) in enumerate(items[:9]):
        if oh[i] > 0:
            assert h[3][do[i]:do[i] + oh[i]].tobytes() == plain[i % 64][:oh[i]]


def test_chain_decode_host_equals_device(native, k4, data):
    plain, enc, bad, gold = data
    b0, b1z = gold["block0.bin"], gold["block1.lz4"]
    items = [(b1z, BS, b0[-65535:]), (b1z, BS, b0[-100:]), (b1z, BS, b""), (enc[1], BS, b"x" * 70000)]
    items += [(b, BS, plain[3][:i * 997]) for i, b in enumerate(bad)]
    items += [(b1z, BS, b0[-65535:]) if i % 2 else (enc[i % 64], BS, plain[i % 64][:i * 31 % BS])
              for i in range(2100)]
    assert sum(len(s) + c + min(len(h), 65535) for s, c, h in items) > 256 << 20
    src, so, sl, dst, do, dc = _layout(items)
    pre = np.array([len(h) for _, _, h in items], dtype=np.int32)
    call = lambda p, out, mk, st: native.k4lz4_decode_chain_batch(*p, out, len(items), mk, st, 0)
    oh, od, h, d = _both(native, call, [src, so, sl, dst, do, dc, pre])
    assert np.array_equal(oh, od)
    assert oh[0] == len(gold["block1.bin"]) and oh[3] == BS
    _check_dst(dst, h[3], d[3], do, oh)
    assert h[3][do[0]:do[0] + oh[0]].tobytes() == gold["block1.bin"]


def test_xxh32_host_equals_device(native, k4, data):
    plain, enc, _, _ = data
    items = [(b"", 0, b""), (b"a", 0, b""), (plain[0][:17], 0, b""), (enc[0], 0, b"")]
    items += [(plain[i % 64], 0, b"") for i in range(4200)]
    assert _staged_bytes(items) > 256 << 20
    src, so, sl = _layout(items)[:3]
    call = lambda p, out, mk, st: native.k4lz4_xxh32_batch(*p, 9, out, len(items), mk, st, 0)
    oh, od, _, _ = _both(native, call, [src, so, sl], np.uint32)
    assert np.array_equal(oh, od)
    for i in range(8):
        assert oh[i] == native.k4lz4_xxh32(src[so[i]:].ctypes.data, int(sl[i]), 9)
