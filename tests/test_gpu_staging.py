"""GPU tests of the synchronous host-memory calls (dictionary, partial and chained decode, chained encode, XXH32,
decoded sizes, and whole-frame encode, decode and content sizes).

Each batch goes through the same export twice, once with host memory (staged in chunks of at most 256 MiB)
and once with device memory, and the two must agree: the same results, the same bytes in every
[dstOff, dstOff + outLen) and the same state records.  Each batch stages more than 256 MiB, so the host call
runs in at least two chunks.  The host call must leave every other destination byte as it was: the 0xCD
sentinels after each outLen and the history bytes in front of each chained slot.  The calls share one staging
area per device, so the last test runs four of them at once from several threads."""
import threading

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


SB = 16400                                             # K4LZ4_CHAIN_STATE_BYTES


def _enc_layout(items):
    """items: (history, source, capacity, state) -> [src, srcOff, srcLen, prefixLen, dst, dstOff, dstCap, states,
    stateOff]: [history | source] 16-aligned, destination slots with 32 sentinel bytes after each, state records
    with 32 sentinel bytes around each."""
    at, parts, pos, soff = {}, [], 0, []
    for h, s, _, _ in items:
        if (h, s) not in at:
            pos = (pos + len(h) + 15) // 16 * 16
            at[(h, s)] = pos
            parts.append((pos, h, s))
            pos += len(s)
        soff.append(at[(h, s)])
    src = np.zeros(pos + 16, dtype=np.uint8)
    for o, h, s in parts:
        src[o - len(h):o + len(s)] = np.frombuffer(h + s, dtype=np.uint8)
    _, _, _, dst, doff, dcap = _layout([(b"", c, b"") for _, _, c, _ in items])
    sto = np.array([32 + k * (SB + 64) for k in range(len(items))], dtype=np.int64)
    st = np.full(len(items) * (SB + 64) + 64, 0xCD, dtype=np.uint8)
    for o, (_, _, _, s) in zip(sto, items):
        st[o:o + SB] = s
    return [src, np.array(soff, dtype=np.int64), np.array([len(s) for _, s, _, _ in items], dtype=np.int32),
            np.array([len(h) for h, _, _, _ in items], dtype=np.int32), dst, doff, dcap, st, sto]


def _enc_call(native, n):
    return lambda p, out, mk, st: native.k4lz4_encode_chain_batch(*p, out, n, 0, mk, st, 0)


def test_chain_encode_host_equals_device(native, k4, data):
    plain = data[0]
    zero = np.zeros(SB, dtype=np.uint8)
    # first blocks of fresh streams: their states after the device arm start the second blocks below
    first = [(b"", plain[i], BS + BS // 255 + 16, zero) for i in range(64)]
    fa = _enc_layout(first)
    oh, od, h, d = _both(native, _enc_call(native, len(first)), fa)
    assert np.array_equal(oh, od) and (oh > 0).all()
    _check_dst(fa[4], h[4], d[4], fa[5], oh)
    assert np.array_equal(h[7], d[7])
    after = [d[7][o:o + SB].copy() for o in fa[8]]
    items = [(b"", plain[0], 100, zero), (b"", b"", 16, zero), (plain[1], plain[2], 10, after[1])]
    items += [(plain[3] + plain[4][:4464], plain[5], BS + 300, zero)]            # 70000 bytes of history
    items += [(plain[i % 64], plain[(i + 1) % 64], BS + 300 if i % 5 else BS - i % 4000, after[i % 64])
              for i in range(1400)]
    assert sum(len(s) + min(c, len(s) + len(s) // 255 + 16) + min(len(h), 65535) + 16 + SB
               for h, s, c, _ in items) > 256 << 20
    a = _enc_layout(items)
    oh, od, h, d = _both(native, _enc_call(native, len(items)), a)
    assert np.array_equal(oh, od)
    assert oh[0] == -1 and oh[1] == 0 and oh[2] == -1 and (oh[4:] > 0).any()
    _check_dst(a[4], h[4], d[4], a[5], oh)
    assert np.array_equal(h[7], d[7]), "state records differ"
    outside = np.ones(a[7].shape, dtype=bool)
    for o in a[8]:
        outside[o:o + SB] = False
    assert (h[7][outside] == 0xCD).all(), "the host call wrote outside the state records"


def test_decoded_size_host_equals_device(native, k4, data):
    plain, enc, bad, _ = data
    items = [(b"", 0, b""), (enc[0][:-1], 0, b"")] + [(b, 0, b"") for b in bad]
    items += [(enc[i % 64] if i % 3 == 0 else plain[i % 64], 0, b"") for i in range(6600)]
    assert _staged_bytes(items) > 256 << 20
    src, so, sl = _layout(items)[:3]
    call = lambda p, out, mk, st: native.k4lz4_decoded_size_batch(*p, out, len(items), mk, st, 0)
    oh, od, _, _ = _both(native, call, [src, so, sl])
    assert np.array_equal(oh, od)
    assert oh[0] == 0 and all(oh[2 + len(bad) + i] == BS for i in range(0, 6600, 3))


@pytest.fixture(scope="module")
def contents(data):
    big = b"".join(data[0])
    sizes = [0, 1, 1000, BS, BS + 1, 300000, 1 << 20, 1500000, 2 << 20, 3000001, len(big) - 5]
    return [big[i * 4099:i * 4099 + n] for i, n in enumerate(sizes)]


def _frame_call(native, what, n, bs=BS, flags=0):
    if what == "encode":
        return lambda p, out, mk, st: native.k4lz4_frame_encode_batch(*p, out, n, bs, flags, 0, mk, st, 0)
    if what == "decode":
        return lambda p, out, mk, st: native.k4lz4_frame_decode_batch(*p, out, n, mk, st, 0)
    return lambda p, out, mk, st: native.k4lz4_frame_content_size_batch(*p, out, n, mk, st, 0)


@pytest.mark.parametrize("flags", [6, 7], ids=["linked", "independent"])
def test_frame_encode_host_equals_device(native, k4, contents, flags):
    bound = lambda c: int(native.k4lz4_frame_bound(len(c), BS, flags))
    items = [(contents[6], 12, b""), (contents[8], 100, b"")]                  # no room for the header / the frame
    items += [(c, bound(c), b"") for c in contents] * 12
    assert _staged_bytes(items) > 256 << 20
    src, so, sl, dst, do, dc = _layout(items)
    oh, od, h, d = _both(native, _frame_call(native, "encode", len(items), flags=flags), [src, so, sl, dst, do, dc])
    assert np.array_equal(oh, od)
    assert oh[0] == -1 and oh[1] == -1 and (oh[2:] > 0).all()
    _check_dst(dst, h[3], d[3], do, oh)


@pytest.fixture(scope="module")
def frames(k4, contents):
    return [k4.frame.write_frames(contents, BS, True, True, chaining=ch) for ch in (True, False)]


def test_frame_decode_host_equals_device(native, k4, contents, frames):
    rng = np.random.default_rng(8)
    lens = [len(c) for c in contents]
    items = [(inputs.mutate(f, rng), n, b"") for fs in frames for f, n in zip(fs, lens) if n > 0]  # corrupt
    items += [(f, n - 1, b"") for f, n in zip(frames[0], lens) if n > 0]                          # too small
    items += [(f, n + (i % 3) * 7, b"") for i in range(12) for fs in frames for f, n in zip(fs, lens)]
    assert _staged_bytes(items) > 256 << 20
    src, so, sl, dst, do, dc = _layout(items)
    oh, od, h, d = _both(native, _frame_call(native, "decode", len(items)), [src, so, sl, dst, do, dc])
    assert np.array_equal(oh, od)
    k = 2 * (len(lens) - 1)
    assert (oh[:k] < 0).any() and (oh[k:k + len(lens) - 1] == k4._native.R_DST_SMALL).all()
    assert oh[k + len(lens) - 1:].tolist() == lens * 24
    _check_dst(dst, h[3], d[3], do, oh)
    for i, c in zip(range(k + len(lens) - 1, len(items)), contents * 24):
        assert h[3][do[i]:do[i] + len(c)].tobytes() == c


def test_frame_content_size_host_equals_device(native, k4, contents, frames):
    rng = np.random.default_rng(9)
    items = [(inputs.mutate(f, rng), 0, b"") for f in frames[0]] + [(b"", 0, b"")]
    while _staged_bytes(items) <= 300 << 20:
        items += [(f, 0, b"") for fs in frames for f in fs]
    src, so, sl = _layout(items)[:3]
    oh, od, _, _ = _both(native, _frame_call(native, "size", len(items)), [src, so, sl])
    assert np.array_equal(oh, od)
    assert oh[len(frames[0]) + 1:].tolist() == [len(c) for c in contents] * ((len(items) - len(frames[0]) - 1)
                                                                            // len(contents))


def test_concurrent_host_calls_equal_alone(native, k4, data, contents):
    """Dictionary decode, chained encode, frame encode and XXH32 with host memory from four threads at once on
    device 0 (ctypes lets go of the GIL during each call): every result and every output byte is that of the same
    call made alone."""
    from k4os.compression.lz4_b200 import _native as N
    plain, enc, _, gold = data
    d0 = np.frombuffer(gold["block0.bin"], dtype=np.uint8).copy()
    dec = _layout([(gold["block1.lz4"], BS, b"")] + [(enc[i % 64], BS, b"") for i in range(900)])
    dio, dil = np.zeros(901, dtype=np.int64), np.full(901, len(d0), dtype=np.int32)
    zero = np.zeros(SB, dtype=np.uint8)
    enc_items = [(plain[i % 64], plain[(i + 1) % 64], BS + 300, zero) for i in range(600)]
    ea = _enc_layout(enc_items)
    fr = _layout([(c, int(native.k4lz4_frame_bound(len(c), BS, 6)), b"") for c in contents] * 8)
    xa = _layout([(plain[i % 64], 0, b"") for i in range(2000)])[:3]

    def dict_decode():
        a = [x.copy() for x in list(dec) + [d0, dio, dil]]
        out = np.full(901, -7, dtype=np.int32)
        N.check(native.k4lz4_decode_dict_batch(*[x.ctypes.data for x in a], out.ctypes.data, 901, N.MEM_HOST, None, 0))
        return out, a[3]

    def chain_encode():
        a = [x.copy() for x in ea]
        out = np.full(len(enc_items), -7, dtype=np.int32)
        N.check(_enc_call(native, len(enc_items))([x.ctypes.data for x in a], out.ctypes.data, N.MEM_HOST, None))
        return out, a[4], a[7]

    def frame_encode():
        a = [x.copy() for x in fr]
        out = np.full(len(a[1]), -7, dtype=np.int32)
        N.check(_frame_call(native, "encode", len(a[1]), flags=6)([x.ctypes.data for x in a], out.ctypes.data,
                                                                  N.MEM_HOST, None))
        return out, a[3]

    def xxh32():
        out = np.zeros(2000, dtype=np.uint32)
        N.check(native.k4lz4_xxh32_batch(*[x.ctypes.data for x in xa], 9, out.ctypes.data, 2000, N.MEM_HOST, None, 0))
        return (out,)

    calls = [dict_decode, chain_encode, frame_encode, xxh32]
    alone = [f() for f in calls]
    assert (alone[0][0][1:] == BS).all() and (alone[1][0] > 0).all() and (alone[2][0] > 0).all()
    got, errors = [[] for _ in calls], []
    start = threading.Barrier(len(calls))

    def worker(k):
        try:
            start.wait()
            for _ in range(3):
                got[k].append(calls[k]())
        except Exception as e:                         # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(len(calls))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for k, f in enumerate(calls):
        assert len(got[k]) == 3
        for res in got[k]:
            assert all(np.array_equal(x, y) for x, y in zip(res, alone[k])), f.__name__
