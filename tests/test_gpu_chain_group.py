"""Chain groups on the GPU (k4lz4_chain_group_*, ChainEncoderGroup / ChainDecoderGroup): every step compared with
the host-resident LZ4FastChainEncoder / LZ4ChainDecoder and with upstream, through host and device memory, with
0xCD sentinels beyond every block's result and the path counters."""
import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests import chain_group_ref as GR
from tests import chain_ref as CR

pytestmark = pytest.mark.gpu
K64 = 65536
GAP = 32


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
    return ER.EncUpstream()


def _datagen(n, seed):
    import oracle
    return oracle.Port().datagen(max(n, 1), 0.63, 0.0, seed)[:n].tobytes()


def _bound(n):
    return n + n // 255 + 16 if n > 0 else 16


def _layout(blocks, caps):
    """Packed sources and 0xCD destination slots with GAP sentinel bytes between them."""
    lens = np.array([len(b) for b in blocks], np.int32)
    so = np.zeros(len(blocks), np.int64)
    so[1:] = np.cumsum(lens[:-1], dtype=np.int64)
    src = np.frombuffer(b"".join(blocks) + b"\0" * 16, np.uint8).copy()
    caps = np.array(caps, np.int32)
    do = GAP + np.concatenate([[0], np.cumsum(np.maximum(caps[:-1], 0).astype(np.int64) + GAP)]).astype(np.int64)
    dst = np.full(int(do[-1]) + max(int(caps[-1]), 0) + GAP, 0xCD, np.uint8) if len(caps) else np.zeros(1, np.uint8)
    return src, so, lens, dst, do, caps


def _check_sentinels(dst, do, caps, out):
    for i in range(len(out)):
        r = max(int(out[i]), 0)
        assert (dst[do[i] + r:do[i] + max(int(caps[i]), 0) + GAP] == 0xCD).all(), i
    assert (dst[:GAP] == 0xCD).all()


def group_call(k4, g, streams, blocks, caps, mem, level=0):
    """One encode or decode step of group g through host or device memory -> (results, list of produced bytes).
    Checks that nothing beyond each result was written (for encoding with device memory: beyond the capacity of
    a block that did not fit, like k4lz4_encode_chain_batch)."""
    import torch
    N = k4._native
    L = N.lib()
    enc = isinstance(g, k4.ChainEncoderGroup)
    src, so, sl, dst, do, dc = _layout(blocks, caps)
    st = np.array(streams, np.int32)
    n = len(blocks)
    if mem == "host":
        out = np.full(n, -7, np.int32)
        args = [g.handle, st.ctypes.data, src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                do.ctypes.data, dc.ctypes.data, out.ctypes.data, n]
        N.check(L.k4lz4_chain_group_encode(*args, level, N.MEM_HOST, None) if enc
                else L.k4lz4_chain_group_decode(*args, N.MEM_HOST, None))
    else:
        dev = torch.device("cuda", 0)
        t = [torch.from_numpy(a).to(dev) for a in (st, src, so, sl, dst, do, dc)]
        t_out = torch.full((n,), -7, dtype=torch.int32, device=dev)
        s = torch.cuda.current_stream().cuda_stream
        ptrs = [x.data_ptr() for x in t] + [t_out.data_ptr(), n]
        if enc:
            g.encode_device(*ptrs, level=level, stream=s)
        else:
            g.decode_device(*ptrs, stream=s)
        torch.cuda.synchronize()
        out, dst = t_out.cpu().numpy(), t[4].cpu().numpy()
    assert (out != -7).all()
    chk = out.copy()
    if enc and mem == "device":
        chk[chk == -1] = np.maximum(dc[chk == -1], 0)
    _check_sentinels(dst, do, dc, chk)
    return out, [dst[do[i]:do[i] + out[i]].tobytes() if out[i] > 0 else b"" for i in range(n)]


def _state_equiv(a, b):
    """Equal records, except that two dictSizes of at least 64 KiB both mean a full window."""
    a, b = a.view(np.uint32), b.view(np.uint32)
    return np.array_equal(a[:4097], b[:4097]) and (a[4097] == b[4097] or min(a[4097], b[4097]) >= K64) and \
        np.array_equal(a[4098:], b[4098:])


# ---- encoder ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mem", ["host", "device"])
def test_encoder_group_many_streams(k4, up, mem):
    """1 024 streams x 8 steps of 64 KiB (ragged: streams skip steps, short and 1-byte blocks), every block and
    state equal to LZ4FastChainEncoder.EncodeMany on the same data; streams 0 and S - 1 equal upstream."""
    S, steps, B = 1024, 8, K64
    rng = np.random.default_rng(11 if mem == "host" else 12)
    pool = _datagen(steps * B + S * 97, 5)
    encs = [k4.LZ4FastChainEncoder(B) for _ in range(S)]
    sent = [[] for _ in range(S)]
    made = {0: [], S - 1: []}
    nblocks = chained = 0
    with k4.ChainEncoderGroup(S, B) as g:
        for step in range(steps):
            full = step < 2 or step == steps - 1
            streams = [s for s in range(S) if full or s in (0, S - 1) or rng.random() < 0.7]
            blocks = []
            for s in streams:
                n = B if full or s in (0, S - 1) else int(rng.choice([B, 1, int(rng.integers(1, B))]))
                o = (s * 97 + step * B) % (len(pool) - n)
                blocks.append(pool[o:o + n])
            caps = [_bound(len(b)) for b in blocks]
            k4.batch.encode_stats(0, reset=True)
            out, got = group_call(k4, g, streams, blocks, caps, mem)
            chained += k4.batch.encode_stats(0, reset=True)["chain"]
            tg = [np.zeros(c, np.uint8) for c in caps]
            for s, b in zip(streams, blocks):
                assert encs[s].Topup(b) == len(b)
            want = k4.LZ4FastChainEncoder.EncodeMany([encs[s] for s in streams], tg)
            assert list(out) == want
            for k, s in enumerate(streams):
                assert got[k] == tg[k][:want[k]].tobytes(), (step, s)
                sent[s].append(blocks[k])
                if s in made:
                    made[s].append(got[k])
            nblocks += len(streams)
            for s in (streams if step in (0, steps - 1) else streams[::37]):
                assert _state_equiv(g.state(s), encs[s]._state), (step, s)
        for s in (0, S - 1):
            assert b"".join(sent[s]) and g.history(s) == b"".join(sent[s])[-K64:]
    assert chained == nblocks
    for s in (0, S - 1):                                       # full 64 KiB blocks: upstream on the contiguous stream
        assert made[s] == up.encode_chain(b"".join(sent[s]), B)


@pytest.mark.parametrize("B,extra", [(1024, 0), (1024, 3), (4 << 20, 0)])
def test_encoder_group_block_sizes(k4, B, extra):
    """Groups of 1 KiB and 4 MiB blocks against LZ4FastChainEncoder(B, extraBlocks) over enough steps to slide."""
    S = 6 if B <= 4096 else 3
    total = 4 * (2 * K64 + max(B, K64))
    steps = total // B if B <= 4096 else 4
    rng = np.random.default_rng(B + extra)
    data = [_datagen(steps * B, 100 + s) for s in range(S)]
    encs = [k4.LZ4FastChainEncoder(B, extra) for _ in range(S)]
    with k4.ChainEncoderGroup(S, B) as g:
        for step in range(steps):
            mem = "host" if step % 2 else "device"
            blocks = []
            for s in range(S):
                n = B if rng.random() < 0.8 else int(rng.integers(1, B + 1))
                blocks.append(data[s][step * B:step * B + n])
                encs[s].Topup(blocks[-1])
            caps = [_bound(len(b)) for b in blocks]
            out, got = group_call(k4, g, list(range(S)), blocks, caps, mem)
            tg = [np.zeros(c, np.uint8) for c in caps]
            want = k4.LZ4FastChainEncoder.EncodeMany(encs, tg)
            assert list(out) == want and got == [t[:r].tobytes() for t, r in zip(tg, want)], step
        for s in range(S):
            assert _state_equiv(g.state(s), encs[s]._state)


def test_encoder_group_failures_reset_and_untouched(k4):
    """A too-small dstCap gives -1 and the stream returns -1 until it is reset, the others unaffected; level >= 3,
    empty blocks, a block longer than B and (device memory) a stream index out of range change nothing; a reset
    mid-stream equals a new encoder."""
    B, S = K64, 4
    data = [_datagen(6 * B, 200 + s) for s in range(S)]
    fresh = k4.LZ4FastChainEncoder(B)
    with k4.ChainEncoderGroup(S, B) as g:
        out, _ = group_call(k4, g, range(S), [d[:B] for d in data], [_bound(B)] * S, "host")
        assert (out > 0).all()
        before = [g.state(s) for s in range(S)]
        out, _ = group_call(k4, g, range(S), [d[B:2 * B] for d in data], [_bound(B)] * S, "host", level=3)
        assert (out == k4._native.R_DELEGATE).all()
        out, _ = group_call(k4, g, [0, 1, 2], [b"", data[1][:B + 1], b""], [16, _bound(B + 1), 16], "device")
        assert list(out) == [0, -1, 0]
        out, _ = group_call(k4, g, [2, 9, -1], [data[2][:100]] * 3, [_bound(100)] * 3, "device")
        assert out[0] > 0 and list(out[1:]) == [-1, -1]
        g.reset([2])
        assert g.history(2) == b"" and not g.state(2).any()
        for s in (0, 1, 3):
            assert np.array_equal(g.state(s), before[s]) and g.history(s) == data[s][:B][-K64:]
        # stream 1 fails: the others go on
        out, got = group_call(k4, g, [0, 1, 3], [d[B:2 * B] for d in (data[0], data[1], data[3])],
                              [_bound(B), 100, _bound(B)], "host")
        assert out[0] > 0 and out[1] == -1 and out[2] > 0
        for mem in ("host", "device"):
            out, _ = group_call(k4, g, [1], [data[1][:10]], [_bound(10)], mem)
            assert list(out) == [-1]
        g.reset([1])
        for s, mem in ((1, "device"), (2, "host")):             # both equal a new encoder now
            out, got = group_call(k4, g, [s], [data[s][2 * B:3 * B]], [_bound(B)], mem)
            tg = [np.zeros(_bound(B), np.uint8)]
            fresh.Topup(data[s][2 * B:3 * B])
            want = k4.LZ4FastChainEncoder.EncodeMany([fresh], tg)
            assert list(out) == want and got[0] == tg[0][:want[0]].tobytes()
            assert np.array_equal(g.state(s), fresh._state)
            fresh = k4.LZ4FastChainEncoder(B)


def test_encoder_group_device_steps_enqueue_without_sync(k4):
    """Several device-memory steps enqueued on one stream with no host synchronisation between them, then one
    synchronise: the results equal the same steps taken one at a time through host memory."""
    import torch
    S, B, steps = 64, K64, 5
    dev = torch.device("cuda", 0)
    data = [_datagen(steps * B, 300 + s) for s in range(S)]
    cap = _bound(B)
    with k4.ChainEncoderGroup(S, B) as gd, k4.ChainEncoderGroup(S, B) as gh:
        streams = torch.arange(S, dtype=torch.int32, device=dev)
        so = torch.arange(S, dtype=torch.int64, device=dev) * B
        sl = torch.full((S,), B, dtype=torch.int32, device=dev)
        do = torch.arange(S, dtype=torch.int64, device=dev) * cap
        dc = torch.full((S,), cap, dtype=torch.int32, device=dev)
        srcs = [torch.from_numpy(np.frombuffer(b"".join(d[k * B:(k + 1) * B] for d in data), np.uint8).copy()).to(dev)
                for k in range(steps)]
        outs = [(torch.zeros(S * cap, dtype=torch.uint8, device=dev), torch.zeros(S, dtype=torch.int32, device=dev))
                for _ in range(steps)]
        torch.cuda.synchronize()
        st = torch.cuda.Stream()
        for step in range(steps):                              # only enqueues: no host synchronisation here
            dst, out = outs[step]
            gd.encode_device(streams.data_ptr(), srcs[step].data_ptr(), so.data_ptr(), sl.data_ptr(), dst.data_ptr(),
                             do.data_ptr(), dc.data_ptr(), out.data_ptr(), S, stream=st.cuda_stream)
        st.synchronize()
        for step in range(steps):
            want, wr = gh.encode([d[step * B:(step + 1) * B] for d in data])
            dst, out = outs[step][0].cpu().numpy(), outs[step][1].cpu().numpy()
            assert np.array_equal(out, wr)
            assert [dst[i * cap:i * cap + out[i]].tobytes() for i in range(S)] == want
        for s in (0, S - 1):
            assert np.array_equal(gd.state(s), gh.state(s)) and gd.history(s) == gh.history(s)


# ---- decoder ---------------------------------------------------------------------------------------------------

def _chained_stream(up, data: bytes, B: int, stored_every: int = 0):
    """Upstream's chained blocks of `data` in B-byte blocks; a block that does not shrink (or every
    `stored_every`-th block, made incompressible) is stored raw, as a linked frame stores it -> [(kind, bytes)]."""
    src = np.frombuffer(data, np.uint8)
    st = up.lib.LZ4_createStream()
    out = []
    try:
        for o in range(0, len(data), B):
            n = min(B, len(data) - o)
            r, enc = up.compress(st, src.ctypes.data + o, n, _bound(n))
            assert r > 0
            out.append(("raw", data[o:o + n]) if r >= n else ("lz4", enc))
    finally:
        up.lib.LZ4_freeStream(st)
    return out


@pytest.mark.parametrize("B,S,nb", [(K64, 512, 6), (256 << 10, 16, 5), (4 << 20, 3, 3)])
def test_decoder_group_streams(k4, up, B, S, nb):
    """Upstream-chained streams (with stored blocks fed through inject) decode to upstream's content and equal
    LZ4ChainDecoder.DecodeMany; history equals Peek; blocks of <= 64 KiB stay on the tile path."""
    rng = np.random.default_rng(B)
    datas, streams = [], []
    for s in range(S):
        d = bytearray(_datagen(nb * B, 400 + s))
        k = int(rng.integers(0, nb))                  # one incompressible block per stream: stored raw
        d[k * B:(k + 1) * B] = rng.integers(0, 256, B, dtype=np.uint8).tobytes()
        datas.append(bytes(d))
        streams.append(_chained_stream(up, datas[-1], B))
    decs = [k4.LZ4ChainDecoder(B) for _ in range(S)]
    n_lz4, tile, generic = 0, 0, 0          # tile: either stage size of the shared-memory tile kernel
    with k4.ChainDecoderGroup(S, B) as g:
        for step in range(nb):
            mem = "host" if step % 2 == 0 else "device"
            raw = [s for s in range(S) if streams[s][step][0] == "raw"]
            lz = [s for s in range(S) if streams[s][step][0] == "lz4"]
            if raw:
                g.inject([streams[s][step][1] for s in raw], raw)
                for s in raw:
                    decs[s].Inject(streams[s][step][1])
            if lz:
                k4.batch.decode_stats(0, reset=True)
                out, got = group_call(k4, g, lz, [streams[s][step][1] for s in lz], [B] * len(lz), mem)
                stats = k4.batch.decode_stats(0, reset=True)
                tile, generic = tile + stats["tile"] + stats["tile_big"], generic + stats["generic"]
                want = k4.LZ4ChainDecoder.DecodeMany([decs[s] for s in lz], [streams[s][step][1] for s in lz])
                assert list(out) == want
                for k, s in enumerate(lz):
                    assert got[k] == datas[s][step * B:step * B + want[k]] == decs[s].Peek(-want[k]).tobytes()
                n_lz4 += len(lz)
            for s in range(0, S, max(S // 8, 1)):
                h = g.history(s)
                assert h == decs[s].Peek(-len(h)).tobytes() and len(h) == min((step + 1) * B, K64)
    if B <= K64:
        assert tile == n_lz4 and generic == 0, (tile, generic, n_lz4)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_decoder_group_malformed_and_script(k4, mem):
    """Random Decode / Inject scripts (tests/chain_group_ref.decode_script: blocks of 1 byte to B, truncated and
    bit-flipped blocks followed by the valid one) on 8 streams at once: results, bytes and history equal the
    group's rule over the prefix-mode restatement; a malformed block leaves its stream unchanged."""
    B, S = 4096, 8
    scripts = [GR.decode_script(1000 + s, B, 150) for s in range(S)]
    models = [GR.GroupDecoder(B, CR.decompress_prefix) for _ in range(S)]
    fails = 0
    with k4.ChainDecoderGroup(S, B) as g:
        for step in range(max(len(x) for x in scripts)):
            live = [s for s in range(S) if step < len(scripts[s])]
            inj = [s for s in live if scripts[s][step][0] == "inj"]
            dec = [s for s in live if scripts[s][step][0] == "dec"]
            if inj:
                g.inject([scripts[s][step][1] for s in inj], inj)
                for s in inj:
                    models[s].inject(scripts[s][step][1])
            if dec:
                before = {s: g.history(s) for s in dec}
                out, got = group_call(k4, g, dec, [scripts[s][step][1] for s in dec],
                                      [scripts[s][step][2] for s in dec], mem)
                for k, s in enumerate(dec):
                    assert (int(out[k]), got[k]) == models[s].decode(scripts[s][step][1], scripts[s][step][2])
                    if out[k] < 0:
                        fails += 1
                        assert g.history(s) == before[s]
            for s in live:
                assert g.history(s) == models[s].ring.history()
    assert fails > 0


def test_group_arguments_with_device(k4):
    """Host-memory argument errors that need a group: stream out of range or listed twice, the other kind, a bad
    level; the group of the other kind is refused by every call."""
    N = k4._native
    L = N.lib()
    with k4.ChainEncoderGroup(4, 1024) as ge, k4.ChainDecoderGroup(4, 1024) as gd:
        for streams in ([0, 4], [1, 1], [-1]):
            with pytest.raises(N.K4Error) as e:
                ge.encode([b"abc"] * len(streams), streams)
            assert e.value.code == N.E_ARG
            with pytest.raises(N.K4Error) as e:
                gd.decode([b"\x10a"] * len(streams), streams)
            assert e.value.code == N.E_ARG
        with pytest.raises(N.K4Error) as e:
            ge.encode([b"abc"], level=256)
        assert e.value.code == N.E_ARG
        a = np.zeros(64, np.uint8)
        p = [a.ctypes.data] * 8
        assert L.k4lz4_chain_group_encode(gd.handle, *p, 1, 0, N.MEM_HOST, None) == N.E_ARG
        assert L.k4lz4_chain_group_decode(ge.handle, *p, 1, N.MEM_HOST, None) == N.E_ARG
        assert L.k4lz4_chain_group_inject(ge.handle, *p[:4], 1, N.MEM_HOST, None) == N.E_ARG
        assert L.k4lz4_chain_group_state(gd.handle, 0, a.ctypes.data) == N.E_ARG
        assert L.k4lz4_chain_group_state(ge.handle, 4, a.ctypes.data) == N.E_ARG
        assert L.k4lz4_chain_group_encode(ge.handle, None, *p[:7], 1, 0, N.MEM_HOST, None) == N.E_ARG
        assert L.k4lz4_chain_group_encode(ge.handle, *p, 0, 0, N.MEM_HOST, None) == N.OK
    import ctypes as C
    h = C.c_void_p(5)
    assert L.k4lz4_chain_group_create(0, 1 << 30, 4 << 20, 0, C.byref(h)) == N.E_NOMEM and h.value is None
