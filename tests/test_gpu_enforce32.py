"""The 32-bit engine (LZ4Codec.Enforce32) on the GPU: every _x32 export against the reference's 32-bit engine.

Chained blocks are compared with upstream's LZ4_compress_fast_continue built as LL32 (oracle/_ref/libk4ref32.so) on
a planted state: result, bytes and the whole state record after every step.  The pickler is compared with its
restatement over LZ4Codec.Encode with enforce32, frames with a frame restatement over the same engines and with
upstream's LZ4F decoder, writer groups and chain groups with the batch calls.
"""
import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests import enforce32_ref as E
from tests import inputs
from tests import test_gpu_chain_encode as CE

pytestmark = pytest.mark.gpu
SB = ER.STATE_BYTES


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


@pytest.fixture(scope="module")
def up32():
    if not E.have_ref32():
        pytest.fail("oracle/_ref/libk4ref32.so missing: run __graft_entry__.build() where the reference is present")
    return E.EncUpstream32()


@pytest.fixture
def enforce32():
    from k4os.compression.lz4_b200 import LZ4Codec
    LZ4Codec.Enforce32 = True
    try:
        yield
    finally:
        LZ4Codec.Enforce32 = False


def _data(n: int, k: int, seed: int) -> np.ndarray:
    """Input kind k % 4: datagen 0.63, datagen 0.55, text, high entropy."""
    import oracle
    if k % 4 < 2:
        return oracle.Port().datagen(max(n, 1), (0.63, 0.55)[k % 4], 0.0, seed)[:n].copy()
    return np.frombuffer(inputs.gen(("lorem", "random")[k % 4 - 2], n, seed), dtype=np.uint8).copy()


def run_x32(k4, items, host, x32=True, level=0):
    """items (history, src, cap, state) through k4lz4_encode_chain_batch(_x32), host or device memory."""
    src, so, sl, pl, dst, do, dc, st, sto = CE._layout(items)
    if host:
        out = k4.batch.encode_chain_batch_host(src, so, sl, pl, dst, do, dc, st, sto, level, x32=x32)
        return out, dst, do, st, sto
    import torch
    dev = torch.device("cuda", 0)
    t = [torch.from_numpy(a).to(dev) for a in (src, so, sl, pl, dst, do, dc, st, sto)]
    t_out = torch.full((len(items),), -7, dtype=torch.int32, device=dev)
    k4.batch.encode_chain_batch_device(*[x.data_ptr() for x in t], t_out.data_ptr(), len(items), level,
                                       torch.cuda.current_stream().cuda_stream, x32=x32)
    torch.cuda.synchronize()
    return t_out.cpu().numpy(), t[4].cpu().numpy(), do, t[7].cpu().numpy(), sto


# ---- 1. many streams x 16 linked blocks, one call per step ------------------------------------------------------

@pytest.mark.parametrize("host", [False, True])
def test_4224_streams_16_linked_blocks(k4, up32, host):
    """4 224 streams (more than one wave of 132 x 32 warps) x 16 linked 4 KiB blocks of four kinds of data."""
    import torch
    S, B, BS = 4224, 16, 4096
    raw = np.concatenate([_data(S // 4 * B * BS, k, 40 + k) for k in range(4)])
    cap = CE._bound(BS)
    stride = SB + 64
    sts = [up32.lib.LZ4_createStream() for _ in range(S)]
    try:
        states = np.full(S * stride, 0xCD, dtype=np.uint8)
        sto = np.arange(S, dtype=np.int64) * stride + 32
        for o in sto:
            states[o:o + SB] = 0
        do = np.arange(S, dtype=np.int64) * (cap + 64) + 32
        dev = torch.device("cuda", 0)
        if not host:
            t_raw, t_st, t_sto, t_do = (torch.from_numpy(a).to(dev) for a in (raw, states, sto, do))
        for k in range(B):
            so = np.arange(S, dtype=np.int64) * (B * BS) + k * BS
            sl, pl, dc = np.full(S, BS, np.int32), np.full(S, k * BS, np.int32), np.full(S, cap, np.int32)
            if host:
                dst = np.full(S * (cap + 64) + 64, 0xCD, dtype=np.uint8)
                out = k4.batch.encode_chain_batch_host(raw, so, sl, pl, dst, do, dc, states, sto, x32=True)
                st_now = states
            else:
                t_dst = torch.full((S * (cap + 64) + 64,), 0xCD, dtype=torch.uint8, device=dev)
                t_out = torch.full((S,), -7, dtype=torch.int32, device=dev)
                ts = [torch.from_numpy(a).to(dev) for a in (so, sl, pl, dc)]
                k4.batch.encode_chain_batch_device(t_raw.data_ptr(), ts[0].data_ptr(), ts[1].data_ptr(),
                                                   ts[2].data_ptr(), t_dst.data_ptr(), t_do.data_ptr(),
                                                   ts[3].data_ptr(), t_st.data_ptr(), t_sto.data_ptr(),
                                                   t_out.data_ptr(), S, 0, torch.cuda.current_stream().cuda_stream,
                                                   x32=True)
                torch.cuda.synchronize()
                out, dst, st_now = t_out.cpu().numpy(), t_dst.cpu().numpy(), t_st.cpu().numpy()
            for s in range(S):
                r, b = up32.compress(sts[s], raw.ctypes.data + int(so[s]), BS, cap)
                assert r > 0 and int(out[s]) == r, (k, s)
                assert dst[do[s]:do[s] + r].tobytes() == b, (k, s)
                assert (dst[do[s] + r:do[s] + cap + 64] == 0xCD).all(), (k, s)
                assert np.array_equal(st_now[sto[s]:sto[s] + SB], up32.state_of(sts[s])), (k, s)
    finally:
        for st in sts:
            up32.lib.LZ4_freeStream(st)


# ---- 2. edge cases on planted states ------------------------------------------------------------------------------

def _hash4_items(up32):
    """Offsets of exactly 65 535 (accepted) and 65 536 (rejected) planted in the hash4 slot; inputs whose 4-byte
    words collide under hash4 at 12 bits, so that a batch's probes share slots and forward stores to each other."""
    rng = np.random.default_rng(4)
    items = []
    H = rng.integers(0, 256, 70000, dtype=np.uint8).tobytes()
    for dist in (65535, 65536):
        t = len(H) + 1 - dist
        src = bytearray(rng.integers(0, 256, 300, dtype=np.uint8).tobytes())
        src[1:41] = H[t:t + 40]
        table = np.zeros(4096, dtype=np.uint32)
        table[E.hash4(H[t:t + 4])] = t
        items.append((H, bytes(src), 400, ER.make_state(table, len(H), len(H))))
    words = rng.integers(0, 1 << 32, 1 << 18, dtype=np.uint64).astype(np.uint32)
    h = ((words.astype(np.uint64) * 2654435761) & 0xFFFFFFFF) >> 20
    bucket = words[h == np.bincount(h.astype(np.int64)).argmax()][:16]
    assert len(bucket) >= 8
    for v, n in enumerate((300, 5000, 70000, 300000)):
        if v % 2:                                # the same colliding words over and over (hits behind misses)
            w = np.tile(bucket[:8], n // 32 + 1)
        else:                                    # colliding words in random order
            w = bucket[rng.integers(0, len(bucket), n // 4 + 1)]
        src = w.view(np.uint8)[:n].copy()
        if v >= 2:                               # and stretches of random bytes between them
            for at in rng.integers(0, n - 64, n // 2000):
                src[at:at + 40] = rng.integers(0, 256, 40, dtype=np.uint8)
        s = src.tobytes()
        items.append((b"", s, CE._bound(n), ER.make_state()))
        items.append((s[: n // 2], s, CE._bound(n), CE._after_block(up32, s[: n // 2])))
    return items


def _edge_items(up32):
    """The chained encoder's edge cases (tests/test_gpu_chain_encode.edge_items, states from the 32-bit engine:
    blocks of 1 byte to 4 MiB, prefixes shorter than 64 KiB, dictSmall, limited capacities, the renormalisation
    past 2 GiB), the empty block, and the hash4 cases."""
    return CE.edge_items(up32) + [(b"abc", b"", 16, ER.make_state())] + _hash4_items(up32)


@pytest.mark.parametrize("host", [False, True])
def test_edge_cases(k4, up32, host):
    items = _edge_items(up32)
    want = [up32.step(s, h, src, cap) if len(src) else (0, b"", s) for h, src, cap, s in items]
    CE.check(items, want, run_x32(k4, items, host))
    assert any(w[0] == 0 for w in want) and sum(w[0] > 0 for w in want) > len(want) // 2


def test_hash4_cases_differ_from_the_plain_engine(up, up32):
    """The collision inputs mean what they say: the two engines encode them differently."""
    items = _hash4_items(up32)[2:]
    assert sum(up.step(s, h, src, cap)[1] != up32.step(s, h, src, cap)[1] for h, src, cap, s in items) >= 4


@pytest.mark.parametrize("host", [False, True])
def test_level_3_delegates_with_the_state_untouched(k4, up32, host):
    items = [(b"", _data(n, 0, n).tobytes(), CE._bound(n), ER.make_state(None, 12345, 678)) for n in (100, 70000)]
    out, _, _, st, sto = run_x32(k4, items, host, level=3)
    assert list(out) == [-2, -2]
    for i, it in enumerate(items):
        assert np.array_equal(st[sto[i]:sto[i] + SB], it[3])


def test_alternating_engines(k4, up, up32):
    """Streams alternate _x32 and plain calls on one state record; the reference's two engines take turns on one
    state the same way."""
    S, B = 12, 10
    rng = np.random.default_rng(8)
    datas = [_data(B * 70000, s, 300 + s).tobytes() for s in range(S)]
    states = [ER.make_state() for _ in range(S)]
    for k in range(B):
        for x32 in (k % 2 == 0, k % 2 == 1):
            items = []
            for s in range(S):
                if (s + k) % 2 == (0 if x32 else 1):
                    P = min(int(rng.integers(0, 80000)), k * 70000)
                    items.append((datas[s][k * 70000 - P:k * 70000], datas[s][k * 70000:k * 70000 + int(rng.integers(1, 70001))],
                                  CE._bound(70000), states[s]))
            if not items:
                continue
            eng = up32 if x32 else up
            want = [eng.step(st, h, src, cap) for h, src, cap, st in items]
            got = run_x32(k4, items, host=False, x32=x32)
            CE.check(items, want, got)
            it = iter(range(len(items)))
            for s in range(S):
                if (s + k) % 2 == (0 if x32 else 1):
                    states[s] = want[next(it)][2]


def test_fast_chain_encoder_under_enforce32(k4, up32, enforce32):
    """LZ4FastChainEncoder reads LZ4Codec.Enforce32 at each Encode: its ring model over the 32-bit engine."""
    from k4os.compression.lz4_b200 import LZ4FastChainEncoder
    rng = np.random.default_rng(9)
    for bs, extra in ((1024, 0), (65536, 1), (256 << 10, 0)):
        data = _data(4 * bs + 70000, bs, bs).tobytes()
        enc, ring = LZ4FastChainEncoder(bs, extra), ER.RingModel(up32, bs, extra)
        cap = CE._bound(enc.BlockSize)
        o = 0
        try:
            while o < len(data):
                k = int(rng.integers(1, enc.BlockSize + 1))
                a = enc.Topup(data[o:o + k])
                assert ring.topup(data[o:o + k]) == a
                o += a
                t = np.full(cap, 0xCD, dtype=np.uint8)
                r = enc.Encode(t, True)
                rr, out, _, _, after = ring.encode(cap, True)
                assert r == rr and t[:abs(r)].tobytes() == out, (bs, o)
                assert np.array_equal(enc._state, after), (bs, o)
        finally:
            ring.close()


# ---- 3. the pickler and the block calls ----------------------------------------------------------------------------

def test_pickler_both_variants(k4, enforce32):
    import oracle
    import torch
    from k4os.compression.lz4_b200 import LZ4Codec, LZ4Pickler
    port = oracle.Port()
    sizes = [100, 65546, 65547, 65548, 100000, 300001, 1 << 20]
    msgs = [_data(n, i, 500 + i).tobytes() for i, n in enumerate(sizes)] + \
           [_data(n, 0, 600 + i).tobytes() for i, n in enumerate((65547, 65548, 200000))]
    want = [E.pickle(port, m) for m in msgs]
    want_w = [E.pickle_writer(port, m) for m in msgs]
    got, _ = k4.batch.pickle_batch_host(msgs, x32=True)
    got_w, _ = k4.batch.pickle_writer_batch_host(msgs, x32=True)
    assert got == want and got_w == want_w
    for m, w, ww in zip(msgs, want, want_w):
        assert LZ4Pickler.Pickle(m) == w and LZ4Pickler.Unpickle(w) == m
        sink = bytearray()
        LZ4Pickler.PickleTo(m, sink)
        assert bytes(sink) == ww
    # the device form
    src, so, sl = k4.batch._pack(msgs)
    dst, do, _ = k4.batch._slots(np.where(sl > 0, sl + 1, 0))
    dev = torch.device("cuda", 0)
    t = [torch.from_numpy(a).to(dev) for a in (src, so, sl, dst, do)]
    t_out = torch.zeros(len(msgs), dtype=torch.int32, device=dev)
    k4.batch.pickle_batch_device(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(),
                                 t_out.data_ptr(), len(msgs), stream=torch.cuda.current_stream().cuda_stream, x32=True)
    torch.cuda.synchronize()
    assert k4.batch._slices(t[3].cpu().numpy(), do, t_out.cpu().numpy()) == want
    # below 65 547 bytes both engines agree; from there on they do for incompressible input only
    plain = [port.pickle(m) for m in msgs]
    assert all(p == w for m, p, w in zip(msgs, plain, want) if len(m) < 65547)
    assert sum(p != w for p, w in zip(plain, want)) >= 6
    for m in msgs:
        t = bytearray(LZ4Codec.MaximumOutputSize(len(m)))
        n = LZ4Codec.Encode(m, t)
        assert (n, bytes(t[:n])) == port.encode(m, len(t), 0, enforce32=True)


# ---- 4. frames, writer groups, chain groups -------------------------------------------------------------------------

def _frame_contents(B):
    rng = np.random.default_rng(B)
    out = []
    for j, n in enumerate((0, 1000, B, 2 * B + 12345)):
        c = _data(n, j, B + j)
        if n > 200000:
            at = int(rng.integers(0, n - 150000))
            c[at:at + 150000] = rng.integers(0, 256, 150000, dtype=np.uint8)
        out.append(c.tobytes())
    return out


@pytest.mark.parametrize("B", [1 << 16, 100000, 1 << 18, 1 << 22])
def test_frame_encode_x32(k4, up32, B, enforce32):
    import oracle
    import torch
    from k4os.compression.lz4_b200 import frame as F
    port, ref = oracle.Port(), oracle.Ref()
    contents = _frame_contents(B)
    for linked in (True, False):
        for bc in (False, True):
            for cc in (False, True):
                want = [E.frame_ref(up32, port, ref.xxh32, c, B, linked, bc, cc) for c in contents]
                frames, out = F.LZ4Frame.EncodeMany(contents, B, linked, bc, cc)
                assert frames == want, (B, linked, bc, cc)
                for c, f in zip(contents, frames):
                    assert ref.frame_decompress(f, len(c) + 16) == c
                assert F.read_frames(frames) == contents
                # device memory
                src, so, sl = k4.batch._pack([np.frombuffer(c, dtype=np.uint8) for c in contents])
                caps = [F.LZ4Frame.Bound(len(c), B, linked, bc, cc) for c in contents]
                dst, do, dc = k4.batch._slots(caps)
                dev = torch.device("cuda", 0)
                t = [torch.from_numpy(a).to(dev) for a in (src, so, sl, dst, do, dc)]
                t_out = torch.zeros(len(contents), dtype=torch.int32, device=dev)
                F.LZ4Frame.encode_many_device(*t, t_out, B, linked, bc, cc,
                                              stream=torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                assert k4.batch._slices(t[3].cpu().numpy(), do, t_out.cpu().numpy()) == want
    if B >= 65547:                                     # independent blocks of this size use the 32-bit engine
        from k4os.compression.lz4_b200 import LZ4Codec
        LZ4Codec.Enforce32 = False
        plain = F.LZ4Frame.EncodeMany(contents[2:], B, False)[0]
        LZ4Codec.Enforce32 = True
        assert plain != F.LZ4Frame.EncodeMany(contents[2:], B, False)[0]


@pytest.mark.parametrize("B,chaining", [(1 << 16, True), (100000, False), (100000, True)])
def test_writer_group_equals_frame_encode(k4, B, chaining, enforce32):
    """1 024 streams, random write cuts, then a close: each stream emits frame_encode_batch_x32 of its content."""
    from k4os.compression.lz4_b200 import frame as F
    from k4os.compression.lz4_b200.groups import FrameWriterGroup
    S = 1024
    rng = np.random.default_rng(B + chaining)
    raw = _data(4 << 20, 0, 77)
    lens = rng.integers(0, 300000, S)
    lens[:4] = [0, 1, B, 3 * B]
    contents = [raw[(s * 3761) % (len(raw) - 400000):][:lens[s]].tobytes() for s in range(S)]
    want = F.LZ4Frame.EncodeMany(contents, B, chaining, True, True)[0]
    got = [[] for _ in range(S)]
    at = [0] * S
    with FrameWriterGroup(S, B, chaining, True, True) as g:
        while True:
            todo = [s for s in range(S) if at[s] < len(contents[s]) or at[s] == 0]
            if not todo:
                break
            chunks = []
            for s in todo:
                k = int(rng.integers(0, 2 * B))
                chunks.append(contents[s][at[s]:at[s] + k])
                at[s] += max(k, 1) if not contents[s] else k
            outs, r = g.write(chunks, todo)
            assert (r >= 0).all()
            for s, o in zip(todo, outs):
                got[s].append(o)
        outs, r = g.close()
        assert (r >= 0).all()
        for s, o in enumerate(outs):
            got[s].append(o)
    assert [b"".join(x) for x in got] == want


def test_writer_group_device_forms(k4, enforce32):
    import torch
    from k4os.compression.lz4_b200 import frame as F
    from k4os.compression.lz4_b200.groups import FrameWriterGroup
    S, B = 64, 100000
    contents = [_data(250000, s, 900 + s).tobytes() for s in range(S)]
    want = F.LZ4Frame.EncodeMany(contents, B, True)[0]
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    got = [[] for _ in range(S)]
    with FrameWriterGroup(S, B) as g:
        streams = torch.arange(S, dtype=torch.int32, device=dev)
        for o in range(0, 250000, 90000):
            chunks = [c[o:o + 90000] for c in contents]
            src, so, sl = k4.batch._pack([np.frombuffer(c, dtype=np.uint8) for c in chunks])
            dst, do, dc = k4.batch._slots([g.bound(len(c)) for c in chunks])
            t = [torch.from_numpy(a).to(dev) for a in (src, so, sl, dst, do, dc)]
            t_out = torch.zeros(S, dtype=torch.int32, device=dev)
            g.write_device(streams.data_ptr(), *[x.data_ptr() for x in t], t_out.data_ptr(), S, st)
            torch.cuda.synchronize()
            for s, b in enumerate(k4.batch._slices(t[3].cpu().numpy(), do, t_out.cpu().numpy())):
                got[s].append(b)
        dst, do, dc = k4.batch._slots([g.close_bound()] * S)
        t = [torch.from_numpy(a).to(dev) for a in (dst, do, dc)]
        t_out = torch.zeros(S, dtype=torch.int32, device=dev)
        g.close_device(streams.data_ptr(), *[x.data_ptr() for x in t], t_out.data_ptr(), S, st)
        torch.cuda.synchronize()
        for s, b in enumerate(k4.batch._slices(t[0].cpu().numpy(), do, t_out.cpu().numpy())):
            got[s].append(b)
    assert [b"".join(x) for x in got] == want


def test_chain_group_agrees_with_the_chain_batch(k4):
    """ChainEncoderGroup under Enforce32, and on alternate steps without it, equals the chain batch call with the
    same engine per step; streams are a subset per call."""
    from k4os.compression.lz4_b200 import LZ4Codec
    from k4os.compression.lz4_b200.groups import ChainEncoderGroup
    S, BS, K = 300, 65536, 6
    rng = np.random.default_rng(12)
    datas = [_data(K * BS, s, 700 + s) for s in range(S)]
    states = [ER.make_state() for _ in range(S)]
    pos = [0] * S
    try:
        with ChainEncoderGroup(S, BS) as g:
            for k in range(K):
                LZ4Codec.Enforce32 = k % 3 != 2
                streams = [s for s in range(S) if rng.random() < 0.8]
                blocks = [datas[s][pos[s]:pos[s] + int(rng.integers(1, BS + 1))].tobytes() for s in streams]
                got, r = g.encode(blocks, streams)
                items = [(datas[s][:pos[s]][-65536:].tobytes(), b, CE._bound(len(b)), states[s])
                         for s, b in zip(streams, blocks)]
                out, dst, do, st, sto = run_x32(k4, items, host=True, x32=LZ4Codec.Enforce32)
                assert list(r) == list(out), k
                assert got == k4.batch._slices(dst, do, out), k
                for i, s in enumerate(streams):
                    states[s] = st[sto[i]:sto[i] + SB].copy()
                    assert np.array_equal(g.state(s)[:4096 * 4 + 4], states[s][:4096 * 4 + 4]), (k, s)
                    pos[s] += len(blocks[i])
    finally:
        LZ4Codec.Enforce32 = False


def test_group_x32_exports_check_arguments_as_their_twins(k4, native):
    from k4os.compression.lz4_b200 import _native as N
    from k4os.compression.lz4_b200.groups import ChainEncoderGroup, FrameWriterGroup
    keep = [np.zeros(64, dtype=np.int64) for _ in range(9)]
    p = [a.ctypes.data for a in keep]
    twice = np.zeros(4, dtype=np.int32)
    far = np.full(4, 999, dtype=np.int32)
    L = native
    with ChainEncoderGroup(4, 65536) as cg, FrameWriterGroup(4, 65536) as fw:
        for streams, n, level, mem in ((p[0], -1, 0, 0), (None, 1, 0, 0), (p[0], 1, 0, 7), (twice.ctypes.data, 2, 0, 0),
                                       (far.ctypes.data, 1, 0, 0), (p[0], 1, 256, 0), (p[0], 1, -1, 0)):
            a = (streams, *p[1:8], n, level, mem, None)
            assert L.k4lz4_chain_group_encode_x32(cg.handle, *a) == L.k4lz4_chain_group_encode(cg.handle, *a) == N.E_ARG
            w = (streams, *p[1:8], n, mem, None)
            if level == 0:
                assert L.k4lz4_frame_writer_group_write_x32(fw.handle, *w) == \
                    L.k4lz4_frame_writer_group_write(fw.handle, *w) == N.E_ARG
                c = (streams, *p[1:5], n, mem, None)
                assert L.k4lz4_frame_writer_group_close_x32(fw.handle, *c) == \
                    L.k4lz4_frame_writer_group_close(fw.handle, *c) == N.E_ARG
    from k4os.compression.lz4_b200.groups import ChainDecoderGroup
    with ChainDecoderGroup(2, 65536) as d:                    # a group of the other kind
        a = (p[0], *p[1:8], 1, 0, 0, None)
        assert L.k4lz4_chain_group_encode_x32(d.handle, *a) == L.k4lz4_chain_group_encode(d.handle, *a) == N.E_ARG


def test_stats_count_x32_chained_blocks(k4):
    B = k4.batch
    B.encode_stats(0, reset=True)
    items = [(b"", _data(n, 0, n).tobytes(), CE._bound(n), ER.make_state()) for n in (100, 65536, 70000, 1 << 20)]
    items.append((b"", b"", 16, ER.make_state()))
    out = run_x32(k4, items, host=False)[0]
    assert out[-1] == 0
    st = B.encode_stats(0, reset=True)
    assert (st["smem"], st["gtab"], st["generic"], st["chain"]) == (0, 0, 0, 4), st
    out = run_x32(k4, items[:2], host=False, level=3)[0]
    assert list(out) == [-2, -2] and B.encode_stats(0, reset=True)["chain"] == 0
