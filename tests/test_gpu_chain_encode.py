"""Chained block encoding on the GPU (k4lz4_encode_chain_batch, LZ4FastChainEncoder, linked frames), compared
with upstream's LZ4_compress_fast_continue for the result, the bytes and the whole state (4 096 slots,
currentOffset, dictSize) after every step.  0xCD sentinels guard every destination slot and state record."""
import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests import inputs

pytestmark = pytest.mark.gpu
SB = ER.STATE_BYTES
GAP = 48


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
    return oracle.Port().datagen(max(n, 1), 0.63, 0.0, seed)[:n]


def _bound(n):
    return n + n // 255 + 16


def _layout(items):
    """items: (history, src, cap, state) -> host arrays: sources [history | src] 16-aligned, 0xCD destination
    slots and state records with GAP sentinel bytes around each."""
    so, at = [], 0
    for h, s, _, _ in items:
        o = (at + len(h) + 15) // 16 * 16
        so.append(o)
        at = o + len(s)
    src = np.zeros(at + 16, dtype=np.uint8)
    for o, (h, s, _, _) in zip(so, items):
        src[o - len(h):o] = np.frombuffer(h, dtype=np.uint8)
        src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    do, at = [], GAP
    for _, _, c, _ in items:
        do.append(at)
        at = (at + max(c, 0) + GAP + 15) // 16 * 16
    dst = np.full(at + GAP, 0xCD, dtype=np.uint8)
    sto = np.array([GAP + 16 + k * (SB + 64) for k in range(len(items))], dtype=np.int64)
    st = np.full(len(items) * (SB + 64) + 128, 0xCD, dtype=np.uint8)
    for o, it in zip(sto, items):
        st[o:o + SB] = it[3]
    return (src, np.array(so, np.int64), np.array([len(i[1]) for i in items], np.int32),
            np.array([len(i[0]) for i in items], np.int32), dst, np.array(do, np.int64),
            np.array([i[2] for i in items], np.int32), st, sto)


def run_host(k4, items, level=0):
    src, so, sl, pl, dst, do, dc, st, sto = _layout(items)
    out = k4.batch.encode_chain_batch_host(src, so, sl, pl, dst, do, dc, st, sto, level)
    return out, dst, do, st, sto


def run_device(k4, items, level=0):
    import torch
    src, so, sl, pl, dst, do, dc, st, sto = _layout(items)
    dev = torch.device("cuda", 0)
    t = [torch.from_numpy(a).to(dev) for a in (src, so, sl, pl, dst, do, dc, st, sto)]
    t_out = torch.full((len(items),), -7, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    k4.batch.encode_chain_batch_device(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(),
                                       t[4].data_ptr(), t[5].data_ptr(), t[6].data_ptr(), t[7].data_ptr(),
                                       t[8].data_ptr(), t_out.data_ptr(), len(items), level, stream)
    torch.cuda.synchronize()
    return t_out.cpu().numpy(), t[4].cpu().numpy(), do, t[7].cpu().numpy(), sto


def check(items, want, got):
    """want[i] = (engine result, bytes, state after); got = run_*(...).  Results follow the ABI: 0 for an empty
    block, -1 for an engine result of 0."""
    out, dst, do, st, sto = got
    for i, (r, b, s) in enumerate(want):
        assert int(out[i]) == (r if r > 0 or not items[i][1] else -1), (i, int(out[i]), r)
        if r > 0:
            assert dst[do[i]:do[i] + r].tobytes() == b, i
        # bytes at index >= outLen inside the slot are untouched (a block that does not fit may have written
        # anything below its capacity, as the reference's engine does), and so are the gaps around it
        if r > 0:
            assert (dst[do[i] + r:do[i] + max(items[i][2], 0)] == 0xCD).all(), i
        cap = max(items[i][2], 0)
        assert (dst[do[i] - GAP:do[i]] == 0xCD).all() and (dst[do[i] + cap:do[i] + cap + GAP] == 0xCD).all(), i
        assert np.array_equal(st[sto[i]:sto[i] + SB], s), (i, _state_diff(st[sto[i]:sto[i] + SB], s))
        assert (st[sto[i] - GAP:sto[i]] == 0xCD).all() and (st[sto[i] + SB:sto[i] + SB + GAP] == 0xCD).all(), i
    assert (dst[-GAP:] == 0xCD).all()


def _state_diff(a, b):
    a, b = a.view(np.uint32), b.view(np.uint32)
    d = np.nonzero(a != b)[0]
    return [(int(j), int(a[j]), int(b[j])) for j in d[:5]], len(d)


def _hash5(b8: bytes) -> int:
    v = int.from_bytes(b8, "little")
    return (((v << 24) * 889523592379) & ((1 << 64) - 1)) >> 52


# ---- 1. many streams, one call per step ------------------------------------------------------------------------

def _streams_through(k4, up, S, B, BS, seed, host):
    """S streams x B linked BS-byte blocks of datagen, one call per step (device memory, or host memory);
    upstream runs the same streams over contiguous buffers.  Compares every block and state."""
    import torch
    raw = _datagen(S * B * BS, seed)
    sts = [up.lib.LZ4_createStream() for _ in range(S)]
    try:
        dev = torch.device("cuda", 0)
        stride = SB + 64
        states = np.full(S * stride, 0xCD, dtype=np.uint8)
        sto = np.arange(S, dtype=np.int64) * stride + 32
        for o in sto:
            states[o:o + SB] = 0
        cap = _bound(BS)
        do = np.arange(S, dtype=np.int64) * (cap + 64) + 32
        if not host:
            t_raw = torch.from_numpy(raw).to(dev)
            t_st = torch.from_numpy(states).to(dev)
            t_sto = torch.from_numpy(sto).to(dev)
            t_do = torch.from_numpy(do).to(dev)
        for k in range(B):
            so = np.arange(S, dtype=np.int64) * (B * BS) + k * BS
            sl = np.full(S, BS, dtype=np.int32)
            pl = np.full(S, k * BS, dtype=np.int32)
            dc = np.full(S, cap, dtype=np.int32)
            if host:
                dst = np.full(S * (cap + 64) + 64, 0xCD, dtype=np.uint8)
                out = k4.batch.encode_chain_batch_host(raw, so, sl, pl, dst, do, dc, states, sto)
                st_now = states
            else:
                t_dst = torch.full((S * (cap + 64) + 64,), 0xCD, dtype=torch.uint8, device=dev)
                t_out = torch.full((S,), -7, dtype=torch.int32, device=dev)
                ts = [torch.from_numpy(a).to(dev) for a in (so, sl, pl, dc)]
                k4.batch.encode_chain_batch_device(t_raw.data_ptr(), ts[0].data_ptr(), ts[1].data_ptr(),
                                                   ts[2].data_ptr(), t_dst.data_ptr(), t_do.data_ptr(),
                                                   ts[3].data_ptr(), t_st.data_ptr(), t_sto.data_ptr(),
                                                   t_out.data_ptr(), S, 0, torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                out, dst, st_now = t_out.cpu().numpy(), t_dst.cpu().numpy(), t_st.cpu().numpy()
            for s in range(S):
                r, b = up.compress(sts[s], raw.ctypes.data + int(so[s]), BS, cap)
                assert r > 0 and int(out[s]) == r, (k, s)
                assert dst[do[s]:do[s] + r].tobytes() == b, (k, s)
                assert (dst[do[s] + r:do[s] + cap + 64] == 0xCD).all(), (k, s)
                assert np.array_equal(st_now[sto[s]:sto[s] + SB], up.state_of(sts[s])), (k, s)
                assert (st_now[sto[s] - 32:sto[s]] == 0xCD).all() and (st_now[sto[s] + SB:sto[s] + SB + 32] == 0xCD).all()
    finally:
        for st in sts:
            up.lib.LZ4_freeStream(st)


@pytest.mark.parametrize("host", [False, True])
def test_1024_streams_linked_blocks(k4, up, host):
    """1 024 streams x 4 x 64 KiB of datagen, one call per step, through device and host memory."""
    _streams_through(k4, up, 1024, 4, 65536, 4321, host)


@pytest.mark.parametrize("host", [False, True])
def test_more_streams_than_one_round(k4, up, host):
    """4 400 streams in one call (warps take several blocks each); through host memory each call stages more
    than 256 MiB, so it is cut into chunks."""
    _streams_through(k4, up, 4400, 2, 65536, 99, host)


# ---- 3. edge cases against the planted-state oracle -------------------------------------------------------------

def _after_block(up, data: bytes, cap=None):
    """The state of a new stream after encoding `data` as one block."""
    a = np.frombuffer(data, dtype=np.uint8)
    st = up.lib.LZ4_createStream()
    try:
        up.compress(st, a.ctypes.data, len(data), cap or _bound(len(data)))
        return up.state_of(st)
    finally:
        up.lib.LZ4_freeStream(st)


def edge_items(up):
    rng = np.random.default_rng(11)
    items = []
    prev = _datagen(100000, 5).tobytes()
    s_prev = _after_block(up, prev)
    for i, n in enumerate([1, 4, 12, 13, 65535, 65536, 65547, 256 << 10, 1 << 20, 4 << 20]):
        src = _datagen(n, 100 + i).tobytes()
        items.append((b"", src, _bound(n), ER.make_state()))                 # a fresh first block
        items.append((prev, src, _bound(n), s_prev))                          # behind a 100 000-byte block
    # prefix lengths: saveDict(0) after 100 000 bytes, and P bytes of the previous block kept
    nxt = prev[50000:] + _datagen(60000, 6).tobytes()                         # refers back into `prev`
    for P in (0, 1, 3, 4, 65534, 65535, 65536, 70000):
        items.append((prev[len(prev) - P:], nxt, _bound(len(nxt)), s_prev))
    small = _after_block(up, prev[:30000])                                    # dictSmall: dictSize < 64 KiB
    items.append((prev[:30000], nxt, _bound(len(nxt)), small))
    # offsets of exactly 65 535 (accepted) and 65 536 (rejected) into the history, planted in the table
    H = rng.integers(0, 256, 70000, dtype=np.uint8).tobytes()
    for dist in (65535, 65536):
        t = len(H) + 1 - dist
        src = bytearray(rng.integers(0, 256, 300, dtype=np.uint8).tobytes())
        src[1:41] = H[t:t + 40]
        table = np.zeros(4096, dtype=np.uint32)
        table[_hash5(H[t:t + 8])] = t
        items.append((H, bytes(src), 400, ER.make_state(table, len(H), len(H))))
    # a catch-up that crosses into the history (and one stopped by a short prefix)
    W = rng.integers(0, 256, 40, dtype=np.uint8).tobytes()
    R = lambda k: rng.integers(0, 256, k, dtype=np.uint8).tobytes()
    hist = R(1000) + W[:20]
    src = W[20:] + R(30) + W + R(100)
    for P in (len(hist), 10):
        items.append((hist[len(hist) - P:], src, 400, ER.make_state(None, len(hist), len(hist))))
    # capacities around the result
    for i, n in enumerate((1000, 65536, 300000)):
        src = _datagen(n, 200 + i).tobytes()
        r, _, _ = up.step(s_prev, prev, src, _bound(n))
        for cap in (r - 1, r, _bound(n), 0):
            items.append((prev, src, cap, s_prev))
    # renormalisation: currentOffset + n just at and just above 0x80000000, random slots below it
    hist = _datagen(70000, 7).tobytes()
    for n in (65536, 300000):
        src = (hist[-20000:] + _datagen(n, 8).tobytes())[:n]
        for cur in (0x80000000 - n, 0x80000000 - n + 1, 0x7FFFFF00):
            table = rng.integers(cur - 200000, cur, 4096).astype(np.uint32)
            table[:100] = rng.integers(0, 1000, 100)
            items.append((hist, src, _bound(n), ER.make_state(table, cur, 70000)))
            items.append((hist, src, _bound(n), ER.make_state(table, cur, 500000)))
    # the adversarial kinds, fresh and behind a block of the same kind
    for kind in inputs.KINDS:
        a = inputs.gen(kind, 65536, 3)
        b = inputs.gen(kind, 200000, 4)
        items.append((b"", a, _bound(len(a)), ER.make_state()))
        items.append((a, b, _bound(len(b)), _after_block(up, a)))
    return items


@pytest.mark.parametrize("host", [False, True])
def test_edge_cases(k4, up, host):
    items = edge_items(up)
    want = [up.step(s, h, src, cap) if len(src) else (0, b"", s) for h, src, cap, s in items]
    got = (run_host if host else run_device)(k4, items)
    check(items, want, got)
    # the cases mean what they say
    assert any(w[0] == 0 for w in want) and sum(w[0] > 0 for w in want) > len(want) // 2


def test_mid_stream_failure_then_more_blocks(k4, up):
    """cap = r - 1 on block 1 of a stream (the engine returns 0, the state advances as upstream's), then blocks
    2 and 3 behind it; cap = r and the bound on the other streams."""
    BS, B = 65536, 4
    raw = _datagen(3 * B * BS, 17)
    probe = ER.EncUpstream.state_of
    caps = {}
    st = up.lib.LZ4_createStream()
    up.compress(st, raw.ctypes.data, BS, _bound(BS))
    r1, _ = up.compress(st, raw.ctypes.data + BS, BS, _bound(BS))
    up.lib.LZ4_freeStream(st)
    caps = [[_bound(BS)] * B, [_bound(BS), r1 - 1, _bound(BS), _bound(BS)], [_bound(BS), r1, _bound(BS), _bound(BS)]]
    sts = [up.lib.LZ4_createStream() for _ in range(3)]
    states = [ER.make_state() for _ in range(3)]
    try:
        for k in range(B):
            items, want = [], []
            for s in range(3):
                base = s * B * BS
                src = raw[base + k * BS:base + (k + 1) * BS].tobytes()
                items.append((raw[base:base + k * BS].tobytes(), src, caps[s][k], states[s]))
                r, b = up.compress(sts[s], raw.ctypes.data + base + k * BS, BS, caps[s][k])
                want.append((r, b, probe(up, sts[s])))
            got = run_device(k4, items)
            check(items, want, got)
            states = [got[3][got[4][s]:got[4][s] + SB].copy() for s in range(3)]
        assert want[1][0] > 0
    finally:
        for x in sts:
            up.lib.LZ4_freeStream(x)


# ---- 4. LZ4FastChainEncoder ---------------------------------------------------------------------------------------

def test_fast_chain_encoder_against_ring_model(k4, up):
    from k4os.compression.lz4_b200 import LZ4FastChainEncoder
    rng = np.random.default_rng(23)
    for bs in (1024, 4096, 65536, 256 << 10, 1 << 20, 4 << 20):
        for extra in (0, 1, 3):
            if bs >= (1 << 20) and extra == 3:
                continue
            for allow in (False, True):
                data = _datagen(int(3.5 * bs) + 70000, bs + extra).tobytes()
                data = data[:len(data) // 2] + rng.integers(0, 256, 5000, dtype=np.uint8).tobytes() + data[len(data) // 2:]
                enc, ring = LZ4FastChainEncoder(bs, extra), ER.RingModel(up, bs, extra)
                cap = _bound(enc.BlockSize)
                o = 0
                try:
                    while o < len(data):
                        k = int(rng.integers(1, enc.BlockSize + 1)) if rng.random() < 0.7 else enc.BlockSize
                        a = enc.Topup(data[o:o + k])
                        assert ring.topup(data[o:o + k]) == a
                        o += a
                        if enc.BytesReady == enc.BlockSize or rng.random() < 0.3 or o >= len(data):
                            t = np.full(cap, 0xCD, dtype=np.uint8)
                            r = enc.Encode(t, allow)
                            rr, out, _, _, after = ring.encode(cap, allow)
                            assert r == rr and t[:abs(r)].tobytes() == out, (bs, extra, allow, o)
                            assert (t[abs(r):] == 0xCD).all()
                            assert np.array_equal(enc._state, after), (bs, extra, allow, o)
                finally:
                    ring.close()


def test_encode_many_equals_alone(k4):
    from k4os.compression.lz4_b200 import LZ4FastChainEncoder
    rng = np.random.default_rng(31)
    N_ = 64
    many = [LZ4FastChainEncoder(65536, i % 3) for i in range(N_)]
    alone = [LZ4FastChainEncoder(65536, i % 3) for i in range(N_)]
    datas = [_datagen(300000, 500 + i).tobytes() for i in range(N_)]
    pos = [0] * N_
    for step in range(6):
        targets = [np.zeros(_bound(65536), dtype=np.uint8) for _ in range(N_)]
        for i in range(N_):
            k = int(rng.integers(1, 65537))
            a = many[i].Topup(datas[i][pos[i]:pos[i] + k])
            assert alone[i].Topup(datas[i][pos[i]:pos[i] + k]) == a
            pos[i] += a
        res = LZ4FastChainEncoder.EncodeMany(many, targets, True)
        for i in range(N_):
            t = np.zeros(_bound(65536), dtype=np.uint8)
            r = alone[i].Encode(t, True)
            assert r == res[i] and t[:abs(r)].tobytes() == targets[i][:abs(r)].tobytes(), (step, i)
            assert np.array_equal(alone[i]._state, many[i]._state)


def test_high_entropy_repeated(k4):
    """LZ4EncoderTests.HighEntropyRepeated (LZ4EncoderTests.cs:85-99)."""
    from k4os.compression.lz4_b200 import LZ4FastChainEncoder
    src = np.random.default_rng(0).integers(0, 256, 256, dtype=np.uint8).tobytes()
    enc = LZ4FastChainEncoder(256)
    target = np.zeros(1024, dtype=np.uint8)
    assert enc.Topup(src) == 256
    assert enc.Encode(target, True) == -256
    assert enc.Topup(src) == 256
    assert 0 < enc.Encode(target, True) < 32


# ---- 5. frames ------------------------------------------------------------------------------------------------------

def test_write_frames_linked(k4, up):
    import oracle
    from k4os.compression.lz4_b200 import frame as F
    ref = oracle.Ref()
    rng = np.random.default_rng(41)
    for bsz in (1 << 16, 1 << 18, 1 << 20, 1 << 22):
        contents = []
        for j in range(5):
            n = [0, 1000, bsz, 2 * bsz + 12345, 3 * bsz + 7][j] if bsz < (1 << 22) else [0, 1000, 9_000_000, bsz, 5_000_000][j]
            c = _datagen(n, bsz + j).copy()
            if n > 200000:
                at = int(rng.integers(0, n - 150000))
                c[at:at + 150000] = rng.integers(0, 256, 150000, dtype=np.uint8)   # incompressible: raw blocks
            contents.append(c.tobytes())
        for bc in (False, True):
            for cc in (False, True):
                frames = F.write_frames(contents, bsz, bc, cc)
                for c, f in zip(contents, frames):
                    assert f == ER.frame_linked_ref(up, c, bsz, bc, cc), (bsz, bc, cc, len(c))
                    assert ref.frame_decompress(f, len(c) + 16) == c
                    assert (f[4] >> 5) & 1 == 0
                assert F.read_frames(frames) == contents
        assert F.write_frame(contents[3], bsz, chaining=True) == F.write_frames([contents[3]], bsz)[0]
    raws = sum(F._Frame(f).raws.count(True) for f in F.write_frames([contents[3]], 1 << 16))
    assert raws > 0


# ---- 6. path counters -----------------------------------------------------------------------------------------------

def test_path_counters(k4):
    B = k4.batch
    B.encode_stats(0, reset=True)
    items = [(b"", _datagen(n, n).tobytes(), _bound(n), ER.make_state()) for n in (100, 65536, 70000, 1 << 20)]
    items.append((b"", b"", 16, ER.make_state()))
    out = run_device(k4, items)[0]
    assert out[-1] == 0
    st = B.encode_stats(0, reset=True)
    assert (st["smem"], st["gtab"], st["generic"], st["chain"]) == (0, 0, 0, 4), st
    out = run_device(k4, items[:2], level=3)[0]
    assert list(out) == [-2, -2] and B.encode_stats(0, reset=True)["chain"] == 0
    blocks = [_datagen(65536, 9 + i).tobytes() for i in range(8)] + [_datagen(100000, 1).tobytes()]
    B.encode_batch_host(blocks)
    st = B.encode_stats(0, reset=True)
    assert st["chain"] == 0 and st["smem"] + st["gtab"] == 8 and st["generic"] == 1, st
