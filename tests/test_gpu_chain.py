"""GPU tests of chained (linked) blocks: k4lz4_decode_chain_batch, LZ4ChainDecoder and linked frames.

Every hand-built case runs through the device path at chosen 16-byte source / destination phases with the
stream's history directly in front of the destination, and asserts
  * the return code, and the bytes where it is >= 0, equal the prefix-mode restatement's (tests/chain_ref.py),
    which is pinned against upstream's LZ4_decompress_safe_continue by tests/test_chain_model.py;
  * the history bytes and every 0xCD sentinel outside [slot, slot + return code) are unchanged (for a
    rejected block: outside the slot);
  * the decoder's path counters equal what the routing model with a history (chain_ref.tile_route_p)
    predicts, engine by engine.
Streams from upstream's chained encoder and upstream's linked frames need the reference engine that
__graft_entry__.build() compiles into oracle/_ref/."""
import collections

import numpy as np
import pytest

from tests import chain_ref as CR
from tests import inputs
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
GOLD = ROOT + "/tests/golden/"


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
    return CR.Upstream()


def run_chain_device(k4, cases, src_ph, dst_ph, gap=48):
    """cases: (stream, cap, history).  One device launch; slot i = [history | cap] with the destination at
    phase dst_ph[i].  -> (outLen, dst bytes, dst offsets, stats)."""
    import torch
    dev = torch.device("cuda", 0)
    n = len(cases)
    soff, pos = [], 16
    for (s, _, _), ph in zip(cases, src_ph):
        pos = (pos + 15) // 16 * 16 + int(ph)
        soff.append(pos)
        pos += len(s) + 16
    src = np.zeros(pos + 16, dtype=np.uint8)
    for o, (s, _, _) in zip(soff, cases):
        src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    doff, pos = [], gap
    for (_, cap, h), ph in zip(cases, dst_ph):
        pos = (pos + len(h) + 15) // 16 * 16 + int(ph)
        doff.append(pos)
        pos += max(cap, 0) + gap
    dst = np.full(pos + gap, 0xCD, dtype=np.uint8)
    for o, (_, _, h) in zip(doff, cases):
        dst[o - len(h):o] = np.frombuffer(h, dtype=np.uint8)
    t_src, t_dst = torch.from_numpy(src).to(dev), torch.from_numpy(dst).to(dev)
    t_soff = torch.tensor(soff, dtype=torch.int64, device=dev)
    t_doff = torch.tensor(doff, dtype=torch.int64, device=dev)
    t_len = torch.tensor([len(s) for s, _, _ in cases], dtype=torch.int32, device=dev)
    t_cap = torch.tensor([c for _, c, _ in cases], dtype=torch.int32, device=dev)
    t_pre = torch.tensor([len(h) for _, _, h in cases], dtype=torch.int32, device=dev)
    t_out = torch.full((n,), -7, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    k4.batch.decode_stats(0, reset=True)
    k4.batch.decode_chain_batch_device(t_src.data_ptr(), t_soff.data_ptr(), t_len.data_ptr(), t_dst.data_ptr(),
                                       t_doff.data_ptr(), t_cap.data_ptr(), t_pre.data_ptr(), t_out.data_ptr(), n, st)
    torch.cuda.synchronize()
    return t_out.cpu().numpy(), t_dst.cpu().numpy(), dst, np.array(doff), k4.batch.decode_stats(0, reset=True)


def check_cases(k4, cases, src_ph, dst_ph):
    got, dst, before, doff, stats = run_chain_device(k4, cases, src_ph, dst_ph)
    want, mask = before.copy(), np.ones(dst.shape, dtype=bool)
    engines = collections.Counter()
    memo, routes = {}, {}
    for i, ((s, cap, h), ph) in enumerate(zip(cases, src_ph)):
        key = (s, cap, h)
        if key not in memo:
            memo[key] = CR.decompress_prefix(s, cap, h)
        r, ref = memo[key]
        assert int(got[i]) == r, (i, int(got[i]), r, len(h))
        if (key, int(ph)) not in routes:
            routes[(key, int(ph))] = CR.tile_route_p(s, cap, len(h), int(ph))
        e = routes[(key, int(ph))]
        assert not (e.startswith("tile") and r < 0), "the model sends a rejected block to the tile path"
        if e != "trivial":
            engines[e] += 1
        o = int(doff[i])
        if r > 0 and not inputs.uses_zero_offset(s):
            want[o:o + r] = np.frombuffer(ref, dtype=np.uint8)
        elif r > 0:
            mask[o:o + r] = False
        elif r < 0:
            mask[o:o + max(cap, 0)] = False
    bad = np.nonzero((dst != want) & mask)[0]
    assert len(bad) == 0, f"{len(bad)} bytes differ, first at {int(bad[0])}"
    assert (stats["tile"], stats["tile_big"], stats["generic"]) == \
        (engines["tile"], engines["tile_big"], engines["generic"]), (stats, engines)


def test_issue64_known_answer(k4):
    """The reference's golden vector: block #1 of assets/issue64 decodes only behind block #0's output."""
    b0 = open(GOLD + "issue64_block0.bin", "rb").read()
    b1z = open(GOLD + "issue64_block1.lz4", "rb").read()
    b1 = open(GOLD + "issue64_block1.bin", "rb").read()
    assert len(b0) == 65536
    assert CR.decompress_prefix(b1z, 65536, b0) == (len(b1), b1)
    check_cases(k4, [(b1z, 65536, b0), (b1z, 65536, b0[-65535:]), (b1z, 65536, b"")], [0, 3, 7], [0, 9, 15])
    # host memory: the history is staged in front of the device slot
    dst = np.zeros(2 * 65536 + 64, dtype=np.uint8)
    dst[:65536] = np.frombuffer(b0, dtype=np.uint8)
    src = np.frombuffer(b1z, dtype=np.uint8)
    out = k4.batch.decode_chain_batch_host(src, [0], [len(b1z)], dst, [65536], [65536], [65536])
    assert int(out[0]) == len(b1) and dst[65536:65536 + len(b1)].tobytes() == b1
    assert dst[:65536].tobytes() == b0


def _filler(rng, n_seq):
    """n_seq short sequences that stay inside the block (1 literal, a 4..8-byte match 5..40 back)."""
    seqs = [(rng.integers(0, 256, 48, dtype=np.uint8).tobytes(), 7, 8)]
    for _ in range(n_seq - 1):
        seqs.append((rng.integers(0, 256, 1, dtype=np.uint8).tobytes(), int(rng.integers(5, 40)),
                     int(rng.integers(4, 9))))
    return seqs


def _out_len(seqs):
    return sum(len(l) + m for l, _, m in seqs)


def hand_cases():
    """(name, stream, cap, history) -- the families of the history window."""
    rng = np.random.default_rng(64)
    rb = lambda k: rng.integers(0, 256, k, dtype=np.uint8).tobytes()
    out = []
    hist = rb(70000)
    for P in (1, 16, 300, 4096):
        h = hist[-P:]
        for L in (0, 3):                                     # offset == op + lit + P: accepted; + 1: rejected
            for ml in (4, 20, 33, 100):
                s, d = CR.build_prefix_block(h, [(rb(L), P + L, ml), (rb(2), 5, 6)], rb(12))
                out.append((f"off=P P{P} L{L} ml{ml}", s, len(d), h))
                m = bytearray(s)
                at = 1 + L
                m[at:at + 2] = (P + L + 1).to_bytes(2, "little")
                out.append((f"off=P+1 P{P} L{L} ml{ml}", bytes(m), len(d) + 64, h))
    h = hist[-5000:]
    for ml in (5, 31, 32, 33, 64, 500):                       # history parts both sides of DT_LSHORT, straddling too
        for back in (ml, ml // 2 + 1, 1):
            s, d = CR.build_prefix_block(h, [(rb(6), 6 + back, ml), (rb(1), 3, 4)], rb(12))
            out.append((f"hist ml{ml} back{back}", s, len(d), h))
    # straddling with off < ml (the remainder reads its own history part), step 0
    for ml, back in ((40, 3), (200, 17), (1000, 100), (36, 35)):
        s, d = CR.build_prefix_block(h, [(rb(2), 2 + back, ml)], rb(12))
        out.append((f"periodic step0 ml{ml} back{back}", s, len(d), h))
    # later steps (> 512 sequences before, Sr ~ 3.6 KB and ~ 7.2 KB): far remainders (shorter than Sr) and near
    # remainders (longer than Sr, with off < remainder: periodic, reading their own history part)
    for n_fill, back, ml in ((600, 10, 30), (600, 40, 5000), (1100, 5, 9000), (1100, 64, 2500)):
        seqs = _filler(rng, n_fill)
        o = _out_len(seqs)
        seqs.append((b"", o + back, ml))
        seqs.append((rb(1), 3, 4))
        s, d = CR.build_prefix_block(h, seqs, rb(12))
        out.append((f"later fill{n_fill} back{back} ml{ml}", s, len(d), h))
    # offset 65535 at output position 0 with every kind of history length
    for P in (0, 1, 65534, 65535, 65536):
        hh = hist[len(hist) - P:]
        for L in (0, 1, 2):
            lit = rb(L)
            if 65535 <= L + P:
                s, d = CR.build_prefix_block(hh, [(lit, 65535, 24)], rb(12))
                cap = len(d)
            else:
                s, _ = CR.build_prefix_block(hist[-65535:], [(lit, 65535, 24)], rb(12))
                cap = 64
            out.append((f"off65535 P{P} L{L}", s, cap, hh))
    return out


def test_history_window_all_phases(k4):
    """Every hand-built case at all 16 x 16 source / destination phases, in one launch per source phase."""
    cases = hand_cases()
    assert sum(1 for n, s, c, h in cases if CR.decompress_prefix(s, c, h)[0] < 0) >= 20
    assert sum(1 for n, s, c, h in cases if CR.tile_route_p(s, c, len(h)) == "tile") >= 60
    for sp in range(16):
        batch = [(s, c, h) for _ in range(16) for _, s, c, h in cases]
        dph = [dp for dp in range(16) for _ in cases]
        check_cases(k4, batch, [sp] * len(batch), dph)


def _chained_streams(up, S, B, seed=1234):
    import oracle
    raw = oracle.Port().datagen(S * B * 65536, 0.63, 0.0, seed)
    comp = [up.encode_chain(raw[s * B * 65536:(s + 1) * B * 65536].tobytes()) for s in range(S)]
    return raw, comp


def test_many_streams_linked_blocks(k4, up):
    """1 024 streams x 4 linked 64 KiB blocks from upstream's chained encoder: one device call per step
    decodes block k of every stream behind its earlier output; byte-identical to the input, every block on the
    tile path."""
    import torch
    S, B, BS = 1024, 4, 65536
    raw, comp = _chained_streams(up, S, B)
    dev = torch.device("cuda", 0)
    out = torch.full((S * B * BS,), 0xCD, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    k4.batch.decode_stats(0, reset=True)
    lens = []
    for k in range(B):
        blocks = [comp[s][k] for s in range(S)]
        ln = np.array([len(b) for b in blocks], dtype=np.int32)
        so = np.zeros(S, dtype=np.int64)
        so[1:] = np.cumsum(ln[:-1])
        t_src = torch.from_numpy(np.frombuffer(b"".join(blocks), dtype=np.uint8).copy()).to(dev)
        t_so, t_ln = torch.from_numpy(so).to(dev), torch.from_numpy(ln).to(dev)
        t_do = torch.arange(S, dtype=torch.int64, device=dev) * (B * BS) + k * BS
        t_cap = torch.full((S,), BS, dtype=torch.int32, device=dev)
        t_pre = torch.full((S,), k * BS, dtype=torch.int32, device=dev)
        t_out = torch.full((S,), -7, dtype=torch.int32, device=dev)
        k4.batch.decode_chain_batch_device(t_src.data_ptr(), t_so.data_ptr(), t_ln.data_ptr(), out.data_ptr(),
                                           t_do.data_ptr(), t_cap.data_ptr(), t_pre.data_ptr(), t_out.data_ptr(), S, st)
        torch.cuda.synchronize()
        lens.append(t_out.cpu().numpy())
    stats = k4.batch.decode_stats(0, reset=True)
    assert all((l == BS).all() for l in lens)
    assert np.array_equal(out.cpu().numpy(), raw)
    assert stats["tile"] + stats["tile_big"] == S * B and stats["generic"] == 0, stats
    # the blocks after the first really reach into the history, and upstream agrees on a sample
    for s in (0, 511, 1023):
        base = raw[s * B * BS:(s + 1) * B * BS].tobytes()
        for k in (1, 3):
            hist = base[(k - 1) * BS:k * BS]
            assert up.decode_prefix(comp[s][k], BS, hist) == (BS, base[k * BS:(k + 1) * BS])
            assert CR.tile_route_p(comp[s][k], BS, BS) != "generic"
    assert sum(CR.tile_route_p(comp[s][1], BS, 0) == "generic" for s in range(0, S, 64)) > 0


def _frame_content(rng, n):
    """datagen-like bytes with incompressible stretches (they become raw blocks)"""
    import oracle
    a = oracle.Port().datagen(n, 0.63, 0.0, int(rng.integers(1, 1 << 30))).copy()
    for _ in range(3):
        at = int(rng.integers(0, max(n - 70000, 1)))
        k = min(70000, n - at)
        a[at:at + k] = rng.integers(0, 256, k, dtype=np.uint8)
    return a.tobytes()


def test_linked_frames_many_per_call(k4, up):
    """Upstream's linked frames (block sizes 64 KiB .. 4 MiB, with and without block / content checksums, with
    raw blocks) read by read_frames, many frames per call, mixed with independent frames from write_frame."""
    from k4os.compression.lz4_b200 import frame as F
    rng = np.random.default_rng(5)
    frames, contents = [], []
    for size_id in (4, 5, 6, 7):
        for bc in (False, True):
            for cc in (False, True):
                n = int(rng.integers(1, 4 << (2 * size_id + 8))) if size_id < 7 else 5_000_000
                c = _frame_content(rng, n)
                frames.append(up.frame_linked(c, size_id, bc, cc))
                contents.append(c)
    for _ in range(24):                                      # many small 64 KiB-block frames in one call
        c = _frame_content(rng, int(rng.integers(70000, 400000)))
        frames.append(up.frame_linked(c, 4, bool(rng.integers(0, 2)), bool(rng.integers(0, 2))))
        contents.append(c)
    c = _frame_content(rng, 300000)
    frames.append(F.write_frame(c, 65536, True, True))
    contents.append(c)
    frames.append(up.frame_linked(b"", 4))
    contents.append(b"")
    raw_blocks, linked = 0, 0
    for f, c in zip(frames[:-2], contents):
        fr = F._Frame(f)
        assert fr.chaining == (len(c) > fr.max_block)         # upstream writes a one-block frame as independent
        linked += fr.chaining
        raw_blocks += sum(fr.raws) if fr.chaining else 0
    assert linked >= 30 and raw_blocks > 0
    assert F.read_frames(frames) == contents
    assert F.read_frame(frames[0]) == contents[0]
    bad = bytearray(frames[1])
    bad[len(bad) // 2] ^= 0x40
    with pytest.raises((F.InvalidDataException,)):
        F.read_frames([frames[0], bytes(bad)])


def test_chain_decoder_random_sequence(k4, up):
    """Eight LZ4ChainDecoders driven through seeded random Decode / Inject / Drain / Peek sequences that wrap
    their rings, with DecodeMany advancing all decoders that decode in the step by one GPU call; each equals the
    reference's class run over upstream's LZ4_decompress_safe_continue."""
    from k4os.compression.lz4_b200 import LZ4ChainDecoder
    import oracle
    rng = np.random.default_rng(11)
    D = 8
    configs = [(4096, 0), (4096, 2), (65536, 0), (20000, 1), (1024, 0), (65536, 1), (8192, 3), (30000, 0)]
    decs = [LZ4ChainDecoder(b, e) for b, e in configs]
    refs = [CR.RingModel(up, b, e) for b, e in configs]
    scripts = []
    for d in decs:
        bs = d.BlockSize
        data = oracle.Port().datagen(60 * bs + 65536, 0.63, 0.0, int(rng.integers(1, 1 << 30))).tobytes()
        st = up.lib.LZ4_createStream()
        buf = np.frombuffer(data, dtype=np.uint8)
        cap = bs + bs // 255 + 16
        tmp = np.zeros(cap, dtype=np.uint8)
        ops, at = [], 0
        try:
            while at < len(data) - bs:
                k = int(rng.integers(1, bs + 1)) if rng.random() < 0.6 else bs
                r = int(up.lib.LZ4_compress_fast_continue(st, buf.ctypes.data + at, tmp.ctypes.data, k, cap, 1))
                assert r > 0
                if rng.random() < 0.15:
                    ops.append(("inject", data[at:at + k]))
                else:
                    ops.append(("decode", tmp[:r].tobytes(), k if rng.random() < 0.5 else 0))
                at += k
        finally:
            up.lib.LZ4_freeStream(st)
        scripts.append(ops)
    try:
        steps = max(len(s) for s in scripts)
        wraps = 0
        for t in range(steps):
            batch = []
            for i, (d, r, ops) in enumerate(zip(decs, refs, scripts)):
                if t >= len(ops):
                    continue
                op = ops[t]
                if op[0] == "inject":
                    assert d.Inject(op[1]) == r.inject(op[1])
                else:
                    batch.append(i)
            if batch:
                before = [decs[i].BytesReady for i in batch]
                got = LZ4ChainDecoder.DecodeMany([decs[i] for i in batch],
                                                 [(scripts[i][t][1], scripts[i][t][2]) for i in batch])
                for i, g, b0 in zip(batch, got, before):
                    assert g == refs[i].decode(scripts[i][t][1], scripts[i][t][2])
                    wraps += decs[i].BytesReady < b0
            for d, r in zip(decs, refs):
                assert d.BytesReady == r.index and d.PrefixSize == r.prefix_size
                k = int(rng.integers(0, d.BytesReady + 1))
                assert d.Peek(-k).tobytes() == r.peek(-k)
                tgt = bytearray(k)
                d.Drain(tgt, -k, k)
                assert bytes(tgt) == r.peek(-k)
        assert wraps >= 8
        # a corrupt block: its decoder throws and stays where it was, the others advance
        d0, d1 = decs[0], decs[1]
        n0, n1 = d0.BytesReady, d1.BytesReady
        with pytest.raises(RuntimeError):
            LZ4ChainDecoder.DecodeMany([d0, d1], [b"\xf0\x01", b"\x40abcd"])
        assert d0.BytesReady in (n0, min(n0, 65536))          # Prepare may have moved the dictionary
        assert d1.BytesReady in (n1 + 4, min(n1, 65536) + 4) and d1.Peek(-4).tobytes() == b"abcd"
    finally:
        for r in refs:
            r.close()
