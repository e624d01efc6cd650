"""GPU edge tests: hand-assembled blocks aimed at the tile decoder's mechanisms, and full-size encode
batches through both encoder warp kinds, against the oracle.

Every decode case runs through the device path with explicit offsets, so that the source and destination
16-byte phases are chosen, and asserts
  * the return code, and the bytes where it is > 0, equal the oracle's (``Port`` restates LL64.dec.cs and is
    the authority on malformed input; content is not compared for streams with an offset-0 match);
  * every byte of the destination buffer outside [slot, slot + return code) keeps its 0xCD sentinel -- for a
    rejected block only outside the slot, since the reference itself writes part of the output before it
    rejects;
  * the decoder's path counters for the batch equal what the routing model (tests/lz4_blocks.py) predicts for
    each block, engine by engine -- so a tile-path bug cannot hide behind the exact fallback.
Encode batches are bigger than one round of the shared-memory-table warps, so the global-table warps run
too; every block is compared with the oracle and the encoder's path counters are checked."""
import collections

import numpy as np
import pytest

from tests import inputs
from tests import lz4_blocks as LB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def port():
    import oracle
    return oracle.Port()


@pytest.fixture(scope="module")
def chk():
    import oracle
    return oracle.best()


def _layout(sizes, phases, gap):
    off, pos = [], gap
    for z, ph in zip(sizes, phases):
        pos = (pos + 15) // 16 * 16 + int(ph)
        off.append(pos)
        pos += max(int(z), 0) + gap
    return np.array(off, dtype=np.int64), pos + gap


def _run_device(k4, encode, srcs, caps, src_ph, dst_ph, gap=48):
    """One device launch over `srcs` at the given 16-byte phases -> (outLen, dst bytes, dst offsets, stats)."""
    import torch
    dev = torch.device("cuda", 0)
    n = len(srcs)
    soff, send = _layout([len(s) for s in srcs], src_ph, 16)
    src = np.zeros(send, dtype=np.uint8)
    for o, s in zip(soff, srcs):
        src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    doff, dend = _layout(caps, dst_ph, gap)
    t_src = torch.from_numpy(src).to(dev)
    t_dst = torch.full((dend,), 0xCD, dtype=torch.uint8, device=dev)
    t_soff, t_doff = torch.from_numpy(soff).to(dev), torch.from_numpy(doff).to(dev)
    t_len = torch.tensor([len(s) for s in srcs], dtype=torch.int32, device=dev)
    t_cap = torch.tensor([int(c) for c in caps], dtype=torch.int32, device=dev)
    t_out = torch.full((n,), -7, dtype=torch.int32, device=dev)
    assert t_src.data_ptr() % 16 == 0 and t_dst.data_ptr() % 16 == 0
    st = torch.cuda.current_stream().cuda_stream
    B = k4.batch
    stats = B.encode_stats if encode else B.decode_stats
    stats(0, reset=True)
    fn = B.encode_batch_device if encode else B.decode_batch_device
    args = (t_src.data_ptr(), t_soff.data_ptr(), t_len.data_ptr(), t_dst.data_ptr(), t_doff.data_ptr(),
            t_cap.data_ptr(), t_out.data_ptr(), n)
    fn(*args, 0, st) if encode else fn(*args, st)
    torch.cuda.synchronize()
    return t_out.cpu().numpy(), t_dst.cpu().numpy(), doff, stats(0, reset=True)


def _compare(got, dst, doff, caps, expect):
    """expect[i] = (return code, bytes or None = content not compared)"""
    want = np.full(dst.shape, 0xCD, dtype=np.uint8)
    mask = np.ones(dst.shape, dtype=bool)
    for i, (r, ref) in enumerate(expect):
        assert int(got[i]) == r, (i, int(got[i]), r)
        o = int(doff[i])
        if r > 0 and ref is not None:
            want[o:o + r] = np.frombuffer(ref, dtype=np.uint8)
        elif r > 0:
            mask[o:o + r] = False
        else:
            mask[o:o + max(int(caps[i]), 0)] = False
    bad = np.nonzero((dst != want) & mask)[0]
    if len(bad):
        i = int(np.searchsorted(doff, bad[0], side="right")) - 1
        pytest.fail(f"byte {int(bad[0])} differs (slot {i} at {int(doff[i])}, cap {caps[i]}, rc {int(got[i])}); "
                    f"{len(bad)} bytes in all")


def decode_case(k4, port, blocks, caps=None, src_ph=None, dst_ph=None, seed=0):
    """blocks: list of (stream, intended bytes or None); caps default to the intended size."""
    rng = np.random.default_rng(seed)
    n = len(blocks)
    streams = [s for s, _ in blocks]
    caps = [len(d) for _, d in blocks] if caps is None else list(caps)
    src_ph = rng.integers(0, 16, n) if src_ph is None else src_ph
    dst_ph = rng.integers(0, 16, n) if dst_ph is None else dst_ph
    expect, engines = [], collections.Counter()
    for (s, d), cap, ph in zip(blocks, caps, src_ph):
        r, ref = port.decode(s, cap)
        if r > 0 and d is not None:
            assert ref == d[:r]                                       # the builder and the oracle agree
        expect.append((r, None if r > 0 and inputs.uses_zero_offset(s) else ref))
        e = LB.expected_engine(s, cap, int(ph))
        assert not (e.startswith("tile") and r <= 0), "the model sends a rejected block to the tile path"
        engines[e] += 1
    got, dst, doff, st = _run_device(k4, False, streams, caps, src_ph, dst_ph)
    _compare(got, dst, doff, caps, expect)
    assert (st["tile"], st["tile_big"], st["generic"]) == (engines["tile"], engines["tile_big"], engines["generic"]), \
        (st, dict(engines))
    return engines


# ---- decode families ------------------------------------------------------------------------------------

def test_density_around_table_flip_and_limits(k4, port):
    """A: dense 3-byte sequences around the flip of pass 2 from the jump table to seq_next, at source phase
    0 and 15; N = 1, 2, 511, 512, 513, 1024; the densest clean tile block; one sequence more; > 16 384
    sequences under a large capacity."""
    rng = np.random.default_rng(1)
    blocks, caps, sph, intact = [], [], [], set()
    for ph in (0, 15):
        for n_seq in range(9358, 9372):
            s, d = LB.dense_block(n_seq, rng)
            blocks.append((s, d)); caps.append(len(d)); sph.append(ph)
            intact.add(LB.tile_route(s, len(d), ph).table_intact)
    assert intact == {True, False}
    lone = LB._rb(rng, 9)
    blocks.append(LB.build_block([], lone)); caps.append(9); sph.append(3)
    for n_seq in (2, 511, 512, 513, 1024):
        s, d = LB.dense_block(n_seq, rng)
        blocks.append((s, d)); caps.append(len(d)); sph.append(int(rng.integers(0, 16)))
    nmax = LB.densest_tile_n()
    for ph in (0, 15):
        s, d = LB.dense_block(nmax, rng, term=5)
        blocks += [(s, d), (s, d)]; caps += [len(d) + 3, len(d)]; sph += [ph, ph]
        s, d = LB.dense_block(LB.densest_tile_n(cap_slack=False), rng)
        blocks.append((s, d)); caps.append(len(d)); sph.append(ph)
        s, d = LB.dense_block(nmax + 1, rng, term=5)
        blocks.append((s, d)); caps.append(len(d) + 3); sph.append(ph)
        s, d = LB.dense_block(17000, rng, term=5)
        blocks.append((s, d)); caps.append(80000); sph.append(ph)
    eng = decode_case(k4, port, blocks, caps, src_ph=sph, seed=1)
    assert eng["tile"] >= 28 and eng["tile_big"] >= 4 and eng["generic"] >= 6, eng


def test_near_match_chains_and_step_boundaries(k4, port):
    """B: dependency chains through whole steps (starting at lane 0, 28, 31, 32, 33), long matches whose
    source spans >= 20 pending near intervals, sources that end at Sr - 1, Sr, Sr + 1."""
    rng = np.random.default_rng(2)
    blocks = [LB.chain_block(rng, 1600, skip) for skip in (0, 28, 31, 32, 33) for _ in range(3)]
    blocks += [LB.chain_block(rng, 2400, 0, lit0=1000)]
    blocks += [LB.wide_source_block(rng, k, 4) for k in (20, 30, 60)]
    blocks += [LB.step_boundary_block(rng, delta) for delta in (-1, 0, 1) for _ in range(2)]
    eng = decode_case(k4, port, blocks, seed=2)
    assert eng["generic"] == 0, eng


def test_copy_forms_at_their_thresholds(k4, port):
    """C: every offset 1..200 x lengths 4..33, 127..129, 159..161, 600 as near matches with literal runs of
    0..40; overlapping matches as far copies at the start of a step."""
    rng = np.random.default_rng(3)
    blocks = LB.copy_grid_blocks(rng)
    blocks += LB.far_overlap_blocks(rng, (1, 2, 3, 4, 7, 8, 15, 16, 31, 32, 33, 63, 64, 100, 127, 128, 159, 160,
                                          161, 199, 200), LB.COPY_LENS)
    eng = decode_case(k4, port, blocks, seed=3)
    assert eng["generic"] == 0 and eng["tile"] + eng["tile_big"] == len(blocks), eng


def test_literal_runs_across_parse_segments(k4, port):
    """D: literal runs spanning 1, 2, k parse segments (80 bytes on the small stage, 128 on the big one) +- 1,
    filled with random bytes or all 0xFF / 0xF0 / 0x0F / 0x00; one run covering nearly the whole stage."""
    rng = np.random.default_rng(4)
    blocks, sph = [], []
    for seg in (LB.SEG_SMALL, LB.SEG_BIG):
        for k in (1, 2, 5, 31, 100):
            for run in (k * seg - 1, k * seg, k * seg + 1):
                for fill in (None, 0xFF, 0xF0, 0x0F, 0x00):
                    blocks.append(LB.literal_run_block(rng, run, fill))
                    sph.append(int(rng.integers(0, 16)))
    for fill in (None, 0xFF, 0xF0, 0x0F, 0x00):
        for ph in (0, 9, 15):
            blocks.append(LB.sized_block(rng, LB.STAGE_SMALL - 16 - ph, fill)); sph.append(ph)
        blocks.append(LB.sized_block(rng, 65535, fill)); sph.append(int(rng.integers(0, 16)))
    eng = decode_case(k4, port, blocks, src_ph=sph, seed=4)
    assert eng["generic"] == 0 and eng["tile_big"] >= 5, eng


def test_every_phase_pair_and_ragged_ends(k4, port):
    """E: every (source phase, destination phase) in 16 x 16 for decoded sizes 1, 15, 16, 17, 4097, 65535 and
    65536, with cap = O and cap = O + 1 (the byte behind the output keeps its sentinel); cap = O - 1 -> -1."""
    sizes = (1, 15, 16, 17, 4097, 65535, 65536)
    enc = {z: port.encode(inputs.gen("text2" if z > 17 else "random", z, z))[1] for z in sizes}
    blocks, caps, sph, dph, zs = [], [], [], [], []
    for z in sizes:
        for sp in range(16):
            for dp in range(16):
                for cap in (z, z + 1) if (sp + dp) % 2 else (z + 1, z - 1 if z > 1 else z):
                    blocks.append((enc[z], None)); caps.append(cap); sph.append(sp); dph.append(dp); zs.append(z)
    eng = decode_case(k4, port, blocks, caps, sph, dph)
    n_short = sum(1 for c, z in zip(caps, zs) if c < z)
    assert n_short > 0 and eng["generic"] == n_short, (eng, n_short)


def test_stage_threshold_sizes(k4, port):
    """F: compressed sizes with shift + n + 16 = 40 960 (small stage) and 40 961 (big stage) for every phase;
    n = 65 535 (big stage) and 65 536 (exact decoder), literal-heavy valid blocks."""
    rng = np.random.default_rng(6)
    blocks, sph = [], []
    for ph in range(16):
        for n in (LB.STAGE_SMALL - 16 - ph, LB.STAGE_SMALL - 15 - ph):
            blocks.append(LB.sized_block(rng, n)); sph.append(ph)
    for ph in (0, 15):
        blocks.append(LB.sized_block(rng, 65535)); sph.append(ph)
        blocks.append(LB.sized_block(rng, 65536)); sph.append(ph)
    eng = decode_case(k4, port, blocks, src_ph=sph, seed=6)
    assert (eng["tile"], eng["tile_big"], eng["generic"]) == (16, 18, 2), eng


def test_big_stage_reuse_across_blocks(k4, port):
    """G: more than three big-stage blocks per persistent CTA: long 0xFF-literal blocks next to short ones (stale
    stage and tile bytes behind n), blocks with many sequences, and blocks the big-stage path declines -- before
    the steps (decoded size > 64 KiB, cap too small) and inside them (an offset reaching before the block)."""
    rng = np.random.default_rng(7)
    kinds = []
    long_ff = [LB.sized_block(rng, n, 0xFF) for n in (65535, 65000, 60001)]
    short = [LB.sized_block(rng, n) for n in (40961, 41000, 42017)]
    mixed = [port.encode(inputs.gen("random", 30000 + 1000 * i, i) + inputs.gen("text2", 35536 - 1000 * i, i))
             for i in range(4)]
    mixed = [(c, None) for _, c in mixed]
    seqs = [(LB._rb(rng, 41000), 1, 4)] + [(b"", int(rng.integers(1, 40000)), 4 + int(rng.integers(0, 20)))
                                           for _ in range(1400)]
    dense = LB.build_block(seqs, LB._rb(rng, 8))
    sq = LB.parse(dense[0])
    bad_off = bytearray(dense[0])
    p = sq[900].lit_pos + sq[900].lit
    bad_off[p:p + 2] = b"\xFF\xFF"                                      # reaches before the block start
    oversize = LB.build_block([(LB._rb(rng, 41000), 7, 30000)], LB._rb(rng, 8))
    for i, k in enumerate(rng.permutation(np.arange(1001) % 7)):
        if k == 0:
            b = long_ff[i % 3]; kinds.append((b, len(b[1])))
        elif k == 1:
            b = short[i % 3]; kinds.append((b, len(b[1])))
        elif k == 2:
            b = mixed[i % 4]; kinds.append((b, 65536))
        elif k == 3:
            kinds.append((dense, len(dense[1])))
        elif k == 4:
            kinds.append(((bytes(bad_off), None), len(dense[1])))
        elif k == 5:
            kinds.append((oversize, 80000))
        else:
            b = long_ff[i % 3]; kinds.append((b, len(b[1]) - 1))           # one byte short
    blocks = [b for b, _ in kinds]
    caps = [c for _, c in kinds]
    eng = decode_case(k4, port, blocks, caps, seed=7)
    assert eng["tile_big"] >= 3 * 132 and eng["generic"] >= 3 * 143, eng


# ---- encode families ------------------------------------------------------------------------------------

def _encode_expect(chk, blocks, caps):
    out = []
    for b, cap in zip(blocks, caps):
        if len(b) == 0:
            out.append((0, None))
            continue
        r, c = chk.encode(b, cap)
        out.append((r, c) if r > 0 else (-1, None))
    return out


def test_encode_full_blocks_through_both_warp_kinds(k4, chk, port):
    """H: >= 4 224 blocks of 64 KiB in one launch -- every input kind, the survey's datagen streams, inputs that
    put the first hit of a search run at probe 64k - 1 / 64k / 64k + 1 and the last match at n - 13 / n - 12,
    and inputs full of hash / tag collisions -- interleaved with blocks of 0..13 bytes and >= 65 547 bytes, all
    byte for byte equal to the reference engine."""
    bs = 65536
    rng = np.random.default_rng(8)
    blocks = []
    for kind in inputs.KINDS:
        raw = inputs.gen(kind, 48 * bs, 17)
        blocks += [raw[i * bs:(i + 1) * bs] for i in range(48)]
    for mp in (0.55, 0.63):
        raw = port.datagen(1800 * bs, mp, 0.0, 4321)
        blocks += [raw[i * bs:(i + 1) * bs].tobytes() for i in range(1800)]
    for i in range(240):
        blocks.append(LB.probe_step_input(rng, tail=12 + i % 2, collide=i % 3 == 2))
    n_full = len(blocks)
    assert n_full >= 4224
    small = [inputs.gen("text2", z, z) for z in range(0, 14) for _ in range(4)]
    large = [inputs.gen(k, z, 5) for k in ("text2", "lowent") for z in (65547, 65548, 70000, 100000, 131072)]
    extra = small + large
    pos = sorted(rng.choice(n_full + len(extra), len(extra), replace=False))
    for p, b in zip(pos, extra):
        blocks.insert(int(p), b)
    caps = [k4.LZ4Codec.MaximumOutputSize(len(b)) for b in blocks]
    got, dst, doff, st = _run_device(k4, True, blocks, caps, [0] * len(blocks), [0] * len(blocks))
    _compare(got, dst, doff, caps, _encode_expect(chk, blocks, caps))
    assert st["smem"] > 0 and st["gtab"] > 0, st
    assert st["generic"] == len(large) and st["smem"] + st["gtab"] == len(blocks) - len(large) - 4, st


def test_encode_limited_output_through_both_warp_kinds(k4, chk):
    """I: ~300 blocks at capacities r - 2 .. r + 10 and MaximumOutputSize - 1, where r is the reference's
    full-capacity length: one launch of more than one round of blocks, return codes and bytes as the reference."""
    rng = np.random.default_rng(9)
    base = []
    for i in range(300):
        z = int(rng.choice([20, 300, 4097, 30000, 65535, 65536, int(rng.integers(1, 65537))]))
        base.append(inputs.gen(inputs.KINDS[i % len(inputs.KINDS)], z, i))
    base += [inputs.gen("text2", 70000, 1), inputs.gen("random", 65547, 2)]
    blocks, caps = [], []
    for b in base:
        r = chk.encode(b)[0]
        for cap in list(range(r - 2, r + 11)) + [k4.LZ4Codec.MaximumOutputSize(len(b)) - 1]:
            blocks.append(b); caps.append(max(cap, 1))
    assert len(blocks) > 132 * 8
    got, dst, doff, st = _run_device(k4, True, blocks, caps, rng.integers(0, 16, len(blocks)),
                                     rng.integers(0, 16, len(blocks)))
    expect = _encode_expect(chk, blocks, caps)
    _compare(got, dst, doff, caps, expect)
    assert st["smem"] > 0 and st["gtab"] > 0 and st["generic"] == 2 * 14, st
    assert sum(1 for r, _ in expect if r < 0) > 300
