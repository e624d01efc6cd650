"""The block decoders on mutated full-size blocks (tests/block_mutants.py), against the oracle.

Real 64 KiB blocks with fields rewritten in place stay on the tile kernel and decode to different content; rewrites
to the accept boundary pin its test deep in a block; chain-breaking mutations check that the tile path hands blocks
over to the exact engine untouched.  Every independent and chained case runs through the device path at random
16-byte source and destination phases and asserts
  * the return code, and the bytes where it is positive, equal the authority's (``oracle.Port`` for independent
    blocks, ``chain_ref.decompress_prefix`` behind a history; content is not compared for offset-0 streams);
  * every 0xCD sentinel outside [slot, slot + rc) is intact (for a rejected block: outside the slot), and the
    history in front of a chained slot is unchanged;
  * the path counters (tile, tile_big, generic) equal the routing model's count, engine by engine, per launch.
Chain decoder groups decode streams whose blocks are sometimes replaced by mutants, against a per-stream history;
the exact engine's dictionary and partial decodes take mutants whose offsets reach into the dictionary or whose
target sits at the rewritten sequence."""
import collections
import time

import numpy as np
import pytest

from tests import block_mutants as BM
from tests import chain_ref as CR
from tests import inputs
from tests.test_gpu_chain import run_chain_device
from tests.test_gpu_chain_group import group_call
from tests.test_gpu_edges import _compare, _run_device

pytestmark = pytest.mark.gpu
K64 = 65536


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
def up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return CR.Upstream()


def _report(family, eng, t0):
    print(f"\n[{family}] {dict(eng)} in {time.time() - t0:.1f} s")


def test_independent_block_mutants(k4, port):
    """~8 000 independent mutants (k4lz4_decode_batch), caps exact + {0, 1, 5, 13, 32}, 65 536 and exact - 1, in two
    launches, the first of more than 4 224 blocks; then a host-memory call over a slice gives the same results."""
    t0 = time.time()
    cases = BM.independent_cases()
    rng = np.random.default_rng(41)
    order = rng.permutation(len(cases))
    expect, engines = [], []
    for m, cap, ph in cases:
        r, ref = port.decode(m.stream, cap)
        if r > 0 and m.kind == "tail":
            assert r == m.size
        expect.append((r, None if r > 0 and inputs.uses_zero_offset(m.stream) else ref))
        e = BM.route(m.parse(), len(m.stream), cap, ph)
        assert not (e.startswith("tile") and r <= 0), "the model sends a rejected block to the tile path"
        engines.append(e)
    total = collections.Counter()
    for part in (order[:4500], order[4500:]):
        streams = [cases[i][0].stream for i in part]
        caps = [cases[i][1] for i in part]
        sph = [cases[i][2] for i in part]
        got, dst, doff, st = _run_device(k4, False, streams, caps, sph, rng.integers(0, 16, len(part)))
        _compare(got, dst, doff, caps, [expect[i] for i in part])
        eng = collections.Counter(engines[i] for i in part)
        assert (st["tile"], st["tile_big"], st["generic"]) == (eng["tile"], eng["tile_big"], eng["generic"]), \
            (st, dict(eng))
        total += eng
    assert len(order[:4500]) > 4224
    sl = order[::13]
    dec, out = k4.batch.decode_batch_host([cases[i][0].stream for i in sl], [cases[i][1] for i in sl])
    for k, i in enumerate(sl):
        r, ref = expect[i]
        assert int(out[k]) == r and (r <= 0 or ref is None or dec[k] == ref), (i, int(out[k]), r)
    _report("independent", total, t0)


def _check_chained(k4, up, cases, rng, tenth):
    """One device launch of (stream, cap, history) cases at random phases, against decompress_prefix (and upstream
    on every tenth case) -> per-engine counts."""
    triples = [(m.stream, cap, h) for m, cap, h in cases]
    sph, dph = rng.integers(0, 16, len(cases)), rng.integers(0, 16, len(cases))
    got, dst, before, doff, stats = run_chain_device(k4, triples, sph, dph)
    want, mask = before.copy(), np.ones(dst.shape, dtype=bool)
    eng = collections.Counter()
    for i, ((m, cap, h), ph) in enumerate(zip(cases, sph)):
        r, ref = CR.decompress_prefix(m.stream, cap, h)
        if (tenth + i) % 10 == 0:
            assert up.decode_prefix(m.stream, cap, h)[0] == r, (m.base.name, m.kind, m.seq, len(h))
        assert int(got[i]) == r, (i, m.base.name, m.kind, m.seq, cap, len(h), int(got[i]), r)
        e = BM.route(m.parse(), len(m.stream), cap, int(ph), len(h))
        assert not (e.startswith("tile") and r < 0), "the model sends a rejected block to the tile path"
        if e != "trivial":
            eng[e] += 1
        o = int(doff[i])
        if r > 0 and not inputs.uses_zero_offset(m.stream):
            want[o:o + r] = np.frombuffer(ref, dtype=np.uint8)
        elif r > 0:
            mask[o:o + r] = False
        elif r < 0:
            mask[o:o + max(cap, 0)] = False
    bad = np.nonzero((dst != want) & mask)[0]
    assert len(bad) == 0, f"{len(bad)} bytes differ, first at {int(bad[0])}"
    assert (stats["tile"], stats["tile_big"], stats["generic"]) == (eng["tile"], eng["tile_big"], eng["generic"]), \
        (stats, dict(eng))
    return eng


def test_chained_block_mutants(k4, up):
    """Upstream's chained blocks behind P = 0, 1, 7, 4 096, 65 534, 65 535, 65 536 and 131 072 bytes of history
    (k4lz4_decode_chain_batch), offset-rewritten -- the boundary op + lit + P and one past it in steps >= 1, half of
    the random offsets reaching into the history -- and end-rule tails behind a history; one launch per P."""
    t0 = time.time()
    rng = np.random.default_rng(42)
    by_p = collections.defaultdict(list)
    for c in BM.chained_cases():
        by_p[len(c[2])].append(c)
    total, k = collections.Counter(), 0
    for P in sorted(by_p):
        total += _check_chained(k4, up, by_p[P], rng, k)
        k += len(by_p[P])
    assert total["tile"] + total["tile_big"] >= 0.5 * k and total["tile_big"] > 0 and total["generic"] > 0, total
    _report("chained", total, t0)


def _group_mutant(rng, block: bytes, hist_len: int, B: int):
    """-> (block or a mutant of it, 'valid' / 'invalid' / 'block'), the kind the mutation aims at; the authority
    decides.  Valid: an offset in range, a shorter match, new literals, or a longer match while the block stays
    within B bytes; invalid: an offset one past the history, a truncated block or a 0xFF token."""
    pa = BM.parsed(block)
    if pa.N < 3:
        return block, "block"
    i = int(rng.integers(0, pa.N - 1))
    d = int(pa.op()[i] + pa.lit[i])
    k = int(rng.integers(0, 8))
    reach = min(d + hist_len, 65535)
    if k <= 1 and reach >= 1:
        return BM.set_offset(block, i, int(rng.integers(max(reach - 2000, 1), reach + 1)))[0], "valid"
    if k == 2 and pa.ml[i] > BM.MINMATCH and pa.ml[i] < 15 + BM.MINMATCH:
        return BM.set_match_len(block, i, BM.MINMATCH)[0], "valid"
    if k == 3 and pa.lit[i] > 0:
        return BM.set_literals(block, i, BM.LB._rb(rng, int(pa.lit[i])))[0], "valid"
    if k == 4 and pa.ml[i] < 4 + BM.MINMATCH:
        return BM.set_match_len(block, i, int(pa.ml[i]) + 10)[0], "valid" if pa.size + 10 <= B - 5 else "invalid"
    if k == 5 and d + hist_len + 1 <= 65535:
        return BM.set_offset(block, i, d + hist_len + 1)[0], "invalid"
    if k == 6:
        return block[:int(rng.integers(1, len(block)))], "invalid"
    m = bytearray(block)
    m[int(pa.tp[i])] = 0xFF
    return bytes(m), "invalid"


def test_chain_decoder_group_with_mutants(k4, up):
    """256 streams x 8 linked 64 KiB blocks through a ChainDecoderGroup whose blockSize leaves room to grow; in about a
    third of the steps a stream gets a mutant instead of its block.  Valid mutants change the stream's content and
    size, so later blocks decode against the changed history; invalid ones fail and leave the stream as it was.
    Calls alternate host and device memory; the authority is decompress_prefix behind a per-stream history that
    grows only on success, and every stream's history() equals it at the end."""
    import oracle
    t0 = time.time()
    S, NB, B = 256, 8, K64 + 4096
    rng = np.random.default_rng(43)
    raw = oracle.Port().datagen(S * NB * K64, 0.63, 0.0, 4343)
    comp = [up.encode_chain(raw[s * NB * K64:(s + 1) * NB * K64].tobytes()) for s in range(S)]
    hist = [b""] * S
    kinds = collections.Counter()
    eng = collections.Counter()
    with k4.ChainDecoderGroup(S, B) as g:
        for step in range(NB):
            blocks, what = [], []
            for s in range(S):
                if rng.random() < 1 / 3:
                    b, w = _group_mutant(rng, comp[s][step], len(hist[s]), B)
                else:
                    b, w = comp[s][step], "block"
                blocks.append(b); what.append(w)
            mem = "host" if step % 2 == 0 else "device"
            k4.batch.decode_stats(0, reset=True)
            out, got = group_call(k4, g, list(range(S)), blocks, [B] * S, mem)
            st = k4.batch.decode_stats(0, reset=True)
            for e in ("tile", "tile_big", "generic"):
                eng[e] += st[e]
            for s in range(S):
                r, ref = CR.decompress_prefix(blocks[s], B, hist[s][-K64:])
                assert int(out[s]) == r, (step, s, what[s], int(out[s]), r)
                if r > 0 and not inputs.uses_zero_offset(blocks[s]):
                    assert got[s] == ref, (step, s, what[s])
                if r >= 0:
                    hist[s] = (hist[s] + ref)[-K64:]
                kinds[(what[s], r >= 0)] += 1
        for s in range(S):
            assert g.history(s) == hist[s], s
    assert kinds[("valid", True)] >= 100 and kinds[("invalid", False)] >= 50, kinds
    assert eng["tile"] + eng["tile_big"] > 0, eng
    _report("group", eng, t0)


def _dict_cases(rng):
    """64 KiB mutants whose offsets reach exactly op + lit + dictLen, one past it, and randomly into the dictionary,
    with dictionaries of 0, 1, 4 095, 65 535, 65 536 and 70 000 bytes -> [(stream, cap, dict)]."""
    out = []
    for L in (0, 1, 4095, 65535, 65536, 70000):
        dic = inputs.gen("text2" if L % 2 else "lowent", L, L + 1)
        for base in BM.independent_bases():
            pa, s = base.pa, base.stream
            for i in BM.target_seqs(pa, len(s), per_segment=1):
                d = int(pa.op()[i] + pa.lit[i])
                vals = [d + L, d + L + 1] + [int(rng.integers(d + 1, min(d + L, 65535) + 1)) for _ in range(2)
                                             if L and d < 65535]
                for v in vals:
                    if 1 <= v <= 65535:
                        m, z = BM.set_offset(s, i, v)
                        out.append((m, z + (0, 5, 32)[len(out) % 3], dic))
    return out


def _partial_cases(rng):
    """Offset and match-length mutants with partial-decode targets at the rewritten sequence's output position
    -1, +0 and +1, and at step boundaries -> [(stream, target)]."""
    out = []
    for base in BM.independent_bases():
        for m in BM.layout_mutants(base, rng, full=False):
            if m.seq < 0 or m.seq >= m.pa.N - 1:
                continue
            op = m.pa.op()
            d = int(op[m.seq] + m.pa.lit[m.seq])
            steps = [int(op[k]) for k in range(BM.DT_K, m.pa.N, BM.DT_K)]
            tg = [d - 1, d, d + 1] + steps[:1]
            out.append((m.stream, max(tg[len(out) % len(tg)], 0)))
    return out


def _device_exact(k4, fn, streams, caps, dicts=None, gap=32):
    """k4lz4_decode_dict_batch (dicts given) or k4lz4_partial_decode_batch with device memory at random phases
    -> (outLen, list of slots' bytes up to outLen, sentinels intact)."""
    import torch
    N = k4._native
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(len(streams))
    src, so, sl = k4.batch._pack(streams)
    caps = np.array(caps, np.int32)
    do, pos = np.zeros(len(caps), np.int64), gap
    for i, c in enumerate(caps):
        pos = (pos + 15) // 16 * 16 + int(rng.integers(0, 16))
        do[i] = pos
        pos += max(int(c), 0) + gap
    dst = torch.full((pos + gap,), 0xCD, dtype=torch.uint8, device=dev)
    t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (src, so, sl, do, caps)]
    out = torch.full((len(caps),), -7, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    if dicts is not None:
        dic, dof, dl = k4.batch._pack(dicts)
        td = [torch.from_numpy(a).to(dev) for a in (dic, dof, dl)]
        N.check(fn(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), dst.data_ptr(), t[3].data_ptr(), t[4].data_ptr(),
                   td[0].data_ptr(), td[1].data_ptr(), td[2].data_ptr(), out.data_ptr(), len(caps), N.MEM_DEVICE,
                   stream, 0))
    else:
        N.check(fn(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), dst.data_ptr(), t[3].data_ptr(), t[4].data_ptr(),
                   out.data_ptr(), len(caps), N.MEM_DEVICE, stream, 0))
    torch.cuda.synchronize()
    o, d = out.cpu().numpy(), dst.cpu().numpy()
    keep = np.ones(d.shape, dtype=bool)
    for i in range(len(caps)):
        keep[do[i]:do[i] + (int(o[i]) if o[i] > 0 else max(int(caps[i]), 0))] = False
    assert (d[keep] == 0xCD).all(), "a byte outside a slot's result was written"
    return o, [d[do[i]:do[i] + o[i]].tobytes() if o[i] > 0 else b"" for i in range(len(caps))]


def test_exact_engine_dictionary_and_partial_mutants(k4, port):
    """k4lz4_decode_dict_batch and k4lz4_partial_decode_batch, host and device memory, on 64 KiB mutants: offsets at
    op + lit + dictLen, one past it and inside the dictionary; partial targets around the rewritten sequence."""
    t0 = time.time()
    rng = np.random.default_rng(44)
    L = k4._native.lib()
    dc = _dict_cases(rng)
    want = [port.decode_dict(s, c, d) if d else port.decode(s, c) for s, c, d in dc]
    assert sum(r > 0 for r, _ in want) >= 0.5 * len(dc) and sum(r < 0 for r, _ in want) >= 100
    for mem in ("host", "device"):
        if mem == "host":
            dec, out = k4.batch.decode_dict_batch_host([s for s, _, _ in dc], [c for _, c, _ in dc],
                                                       [d for _, _, d in dc])
        else:
            out, dec = _device_exact(k4, L.k4lz4_decode_dict_batch, [s for s, _, _ in dc], [c for _, c, _ in dc],
                                     [d for _, _, d in dc])
        for i, ((s, c, d), (r, ref)) in enumerate(zip(dc, want)):
            assert int(out[i]) == r, (mem, i, len(d), int(out[i]), r)
            assert r <= 0 or inputs.uses_zero_offset(s) or dec[i] == ref, (mem, i, len(d))
    pc = _partial_cases(rng)
    want = [port.partial_decode(s, t) for s, t in pc]
    assert sum(r > 0 for r, _ in want) >= 0.5 * len(pc)
    for mem in ("host", "device"):
        if mem == "host":
            dec, out = k4.batch.partial_decode_batch_host([s for s, _ in pc], [t for _, t in pc])
        else:
            out, dec = _device_exact(k4, L.k4lz4_partial_decode_batch, [s for s, _ in pc], [t for _, t in pc])
        for i, ((s, t), (r, ref)) in enumerate(zip(pc, want)):
            assert int(out[i]) == r, (mem, i, t, int(out[i]), r)
            assert r <= 0 or inputs.uses_zero_offset(s) or dec[i] == ref, (mem, i, t)
    _report("dict/partial", {"dict": len(dc), "partial": len(pc)}, t0)
