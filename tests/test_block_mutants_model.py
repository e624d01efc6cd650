"""The block-mutant generator (tests/block_mutants.py) checked without a device: its rewrites keep the layout they
promise, its array parse and routing model equal the list forms of tests/lz4_blocks.py and tests/chain_ref.py, the
three CPU engines agree on its mutants, and the GPU suite built on it (tests/test_gpu_decode_mutants.py) reaches the
tile kernel, not only the exact fallback."""
import collections

import numpy as np
import pytest

from tests import block_mutants as BM
from tests import chain_ref as CR
from tests import inputs
from tests import lz4_blocks as LB


def _have_ref() -> bool:
    import oracle
    return oracle.have_ref()


def _need_ref():
    if not _have_ref():
        pytest.skip("upstream's engine (oracle/_ref/) is needed for chained blocks")


@pytest.fixture(scope="module")
def ind():
    return BM.independent_cases()


@pytest.fixture(scope="module")
def chained():
    _need_ref()
    return BM.chained_cases()


def _same(a: BM.Parsed, b: BM.Parsed) -> bool:
    return all(np.array_equal(getattr(a, f), getattr(b, f)) for f in BM.Parsed.FIELDS)


def test_layout_preserving_rewrites_keep_the_layout(ind):
    """Offset, match-length and literal rewrites keep len(stream) and every token position; the parse they report
    (and so the decoded size) is the list-form parse of the mutant."""
    rng = np.random.default_rng(1)
    by_kind = collections.defaultdict(list)
    for m, _, _ in ind:
        if m.kind != "tail" and m.seq >= 0 and m.pa is not None:
            by_kind[m.kind].append(m)
    checked = 0
    for kind, ms in sorted(by_kind.items()):
        for j in rng.choice(len(ms), min(len(ms), 12), replace=False):
            m = ms[int(j)]
            full = BM.Parsed.from_seqs(LB.parse(m.stream))
            assert len(m.stream) == len(m.base.stream), kind
            assert np.array_equal(full.tp, m.base.pa.tp), kind
            assert _same(full, m.pa), (kind, m.base.name, m.seq)
            assert m.size == sum(s.lit + s.ml for s in LB.parse(m.stream)), kind
            checked += 1
    assert len(by_kind) >= 10 and checked >= 100, (sorted(by_kind), checked)
    s = BM.independent_bases()[4].stream                            # runs: long matches
    pa = BM.parsed(s)
    i = int(np.flatnonzero(pa.ml[:-1] >= 19)[0])                     # a length-extension byte
    m, z = BM.set_match_len(s, i, int(pa.ml[i]) + 1)
    assert z == pa.size + 1 and LB.parse(m)[i].ml == pa.ml[i] + 1
    with pytest.raises(ValueError):
        BM.set_offset(s, pa.N - 1, 5)                                # the terminal sequence has no offset


def test_array_parse_and_route_restate_the_list_forms(ind):
    """parse(stream, like=base) equals lz4_blocks.parse for chain-breaking mutants of every kind; route equals
    lz4_blocks.expected_engine at the cases' caps and source phases, and chain_ref.tile_route_p with histories."""
    rng = np.random.default_rng(2)
    by_kind = collections.defaultdict(list)
    for c in ind:
        by_kind[c[0].kind.split(":")[0]].append(c)
    n = 0
    for kind, cs in sorted(by_kind.items()):
        for j in rng.choice(len(cs), min(len(cs), 6 if kind != "tail" else 3), replace=False):
            m, cap, ph = cs[int(j)]
            assert _same(BM.parse(m.stream, (m.base.stream, m.base.pa)), BM.Parsed.from_seqs(LB.parse(m.stream))), kind
            for c in (cap, m.size, m.size - 1, BM.K64):
                assert BM.route(m.parse(), len(m.stream), c, ph) == LB.expected_engine(m.stream, c, ph), (kind, c)
                for P in (1, 4096, 70000) if kind == "offset" else ():
                    assert BM.route(m.parse(), len(m.stream), c, ph, P) == CR.tile_route_p(m.stream, c, P, ph)
            n += 1
    assert n >= 60


def _authority(b, cap, h):
    return CR.decompress_prefix(b.stream, cap, h)


def _agree(r1, r2, stream):
    if r1[0] != r2[0]:
        return False
    return r1[0] <= 0 or inputs.uses_zero_offset(stream) or r1[1] == r2[1]


def test_three_engines_agree_on_independent_mutants(ind):
    """oracle.Port, upstream (oracle.Ref) and chain_ref.decompress_prefix with no history agree on return code and
    bytes for every 8th case; the accept boundary op + lit is accepted and one past it rejected wherever the cap
    holds the block."""
    import oracle
    port = oracle.Port()
    ref = oracle.Ref() if _have_ref() else None
    n_bound = collections.Counter()
    for k, (m, cap, _) in enumerate(ind):
        bound = m.kind in ("offset:boundary", "offset:boundary+1")
        if k % 8 and not bound:
            continue
        r = port.decode(m.stream, cap)
        assert _agree(r, CR.decompress_prefix(m.stream, cap), m.stream), (m.base.name, m.kind, m.seq, cap)
        if ref is not None:
            assert _agree(r, ref.decode(m.stream, cap), m.stream), (m.base.name, m.kind, m.seq, cap)
        if bound and cap >= m.size:
            assert r[0] == (m.size if m.kind == "offset:boundary" else -1), (m.base.name, m.kind, m.seq, cap)
            n_bound[m.kind] += 1
    assert n_bound["offset:boundary"] >= 40 and n_bound["offset:boundary+1"] >= 40, n_bound


def test_three_engines_agree_on_chained_mutants(chained):
    """Behind their histories, chain_ref.decompress_prefix and upstream's decoder (Upstream.decode_prefix, negative
    codes read as -1) agree on every 6th chained case; oracle.Port agrees where there is no history.  The accept
    boundary op + lit + P is accepted and one past it rejected, in steps >= 1 too."""
    import oracle
    up, port = CR.Upstream(), oracle.Port()
    steps = collections.Counter()
    valid = {}          # a base with no literal in front of its first match has no valid offset there without history
    for k, (m, cap, h) in enumerate(chained):
        bound = m.kind in ("offset:boundary", "offset:boundary+1")
        if k % 6 and not (bound and k % 2 == 0):
            continue
        r = _authority(m, cap, h)
        assert _agree(r, up.decode_prefix(m.stream, cap, h), m.stream), (m.base.name, m.kind, m.seq, cap, len(h))
        if not h:
            assert _agree(r, port.decode(m.stream, cap), m.stream)
        if bound and cap >= m.size and valid.setdefault(m.base, _authority(m.base, m.size, h)[0] == m.size):
            assert r[0] == (m.size if m.kind == "offset:boundary" else -1), (m.base.name, m.kind, m.seq, len(h))
            steps[(m.kind, min(m.seq // BM.DT_K, 2))] += 1
    for kind in ("offset:boundary", "offset:boundary+1"):
        assert steps[(kind, 0)] > 0 and steps[(kind, 1)] > 0 and steps[(kind, 2)] > 0, steps


def test_model_never_sends_a_rejected_block_to_the_tile_path(ind, chained):
    """decode_case's assert over every mutant: a block the authority rejects is never routed to tile / tile_big
    (independent: oracle.Port; chained: upstream's prefix-mode decoder, held equal to the restatement above)."""
    import oracle
    port, up = oracle.Port(), CR.Upstream()
    for m, cap, ph in ind:
        e = BM.route(m.parse(), len(m.stream), cap, ph)
        assert not (e.startswith("tile") and port.decode(m.stream, cap)[0] <= 0), (m.base.name, m.kind, m.seq, cap)
    for m, cap, h in chained:
        e = BM.route(m.parse(), len(m.stream), cap, 0, len(h))
        assert not (e.startswith("tile") and up.decode_prefix(m.stream, cap, h)[0] < 0), (m.base.name, m.kind, m.seq)


def test_coverage_floors(ind, chained):
    """The GPU file cannot drift into testing only the fallback: >= 40 % of independent cases on the tile kernel and
    >= 500 of them on the big stage; rewritten sequences in steps 0, 1 and >= 2 and the last sequence, on the tile
    path; >= 1 000 chained mutants on the tile path whose rewritten match reads the history, over >= 3 steps."""
    eng, steps = collections.Counter(), collections.Counter()
    for m, cap, ph in ind:
        e = BM.route(m.parse(), len(m.stream), cap, ph)
        eng[e] += 1
        if e.startswith("tile") and m.seq >= 0:
            steps["last" if m.seq == m.pa.N - 1 else min(m.seq // BM.DT_K, 2)] += 1
    assert eng["tile"] + eng["tile_big"] >= 0.4 * len(ind) and eng["tile_big"] >= 500, eng
    assert all(steps[k] >= 50 for k in (0, 1, 2, "last")), steps
    hist_steps = collections.Counter()
    for m, cap, h in chained:
        if m.kind == "tail" or not h:
            continue
        i, pa = m.seq, m.pa
        if int(pa.off[i]) > int(pa.op()[i] + pa.lit[i]) and BM.route(pa, len(m.stream), cap, 0, len(h)) != "generic":
            hist_steps[i // BM.DT_K] += 1
    assert sum(hist_steps.values()) >= 1000 and len(hist_steps) >= 3, hist_steps
