"""The chain_windows cases mean what they say: the plain restatement of upstream's fast loop
(tests/chain_search_ref.py) equals upstream on every case -- result, bytes and the whole state record -- and its
event log shows that the cases reach every batch position, store pattern and check they are built for."""
import numpy as np
import pytest

from tests import chain_search_ref as SR
from tests import chain_windows as CW


@pytest.fixture(scope="module")
def engines():
    import oracle
    from tests import dict_enc_ref as DR
    from tests import enforce32_ref as E32
    if not oracle.have_ref() or not E32.have_ref32():
        pytest.fail("oracle/_ref missing: run __graft_entry__.build() where the reference is present")
    return DR.DictUpstream(), E32.EncUpstream32()


@pytest.fixture(scope="module")
def runs(engines):
    """Every case through upstream and the restatement: (cases, tight cases, upstream's results, events)."""
    up, up32 = engines
    cases = CW.family_cases(up, up32)
    ev, want, bad = SR.Events(), {}, []
    for c in cases:
        w = SR.upstream_case(up, up32, c)
        want[c.name] = w
    tight = CW.tight_cases(cases, {k: v[1] for k, v in want.items()})
    for c in tight:
        want[c.name] = SR.upstream_case(up, up32, c)
    for c in cases + tight:
        r, b, s, e = SR.run_case(c)
        ev.merge(e)
        w = want[c.name]
        if not (r == w[0] and b == w[1] and np.array_equal(s, w[2])):
            bad.append(c.name)
    return cases, tight, want, ev, bad


def test_restatement_equals_upstream(runs):
    cases, tight, want, ev, bad = runs
    assert not bad, f"{len(bad)} cases differ from upstream, first {bad[:5]}"
    assert len(cases) + len(tight) < 1500
    assert all(want[c.name][0] > 0 for c in cases)
    assert all(want[c.name][0] == 0 for c in tight)


def test_every_target_hits_in_both_layouts(runs):
    at = runs[3].at["hit"]
    for q in CW.TARGETS:
        assert (q, "first") in at and (q, "post") in at, q


def test_every_event_kind_is_reached(runs):
    ev = runs[3]
    need = {"hit": 5000, "post_hit": 200, "offset2": 200, "reject_dist": 1000, "reject_small": 1000,
            "reject_cmp": 10000, "dist_65535": 8, "lane_forward": 1000, "slot_twice": 1000, "slot_thrice": 100,
            "h2_forward": 500, "same2": 500, "end": 300, "end_committed": 300, "catchup_history": 30,
            "catchup_floor": 30, "straddle": 30, "fail_lit": 50, "fail_match": 50, "fail_last": 30}
    assert set(need) == set(SR.EVENT_KINDS)
    low = {k: (ev.count[k], v) for k, v in need.items() if ev.count[k] < v}
    assert not low, low


def test_batch_positions_are_reached(runs):
    at = runs[3].at
    lanes = set(range(32))
    # the run ends at every lane of its batch, in both layouts (lane 0 of the block's first batch is never
    # reached: a block of 13 bytes or more always has a valid probe 0), with stores before it committed
    assert {l for l, lay in at["end"] if lay == "post"} == lanes
    assert {l for l, lay in at["end"] if lay == "first"} == lanes
    assert at["end_committed"] == lanes - {0}
    # put(ip-2) read back by the post lane and by later lanes, and dropped for later lanes at every position
    assert {0, 1, 2, 3} <= at["h2_forward"] and len(at["h2_forward"]) >= 16
    assert {0, 1, 31} <= at["same2"] and len(at["same2"]) >= 16
    # in-batch forwards from near and far lanes, in both layouts
    assert {(k, lay) for k in (1, 5, 10, 15) for lay in ("first", "post")} <= at["lane_forward"]
    assert {"first", "post"} <= at["slot_thrice"]
    # 65 535 back is accepted at lanes >= 1, mid-batch and at the batch's end
    assert {1, 7, 30, 31} <= at["dist_65535"]
    # dictSmall and distance rejections mid-batch, and the post lane's rejections
    assert {l for _, l, _ in at["reject_small"]} == lanes
    assert {l for _, l, _ in at["reject_dist"]} == lanes
    assert {"prefix", "ext"} <= at["catchup_history"]
    assert at["catchup_floor"] == {"prefix", "dict", "src"}
    assert at["post_hit"] == {"h2", "table"}


def test_straddles_reach_every_phase(runs):
    """Dictionary matches whose count runs over the dictionary's end into src[0]: the count starts 4..11 bytes
    before the end (every phase of a 4-byte word and of an 8-byte one), and runs 0 to 5 bytes into the source."""
    at = runs[3].at["straddle"]
    assert {b for b, _ in at} >= set(range(4, 12))
    assert {k for _, k in at} >= set(range(0, 6))
    names = {c.name.rsplit("-", 1)[0] for c in runs[0] if c.family == "straddle"}
    assert names == {f"straddle-d{d}" for d in CW.DICT_SIZES}


def test_each_check_fails_first_somewhere(runs):
    tight = runs[1]
    for check in ("lit", "match", "last"):
        assert sum(c.name.rsplit("-", 1)[1].startswith(check) for c in tight) >= 30, check
    assert {c.ext for c in tight} == {False, True} and {c.h4 for c in tight} == {False, True}


def test_collisions_share_the_slot_with_other_bytes():
    rng = np.random.default_rng(3)
    for h4 in (False, True):
        H, unit = (CW.hash4_12, 4) if h4 else (CW.hash5_12, 8)
        for _ in range(200):
            buf = bytearray(rng.integers(0, 256, 40, dtype=np.uint8).tobytes())
            CW.collide(buf, 20, 4, rng, h4)
            assert H(buf[20:20 + unit]) == H(buf[4:4 + unit]) and buf[20:24] != buf[4:8]


def test_tight_caps_follow_the_token_walk(engines):
    """tight_caps on a block of known sequences: the first capacity of each check is one byte short of it."""
    up, _ = engines
    src = bytes(range(40)) + bytes(range(40)) + bytes(64) + bytes(range(100, 130))
    r, block = up.encode(src, b"")
    caps = CW.tight_caps(block)
    assert caps["last"] == [r - 1]
    assert caps["lit"][0] == 1 + 40 + 8 - 1
