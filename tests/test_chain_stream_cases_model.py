"""The model of k4lz4_decode_chain_streams (tests/chain_stream_ref.py) on the adversarial stream families of
tests/stream_cases.py, against upstream's chained decoder stepped block by block.

Every family must decode exactly as upstream does, must reach its coverage target in the model's counters (which
rule of pass 2 or of the replay it exercised, and how often), and must not contain the GPU tests' fill byte.  The
last tests check that the families catch a wrong replay rule: the model run with that rule must fail.
"""
import functools

import pytest

from tests import chain_ref as CR
from tests import chain_stream_ref as SR
from tests import inputs as IN
from tests import stream_cases as SC

pytestmark = pytest.mark.skipif(not __import__("oracle").have_ref(), reason="needs the reference's C engine")

NAMES = ["history", "depth", "own-intervals", "phase-a", "phase-b-runs", "periodic", "zero-offset", "budget",
         "mutants"]


@functools.lru_cache(maxsize=None)
def _up():
    return CR.Upstream()


class _Restated:
    """chain_ref's Python restatement in Upstream's place: offset 0 writes zeros, as the kernels do"""
    decode_prefix = staticmethod(CR.decompress_prefix)


@pytest.mark.parametrize("name", NAMES)
def test_family_matches_upstream(name):
    f = SC.families()[name]
    st = SR.Stats()
    got = SR.decode_streams([(h, len(h), e) for h, e in f.streams], stats=st)
    for s, ((h, es), (ol, data)) in enumerate(zip(f.streams, got)):
        want_len, want = SR.step_reference(_up(), h, len(h), es)
        assert ol == want_len, f"{name} stream {s}: lengths"
        if f.zero_offset:
            assert any(IN.uses_zero_offset(src) for src, _, raw in es if not raw)
            want = SR.step_reference(_Restated(), h, len(h), es)[1]
        assert data == want, f"{name} stream {s}: bytes"
        assert SC.FILL not in data, f"{name} stream {s}: decodes to the fill byte"
    missed = [what for what, ok in f.target(st).items() if not ok]
    assert not missed, (name, missed, st)


def _model(name, rules):
    f = SC.families()[name]
    st = SR.Stats()
    SR.decode_streams([(h, len(h), e) for h, e in f.streams], stats=st, rules=rules)
    return f, st


@pytest.mark.parametrize("rules,name", [(SR.Rules(dep_gap=1), "phase-b-runs"), (SR.Rules(phase_a_hi=1), "phase-a")],
                         ids=["adjacent-lane-dependency-missed", "phase-a-takes-hi-1"])
def test_wrong_replay_rule_reads_a_byte_before_it_is_final(rules, name):
    """A phase-B window that misses the dependency of a lane on the lane just before it, or a phase A that takes a
    record whose source ends one byte into the block (the block's byte 0 being deferred itself): some run of copies
    then reads a byte before the record that writes it has run."""
    with pytest.raises(AssertionError, match="not final yet"):
        _model(name, rules)


def test_lane_copy_limit_is_pinned_by_the_counters():
    """A lane copy limit of 65 instead of 64 changes no byte (a lane copies a 65-byte record exactly as the warp
    does), so only the partition shows it: the 65-byte records stop being long."""
    for name, what in (("phase-a", "long phase-A records"), ("periodic", "phase-A periodic")):
        f, st = _model(name, SR.Rules(lane_copy=65))
        assert not f.target(st)[what], (name, what)
