"""Encoding into a fixed-size destination: the sequence-level model of upstream's LZ4_compress_destSize
(tests/dest_size_ref.py) that k4lz4_encode_dest_size_batch's fill policy follows, checked against upstream lz4 on
the oracle's reference engine, and the call's argument checks.  CPU only."""
import ctypes as C

import numpy as np
import pytest

oracle = pytest.importorskip("oracle")
if not oracle.have_ref():
    pytest.skip("reference engine not built", allow_module_level=True)

from tests import dest_size_ref as D
from tests.lz4_blocks import parse

GRID_EXTRA = 48          # seeded random targets per input on top of the fixed ones


@pytest.fixture(scope="module")
def up():
    return D.Upstream()


@pytest.fixture(scope="module")
def grid(up):
    """[(kind, n, src, seqs, targets)] over every size and content of the grid."""
    out = []
    for kind in D.KINDS:
        for n in D.SIZES:
            src = D.content(kind, n, 7 + n)
            out.append((kind, n, src, parse(up.plain(src)) if n else [], D.targets(n, 11 + n, GRID_EXTRA)))
    return out


def test_model_equals_upstream_on_the_grid(up, grid):
    pairs = 0
    for kind, n, src, seqs, ts in grid:
        for t in ts:
            r, used, _ = up.dest_size(src, t)
            if r == 0:
                used = 0                                   # the library's convention where nothing is written
            assert (r, used) == D.model(seqs, n, t)[:2], (kind, n, t)
            pairs += 1
    assert pairs >= 2000, pairs


def test_every_rule_is_reached_on_both_sides_of_the_u16_limit(up, grid):
    seen = set()
    for kind, n, src, seqs, ts in grid:
        found = D.rule_targets(seqs, n)
        for rule, t in found.items():
            r, used, _ = up.dest_size(src, t)
            assert (r, used) == D.model(seqs, n, t)[:2], (kind, n, t, rule)
            seen.add((rule, n >= D.LIMIT_64K))
        for t in ts:
            rule = D.model(seqs, n, t)[2]
            if rule is not None:
                seen.add((rule, n >= D.LIMIT_64K))
        if n < D.MFLIMIT + 1:                              # no sequences: only the last run can be cut
            assert set(found) <= {4}
    assert seen == {(r, big) for r in (1, 2, 3, 4) for big in (False, True)}, sorted(seen)


def test_last_run_formula_follows_upstream_not_1_9_2(up):
    """100 000 random bytes into 4 096: upstream consumes 4 079 bytes and fills every byte; lz4 1.9.2's formula
    (the reference's unreachable branch) would consume 4 078."""
    src = D.content("random", 100000, 1)
    assert up.dest_size(src, 4096)[:2] == (4096, 4079)
    assert up.model(src, 4096)[:2] == (4096, 4079)
    assert up.model(src, 4096, D.last_cut_1_9_2)[:2] == (4095, 4078)


def test_every_result_decodes_to_the_consumed_prefix(up, grid):
    for kind, n, src, seqs, ts in grid:
        for t in ts[::3]:
            r, used, block = up.dest_size(src, t)
            if r > 0:
                assert up.decode(block, max(used, 1)) == src[:used], (kind, n, t)


def test_argument_codes_without_a_device(native):
    """check()'s order: unknown memKind, bad block count, null pointer; the same codes with and without a GPU."""
    from k4os.compression.lz4_b200 import _native as N
    keep = [np.zeros(16, dtype=np.int64) for _ in range(8)]
    real = [a.ctypes.data for a in keep]
    f = native.k4lz4_encode_dest_size_batch
    assert f(*[None] * 8, 1, 7, None, 0) == N.E_ARG                  # memKind first, even with null pointers
    assert f(*real, -1, N.MEM_HOST, None, 0) == N.E_ARG               # then the count
    assert f(*real, -1, N.MEM_DEVICE, None, 0) == N.E_ARG
    for i in range(8):                                                # then every pointer, srcUsed included
        ptrs = list(real)
        ptrs[i] = None
        assert f(*ptrs, 1, N.MEM_HOST, None, 0) == N.E_ARG, i
        assert f(*ptrs, 1, N.MEM_DEVICE, None, 0) == N.E_ARG, i
    empty = f(*[None] * 8, 0, N.MEM_HOST, None, 0)
    assert empty == (N.OK if native.k4lz4_device_count() > 0 else N.E_NODEVICE)


def test_single_call_answers_that_need_no_device(native):
    """Nothing written: result 0 and *srcSize 0; an empty source: upstream's one-byte block."""
    from k4os.compression.lz4_b200 import _native as N
    src = np.arange(100, dtype=np.uint8)
    dst = np.full(32, 0xCD, dtype=np.uint8)
    for n, t in [(100, 0), (100, -5), (-1, 100), (0x7E000001, 100), (0, 0)]:
        size = C.c_int32(n)
        assert native.k4lz4_encode_dest_size(src.ctypes.data, dst.ctypes.data, C.byref(size), t) == 0
        assert size.value == 0 and (dst == 0xCD).all()
    size = C.c_int32(0)
    assert native.k4lz4_encode_dest_size(None, dst.ctypes.data, C.byref(size), 1) == 1
    assert size.value == 0 and dst[0] == 0 and (dst[1:] == 0xCD).all()
    assert native.k4lz4_encode_dest_size(src.ctypes.data, dst.ctypes.data, None, 16) == N.E_ARG
    assert native.k4lz4_encode_dest_size(src.ctypes.data, None, C.byref(C.c_int32(10)), 16) == N.E_ARG
