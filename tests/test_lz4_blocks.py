"""CPU tests of the block builder and of the tile decoder's routing model (tests/lz4_blocks.py).

The builder's blocks must decode, in the restatement of LL64.dec.cs (and the reference's own engine where it
is built), to the bytes the builder says; the model must agree with what the GPU suite already proves about
the kernel's routing and must pin the boundaries it claims (densest tile block, table/descriptor collision,
stage thresholds)."""
import numpy as np
import pytest

import oracle
from tests import inputs
from tests import lz4_blocks as LB


@pytest.fixture(scope="module")
def checkers():
    out = [oracle.Port()]
    if oracle.have_ref():
        out.append(oracle.Ref())
    return out


def _decodes_to(checkers, stream, want, cap=None):
    cap = len(want) if cap is None else cap
    for c in checkers:
        r, got = c.decode(stream, cap)
        assert (r, got) == (len(want), want), (c.kind, len(stream), r, len(want))


def test_builder_length_chains():
    rng = np.random.default_rng(1)
    for L in (0, 1, 14, 15, 16, 269, 270, 271, 524, 525, 1000):
        for M in (4, 18, 19, 20, 273, 274, 275, 528, 529, 3000):
            lit = LB._rb(rng, L)
            s, d = LB.build_block([(b"abcdefgh" + lit, 8, M)], b"tail!")
            exp = bytearray(b"abcdefgh" + lit)
            for _ in range(M):
                exp.append(exp[-8])
            assert d == bytes(exp) + b"tail!"
            sq = LB.parse(s)
            assert [(q.lit, q.ml, q.off) for q in sq] == [(8 + L, M, 8), (5, 0, 0)]
            assert sq[-1].next == len(s) and not any(q.flags & LB.SQ_BAD for q in sq)
    with pytest.raises(ValueError):
        LB.build_block([(b"ab", 3, 4)])                       # reaches before the block start


def test_builder_blocks_decode_to_intended_bytes(checkers):
    rng = np.random.default_rng(2)
    blocks = [LB.dense_block(n, rng) for n in (2, 3, 511, 512, 513, 1024, 9365)]
    blocks += [LB.chain_block(rng, 1100, skip) for skip in (0, 28, 31, 32, 33)]
    blocks += [LB.wide_source_block(rng), LB.step_boundary_block(rng, -1), LB.step_boundary_block(rng, 0),
               LB.step_boundary_block(rng, 1)]
    blocks += LB.copy_grid_blocks(rng, offsets=range(1, 201, 7))
    blocks += LB.far_overlap_blocks(rng, (1, 2, 31, 32, 33, 160), (33, 128, 600))
    blocks += [LB.literal_run_block(rng, run, fill) for run in (79, 80, 81, 161, 1000) for fill in (None, 0xFF, 0x00)]
    blocks += [LB.sized_block(rng, n) for n in (20, 40944, 40945, 65535)]
    for s, d in blocks:
        _decodes_to(checkers, s, d)
        _decodes_to(checkers[:1], s, d, cap=len(d) + 64)


def test_model_says_tile_for_datagen_blocks():
    """test_datagen_blocks_encode_and_decode_gpu proves these stay on the tile path."""
    port = oracle.Port()
    bs = 65536
    for mp in (0.63, 0.55):
        raw = port.datagen(12 * bs, mp, 0.0, 1234)
        for i in range(12):
            c = port.encode(raw[i * bs:(i + 1) * bs].tobytes())[1]
            for ph in (0, 7, 15):
                assert LB.expected_engine(c, bs, ph) in ("tile", "tile_big"), (mp, i, ph)
    for kind in ("text2", "lorem", "runs", "synth525"):                  # test_tile_path_with_oversized_capacity
        c = port.encode(inputs.gen(kind, 40000, 3))[1]
        assert LB.expected_engine(c, 65537) in ("tile", "tile_big"), kind


def test_model_trivial_and_generic_routes():
    port = oracle.Port()
    assert LB.expected_engine(b"", 10) == "trivial" and LB.expected_engine(b"\x10a", 0) == "trivial"
    assert LB.expected_engine(b"\x00", 10) == "generic"                  # decodes to nothing: O == 0
    rnd = port.encode(inputs.gen("random", 65536, 1))[1]
    assert len(rnd) > 65535 and LB.expected_engine(rnd, 65536) == "generic"
    s, d = LB.build_block([(b"abcdefgh", 8, 100)], b"12345")
    O = len(d)
    assert LB.expected_engine(s, O) == "tile" and LB.expected_engine(s, O - 1) == "generic"
    assert LB.expected_engine(s[:-1], O) == "generic"                   # truncated terminal run
    s0, _ = LB.build_block([(b"abcdefgh", 8, 20), (b"x", 1, 4)], b"12345")
    z = bytearray(s0); z[9] = 0; z[10] = 0                              # offset 0 on the first match
    assert LB.expected_engine(bytes(z), 100) == "generic"


def test_densest_tile_block_and_one_sequence_more(checkers):
    """No clean block reaches DT_NMAX = 16384 sequences on the tile path: the densest has 16383 (cap with
    3 bytes of slack) or 16382 (cap == decoded size); one sequence more is declined."""
    rng = np.random.default_rng(3)
    nmax = LB.densest_tile_n()
    s, d = LB.dense_block(nmax, rng, term=5)
    r = LB.tile_route(s, len(d) + 3)
    assert (r.engine, r.n_seq, r.out) == ("tile_big", 16383, 65534) and not r.table_intact
    _decodes_to(checkers, s, d, cap=len(d) + 3)
    assert LB.expected_engine(s, len(d)) == "generic"                   # last match starts after cap - 12
    s2, d2 = LB.dense_block(LB.densest_tile_n(cap_slack=False), rng, term=8)
    assert LB.expected_engine(s2, len(d2)) == "tile_big"
    _decodes_to(checkers, s2, d2)
    for term in range(0, 8):                                            # one more sequence: never the tile path
        s3, d3 = LB.dense_block(nmax + 1, rng, term=term)
        assert LB.expected_engine(s3, 1 << 20) == "generic", term
    big, dbig = LB.dense_block(17000, rng, term=5)                             # > DT_NMAX: accepted by the reference
    rb = LB.tile_route(big, 80000)
    assert rb.engine == "generic" and rb.n_seq == 17000 and rb.n_seq > LB.DT_NMAX
    _decodes_to(checkers, big, dbig, cap=80000)


@pytest.mark.parametrize("phase", [0, 15])
def test_table_collision_flip_is_on_the_small_stage(phase):
    """Pass 2 walks the jump table while shift + n + 4 + 4N <= 65 568 and falls back to seq_next above
    (decode_tile.cuh:477); dense 3-byte sequences flip it at N ~ 9 365 with the block still on the small stage."""
    rng = np.random.default_rng(4)
    seen = {}
    for n_seq in range(9355, 9376):
        s, d = LB.dense_block(n_seq, rng, term=8)
        r = LB.tile_route(s, len(d), phase)
        assert r.engine == "tile", (n_seq, r)
        seen.setdefault(r.table_intact, n_seq)
    assert set(seen) == {True, False}, seen


def test_stage_threshold_sizes():
    rng = np.random.default_rng(5)
    for ph in (0, 1, 15):
        s, d = LB.sized_block(rng, LB.STAGE_SMALL - 16 - ph)
        assert LB.expected_engine(s, len(d), ph) == "tile"
        s, d = LB.sized_block(rng, LB.STAGE_SMALL - 15 - ph)
        assert LB.expected_engine(s, len(d), ph) == "tile_big"
    s, d = LB.sized_block(rng, 65535)
    assert LB.expected_engine(s, len(d), 15) == "tile_big"
    s, d = LB.sized_block(rng, 65536)
    assert LB.expected_engine(s, len(d)) == "generic"


def test_families_reach_what_they_aim_at():
    rng = np.random.default_rng(6)
    # the chain: every sequence of a step but the first is near
    s, _ = LB.chain_block(rng, 1100)
    nf = LB.near_flags(s)
    assert sum(nf[513:1024]) == 511
    # the wide source: the long match's source covers >= 20 near intervals of its own step
    s, _ = LB.wide_source_block(rng)
    sq, nf = LB.parse(s), LB.near_flags(s)
    longs = [i for i, q in enumerate(sq) if q.ml == 600]
    assert longs and all(nf[i] and sum(nf[i - 30:i]) >= 20 for i in longs if i % LB.DT_K >= 30)
    # the step boundary: delta -1 / 0 -> far, +1 -> near, for the sequences after the first
    for delta, want in ((-1, False), (0, False), (1, True)):
        s, _ = LB.step_boundary_block(rng, delta)
        nf = LB.near_flags(s)
        for r in range(1, 7):
            assert not nf[r * LB.DT_K] and all(nf[r * LB.DT_K + j] == want for j in (1, 2, 3)), (delta, r)
    # copy grid: overlapping matches are near; the far-overlap blocks put them first in their step, far
    for s, _ in LB.copy_grid_blocks(rng, offsets=(1, 50, 160, 199)):
        sq, nf = LB.parse(s), LB.near_flags(s)
        assert all(nf[i] for i, q in enumerate(sq) if 0 < q.off < q.ml and i % LB.DT_K)
    for s, _ in LB.far_overlap_blocks(rng, (1, 33, 160), (128, 600)):
        sq, nf = LB.parse(s), LB.near_flags(s)
        firsts = [i for i in range(LB.DT_K, len(sq) - 1, LB.DT_K)]
        assert firsts and all(sq[i].off < sq[i].ml and not nf[i] for i in firsts)


def test_probe_step_and_collision_inputs(checkers):
    """The adversarial encoder inputs are deterministic, full-size, and plant the hash/tag collisions they
    promise (same 13-bit hash and, for some, the same 16-bit tag, different words)."""
    rng = np.random.default_rng(7)
    a = LB.probe_step_input(rng, tail=13)
    b = LB.probe_step_input(np.random.default_rng(7), tail=13)
    assert a == b and len(a) == 65536
    c = LB.probe_step_input(rng, tail=12, collide=True)
    tag_pairs = hash_pairs = 0
    for o in range(4):                                 # words 4 bytes apart at every alignment
        words = np.frombuffer(c[o:o + 16380 * 4], dtype="<u4")
        prod = (words.astype(np.uint64) * LB.ENC_HASH_MUL) & 0xFFFFFFFF
        h, tag = prod >> 19, (prod >> 3) & 0xFFFF
        same_h = (h[:-1] == h[1:]) & (words[:-1] != words[1:])
        hash_pairs += int(same_h.sum())
        tag_pairs += int((same_h & (tag[:-1] == tag[1:])).sum())
    assert tag_pairs > 50 and hash_pairs > tag_pairs + 20, (tag_pairs, hash_pairs)
    for d in (a, c):                                   # and they encode / decode in the checkers
        for ch in checkers:
            r, enc = ch.encode(d)
            assert r > 0 and ch.decode(enc, len(d)) == (len(d), d)
