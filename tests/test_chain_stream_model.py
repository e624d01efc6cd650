"""The model of k4lz4_decode_chain_streams (tests/chain_stream_ref.py) against upstream's chained decoder.

The streams are upstream's own LZ4_compress_fast_continue output over datagen 0.63, in 4 KiB, 64 KiB, 256 KiB and
4 MiB blocks, behind histories of 0 .. 65 536 bytes, with stored blocks interleaved and mutated blocks
(tests/block_mutants.py) at the first, a middle and the last position.  The model's every copy asserts that it
reads only final bytes; the test holds its lengths and bytes to upstream stepped block by block.  It also counts
the data properties the design rests on: the share of bytes deferred and the blocks that overflow the budget.
"""
import functools

import pytest

from tests import block_mutants as BM
from tests import chain_ref as CR
from tests import chain_stream_ref as SR

pytestmark = pytest.mark.skipif(not __import__("oracle").have_ref(), reason="needs the reference's C engine")

SIZES = {4096: 48, 65536: 12, 262144: 4, 4 << 20: 2}      # block size -> blocks


@functools.lru_cache(maxsize=None)
def _up():
    return CR.Upstream()


@functools.lru_cache(maxsize=None)
def _chain(block: int, nblocks: int, seed: int = 63):
    import oracle
    data = oracle.Port().datagen(block * nblocks, 0.63, 0.0, seed).tobytes()
    return data, _up().encode_chain(data, block)


def _check(hist: bytes, entries, stats=None):
    (got_len, got), = SR.decode_streams([(hist, len(hist), entries)], stats=stats)
    want_len, want = SR.step_reference(_up(), hist, len(hist), entries)
    assert got_len == want_len
    assert got == want
    return got_len


@pytest.mark.parametrize("block", sorted(SIZES))
def test_model_matches_upstream_on_linked_blocks(block):
    data, blocks = _chain(block, SIZES[block])
    st = SR.Stats()
    lens = _check(b"", [(b, block, False) for b in blocks], st)
    assert sum(lens) == len(data)
    assert st.deferred_bytes > 0                    # datagen 0.63 matches reach back into earlier blocks
    print(f"\n{block} B blocks: {st.blocks} blocks, {100 * st.deferred_bytes / st.out_bytes:.1f} % of bytes deferred, "
          f"{st.deferred_copies / st.blocks:.0f} deferred copies per block (max {st.max_copies}), "
          f"{st.whole_blocks} over the budget of {SR.BUDGET}")


def test_model_history_lengths():
    """prefixLen 0, 1, 65 534, 65 535, 65 536: the first block reads the caller's history."""
    data, blocks = _chain(65536, 6, seed=64)
    for P in (0, 1, 65534, 65535, 65536):
        hist = data[2 * 65536 - P:2 * 65536] if P else b""
        entries = [(b, 65536, False) for b in blocks[2:]]
        lens = _check(hist, entries)
        if P >= 65535:
            assert min(lens) > 0                    # the full window: every block decodes


def test_model_deepest_chain_and_budget():
    """A repetitive input: every block depends on the one before.  With budget 0 every block with a deferred match
    is decoded whole; with the default budget none is."""
    data = (b"abcdefghij" * 7 + b"0123456789ABCDEF" * 3) * 40000
    blocks = _up().encode_chain(data, 4096)[:64]
    entries = [(b, 4096, False) for b in blocks]
    st = SR.Stats()
    lens = _check(b"", entries, st)
    assert sum(lens) == 64 * 4096 and st.whole_blocks == 0 and min(st.per_block[1:]) > 0
    st0 = SR.Stats()
    (l0, d0), = SR.decode_streams([(b"", 0, entries)], budget=0, stats=st0)
    assert l0 == lens and st0.whole_blocks >= 63


def test_model_raw_entries_interleaved():
    data, blocks = _chain(65536, 8, seed=65)
    entries = []
    for k, b in enumerate(blocks):
        raw = k % 3 == 1
        entries.append((data[k * 65536:(k + 1) * 65536] if raw else b, 65536, raw))
    entries.insert(4, (b"", 65536, True))          # an empty stored entry
    entries.insert(6, (b"x" * 70000, 65536, True))  # a stored entry larger than its capacity fails the stream
    lens = _check(b"", entries)
    assert lens[:6] == [65536, 65536, 65536, 65536, 0, 65536] and set(lens[6:]) == {-1}


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_model_mutated_blocks(where):
    """Mutants of one block: layout-preserving offset rewrites (valid, different content that later blocks copy)
    and chain-breaking ones (the stream fails there: -1 from that block on, exact bytes before it)."""
    data, blocks = _chain(65536, 8, seed=66)
    k = {"first": 0, "middle": 4, "last": 7}[where]
    pa = BM.parsed(blocks[k])
    muts = []
    for i in (1, pa.N // 2, pa.N - 2):
        op_lit = int(pa.op()[i] + pa.lit[i])
        v = max(8, min(65535, op_lit + 65536 * k // 2)) if k else max(8, min(int(pa.off[i]), op_lit))
        muts.append(BM.set_offset(blocks[k], i, v)[0])
    s = blocks[k]
    muts += [s[:-3], s + b"\x00", bytes([0xFF]) + s[1:], s[:len(s) // 2]]
    failed = 0
    for m in muts:
        entries = [(b, 65536, False) for b in blocks]
        entries[k] = (m, 65536, False)
        lens = _check(b"", entries)
        if -1 in lens:
            first = lens.index(-1)
            assert set(lens[first:]) == {-1}
            failed += 1
    assert failed >= 3
