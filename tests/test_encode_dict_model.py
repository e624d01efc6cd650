"""Encoding against an external dictionary: the facts about upstream's LZ4_loadDict + LZ4_compress_fast_continue
that k4lz4_encode_dict_batch (csrc/encode_dict.cuh) relies on, checked on the oracle engine.  CPU only."""
import numpy as np
import pytest

oracle = pytest.importorskip("oracle")
if not oracle.have_ref():
    pytest.skip("reference engine not built", allow_module_level=True)

from tests import dict_enc_ref as DR

LENGTHS = [0, 1, 7, 8, 9, 3000, 65535, 65536, 65537, 200000]


@pytest.fixture(scope="module")
def up():
    return DR.DictUpstream()


def _collisions(n: int, seed: int) -> bytes:
    """A few distinct 8-byte words repeated: every load position hashes into a handful of slots."""
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 256, (4, 8), dtype=np.uint8)
    pick = rng.integers(0, 4, n // 8 + 1)
    return words[pick].reshape(-1)[:n].tobytes()


@pytest.mark.parametrize("kind", ["random", "collisions"])
@pytest.mark.parametrize("n", LENGTHS)
def test_load_is_last_writer_per_slot(up, n, kind):
    rng = np.random.default_rng(n)
    d = rng.integers(0, 256, n, dtype=np.uint8).tobytes() if kind == "random" else _collisions(n, n)
    assert np.array_equal(DR.load_table(d), up.loaded(d))


def test_short_dictionaries_encode_like_none(up):
    src = DR.records(4096, 3)
    want = up.encode(src, b"")
    for n in (1, 7):
        assert up.encode(src, b"\x7b" * n) == want
        assert up.encode(src, src[:n]) == want


def test_long_dictionary_encodes_like_its_last_64k(up):
    d = DR.records(200000, 4)
    for size in (256, 4096, 100000):
        src = DR.records(size, 10 + size)
        assert up.encode(src, d) == up.encode(src, d[-65536:])


def test_extdict_differs_from_prefix_mode_on_catchup(up):
    """A match found in the source catches up no further than the source's start in the extDict mode; in the prefix
    mode it runs on into the dictionary in front."""
    src, d = DR.catchup_input()
    ext, pre = up.encode(src, d), up.encode_prefix(src, d)
    assert ext[0] > 0 and pre[0] > 0 and ext[1] != pre[1]
    assert up.decode(ext[1], len(src), d) == (len(src), src)
