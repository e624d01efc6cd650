"""CPU test of tools/enc_traffic.py: the model of the encoder's search batches emits the reference engine's bytes,
so the request counts it reports describe the real parse -- on the bench's encode data and on the window-edge
inputs of tests/test_gpu_encode_windows.py, at several first-batch widths."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import enc_traffic as E  # noqa: E402

from tests.test_gpu_encode_windows import window_block  # noqa: E402


@pytest.fixture(scope="module")
def chk():
    import oracle
    return oracle.best()


def test_model_bytes_on_bench_data(chk):
    import bench
    raw = bench.gen_blocks(2, bench.MP_ENCODE, 0)
    for i in range(2):
        b = raw[i * bench.BLOCK:(i + 1) * bench.BLOCK].tobytes()
        want = chk.encode(b)[1]
        counts = []
        for win in (32, 8, 3):
            got, c = E.encode_block(b, win)
            assert got == want, (i, win)
            counts.append(c)
        # the width changes the requests, never the parse
        assert len({(c["seqs"], c["runs"], c["probes"]) for c in counts}) == 1
        assert counts[1]["slot"] < counts[0]["slot"] and counts[1]["batches"] > counts[0]["batches"]


@pytest.mark.parametrize("mode", ["hit", "split", "post"])
def test_model_bytes_on_window_edges(chk, mode):
    rng = np.random.default_rng(5)
    for n, tail in ((65536, 12), (65535, 19), (65546, 13), (700, 15)):
        b = window_block(rng, 8, n=n, tail=tail, mode=mode)
        want = chk.encode(b)[1]
        for win in (32, 8):
            assert E.encode_block(b, win)[0] == want, (n, tail, win)


def test_model_small_blocks(chk):
    rng = np.random.default_rng(6)
    for n in range(0, 40):
        b = rng.integers(0, 3, n, dtype=np.uint8).tobytes()
        if n == 0:
            continue
        assert E.encode_block(b, 8)[0] == chk.encode(b)[1], n
