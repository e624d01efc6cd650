"""CPU test of the decoder's jump table (csrc/parse_table.cuh): the SAME header the CUDA kernel uses is
compiled for the host and compared, position by position, with a strict restatement of the block format's
length decoding -- on valid streams (oracle encoder), mutated streams and random bytes, at every stage
alignment, with 0x00 / 0xFF or random bytes (what the big-stage kernel leaves from the previous block) behind
the end of the stream."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle
from tests import inputs

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "parse_table_check.cpp")
SO = os.path.join(HERE, "native", "_parse_table_check.so")


@pytest.fixture(scope="module")
def chk():
    hdr = os.path.join(HERE, "..", "k4os", "compression", "lz4_b200", "csrc", "parse_table.cuh")
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(SRC), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-std=c++17", "-x", "c++", "-shared", "-fPIC", "-o", SO, SRC], check=True)
    lib = C.CDLL(SO)
    lib.jt_check.restype = C.c_int
    lib.jt_check.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]

    def run(stream: bytes, shift=0, fill=0xFF, seg=0, warm=0):
        a = np.frombuffer(stream, dtype=np.uint8)
        st = np.zeros(8, dtype=np.int64)
        fails = lib.jt_check(a.ctypes.data, len(a), shift, fill, seg, warm, st.ctypes.data)
        return fails, st
    return run


def _streams():
    port = oracle.Port()
    rng = np.random.default_rng(7)
    out = []
    dg = port.datagen(8 * 65536, 0.63, 0.0, 1234)
    for i in range(8):
        out.append(port.encode(dg[i * 65536:(i + 1) * 65536].tobytes())[1])
    for kind in ("text2", "lowent", "repeat", "random", "runs", "lorem"):
        for n in (13, 100, 4000, 65536):
            out.append(port.encode(inputs.gen(kind, n, seed=n))[1])
    # long literal runs and long matches: extension chains of every length
    for lit in (14, 15, 16, 238, 239, 240, 269, 270, 271, 524, 525, 526, 1000):
        raw = rng.integers(0, 256, lit, dtype=np.uint8).tobytes() + b"abcd" * 400 + bytes(rng.integers(0, 256, 64, dtype=np.uint8))
        out.append(port.encode(raw)[1])
    return out


def test_table_matches_format_on_valid_streams(chk):
    tot = np.zeros(8, dtype=np.int64)
    for s in _streams():
        for shift in (0, 1, 2, 3, 7, 15):
            for fill in (0x00, 0xFF, 0x100 + shift):            # > 255: pseudo-random bytes seeded by it
                fails, st = chk(s, shift, fill)
                assert fails == 0, (len(s), shift, fill, int(st[4]) - 1)
                tot += st
    assert tot[0] > 1_000_000
    # the table must actually serve the hops: escapes are rare among true tokens
    assert tot[3] < 0.05 * tot[2], (int(tot[3]), int(tot[2]))


def test_table_on_mutated_and_random_streams(chk):
    rng = np.random.default_rng(11)
    base = _streams()[:8]
    n_checked = 0
    for it in range(300):
        s = bytearray(base[it % len(base)][: int(rng.integers(20, 6000))])
        for _ in range(int(rng.integers(1, 12))):
            s[int(rng.integers(0, len(s)))] = int(rng.choice([0, 15, 0xF0, 0xFF, 0xEF, 0xFE, int(rng.integers(0, 256))]))
        fails, st = chk(bytes(s), int(rng.integers(0, 16)), int(rng.choice([0, 0xFF, 0xF0, 0x100 + it])))
        assert fails == 0, (it, int(st[4]) - 1)
        n_checked += int(st[0])
    for it in range(100):
        p = rng.choice([0.02, 0.2, 0.5])
        s = np.where(rng.random(3000) < p, 0xFF, rng.integers(0, 256, 3000)).astype(np.uint8).tobytes()
        fails, st = chk(s, it % 16, 0xFF if it % 2 else 0x1000 + it)
        assert fails == 0, (it, int(st[4]) - 1)
    assert n_checked > 100_000
