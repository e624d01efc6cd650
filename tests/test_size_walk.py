"""CPU test of the warp-parallel size walk (csrc/size_walk.cuh): the SAME header the CUDA kernels use is compiled for
the host, and tests/native/size_walk_check.cpp runs its windows, speculative lanes and link repair lane by lane.
The result must equal the serial walk (test_frame_model.walk) on valid streams (oracle encoder), mutated full-size
blocks (tests/block_mutants.py), truncated tails, random bytes and hand-built chains whose 255-extension runs and
literal runs cross segment and window edges -- at every segment phase, for the shipped segment length and warm-up
and for others."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import block_mutants as BM
from tests import inputs
from tests import lz4_blocks as LB
from tests.test_frame_model import walk

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "size_walk_check.cpp")
SEG, WARM = 128, 64                      # K4_SW_SEG / K4_SW_WARM as shipped
SHAPES = ((SEG, WARM), (32, 0), (32, 32), (64, 64), (64, 256))


@pytest.fixture(scope="module")
def sw(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("size_walk") / "size_walk_check.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-x", "c++", "-shared", "-fPIC", "-o", so, SRC], check=True)
    lib = C.CDLL(so)
    lib.sw_sim.restype = C.c_longlong
    lib.sw_sim.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p]
    lib.sw_serial.restype = C.c_longlong
    lib.sw_serial.argtypes = [C.c_void_p, C.c_longlong]

    class Check:
        stats = np.zeros(8, dtype=np.int64)

        def run(self, s: bytes, seg=SEG, warm=WARM):
            """-> (simulated walk, serial walk); asserts that no byte outside the block was read"""
            a = np.frombuffer(s, dtype=np.uint8) if s else np.zeros(1, dtype=np.uint8)
            st = np.zeros(8, dtype=np.int64)
            got = lib.sw_sim(a.ctypes.data, len(s), seg, warm, st.ctypes.data)
            assert st[6] == 0, ("read outside the block", len(s), seg, warm)
            self.stats += st
            return got, lib.sw_serial(a.ctypes.data, len(s))

        def same(self, s: bytes, shapes=SHAPES):
            for seg, warm in shapes:
                got, want = self.run(s, seg, warm)
                assert got == want, (len(s), seg, warm, got, want)
            return want
    return Check()


def shifted(stream: bytes, d: int, rng) -> bytes:
    """`stream` with d more literals in its first sequence: every later token moves d bytes against the segment
    grid, and the walk grows by d."""
    tok, p = stream[0], 1
    lit = tok >> 4
    if lit == 15:
        while True:
            x = stream[p]; p += 1; lit += x
            if x != 255:
                break
    L = lit + d
    head = bytes([(min(L, 15) << 4) | (tok & 15)]) + (LB._ext(L - 15) if L >= 15 else b"")
    return head + stream[p:p + lit] + bytes(rng.integers(0, 256, d, dtype=np.uint8)) + stream[p + lit:]


def _valid_streams():
    import oracle
    port = oracle.Port()
    out = []
    dg = port.datagen(4 * 65536, 0.63, 0.0, 99)
    out += [port.encode(dg[i * 65536:(i + 1) * 65536].tobytes())[1] for i in range(4)]
    for kind in ("text2", "lowent", "repeat", "random", "runs", "lorem"):
        for n in (13, 100, 2047, 2048, 2049, 4000, 65536):
            out.append(port.encode(inputs.gen(kind, n, seed=n))[1])
    out.append(port.encode(bytes(65536))[1])               # one match with a 257-byte extension run
    return out


def test_valid_streams_at_every_phase(sw):
    rng = np.random.default_rng(3)
    streams = _valid_streams()
    for s in streams[:4]:
        assert sw.same(s) == 65536 and walk(s) == 65536
    for s in streams:
        want = walk(s)
        assert sw.same(s) == want
        for d in range(1, SEG, 3) if len(s) > 4000 else range(SEG):
            assert sw.same(shifted(s, d, rng), ((SEG, WARM),)) == want + d
    # the shipped shape resolves most lanes speculatively
    assert sw.stats[2] < 0.5 * sw.stats[1], sw.stats


def test_mutated_full_size_blocks(sw):
    rng = np.random.default_rng(5)
    n, differ = 0, 0
    for base in BM.independent_bases():
        for m in BM.chain_breaking(base, rng):
            w = sw.same(m.stream, ((SEG, WARM), (32, 32)))
            differ += w != base.size
            n += 1
        for m in BM.layout_mutants(base, rng)[::7]:
            assert sw.same(m.stream, ((SEG, WARM),)) == m.size
    assert n > 1000 and differ > 100
    for m in BM.chain_breaking(BM.independent_bases()[1], rng)[::25]:
        assert sw.run(m.stream)[0] == walk(m.stream)


def test_truncated_tails_and_random_bytes(sw):
    rng = np.random.default_rng(7)
    for s in _valid_streams()[:2]:
        for c in range(len(s) - 20, len(s) + 1):
            got, want = sw.run(s[:c])
            assert got == want == walk(s[:c]), c
    for it in range(300):
        p = (0.02, 0.2, 0.5, 0.95)[it % 4]
        n = int(rng.integers(1, 9000))
        s = np.where(rng.random(n) < p, 0xFF, rng.integers(0, 256, n)).astype(np.uint8).tobytes()
        sw.same(s)
    assert sw.same(b"") == -1 and walk(b"") == -1
    for s in (b"\x00", b"\x10a", b"\xf0" + b"\xff" * 3, b"\x0f\x01\x00\xff\x00"):
        assert sw.same(s) == walk(s)


def test_extension_runs_across_segment_and_window_edges(sw):
    """Hand-built chains: literal runs and matches whose 255-extension runs start, end or lie wholly inside a segment
    and cross window edges (32 segments), behind a first literal run of every length 0 .. SEG - 1."""
    rng = np.random.default_rng(9)
    rb = lambda k: bytes(rng.integers(0, 256, k, dtype=np.uint8))
    lens = (14, 15, 16, 269, 270, 271, 524, 525, 255 * 64 + 14, 255 * 64 + 15, 255 * 64 + 16, 255 * 130 + 3)
    n = 0
    for L in lens:
        for M in lens:
            for lead in range(0, SEG, 5):
                seqs = [(rb(lead + 1), 1, 4), (rb(L), 1, M + 4), (rb(3), 2, 4), (rb(L // 3), 7, M // 2 + 4)]
                s, dec = LB.build_block(seqs, rb(int(rng.integers(0, 40))))
                assert sw.same(s) == len(dec)
                n += 1
    # a run of single-literal sequences with long matches: many tokens per segment, every phase
    seqs = [(rb(1), 1, int(x)) for x in rng.integers(4, 2000, 600)]
    for lead in range(SEG):
        s, dec = LB.build_block([(rb(lead + 1), 1, 4)] + seqs, rb(5))
        assert sw.same(s, ((SEG, WARM),)) == len(dec)
    assert n > 1000


def test_long_extension_run_is_read_once(sw):
    """A 1 MB run of 0xFF match-extension bytes: only the exact lane reads it; speculative lanes stop one segment
    past their own."""
    s = b"\x0f\x01\x00" + b"\xff" * 1_000_000 + b"\x00\x00"
    sw.stats[:] = 0
    got, want = sw.run(s)
    assert got == want == 15 + 255 * 1_000_000 + 4
    assert sw.stats[7] < 1.2 * len(s), sw.stats
