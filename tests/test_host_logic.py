"""Host-side logic that needs no GPU: the Python mirror's argument rules, batch packing, the
block-list sharding used for N>1 (exercised with a real 2-process gloo group)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import ROOT


def test_validate_rules(native):
    """Internal/Extensions.cs:37-52 via the array overloads (LZ4Codec.cs:82-96,225-237)."""
    from k4os.compression.lz4_b200 import LZ4Codec
    src = bytearray(b"abcdef" * 10)
    dst = bytearray(100)
    with pytest.raises(ValueError):
        LZ4Codec.Encode(src, 0, 61, dst, 0, 100)
    with pytest.raises(ValueError):
        LZ4Codec.Encode(src, -1, 10, dst, 0, 100)
    with pytest.raises(ValueError):
        LZ4Codec.Decode(src, 0, 10, dst, 50, 51)
    with pytest.raises(ValueError):
        LZ4Codec.Encode(None, 0, 0, dst, 0, 100)
    assert LZ4Codec.Encode(src, 5, 0, dst, 0, 100) == 0      # empty slice -> 0
    with pytest.raises(TypeError):
        LZ4Codec.Decode(b"\x10a", b"readonly-target")


def test_level_enum_matches_reference():
    from k4os.compression.lz4_b200 import LZ4Level
    assert LZ4Level.L00_FAST == 0 and LZ4Level.L03_HC == 3 and LZ4Level.L09_HC == 9
    assert LZ4Level.L10_OPT == 10 and LZ4Level.L12_MAX == 12 and len(LZ4Level) == 11


def test_pack_helper():
    from k4os.compression.lz4_b200.batch import _pack
    base, off, ln = _pack([b"abc", b"", b"defgh"])
    assert base.tobytes() == b"abcdefgh" and off.tolist() == [0, 3, 3] and ln.tolist() == [3, 0, 5]
    base, off, ln = _pack([])
    assert len(off) == 0 and len(ln) == 0


def test_shard_ranges_cover_everything():
    sys.path.insert(0, ROOT)
    import bench
    for n in (0, 1, 7, 8, 65536, 524288):
        for w in (1, 2, 3, 4, 8):
            ranges = [bench.shard_range(n, r, w) for r in range(w)]
            assert ranges[0][0] == 0 and ranges[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
            sizes = [hi - lo for lo, hi in ranges]
            assert max(sizes) - min(sizes) <= 1


def test_bench_dump_outputs_format(tmp_path):
    """--dump-outputs: float .npy files, a sample fixed by the seed, bytes past a returned length masked,
    at most 64 MB at the default batch size."""
    import torch
    sys.path.insert(0, ROOT)
    import bench
    nb = 100
    assert np.array_equal(bench.dump_sample(nb), bench.dump_sample(nb)) and len(bench.dump_sample(nb)) == bench.DUMP_BLOCKS
    slots = torch.randint(0, 256, (nb * bench.BOUND,), dtype=torch.uint8)
    enc_len = torch.randint(1, bench.BOUND, (nb,), dtype=torch.int32)
    out = torch.randint(0, 256, (nb * bench.BLOCK,), dtype=torch.uint8)
    out_len = torch.full((nb,), bench.BLOCK, dtype=torch.int32)
    bench.dump_outputs(str(tmp_path), slots, enc_len, out, out_len, nb)
    files = {p.stem: np.load(p) for p in tmp_path.glob("*.npy")}
    assert set(files) == {"encode_len", "encode_bytes_sample", "decode_len", "decode_bytes_sample", "sample_blocks"}
    assert all(a.dtype in (np.float32, np.float64) for a in files.values())
    idx = files["sample_blocks"].astype(np.int64)
    assert np.array_equal(idx, bench.dump_sample(nb))
    for row, b in zip(files["encode_bytes_sample"], idx):
        n = int(enc_len[b])
        assert np.array_equal(row[:n], slots.view(nb, bench.BOUND)[b, :n].numpy()) and (row[n:] == -1).all()
    assert np.array_equal(files["decode_bytes_sample"], out.view(nb, bench.BLOCK)[idx].numpy())
    full = bench.BLOCKS_PER_GPU
    assert 4 * (2 * full + bench.DUMP_BLOCKS * (bench.BOUND + bench.BLOCK)) + 8 * bench.DUMP_BLOCKS <= 64 << 20


def test_two_rank_gloo_sharding_and_timing_reduce():
    """world_size 2 on CPU (gloo): the N>1 plumbing of bench.py -- shard, max-over-ranks
    timing reduce, sum of units -- without touching a GPU."""
    code = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %r)
import bench
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%%s" %% os.environ["K4_PORT"],
                        rank=int(os.environ["RANK"]), world_size=2)
r, w = dist.get_rank(), dist.get_world_size()
lo, hi = bench.shard_range(1001, r, w)
t = bench.reduce_max_seconds(0.25 * (r + 1), device="cpu")
units = bench.reduce_sum_int(hi - lo, device="cpu")
assert abs(t - 0.5) < 1e-6, t
assert units == 1001, units
dist.barrier(); dist.destroy_process_group()
print("rank", r, "ok")
""" % ROOT
    port = 29500 + (os.getpid() % 2000)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", K4_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, "-c", code], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=180)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o
        assert "ok" in o
