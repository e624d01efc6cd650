"""Upstream's frames on the GPU (k4lz4_lz4f_compress_batch, LZ4F / lz4f_compress): every frame of the grid in
tests/lz4f_ref.py byte for byte what LZ4F_compressFrame writes, one batched call per (block size, flags), in host and
device memory, with the destinations' slack and surroundings untouched.  Also: the results of small destinations and
of the levels upstream's call would run with HC or acceleration, a call large enough for every encoder warp kind, and
round trips through the reference-semantics frame calls.  Needs the reference engine that __graft_entry__.build()
compiles into oracle/_ref/."""
import numpy as np
import pytest

from tests import lz4f_ref as R
from tests.test_gpu_frames import CD, GAP, layout

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return R.Lz4fUpstream()


def run(k4, items, caps, bs, flags, level=0, mem="device"):
    """One k4lz4_lz4f_compress_batch call -> (results, dst, dstOff, dstCap)."""
    N = k4._native
    src, so, sl, dst, do, dc = layout(items, caps)
    n = len(items)
    out = np.full(n, 12345, dtype=np.int32)
    if mem == "host":
        N.check(N.lib().k4lz4_lz4f_compress_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                  do.ctypes.data, dc.ctypes.data, out.ctypes.data, n, bs, flags,
                                                  level, N.MEM_HOST, None, 0))
        return out, dst, do, dc
    import torch
    dev = torch.device("cuda", 0)
    t = {k: torch.from_numpy(v.copy()).to(dev) for k, v in dict(src=src, so=so, sl=sl, dst=dst, do=do, dc=dc).items()}
    o = torch.from_numpy(out).to(dev)
    k4.LZ4F.compress_many_device(t["src"], t["so"], t["sl"], t["dst"], t["do"], t["dc"], o, bs,
                                 not (flags & R.INDEPENDENT), bool(flags & R.BLOCK_CHECKSUM),
                                 bool(flags & R.CONTENT_CHECKSUM), bool(flags & R.CONTENT_SIZE), level,
                                 torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return o.cpu().numpy(), t["dst"].cpu().numpy(), do, dc


def frames_of(out, dst, do, dc):
    """The frames; every byte of a slot behind its frame (the whole slot where it failed) and the gaps around it
    still hold the fill byte."""
    res = []
    for i in range(len(out)):
        r, a, c = int(out[i]), int(do[i]), int(dc[i])
        assert (dst[a - GAP:a] == CD).all() and (dst[a + c:a + c + GAP] == CD).all(), f"canary of frame {i}"
        if r >= 0:
            assert (dst[a + r:a + c] == CD).all(), f"slack of frame {i}"
        res.append(dst[a:a + r].tobytes() if r >= 0 else None)
    return res


@pytest.mark.parametrize("mem", ["device", "host"])
def test_grid_equals_upstream(k4, up, mem):
    for (bs, fl), items in R.groups().items():
        caps = [up.bound(len(x), bs, fl) + 5 for x in items]
        got = frames_of(*run(k4, items, caps, bs, fl, mem=mem))
        for g, x in zip(got, items):
            assert g == up.frame(x, bs, fl), (len(x), bs, fl)


def test_small_destinations(k4, up):
    """A frame that does not fit gives -1 and writes nothing beyond its slot; one that fits exactly succeeds."""
    items, caps, want = [], [], []
    for i, n in enumerate((0, 13, 5000, 70000, 300000)):
        x = R.content("text" if i % 2 else "random", n, 77 * i)
        f = up.frame(x, 1 << 18, R.CONTENT_SIZE | R.CONTENT_CHECKSUM)
        for c in (len(f) - 1, len(f), 0, 7):
            items.append(x); caps.append(c); want.append(f if c >= len(f) else None)
    for mem in ("device", "host"):
        got = frames_of(*run(k4, items, caps, 1 << 18, R.CONTENT_SIZE | R.CONTENT_CHECKSUM, mem=mem))
        assert got == want


@pytest.mark.parametrize("level", [3, 9, 12, -1, -5])
def test_levels_upstream_runs_elsewhere_delegate(k4, up, level):
    from k4os.compression.lz4_b200 import _native as N
    items = [R.content("text", n, n) for n in (0, 100, 70000)]
    caps = [up.bound(len(x), 1 << 16, 0) for x in items]
    for mem in ("device", "host"):
        out, dst, do, dc = run(k4, items, caps, 1 << 16, 0, level, mem)
        assert (out == N.R_DELEGATE).all()
        assert (dst == CD).all()
    with pytest.raises(NotImplementedError):
        k4.lz4f_compress(b"abc", level=level)


def test_levels_1_and_2_are_level_0(k4, up):
    x = R.content("text", 300000, 3)
    for level in (1, 2):
        assert k4.lz4f_compress(x, 1 << 16, content_size=True, level=level) == up.frame(x, 1 << 16, R.CONTENT_SIZE)


def test_every_engine_in_one_call(k4, up):
    """One call with frames of every kind: many small ones (the warps for blocks below 65 547 bytes), single-block
    frames above 65 547 bytes (independent: the big-block warp) and linked 1 MiB-block frames (the chained encoder);
    every frame equals upstream's."""
    from k4os.compression.lz4_b200 import batch
    rng = np.random.default_rng(8)
    items = [R.content("text", int(rng.integers(13, 8192)), i * 4096) for i in range(6000)]
    items += [R.content("text", int(rng.integers(65548, 1 << 20)), i * 777) for i in range(40)]
    items += [R.content("mixed", (2 << 20) + 12345 * i, i * 999, 1 << 20) for i in range(6)]
    fl = R.CONTENT_SIZE
    caps = [up.bound(len(x), 1 << 20, fl) for x in items]
    batch.encode_stats(0, reset=True)
    got = frames_of(*run(k4, items, caps, 1 << 20, fl))
    st = batch.encode_stats(0, reset=True)
    assert st["smem"] + st["gtab"] == 6000 and st["generic"] == 40 and st["chain"] > 0, st
    for g, x in zip(got, items):
        assert g == up.frame(x, 1 << 20, fl), len(x)


def test_round_trips_with_the_frame_calls(k4, up):
    """k4lz4_frame_decode_batch reads the frames written without a content size, and upstream reads them back."""
    from k4os.compression.lz4_b200 import LZ4F, LZ4Frame
    for bs in R.BLOCK_SIZES:
        for linked in (True, False):
            items = [x for x in R.groups()[(bs, R.flags_of(linked, True, True, False))]]
            frames, out = LZ4F.compress_many(items, bs, linked, True, True, False)
            assert (out > 0).all()
            contents, res = LZ4Frame.DecodeMany(frames)
            assert list(res) == [len(x) for x in items] and contents == items
            for f, x in zip(frames, items):
                assert up.ref.frame_decompress(f, len(x)) == x


def test_linked_steps_follow_the_linked_frames(k4, up):
    """Thousands of one-block frames beside one linked frame of five 4 MiB blocks: the linked steps run over the
    linked frame alone (one chunk), not over every frame of the call, and every frame equals upstream's."""
    N = k4._native
    items = [R.content("text", 100 + i % 900, i * 64) for i in range(3000)]
    items.append(R.content("zeros", (4 << 22) + 77, 0))
    fl = R.CONTENT_CHECKSUM
    caps = [up.bound(len(x), 1 << 22, fl) for x in items]
    before = N.lib().k4lz4_launch_count()
    got = frames_of(*run(k4, items, caps, 1 << 22, fl))
    launches = N.lib().k4lz4_launch_count() - before
    # 3000 independent blocks go in chunks of 127 4-MiB scratch slots (24 chunks of about 7 launches); the linked
    # pass is one chunk of 5 steps.  Steps over all 3001 frames would add about 24 x 5 x 7 = 840 more.
    assert launches < 400, launches
    for g, x in zip(got, items):
        assert g == up.frame(x, 1 << 22, fl), len(x)
