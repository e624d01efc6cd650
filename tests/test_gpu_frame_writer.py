"""Frame writer groups on the GPU (k4lz4_frame_writer_group_*, FrameWriterGroup): every write's and close's bytes
equal the incremental LZ4FrameWriter model over upstream's engine (tests/frame_writer_ref.py), through host and
device memory alternately, with 0xCD canaries around every destination slot.  Closed frames decode with upstream
lz4frame.c and with k4lz4_frame_decode_batch.  Needs the reference engine that __graft_entry__.build() compiles
into oracle/_ref/."""
import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests import frame_writer_ref as FW

pytestmark = pytest.mark.gpu
CD = 0xCD
GAP = 32


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def ref():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return oracle.Ref()


@pytest.fixture(scope="module")
def up(ref):
    return ER.EncUpstream()


def pool(n: int, seed: int) -> bytes:
    """datagen 0.63 with incompressible stretches (raw blocks) and an all-zero stretch."""
    import oracle
    rng = np.random.default_rng(seed)
    a = oracle.Port().datagen(n, 0.63, 0.0, seed).copy()
    for _ in range(max(n // 400000, 1)):
        at = int(rng.integers(0, n - 80000))
        a[at:at + 80000] = rng.integers(0, 256, 80000, dtype=np.uint8)
    at = int(rng.integers(0, n - 300000))
    a[at:at + 300000] = 0
    return a.tobytes()


def call(k4, g, mem, streams, chunks=None, caps=None):
    """One write (chunks given) or close of group g through host or device memory -> (results, produced bytes).
    Checks that nothing outside [dstOff, dstOff + result) changed."""
    import torch
    N = k4._native
    L = N.lib()
    n = len(streams)
    if chunks is not None:
        lens = np.array([len(c) for c in chunks], np.int32)
        so = np.zeros(n, np.int64)
        so[1:] = np.cumsum(lens[:-1], dtype=np.int64)
        src = np.frombuffer(b"".join(chunks) + b"\0" * 16, np.uint8).copy()
        if caps is None:
            caps = [g.bound(int(x)) for x in lens]
    elif caps is None:
        caps = [g.close_bound()] * n
    dc = np.array(caps, np.int32)
    do = GAP + np.concatenate([[0], np.cumsum(np.maximum(dc[:-1], 0).astype(np.int64) + GAP)]).astype(np.int64)
    dst = np.full(int(do[-1]) + max(int(dc[-1]), 0) + GAP, CD, np.uint8)
    st = np.array(streams, np.int32)
    out = np.full(n, -7, np.int32)
    if mem == "host":
        if chunks is not None:
            rc = L.k4lz4_frame_writer_group_write(g.handle, st.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                  lens.ctypes.data, dst.ctypes.data, do.ctypes.data, dc.ctypes.data,
                                                  out.ctypes.data, n, N.MEM_HOST, None)
        else:
            rc = L.k4lz4_frame_writer_group_close(g.handle, st.ctypes.data, dst.ctypes.data, do.ctypes.data,
                                                  dc.ctypes.data, out.ctypes.data, n, N.MEM_HOST, None)
        N.check(rc)
    else:
        dev = torch.device("cuda", 0)
        T = lambda a: torch.from_numpy(a).to(dev)
        t_st, t_dst, t_do, t_dc = T(st), T(dst), T(do), T(dc)
        t_out = torch.full((n,), -7, dtype=torch.int32, device=dev)
        s = torch.cuda.current_stream().cuda_stream
        if chunks is not None:
            t_src, t_so, t_sl = T(src), T(so), T(lens)
            g.write_device(t_st.data_ptr(), t_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(), t_dst.data_ptr(),
                           t_do.data_ptr(), t_dc.data_ptr(), t_out.data_ptr(), n, stream=s)
        else:
            g.close_device(t_st.data_ptr(), t_dst.data_ptr(), t_do.data_ptr(), t_dc.data_ptr(), t_out.data_ptr(), n,
                           stream=s)
        torch.cuda.synchronize()
        out, dst = t_out.cpu().numpy(), t_dst.cpu().numpy()
    mask = np.ones(dst.shape[0], bool)
    for o, r in zip(do, out):
        mask[o:o + max(int(r), 0)] = False
    assert (dst[mask] == CD).all(), np.nonzero(dst[mask] != CD)[0][:8]
    return out, [dst[o:o + r].tobytes() if r > 0 else b"" for o, r in zip(do, out)]


def decode_all(k4, ref, frames, contents):
    assert k4.frame.read_frames(frames) == contents
    for f, c in zip(frames[::7], contents[::7]):
        assert ref.frame_decompress(f, len(c) + 16) == c


def run_streams(k4, ref, up, g, S, bs, fl, rng, data, calls, picks):
    """`calls` writes of random subsets with chunk sizes from `picks`, alternating host and device memory, with
    one entry per call at dstCap = bound - 1 (-1, retried at the bound in the next call); then a close of every
    stream.  Each result equals the model's emission."""
    chaining, bc, cc = not fl & 1, bool(fl & 2), bool(fl & 4)
    models = [FW.Writer(bs, chaining, bc, cc, FW.UpstreamEngine(up, ref, chaining), ref.xxh32) for _ in range(S)]
    content = [[] for _ in range(S)]
    frames = [[] for _ in range(S)]
    at = [int(rng.integers(0, len(data) // 2)) for _ in range(S)]
    retry = {}
    for c in range(calls):
        mem = "host" if c % 2 == 0 else "device"
        streams = [s for s in range(S) if s in retry or rng.random() < 0.7]
        rng.shuffle(streams)
        chunks = []
        for s in streams:
            if s in retry:
                chunks.append(retry.pop(s))
                continue
            k = int(picks[int(rng.integers(0, len(picks)))])
            if s % 11 == 3:
                chunks.append(bytes(k))                   # all-zero content
            else:
                o = at[s] % (len(data) - k)
                chunks.append(data[o:o + k])
                at[s] += k + 1
        caps = [g.bound(len(x)) for x in chunks]
        short = int(rng.integers(0, len(streams))) if streams else -1
        if short >= 0:
            caps[short] -= 1
        res, got = call(k4, g, mem, streams, chunks, caps)
        for i, s in enumerate(streams):
            if i == short:
                assert res[i] == -1
                retry[s] = chunks[i]
                continue
            want = models[s].write(chunks[i])
            content[s].append(chunks[i])
            assert res[i] == len(want) and got[i] == want, (c, mem, s, len(chunks[i]))
            frames[s].append(got[i])
    for s, chunk in retry.items():                       # every retry at the bound
        res, got = call(k4, g, "device", [s], [chunk])
        assert got[0] == models[s].write(chunk)
        content[s].append(chunk)
        frames[s].append(got[0])
    streams = list(range(S))
    res, got = call(k4, g, "host" if calls % 2 else "device", streams)
    for s in streams:
        want = models[s].close()
        assert res[s] == len(want) and got[s] == want, s
        frames[s].append(got[s])
    return [b"".join(f) for f in frames], [b"".join(c) for c in content]


@pytest.mark.parametrize("fl", range(8))
def test_many_streams_equal_model(k4, ref, up, fl):
    """4 224 streams of 64 KiB blocks: enough entries per step that independent frames use both encoder warp kinds."""
    S, bs = 4224, 65536
    rng = np.random.default_rng(100 + fl)
    data = pool(8 << 20, 100 + fl)
    picks = [0, 1, 15, 16, 17, bs - 1, bs, bs + 1, 3 * bs + 17, 300, 5000, 20000]
    k4.batch.encode_stats(0, reset=True)
    with k4.FrameWriterGroup(S, bs, chaining=not fl & 1, block_checksum=bool(fl & 2),
                             content_checksum=bool(fl & 4)) as g:
        frames, contents = run_streams(k4, ref, up, g, S, bs, fl, rng, data, 3, picks)
    stats = np.zeros(4, np.uint64)
    k4._native.check(k4._native.lib().k4lz4_encode_stats(0, stats.ctypes.data, 1))
    if fl & 1:
        assert stats[0] > 0 and stats[1] > 0 and stats[3] == 0, stats
    else:
        assert stats[3] > 0 and stats[0] == 0 and stats[1] == 0, stats
    decode_all(k4, ref, [f for f in frames if f], [c for f, c in zip(frames, contents) if f])


@pytest.mark.parametrize("bs", [1 << 18, 1 << 20, 4 << 20, 100000])
def test_block_sizes_equal_model(k4, ref, up, bs):
    B = FW.rounded_block(bs)
    S = 6 if bs == 4 << 20 else 24
    rng = np.random.default_rng(bs)
    data = pool(max(12 * B, 4 << 20), bs)
    picks = [0, 1, 15, 16, 17, B - 1, B, B + 1, 3 * B + 17, 1000]
    for fl in (0, 7, 1, 6):
        with k4.FrameWriterGroup(S, bs, chaining=not fl & 1, block_checksum=bool(fl & 2),
                                 content_checksum=bool(fl & 4)) as g:
            frames, contents = run_streams(k4, ref, up, g, S, bs, fl, rng, data, 4, picks)
        nz = [i for i, f in enumerate(frames) if f]
        decode_all(k4, ref, [frames[i] for i in nz], [contents[i] for i in nz])
        if bs == 100000:
            assert all(f[5] == 5 << 4 for f in frames if f)


def test_lifecycle(k4, ref, up):
    """Close of a never-written stream: 0 bytes.  write(0) + close: header, end mark, XXH32 of nothing.  Reset in
    the middle of a frame, then reuse of closed and reset streams."""
    import struct
    for mem in ("host", "device"):
        with k4.FrameWriterGroup(4, 65536, content_checksum=True) as g:
            res, got = call(k4, g, mem, [0, 1, 2, 3])
            assert res.tolist() == [0] * 4 and got == [b""] * 4
            res, got = call(k4, g, mem, [2], [b""])
            assert got[0] == FW.header(65536, True, False, True)
            res, got = call(k4, g, mem, [2, 3])
            assert got == [struct.pack("<II", 0, ref.xxh32(b"")), b""]
            data = pool(1 << 20, 5)
            models = [FW.Writer(65536, True, False, True, FW.UpstreamEngine(up, ref, True), ref.xxh32) for _ in range(4)]
            res, got = call(k4, g, mem, [0, 1], [data[:100000], data[5:70000]])
            assert got == [models[0].write(data[:100000]), models[1].write(data[5:70000])]
            if mem == "host":
                g.reset([1])
            else:
                import torch
                t = torch.tensor([1], dtype=torch.int32, device="cuda")
                g.reset_device(t.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)
            models[1] = FW.Writer(65536, True, False, True, FW.UpstreamEngine(up, ref, True), ref.xxh32)
            res, got = call(k4, g, mem, [1])
            assert res[0] == 0                                           # reset: nothing to close
            chunks = [data[300000:450000], data[:1000], data[7:200000]]
            res, got = call(k4, g, mem, [0, 1, 2], chunks)
            assert got == [models[i].write(c) for i, c in zip((0, 1, 2), chunks)]
            res, got = call(k4, g, mem, [0, 1, 2])
            frames = [models[i].close() for i in (0, 1, 2)]
            assert got == frames


def test_argument_errors(k4):
    N = k4._native
    L = N.lib()
    with k4.FrameWriterGroup(4, 65536) as g:
        s = np.array([0, 0], np.int32)
        src = np.zeros(32, np.uint8)
        so = np.zeros(2, np.int64)
        sl = np.array([1, 1], np.int32)
        dc = np.array([100, 100], np.int32)
        out = np.zeros(2, np.int32)
        args = [src.ctypes.data, so.ctypes.data, sl.ctypes.data, src.ctypes.data, so.ctypes.data, dc.ctypes.data,
                out.ctypes.data]
        assert L.k4lz4_frame_writer_group_write(g.handle, s.ctypes.data, *args, 2, N.MEM_HOST, None) == N.E_ARG
        s[1] = 4
        assert L.k4lz4_frame_writer_group_write(g.handle, s.ctypes.data, *args, 2, N.MEM_HOST, None) == N.E_ARG
        assert L.k4lz4_frame_writer_group_write(g.handle, s.ctypes.data, *args, 2, 5, None) == N.E_ARG
        assert L.k4lz4_frame_writer_group_write(g.handle, s.ctypes.data, *args, -1, N.MEM_HOST, None) == N.E_ARG
        s[1] = 1
        sl[1] = 0x7FFFFF00                               # its bound exceeds 2^31 - 1
        assert L.k4lz4_frame_writer_group_write(g.handle, s.ctypes.data, *args, 2, N.MEM_HOST, None) == N.E_ARG
        assert g.bound(0) == 7 and g.bound(1) == 7 + 4 + 65536 and g.close_bound() == 4 + 65536 + 4
        assert L.k4lz4_frame_writer_bound(g.handle, -1) == N.E_ARG
    with k4.FrameWriterGroup(2, 65536, block_checksum=True, content_checksum=True) as g:
        assert g.bound(65537) == 7 + 2 * (4 + 65536 + 4) and g.close_bound() == 4 + 65536 + 4 + 4 + 4
        # device memory: an index out of range gives -1 and changes nothing
        res, got = call(k4, g, "device", [5, 0], [b"abc", b"def"])
        assert res[0] == -1 and res[1] == 7
        res, got = call(k4, g, "device", [0, 7])
        # the pending "def": length code (raw), body, block checksum; the end mark; the content checksum
        assert res[1] == -1 and res[0] == 19 and got[0][:7] == b"\x03\x00\x00\x80def"


def test_staging_split(k4, ref):
    """One host call with more source than one staging piece (256 MiB): the bytes equal the frame call's on the
    whole content, and decode."""
    import oracle
    n = 150 << 20
    a = oracle.Port().datagen(n, 0.63, 0.0, 77)
    chunks = [a.tobytes(), a[7:].tobytes(), b"x" * 1000]
    with k4.FrameWriterGroup(3, 1 << 20, block_checksum=True, content_checksum=True) as g:
        res, got = call(k4, g, "host", [0, 1, 2], chunks)
        assert (res > 0).all()
        res2, got2 = call(k4, g, "host", [2, 1, 0])
    frames = [got[0] + got2[2], got[1] + got2[1], got[2] + got2[0]]
    want, res = k4.LZ4Frame.EncodeMany(chunks, 1 << 20, True, True, True)
    assert frames == want
    assert k4.frame.read_frames(frames[2:]) == chunks[2:]
    assert ref.frame_decompress(frames[1], len(chunks[1]) + 16) == chunks[1]
