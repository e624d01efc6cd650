"""Frame reader groups on the GPU (k4lz4_frame_reader_group_*, FrameReaderGroup): every read's result, bytes
consumed, frame end and content equal the incremental LZ4FrameReader model (tests/frame_reader_ref.py) over
upstream's engines, through host and device memory alternately, with 0xCD canaries around every destination.
Verdicts equal k4lz4_frame_decode_batch's.  Needs the reference engine that __graft_entry__.build() compiles into
oracle/_ref/."""
import numpy as np
import pytest

from tests import frame_reader_ref as FR
from tests.test_frame_reader_model import content, corruptions, frame

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
def eng():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    from tests import chain_enc_ref as ER
    from tests import chain_ref as CR
    up, ref = CR.Upstream(), oracle.Ref()
    return up, ref, ER.EncUpstream(), FR.upstream_engine(up, ref)


def call(k4, g, mem, streams, chunks, caps):
    """One read through host or device memory -> (results, used, ended, contents); checks the canaries."""
    import torch
    N = k4._native
    L = N.lib()
    n = len(streams)
    lens = np.array([len(c) for c in chunks], np.int32)
    so = np.zeros(n, np.int64)
    so[1:] = np.cumsum(lens[:-1], dtype=np.int64)
    src = np.frombuffer(b"".join(chunks) + b"\0" * 16, np.uint8).copy()
    dc = np.array(caps, np.int32)
    do = GAP + np.concatenate([[0], np.cumsum(np.maximum(dc[:-1], 0).astype(np.int64) + GAP)]).astype(np.int64)
    dst = np.full(int(do[-1]) + max(int(dc[-1]), 0) + GAP, CD, np.uint8)
    st = np.array(streams, np.int32)
    out = np.full(n, -7, np.int32)
    used = np.full(n, -7, np.int32)
    ended = np.full(n, -7, np.int32)
    if mem == "host":
        N.check(L.k4lz4_frame_reader_group_read(g.handle, st.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                lens.ctypes.data, used.ctypes.data, dst.ctypes.data, do.ctypes.data,
                                                dc.ctypes.data, out.ctypes.data, ended.ctypes.data, n, N.MEM_HOST,
                                                None))
    else:
        dev = torch.device("cuda", 0)
        T = lambda a: torch.from_numpy(a).to(dev)
        t = [T(a) for a in (st, src, so, lens, used, dst, do, dc, out, ended)]
        g.read_device(*[x.data_ptr() for x in t], n, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        used, dst, out, ended = t[4].cpu().numpy(), t[5].cpu().numpy(), t[8].cpu().numpy(), t[9].cpu().numpy()
    mask = np.ones(dst.shape[0], bool)
    for o, r, c in zip(do, out, dc):
        mask[o:o + (max(int(r), 0) if r >= 0 else max(int(c), 0))] = False
    assert (dst[mask] == CD).all(), np.nonzero(dst[mask] != CD)[0][:8]
    return out, used, ended, [dst[o:o + r].tobytes() if r > 0 else b"" for o, r in zip(do, out)]


def frame_decode(k4, f: bytes) -> int:
    """k4lz4_frame_decode_batch's result for one frame, with room for 2 MiB of content."""
    N = k4._native
    src = np.frombuffer(f + b"\0" * 16, np.uint8)
    zero = np.zeros(1, np.int64)
    sl = np.array([len(f)], np.int32)
    dc = np.array([1 << 21], np.int32)
    dst = np.zeros(1 << 21, np.uint8)
    r = np.zeros(1, np.int32)
    N.check(N.lib().k4lz4_frame_decode_batch(src.ctypes.data, zero.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                             zero.ctypes.data, dc.ctypes.data, r.ctypes.data, 1, N.MEM_HOST, None, 0))
    return int(r[0])


def end(k4, g, mem, streams):
    import torch
    if mem == "host":
        return g.end(streams)
    t = torch.tensor(streams, dtype=torch.int32, device="cuda")
    o = torch.full((len(streams),), -7, dtype=torch.int32, device="cuda")
    g.end_device(t.data_ptr(), o.data_ptr(), len(streams), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return o.cpu().numpy()


def drive(k4, g, models, blobs, rng, picks, cap_picks, max_calls=10000):
    """Feeds every stream its blob in random chunks, re-feeding what was not consumed, host and device memory
    alternating; every call equals the model.  -> the content per stream."""
    S = len(blobs)
    at = [0] * S
    got = [[] for _ in range(S)]
    for c in range(max_calls):
        live = [s for s in range(S) if at[s] < len(blobs[s])]
        if not live:
            break
        streams = [s for s in live if rng.random() < 0.8] or live[:1]
        rng.shuffle(streams)
        chunks = [blobs[s][at[s]:at[s] + int(picks[int(rng.integers(0, len(picks)))])] for s in streams]
        caps = [int(cap_picks[int(rng.integers(0, len(cap_picks)))]) for _ in streams]
        mem = "host" if c % 2 == 0 else "device"
        out, used, ended, data = call(k4, g, mem, streams, chunks, caps)
        for k, s in enumerate(streams):
            want = models[s].read(chunks[k], caps[k])
            assert (out[k], used[k], ended[k]) == want[:3], (c, mem, s, len(chunks[k]), caps[k], want[:3])
            assert data[k] == want[3]
            at[s] += int(used[k])
            got[s].append(data[k])
    for s in range(S):
        assert at[s] >= len(blobs[s])
    return [b"".join(x) for x in got]


def test_many_streams_equal_model(k4, eng):
    """4 224 streams, more than one wave of the decoder's CTA slots: the library's frames (linked / independent x
    block checksum x content checksum), upstream's linked and independent frames, empty frames, frames with a
    content-size field and raw stretches, two or three concatenated frames per stream."""
    up, ref, _, dec = eng
    S = 4224
    rng = np.random.default_rng(5)
    pool = content(3 << 20, 5)
    blobs, contents = [], []
    for s in range(S):
        parts, frames = [], []
        for j in range(2 + s % 2):
            n = [0, 17, 5000, 70000, 140000][int(rng.integers(0, 5))]
            o = int(rng.integers(0, len(pool) - n))
            d = pool[o:o + n]
            kind = (s + j) % 10
            if kind < 8:
                f = frame(eng, d, kind)
            elif kind == 8:
                f = up.frame_linked(d, 4, bool(s & 1), bool(s & 2))
            else:
                f = ref.frame_compress(d, bool(s & 1), bool(s & 2))
            parts.append(d)
            frames.append(f)
        blobs.append(b"".join(frames))
        contents.append(b"".join(parts))
    models = [FR.Reader(65536, dec, ref.xxh32) for _ in range(S)]
    k4.batch.decode_stats(0, reset=True)
    with k4.FrameReaderGroup(S, 65536) as g:
        got = drive(k4, g, models, blobs, rng, [1, 5, 19, 4095, 65537, 300000], [65535, 65544, 3 * 65544, 16 * 65544])
        st = end(k4, g, "device", list(range(S)))
        assert st.tolist() == [m.end() for m in models] and (st == 0).all()
    assert got == contents


def test_content_size_field_and_big_blocks(k4, eng):
    """Upstream linked frames at BD 4-7 in a 4 MiB group; a content-size field (built by hand)."""
    import struct
    from tests import frame_writer_ref as FW
    up, ref, _, dec = eng
    rng = np.random.default_rng(9)
    pool = content(6 << 20, 9)
    S = 24
    blobs, contents = [], []
    for s in range(S):
        n = int(rng.integers(0, 5 << 20))
        d = pool[:n]
        f = up.frame_linked(d, 4 + s % 4, bool(s & 1), bool(s & 2))
        if s % 5 == 0:                                   # the same frame with a content-size field
            flg = f[4] | 8
            h = bytes([flg, f[5]]) + struct.pack("<Q", n)
            f = f[:4] + h + bytes([(FW.xxh32(h) >> 8) & 0xFF]) + f[7:]
        blobs.append(f)
        contents.append(d)
    models = [FR.Reader(4 << 20, dec, ref.xxh32) for _ in range(S)]
    with k4.FrameReaderGroup(S, 4 << 20) as g:
        got = drive(k4, g, models, blobs, rng, [19, 65537, 1 << 20, 5 << 20], [(4 << 20) + 8, 3 << 22])
    assert got == contents


def test_verdicts_equal_frame_decode(k4, eng):
    """Every corruption class next to good streams in the same call; each verdict equals k4lz4_frame_decode_batch's
    on that frame; a failed stream stays failed, and reads a fresh frame after reset."""
    up, ref, _, dec = eng
    bad = corruptions(eng)
    good = frame(eng, content(100000, 1), 6)
    frames = [f for _, f in bad]
    for mem in ("host", "device"):
        with k4.FrameReaderGroup(2 * len(bad), 65536) as g:
            streams = list(range(2 * len(bad)))
            chunks = [x for f in frames for x in (f, good)]
            out, used, ended, data = call(k4, g, mem, streams, chunks, [1 << 22] * len(chunks))
            for k, (name, f) in enumerate(bad):
                r = frame_decode(k4, f)
                v = out[2 * k] if out[2 * k] < 0 else int(end(k4, g, mem, [2 * k])[0])
                if name == "big bd":
                    assert v == FR.DELEGATE and r == 1000
                else:
                    assert v == r, (name, v, r)
                assert out[2 * k + 1] == 100000 and ended[2 * k + 1] == 1
            failed = [2 * k for k in range(len(bad)) if out[2 * k] < 0]
            out2, used2, _, _ = call(k4, g, mem, failed, [good] * len(failed), [1 << 22] * len(failed))
            assert (out2 == out[failed]).all() and (used2 == 0).all()
            g.reset(failed)
            out3, _, ended3, d3 = call(k4, g, mem, failed, [good] * len(failed), [1 << 22] * len(failed))
            assert (out3 == 100000).all() and (ended3 == 1).all()


def test_verdicts_in_pieces(k4, eng):
    """The same corruptions fed in pieces of 13 (1 001 for long frames) and 5 000 bytes, so that long compressed blocks are skipped and
    their checksums cut across reads: each verdict (from a read, or from end()) equals the model's and, but for the
    BD above the group's maximum, k4lz4_frame_decode_batch's."""
    up, ref, _, dec = eng
    bad = corruptions(eng)
    want = [FR.DELEGATE if name == "big bd" else frame_decode(k4, f) for name, f in bad]
    for w in (13, 5000):
        models = [FR.Reader(65536, dec, ref.xxh32) for _ in bad]
        blobs = [f for _, f in bad]
        at = [0] * len(bad)
        verdict = [None] * len(bad)
        with k4.FrameReaderGroup(len(bad), 65536) as g:
            for c in range(100000):
                live = [k for k in range(len(bad)) if verdict[k] is None and at[k] < len(blobs[k])]
                if not live:
                    break
                # pieces of 13 bytes cut headers and checksums; the long frames take 1 001-byte pieces
                chunks = [blobs[k][at[k]:at[k] + (w if len(blobs[k]) < 4096 else max(w, 1001))] for k in live]
                out, used, ended, data = call(k4, g, "host" if c % 2 else "device", live, chunks, [1 << 20] * len(live))
                for j, k in enumerate(live):
                    m = models[k].read(chunks[j], 1 << 20)
                    assert (out[j], used[j], ended[j]) == m[:3] and data[j] == m[3], (bad[k][0], w, c)
                    if out[j] < 0:
                        verdict[k] = int(out[j])
                    at[k] += int(used[j])
            st = end(k4, g, "device", list(range(len(bad))))
        for k, (name, _) in enumerate(bad):
            v = verdict[k] if verdict[k] is not None else int(st[k])
            assert v == models[k].end() == want[k], (name, w, v, want[k])


def test_end_room_and_counters(k4, eng):
    """end() at every phase of a frame; dstCap < blockCap consumes a header and a complete end mark but no block
    byte; clean linked data never reaches the exact engine."""
    up, ref, _, dec = eng
    f = frame(eng, content(70000, 3), 6)
    cuts = list(range(0, 20)) + [len(f) - k for k in range(0, 12)] + list(range(20, len(f), 997))
    with k4.FrameReaderGroup(len(cuts), 65536) as g:
        for mem in ("host", "device"):
            out, used, ended, _ = call(k4, g, mem, list(range(len(cuts))), [f[:c] for c in cuts], [1 << 20] * len(cuts))
            st = end(k4, g, mem, list(range(len(cuts))))
            for k, c in enumerate(cuts):
                assert st[k] == (0 if c in (0, len(f)) else FR.CORRUPT), c
    e = frame(eng, b"", 4)
    with k4.FrameReaderGroup(2, 65536) as g:
        for mem in ("host", "device"):
            out, used, ended, _ = call(k4, g, mem, [0, 1], [f, e], [65535, 0])
            assert used.tolist() == [7, len(e)] and ended.tolist() == [0, 1] and out.tolist() == [0, 0]
            g.reset()
    data = content(1 << 20, 4)
    fr = [frame(eng, data, 0) for _ in range(64)]
    k4.batch.decode_stats(0, reset=True)
    with k4.FrameReaderGroup(64, 65536) as g:
        got, res = g.read_all(fr, 16 * 65536)
    stats = k4.batch.decode_stats(0, reset=True)
    assert got == [data] * 64 and (res == len(data)).all()
    assert stats["generic"] == 0 and stats["tile"] > 0, stats
