"""Byte reads of frame reader groups on the GPU (k4lz4_frame_reader_group_read_bytes, FrameReaderGroup.read_bytes):
every call's result, bytes consumed, frame end and content equal the push model (tests/frame_reader_bytes_ref.py)
over upstream's engines, through host and device memory alternately, with 0xCD canaries around every destination;
caps of any size, both modes, 64 KiB and 4 MiB blocks (first blocks above 64 KiB: the deferred slide).  Verdicts
equal k4lz4_frame_decode_batch's; mixing with read, end and reset; sub-reads.  Needs oracle/_ref/."""
import numpy as np
import pytest

from tests import frame_reader_bytes_ref as RB
from tests import frame_reader_ref as FR
from tests.test_frame_reader_model import content, corruptions, frame
from tests.test_gpu_frame_reader import GAP, CD, end, eng, frame_decode, k4  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
CAPS = [0, 1, 3, 4096, 65535, 65536, 65544, 200000]


def call(k4, g, mem, streams, chunks, caps, interactive=False, plain=False):
    """One read_bytes (plain: read) through host or device memory -> (results, used, ended, contents)."""
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
    fl = N.READ_INTERACTIVE if interactive else 0
    if mem == "host":
        args = [g.handle, st.ctypes.data, src.ctypes.data, so.ctypes.data, lens.ctypes.data, used.ctypes.data,
                dst.ctypes.data, do.ctypes.data, dc.ctypes.data, out.ctypes.data, ended.ctypes.data, n]
        if plain:
            N.check(L.k4lz4_frame_reader_group_read(*args, N.MEM_HOST, None))
        else:
            N.check(L.k4lz4_frame_reader_group_read_bytes(*args, fl, N.MEM_HOST, None))
    else:
        dev = torch.device("cuda", 0)
        t = [torch.from_numpy(a).to(dev) for a in (st, src, so, lens, used, dst, do, dc, out, ended)]
        ptrs = [x.data_ptr() for x in t]
        s = torch.cuda.current_stream().cuda_stream
        if plain:
            g.read_device(*ptrs, n, stream=s)
        else:
            g.read_bytes_device(*ptrs, n, interactive=interactive, stream=s)
        torch.cuda.synchronize()
        used, dst, out, ended = t[4].cpu().numpy(), t[5].cpu().numpy(), t[8].cpu().numpy(), t[9].cpu().numpy()
    mask = np.ones(dst.shape[0], bool)
    for o, r, c in zip(do, out, dc):
        mask[o:o + (max(int(r), 0) if r >= 0 else max(int(c), 0))] = False
    assert (dst[mask] == CD).all(), np.nonzero(dst[mask] != CD)[0][:8]
    assert all(r <= max(c, 0) for r, c in zip(out, dc))
    return out, used, ended, [dst[o:o + r].tobytes() if r > 0 else b"" for o, r in zip(do, out)]


def drive(k4, g, models, blobs, rng, picks, cap_picks, max_calls=20000):
    """Feeds every stream its blob in random chunks with random caps and modes until it is consumed and drained;
    every call equals the model.  -> the content per stream."""
    S = len(blobs)
    at = [0] * S
    got = [[] for _ in range(S)]
    for c in range(max_calls):
        live = [s for s in range(S) if at[s] < len(blobs[s]) or models[s].pending]
        if not live:
            break
        streams = [s for s in live if rng.random() < 0.8] or live[:1]
        rng.shuffle(streams)
        chunks = [blobs[s][at[s]:at[s] + int(picks[int(rng.integers(0, len(picks)))])] for s in streams]
        caps = [int(cap_picks[int(rng.integers(0, len(cap_picks)))]) for _ in streams]
        inter = bool(c % 3 == 2)
        mem = "host" if c % 2 == 0 else "device"
        out, used, ended, data = call(k4, g, mem, streams, chunks, caps, inter)
        for k, s in enumerate(streams):
            want = models[s].read_bytes(chunks[k], caps[k], inter)
            assert (out[k], used[k], ended[k]) == want[:3], (c, mem, inter, s, len(chunks[k]), caps[k], want[:3])
            assert data[k] == want[3], (c, mem, s)
            at[s] += int(used[k])
            got[s].append(data[k])
    assert all(at[s] >= len(blobs[s]) and not models[s].pending for s in range(S))
    return [b"".join(x) for x in got]


def test_many_streams_equal_model(k4, eng):
    """4 224 streams: linked and independent frames with and without both checksums, upstream's frames, empty
    frames, two or three concatenated frames per stream."""
    up, ref, _, dec = eng
    S = 4224
    rng = np.random.default_rng(15)
    pool = content(3 << 20, 15)
    blobs, contents = [], []
    for s in range(S):
        parts, frames = [], []
        for j in range(2 + s % 2):
            n = [0, 17, 5000, 70000, 140000][int(rng.integers(0, 5))]
            o = int(rng.integers(0, len(pool) - n))
            d = pool[o:o + n]
            kind = (s + j) % 10
            f = frame(eng, d, kind) if kind < 8 else (up.frame_linked(d, 4, bool(s & 1), bool(s & 2)) if kind == 8
                                                      else ref.frame_compress(d, bool(s & 1), bool(s & 2)))
            parts.append(d)
            frames.append(f)
        blobs.append(b"".join(frames))
        contents.append(b"".join(parts))
    models = [RB.BytesReader(65536, dec, ref.xxh32) for _ in range(S)]
    with k4.FrameReaderGroup(S, 65536) as g:
        got = drive(k4, g, models, blobs, rng, [1, 5, 19, 4095, 65537, 300000], CAPS)
        st = end(k4, g, "device", list(range(S)))
        assert st.tolist() == [m.end() for m in models] and (st == 0).all()
    assert got == contents


def test_big_blocks_and_the_slide(k4, eng):
    """4 MiB groups: upstream linked frames at BD 4-7 whose first block exceeds 64 KiB, drained a little at a time
    so that more than 64 KiB stay undrained when the ring would slide."""
    up, ref, _, dec = eng
    rng = np.random.default_rng(19)
    pool = content(6 << 20, 19)
    S = 16
    blobs, contents = [], []
    for s in range(S):
        n = int(rng.integers(1 << 20, 5 << 20))
        d = pool[:n]
        blobs.append(up.frame_linked(d, 4 + s % 4, bool(s & 1), bool(s & 2)))
        contents.append(d)
    models = [RB.BytesReader(4 << 20, dec, ref.xxh32) for _ in range(S)]
    with k4.FrameReaderGroup(S, 4 << 20) as g:
        got = drive(k4, g, models, blobs, rng, [65537, 1 << 20, 5 << 20], [4096, 65536, 200000, 3 << 20], 5000)
    assert got == contents


def test_verdicts_equal_frame_decode(k4, eng):
    up, ref, _, dec = eng
    bad = [(n, f) for n, f in corruptions(eng) if n != "big bd"]
    for mem, cap in (("host", 4096), ("device", 65536), ("host", 1 << 22)):
        models = [RB.BytesReader(65536, dec, ref.xxh32) for _ in bad]
        with k4.FrameReaderGroup(len(bad), 65536) as g:
            at = [0] * len(bad)
            verdict = [None] * len(bad)
            for c in range(10000):
                live = [k for k in range(len(bad)) if verdict[k] is None and
                        (at[k] < len(bad[k][1]) or models[k].pending)]
                if not live:
                    break
                chunks = [bad[k][1][at[k]:at[k] + 5000] for k in live]
                out, used, ended, data = call(k4, g, mem if c % 2 else "device", live, chunks, [cap] * len(live))
                stuck = []
                for j, k in enumerate(live):
                    m = models[k].read_bytes(chunks[j], cap)
                    assert (out[j], used[j], ended[j]) == m[:3] and data[j] == m[3], (bad[k][0], c)
                    if out[j] < 0:
                        verdict[k] = int(out[j])
                    at[k] += int(used[j])
                    if used[j] == 0 and out[j] == 0 and not ended[j]:
                        stuck.append(k)
                for k in stuck:
                    verdict[k] = "end"
            st = end(k4, g, "device", list(range(len(bad))))
        for k, (name, f) in enumerate(bad):
            v = verdict[k] if isinstance(verdict[k], int) else int(st[k])
            assert v == frame_decode(k4, f), (name, mem, v)


def test_mixing_end_reset_and_sub_reads(k4, eng):
    """read on a stream with undrained bytes: K4LZ4_E_ARG, nothing consumed, not failed, and read_bytes goes on;
    end and reset discard undrained bytes (end: R_CORRUPT); a host read equals the same read cut in two."""
    up, ref, _, dec = eng
    data = content(300000, 21)
    f = frame(eng, data, 6)
    for mem in ("host", "device"):
        with k4.FrameReaderGroup(4, 65536) as g:
            out, used, ended, d = call(k4, g, mem, [0, 1, 2, 3], [f] * 4, [4096] * 4)
            assert (out == 4096).all()
            o2, u2, e2, _ = call(k4, g, mem, [0], [f[used[0]:]], [1 << 20], plain=True)
            assert o2[0] == FR.ARG and u2[0] == 0
            rest, at = [d[0]], int(used[0])
            while True:
                o, u, e, dd = call(k4, g, mem, [0], [f[at:]], [1 << 20])
                rest.append(dd[0])
                at += int(u[0])
                if e[0]:
                    break
            assert b"".join(rest) == data
            assert end(k4, g, mem, [1]).tolist() == [FR.CORRUPT]
            g.reset([2])
            for s in (1, 2):
                o, u, e, dd = call(k4, g, mem, [s], [f], [1 << 22])
                assert o[0] == len(data) and e[0] == 1 and dd[0] == data
    # flags other than 0 or K4LZ4_READ_INTERACTIVE: K4LZ4_E_ARG, after _read's checks, with n = 0 as well
    N = k4._native
    with k4.FrameReaderGroup(2, 65536) as g:
        z = np.zeros(4, np.int32)
        o = np.zeros(4, np.int64)
        bb = np.zeros(16, np.uint8)
        p = [z.ctypes.data, bb.ctypes.data, o.ctypes.data, z.ctypes.data, z.ctypes.data, bb.ctypes.data,
             o.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data]
        for flags in (2, -1, 3):
            for cnt in (0, 1):
                assert N.lib().k4lz4_frame_reader_group_read_bytes(g.handle, *p, cnt, flags, N.MEM_HOST, None) == -102
        assert N.lib().k4lz4_frame_reader_group_read_bytes(g.handle, *p, -1, 2, N.MEM_HOST, None) == -102
        assert N.lib().k4lz4_frame_reader_group_read_bytes(g.handle, *p, 1, 0, 7, None) == -102
    # sub-reads: the reader's host path cuts a read into pieces of at most 256 MiB; a frame fed in two calls of
    # one byte-read each equals one call (cutting changes nothing)
    with k4.FrameReaderGroup(2, 65536) as g:
        whole = call(k4, g, "host", [0], [f], [200000])
        a = call(k4, g, "host", [1], [f[:1000]], [200000])
        b = call(k4, g, "host", [1], [f[int(a[1][0]):]], [200000 - int(a[0][0])])
        assert a[3][0] + b[3][0] == whole[3][0] and int(a[1][0]) + int(b[1][0]) == int(whole[1][0])


def zero_block() -> bytes:
    """An LZ4 block of 65 536 zero bytes in 267: one literal, a match at offset 1 over 65 530 bytes, 5 literals."""
    ext = 65530 - 4 - 15
    return bytes([0x1F, 0x00, 0x01, 0x00]) + b"\xff" * (ext // 255) + bytes([ext % 255, 0x50]) + bytes(5)


def test_int32_max_cap_through_host_staging(k4, eng):
    """dstCap = INT32_MAX on a frame of 32 768 zero blocks (2 GiB of content in 8.7 MB), through the Python host
    wrapper: the read fills all 2^31 - 1 bytes of room, leaves the last byte undrained and the end mark unread;
    the next read returns that byte and ends the frame."""
    import struct
    from tests import frame_writer_ref as FW
    up, ref, _, dec = eng
    blk = zero_block()
    assert ref.decode(blk, 65544) == (65536, bytes(65536))
    f = FW.header(65536, False, False, False) + (struct.pack("<I", len(blk)) + blk) * 32768 + bytes(4)
    cap = (1 << 31) - 1
    with k4.FrameReaderGroup(1, 65536) as g:
        got, out, used, ended = g.read_bytes([f], [cap])
        assert (int(out[0]), int(used[0]), int(ended[0])) == (cap, len(f) - 4, 0)
        assert len(got[0]) == cap and not np.frombuffer(got[0], np.uint8).any()
        del got
        got, out, used, ended = g.read_bytes([f[len(f) - 4:]], [16])
        assert (int(out[0]), int(used[0]), int(ended[0])) == (1, 4, 1) and got[0] == b"\0"
        assert g.end([0]).tolist() == [0]


@pytest.mark.parametrize("interactive", [False, True])
def test_host_read_over_256_mib_in_sub_reads(k4, eng, interactive):
    """One host read whose chunks total more than 256 MiB, so that it runs as several sub-reads, at small and large
    caps and a second read from where the first stopped: every entry equals the push model and the same reads
    through device memory.  Plain reads too, whose room in blocks carries over from one sub-read to the next."""
    up, ref, _, dec = eng
    rng = np.random.default_rng(23)
    noise = rng.integers(0, 256, 24 << 20, dtype=np.uint8).tobytes()
    text = content(12 << 20, 23)
    S = 80
    blobs = []
    for s in range(S):
        o1, o2 = int(rng.integers(0, 20 << 20)), int(rng.integers(0, 9 << 20))
        d = noise[o1:o1 + (3 << 20)] + text[o2:o2 + (2 << 20) + s * 4099]
        fr, _ = k4.LZ4Frame.EncodeMany([d], 65536, not s & 1, bool(s & 2), bool(s & 4))
        blobs.append(fr[0])
    assert sum(len(b) for b in blobs) > 300 << 20
    arms = [(cap, False) for cap in (4096, 16 << 20)]
    if not interactive:
        arms += [(cap, True) for cap in (1 << 20, 16 << 20)]
    for cap, plain in arms:
        models = [RB.BytesReader(65536, dec, ref.xxh32) for _ in range(S)]
        at = [0] * S
        streams = list(range(S))[::-1]
        with k4.FrameReaderGroup(S, 65536) as gh, k4.FrameReaderGroup(S, 65536) as gd:
            for rnd in range(2):
                chunks = [blobs[s][at[s]:] for s in streams]
                if plain:
                    got, out, used, ended = gh.read(chunks, [cap] * S, streams)
                else:
                    got, out, used, ended = gh.read_bytes(chunks, [cap] * S, streams, interactive=interactive)
                dout, dused, dended, dgot = call(k4, gd, "device", streams, chunks, [cap] * S, interactive, plain)
                assert out.tolist() == dout.tolist() and used.tolist() == dused.tolist()
                assert ended.tolist() == dended.tolist() and got == dgot
                for k, s in enumerate(streams):
                    m = models[s]
                    want = m.read(chunks[k], cap) if plain else m.read_bytes(chunks[k], cap, interactive)
                    assert (out[k], used[k], ended[k]) == want[:3], (cap, plain, rnd, s, want[:3])
                    assert got[k] == want[3], (cap, plain, rnd, s)
                    at[s] += int(used[k])
