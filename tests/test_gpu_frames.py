"""Whole LZ4 frames on the GPU (k4lz4_frame_encode_batch / _decode_batch / _content_size_batch, LZ4Frame).

Encoded frames are compared byte for byte with the reference's writer restated over upstream's engine
(tests/chain_enc_ref.frame_linked_ref for linked blocks, `indep_ref` below for independent ones) and decoded by
upstream lz4frame.c; decoded frames come from upstream's writer, the reference's writer and ours.  Destinations
are surrounded by 0xCD canaries.  Needs the reference engine that __graft_entry__.build() compiles into
oracle/_ref/."""
import struct

import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests import chain_ref as CR

pytestmark = pytest.mark.gpu
CD = 0xCD
GAP = 64


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


def indep_ref(ref, data: bytes, bs: int, bc: bool, cc: bool) -> bytes:
    """LZ4FrameWriter with Chaining = false: every block through upstream's LZ4_compress_fast with capacity
    MaximumOutputSize(blockSize), stored raw when it does not shrink."""
    code = {1 << 16: 4, 1 << 18: 5, 1 << 20: 6, 1 << 22: 7}[bs]
    head = struct.pack("<IBB", 0x184D2204, 0x40 | 0x20 | (int(bc) << 4) | (int(cc) << 2), code << 4)
    out = [head, bytes([(ref.xxh32(head[4:6]) >> 8) & 0xFF])]
    for o in range(0, len(data), bs):
        blk = data[o:o + bs]
        r, enc = ref.encode(blk, bs + bs // 255 + 16)
        assert r > 0
        body = blk if r >= len(blk) else enc
        out.append(struct.pack("<I", len(body) | (0x80000000 if r >= len(blk) else 0)))
        out.append(body)
        if bc:
            out.append(struct.pack("<I", ref.xxh32(body)))
    out.append(struct.pack("<I", 0))
    if cc:
        out.append(struct.pack("<I", ref.xxh32(data)))
    return b"".join(out)


def content(rng, n: int, noise: bool = True) -> bytes:
    """datagen 0.63 with an incompressible stretch (it becomes a raw block)."""
    import oracle
    a = oracle.Port().datagen(max(n, 1), 0.63, 0.0, int(rng.integers(1, 1 << 30)))[:n].copy()
    if noise and n > 1000:
        at = int(rng.integers(0, n // 2))
        k = min(n - at, 70000)
        a[at:at + k] = rng.integers(0, 256, k, dtype=np.uint8)
    return a.tobytes()


def layout(sizes, caps):
    """Packed sources and canaried destination slots -> (src, srcOff, srcLen, dst, dstOff, dstCap)."""
    so = np.zeros(len(sizes), dtype=np.int64)
    at = 0
    for i, s in enumerate(sizes):
        so[i] = at
        at += len(s) + 3                     # odd phases
    src = np.zeros(at + 16, dtype=np.uint8)
    for o, s in zip(so, sizes):
        src[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    do = np.zeros(len(caps), dtype=np.int64)
    at = GAP
    for i, c in enumerate(caps):
        do[i] = at
        at += max(int(c), 0) + GAP + (i % 5)
    dst = np.full(at + GAP, CD, dtype=np.uint8)
    return src, so, np.array([len(s) for s in sizes], dtype=np.int32), dst, do, np.array(caps, dtype=np.int32)


def run(k4, what, items, caps=None, mem="device", **kw):
    """One frame call through device or host memory -> (results, dst, dstOff, dstCap)."""
    import torch
    N = k4._native
    L = N.lib()
    src, so, sl, dst, do, dc = layout(items, caps if caps is not None else [0] * len(items))
    n = len(items)
    out = np.full(n, 12345, dtype=np.int32)
    if mem == "host":
        if what == "encode":
            rc = L.k4lz4_frame_encode_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                            do.ctypes.data, dc.ctypes.data, out.ctypes.data, n, kw["bs"], kw["flags"],
                                            kw.get("level", 0), N.MEM_HOST, None, 0)
        elif what == "decode":
            rc = L.k4lz4_frame_decode_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                            do.ctypes.data, dc.ctypes.data, out.ctypes.data, n, N.MEM_HOST, None, 0)
        else:
            rc = L.k4lz4_frame_content_size_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, out.ctypes.data, n,
                                                  N.MEM_HOST, None, 0)
        N.check(rc)
        return out, dst, do, dc
    dev = torch.device("cuda", 0)
    t = {k: torch.from_numpy(v.copy()).to(dev) for k, v in dict(src=src, so=so, sl=sl, dst=dst, do=do, dc=dc).items()}
    o = torch.from_numpy(out).to(dev)
    st = torch.cuda.current_stream().cuda_stream
    F = k4.LZ4Frame
    if what == "encode":
        F.encode_many_device(t["src"], t["so"], t["sl"], t["dst"], t["do"], t["dc"], o, kw["bs"],
                             not (kw["flags"] & 1), bool(kw["flags"] & 2), bool(kw["flags"] & 4), kw.get("level", 0), st)
    elif what == "decode":
        F.decode_many_device(t["src"], t["so"], t["sl"], t["dst"], t["do"], t["dc"], o, st)
    else:
        F.content_sizes_device(t["src"], t["so"], t["sl"], o, st)
    torch.cuda.synchronize()
    return o.cpu().numpy(), t["dst"].cpu().numpy(), do, dc


def check_canaries(dst, do, dc, res):
    """Bytes outside every destination, and inside it beyond a successful result, are still 0xCD."""
    mask = np.ones(dst.shape[0], dtype=bool)
    for o, c, r in zip(do, dc, res):
        mask[o:o + (c if r < 0 else r)] = False
    assert (dst[mask] == CD).all(), np.nonzero(dst[mask] != CD)[0][:8]


def flags_of(chaining, bc, cc):
    return (0 if chaining else 1) | (2 if bc else 0) | (4 if cc else 0)


# ---- encode -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bs", [1 << 16, 1 << 18, 1 << 20, 1 << 22])
def test_encode_bytes_equal_reference_writer(k4, ref, up, bs):
    rng = np.random.default_rng(bs)
    sizes = [0, 1, bs - 1, bs, bs + 1, 2 * bs + bs // 3] if bs < (1 << 22) else [0, 1, bs - 1, bs + 1, 2 * bs + 7]
    items = [content(rng, n) for n in sizes]
    combos = [(False, False), (True, False), (False, True), (True, True)] if bs == 1 << 16 else [(False, False), (True, True)]
    raws = 0
    for chaining in (True, False):
        for bc, cc in combos:
            fl = flags_of(chaining, bc, cc)
            caps = [int(k4._native.lib().k4lz4_frame_bound(len(c), bs, fl)) for c in items]
            res, dst, do, dc = run(k4, "encode", items, caps, bs=bs, flags=fl)
            check_canaries(dst, do, dc, res)
            for c, r, o in zip(items, res, do):
                f = dst[o:o + r].tobytes()
                want = ER.frame_linked_ref(up, c, bs, bc, cc) if chaining else indep_ref(ref, c, bs, bc, cc)
                assert f == want, (bs, chaining, bc, cc, len(c))
                assert ref.frame_decompress(f, len(c) + 16) == c
                raws += sum(k4.frame._Frame(f).raws)
    assert raws > 0


def test_encode_many_frames_host_equals_device(k4, ref, up):
    rng = np.random.default_rng(3)
    items = [content(rng, int(n), noise=bool(i % 3 == 0)) for i, n in enumerate(rng.integers(0, 300000, 260))]
    items[5] = b""
    for chaining in (True, False):
        fl = flags_of(chaining, True, True)
        caps = [int(k4._native.lib().k4lz4_frame_bound(len(c), 65536, fl)) for c in items]
        # do not fit: -1, nothing at or beyond dstCap -- no room for the header / one byte short of the frame
        exact8 = ER.frame_linked_ref(up, items[8], 65536, True, True) if chaining else indep_ref(ref, items[8], 65536, True, True)
        caps[7], caps[8] = 12, len(exact8) - 1
        rd, dd, do, dc = run(k4, "encode", items, caps, bs=65536, flags=fl)
        rh, dh, _, _ = run(k4, "encode", items, caps, mem="host", bs=65536, flags=fl)
        assert rd.tolist() == rh.tolist() and rd[7] == -1 and rd[8] == -1
        check_canaries(dd, do, dc, rd)
        for i, c in enumerate(items):
            if i in (7, 8):
                continue
            f = dd[do[i]:do[i] + rd[i]].tobytes()
            assert f == dh[do[i]:do[i] + rh[i]].tobytes()
            if i % 37 == 0:
                want = ER.frame_linked_ref(up, c, 65536, True, True) if chaining else indep_ref(ref, c, 65536, True, True)
                assert f == want
        res, dst, do, dc = run(k4, "encode", items[:4], [1 << 20] * 4, bs=65536, flags=fl, level=3)
        assert res.tolist() == [k4._native.R_DELEGATE] * 4 and (dst == CD).all()


def test_write_frames_python_mirror(k4, up):
    from k4os.compression.lz4_b200 import frame as F
    rng = np.random.default_rng(9)
    items = [content(rng, n) for n in (0, 100, 200000)]
    assert F.write_frames(items, 65536, True, False) == [ER.frame_linked_ref(up, c, 65536, True, False) for c in items]
    assert F.read_frames(F.write_frames(items, 1 << 20)) == items
    assert F.LZ4Frame.Decode(F.LZ4Frame.Encode(items[2], 1 << 18, chaining=False)) == items[2]
    with pytest.raises(NotImplementedError):
        F.write_frames(items, 65536, level=3)
    with pytest.raises(RuntimeError):
        F.write_frame(items[1], 65536, level=9)
    with pytest.raises(ValueError):
        F.write_frame(items[1], (4 << 20) + 1)


# ---- decode -------------------------------------------------------------------------------------------------

def test_decode_mixed_batch(k4, ref, up):
    rng = np.random.default_rng(11)
    frames, contents = [], []
    cup = CR.Upstream()
    for sid in (4, 5, 6, 7):
        for bc, cc in ((False, False), (True, True), (True, False)):
            n = int(rng.integers(1, 3 << (2 * sid + 8))) if sid < 7 else 9_000_000
            c = content(rng, n)
            frames.append(cup.frame_linked(c, sid, bc, cc)); contents.append(c)
    for _ in range(24):
        c = content(rng, int(rng.integers(70000, 400000)))
        frames.append(cup.frame_linked(c, 4, bool(rng.integers(0, 2)), bool(rng.integers(0, 2)))); contents.append(c)
    for bc, cc in ((False, False), (True, True)):
        c = content(rng, 300000)
        frames.append(ref.frame_compress(c, bc, cc)); contents.append(c)
        frames.append(indep_ref(ref, c, 1 << 18, bc, cc)); contents.append(c)
        frames.append(ER.frame_linked_ref(up, c, 1 << 16, bc, cc)); contents.append(c)
    for bc, cc in ((False, False), (True, True)):
        frames.append(ER.frame_linked_ref(up, b"", 1 << 16, bc, cc)); contents.append(b"")
        frames.append(cup.frame_linked(b"", 4, bc, cc)); contents.append(b"")
        frames.append(cup.frame_linked(b"x", 4, bc, cc)); contents.append(b"x")
    lens = [len(c) for c in contents]
    for mem in ("device", "host"):
        sz, _, _, _ = run(k4, "size", frames, mem=mem)
        assert sz.tolist() == lens
        res, dst, do, dc = run(k4, "decode", frames, lens, mem=mem)
        assert res.tolist() == lens
        check_canaries(dst, do, dc, res)
        assert [dst[o:o + n].tobytes() for o, n in zip(do, lens)] == contents
    assert k4.frame.read_frames(frames) == contents
    # clean 64 KiB-block frames never leave the tile path
    clean = [cup.frame_linked(content(rng, 1 << 20, noise=False), 4) for _ in range(16)]
    clean += [k4.frame.write_frame(content(rng, 1 << 20, noise=False), 65536) for _ in range(16)]
    k4.batch.decode_stats(0, reset=True)
    res, _, _, _ = run(k4, "decode", clean, [1 << 20] * 32)
    stats = k4.batch.decode_stats(0, reset=True)
    assert res.tolist() == [1 << 20] * 32
    assert stats["generic"] == 0 and stats["tile"] + stats["tile_big"] > 0, stats


def _hdr(flg: int, bd: int = 0x40) -> bytes:
    import oracle
    h = struct.pack("<IBB", 0x184D2204, flg, bd)
    return h + bytes([(oracle.Port().xxh32(np.frombuffer(h[4:6], dtype=np.uint8)) >> 8) & 0xFF])


def test_error_classes_in_one_call(k4, up):
    N = k4._native
    rng = np.random.default_rng(21)
    c = content(rng, 200000)
    good = ER.frame_linked_ref(up, c, 65536, True, True)
    fr = k4.frame._Frame(good)
    cases = []

    def bad(edit, code):
        f = bytearray(good)
        f = edit(f)
        cases.append((bytes(f), code))

    def put(f, at, v):
        f[at] ^= v
        return f
    bad(lambda f: put(f, 0, 1), N.R_CORRUPT)                                     # magic
    bad(lambda f: put(f, 4, 0xC0), N.R_CORRUPT)                                  # version 10 (0x11 mask: 0)
    bad(lambda f: put(f, 6, 1), N.R_CORRUPT)                                     # header checksum
    bad(lambda f: f[:9], N.R_CORRUPT)                                            # length code cut off
    bad(lambda f: f[:fr.pos[1] + 100], N.R_CORRUPT)                              # body cut off
    bad(lambda f: put(f, fr.pos[0] + fr.lens[0], 1), N.R_CORRUPT)                # block checksum
    bad(lambda f: put(f, len(f) - 1, 1), N.R_CORRUPT)                            # content checksum
    bad(lambda f: put(f, 4, 1), N.R_DELEGATE)                                    # dictionary id flag
    blk = bytes([0x10, 0x61, 0x64, 0x00, 0x50]) + b"bcdef"                       # offset 100 behind 1 byte
    corrupt = _hdr(0x60) + struct.pack("<I", len(blk)) + blk + struct.pack("<I", 0)
    cases.append((corrupt, -1))
    big = bytes(rng.integers(0, 256, 65545, dtype=np.uint8))
    cases.append((_hdr(0x60) + struct.pack("<I", 0x80000000 | len(big)) + big + struct.pack("<I", 0), N.R_CORRUPT))
    cases.append((_hdr(0x40) + struct.pack("<I", 0x80000000 | 65537) + big[:65537] + struct.pack("<I", 0), N.R_CORRUPT))
    ok_linked = _hdr(0x40) + struct.pack("<I", 0x80000000 | 65536) + big[:65536] + struct.pack("<I", 0)
    frames = [good] + [f for f, _ in cases] + [good, ok_linked, good]
    want = [len(c)] + [w for _, w in cases] + [N.R_DST_SMALL, 65536, len(c)]
    caps = [len(c)] + [len(c)] * len(cases) + [len(c) - 1, 65536, len(c)]
    for mem in ("device", "host"):
        res, dst, do, dc = run(k4, "decode", frames, caps, mem=mem)
        assert res.tolist() == want, mem
        check_canaries(dst, do, dc, res)
        for i in (0, len(frames) - 1):
            assert dst[do[i]:do[i] + len(c)].tobytes() == c
    sz, _, _, _ = run(k4, "size", frames)
    assert sz[0] == len(c) and sz[1:4].tolist() == [N.R_CORRUPT] * 3 and sz[8] == N.R_DELEGATE
    assert sz[4] == N.R_CORRUPT and sz[9] == 10
    with pytest.raises(k4.frame.InvalidDataException):
        k4.frame.read_frame(corrupt)
    with pytest.raises(NotImplementedError):
        k4.frame.read_frame(cases[7][0])


@pytest.mark.parametrize("chaining", [True, False])
def test_untouched_bytes_and_scratch_slots(k4, up, ref, chaining):
    """dstCap exact (the last blocks need the reference's slack beyond it: scratch slots), larger, one short;
    frames of 1 KiB blocks declare 64 KiB, so every block of their last 64 KiB decodes in a scratch slot."""
    rng = np.random.default_rng(31 + chaining)
    cs = [content(rng, n) for n in (3 * 65536 + 100, 4 * 65536, 65536 - 3, 150000, 5000)]
    frames = k4.frame.write_frames(cs[:4], 65536, True, True, chaining=chaining)
    frames += k4.frame.write_frames(cs[3:], 1024, True, True, chaining=chaining)
    cs = cs[:4] + cs[3:]
    for f, c in zip(frames, cs):
        assert ref.frame_decompress(f, len(c) + 16) == c
    lens = [len(c) for c in cs]
    for extra, want in ((0, lens), (37, lens), (-1, [k4._native.R_DST_SMALL] * len(cs))):
        for mem in ("device", "host"):
            res, dst, do, dc = run(k4, "decode", frames, [n + extra for n in lens], mem=mem)
            assert res.tolist() == want, (extra, mem)
            check_canaries(dst, do, dc, res)
            if extra >= 0:
                assert [dst[o:o + n].tobytes() for o, n in zip(do, lens)] == cs
