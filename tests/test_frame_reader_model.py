"""Frame reader groups without a GPU: the incremental LZ4FrameReader model (tests/frame_reader_ref.py) over
upstream's engines, against upstream's whole-frame decoder, on every cut of small frames and random cuts of 1 MiB
frames, and its verdicts against the whole-frame verdict order.  Needs upstream's engine (oracle/_ref/)."""
import struct

import numpy as np
import pytest

from tests import frame_reader_ref as FR
from tests import frame_writer_ref as FW


@pytest.fixture(scope="module")
def eng():
    import oracle
    if not oracle.have_ref():
        pytest.skip("upstream's engine (oracle/_ref/) is not built")
    from tests import chain_enc_ref as ER
    from tests import chain_ref as CR
    up, ref = CR.Upstream(), oracle.Ref()
    return up, ref, ER.EncUpstream(), FR.upstream_engine(up, ref)


def content(n, seed):
    import oracle
    a = oracle.Port().datagen(max(n, 1), 0.63, 0.0, seed)[:n].copy()
    if n > 3000:
        rng = np.random.default_rng(seed)
        at = int(rng.integers(0, n // 2))
        k = min(n - at, 70000)
        a[at:at + k] = rng.integers(0, 256, k, dtype=np.uint8)
    return a.tobytes()


def frame(eng, data, fl, bs=65536):
    up, ref, eup, _ = eng
    chaining = not fl & 1
    w = FW.Writer(bs, chaining, bool(fl & 2), bool(fl & 4), FW.UpstreamEngine(eup, ref, chaining), ref.xxh32)
    return b"".join(FW.emit(w, [data]))


def feed(reader, data, cuts, cap):
    """Feeds data cut at `cuts`, re-feeding unconsumed bytes -> (content, results per call)."""
    out, calls, at = [], [], 0
    bounds = sorted(set(c for c in cuts if 0 < c < len(data))) + [len(data)]
    for b in bounds:
        while at < b:
            res, used, ended, got = reader.read(data[at:b], cap)
            calls.append((res, used, ended))
            assert res >= 0, calls[-1]
            out.append(got)
            at += used
            if used == 0 and not ended:
                break
    return b"".join(out), calls


@pytest.mark.parametrize("fl", range(8))
def test_every_cut_of_small_frames(eng, fl):
    """Every single cut and caps {0, blockCap - 1, blockCap, 3 blockCap}: the content equals upstream's decoder."""
    up, ref, _, dec = eng
    for n in (0, 5, 100):
        data = content(n, n + fl)
        f = frame(eng, data, fl)
        cap_b = 65536 + (8 if fl & 1 else 0)
        assert ref.frame_decompress(f, n + 16) == data
        for cap in (0, cap_b - 1, cap_b, 3 * cap_b):
            for c in range(len(f) + 1):
                r = FR.Reader(65536, dec, ref.xxh32)
                got, calls = feed(r, f, [c], cap)
                if cap < cap_b and n > 0:
                    assert got == b"" and r.end() == FR.CORRUPT
                    continue
                assert got == data, (n, cap, c)
                assert calls[-1][2] == 1 and r.end() == 0


@pytest.mark.parametrize("fl", [0, 7])
def test_random_cuts_of_big_frames(eng, fl):
    up, ref, _, dec = eng
    rng = np.random.default_rng(fl)
    data = content(1 << 20, 11 + fl)
    f = frame(eng, data, fl)
    cap_b = 65536 + (8 if fl & 1 else 0)
    for w in (1, 3, 4, 5, 19, 4095, 65535, 65536, 65537):
        cuts, at = [], 0
        while at < len(f):
            at += int(rng.integers(1, 2 * w + 1)) if w > 1 else 1
            cuts.append(at)
        got, calls = feed(FR.Reader(65536, dec, ref.xxh32), f, cuts, 16 * cap_b)
        assert got == data, w
        assert all(c[1] <= len(f) for c in calls)


def test_concatenated_frames_and_frame_ends(eng):
    """srcUsed never passes a frame end: each frame ends one read, the next read starts the next frame."""
    up, ref, _, dec = eng
    parts = [content(n, n) for n in (0, 1000, 200000, 17)]
    frames = [frame(eng, d, fl) for d, fl in zip(parts, (0, 7, 1, 4))]
    frames.append(up.frame_linked(parts[2], 5, True, True))
    frames.append(ref.frame_compress(parts[1], True, False))
    parts.append(parts[2])
    parts.append(parts[1])
    blob = b"".join(frames)
    r = FR.Reader(1 << 18, dec, ref.xxh32)
    at, k = 0, 0
    while at < len(blob):
        res, used, ended, got = r.read(blob[at:], 1 << 22)
        assert res == len(parts[k]) and got == parts[k] and ended == 1 and used == len(frames[k])
        at += used
        k += 1
    assert k == len(frames) and r.end() == 0


def test_end_at_every_phase(eng):
    up, ref, _, dec = eng
    f = frame(eng, content(70000, 3), 6)
    for c in range(len(f) + 1):
        r = FR.Reader(65536, dec, ref.xxh32)
        r.read(f[:c], 1 << 20)
        assert r.end() == (0 if c in (0, len(f)) else FR.CORRUPT), c
        res, used, ended, got = r.read(f, 1 << 20)          # new again
        assert ended == 1 and used == len(f)


def test_room_rule(eng):
    """dstCap < blockCap consumes a header and a complete end mark, but no block byte."""
    up, ref, _, dec = eng
    f = frame(eng, content(1000, 4), 4)
    r = FR.Reader(65536, dec, ref.xxh32)
    assert r.read(f, 65535)[:3] == (0, 7, 0)
    e = frame(eng, b"", 4)
    r = FR.Reader(65536, dec, ref.xxh32)
    assert r.read(e, 0)[:3] == (0, len(e), 1)


def corruptions(eng):
    """(name, frame) pairs: one of every verdict class."""
    up, ref, _, _ = eng
    data = content(300000, 9)
    good = frame(eng, data, 6)
    ind = frame(eng, data, 7)
    out = []
    b = bytearray(good); b[0] ^= 1; out.append(("magic", bytes(b)))
    out.append(("skippable", struct.pack("<II", 0x184D2A50, 4) + b"abcd"))
    out.append(("legacy", struct.pack("<I", 0x184C2102) + good[4:]))
    b = bytearray(good); b[4] ^= 0x80; out.append(("version", bytes(b)))
    b = bytearray(good); b[6] ^= 1; out.append(("hc", bytes(b)))
    b = bytearray(good); b[4] |= 1; out.append(("dict", bytes(b)))
    b = bytearray(good); b[200] ^= 0x10; out.append(("block sum", bytes(b)))
    b = bytearray(good); b[-1] ^= 1; out.append(("content sum", bytes(b)))
    b = bytearray(good[:7] + struct.pack("<I", 0x80000000 | 65537) + bytes(65541) + good[7:]); out.append(("raw", bytes(b)))
    # a rejected block: an offset before the start of an independent frame's first block (checksums recomputed)
    blk = bytes([0x0F, 0x40, 0x00])
    h = FW.header(65536, False, False, False)
    out.append(("rejected", h + struct.pack("<I", len(blk)) + blk + b"\0\0\0\0"))
    out.append(("big bd", frame(eng, data[:1000], 0, bs=4 << 20)))
    out.append(("truncated", good[:-9]))
    # compressed length codes too long for any block the decoder accepts: complete (the decoder's -1), with a bad
    # block checksum, cut off, and a flipped bit in a real frame's first length code (cut off: R_CORRUPT)
    zeros = bytes(70000)
    for bc in (True, False):
        h = FW.header(65536, False, bc, False) + struct.pack("<I", len(zeros)) + zeros
        s = struct.pack("<I", ref.xxh32(zeros)) if bc else b""
        out.append((f"long block {bc}", h + s + bytes(4)))
        out.append((f"long block cut {bc}", h[:40000]))
    out.append(("long block sum", FW.header(65536, False, True, False) + struct.pack("<I", len(zeros)) + zeros +
                struct.pack("<I", ref.xxh32(zeros) ^ 1) + bytes(4)))
    for name, f in (("length flip", ind), ("length flip linked", good)):
        code = struct.unpack_from("<I", f, 7)[0]
        out.append((name, f[:7] + struct.pack("<I", (code & 0x7FFFFFFF) | 0x00100000) + f[11:]))
    return out


def test_verdicts_equal_whole_frame(eng):
    up, ref, _, dec = eng
    want = {"magic": FR.CORRUPT, "skippable": FR.CORRUPT, "legacy": FR.CORRUPT, "version": FR.CORRUPT,
            "hc": FR.CORRUPT, "dict": FR.DELEGATE, "block sum": FR.CORRUPT, "content sum": FR.CORRUPT,
            "raw": FR.CORRUPT, "rejected": -1, "truncated": FR.CORRUPT, "long block True": -1,
            "long block False": -1, "long block cut True": FR.CORRUPT, "long block cut False": FR.CORRUPT,
            "long block sum": FR.CORRUPT, "length flip": FR.CORRUPT, "length flip linked": FR.CORRUPT}
    for name, f in corruptions(eng):
        if name == "big bd":
            r = FR.Reader(65536, dec, ref.xxh32)
            assert r.read(f, 1 << 20)[0] == FR.DELEGATE
            assert FR.whole_frame_verdict(f, dec, ref.xxh32) == 1000
            continue
        v = FR.whole_frame_verdict(f, dec, ref.xxh32)
        assert v == want[name], name
        for w in (7, 1000, 65536):
            r = FR.Reader(65536, dec, ref.xxh32)
            res, at = 0, 0
            while at < len(f):
                res, used, ended, _ = r.read(f[at:at + w], 1 << 20)
                if res < 0 or (used == 0 and not ended):
                    break
                at += used
            if res >= 0:                                         # truncated: end() tells
                assert r.end() == v, (name, w)
                continue
            assert res == v, (name, w)
            assert r.read(f, 1 << 20)[0] == v                   # failed: sticky
            assert r.end() == v and r.read(b"", 0)[0] == 0      # ended: new
