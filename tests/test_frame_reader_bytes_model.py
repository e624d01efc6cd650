"""Byte reads of frame reader groups without a GPU: the push model (tests/frame_reader_bytes_ref.py) over
upstream's engines against upstream's whole-frame decoder on every cut of small frames, call by call against the
pull restatement of ReadManyBytes, on hand-built frames with empty blocks, on concatenated frames, and its
verdicts against the whole-frame verdict order.  Needs upstream's engine (oracle/_ref/)."""
import struct

import pytest

from tests import frame_reader_bytes_ref as RB
from tests import frame_reader_ref as FR
from tests import frame_writer_ref as FW
from tests.test_frame_reader_model import content, corruptions, eng, frame  # noqa: F401  (eng: a fixture)


def feed_bytes(reader, data, cuts, cap, interactive):
    """Feeds data cut at `cuts` with read_bytes, re-feeding unconsumed bytes, then drains -> content."""
    out, at = [], 0
    bounds = sorted(set(c for c in cuts if 0 < c < len(data))) + [len(data)]
    for b in bounds:
        while at < b or (b == len(data) and reader.pending):
            res, used, ended, got = reader.read_bytes(data[at:b], cap, interactive)
            assert res >= 0 and res <= max(cap, 0) and len(got) == res
            out.append(got)
            at += used
            if used == 0 and res == 0 and not ended:
                break
    return b"".join(out)


def caps_of(cap_b):
    return (0, 1, 7, cap_b - 1, cap_b, cap_b + 1, 3 * cap_b + 5)


@pytest.mark.parametrize("fl", range(8))
def test_every_cut_of_small_frames(eng, fl):
    """Every single cut, caps {0, 1, 7, blockCap - 1, blockCap, blockCap + 1, 3 blockCap + 5}, both modes: the
    content equals upstream's decoder and end() is 0 after the frame."""
    up, ref, _, dec = eng
    for n in (0, 5, 100, 70000):
        data = content(n, n + fl)
        f = frame(eng, data, fl)
        cap_b = 65536 + (8 if fl & 1 else 0)
        assert ref.frame_decompress(f, n + 16) == data
        step = 1 if n < 1000 else 4999
        for cap in caps_of(cap_b):
            for interactive in (False, True):
                for c in list(range(0, len(f) + 1, step)) + [len(f) - 1]:
                    r = RB.BytesReader(65536, dec, ref.xxh32)
                    if cap == 0:
                        assert r.read_bytes(f, 0, interactive)[:3] == (0, 7, 0)     # the header only
                        continue
                    got = feed_bytes(r, f, [c], cap, interactive)
                    assert got == data, (n, cap, c, interactive)
                    assert r.phase == "idle" and r.end() == 0


@pytest.mark.parametrize("fl", [0, 1, 6, 7])
@pytest.mark.parametrize("interactive", [False, True])
def test_calls_equal_pull_model(eng, fl, interactive):
    """Each chunk is the whole remaining input: every call's (result, frameEnded) equals ReadManyBytes'."""
    up, ref, _, dec = eng
    data = content(300000, 3 + fl)
    f = frame(eng, data, fl) + frame(eng, data[:1000], fl ^ 1)
    cap_b = 65536 + (8 if fl & 1 else 0)
    for cap in (1, 4096, cap_b - 1, cap_b, cap_b + 1, 200000):
        push, pull = RB.BytesReader(65536, dec, ref.xxh32), RB.Pull(f, 65536, dec, ref.xxh32)
        at, calls = 0, 0
        while at < len(f) or push.pending:
            res, used, ended, got = push.read_bytes(f[at:], cap, interactive)
            want = pull.read(cap, interactive)
            assert (res, ended) == want and got == pull.last, (cap, calls)
            at += used
            calls += 1
        assert pull.read(cap, interactive) == (0, 0) and push.end() == 0


def handmade(blocks, fl=0):
    """A frame of raw length codes and bodies (fl: FW flags bits: 1 independent, 2 block sum, 4 content sum)."""
    h = FW.header(65536, not fl & 1, bool(fl & 2), bool(fl & 4))
    out, content_ = [h], []
    for code, body, data in blocks:
        out.append(struct.pack("<I", code) + body + (struct.pack("<I", FW.xxh32(body)) if fl & 2 else b""))
        content_.append(data)
    c = b"".join(content_)
    out.append(b"\0\0\0\0" + (struct.pack("<I", FW.xxh32(c)) if fl & 4 else b""))
    return b"".join(out), c


def test_empty_blocks_stop_a_read(eng):
    """A compressed block that decodes to 0 bytes and a raw block 0x80000000 stop a read without closing the
    frame, as ReadBlock returning 0 breaks the reference's loop."""
    up, ref, _, dec = eng
    zero = bytes([0x00])                                  # one token, no literals: decodes to 0 bytes
    # (upstream's independent decoder rejects the 1-byte block, so independent frames take two raw empty blocks)
    for fl in (0, 1, 6, 7):
        empty = (len(zero), zero, b"") if not fl & 1 else (0x80000000, b"", b"")
        f, data = handmade([(0x80000003, b"abc", b"abc"), empty, (0x80000000, b"", b""),
                            (0x80000002, b"de", b"de")], fl)
        assert FR.whole_frame_verdict(f, dec, ref.xxh32) == 5
        for interactive in (False, True):
            push, pull = RB.BytesReader(65536, dec, ref.xxh32), RB.Pull(f, 65536, dec, ref.xxh32)
            at, seen = 0, []
            while True:
                res, used, ended, got = push.read_bytes(f[at:], 100, interactive)
                assert (res, ended) == pull.read(100, interactive) and got == pull.last
                seen.append((res, ended))
                at += used
                if ended:
                    break
            # non-interactive, the first read goes on past "abc" to the empty compressed block and stops there
            want = [(3, 0), (0, 0), (0, 0), (2, 0), (0, 1)] if interactive else [(3, 0), (0, 0), (2, 1)]
            assert seen == want, (fl, interactive, seen)
            assert push.end() == 0


def test_concatenated_frames(eng):
    up, ref, _, dec = eng
    parts = [content(n, n) for n in (0, 1000, 200000, 17)]
    frames = [frame(eng, d, fl) for d, fl in zip(parts, (0, 7, 1, 4))]
    blob = b"".join(frames)
    for cap in (3, 4096, 65536, 1 << 22):
        r = RB.BytesReader(1 << 18, dec, ref.xxh32)
        at, got, ends = 0, [], 0
        while at < len(blob) or r.pending:
            res, used, ended, d = r.read_bytes(blob[at:], cap)
            assert used <= len(blob) - at
            got.append(d)
            at += used
            ends += ended
        assert b"".join(got) == b"".join(parts) and ends == len(frames) and r.end() == 0


def test_mixing_and_end(eng):
    """read() on a stream holding undrained bytes: K4LZ4_E_ARG, nothing consumed, the stream not failed; end()
    inside a frame with undrained bytes: R_CORRUPT, and the stream is new."""
    up, ref, _, dec = eng
    data = content(100000, 8)
    f = frame(eng, data, 0)
    r = RB.BytesReader(65536, dec, ref.xxh32)
    res, used, ended, got = r.read_bytes(f, 4096)
    assert res == 4096 and r.pending
    assert r.read(f[used:], 1 << 20) == (FR.ARG, 0, 0, b"")
    rest = feed_bytes(r, f[used:], [], 1 << 20, False)
    assert got + rest == data and r.end() == 0
    r.read_bytes(f, 10)
    assert r.end() == FR.CORRUPT and r.read_bytes(f, 1 << 20)[2] == 1


def test_verdicts_equal_whole_frame(eng):
    up, ref, _, dec = eng
    for name, f in corruptions(eng):
        if name == "big bd":
            continue
        v = FR.whole_frame_verdict(f, dec, ref.xxh32)
        for w, cap in ((7, 1 << 20), (1000, 4096), (65536, 65535), (len(f), 50000)):
            r = RB.BytesReader(65536, dec, ref.xxh32)
            res, at = 0, 0
            while True:
                res, used, ended, _ = r.read_bytes(f[at:at + w], cap)
                if res < 0 or (used == 0 and res == 0 and not ended):
                    break
                at += used
            if res >= 0:
                assert r.end() == v, (name, w, cap)
                continue
            assert res == v, (name, w, cap)
            assert r.read_bytes(f, 1 << 20)[0] == v
