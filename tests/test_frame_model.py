"""CPU restatements behind the frame calls: k4lz4_frame_bound's arithmetic, the token-chain size walk of
block_size_walk_kernel (csrc/frame.cuh) against the oracle decoder, and _Frame's parse -- the device parse's
order of checks -- with the error class each corruption maps to."""
import struct

import numpy as np
import pytest

from tests import inputs
from tests import lz4_blocks as LB


def walk(s: bytes) -> int:
    """frame_walk: literal runs plus matchlen + 4, offsets unread; -1 where the chain runs past the end."""
    p, out, n = 0, 0, len(s)
    while p < n:
        tok = s[p]; p += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                if p >= n:
                    return -1
                x = s[p]; p += 1; lit += x
                if x != 255:
                    break
        out += lit; p += lit
        if p == n:
            return out
        if p + 2 > n:
            return -1
        p += 2
        ml = tok & 15
        if ml == 15:
            while True:
                if p >= n:
                    return -1
                x = s[p]; p += 1; ml += x
                if x != 255:
                    break
        out += ml + 4
    return -1


def lower_bound(n: int) -> int:
    return (n - 2) * 255 // 256 if n > 2 else 0


@pytest.mark.parametrize("flags", range(8))
def test_frame_bound(native, flags):
    for bs_in, bs in ((1, 1024), (1000, 1024), (65536, 65536), (65537, 66560), (4 << 20, 4 << 20)):
        for n in (0, 1, bs - 1, bs, bs + 1, 7 * bs + 3):
            nb = -(-n // bs)
            want = 7 + nb * (4 + (4 if flags & 2 else 0)) + n + 4 + (4 if flags & 4 else 0)
            assert native.k4lz4_frame_bound(n, bs_in, flags) == want
    E_ARG = -102
    assert native.k4lz4_frame_bound(10, 0, flags) == E_ARG
    assert native.k4lz4_frame_bound(10, (4 << 20) + 1, flags) == E_ARG
    assert native.k4lz4_frame_bound(-1, 65536, flags) == E_ARG
    assert native.k4lz4_frame_bound(10, 65536, flags | 8) == E_ARG


def test_size_walk_equals_decoder(port):
    rng = np.random.default_rng(1)
    streams = []
    for _, data in inputs.corpus(sizes=[1, 13, 100, 5000, 65536]):
        r, enc = port.encode(data)
        if r > 0:
            streams.append(enc)
            streams += [inputs.mutate(enc, rng) for _ in range(6)]
    for _ in range(200):
        n = int(rng.integers(0, 6))
        seqs = [(bytes(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)), 1,
                 int(rng.integers(4, 600))) for _ in range(n)]
        s, _ = LB.build_block(seqs, bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8)))
        streams.append(s)
    streams += [b"\x00", b"\x10a", b"\xf0" + b"\xff" * 3, bytes([0x10, 0x61, 0x64, 0x00, 0x50]) + b"bcdef"]
    accepted = 0
    for s in streams:
        r, _ = port.decode(s, 1 << 20)
        if r >= 0 and s:
            accepted += 1
            assert walk(s) == r, s[:32]
            assert r >= lower_bound(len(s))
    assert accepted > 150


def _hdr(port, flg: int, bd: int = 0x40, extra: bytes = b"") -> bytes:
    h = struct.pack("<IBB", 0x184D2204, flg, bd) + extra
    return h + bytes([(port.xxh32(np.frombuffer(h[4:], dtype=np.uint8)) >> 8) & 0xFF])


def test_frame_parse_error_classes(port):
    """_Frame's verdicts, in the device parse's order: magic, version (the reference's 0x11 mask), dictionary flag
    (K4LZ4_R_DELEGATE: NotImplementedError), header checksum, then the blocks (K4LZ4_R_CORRUPT: InvalidData)."""
    from k4os.compression.lz4_b200 import frame as F
    blk = port.encode(b"abcd" * 300)[1]
    body = struct.pack("<I", len(blk)) + blk + struct.pack("<I", 0x80000003) + b"xyz"
    good = _hdr(port, 0x40 | 0x04) + body + struct.pack("<I", 0) + struct.pack("<I", port.xxh32(np.frombuffer(b"abcd" * 300 + b"xyz", dtype=np.uint8)))
    fr = F._Frame(good)
    assert fr.chaining and fr.lens == [len(blk), 3] and fr.raws == [False, True] and fr.max_block == 65536
    sized = _hdr(port, 0x40 | 0x08, 0x70, struct.pack("<Q", 1203)) + body + struct.pack("<I", 0)
    assert F._Frame(sized).max_block == 4 << 20
    cases = [
        (good[:6], F.InvalidDataException),                              # magic (short)
        (b"\x05" + good[1:], F.InvalidDataException),                    # magic
        (good[:4] + bytes([good[4] ^ 0xC0]) + good[5:], F.InvalidDataException),   # version
        (good[:4] + bytes([good[4] | 1]) + good[5:], NotImplementedError),          # dictionary id
        (good[:6] + bytes([good[6] ^ 1]) + good[7:], F.InvalidDataException),      # header checksum
        (good[:9], F.InvalidDataException),                              # length code cut off
        (good[:20], F.InvalidDataException),                             # body cut off
        (good[:-2], F.InvalidDataException),                             # content checksum cut off
    ]
    for f, exc in cases:
        with pytest.raises(exc):
            F._Frame(f)
    # a version byte with bit 7 set but 6 set passes the reference's mask (0x11 keeps only bit 6 of FLG >> 6)
    assert F._Frame(good[:4] + bytes([good[4] | 0x80]) + good[5:6] + _hdr(port, good[4] | 0x80)[6:7] + good[7:])
