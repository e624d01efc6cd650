"""LZ4FrameWriter restated incrementally (Streams/Frames/LZ4FrameWriter.cs, LZ4FrameWriter.blocking.cs,
LZ4EncoderExtensions.cs:190-210): what each write and the close of one LZ4EncoderStream emit, at L00_FAST.

* The first write of a frame, even of 0 bytes, emits the 7-byte header.
* A block is emitted by the write that fills it; a write may fill any number of blocks.  Each block is encoded with
  capacity MaximumOutputSize(B) and stored raw when the result does not shrink it.
* Close emits the partial block, the end mark and the XXH32 of all the content (content checksum); a writer that
  was never written emits nothing.  After a close the writer starts a new frame.

The block engine is pluggable: ``Writer(..., engine)`` with ``engine(ctx, history, block, cap) -> (result,
bytes)``, ctx being what ``engine.start()`` returned for the frame and history the last min(content so far,
64 KiB) bytes of the frame for linked frames and b"" for independent ones.  ``UpstreamEngine`` gives upstream's LZ4_compress_fast_continue on a carried LZ4_stream_t
(chain_enc_ref.EncUpstream.step) or LZ4_compress_fast (oracle.Ref.encode).  ``XXH32Stream`` restates xxhash.c's
streaming XXH32 (XXH32_update / XXH32_digest).
"""
from __future__ import annotations

import struct

K64 = 65536
P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
M32 = 0xFFFFFFFF


def rounded_block(block_size: int) -> int:
    """LZ4EncoderBase.cs:29: max(1024, blockSize rounded up to 1 KiB)."""
    return max(1024, (block_size + 1023) // 1024 * 1024)


def bd_code(block_size: int) -> int:
    """LZ4FrameWriter.cs:183-188: the BD code of the caller's block size."""
    return 4 if block_size <= 1 << 16 else 5 if block_size <= 1 << 18 else 6 if block_size <= 1 << 20 else 7


def write_bound(length: int, block_size: int, bc: bool) -> int:
    B = rounded_block(block_size)
    return 7 + (B - 1 + length) // B * (4 + B + 4 * bc)


def close_bound(block_size: int, bc: bool, cc: bool) -> int:
    return 4 + rounded_block(block_size) + 4 * bc + 4 + 4 * cc


def _rotl(x: int, r: int) -> int:
    return ((x << r) | (x >> (32 - r))) & M32


def _round(v: int, w: int) -> int:
    return (_rotl((v + w * P2) & M32, 13) * P1) & M32


class XXH32Stream:
    """xxhash.c's XXH32_state_t with seed 0: four accumulators, a 16-byte carry, the total length and large_len."""

    def __init__(self):
        self.v = [(P1 + P2) & M32, P2, 0, (-P1) & M32]
        self.mem = b""
        self.total = 0

    def update(self, data: bytes) -> None:
        self.total += len(data)
        buf = self.mem + bytes(data)
        n = len(buf) // 16 * 16
        for o in range(0, n, 16):
            w = struct.unpack_from("<4I", buf, o)
            self.v = [_round(self.v[g], w[g]) for g in range(4)]
        self.mem = buf[n:]

    def digest(self) -> int:
        if self.total >= 16:                                  # large_len
            h = (_rotl(self.v[0], 1) + _rotl(self.v[1], 7) + _rotl(self.v[2], 12) + _rotl(self.v[3], 18)) & M32
        else:
            h = (self.v[2] + P5) & M32
        h = (h + self.total) & M32
        t, i = self.mem, 0
        while i + 4 <= len(t):
            h = (_rotl((h + struct.unpack_from("<I", t, i)[0] * P3) & M32, 17) * P4) & M32
            i += 4
        while i < len(t):
            h = (_rotl((h + t[i] * P5) & M32, 11) * P1) & M32
            i += 1
        h ^= h >> 15
        h = (h * P2) & M32
        h ^= h >> 13
        h = (h * P3) & M32
        h ^= h >> 16
        return h


def header(block_size: int, chaining: bool, bc: bool, cc: bool) -> bytes:
    flg = (1 << 6) | ((not chaining) << 5) | (bc << 4) | (cc << 2)
    h = struct.pack("<IBB", 0x184D2204, flg, bd_code(block_size) << 4)
    s = XXH32Stream()
    s.update(h[4:6])
    return h + bytes([(s.digest() >> 8) & 0xFF])


def xxh32(data: bytes) -> int:
    s = XXH32Stream()
    s.update(data)
    return s.digest()


class Writer:
    """One LZ4EncoderStream over LZ4FrameWriter.  write() and close() return the bytes each emits."""

    def __init__(self, block_size: int, chaining: bool, bc: bool, cc: bool, engine, hash32=None):
        self.block_size, self.B = block_size, rounded_block(block_size)
        self.chaining, self.bc, self.cc = chaining, bc, cc
        self.engine = engine
        self.hash32 = hash32                                # a faster whole-buffer XXH32, else XXH32Stream
        self.open = False

    def _start(self):
        self.open = True
        self.pending = b""
        self.history = b""                                  # the last <= 64 KiB of content already encoded
        self.sum = XXH32Stream()
        self.content = []
        self.ctx = self.engine.start() if hasattr(self.engine, "start") else None

    def _block(self, blk: bytes) -> bytes:
        cap = self.B + self.B // 255 + 16
        r, enc = self.engine(self.ctx, self.history if self.chaining else b"", blk, cap)
        assert r > 0
        raw = r >= len(blk)
        body = blk if raw else enc
        out = struct.pack("<I", len(body) | (0x80000000 if raw else 0)) + body
        if self.bc:
            out += struct.pack("<I", (self.hash32 or xxh32)(body))
        if self.chaining:
            self.history = (self.history + blk)[-K64:]
        return out

    def write(self, data: bytes) -> bytes:
        out = []
        if not self.open:
            self._start()
            out.append(header(self.block_size, self.chaining, self.bc, self.cc))
        if self.hash32:
            self.content.append(bytes(data))
        else:
            self.sum.update(data)
        buf = self.pending + bytes(data)
        o = 0
        while len(buf) - o >= self.B:
            out.append(self._block(buf[o:o + self.B]))
            o += self.B
        self.pending = buf[o:]
        return b"".join(out)

    def close(self) -> bytes:
        if not self.open:
            return b""
        out = [self._block(self.pending)] if self.pending else []
        out.append(struct.pack("<I", 0))
        if self.cc:
            out.append(struct.pack("<I", self.hash32(b"".join(self.content)) if self.hash32 else self.sum.digest()))
        self.open = False
        return b"".join(out)


class UpstreamEngine:
    """Upstream's blocks: LZ4_compress_fast_continue on a carried state (linked; chain_enc_ref.EncUpstream.step with
    the history in front of the block) or LZ4_compress_fast (independent)."""

    def __init__(self, up, ref, chaining: bool):
        self.up, self.ref, self.chaining = up, ref, chaining

    def start(self):
        from tests import chain_enc_ref as ER
        return [ER.make_state()]

    def __call__(self, ctx, history: bytes, blk: bytes, cap: int):
        if not self.chaining:
            return self.ref.encode(blk, cap)
        r, out, after = self.up.step(ctx[0], history, blk, cap)
        ctx[0] = after
        return r, out


def emit(writer: Writer, chunks) -> list:
    """The bytes each write emits, then the close's."""
    return [writer.write(c) for c in chunks] + [writer.close()]
