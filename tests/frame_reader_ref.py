"""LZ4FrameReader restated for a push contract (Streams/Frames/LZ4FrameReader.async.cs:46-172, LZ4FrameReader.cs,
Internal/ReaderExtensions.cs): what each read of one stream of a frame reader group consumes, decodes and returns.

* Bytes arrive in chunks cut anywhere.  A cut header, block ([length code | body | checksum]) or content checksum
  waits in a stash for the next chunk.
* A read consumes bytes of at most one frame: it stops after the end mark, or after the content checksum when the
  frame has one (the reference's Read returns at the end mark; its next Read opens the next frame).
* Room rule: at most floor(cap / blockCap) blocks per read (blockCap = BD maximum, + 8 for independent frames);
  once spent the read stops before the next length code, except that a complete end mark and the content checksum
  behind it are still consumed.  Header bytes need no room.
* Verdicts: the first problem in stream order, k4lz4_frame_decode_batch's codes (CORRUPT, -1 from the block
  decoder, DELEGATE for a dictionary id or a BD above the group's maximum).  A compressed block too long to decode
  within blockCap is skipped, not stashed: its checksum (CORRUPT) or its truncation (CORRUPT from end()) still come
  before the decoder's -1.  A failed stream returns its code and
  consumes nothing until ``end()``, which returns 0 between frames, CORRUPT inside one, or the failure, and makes
  the stream new.

Block engines are pluggable: ``decode(src, cap, history) -> (r, bytes)`` with r < 0 for a rejected block; linked
frames pass the last min(content, 64 KiB) bytes of the frame as history (chain_group_ref.GroupRing), independent
ones b"".  ``upstream_engine`` gives LZ4_decompress_safe / the prefix decode of chain_ref.Upstream.
"""
from __future__ import annotations

import struct

from tests.frame_writer_ref import XXH32Stream

MAGIC = 0x184D2204
CORRUPT, DELEGATE, ARG = -1000, -2, -102
K64 = 65536


def max_block(code: int) -> int:
    return {7: 1 << 22, 6: 1 << 20, 5: 1 << 18}.get(code, 1 << 16)


def stash_body(max_block_size: int) -> int:
    """The longest compressed block a reader stashes: any longer one decodes to more than maxBlockSize + 8 bytes."""
    m = max_block_size + 8
    return m + m // 255 + 4


def header_check(h: bytes):
    """frame.cuh's frame_header_check on the bytes of a header: -> (status, FLG, BD, header length)."""
    L = len(h)
    st = 0
    if L < 7 or struct.unpack_from("<I", h)[0] != MAGIC:
        st = CORRUPT
    flg, bd = (h[4], h[5]) if L >= 7 else (0, 0)
    if not st and ((flg >> 6) & 0x11) != 1:
        st = CORRUPT
    if not st and flg & 1:
        st = DELEGATE
    p = 6 + (8 if flg & 8 else 0)
    if not st:
        if L < p + 1:
            st = CORRUPT
        else:
            s = XXH32Stream()
            s.update(h[4:p])
            if (s.digest() >> 8) & 0xFF != h[p]:
                st = CORRUPT
    return st, flg, bd, p + 1


def _xxh32(data: bytes) -> int:
    s = XXH32Stream()
    s.update(data)
    return s.digest()


class Reader:
    """One stream.  hash32: a faster whole-buffer XXH32 (else XXH32Stream)."""

    def __init__(self, max_block_size: int, decode, hash32=None):
        self.G, self.decode, self.hash32 = max_block_size, decode, hash32
        self._new()

    def _new(self):
        self.phase, self.item, self.err = "idle", bytearray(), 0
        self.history = b""

    def _hash(self, parts) -> int:
        return self.hash32(b"".join(parts)) if self.hash32 else _xxh32(b"".join(parts))

    def end(self) -> int:
        r = self.err if self.err else (0 if self.phase == "idle" else CORRUPT)
        self._new()
        return r

    def read(self, chunk: bytes, cap: int):
        """-> (result, bytes consumed (0 on a verdict), frame ended, content)."""
        if self.err:
            return self.err, 0, 0, b""
        chunk = bytes(chunk)
        n = len(chunk)
        q, out, blocks = 0, [], 0
        budget = None

        def fail(code):
            self.err = code
            return code, 0, 0, b""

        def done(ended):
            data = b"".join(out)
            return len(data), q, ended, data

        while True:
            if self.phase == "idle":
                if q >= n:
                    break
                self.phase, self.item = "header", bytearray()
            if self.phase == "header":
                opened = False
                while True:
                    h = self.item
                    need = 4 if len(h) < 4 else 7 if len(h) < 7 else (15 if h[4] & 8 else 7)
                    k = max(min(need - len(h), n - q), 0)
                    h += chunk[q:q + k]
                    q += k
                    if len(h) < need:
                        break
                    if need == 4:
                        if struct.unpack_from("<I", h)[0] != MAGIC:
                            return fail(CORRUPT)
                        continue
                    st, flg, bd, hl = header_check(bytes(h))
                    if st == CORRUPT and hl > len(h):
                        continue
                    if not st and max_block((bd >> 4) & 7) > self.G:
                        st = DELEGATE
                    if st:
                        return fail(st)
                    self.linked, self.bc, self.cc = not flg & 0x20, bool(flg & 0x10), bool(flg & 4)
                    self.mb = max_block((bd >> 4) & 7)
                    opened = True
                    break
                if not opened:
                    break
                self.phase, self.item, self.history, self.content = "block", bytearray(), b"", []
            if self.phase == "block":
                cap_b = self.mb if self.linked else self.mb + 8
                if budget is None:
                    budget = max(cap, 0) // cap_b
                it = self.item
                if len(it) + (n - q) < 4:
                    if blocks >= budget:                # stops before the length code
                        break
                    it += chunk[q:]
                    q = n
                    break
                code = struct.unpack_from("<I", bytes(it[:4]) + chunk[q:q + max(4 - len(it), 0)])[0]
                if code == 0:                           # the end mark: consumed whatever the budget
                    q += 4 - len(it)
                    self.item = bytearray()
                    if not self.cc:
                        self.phase = "idle"
                        return done(1)
                    self.phase = "tail"
                else:
                    if blocks >= budget:
                        break
                    blen, raw = code & 0x7FFFFFFF, code >> 31
                    if raw and blen > cap_b:
                        return fail(CORRUPT)
                    if not raw and blen > stash_body(self.G):
                        q += 4 - len(it)
                        self.item, self.skip, self.skipped, self.phase = bytearray(), blen, [], "skip"
                        continue
                    total = 4 + blen + 4 * self.bc
                    if len(it) + (n - q) < total:
                        it += chunk[q:]
                        q = n
                        break
                    blk = bytes(it) + chunk[q:q + total - len(it)]
                    q += total - len(it)
                    self.item = bytearray()
                    blocks += 1
                    body = blk[4:4 + blen]
                    if self.bc and self._hash([body]) != struct.unpack_from("<I", blk, 4 + blen)[0]:
                        return fail(CORRUPT)
                    if raw:
                        data = body
                    else:
                        r, data = self.decode(body, cap_b, self.history if self.linked else b"")
                        if r < 0:
                            return fail(-1)
                    out.append(data)
                    if self.cc:
                        self.content.append(data)
                    if self.linked:
                        self.history = (self.history + data)[-K64:]
                    continue
            if self.phase == "skip":
                k = min(self.skip, n - q)
                if self.bc:
                    self.skipped.append(chunk[q:q + k])
                q += k
                self.skip -= k
                if self.skip:
                    break
                if not self.bc:
                    return fail(-1)
                k = min(4 - len(self.item), n - q)
                self.item += chunk[q:q + k]
                q += k
                if len(self.item) < 4:
                    break
                return fail(CORRUPT if self._hash(self.skipped) != struct.unpack_from("<I", self.item)[0] else -1)
            if self.phase == "tail":
                k = min(4 - len(self.item), n - q)
                self.item += chunk[q:q + k]
                q += k
                if len(self.item) < 4:
                    break
                if struct.unpack_from("<I", self.item)[0] != self._hash(self.content):
                    return fail(CORRUPT)
                self.phase, self.item = "idle", bytearray()
                return done(1)
        return done(0)


def upstream_engine(up, ref):
    """Upstream's engines: LZ4_decompress_safe (independent) and the prefix decode (linked)."""
    def decode(src, cap, history):
        if history:
            return up.decode_prefix(src, cap, history)
        return ref.decode(src, cap) if src else (-1, b"")
    return decode


def whole_frame_verdict(frame: bytes, decode, hash32=None) -> int:
    """k4lz4_frame_decode_batch's result on one whole frame with room for all of it, restated from frame.cuh
    independently of Reader: the header (frame_parse_kernel's order), then block by block in order -- cut off,
    checksum mismatch, a raw block above its limit, the decoder's rejection -- then the end mark and the content
    checksum.  The first problem in that order decides (the smallest error key).  -> the content length or the
    verdict."""
    h = hash32 or _xxh32
    L = len(frame)
    st, flg, bd, hl = header_check(frame[:15])
    if st:
        return st
    linked, bc, cc = not flg & 0x20, bool(flg & 0x10), bool(flg & 4)
    mb = max_block((bd >> 4) & 7)
    cap = mb if linked else mb + 8
    raw_limit = max(mb, K64) if linked else mb + 8
    p, out, hist = hl, [], b""
    while True:
        if p + 4 > L:
            return CORRUPT
        code = struct.unpack_from("<I", frame, p)[0]
        p += 4
        if code == 0:
            break
        blen, raw = code & 0x7FFFFFFF, code >> 31
        if p + blen + 4 * bc > L:
            return CORRUPT
        body = frame[p:p + blen]
        if bc and h(body) != struct.unpack_from("<I", frame, p + blen)[0]:
            return CORRUPT
        if raw:
            if blen > raw_limit:
                return CORRUPT
            data = body
        else:
            r, data = decode(body, cap, hist if linked else b"")
            if r < 0:
                return -1
        out.append(data)
        hist = (hist + data)[-K64:]
        p += blen + 4 * bc
    content = b"".join(out)
    if cc:
        if p + 4 > L or struct.unpack_from("<I", frame, p)[0] != h(content):
            return CORRUPT
    return len(content)
