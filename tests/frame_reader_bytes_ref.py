"""Byte-granular reads of a frame reader group (k4lz4_frame_reader_group_read_bytes), restated twice:

* ``Pull``: the reference's ReadManyBytes / ReadBlock / Drain (Streams/Frames/LZ4FrameReader.blocking.cs,
  LZ4FrameReader.cs) line by line over an in-memory source, with exceptions turned into the library's codes.
* ``BytesReader``: the push contract of k4lz4.h.  A read first drains min(cap, undrained) bytes of the stream's
  current decoded block, then, while room is left, decodes the next complete block (of the chunk, or the stashed
  one) and appends as much of it as fits; the rest stays undrained.  It stops when the destination is full, when
  the chunk holds no further complete block, at the frame's end, or after a block that decodes to 0 bytes;
  interactively, after the first drain that appended anything.  A length code, end mark or cut block is touched
  only when the loop reaches it.  Headers, cut content checksums and skipped blocks go on as in frame_reader_ref.

Block engines are frame_reader_ref's: ``decode(src, cap, history) -> (r, bytes)``.
"""
from __future__ import annotations

import struct

from tests import frame_reader_ref as FR

CORRUPT, DELEGATE, ARG, K64 = FR.CORRUPT, FR.DELEGATE, FR.ARG, FR.K64


class BytesReader(FR.Reader):
    """One stream of a frame reader group read with read_bytes (and, for mixing, read)."""

    def _new(self):
        super()._new()
        self.pending = b""

    def read(self, chunk: bytes, cap: int):
        if self.pending and not self.err:
            return ARG, 0, 0, b""
        return super().read(chunk, cap)

    def read_bytes(self, chunk: bytes, cap: int, interactive: bool = False):
        """-> (result, bytes consumed (0 on a verdict), frame ended, content)."""
        if self.err:
            return self.err, 0, 0, b""
        chunk = bytes(chunk)
        n = len(chunk)
        q, out = 0, bytearray()
        count = max(cap, 0)

        def fail(code):
            self.err = code
            self.pending = b""
            return code, 0, 0, b""

        def done(ended):
            return len(out), q, ended, bytes(out)

        take = min(count, len(self.pending))           # Drain: the rest of the current block first
        out += self.pending[:take]
        self.pending = self.pending[take:]
        count -= take
        go = count > 0 and not (interactive and take > 0)
        while True:
            if self.phase == "idle":
                if q >= n:
                    break
                self.phase, self.item = "header", bytearray()
            if self.phase == "header":                  # EnsureHeader: whatever the room
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
                        if struct.unpack_from("<I", h)[0] != FR.MAGIC:
                            return fail(CORRUPT)
                        continue
                    st, flg, bd, hl = FR.header_check(bytes(h))
                    if st == CORRUPT and hl > len(h):
                        continue
                    if not st and FR.max_block((bd >> 4) & 7) > self.G:
                        st = DELEGATE
                    if st:
                        return fail(st)
                    self.linked, self.bc, self.cc = not flg & 0x20, bool(flg & 0x10), bool(flg & 4)
                    self.mb = FR.max_block((bd >> 4) & 7)
                    opened = True
                    break
                if not opened:
                    break
                self.phase, self.item, self.history, self.content = "block", bytearray(), b"", []
            if self.phase == "block":
                if not go:                               # the loop does not reach this length code
                    break
                cap_b = self.mb if self.linked else self.mb + 8
                it = self.item
                if len(it) + (n - q) < 4:
                    it += chunk[q:]
                    q = n
                    break
                code = struct.unpack_from("<I", bytes(it[:4]) + chunk[q:q + max(4 - len(it), 0)])[0]
                if code == 0:
                    q += 4 - len(it)
                    self.item = bytearray()
                    if not self.cc:
                        self.phase = "idle"
                        return done(1)
                    self.phase = "tail"
                else:
                    blen, raw = code & 0x7FFFFFFF, code >> 31
                    if raw and blen > cap_b:
                        return fail(CORRUPT)
                    if not raw and blen > FR.stash_body(self.G):
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
                    body = blk[4:4 + blen]
                    if self.bc and self._hash([body]) != struct.unpack_from("<I", blk, 4 + blen)[0]:
                        return fail(CORRUPT)
                    if raw:
                        data = body
                    else:
                        r, data = self.decode(body, cap_b, self.history if self.linked else b"")
                        if r < 0:
                            return fail(-1)
                    if self.cc:
                        self.content.append(data)
                    if self.linked:
                        self.history = (self.history + data)[-K64:]
                    take = min(count, len(data))
                    out += data[:take]
                    self.pending = data[take:]
                    count -= take
                    go = count > 0 and not interactive and len(data) > 0
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


class _Fail(Exception):
    def __init__(self, code):
        super().__init__(code)
        self.code = code


class Pull:
    """LZ4FrameReader over a whole in-memory source, restated from the reference: read(count, interactive) is
    ReadManyBytes; the source is pulled as it goes.  -> (result, frame ended) per call; a failure is sticky."""

    def __init__(self, source: bytes, max_block_size: int, decode, hash32=None):
        self.src, self.p, self.G, self.decode = bytes(source), 0, max_block_size, decode
        self.hash = hash32 or FR._xxh32
        self.desc, self.decoded, self.block, self.err = None, 0, b"", 0
        self.history = b""

    def _peek(self, k):
        if self.p + k > len(self.src):
            raise _Fail(CORRUPT)                           # EndOfStreamException inside a frame
        b = self.src[self.p:self.p + k]
        self.p += k
        return b

    def _ensure_header(self):                              # EnsureHeader
        if self.desc is not None:
            return True
        if self.p >= len(self.src):
            return False
        if struct.unpack_from("<I", self._peek(4))[0] != FR.MAGIC:
            raise _Fail(CORRUPT)
        h = FR.MAGIC.to_bytes(4, "little") + self._peek(2)
        if h[4] & 8:
            h += self._peek(8)
        h += self._peek(1)
        st, flg, bd, hl = FR.header_check(h)
        if not st and FR.max_block((bd >> 4) & 7) > self.G:
            st = DELEGATE
        if st:
            raise _Fail(st)
        self.desc = (not flg & 0x20, bool(flg & 0x10), bool(flg & 4), FR.max_block((bd >> 4) & 7))
        self.history, self.content = b"", []
        return True

    def _read_block(self):                                 # ReadBlock
        linked, bc, cc, mb = self.desc
        length = struct.unpack("<I", self._peek(4))[0]
        if length == 0:
            if cc and struct.unpack("<I", self._peek(4))[0] != self.hash(b"".join(self.content)):
                raise _Fail(CORRUPT)
            self.desc = None                               # CloseFrame
            self.ended = 1
            return 0
        raw, length = length >> 31, length & 0x7FFFFFFF
        cap = mb if linked else mb + 8
        if raw and length > cap:
            raise _Fail(CORRUPT)
        body = self._peek(length)
        if bc and struct.unpack("<I", self._peek(4))[0] != self.hash(body):
            raise _Fail(CORRUPT)
        if raw:
            data = body
        else:
            r, data = self.decode(body, cap, self.history if linked else b"")
            if r < 0:
                raise _Fail(-1)
        if linked:
            self.history = (self.history + data)[-K64:]
        if cc:
            self.content.append(data)
        self.block = data
        return len(data)

    def read(self, count: int, interactive: bool = False):
        if self.err:
            return self.err, 0
        self.ended = 0
        try:
            if not self._ensure_header():
                return 0, 0
            read, out = 0, []
            while count > 0:
                if self.decoded <= 0:
                    self.decoded = self._read_block()
                    if self.decoded == 0:
                        break
                k = min(count, self.decoded)                # Drain
                at = len(self.block) - self.decoded
                out.append(self.block[at:at + k])
                self.decoded -= k
                count -= k
                read += k
                if interactive:
                    break
            self.last = b"".join(out)
            return read, self.ended
        except _Fail as f:
            self.err = f.code
            return f.code, 0
