"""Chain groups (k4lz4_chain_group_*): the history rule restated in Python, and reference ring models to hold it
against.

* ``GroupRing`` is one stream of a group: a ring of 128 KiB + max(B, 64 KiB) bytes, the write position, the
  history (the last min(pos, 65 536) bytes) and the slide of the last 64 KiB to the front (chain_group.cuh).
* ``GroupEncoder`` drives a GroupRing and a state record through ``EncUpstream.step`` (upstream's
  LZ4_compress_fast_continue with the kernel's dictionary rule min(state.dictSize, prefixLen)).
* ``GroupDecoder`` drives a GroupRing through a prefix-mode decode function: upstream's, or the restatement
  ``chain_ref.decompress_prefix``.  A failed block leaves the stream as it was; Inject keeps the last 64 KiB.
* ``RefDecoder`` restates LZ4ChainDecoder.cs (the ring, CopyDict / ApplyDict, prefixSize) over the same decode
  function, for runs without upstream's LZ4_streamDecode_t.
"""
from __future__ import annotations

import numpy as np

from tests import chain_enc_ref as ER
from tests import chain_ref as CR

K64 = 65536


class GroupRing:
    def __init__(self, block_size: int):
        self.slot = max((block_size + 15) // 16 * 16, K64)
        self.size = 2 * K64 + self.slot
        self.buf = np.zeros(self.size, dtype=np.uint8)
        self.pos = 0
        self.slides = 0

    @property
    def prefix(self) -> int:
        return min(self.pos, K64)

    def history(self) -> bytes:
        return self.buf[self.pos - self.prefix:self.pos].tobytes()

    def append(self, data: bytes) -> None:
        """The commit: `data` was written at the write position; slide when the next block might not fit."""
        n = len(data)
        assert self.pos + n <= self.size
        self.buf[self.pos:self.pos + n] = np.frombuffer(data, dtype=np.uint8)
        self.pos += n
        if self.pos + self.slot > self.size:
            assert self.pos - K64 >= K64                    # the slide never overlaps its destination
            self.buf[:K64] = self.buf[self.pos - K64:self.pos].copy()
            self.pos = K64
            self.slides += 1


class GroupEncoder:
    """One encoder stream of a group: the kernel's rule over upstream, block by block."""

    def __init__(self, up: "ER.EncUpstream", block_size: int):
        self.up, self.B = up, block_size
        self.ring = GroupRing(block_size)
        self.state = ER.make_state()
        self.failed = False

    def encode(self, src: bytes, cap: int):
        """-> (result as the group returns it, bytes).  Empty: 0, stream untouched; too long or failed stream: -1."""
        if self.failed or len(src) > self.B:
            return -1, b""
        if not src:
            return 0, b""
        r, out, after = self.up.step(self.state, self.ring.history(), src, cap)
        self.state = after
        if r <= 0:
            self.failed = True
            return -1, b""
        self.ring.append(src)
        return r, out


class GroupDecoder:
    def __init__(self, block_size: int, decode):
        self.B, self.decode_fn = block_size, decode
        self.ring = GroupRing(block_size)

    def decode(self, src: bytes, cap: int):
        if cap > self.B:
            return -1, b""
        r, out = self.decode_fn(src, cap, self.ring.history())
        if r < 0:
            return -1, b""
        self.ring.append(out)
        return r, out

    def inject(self, data: bytes) -> None:
        if data:
            self.ring.append(data[-K64:])


class RefDecoder:
    """LZ4ChainDecoder.cs:26-143 restated: the ring, Prepare / CopyDict, Inject / ApplyDict and prefixSize, with
    blocks decoded by `decode(src, cap, history)` behind the prefixSize bytes in front of the write position."""

    def __init__(self, block_size: int, extra: int, decode):
        self.block = (max(block_size, 1024) + 1023) // 1024 * 1024
        self.out_len = K64 + (1 + max(extra, 0)) * self.block + 32
        self.buf = np.zeros(self.out_len + 8, dtype=np.uint8)
        self.index = self.prefix = 0
        self.decode_fn = decode

    def decode(self, src: bytes, bs: int = 0) -> int:
        bs = bs if bs > 0 else self.block
        if self.index + bs > self.out_len:
            start = max(self.index - K64, 0)
            size = self.index - start
            self.buf[:size] = self.buf[start:self.index].copy()
            self.index = self.prefix = size
        P = min(self.prefix, self.index)
        r, out = self.decode_fn(src, bs, self.buf[self.index - P:self.index].tobytes())
        if r < 0:
            raise RuntimeError("InvalidOperationException")
        self.buf[self.index:self.index + r] = np.frombuffer(out, dtype=np.uint8)
        self.index += r
        if r > 0:
            self.prefix = r if self.prefix == 0 else self.prefix + r
        return r

    def inject(self, src: bytes) -> int:
        n = len(src)
        if n <= 0:
            return 0
        a = np.frombuffer(src, dtype=np.uint8)
        if self.index + n < self.out_len:
            self.buf[self.index:self.index + n] = a
            self.index += n
        elif n >= K64:
            self.buf[:n] = a
            self.index = n
        else:
            tail = min(K64 - n, self.index)
            self.buf[:tail] = self.buf[self.index - tail:self.index].copy()
            self.buf[tail:tail + n] = a
            self.index = tail + n
        self.prefix = min(self.index, K64)
        return n

    def peek(self, offset: int) -> bytes:
        return self.buf[self.index + offset:self.index].tobytes()


def decode_script(seed: int, block: int, n_ops: int):
    """A random Decode / Inject sequence of one stream: ops ("dec", block, cap) or ("inj", raw).  Valid blocks are
    built against the stream's true history (chain_ref.build_prefix_block), with matches reaching up to 65 535
    bytes back; about one in six is first sent truncated or with one bit flipped.  Blocks of 1 byte up to `block` bytes."""
    rng = np.random.default_rng(seed)
    hist = b""                           # the stream so far, as a valid decoder sees it (mutations aside)
    ops = []
    for k in range(n_ops):
        size = int(rng.choice([1, 5, 13, 100, block, int(rng.integers(1, block + 1))]))
        if rng.random() < 0.25:
            size = int(rng.choice([size, size, K64 - 1, K64]))
            raw = rng.integers(0, 256, min(size, max(block, K64)), dtype=np.uint8).tobytes()
            ops.append(("inj", raw))
            hist = (hist + raw)[-K64:]
            continue
        seqs, out = [], 0
        lits = rng.integers(0, 4, 64, dtype=np.uint8).tobytes()
        while out + 40 < size - 12:
            L = int(rng.integers(0, 12))
            reach = len(hist) + out + L
            off = int(rng.integers(1, min(reach, 65535) + 1)) if reach else 0
            ml = int(rng.integers(4, 40))
            if off == 0 or out + L + ml > size - 12:
                break
            seqs.append((lits[:L], off, ml))
            out += L + ml
        last = rng.integers(0, 256, max(size - out, 0), dtype=np.uint8).tobytes()
        src, dec = CR.build_prefix_block(hist[-K64:], seqs, last)
        if rng.random() < 1 / 6 and len(src) > 2:
            m = bytearray(src[:-1]) if rng.random() < 0.5 else bytearray(src)     # truncated, or one bit flipped
            m[int(rng.integers(0, len(m)))] ^= 1 << int(rng.integers(0, 8))
            ops.append(("dec", bytes(m), size))      # the valid block follows: the stream must be able to go on
        ops.append(("dec", src, size))
        hist = (hist + dec)[-K64:]
    return ops
