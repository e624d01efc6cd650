"""Independent-block stream pair with a BATCHED top-up (SURVEY.md 8f row 1).

Mirrors of the reference's only in-product callers of the block codec,
    Encoders/LZ4EncoderBase.cs:27-97, Encoders/LZ4BlockEncoder.cs:7-23, Encoders/LZ4BlockDecoder.cs:11-102,
with the same member names and error behaviour, plus the one thing a GPU needs: instead of one
`LZ4Codec.Encode` per 64 KiB block (one PCIe round trip each) the encoder queues up to
`batch_blocks` full blocks and encodes them with ONE `k4lz4_encode_batch` call; the decoder takes a
list of compressed blocks and decodes them with ONE `k4lz4_decode_batch` call.  Every block's bytes
and return value equal what the reference's per-block call produces (independent blocks: no
dictionary, fresh table per block -- LZ4BlockEncoder.cs:18-23).

`LZ4FastChainEncoder` (Encoders/LZ4FastChainEncoder.cs) encodes dependent blocks at L00_FAST, and
`LZ4ChainDecoder` (Encoders/LZ4ChainDecoder.cs) decodes them.  One stream's blocks are serial, but the blocks
of MANY streams are not: `LZ4FastChainEncoder.EncodeMany` and `LZ4ChainDecoder.DecodeMany` advance many
encoders or decoders by one block each with ONE `k4lz4_encode_chain_batch` / `k4lz4_decode_chain_batch` call.
The chained HC encoder stays with the managed engine.

"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .batch import (decode_batch_flat_host, decode_chain_blocks_host, decode_chain_streams_host, encode_batch_flat_host,
                    encode_chain_batch_host)
from .codec import LZ4Codec, LZ4Level

K1 = 1024
K64 = 65536


def _round_up(v: int, step: int) -> int:      # Mem.RoundUp
    return (v + step - 1) // step * step


class LZ4BlockEncoder:
    """LZ4BlockEncoder(level, blockSize) -- LZ4BlockEncoder.cs:11-15; `batch_blocks` blocks are held
    back and encoded by one GPU call."""

    def __init__(self, level: LZ4Level = LZ4Level.L00_FAST, blockSize: int = 65536, batch_blocks: int = 256):
        self._level = LZ4Level(level)
        self._block = _round_up(max(int(blockSize), K1), K1)            # LZ4EncoderBase.cs:29
        self._depth = max(int(batch_blocks), 1)
        self._buf = np.zeros(self._depth * self._block, dtype=np.uint8)   # queue of block slots
        self._fill = np.zeros(self._depth, dtype=np.int32)               # bytes in each slot
        self._cur = 0                                                      # slot being topped up
        self._disposed = False

    # -- ILZ4Encoder ----------------------------------------------------------------------------
    @property
    def BlockSize(self) -> int:
        return self._block

    @property
    def BytesReady(self) -> int:
        """Bytes waiting in the block that is being filled (LZ4EncoderBase.cs:44)."""
        return int(self._fill[self._cur]) if self._cur < self._depth else 0

    @property
    def BlocksQueued(self) -> int:
        return int((self._fill > 0).sum())

    def Topup(self, source) -> int:
        """Adds bytes to the current block; returns how many were taken (0 when the block is full,
        LZ4EncoderBase.cs:47-62)."""
        self._check()
        src = np.frombuffer(source, dtype=np.uint8) if not isinstance(source, np.ndarray) else source
        if src.size == 0 or self._cur >= self._depth:
            return 0
        left = self._block - int(self._fill[self._cur])
        if left <= 0:
            return 0
        chunk = min(left, int(src.size))
        at = self._cur * self._block + int(self._fill[self._cur])
        self._buf[at:at + chunk] = src[:chunk]
        self._fill[self._cur] += chunk
        return chunk

    def TopupMany(self, source) -> int:
        """Batched top-up: fills block after block until the queue or the source is exhausted."""
        self._check()
        src = np.frombuffer(source, dtype=np.uint8) if not isinstance(source, np.ndarray) else source
        taken = 0
        while taken < src.size and self._cur < self._depth:
            got = self.Topup(src[taken:])
            taken += got
            if int(self._fill[self._cur]) == self._block:
                self._cur += 1
            elif got == 0:
                break
        return taken

    def Encode(self, target, allowCopy: bool = True) -> int:
        """Encodes the (single) pending block into `target` -- LZ4EncoderBase.cs:65-87: returns the
        encoded length, or -length when allowCopy stored the block raw; 0 when nothing is pending."""
        out = self.EncodeMany(allowCopy, _targets=[target])
        return out[0][0] if out else 0

    def EncodeMany(self, allowCopy: bool = True, _targets=None):
        """Encodes every queued block with one GPU call.  Returns [(encoded, bytes)] in block order
        with the reference's per-block convention (encoded < 0: stored raw, |encoded| bytes)."""
        self._check()
        nb = int((self._fill > 0).sum())
        if nb == 0:
            return []
        lens = self._fill[:nb].copy()
        if self._level >= LZ4Level.L03_HC:
            from .codec import DelegateToManagedEngine
            raise DelegateToManagedEngine("HC/OPT levels stay with the managed engine")
        bound = LZ4Codec.MaximumOutputSize(self._block)
        src_off = np.arange(nb, dtype=np.int64) * self._block
        if _targets is None:
            caps = np.full(nb, bound, dtype=np.int32)
        else:
            caps = np.array([len(t) for t in _targets], dtype=np.int32)
            assert len(_targets) == nb, "Encode() handles exactly one pending block"
        dst_off = np.zeros(nb, dtype=np.int64)
        dst_off[1:] = np.cumsum(caps[:-1].astype(np.int64))
        dst = np.zeros(int(caps.astype(np.int64).sum()) + 16, dtype=np.uint8)
        out_len = encode_batch_flat_host(self._buf, src_off, lens, dst, dst_off, caps, int(self._level),
                                         x32=LZ4Codec.Enforce32)
        res = []
        for i in range(nb):
            enc = int(out_len[i])
            if enc <= 0:                                                  # LZ4EncoderBase.cs:75-77
                raise RuntimeError("Failed to encode chunk. Target buffer too small.")   # InvalidOperationException
            n = int(lens[i])
            if allowCopy and enc >= n:                                    # :79-83
                data = self._buf[i * self._block:i * self._block + n].tobytes()
                enc = -n
            else:
                data = dst[dst_off[i]:dst_off[i] + enc].tobytes()
            if _targets is not None:
                t = np.frombuffer(_targets[i], dtype=np.uint8) if not isinstance(_targets[i], np.ndarray) else _targets[i]
                t[:len(data)] = np.frombuffer(data, dtype=np.uint8)
            res.append((enc, data))
        self._fill[:] = 0                                                 # Commit(), :89-96 (no dictionary)
        self._cur = 0
        return res

    def Dispose(self) -> None:
        self._disposed = True

    def _check(self) -> None:
        if self._disposed:
            raise RuntimeError("ObjectDisposedException")


class LZ4BlockDecoder:
    """LZ4BlockDecoder(blockSize) -- LZ4BlockDecoder.cs:22-30, with DecodeMany for whole batches."""

    def __init__(self, blockSize: int = 65536):
        self._block = _round_up(max(int(blockSize), K1), K1)
        self._out_len = self._block + 8                                   # LZ4BlockDecoder.cs:26
        self._out = np.zeros(self._out_len + 8, dtype=np.uint8)
        self._index = 0
        self._disposed = False

    @property
    def BlockSize(self) -> int:
        return self._block

    @property
    def BytesReady(self) -> int:
        return self._index

    def Decode(self, source, blockSize: int = 0) -> int:
        """LZ4BlockDecoder.cs:39-55."""
        self._check()
        if blockSize <= 0:
            blockSize = self._block
        if blockSize > self._block:
            raise RuntimeError("InvalidOperationException")
        decoded = LZ4Codec.Decode(bytes(source), self._out[:self._out_len])
        if decoded < 0:
            raise RuntimeError("InvalidOperationException")
        self._index = decoded
        return decoded

    def DecodeMany(self, blocks):
        """Decodes a list of blocks with one GPU call.  An item is compressed bytes, or a tuple
        (bytes, True) for a block that was stored raw (the encoder's negative length).  Returns the
        list of decoded blocks; raises like Decode() if any block is malformed or larger than the
        block size.  The last block stays available through Drain/Peek."""
        self._check()
        comp, raw_at = [], {}
        for i, b in enumerate(blocks):
            if isinstance(b, tuple) and b[1]:
                raw_at[i] = bytes(b[0])
                comp.append(b"")
            else:
                comp.append(bytes(b[0] if isinstance(b, tuple) else b))
        n = len(comp)
        if n == 0:
            return []
        src = np.frombuffer(b"".join(comp) or b"\x00", dtype=np.uint8)
        lens = np.array([len(c) for c in comp], dtype=np.int32)
        off = np.zeros(n, dtype=np.int64)
        off[1:] = np.cumsum(lens[:-1].astype(np.int64))
        caps = np.full(n, self._out_len, dtype=np.int32)
        doff = np.arange(n, dtype=np.int64) * self._out_len
        dst = np.zeros(n * self._out_len + 16, dtype=np.uint8)
        out_len = decode_batch_flat_host(src, off, lens, dst, doff, caps)
        res = []
        for i in range(n):
            if i in raw_at:
                if len(raw_at[i]) > self._out_len:
                    raise RuntimeError("InvalidOperationException")
                res.append(raw_at[i])
                continue
            r = int(out_len[i])
            if r < 0 or (r == 0 and lens[i] > 0):
                raise RuntimeError("InvalidOperationException")
            res.append(dst[doff[i]:doff[i] + r].tobytes())
        last = res[-1]
        self._out[:len(last)] = np.frombuffer(last, dtype=np.uint8)
        self._index = len(last)
        return res

    def Inject(self, source) -> int:
        """LZ4BlockDecoder.cs:58-71."""
        self._check()
        n = len(source)
        if n <= 0:
            self._index = 0
            return 0
        if n > self._out_len:
            raise RuntimeError("InvalidOperationException")
        self._out[:n] = np.frombuffer(bytes(source), dtype=np.uint8)
        self._index = n
        return n

    def Drain(self, target, offset: int, length: int) -> None:
        """LZ4BlockDecoder.cs:74-83 (offset is negative: counted from the end of the block)."""
        self._check()
        offset = self._index + offset
        if offset < 0 or length < 0 or offset + length > self._index:
            raise RuntimeError("InvalidOperationException")
        t = np.frombuffer(target, dtype=np.uint8) if not isinstance(target, np.ndarray) else target
        t[:length] = self._out[offset:offset + length]

    def Peek(self, offset: int) -> np.ndarray:
        self._check()
        offset = self._index + offset
        if offset < 0 or offset > self._index:
            raise RuntimeError("InvalidOperationException")
        return self._out[offset:self._index]

    def Dispose(self) -> None:
        self._disposed = True

    def _check(self) -> None:
        if self._disposed:
            raise RuntimeError("ObjectDisposedException")


class LZ4ChainDecoder:
    """LZ4ChainDecoder(blockSize, extraBlocks) -- LZ4ChainDecoder.cs:26-36: the same ring buffer of
    64 KiB + (1 + extraBlocks) * blockSize + 32 bytes, the same CopyDict / ApplyDict bookkeeping, and the
    prefix size LZ4_streamDecode_t would hold (LL64.dec.cs:558-592; the reference's decoder only ever takes
    the prefix branches of LZ4_decompress_safe_continue, so the end of the prefix is always the write
    position).  Decoding runs on the GPU; DecodeMany advances many decoders with one call."""

    def __init__(self, blockSize: int = 65536, extraBlocks: int = 0):
        self._block = _round_up(max(int(blockSize), K1), K1)
        extra = max(int(extraBlocks), 0)
        self._out_len = K64 + (1 + extra) * self._block + 32
        self._out = np.zeros(self._out_len + 8, dtype=np.uint8)
        self._index = 0
        self._prefix = 0                  # lz4sd->prefixSize
        self._disposed = False

    @property
    def BlockSize(self) -> int:
        return self._block

    @property
    def BytesReady(self) -> int:
        return self._index

    @property
    def PrefixSize(self) -> int:
        """The history length the next Decode passes to the GPU (LZ4_streamDecode_t.prefixSize)."""
        return self._prefix

    def Decode(self, source, blockSize: int = 0) -> int:
        """LZ4ChainDecoder.cs:45-61: decodes one block behind the previous output; returns its length."""
        return LZ4ChainDecoder.DecodeMany([self], [(source, blockSize)])[0]

    @staticmethod
    def DecodeMany(decoders, blocks, device: int = 0) -> list:
        """Decode() on every decoder at once: decoders[i] decodes blocks[i] (compressed bytes, or a tuple
        (bytes, blockSize)), all of them in ONE GPU call.  The decoders must be distinct.  Returns the decoded
        lengths.  If a block is malformed its decoder's write position does not move (Decode throws before
        `_outputIndex += decoded`) and InvalidOperationException is raised after every other decoder has been
        advanced."""
        decoders = list(decoders)
        if len(decoders) != len(blocks):
            raise ValueError("one block per decoder")
        if len({id(d) for d in decoders}) != len(decoders):
            raise ValueError("a decoder may take only one block per call")
        n = len(decoders)
        if n == 0:
            return []
        srcs, caps = [], []
        for d, b in zip(decoders, blocks):
            d._check()
            data, bs = (b if isinstance(b, tuple) else (b, 0))
            bs = int(bs) if int(bs) > 0 else d._block
            if K64 + bs > d._out_len:
                raise RuntimeError("InvalidOperationException")       # the block cannot fit behind the dictionary
            d._prepare(bs)
            srcs.append(bytes(data))
            caps.append(bs)
        hist = [d._out[d._index - min(d._prefix, d._index, 65535):d._index] for d in decoders]
        out, data = decode_chain_blocks_host(srcs, hist, caps, device)
        res, failed = [], False
        for i, d in enumerate(decoders):
            r = int(out[i])
            if r < 0:
                failed = True
                res.append(r)
                continue
            d._out[d._index:d._index + r] = np.frombuffer(data[i], dtype=np.uint8)
            d._index += r
            if r > 0:                                                  # LL64.dec.cs:566-590
                d._prefix = r if d._prefix == 0 else d._prefix + r
            res.append(r)
        if failed:
            raise RuntimeError("InvalidOperationException")
        return res

    def DecodeBlocks(self, blocks, raw=None, device: int = 0) -> bytes:
        """Decode() over many consecutive blocks of this decoder's stream in ONE GPU call
        (k4lz4_decode_chain_streams): every block is in flight at once.  An item is compressed bytes or a tuple
        (bytes, blockSize); where raw[i] is true the item is a block stored uncompressed and goes in by Inject().
        Returns the decoded bytes of all the blocks.  Leaves the decoder exactly as the same sequence of Decode /
        Inject calls would (write position, ring contents, PrefixSize); where one of them would throw, the blocks
        before it are applied and InvalidOperationException is raised.  Not a speed-up today: on an H100 one stream
        decodes about 4x slower this way than by a loop of Decode calls (DESIGN 4.11)."""
        self._check()
        items = []
        for i, b in enumerate(blocks):
            data, bs = (b if isinstance(b, tuple) else (b, 0))
            data = bytes(data)
            is_raw = bool(raw[i]) if raw is not None else False
            items.append((data, len(data) if is_raw else (int(bs) if int(bs) > 0 else self._block), is_raw))
        if not items:
            return b""
        hl = min(self._prefix, self._index, 65535)
        src = np.frombuffer(b"".join(d for d, _, _ in items) or b"\x00", dtype=np.uint8)
        lens = np.array([len(d) for d, _, _ in items], dtype=np.int32)
        offs = np.zeros(len(items), dtype=np.int64)
        offs[1:] = np.cumsum(lens[:-1], dtype=np.int64)
        caps = np.array([bs for _, bs, _ in items], dtype=np.int32)
        dst = np.zeros(hl + int(caps.astype(np.int64).sum()) + 16, dtype=np.uint8)
        dst[:hl] = self._out[self._index - hl:self._index]
        out = decode_chain_streams_host(src, offs, lens, caps, [0, len(items)], dst, [hl], [hl],
                                        raw=[r for _, _, r in items], device=device)
        at = hl
        for i, (data, bs, is_raw) in enumerate(items):
            r = int(out[i])
            if is_raw:
                self.Inject(data)                                      # raises where Inject would
            elif r < 0 or K64 + bs > self._out_len:
                raise RuntimeError("InvalidOperationException")
            else:
                self._prepare(bs)
                self._out[self._index:self._index + r] = dst[at:at + r]
                self._index += r
                if r > 0:                                              # LL64.dec.cs:566-590
                    self._prefix = r if self._prefix == 0 else self._prefix + r
            at += max(r, 0)
        return dst[hl:at].tobytes()

    def Inject(self, source) -> int:
        """LZ4ChainDecoder.cs:64-93."""
        self._check()
        src = np.frombuffer(bytes(source), dtype=np.uint8)
        length = int(src.size)
        if length <= 0:
            return 0
        if length > max(self._block, K64):
            raise RuntimeError("InvalidOperationException")
        if self._index + length < self._out_len:
            self._out[self._index:self._index + length] = src
            self._index = self._apply_dict(self._index + length)
        elif length >= K64:
            self._out[:length] = src
            self._index = self._apply_dict(length)
        else:
            tail = min(K64 - length, self._index)
            self._out[:tail] = self._out[self._index - tail:self._index].copy()
            self._out[tail:tail + length] = src
            self._index = self._apply_dict(tail + length)
        return length

    def Drain(self, target, offset: int, length: int) -> None:
        """LZ4ChainDecoder.cs:96-103 (offset is negative: counted from the write position)."""
        self._check()
        offset = self._index + offset
        if offset < 0 or length < 0 or offset + length > self._index:
            raise RuntimeError("InvalidOperationException")
        t = np.frombuffer(target, dtype=np.uint8) if not isinstance(target, np.ndarray) else target
        t[:length] = self._out[offset:offset + length]

    def Peek(self, offset: int) -> np.ndarray:
        """LZ4ChainDecoder.cs:106-115: the bytes from `offset` (negative) to the write position."""
        self._check()
        offset = self._index + offset
        if offset < 0 or offset > self._index:
            raise RuntimeError("InvalidOperationException")
        return self._out[offset:self._index]

    def Dispose(self) -> None:
        self._disposed = True

    # -- LZ4ChainDecoder.cs:117-140 --------------------------------------------------------------------------
    def _prepare(self, block_size: int) -> None:
        if self._index + block_size <= self._out_len:
            return
        self._index = self._copy_dict(self._index)

    def _copy_dict(self, index: int) -> int:
        start = max(index - K64, 0)
        size = index - start
        self._out[:size] = self._out[start:index].copy()
        self._prefix = size                                            # LZ4_setStreamDecode(ctx, buffer, size)
        return size

    def _apply_dict(self, index: int) -> int:
        self._prefix = index - max(index - K64, 0)                    # LZ4_setStreamDecode(ctx, buffer + start, size)
        return index

    def _check(self) -> None:
        if self._disposed:
            raise RuntimeError("ObjectDisposedException")


class LZ4FastChainEncoder:
    """LZ4FastChainEncoder(blockSize, extraBlocks) -- LZ4FastChainEncoder.cs:14-41 over LZ4EncoderBase.cs:27-97:
    the same input ring of 64 KiB + (1 + extraBlocks) * blockSize + 32 bytes, Topup / Encode / Commit, and
    CopyDict = LZ4_saveDict (the last <= 64 KiB move to the front of the ring).  The LZ4_stream_t lives in a
    16 400-byte state record (K4LZ4_CHAIN_STATE_BYTES, zero = LZ4_createStream); blocks are encoded on the GPU
    by LZ4_compress_fast_continue's rules with the bytes in front of the block in the ring as history, and
    EncodeMany advances many encoders with one call.  After a failed Encode (target too small) the state has
    advanced as the reference's has; encoding the same bytes again would take upstream's external-dictionary
    branch, which the GPU does not reproduce, so such an encoder should be discarded, as the exception suggests."""

    def __init__(self, blockSize: int = 65536, extraBlocks: int = 0):
        self._block = _round_up(max(int(blockSize), K1), K1)              # LZ4EncoderBase.cs:29-35
        extra = max(int(extraBlocks), 0)
        self._in_len = K64 + (1 + extra) * self._block + 32
        self._in = np.zeros(self._in_len + 8, dtype=np.uint8)
        self._index = 0                                                   # _inputIndex
        self._pointer = 0                                                 # _inputPointer
        self._state = np.zeros(N.CHAIN_STATE_BYTES, dtype=np.uint8)
        self._disposed = False

    @property
    def BlockSize(self) -> int:
        return self._block

    @property
    def BytesReady(self) -> int:
        return self._pointer - self._index

    @property
    def State(self) -> np.ndarray:
        """The stream state: uint32 hashTable[4096], currentOffset, dictSize, reserved[2] (a view)."""
        return self._state.view(np.uint32)

    def Topup(self, source) -> int:
        """LZ4EncoderBase.cs:46-62: adds up to the rest of the current block; returns the bytes taken."""
        self._check()
        src = np.frombuffer(bytes(source), dtype=np.uint8) if not isinstance(source, np.ndarray) else source
        if src.size == 0:
            return 0
        left = self._index + self._block - self._pointer
        if left <= 0:
            return 0
        chunk = min(left, int(src.size))
        self._in[self._pointer:self._pointer + chunk] = src[:chunk]
        self._pointer += chunk
        return chunk

    def Encode(self, target, allowCopy: bool = False) -> int:
        """LZ4EncoderBase.cs:65-88: encodes the pending bytes into `target` (a writable uint8 array; its length
        is the capacity).  Returns the encoded length, -length when allowCopy stored the block raw, 0 when nothing
        is pending; raises like the reference when the block does not fit."""
        return LZ4FastChainEncoder.EncodeMany([self], [target], allowCopy)[0]

    @staticmethod
    def EncodeMany(encoders, targets, allowCopy: bool = False, device: int = 0) -> list:
        """Encode() on every encoder at once: encoders[i] encodes its pending bytes into targets[i] (writable
        uint8 arrays), all in ONE GPU call.  The encoders must be distinct.  Returns the per-encoder results of
        Encode.  If a block does not fit, its encoder is not committed (Encode throws before Commit) and
        InvalidOperationException is raised after every other encoder has been advanced."""
        encoders = list(encoders)
        if len(encoders) != len(targets):
            raise ValueError("one target per encoder")
        if len({id(e) for e in encoders}) != len(encoders):
            raise ValueError("an encoder may take only one block per call")
        for e in encoders:
            e._check()
        todo = [i for i, e in enumerate(encoders) if e._pointer - e._index > 0]
        res = [0] * len(encoders)
        if not todo:
            return res
        tg = [targets[i] if isinstance(targets[i], np.ndarray) else np.frombuffer(targets[i], dtype=np.uint8)
              for i in todo]
        # every ring and state goes up as it is: block k starts at ring k's _inputIndex, behind its history
        rings = [encoders[i]._in for i in todo]
        base = np.concatenate(rings)
        roff = np.zeros(len(todo), dtype=np.int64)
        roff[1:] = np.cumsum([r.size for r in rings[:-1]])
        src_off = roff + np.array([encoders[i]._index for i in todo], dtype=np.int64)
        src_len = np.array([encoders[i]._pointer - encoders[i]._index for i in todo], dtype=np.int32)
        prefix = np.array([encoders[i]._index for i in todo], dtype=np.int32)
        caps = np.array([t.size for t in tg], dtype=np.int32)
        dst = np.zeros(int(caps.astype(np.int64).sum()) + 16, dtype=np.uint8)
        doff = np.zeros(len(todo), dtype=np.int64)
        doff[1:] = np.cumsum(caps[:-1].astype(np.int64))
        state = np.concatenate([encoders[i]._state for i in todo])
        soff = np.arange(len(todo), dtype=np.int64) * N.CHAIN_STATE_BYTES
        out = encode_chain_batch_host(base, src_off, src_len, prefix, dst, doff, caps, state, soff, 0, device,
                                      LZ4Codec.Enforce32)
        failed = False
        for k, i in enumerate(todo):
            e, r, n = encoders[i], int(out[k]), int(src_len[k])
            e._state[:] = state[soff[k]:soff[k] + N.CHAIN_STATE_BYTES]  # the engine advanced it, fit or not
            if r <= 0:                                                    # LZ4EncoderBase.cs:75-77
                failed = True
                res[i] = r
                continue
            if allowCopy and r >= n:                                      # :79-83
                tg[k][:n] = e._in[e._index:e._index + n]
                r = -n
            else:
                tg[k][:r] = dst[doff[k]:doff[k] + r]
            e._commit()
            res[i] = r
        if failed:
            raise RuntimeError("Failed to encode chunk. Target buffer too small.")   # InvalidOperationException
        return res

    def Dispose(self) -> None:
        self._disposed = True

    # -- LZ4EncoderBase.cs:90-97, LZ4FastChainEncoder.cs:40-41 ---------------------------------------------------
    def _commit(self) -> None:
        self._index = self._pointer
        if self._index + self._block <= self._in_len:
            return
        self._index = self._pointer = self._copy_dict(self._pointer)

    def _copy_dict(self, length: int) -> int:
        """LZ4_saveDict(ctx, buffer, length): the last min(length, 64 KiB, dictSize) bytes move to the front.  The
        state's dictSize is not written: the next block passes this length as its prefix, and the GPU clamps
        dictSize to it the same way."""
        size = min(length, K64, int(self.State[4097]))
        self._in[:size] = self._in[self._index - size:self._index].copy()
        return size

    def _check(self) -> None:
        if self._disposed:
            raise RuntimeError("ObjectDisposedException")


class LZ4Encoder:
    """LZ4Encoder.Create -- Encoders/LZ4Encoder.cs:14-29."""

    @staticmethod
    def Create(chaining: bool, level: LZ4Level = LZ4Level.L00_FAST, blockSize: int = 65536, extraBlocks: int = 0):
        if not chaining:
            return LZ4BlockEncoder(level, blockSize)
        if LZ4Level(level) < LZ4Level.L03_HC:
            return LZ4FastChainEncoder(blockSize, extraBlocks)
        raise NotImplementedError("LZ4HighChainEncoder (chained HC levels) stays with the managed engine")


class LZ4Decoder:
    """LZ4Decoder.Create -- Encoders/LZ4Decoder.cs:13-15."""

    @staticmethod
    def Create(chaining: bool, blockSize: int, extraBlocks: int = 0):
        return LZ4ChainDecoder(blockSize, extraBlocks) if chaining else LZ4BlockDecoder(blockSize)
