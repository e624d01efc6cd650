"""LZ4 Frame container around BATCHED independent blocks (SURVEY.md 8f row 2).

Writer and reader follow the reference's frame code for the case this library accelerates --
independent blocks (`Chaining = false`), `L00_FAST`:
    Streams/Frames/LZ4FrameWriter.cs:57-108 (header: magic 0x184D2204, FLG, BD, HC),
    :159-189 (block length code with bit 31 = stored raw, XXH32 block / content checksums),
    LZ4FrameWriter.blocking.cs:22-33,88-97 (block = length code, data, [checksum]; tail = end mark,
    [content checksum]), LZ4FrameReader.blocking.cs:57-144 (header / block parsing and checks);
    format: orig/doc/lz4_Frame_format.md.
All blocks of a frame go through ONE k4lz4_encode_batch / k4lz4_decode_batch call and ONE
k4lz4_xxh32_batch call; only the serial parts (header byte, content checksum, byte layout) run
on the host.  Frames are interoperable with upstream lz4 (tests decode them with
orig/lib/lz4frame.c and decode upstream's frames here).  Frames of linked blocks (the reference's
default, LZ4EncoderSettings.ChainBlocks) are written (write_frames, L00_FAST) and read (read_frames) on the
GPU as well, batched across frames; content size and dictionary ids are not written (the reference itself
throws NotImplemented for them, LZ4FrameWriter.cs:89-95).
"""
from __future__ import annotations

import struct

import numpy as np

from . import _native as N
from .batch import decode_batch_flat_host, decode_chain_blocks_host, encode_batch_flat_host, encode_chain_batch_host

MAGIC = 0x184D2204
_BLOCK_SIZES = {4: 1 << 16, 5: 1 << 18, 6: 1 << 20, 7: 1 << 22}


class InvalidDataException(ValueError):
    """Malformed frame (the reference throws InvalidDataException from LZ4FrameReader)."""


def xxh32(data, seed: int = 0) -> int:
    a = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    return int(N.lib().k4lz4_xxh32(a.ctypes.data if a.size else None, int(a.size), seed))


def xxh32_batch(base: np.ndarray, off, length, seed: int = 0, device: int = 0) -> np.ndarray:
    off = np.ascontiguousarray(off, dtype=np.int64)
    length = np.ascontiguousarray(length, dtype=np.int32)
    out = np.zeros(len(length), dtype=np.uint32)
    if len(length):
        N.check(N.lib().k4lz4_xxh32_batch(base.ctypes.data, off.ctypes.data, length.ctypes.data, seed,
                                          out.ctypes.data, len(length), N.MEM_HOST, None, device))
    return out


def _block_size_code(block_size: int) -> int:                # LZ4FrameWriter.cs:183-188
    for code in (4, 5, 6, 7):
        if block_size <= _BLOCK_SIZES[code]:
            return code
    raise ValueError(f"Invalid block size {block_size} for stream")


def _header(code: int, chaining: bool, block_checksum: bool, content_checksum: bool) -> list:
    flg = (1 << 6) | (int(not chaining) << 5) | (int(block_checksum) << 4) | (int(content_checksum) << 2)
    head = struct.pack("<IBB", MAGIC, flg, code << 4)
    return [head, bytes([(xxh32(head[4:6]) >> 8) & 0xFF])]       # HC, LZ4FrameWriter.cs:100-102


def _blocks(out: list, stored, raw, block_checksum: bool, device: int) -> None:
    """Appends the blocks of a frame (length code with bit 31 = stored raw, data, [XXH32 of the stored bytes],
    LZ4FrameWriter.cs:159-175) and the end mark."""
    if block_checksum and stored:
        base = np.frombuffer(b"".join(stored), dtype=np.uint8)
        ln = np.array([len(b) for b in stored], dtype=np.int32)
        off = np.zeros(len(stored), dtype=np.int64)
        off[1:] = np.cumsum(ln[:-1].astype(np.int64))
        sums = xxh32_batch(base, off, ln, 0, device)
    for i, body in enumerate(stored):
        out.append(struct.pack("<I", len(body) | (0x80000000 if raw[i] else 0)))
        out.append(body)
        if block_checksum:
            out.append(struct.pack("<I", int(sums[i])))
    out.append(struct.pack("<I", 0))                            # end mark, blocking.cs:94


def write_frames(datas, block_size: int = 65536, block_checksum: bool = False, content_checksum: bool = False,
                 level: int = 0, device: int = 0, chaining: bool = True) -> list:
    """Many LZ4 frames, one per item of `datas` (LZ4FrameWriter with the default Chaining = true, L00_FAST).
    Linked frames are encoded together: step k encodes block k of every frame that has one with ONE
    k4lz4_encode_chain_batch call, each frame's earlier blocks being its history (LZ4FastChainEncoder).  A block
    is encoded with capacity MaximumOutputSize(blockSize) and stored raw when it does not shrink
    (LZ4FrameWriter.cs:105,130-157); a raw block stays history.  chaining=False writes independent frames
    (write_frame).  Chained HC levels stay with the managed engine (NotImplementedError)."""
    if not chaining:
        return [write_frame(d, block_size, block_checksum, content_checksum, level, device) for d in datas]
    if level >= 3:
        raise NotImplementedError("LZ4HighChainEncoder (chained HC levels) stays with the managed engine")
    srcs = [np.frombuffer(bytes(d), dtype=np.uint8) if not isinstance(d, np.ndarray) else d for d in datas]
    code = _block_size_code(block_size)
    bs = max(1024, (block_size + 1023) // 1024 * 1024)          # LZ4EncoderBase.cs:29
    bound = N.lib().k4lz4_max_output_size(bs)
    nf = len(srcs)
    base = np.concatenate(srcs) if nf and sum(int(s.size) for s in srcs) else np.zeros(1, dtype=np.uint8)
    foff = np.zeros(nf, dtype=np.int64)
    if nf:
        foff[1:] = np.cumsum([int(s.size) for s in srcs[:-1]])
    nbs = [(int(s.size) + bs - 1) // bs for s in srcs]
    state = np.zeros(nf * N.CHAIN_STATE_BYTES, dtype=np.uint8)
    stored = [[] for _ in srcs]
    raws = [[] for _ in srcs]
    for k in range(max(nbs, default=0)):
        fs = [j for j in range(nf) if k < nbs[j]]
        so = np.array([foff[j] + k * bs for j in fs], dtype=np.int64)
        sl = np.array([min(bs, int(srcs[j].size) - k * bs) for j in fs], dtype=np.int32)
        pl = np.full(len(fs), min(k * bs, 0x7FFFFFFF), dtype=np.int32)   # the frame so far, in front
        caps = np.full(len(fs), bound, dtype=np.int32)
        doff = np.arange(len(fs), dtype=np.int64) * bound
        dst = np.zeros(len(fs) * bound + 16, dtype=np.uint8)
        st_off = np.array(fs, dtype=np.int64) * N.CHAIN_STATE_BYTES
        enc = encode_chain_batch_host(base, so, sl, pl, dst, doff, caps, state, st_off, level, device)
        if (enc <= 0).any():
            raise RuntimeError("Failed to encode chunk. Target buffer too small.")   # LZ4EncoderBase.cs:75-77
        for i, j in enumerate(fs):
            raw = int(enc[i]) >= int(sl[i])                      # allowCopy, :79-83
            body = base[so[i]:so[i] + sl[i]] if raw else dst[doff[i]:doff[i] + enc[i]]
            stored[j].append(body.tobytes())
            raws[j].append(raw)
    frames = []
    for j in range(nf):
        out = _header(code, True, block_checksum, content_checksum)
        _blocks(out, stored[j], raws[j], block_checksum, device)
        if content_checksum:
            out.append(struct.pack("<I", xxh32(srcs[j])))       # :95
        frames.append(b"".join(out))
    return frames


def write_frame(data, block_size: int = 65536, block_checksum: bool = False,
                content_checksum: bool = False, level: int = 0, device: int = 0, chaining: bool = False) -> bytes:
    """One LZ4 frame holding `data`: independent blocks (LZ4FrameWriter with Chaining = false), or with
    chaining=True linked blocks (write_frames)."""
    if chaining:
        return write_frames([data], block_size, block_checksum, content_checksum, level, device)[0]
    src = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    code = _block_size_code(block_size)
    bs = max(1024, (block_size + 1023) // 1024 * 1024)          # LZ4EncoderBase.cs:29
    flg = (1 << 6) | (1 << 5) | (int(block_checksum) << 4) | (int(content_checksum) << 2)
    bd = code << 4
    head = struct.pack("<IBB", MAGIC, flg, bd)
    out = [head, bytes([(xxh32(head[4:6]) >> 8) & 0xFF])]       # HC, LZ4FrameWriter.cs:100-102
    n = int(src.size)
    nb = (n + bs - 1) // bs
    if nb:
        lens = np.full(nb, bs, dtype=np.int32)
        lens[-1] = n - (nb - 1) * bs
        off = np.arange(nb, dtype=np.int64) * bs
        bound = N.lib().k4lz4_max_output_size(bs)
        caps = np.full(nb, bound, dtype=np.int32)
        doff = np.arange(nb, dtype=np.int64) * bound
        dst = np.zeros(nb * bound + 16, dtype=np.uint8)
        enc = encode_batch_flat_host(src, off, lens, dst, doff, caps, level, device)
        if (enc <= 0).any():
            raise RuntimeError("Failed to encode chunk. Target buffer too small.")   # LZ4EncoderBase.cs:75-77
        raw = enc >= lens                                       # allowCopy: stored as is, :79-83
        store_len = np.where(raw, lens, enc).astype(np.int32)
        if block_checksum:                                      # checksum of the bytes as stored, :169-175
            cbase = np.concatenate([dst, src]) if raw.any() else dst
            coff = np.where(raw, off + dst.size, doff)
            sums = xxh32_batch(cbase, coff, store_len, 0, device)
        for i in range(nb):
            body = src[off[i]:off[i] + lens[i]] if raw[i] else dst[doff[i]:doff[i] + enc[i]]
            out.append(struct.pack("<I", int(store_len[i]) | (0x80000000 if raw[i] else 0)))   # :159-160
            out.append(body.tobytes())
            if block_checksum:
                out.append(struct.pack("<I", int(sums[i])))
    out.append(struct.pack("<I", 0))                            # end mark, blocking.cs:94
    if content_checksum:
        out.append(struct.pack("<I", xxh32(src)))               # :95
    return b"".join(out)


class _Frame:
    """A parsed frame: header flags and the position, length and raw flag of every block."""

    def __init__(self, f: bytes):
        if len(f) < 7 or struct.unpack_from("<I", f, 0)[0] != MAGIC:
            raise InvalidDataException("LZ4 frame magic number expected")
        flg, bd = f[4], f[5]
        if (flg >> 6) & 0x11 != 1:                               # sic: the reference masks with 0x11, :85
            raise InvalidDataException(f"LZ4 frame version unknown: {(flg >> 6) & 0x11}")
        self.chaining = ((flg >> 5) & 1) == 0
        self.block_checksum = bool((flg >> 4) & 1)
        has_size = bool((flg >> 3) & 1)
        content_checksum = bool((flg >> 2) & 1)
        if flg & 1:
            raise NotImplementedError("Predefined dictionaries feature is not implemented")   # :108-110
        p = 6 + (8 if has_size else 0)
        if len(f) < p + 1 or ((xxh32(f[4:p]) >> 8) & 0xFF) != f[p]:
            raise InvalidDataException("Invalid LZ4 frame header checksum")
        p += 1
        self.max_block = _BLOCK_SIZES.get((bd >> 4) & 7, 1 << 16)    # LZ4FrameReader.cs:55-59
        pos, lens, raws, sums = [], [], [], []
        while True:
            if p + 4 > len(f):
                raise InvalidDataException("Unexpected end of stream")
            code = struct.unpack_from("<I", f, p)[0]
            p += 4
            if code == 0:
                break
            blen = code & 0x7FFFFFFF
            if p + blen + (4 if self.block_checksum else 0) > len(f):
                raise InvalidDataException("Unexpected end of stream")
            pos.append(p); lens.append(blen); raws.append(bool(code & 0x80000000))
            p += blen
            if self.block_checksum:
                sums.append(struct.unpack_from("<I", f, p)[0])
                p += 4
        self.expect_content = None
        if content_checksum:
            if p + 4 > len(f):
                raise InvalidDataException("Unexpected end of stream")
            self.expect_content = struct.unpack_from("<I", f, p)[0]
        self.f, self.pos, self.lens, self.raws, self.sums = f, pos, lens, raws, sums

    def check_blocks(self, device: int) -> None:
        if self.block_checksum and self.pos:
            base = np.frombuffer(self.f, dtype=np.uint8)
            got = xxh32_batch(base, np.array(self.pos, dtype=np.int64), np.array(self.lens, dtype=np.int32), 0, device)
            if (got != np.array(self.sums, dtype=np.uint32)).any():
                raise InvalidDataException("Invalid block checksum")

    def check_content(self, content: bytes) -> bytes:
        if self.expect_content is not None and xxh32(content) != self.expect_content:
            raise InvalidDataException("Invalid content checksum")
        return content


def _read_independent(fr: _Frame, device: int) -> bytes:
    f, pos, lens, max_block = fr.f, fr.pos, fr.lens, fr.max_block
    nb = len(pos)
    if nb == 0:
        return b""
    base = np.frombuffer(f, dtype=np.uint8)
    off = np.array(pos, dtype=np.int64)
    ln = np.array(lens, dtype=np.int32)
    fr.check_blocks(device)
    is_raw = np.array(fr.raws, dtype=bool)
    caps = np.full(nb, max_block + 8, dtype=np.int32)           # LZ4BlockDecoder.cs:26
    doff = np.arange(nb, dtype=np.int64) * (max_block + 8)
    dst = np.zeros(nb * (max_block + 8) + 16, dtype=np.uint8)
    dec_len = np.where(is_raw, 0, ln).astype(np.int32)           # raw blocks are injected, not decoded
    out_len = decode_batch_flat_host(base, off, dec_len, dst, doff, caps, device)
    parts = []
    for i in range(nb):
        if is_raw[i]:
            if lens[i] > max_block + 8:
                raise InvalidDataException("block larger than the declared block size")
            parts.append(f[pos[i]:pos[i] + lens[i]])
        else:
            r = int(out_len[i])
            if r < 0 or (r == 0 and lens[i] > 0):
                raise InvalidDataException("corrupted block")   # InvalidOperationException in LZ4BlockDecoder.cs:50-51
            parts.append(dst[doff[i]:doff[i] + r].tobytes())
    return b"".join(parts)


def _read_linked(frames: list, device: int) -> list:
    """Linked-block frames, batched ACROSS frames: step k decodes block k of every frame that has one with ONE
    k4lz4_decode_chain_batch call.  A block decodes with dstCap = the frame's maximum block size and the
    frame's output so far as history (LZ4ChainDecoder, LZ4FrameReader.cs:93-106); a raw block is history too
    (Inject, :93-96)."""
    for fr in frames:
        fr.check_blocks(device)
    outs = [bytearray() for _ in frames]
    steps = max((len(fr.pos) for fr in frames), default=0)
    for k in range(steps):
        todo = []
        for j, fr in enumerate(frames):
            if k >= len(fr.pos):
                continue
            blk = fr.f[fr.pos[k]:fr.pos[k] + fr.lens[k]]
            if fr.raws[k]:
                if fr.lens[k] > max(fr.max_block, 65536):            # LZ4ChainDecoder.Inject, :69-70
                    raise InvalidDataException("block larger than the declared block size")
                outs[j] += blk
            else:
                todo.append((j, blk))
        if not todo:
            continue
        res, data = decode_chain_blocks_host([b for _, b in todo], [outs[j] for j, _ in todo],
                                             [frames[j].max_block for j, _ in todo], device)
        for i, (j, _) in enumerate(todo):
            if res[i] < 0:
                raise InvalidDataException("corrupted block")   # InvalidOperationException in LZ4ChainDecoder.cs:55-56
            outs[j] += data[i]
    return [fr.check_content(bytes(o)) for fr, o in zip(frames, outs)]


def read_frames(frames, device: int = 0) -> list:
    """Decodes many frames, linked or independent; returns their contents in order.  Independent frames are
    read as by read_frame; the linked ones together, one block of every frame per GPU call.  Raises like
    read_frame for the first bad frame."""
    parsed = [_Frame(bytes(f)) for f in frames]
    out = [None] * len(parsed)
    linked = [i for i, fr in enumerate(parsed) if fr.chaining]
    for i, fr in enumerate(parsed):
        if not fr.chaining:
            out[i] = fr.check_content(_read_independent(fr, device))
    for i, content in zip(linked, _read_linked([parsed[i] for i in linked], device)):
        out[i] = content
    return out


def read_frame(frame, device: int = 0) -> bytes:
    """Decodes one frame (LZ4FrameReader.blocking.cs:57-144); raises InvalidDataException on a bad magic
    number, header checksum, block or content checksum or a corrupted block.  A frame of linked blocks goes
    through read_frames."""
    fr = _Frame(bytes(frame))
    if fr.chaining:
        return read_frames([fr.f], device)[0]
    return fr.check_content(_read_independent(fr, device))
