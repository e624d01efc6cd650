"""LZ4 Frame container, batched across frames on the GPU (SURVEY.md 8f row 2).

Writer and reader follow the reference's frame code at `L00_FAST`:
    Streams/Frames/LZ4FrameWriter.cs:57-108 (header: magic 0x184D2204, FLG, BD, HC),
    :159-189 (block length code with bit 31 = stored raw, XXH32 block / content checksums),
    LZ4FrameWriter.blocking.cs:22-33,88-97 (block = length code, data, [checksum]; tail = end mark,
    [content checksum]), LZ4FrameReader.blocking.cs:57-144 (header / block parsing and checks);
    format: orig/doc/lz4_Frame_format.md.
Whole frames, linked (the reference's default, LZ4EncoderSettings.ChainBlocks) or independent, are encoded and
decoded by the library's frame calls (k4lz4_frame_encode_batch / _decode_batch / _content_size_batch), many frames
per call: header, block walk, raw/compressed choice, layout and checksums run on the GPU.  This module is a thin
mirror over them.  Frames are interoperable with upstream lz4 (tests decode them with orig/lib/lz4frame.c and
decode upstream's frames here); content size and dictionary ids are not written (the reference itself throws
NotImplemented for them, LZ4FrameWriter.cs:89-95).  The *WithDictionary calls and Info go beyond the reference:
upstream's frames against a dictionary (LZ4F_compressBegin_usingCDict, lz4 -D), encoded and decoded on the GPU.
_Frame restates the device parse on the CPU (dictionary=True: the dictionary calls' parse).
"""
from __future__ import annotations

import struct

import numpy as np

from . import _native as N
from .batch import _pack, _slices, _slots, encoder_fn
from .codec import LZ4Codec

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


def _flags(chaining: bool, block_checksum: bool, content_checksum: bool) -> int:
    return ((0 if chaining else N.FRAME_INDEPENDENT) | (N.FRAME_BLOCK_CHECKSUM if block_checksum else 0) |
            (N.FRAME_CONTENT_CHECKSUM if content_checksum else 0))


def _u8(d) -> np.ndarray:
    return d if isinstance(d, np.ndarray) else np.frombuffer(bytes(d), dtype=np.uint8)


def _native_block_size(block_size: int) -> int:
    _block_size_code(block_size)                                # ValueError beyond 4 MiB, as before
    return max(int(block_size), 1)                              # <= 0 rounds to 1 KiB either way (LZ4EncoderBase.cs:29)


class LZ4Frame:
    """LZ4Frame.Encode / Decode over whole buffers (k4lz4_frame_*): every frame of a call is encoded or decoded on
    the GPU, header, block walk, layout and checksums included.  Encoding follows LZ4Codec.Enforce32 at each call.  Host memory takes bytes / numpy arrays; the
    *_device forms take torch tensors on the GPU (uint8 data, int64 offsets, int32 lengths and results) and only
    enqueue work on `stream` (after one wait for the block and step counts)."""

    @staticmethod
    def Bound(length: int, block_size: int = 65536, chaining: bool = True, block_checksum: bool = False,
              content_checksum: bool = False) -> int:
        r = int(N.lib().k4lz4_frame_bound(int(length), _native_block_size(block_size),
                                           _flags(chaining, block_checksum, content_checksum)))
        if r < 0:
            N.check(r)
        return r

    @staticmethod
    def EncodeMany(datas, block_size: int = 65536, chaining: bool = True, block_checksum: bool = False,
                   content_checksum: bool = False, level: int = 0, device: int = 0):
        """-> (list of frames, int32 results): the frame's length, or K4LZ4_R_DELEGATE for level >= 3."""
        src, so, sl = _pack([_u8(d) for d in datas])
        bs, fl = _native_block_size(block_size), _flags(chaining, block_checksum, content_checksum)
        caps = [LZ4Frame.Bound(int(x), block_size, chaining, block_checksum, content_checksum) for x in sl]
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(encoder_fn("k4lz4_frame_encode_batch", LZ4Codec.Enforce32)(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                 do.ctypes.data, dc.ctypes.data, out.ctypes.data, len(sl), bs, fl,
                                                 int(level), N.MEM_HOST, None, int(device)))
        return _slices(dst, do, out), out

    @staticmethod
    def ContentSizes(frames, device: int = 0) -> np.ndarray:
        src, so, sl = _pack([_u8(f) for f in frames])
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(N.lib().k4lz4_frame_content_size_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data,
                                                       out.ctypes.data, len(sl), N.MEM_HOST, None, int(device)))
        return out

    @staticmethod
    def DecodeMany(frames, caps=None, device: int = 0):
        """-> (list of contents, int32 results).  caps default to each frame's content size."""
        frames = [_u8(f) for f in frames]
        if caps is None:
            caps = np.maximum(LZ4Frame.ContentSizes(frames, device), 0)
        src, so, sl = _pack(frames)
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(N.lib().k4lz4_frame_decode_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                 do.ctypes.data, dc.ctypes.data, out.ctypes.data, len(sl),
                                                 N.MEM_HOST, None, int(device)))
        return _slices(dst, do, out), out

    @staticmethod
    def Encode(data, block_size: int = 65536, chaining: bool = True, block_checksum: bool = False,
               content_checksum: bool = False, level: int = 0, device: int = 0) -> bytes:
        return write_frames([data], block_size, block_checksum, content_checksum, level, device, chaining)[0]

    @staticmethod
    def Decode(frame, device: int = 0) -> bytes:
        return read_frames([frame], device)[0]

    @staticmethod
    def ContentSize(frame, device: int = 0) -> int:
        r = int(LZ4Frame.ContentSizes([frame], device)[0])
        _raise_for(r)
        return r

    @staticmethod
    def encode_many_device(src, src_off, src_len, dst, dst_off, dst_cap, out_len, block_size: int = 65536,
                           chaining: bool = True, block_checksum: bool = False, content_checksum: bool = False,
                           level: int = 0, stream: int = 0, device: int = -1) -> None:
        N.check(encoder_fn("k4lz4_frame_encode_batch", LZ4Codec.Enforce32)(
            src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(), dst.data_ptr(), dst_off.data_ptr(),
            dst_cap.data_ptr(), out_len.data_ptr(), int(src_len.numel()), _native_block_size(block_size),
            _flags(chaining, block_checksum, content_checksum), int(level), N.MEM_DEVICE, stream or None, int(device)))

    @staticmethod
    def content_sizes_device(src, src_off, src_len, out_size, stream: int = 0, device: int = -1) -> None:
        N.check(N.lib().k4lz4_frame_content_size_batch(src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(),
                                                       out_size.data_ptr(), int(src_len.numel()), N.MEM_DEVICE,
                                                       stream or None, int(device)))

    @staticmethod
    def decode_many_device(src, src_off, src_len, dst, dst_off, dst_cap, out_len, stream: int = 0,
                           device: int = -1) -> None:
        N.check(N.lib().k4lz4_frame_decode_batch(src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(),
                                                 dst.data_ptr(), dst_off.data_ptr(), dst_cap.data_ptr(),
                                                 out_len.data_ptr(), int(src_len.numel()), N.MEM_DEVICE,
                                                 stream or None, int(device)))

    # ---- against a dictionary (k4lz4_frame_encode_dict_batch / _decode_dict_batch / k4lz4_frame_info_batch):
    # upstream's LZ4F_compressBegin_usingCDict frames and lz4 -D; the reference has no dictionary frames.

    @staticmethod
    def EncodeManyWithDictionary(datas, dictionaries, dict_ids=None, block_size: int = 65536, chaining: bool = True,
                                 block_checksum: bool = False, content_checksum: bool = False, level: int = 0,
                                 device: int = 0):
        """-> (list of frames, int32 results): frame i of datas[i] against dictionaries[i], byte for byte upstream's
        CDict frame (dictID = dict_ids[i]; 0 or None writes no ID); K4LZ4_R_DELEGATE for level >= 3.  block_size is
        64 KiB, 256 KiB, 1 MiB or 4 MiB."""
        src, so, sl = _pack([_u8(d) for d in datas])
        dic, do_, dl = _pack([_u8(d) for d in dictionaries])
        ids = np.zeros(len(sl), dtype=np.uint32) if dict_ids is None else np.ascontiguousarray(dict_ids, dtype=np.uint32)
        if len(dl) != len(sl) or len(ids) != len(sl):
            raise ValueError("one dictionary and one ID per frame")
        fl = _flags(chaining, block_checksum, content_checksum)
        caps = [LZ4Frame.Bound(int(x), block_size, chaining, block_checksum, content_checksum) + (4 if ids[i] else 0)
                for i, x in enumerate(sl)]
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(N.lib().k4lz4_frame_encode_dict_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                      do.ctypes.data, dc.ctypes.data, dic.ctypes.data,
                                                      do_.ctypes.data, dl.ctypes.data, ids.ctypes.data,
                                                      out.ctypes.data, len(sl), int(block_size), fl, int(level),
                                                      N.MEM_HOST, None, int(device)))
        return _slices(dst, do, out), out

    @staticmethod
    def Info(frames, device: int = 0):
        """-> (int32 content sizes or verdicts, as ContentSizes but with the dictionary flag accepted;
        int64 dictIDs, -1 for a frame without a dictID field)."""
        src, so, sl = _pack([_u8(f) for f in frames])
        out = np.full(len(sl), -1, dtype=np.int32)
        ids = np.full(len(sl), -1, dtype=np.int64)
        N.check(N.lib().k4lz4_frame_info_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, out.ctypes.data,
                                               ids.ctypes.data, len(sl), N.MEM_HOST, None, int(device)))
        return out, ids

    @staticmethod
    def DecodeManyWithDictionary(frames, dictionaries, caps=None, device: int = 0):
        """-> (list of contents, int32 results), frame i against dictionaries[i] (with or without a dictID field:
        the ID is not checked).  caps default to each frame's content size."""
        frames = [_u8(f) for f in frames]
        if caps is None:
            caps = np.maximum(LZ4Frame.Info(frames, device)[0], 0)
        src, so, sl = _pack(frames)
        dic, do_, dl = _pack([_u8(d) for d in dictionaries])
        if len(dl) != len(sl):
            raise ValueError("one dictionary per frame")
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(N.lib().k4lz4_frame_decode_dict_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                      do.ctypes.data, dc.ctypes.data, dic.ctypes.data,
                                                      do_.ctypes.data, dl.ctypes.data, out.ctypes.data, len(sl),
                                                      N.MEM_HOST, None, int(device)))
        return _slices(dst, do, out), out

    @staticmethod
    def EncodeWithDictionary(data, dictionary, dict_id: int = 0, block_size: int = 65536, chaining: bool = True,
                             block_checksum: bool = False, content_checksum: bool = False, level: int = 0,
                             device: int = 0) -> bytes:
        if level >= 3:
            raise NotImplementedError("dictionary frames at the HC levels are not implemented")
        frames, out = LZ4Frame.EncodeManyWithDictionary([data], [dictionary], [dict_id], block_size, chaining,
                                                        block_checksum, content_checksum, level, device)
        if out[0] < 0:
            raise RuntimeError("Failed to encode the frame")
        return frames[0]

    @staticmethod
    def DecodeWithDictionary(frame, dictionary, device: int = 0) -> bytes:
        contents, out = LZ4Frame.DecodeManyWithDictionary([frame], [dictionary], None, device)
        _raise_for(int(out[0]))
        return contents[0]

    @staticmethod
    def encode_many_with_dictionary_device(src, src_off, src_len, dst, dst_off, dst_cap, dict_base, dict_off,
                                           dict_len, dict_id, out_len, block_size: int = 65536, chaining: bool = True,
                                           block_checksum: bool = False, content_checksum: bool = False,
                                           level: int = 0, stream: int = 0, device: int = -1) -> None:
        """dict_id: a uint32-sized tensor (torch.int32 holding the IDs' bits) or None."""
        N.check(N.lib().k4lz4_frame_encode_dict_batch(
            src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(), dst.data_ptr(), dst_off.data_ptr(),
            dst_cap.data_ptr(), dict_base.data_ptr(), dict_off.data_ptr(), dict_len.data_ptr(),
            dict_id.data_ptr() if dict_id is not None else None, out_len.data_ptr(), int(src_len.numel()),
            int(block_size), _flags(chaining, block_checksum, content_checksum), int(level), N.MEM_DEVICE,
            stream or None, int(device)))

    @staticmethod
    def decode_many_with_dictionary_device(src, src_off, src_len, dst, dst_off, dst_cap, dict_base, dict_off,
                                           dict_len, out_len, stream: int = 0, device: int = -1) -> None:
        """dict_base None: no dictionaries (dict_off / dict_len are then ignored)."""
        N.check(N.lib().k4lz4_frame_decode_dict_batch(
            src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(), dst.data_ptr(), dst_off.data_ptr(),
            dst_cap.data_ptr(), dict_base.data_ptr() if dict_base is not None else None,
            dict_off.data_ptr() if dict_base is not None else None,
            dict_len.data_ptr() if dict_base is not None else None, out_len.data_ptr(), int(src_len.numel()),
            N.MEM_DEVICE, stream or None, int(device)))

    @staticmethod
    def info_device(src, src_off, src_len, out_size, out_dict_id, stream: int = 0, device: int = -1) -> None:
        N.check(N.lib().k4lz4_frame_info_batch(src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(),
                                               out_size.data_ptr(), out_dict_id.data_ptr(), int(src_len.numel()),
                                               N.MEM_DEVICE, stream or None, int(device)))


class LZ4F:
    """Frames as upstream lz4 writes them (k4lz4_lz4f_compress_batch): LZ4F_compressFrame byte for byte, many frames
    per call.  Unlike LZ4Frame, each frame's block size shrinks to fit small contents, a one-block frame is written
    independent, every block is encoded with capacity n - 1 and stored raw when that fails, and the content size can
    be written (content_size=True, as python-lz4's store_size).  block_size is 64 KiB, 256 KiB, 1 MiB or 4 MiB;
    level 0..2 (acceleration 1).  The reference has no such call: it is liblz4's, the lz4 CLI's and python-lz4's."""

    BLOCK_SIZES = (1 << 16, 1 << 18, 1 << 20, 1 << 22)

    @staticmethod
    def flags(linked: bool = True, block_checksum: bool = False, content_checksum: bool = False,
              content_size: bool = False) -> int:
        return _flags(linked, block_checksum, content_checksum) | (N.FRAME_CONTENT_SIZE if content_size else 0)

    @staticmethod
    def bound(length: int, block_size: int = 65536, linked: bool = True, block_checksum: bool = False,
              content_checksum: bool = False, content_size: bool = False) -> int:
        """LZ4F_compressFrameBound for these preferences."""
        r = int(N.lib().k4lz4_lz4f_compress_bound(int(length), int(block_size),
                                                   LZ4F.flags(linked, block_checksum, content_checksum, content_size)))
        if r < 0:
            N.check(r)
        return r

    @staticmethod
    def compress_many(datas, block_size: int = 65536, linked: bool = True, block_checksum: bool = False,
                      content_checksum: bool = False, content_size: bool = False, level: int = 0, device: int = 0):
        """-> (list of frames, int32 results): the frame's length, or K4LZ4_R_DELEGATE for level >= 3 or < 0."""
        src, so, sl = _pack([_u8(d) for d in datas])
        fl = LZ4F.flags(linked, block_checksum, content_checksum, content_size)
        caps = [LZ4F.bound(int(x), block_size, linked, block_checksum, content_checksum, content_size) for x in sl]
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(N.lib().k4lz4_lz4f_compress_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                  do.ctypes.data, dc.ctypes.data, out.ctypes.data, len(sl),
                                                  int(block_size), fl, int(level), N.MEM_HOST, None, int(device)))
        return _slices(dst, do, out), out

    @staticmethod
    def compress_many_device(src, src_off, src_len, dst, dst_off, dst_cap, out_len, block_size: int = 65536,
                             linked: bool = True, block_checksum: bool = False, content_checksum: bool = False,
                             content_size: bool = False, level: int = 0, stream: int = 0, device: int = -1) -> None:
        """Torch tensors on the GPU (uint8 data, int64 offsets, int32 lengths and results); only enqueues work on
        `stream`, after one wait for the block and step counts."""
        N.check(N.lib().k4lz4_lz4f_compress_batch(
            src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(), dst.data_ptr(), dst_off.data_ptr(),
            dst_cap.data_ptr(), out_len.data_ptr(), int(src_len.numel()), int(block_size),
            LZ4F.flags(linked, block_checksum, content_checksum, content_size), int(level), N.MEM_DEVICE,
            stream or None, int(device)))

    @staticmethod
    def decompressed_sizes(streams, device: int = 0):
        """-> (int32 sizes, int32 errors, int32 ends) of whole .lz4 streams (k4lz4_lz4f_decompressed_size_batch): the
        content length, or -1 with the error that needs no decoding; see decompress_many for the codes."""
        src, so, sl = _pack([_u8(s) for s in streams])
        out, err, end = (np.zeros(len(sl), dtype=np.int32) for _ in range(3))
        N.check(N.lib().k4lz4_lz4f_decompressed_size_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data,
                                                           out.ctypes.data, err.ctypes.data, end.ctypes.data,
                                                           len(sl), N.MEM_HOST, None, int(device)))
        return out, err, end

    @staticmethod
    def decompress_many(streams, dictionaries=None, caps=None, device: int = 0):
        """Whole .lz4 streams read as `lz4 -d [-D dict]` reads them (k4lz4_lz4f_decompress_batch): concatenated
        frames, skippable frames, legacy members, trailing data.  -> (list of contents, int32 results, int32 errors,
        int32 ends).  A result is the content length, -1 on an error or K4LZ4_R_DST_SMALL; an error is
        (cli << 8) | lz4f, cli being the lz4 CLI's exit code and lz4f the LZ4F_errorCodes value for cli = 66; an end
        is where reading stopped (the stream's length, or the start of undecodable trailing data).  caps default to
        each stream's decompressed size."""
        streams = [_u8(s) for s in streams]
        if caps is None:
            caps = np.maximum(LZ4F.decompressed_sizes(streams, device)[0], 0)
        src, so, sl = _pack(streams)
        dic = do_ = dl = None
        if dictionaries is not None:
            dic, do_, dl = _pack([_u8(d) for d in dictionaries])
            if len(dl) != len(sl):
                raise ValueError("one dictionary per stream")
        dst, do, dc = _slots(caps)
        out, err, end = (np.zeros(len(sl), dtype=np.int32) for _ in range(3))
        N.check(N.lib().k4lz4_lz4f_decompress_batch(
            src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data, do.ctypes.data, dc.ctypes.data,
            None if dic is None else dic.ctypes.data, None if dic is None else do_.ctypes.data,
            None if dic is None else dl.ctypes.data, out.ctypes.data, err.ctypes.data, end.ctypes.data, len(sl),
            N.MEM_HOST, None, int(device)))
        return _slices(dst, do, out), out, err, end

    @staticmethod
    def decompress_many_device(src, src_off, src_len, dst, dst_off, dst_cap, out_len, out_err, out_end,
                               dict_base=None, dict_off=None, dict_len=None, stream: int = 0,
                               device: int = -1) -> None:
        """Torch tensors on the GPU (uint8 data, int64 offsets, int32 lengths, results, errors and ends); only
        enqueues work on `stream`, after one wait for the block, member and step counts."""
        ptr = (lambda t: None if t is None else t.data_ptr())
        N.check(N.lib().k4lz4_lz4f_decompress_batch(
            src.data_ptr(), src_off.data_ptr(), src_len.data_ptr(), dst.data_ptr(), dst_off.data_ptr(),
            dst_cap.data_ptr(), ptr(dict_base), ptr(dict_off), ptr(dict_len), out_len.data_ptr(), out_err.data_ptr(),
            out_end.data_ptr(), int(src_len.numel()), N.MEM_DEVICE, stream or None, int(device)))


class LZ4FError(ValueError):
    """A .lz4 stream `lz4 -d` refuses: `cli` is the CLI's exit code, `lz4f` the LZ4F_errorCodes value (cli 66)."""

    def __init__(self, cli: int, lz4f: int):
        super().__init__(f"lz4 -d error {cli}" + (f" (LZ4F error {lz4f})" if lz4f else ""))
        self.cli, self.lz4f = cli, lz4f


def lz4f_decompress(data, dictionary=None, device: int = 0) -> bytes:
    """One whole .lz4 stream, as `lz4 -d -c [-D dictionary]` decodes it; undecodable data after the first member is
    ignored, as the CLI does.  Raises LZ4FError where the CLI fails."""
    contents, out, err, _ = LZ4F.decompress_many([data], None if dictionary is None else [dictionary], None, device)
    if int(err[0]):
        raise LZ4FError(int(err[0]) >> 8, int(err[0]) & 0xFF)
    return contents[0]


def lz4f_compress(data, block_size: int = 65536, linked: bool = True, block_checksum: bool = False,
                  content_checksum: bool = False, content_size: bool = False, level: int = 0,
                  device: int = 0) -> bytes:
    """One frame, as LZ4F_compressFrame writes it.  Raises NotImplementedError for HC levels (>= 3) and
    accelerations (< 0), which this library does not encode."""
    frames, out = LZ4F.compress_many([data], block_size, linked, block_checksum, content_checksum, content_size,
                                     level, device)
    if int(out[0]) == N.R_DELEGATE:
        raise NotImplementedError(f"LZ4F_compressFrame at level {level} is not implemented")
    if int(out[0]) < 0:
        raise RuntimeError("ERROR_dstMaxSize_tooSmall")
    return frames[0]


def write_frames(datas, block_size: int = 65536, block_checksum: bool = False, content_checksum: bool = False,
                 level: int = 0, device: int = 0, chaining: bool = True) -> list:
    """Many LZ4 frames, one per item of `datas` (LZ4FrameWriter with the default Chaining = true, L00_FAST), in one
    k4lz4_frame_encode_batch call.  A block is encoded with capacity MaximumOutputSize(blockSize) and stored raw when
    it does not shrink (LZ4FrameWriter.cs:105,130-157).  chaining=False writes independent frames.  Chained HC
    levels stay with the managed engine (NotImplementedError)."""
    if chaining and level >= 3:
        raise NotImplementedError("LZ4HighChainEncoder (chained HC levels) stays with the managed engine")
    frames, out = LZ4Frame.EncodeMany(datas, block_size, chaining, block_checksum, content_checksum, level, device)
    if (out <= 0).any():
        raise RuntimeError("Failed to encode chunk. Target buffer too small.")   # LZ4EncoderBase.cs:75-77
    return frames


def write_frame(data, block_size: int = 65536, block_checksum: bool = False,
                content_checksum: bool = False, level: int = 0, device: int = 0, chaining: bool = False) -> bytes:
    """One LZ4 frame holding `data`: independent blocks (LZ4FrameWriter with Chaining = false), or with
    chaining=True linked blocks."""
    return write_frames([data], block_size, block_checksum, content_checksum, level, device, chaining)[0]

class _Frame:
    """A parsed frame: header flags and the position, length and raw flag of every block."""

    def __init__(self, f: bytes, dictionary: bool = False):
        if len(f) < 7 or struct.unpack_from("<I", f, 0)[0] != MAGIC:
            raise InvalidDataException("LZ4 frame magic number expected")
        flg, bd = f[4], f[5]
        if (flg >> 6) & 0x11 != 1:                               # sic: the reference masks with 0x11, :85
            raise InvalidDataException(f"LZ4 frame version unknown: {(flg >> 6) & 0x11}")
        self.chaining = ((flg >> 5) & 1) == 0
        self.block_checksum = bool((flg >> 4) & 1)
        has_size = bool((flg >> 3) & 1)
        content_checksum = bool((flg >> 2) & 1)
        if flg & 1 and not dictionary:
            raise NotImplementedError("Predefined dictionaries feature is not implemented")   # :108-110
        p = 6 + (8 if has_size else 0) + (4 if flg & 1 else 0)
        if len(f) < p + 1 or ((xxh32(f[4:p]) >> 8) & 0xFF) != f[p]:
            raise InvalidDataException("Invalid LZ4 frame header checksum")
        self.dict_id = struct.unpack_from("<I", f, p - 4)[0] if flg & 1 else None
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


def _raise_for(r: int) -> None:
    if r == N.R_DELEGATE:
        raise NotImplementedError("Predefined dictionaries feature is not implemented")   # :108-110
    if r == -1:
        raise InvalidDataException("corrupted block")   # InvalidOperationException in the block decoders
    if r < 0:
        raise InvalidDataException("Invalid LZ4 frame")


def read_frames(frames, device: int = 0) -> list:
    """Decodes many frames, linked or independent, in one k4lz4_frame_decode_batch call; returns their contents in
    order.  Raises for the first bad frame: InvalidDataException (bad magic number, header, block or content
    checksum, truncation, a corrupted block), NotImplementedError for a dictionary id."""
    contents, out = LZ4Frame.DecodeMany(frames, None, device)
    for r in out:
        _raise_for(int(r))
    return contents


def read_frame(frame, device: int = 0) -> bytes:
    """Decodes one frame (LZ4FrameReader.blocking.cs:57-144); raises like read_frames."""
    return read_frames([frame], device)[0]
