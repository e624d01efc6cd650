"""Chain groups (k4lz4_chain_group_*): many chained streams whose context stays on one GPU between calls.

``LZ4FastChainEncoder.EncodeMany`` and ``LZ4ChainDecoder.DecodeMany`` keep each stream's history and state on the
host, so every call sends all of it up and brings the states back.  A group keeps them on the device: a call
sends only the blocks and brings back only the bytes produced (host entry points), or moves nothing across PCIe
at all (``*_device`` entry points, which take ``data_ptr()``s and a CUDA stream and only enqueue work).

Each call advances any subset of the group's streams by one block each.  A block's bytes and result equal what
the stream's ``LZ4FastChainEncoder`` / ``LZ4ChainDecoder`` gives for it, whatever that object's blockSize and
extraBlocks.  Like those objects a group is not thread-safe; ``close()`` (or ``with``) frees its device memory.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from . import _native as N
from .batch import _i32, _pack, _slices, _slots, encoder_fn
from .codec import LZ4Codec


class _Group:
    """What every resident group's mirror shares: the handle, with-blocks, and the kind's destroy and reset."""
    _destroy = _reset = ""            # names of the kind's k4lz4_*_destroy / k4lz4_*_reset

    @property
    def handle(self) -> int:
        if not self._h:
            raise RuntimeError("ObjectDisposedException")
        return self._h

    def _free(self) -> None:
        if getattr(self, "_h", None):
            getattr(N.lib(), self._destroy)(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self._free()

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass

    def _streams(self, streams, n: int) -> np.ndarray:
        return _i32(np.arange(n) if streams is None else streams)

    def reset(self, streams: Sequence[int] | None = None) -> None:
        """Streams (default: all) become new; what they held is dropped (a writer's open frames emit nothing)."""
        s = self._streams(streams, self.n_streams)
        N.check(getattr(N.lib(), self._reset)(self.handle, s.ctypes.data, len(s), N.MEM_HOST, None))

    def reset_device(self, streams_ptr: int, n: int, stream: int = 0) -> None:
        N.check(getattr(N.lib(), self._reset)(self.handle, streams_ptr, int(n), N.MEM_DEVICE, stream or None))


class _ChainGroup(_Group):
    _kind = -1
    _destroy, _reset = "k4lz4_chain_group_destroy", "k4lz4_chain_group_reset"

    def __init__(self, n_streams: int, block_size: int, device: int = 0):
        h = C.c_void_p()
        N.check(N.lib().k4lz4_chain_group_create(self._kind, int(n_streams), int(block_size), int(device),
                                                 C.byref(h)))
        self._h = h.value
        self.n_streams, self.block_size = int(n_streams), int(block_size)

    close = _Group._free

    def history(self, i: int) -> bytes:
        """The stream's history: its last <= 65 536 bytes (waits for the device)."""
        out = np.zeros(65536, dtype=np.uint8)
        k = N.lib().k4lz4_chain_group_history(self.handle, int(i), out.ctypes.data, out.size)
        N.check(min(k, 0))
        return out[:k].tobytes()


class ChainEncoderGroup(_ChainGroup):
    """S LZ4FastChainEncoder streams at L00_FAST whose input rings and LZ4_stream_t records live on the GPU.  Each
    call encodes with the engine LZ4Codec.Enforce32 names at that call."""
    _kind = N.CHAIN_ENCODER

    def encode(self, blocks: Sequence, streams: Sequence[int] | None = None, caps: Sequence[int] | None = None,
               level: int = 0):
        """blocks[i] is the next block of stream streams[i] (default: stream i), caps[i] its capacity (default
        MaximumOutputSize).  -> (list of encoded bytes, int32 results as k4lz4_encode_chain_batch gives them)."""
        src, so, sl = _pack(blocks)
        s = self._streams(streams, len(sl))
        if caps is None:
            caps = [N.lib().k4lz4_max_output_size(int(x)) for x in sl]
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(encoder_fn("k4lz4_chain_group_encode", LZ4Codec.Enforce32)(self.handle, s.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                 sl.ctypes.data, dst.ctypes.data, do.ctypes.data, dc.ctypes.data,
                                                 out.ctypes.data, len(sl), int(level), N.MEM_HOST, None))
        return _slices(dst, do, out), out

    def encode_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int, dst_ptr: int,
                      dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int, n: int, level: int = 0,
                      stream: int = 0) -> None:
        """Device-pointer form of encode: only enqueues work on `stream`."""
        N.check(encoder_fn("k4lz4_chain_group_encode", LZ4Codec.Enforce32)(self.handle, streams_ptr, src_ptr, src_off_ptr, src_len_ptr, dst_ptr,
                                                 dst_off_ptr, dst_cap_ptr, out_len_ptr, int(n), int(level),
                                                 N.MEM_DEVICE, stream or None))

    def state(self, i: int) -> np.ndarray:
        """Stream i's K4LZ4_CHAIN_STATE_BYTES record (waits for the device)."""
        out = np.zeros(N.CHAIN_STATE_BYTES, dtype=np.uint8)
        N.check(N.lib().k4lz4_chain_group_state(self.handle, int(i), out.ctypes.data))
        return out


class ChainDecoderGroup(_ChainGroup):
    """S LZ4ChainDecoder streams whose output rings live on the GPU."""
    _kind = N.CHAIN_DECODER

    def decode(self, blocks: Sequence, streams: Sequence[int] | None = None, caps: Sequence[int] | None = None):
        """blocks[i] (compressed) is the next block of stream streams[i] (default: stream i), decoded into at most
        caps[i] <= block_size bytes (default block_size).  -> (list of decoded bytes, int32 results as
        k4lz4_decode_chain_batch gives them)."""
        src, so, sl = _pack(blocks)
        s = self._streams(streams, len(sl))
        dst, do, dc = _slots([self.block_size] * len(sl) if caps is None else caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(N.lib().k4lz4_chain_group_decode(self.handle, s.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                 sl.ctypes.data, dst.ctypes.data, do.ctypes.data, dc.ctypes.data,
                                                 out.ctypes.data, len(sl), N.MEM_HOST, None))
        return _slices(dst, do, out), out

    def decode_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int, dst_ptr: int,
                      dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int, n: int, stream: int = 0) -> None:
        """Device-pointer form of decode: only enqueues work on `stream`."""
        N.check(N.lib().k4lz4_chain_group_decode(self.handle, streams_ptr, src_ptr, src_off_ptr, src_len_ptr, dst_ptr,
                                                 dst_off_ptr, dst_cap_ptr, out_len_ptr, int(n), N.MEM_DEVICE,
                                                 stream or None))

    def inject(self, blocks: Sequence, streams: Sequence[int] | None = None) -> None:
        """LZ4ChainDecoder.Inject: blocks[i] (raw bytes) become the end of stream streams[i]'s history."""
        src, so, sl = _pack(blocks)
        s = self._streams(streams, len(sl))
        N.check(N.lib().k4lz4_chain_group_inject(self.handle, s.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                 sl.ctypes.data, len(sl), N.MEM_HOST, None))

    def inject_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int, n: int,
                      stream: int = 0) -> None:
        N.check(N.lib().k4lz4_chain_group_inject(self.handle, streams_ptr, src_ptr, src_off_ptr, src_len_ptr, int(n),
                                                 N.MEM_DEVICE, stream or None))


class FrameWriterGroup(_Group):
    """S LZ4EncoderStream / LZ4FrameWriter streams at L00_FAST (k4lz4_frame_writer_group_*) whose partial blocks,
    chain states and content checksums live on the GPU.  Each call writes one chunk of any size to (or closes) any
    subset of the streams and returns the frame bytes it produced; for every stream the concatenation of what its
    writes and its close returned is the LZ4 frame of everything written to it.  ``close(streams)`` ends frames;
    ``free()`` (or ``with``) frees the group's device memory, abandoning frames not closed.  Each write and close
    encodes with the engine LZ4Codec.Enforce32 names at that call."""
    _destroy, _reset = "k4lz4_frame_writer_group_destroy", "k4lz4_frame_writer_group_reset"

    def __init__(self, n_streams: int, block_size: int = 65536, chaining: bool = True, block_checksum: bool = False,
                 content_checksum: bool = False, level: int = 0, device: int = 0):
        self.flags = (0 if chaining else N.FRAME_INDEPENDENT) | (N.FRAME_BLOCK_CHECKSUM if block_checksum else 0) | \
            (N.FRAME_CONTENT_CHECKSUM if content_checksum else 0)
        h = C.c_void_p()
        rc = N.lib().k4lz4_frame_writer_group_create(int(n_streams), int(block_size), self.flags, int(level),
                                                     int(device), C.byref(h))
        if rc == N.R_DELEGATE:
            raise NotImplementedError("LZ4HighChainEncoder (chained HC levels) stays with the managed engine")
        N.check(rc)
        self._h = h.value
        self.n_streams, self.block_size = int(n_streams), int(block_size)

    free = _Group._free

    def bound(self, length: int) -> int:
        """The most one write of `length` bytes appends."""
        return int(N.lib().k4lz4_frame_writer_bound(self.handle, int(length)))

    def close_bound(self) -> int:
        """The most one close appends."""
        return int(N.lib().k4lz4_frame_writer_close_bound(self.handle))

    def write(self, chunks: Sequence, streams: Sequence[int] | None = None, caps: Sequence[int] | None = None):
        """chunks[i] is written to stream streams[i] (default: stream i), into caps[i] bytes (default: the bound).
        -> (list of frame bytes each write produced, int32 results: bytes appended, or -1 where caps[i] is below
        the bound)."""
        src, so, sl = _pack(chunks)
        s = self._streams(streams, len(sl))
        dst, do, dc = _slots([self.bound(int(x)) for x in sl] if caps is None else caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        N.check(encoder_fn("k4lz4_frame_writer_group_write", LZ4Codec.Enforce32)(self.handle, s.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                       sl.ctypes.data, dst.ctypes.data, do.ctypes.data,
                                                       dc.ctypes.data, out.ctypes.data, len(sl), N.MEM_HOST, None))
        return _slices(dst, do, out), out

    def close(self, streams: Sequence[int] | None = None, caps: Sequence[int] | None = None):
        """Closes streams (default: all): their pending block, end mark and content checksum.  -> (list of frame
        bytes, int32 results; 0 and no bytes for a stream that was not written since it was new)."""
        s = self._streams(streams, self.n_streams)
        dst, do, dc = _slots([self.close_bound()] * len(s) if caps is None else caps)
        out = np.full(len(s), -1, dtype=np.int32)
        N.check(encoder_fn("k4lz4_frame_writer_group_close", LZ4Codec.Enforce32)(self.handle, s.ctypes.data, dst.ctypes.data, do.ctypes.data,
                                                       dc.ctypes.data, out.ctypes.data, len(s), N.MEM_HOST, None))
        return _slices(dst, do, out), out

    def write_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int, dst_ptr: int,
                     dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int, n: int, stream: int = 0) -> None:
        """Device-pointer form of write: enqueues work on `stream` (and waits once for the number of steps)."""
        N.check(encoder_fn("k4lz4_frame_writer_group_write", LZ4Codec.Enforce32)(self.handle, streams_ptr, src_ptr, src_off_ptr, src_len_ptr,
                                                       dst_ptr, dst_off_ptr, dst_cap_ptr, out_len_ptr, int(n),
                                                       N.MEM_DEVICE, stream or None))

    def close_device(self, streams_ptr: int, dst_ptr: int, dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int,
                     n: int, stream: int = 0) -> None:
        """Device-pointer form of close: only enqueues work on `stream`."""
        N.check(encoder_fn("k4lz4_frame_writer_group_close", LZ4Codec.Enforce32)(self.handle, streams_ptr, dst_ptr, dst_off_ptr, dst_cap_ptr,
                                                       out_len_ptr, int(n), N.MEM_DEVICE, stream or None))


class FrameReaderGroup(_Group):
    """S LZ4DecoderStream / LZ4FrameReader streams (k4lz4_frame_reader_group_*) whose partial headers and blocks,
    histories and content checksums live on the GPU.  Each call feeds one chunk of compressed bytes, cut anywhere,
    to any subset of the streams and returns the content it decoded; a call consumes bytes of at most one frame and
    decodes at most floor(cap / blockCap) blocks (blockCap: the frame's BD maximum, + 8 for independent blocks), so
    a caller re-feeds what was not consumed.  ``end(streams)`` reports whether each input stopped between frames;
    ``free()`` (or ``with``) frees the group's device memory."""
    _destroy, _reset = "k4lz4_frame_reader_group_destroy", "k4lz4_frame_reader_group_reset"

    def __init__(self, n_streams: int, max_block_size: int = 65536, device: int = 0):
        h = C.c_void_p()
        N.check(N.lib().k4lz4_frame_reader_group_create(int(n_streams), int(max_block_size), int(device), C.byref(h)))
        self._h = h.value
        self.n_streams, self.max_block_size = int(n_streams), int(max_block_size)

    free = _Group._free

    def read(self, chunks: Sequence, caps: Sequence[int], streams: Sequence[int] | None = None):
        """chunks[i] is fed to stream streams[i] (default: stream i) with caps[i] bytes of room.  -> (list of
        content each entry decoded, int32 results: bytes appended or the verdict, int32 bytes consumed, int32 1
        where the entry ended a frame)."""
        return self._read(chunks, caps, streams, None)

    def read_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int, src_used_ptr: int,
                    dst_ptr: int, dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int, frame_ended_ptr: int, n: int,
                    stream: int = 0) -> None:
        """Device-pointer form of read: enqueues work on `stream` (and waits once for the row and step counts)."""
        self._call(None, streams_ptr, src_ptr, src_off_ptr, src_len_ptr, src_used_ptr, dst_ptr, dst_off_ptr,
                   dst_cap_ptr, out_len_ptr, frame_ended_ptr, int(n), mem=N.MEM_DEVICE, stream=stream or None)

    def read_bytes(self, chunks: Sequence, caps: Sequence[int], streams: Sequence[int] | None = None,
                   interactive: bool = False):
        """LZ4DecoderStream.Read with a buffer of any size: each entry first drains what is left of its stream's
        current block, then decodes blocks while room is left; what does not fit stays on the device for the next
        call (k4lz4_frame_reader_group_read_bytes).  interactive: stop after the first drain that appended
        anything.  -> as read."""
        return self._read(chunks, caps, streams, N.READ_INTERACTIVE if interactive else 0)

    def read_bytes_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int,
                          src_used_ptr: int, dst_ptr: int, dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int,
                          frame_ended_ptr: int, n: int, interactive: bool = False, stream: int = 0) -> None:
        """Device-pointer form of read_bytes: enqueues work on `stream` (and waits once for the candidate rows)."""
        self._call(N.READ_INTERACTIVE if interactive else 0, streams_ptr, src_ptr, src_off_ptr, src_len_ptr,
                   src_used_ptr, dst_ptr, dst_off_ptr, dst_cap_ptr, out_len_ptr, frame_ended_ptr, int(n),
                   mem=N.MEM_DEVICE, stream=stream or None)

    def _call(self, flags, *args, mem, stream):
        """k4lz4_frame_reader_group_read (flags None) or _read_bytes with these flags."""
        if flags is None:
            N.check(N.lib().k4lz4_frame_reader_group_read(self.handle, *args, mem, stream))
        else:
            N.check(N.lib().k4lz4_frame_reader_group_read_bytes(self.handle, *args, flags, mem, stream))

    def _read(self, chunks, caps, streams, flags):
        src, so, sl = _pack(chunks)
        s = self._streams(streams, len(sl))
        dst, do, dc = _slots(caps)
        out = np.full(len(sl), -1, dtype=np.int32)
        used = np.zeros(len(sl), dtype=np.int32)
        ended = np.zeros(len(sl), dtype=np.int32)
        self._call(flags, s.ctypes.data, src.ctypes.data, so.ctypes.data, sl.ctypes.data, used.ctypes.data,
                   dst.ctypes.data, do.ctypes.data, dc.ctypes.data, out.ctypes.data, ended.ctypes.data, len(sl),
                   mem=N.MEM_HOST, stream=None)
        return _slices(dst, do, out), out, used, ended

    def end(self, streams: Sequence[int] | None = None) -> np.ndarray:
        """The input of streams (default: all) has ended.  -> int32 statuses: 0 between frames, R_CORRUPT inside a
        frame, a failed stream's verdict.  The streams become new."""
        s = self._streams(streams, self.n_streams)
        out = np.zeros(len(s), dtype=np.int32)
        N.check(N.lib().k4lz4_frame_reader_group_end(self.handle, s.ctypes.data, out.ctypes.data, len(s), N.MEM_HOST,
                                                     None))
        return out

    def end_device(self, streams_ptr: int, status_ptr: int, n: int, stream: int = 0) -> None:
        N.check(N.lib().k4lz4_frame_reader_group_end(self.handle, streams_ptr, status_ptr, int(n), N.MEM_DEVICE,
                                                     stream or None))

    def read_all(self, chunks: Sequence, cap: int, streams: Sequence[int] | None = None):
        """Feeds chunks[i] to stream streams[i] (default: stream i) whole, re-feeding what each call leaves, across
        frame ends, until every chunk is consumed or its stream fails, then ends the streams (they become new).
        -> (list of content, int32 results: total bytes, or the verdict -- R_CORRUPT where a chunk stops inside
        a frame).  Each call is fed at most what it can consume: its blocks at `cap`, a header and an end mark."""
        s = [int(x) for x in self._streams(streams, len(chunks))]
        data = [memoryview(bytes(c)) for c in chunks]
        # a block's stored bytes never exceed max_block_size + 8 + (max_block_size + 8) // 255 + 16 (longer
        # compressed blocks are skipped in pieces), so a window this long holds everything one call consumes
        m = self.max_block_size + 8
        window = (max(int(cap), 0) // 65536 + 1) * (m + m // 255 + 16) + 64
        at = [0] * len(data)
        got = [[] for _ in data]
        res = np.zeros(len(data), dtype=np.int32)
        todo = [i for i in range(len(data)) if len(data[i])]
        while todo:
            outs, r, used, _ = self.read([data[i][at[i]:at[i] + window] for i in todo], [cap] * len(todo),
                                         [s[i] for i in todo])
            nxt = []
            for k, i in enumerate(todo):
                if r[k] < 0:
                    res[i] = r[k]
                    continue
                got[i].append(outs[k])
                res[i] += r[k]
                at[i] += int(used[k])
                if at[i] < len(data[i]):
                    if used[k] == 0 and r[k] == 0:
                        raise ValueError(f"stream {s[i]}: cap {cap} leaves no room for a block")
                    nxt.append(i)
            todo = nxt
        st = self.end(s)
        res = np.where(res < 0, res, np.where(st < 0, st, res)).astype(np.int32)
        return [b"".join(g) for g in got], res
