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
from .batch import _i32, _pack, _slices, _slots


class _ChainGroup:
    _kind = -1

    def __init__(self, n_streams: int, block_size: int, device: int = 0):
        h = C.c_void_p()
        N.check(N.lib().k4lz4_chain_group_create(self._kind, int(n_streams), int(block_size), int(device),
                                                 C.byref(h)))
        self._h = h.value
        self.n_streams, self.block_size = int(n_streams), int(block_size)

    @property
    def handle(self) -> int:
        if not self._h:
            raise RuntimeError("ObjectDisposedException")
        return self._h

    def close(self) -> None:
        if getattr(self, "_h", None):
            N.lib().k4lz4_chain_group_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _streams(self, streams, n: int) -> np.ndarray:
        return _i32(np.arange(n) if streams is None else streams)

    def reset(self, streams: Sequence[int] | None = None) -> None:
        """Streams (default: all) become new."""
        s = self._streams(streams, self.n_streams)
        N.check(N.lib().k4lz4_chain_group_reset(self.handle, s.ctypes.data, len(s), N.MEM_HOST, None))

    def reset_device(self, streams_ptr: int, n: int, stream: int = 0) -> None:
        N.check(N.lib().k4lz4_chain_group_reset(self.handle, streams_ptr, int(n), N.MEM_DEVICE, stream or None))

    def history(self, i: int) -> bytes:
        """The stream's history: its last <= 65 536 bytes (waits for the device)."""
        out = np.zeros(65536, dtype=np.uint8)
        k = N.lib().k4lz4_chain_group_history(self.handle, int(i), out.ctypes.data, out.size)
        N.check(min(k, 0))
        return out[:k].tobytes()


class ChainEncoderGroup(_ChainGroup):
    """S LZ4FastChainEncoder streams at L00_FAST whose input rings and LZ4_stream_t records live on the GPU."""
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
        N.check(N.lib().k4lz4_chain_group_encode(self.handle, s.ctypes.data, src.ctypes.data, so.ctypes.data,
                                                 sl.ctypes.data, dst.ctypes.data, do.ctypes.data, dc.ctypes.data,
                                                 out.ctypes.data, len(sl), int(level), N.MEM_HOST, None))
        return _slices(dst, do, out), out

    def encode_device(self, streams_ptr: int, src_ptr: int, src_off_ptr: int, src_len_ptr: int, dst_ptr: int,
                      dst_off_ptr: int, dst_cap_ptr: int, out_len_ptr: int, n: int, level: int = 0,
                      stream: int = 0) -> None:
        """Device-pointer form of encode: only enqueues work on `stream`."""
        N.check(N.lib().k4lz4_chain_group_encode(self.handle, streams_ptr, src_ptr, src_off_ptr, src_len_ptr, dst_ptr,
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
