"""Host-side mirror of the reference's public block API for the accelerated path.

Same names, argument meaning and error behaviour as
``/root/reference/src/K4os.Compression.LZ4/LZ4Codec.cs`` (Encode :40-96, Decode :104-237,
MaximumOutputSize :30-31) and ``LZ4Level.cs:6-39``.  Every call goes through the C ABI of
``libk4lz4.so`` (``include/k4lz4.h``) and therefore through the CUDA kernels; nothing is
computed in Python and there is no CPU fallback.

Buffers: ``source`` is any object exposing the buffer protocol (bytes, bytearray, memoryview,
numpy uint8 array); ``target`` must be writable (bytearray, memoryview, numpy).  They play the
role of ``ReadOnlySpan<byte>`` / ``Span<byte>``.
"""
from __future__ import annotations

import ctypes as C
from enum import IntEnum

import numpy as np

from . import _native as N


class LZ4Level(IntEnum):
    """LZ4Level.cs:6-39.  Only L00_FAST runs natively; HC/OPT levels keep delegating."""
    L00_FAST = 0
    L03_HC = 3
    L04_HC = 4
    L05_HC = 5
    L06_HC = 6
    L07_HC = 7
    L08_HC = 8
    L09_HC = 9
    L10_OPT = 10
    L11_OPT = 11
    L12_MAX = 12


class DelegateToManagedEngine(NotImplementedError):
    """Raised for levels >= L03_HC: outside the accelerated path (LZ4Codec.cs:48-50 routes
    them to LZ4_compress_HC, which stays with the reference)."""


def _ro(buf) -> np.ndarray:
    if isinstance(buf, np.ndarray):
        if buf.dtype != np.uint8 or not buf.flags.c_contiguous:
            raise TypeError("numpy buffers must be contiguous uint8")
        return buf
    return np.frombuffer(buf, dtype=np.uint8)


def _rw(buf) -> np.ndarray:
    a = _ro(buf)
    if not a.flags.writeable:
        raise TypeError("target buffer must be writable")
    return a


def _validate(buffer, offset: int, length: int, name: str) -> None:
    """Internal/Extensions.cs:37-52 (Validate)."""
    if buffer is None:
        raise ValueError(f"{name}: cannot be null")           # ArgumentNullException
    if not (offset >= 0 and length >= 0 and offset + length <= len(buffer)):
        raise ValueError(f"invalid offset/length combination: {offset}/{length}")   # ArgumentException


class LZ4Codec:
    """Static class exposing LZ4 block compression methods (LZ4Codec.cs:10-266)."""

    Version = 192                      # LZ4Codec.cs:13

    # LZ4Codec.Enforce32 (LZ4Codec.cs:21-25, Engine/LL.tools.cs:29-36): every L00_FAST encode call made while it is
    # set uses the 32-bit engine LL32 (hash4 for the u32 table), so its bytes differ from LL64's for inputs of
    # >= 65 547 bytes and for chained blocks of any size.  Read at each call, as the reference reads it
    # (Engine/LLxx.cs:65-91): Encode, LZ4Pickler.Pickle / PickleTo, LZ4BlockEncoder, LZ4FastChainEncoder,
    # LZ4Frame / write_frames, ChainEncoderGroup.encode and FrameWriterGroup.write / close.  Decoding is unaffected.
    Enforce32 = False

    @staticmethod
    def MaximumOutputSize(length: int) -> int:
        """LZ4Codec.cs:30-31."""
        return int(N.lib().k4lz4_max_output_size(int(length)))

    # -- Encode ---------------------------------------------------------------------------
    @staticmethod
    def Encode(source, *args, **kw) -> int:
        """Encode(source, target, level=L00_FAST)                         -- LZ4Codec.cs:59-71
        Encode(source, sourceOffset, sourceLength, target, targetOffset, targetLength, level)
                                                                          -- LZ4Codec.cs:82-96
        Returns bytes written, 0 for empty input, negative if the target is too small."""
        level = kw.pop("level", None)
        if len(args) >= 5 and isinstance(args[0], int):
            s_off, s_len, target, t_off, t_len = args[:5]
            if len(args) > 5:
                level = args[5]
            _validate(source, s_off, s_len, "source")
            _validate(target, t_off, t_len, "target")
            src = _ro(source)[s_off:s_off + s_len]
            dst = _rw(target)[t_off:t_off + t_len]
        else:
            target = args[0]
            if len(args) > 1:
                level = args[1]
            src, dst = _ro(source), _rw(target)
        level = LZ4Level.L00_FAST if level is None else level
        n = int(src.shape[0])
        if n <= 0:
            return 0                                                      # LZ4Codec.cs:45-46,64-65
        enc = N.lib().k4lz4_encode_x32 if LZ4Codec.Enforce32 else N.lib().k4lz4_encode
        r = int(enc(src.ctypes.data, n, dst.ctypes.data, int(dst.shape[0]), int(level)))
        if r == N.R_DELEGATE:
            raise DelegateToManagedEngine(f"level {int(level)} is not on the accelerated path")
        if r <= N.E_NODEVICE:
            N.check(r)
        return r

    # -- Decode ---------------------------------------------------------------------------
    @staticmethod
    def Decode(source, *args) -> int:
        """Decode(source, target[, dictionary])                            -- LZ4Codec.cs:179-191, :200-214
        Decode(source, sourceOffset, sourceLength, target, targetOffset, targetLength)
                                                                          -- LZ4Codec.cs:225-237
        Returns bytes written, 0 for empty input, negative on malformed input / small target."""
        dic = None
        if len(args) >= 5:
            s_off, s_len, target, t_off, t_len = args[:5]
            _validate(source, s_off, s_len, "source")
            _validate(target, t_off, t_len, "target")
            src = _ro(source)[s_off:s_off + s_len]
            dst = _rw(target)[t_off:t_off + t_len]
            if len(args) >= 8:                                            # ..., dictionary, dictOffset, dictLength
                dictionary, d_off, d_len = args[5:8]
                if dictionary is not None or d_len:
                    _validate(dictionary, d_off, d_len, "dictionary")
                    dic = _ro(dictionary)[d_off:d_off + d_len]
        else:
            src, dst = _ro(source), _rw(args[0])
            if len(args) >= 2 and args[1] is not None:                    # Decode(source, target, dictionary)
                dic = _ro(args[1])
        n = int(src.shape[0])
        if n <= 0:
            return 0
        if dic is not None and int(dic.shape[0]) > 0:                     # LZ4Codec.cs:144-157, :200-214, :246-265
            r = int(N.lib().k4lz4_decode_dict(src.ctypes.data, n, dst.ctypes.data, int(dst.shape[0]),
                                              dic.ctypes.data, int(dic.shape[0])))
        else:
            r = int(N.lib().k4lz4_decode(src.ctypes.data, n, dst.ctypes.data, int(dst.shape[0])))
        if r <= N.E_NODEVICE:
            N.check(r)
        return r

    @staticmethod
    def PartialDecode(source, *args) -> int:
        """PartialDecode(source, target)                                   -- LZ4Codec.cs:163-173
        PartialDecode(source, sourceOffset, sourceLength, target, targetOffset, targetLength)
        Decoding stops at the end of the target; returns bytes written, negative on failure."""
        if len(args) >= 5:
            s_off, s_len, target, t_off, t_len = args[:5]
            _validate(source, s_off, s_len, "source")
            _validate(target, t_off, t_len, "target")
            src = _ro(source)[s_off:s_off + s_len]
            dst = _rw(target)[t_off:t_off + t_len]
        else:
            src, dst = _ro(source), _rw(args[0])
        n = int(src.shape[0])
        if n <= 0:
            return 0
        r = int(N.lib().k4lz4_partial_decode(src.ctypes.data, n, dst.ctypes.data, int(dst.shape[0])))
        if r <= N.E_NODEVICE:
            N.check(r)
        return r
