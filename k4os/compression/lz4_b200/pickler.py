"""Host-side mirror of ``LZ4Pickler`` (byte[] variant) for the accelerated path.

Reference: ``/root/reference/src/K4os.Compression.LZ4/LZ4Pickler.pickle.cs:51-106`` and
``LZ4Pickler.unpickle.cs:39-50,83-129``.  ``InvalidDataException`` is mirrored by
:class:`InvalidDataException`.  Single-message calls are batches of one through the C ABI.
"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .batch import pickle_batch_host, pickle_writer_batch_host, unpickle_batch_host, unpickled_size_batch_host
from .codec import LZ4Codec, LZ4Level, DelegateToManagedEngine, _ro, _rw


class InvalidDataException(ValueError):
    """Stands for System.IO.InvalidDataException ("Pickle is corrupted: ...")."""


class LZ4Pickler:
    @staticmethod
    def Pickle(source, level: LZ4Level = LZ4Level.L00_FAST) -> bytes:
        """LZ4Pickler.pickle.cs:51-74."""
        src = _ro(source)
        if src.shape[0] == 0:
            return b""
        out, lens = pickle_batch_host([src], level=int(level), x32=LZ4Codec.Enforce32)
        if lens[0] == N.R_DELEGATE:
            raise DelegateToManagedEngine(f"level {int(level)} is not on the accelerated path")
        return out[0]

    @staticmethod
    def PickleTo(source, writer, level: LZ4Level = LZ4Level.L00_FAST) -> None:
        """Pickle<TBufferWriter>(source, writer, level) -- LZ4Pickler.pickle.cs:113-148.  `writer` is
        anything with write(bytes) (or a bytearray, which is extended): the IBufferWriter mirror.
        NOTE the bytes differ from Pickle(): pessimistic header width, capacity-n encode."""
        if writer is None:
            raise ValueError("writer: cannot be null")                    # ArgumentNullException, :118-119
        src = _ro(source)
        if src.shape[0] == 0:
            return
        out, lens = pickle_writer_batch_host([src], level=int(level), x32=LZ4Codec.Enforce32)
        if lens[0] == N.R_DELEGATE:
            raise DelegateToManagedEngine(f"level {int(level)} is not on the accelerated path")
        if isinstance(writer, bytearray):
            writer.extend(out[0])
        else:
            writer.write(out[0])

    @staticmethod
    def UnpickledSize(source) -> int:
        """LZ4Pickler.unpickle.cs:83-92."""
        src = _ro(source)
        if src.shape[0] == 0:
            raise IndexError("source is empty")       # source[0] on an empty span throws
        size = int(unpickled_size_batch_host([src])[0])
        if size == N.R_CORRUPT:
            raise InvalidDataException("Pickle is corrupted")
        return size

    @staticmethod
    def Unpickle(source, output=None):
        """Unpickle(source) -> bytes                        -- LZ4Pickler.unpickle.cs:39-50
        Unpickle(source, output) -> None (fills output)    -- LZ4Pickler.unpickle.cs:99-107"""
        src = _ro(source)
        if src.shape[0] == 0:
            return b"" if output is None else None
        if output is None:
            size = LZ4Pickler.UnpickledSize(src)
            if size == 0:
                return b""
            out = np.zeros(size, dtype=np.uint8)
        else:
            out = _rw(output)
        r = int(unpickle_batch_host([src], [out])[0])
        if r == N.R_CORRUPT:
            raise InvalidDataException("Pickle is corrupted")
        return out.tobytes() if output is None else None
