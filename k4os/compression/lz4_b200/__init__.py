"""k4os.compression.lz4_b200 -- H100-native (sm_90a CUDA) drop-in for one hot path of
K4os.Compression.LZ4: ``LZ4Codec.Encode`` at ``L00_FAST``, ``LZ4Codec.Decode`` and
``LZ4Pickler.Pickle/Unpickle`` over batches of independent blocks (plus ``Decode`` with a
dictionary, ``PartialDecode`` and the independent-block ``LZ4BlockEncoder`` / ``LZ4BlockDecoder``
pair with a batched top-up, and ``LZ4FastChainEncoder`` / ``LZ4ChainDecoder`` for chained blocks, batched
across streams, with ``ChainEncoderGroup`` / ``ChainDecoderGroup`` keeping such streams resident on the GPU, and whole ``LZ4Frame`` buffers, batched across frames, with ``FrameWriterGroup`` / ``FrameReaderGroup`` writing and reading many frames incrementally).

The product is ``libk4lz4.so`` (C ABI in ``include/k4lz4.h``, kernels in ``csrc/``); this
package is the host-side mirror of the reference's public interface for that path plus the
batched entry points.  Importing it never imports ``oracle/``.
"""
from . import _native
from .codec import LZ4Codec, LZ4Level, DelegateToManagedEngine
from .pickler import LZ4Pickler, InvalidDataException
from . import batch
from .encoders import (LZ4BlockEncoder, LZ4BlockDecoder, LZ4ChainDecoder, LZ4Decoder, LZ4Encoder,
                       LZ4FastChainEncoder)
from .groups import ChainDecoderGroup, ChainEncoderGroup, FrameReaderGroup, FrameWriterGroup
from .frame import LZ4Frame

__all__ = ["LZ4Codec", "LZ4Level", "LZ4Pickler", "InvalidDataException",
           "DelegateToManagedEngine", "batch", "_native", "LZ4BlockEncoder", "LZ4BlockDecoder",
           "LZ4ChainDecoder", "LZ4Decoder", "LZ4Encoder", "LZ4FastChainEncoder", "ChainEncoderGroup",
           "ChainDecoderGroup", "LZ4Frame", "FrameWriterGroup", "FrameReaderGroup"]
