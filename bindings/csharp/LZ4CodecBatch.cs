// LZ4CodecBatch.cs -- the batched public surface next to LZ4Codec (same return conventions per block:
// lengths[i] is exactly what LZ4Codec.Encode / LZ4Codec.Decode would return for block i).
// Not compiled in this repository (no .NET SDK in the build image); see INTEGRATION.md.
using System;
using K4os.Compression.LZ4.Engine.Native;

namespace K4os.Compression.LZ4
{
    public static unsafe class LZ4CodecBatch
    {
        public static bool IsAvailable => K4Lz4Native.k4lz4_device_count() > 0;

        public static void Encode(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            Span<int> lengths, LZ4Level level = LZ4Level.L00_FAST)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (int* ol = lengths)
                Check(K4Lz4Native.k4lz4_encode_batch(s, so, sl, d, dof, dc, ol, lengths.Length,
                    (int)level, K4Lz4Native.MEM_HOST, null, K4Lz4Native.ALL_DEVICES));
        }

        public static void Decode(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            Span<int> lengths)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (int* ol = lengths)
                Check(K4Lz4Native.k4lz4_decode_batch(s, so, sl, d, dof, dc, ol, lengths.Length,
                    K4Lz4Native.MEM_HOST, null, K4Lz4Native.ALL_DEVICES));
        }

        // Block i against dictionaryBase[dictionaryOffsets[i] .. +dictionaryLengths[i]): what
        // LZ4Codec.Decode(source, target, dictionary) reads back.  Blocks with equal (offset, length) share one
        // loaded table and one staged copy of the dictionary.  lengths[i]: bytes written, 0 for an empty block,
        // -1 where it does not fit targetCapacities[i].
        public static void EncodeWithDictionary(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            ReadOnlySpan<byte> dictionaryBase, ReadOnlySpan<long> dictionaryOffsets,
            ReadOnlySpan<int> dictionaryLengths, Span<int> lengths)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (byte* x = dictionaryBase) fixed (long* xo = dictionaryOffsets) fixed (int* xl = dictionaryLengths)
            fixed (int* ol = lengths)
                Check(K4Lz4Native.k4lz4_encode_dict_batch(s, so, sl, d, dof, dc, x, xo, xl, ol, lengths.Length,
                    K4Lz4Native.MEM_HOST, null, K4Lz4Native.ALL_DEVICES));
        }

        // Fixed-size destinations (k4lz4_encode_dest_size_batch; the reference has no such call): block i encodes the
        // longest prefix of its source whose block fits targetCapacities[i], as upstream's LZ4_compress_destSize.
        // lengths[i]: bytes written; consumed[i]: the source bytes the block holds (both 0 where nothing is written).
        public static void EncodeDestSize(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            Span<int> lengths, Span<int> consumed)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (int* ol = lengths) fixed (int* su = consumed)
                Check(K4Lz4Native.k4lz4_encode_dest_size_batch(s, so, sl, d, dof, dc, ol, su, lengths.Length,
                    K4Lz4Native.MEM_HOST, null, K4Lz4Native.ALL_DEVICES));
        }

        // LZ4 frames as upstream's LZ4F_compressFrame writes them (k4lz4_lz4f_compress_batch; the reference has no
        // such call): frame i holds source i; each frame's block size shrinks to fit it, a one-block frame is
        // independent, and FRAME_CONTENT_SIZE writes the content size.  blockSize: 64 KiB, 256 KiB, 1 MiB or 4 MiB;
        // flags: K4Lz4Native.FRAME_*; size targets with k4lz4_lz4f_compress_bound.  lengths[i]: the frame's length,
        // -1 where it does not fit targetCapacities[i], K4Lz4Native.R_DELEGATE for HC levels.
        public static void CompressFramesUpstream(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            Span<int> lengths, int blockSize = 65536, int flags = 0, LZ4Level level = LZ4Level.L00_FAST)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (int* ol = lengths)
                Check(K4Lz4Native.k4lz4_lz4f_compress_batch(s, so, sl, d, dof, dc, ol, lengths.Length, blockSize,
                    flags, (int)level, K4Lz4Native.MEM_HOST, null, 0));
        }

        // Whole .lz4 inputs as upstream's `lz4 -d [-D dict]` reads them (k4lz4_lz4f_decompress_batch): concatenated
        // frames, skippable frames, legacy members.  lengths[i]: the content length, -1 on an error, R_DST_SMALL;
        // errors[i]: (cliError << 8) | LZ4F code, 0 on success; ends[i]: where reading stopped.  An empty
        // dictionaryLengths span: no dictionaries.  Size targets with k4lz4_lz4f_decompressed_size_batch.
        public static void DecompressFramesUpstream(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            ReadOnlySpan<byte> dictionaryBase, ReadOnlySpan<long> dictionaryOffsets,
            ReadOnlySpan<int> dictionaryLengths, Span<int> lengths, Span<int> errors, Span<int> ends)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (byte* k = dictionaryBase) fixed (long* ko = dictionaryOffsets) fixed (int* kl = dictionaryLengths)
            fixed (int* ol = lengths) fixed (int* oe = errors) fixed (int* oz = ends)
                Check(K4Lz4Native.k4lz4_lz4f_decompress_batch(s, so, sl, d, dof, dc,
                    dictionaryLengths.IsEmpty ? null : k, ko, kl, ol, oe, oz, lengths.Length,
                    K4Lz4Native.MEM_HOST, null, 0));
        }

        // LZ4 frames against a dictionary, as upstream's LZ4F_compressBegin_usingCDict writes them
        // (k4lz4_frame_encode_dict_batch): frame i holds source i, encoded against dictionary i, with the dictID
        // dictionaryIds[i] unless it is 0 (an empty span: no IDs).  blockSize: 64 KiB, 256 KiB, 1 MiB or 4 MiB; flags:
        // K4Lz4Native.FRAME_*.  lengths[i]: the frame's length, -1 where it does not fit targetCapacities[i].
        public static void EncodeFramesWithDictionary(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            ReadOnlySpan<byte> dictionaryBase, ReadOnlySpan<long> dictionaryOffsets,
            ReadOnlySpan<int> dictionaryLengths, ReadOnlySpan<uint> dictionaryIds, Span<int> lengths,
            int blockSize = 65536, int flags = 0)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (byte* x = dictionaryBase) fixed (long* xo = dictionaryOffsets) fixed (int* xl = dictionaryLengths)
            fixed (uint* xi = dictionaryIds) fixed (int* ol = lengths)
                Check(K4Lz4Native.k4lz4_frame_encode_dict_batch(s, so, sl, d, dof, dc, x, xo, xl,
                    dictionaryIds.Length > 0 ? xi : null, ol, lengths.Length, blockSize, flags, 0,
                    K4Lz4Native.MEM_HOST, null, 0));
        }

        // Frames against a dictionary, with or without a dictID field (k4lz4_frame_decode_dict_batch); lengths[i]
        // as k4lz4_frame_decode_batch gives them.  Pick the dictionaries with FrameInfo.
        public static void DecodeFramesWithDictionary(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> targetCapacities,
            ReadOnlySpan<byte> dictionaryBase, ReadOnlySpan<long> dictionaryOffsets,
            ReadOnlySpan<int> dictionaryLengths, Span<int> lengths)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* d = targetBase) fixed (long* dof = targetOffsets) fixed (int* dc = targetCapacities)
            fixed (byte* x = dictionaryBase) fixed (long* xo = dictionaryOffsets) fixed (int* xl = dictionaryLengths)
            fixed (int* ol = lengths)
                Check(K4Lz4Native.k4lz4_frame_decode_dict_batch(s, so, sl, d, dof, dc, x, xo, xl, ol, lengths.Length,
                    K4Lz4Native.MEM_HOST, null, 0));
        }

        // sizes[i]: the content size (the dictionary flag accepted); dictionaryIds[i]: the header's dictID, -1 without
        // a dictID field (k4lz4_frame_info_batch).
        public static void FrameInfo(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<int> sizes, Span<long> dictionaryIds)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (int* os = sizes) fixed (long* oi = dictionaryIds)
                Check(K4Lz4Native.k4lz4_frame_info_batch(s, so, sl, os, oi, sizes.Length,
                    K4Lz4Native.MEM_HOST, null, 0));
        }

        // sizes[i]: what Decode needs as targetCapacities[i] -- 0 for an empty block, -1 where the token chain does
        // not parse (Decode then fails at any capacity)
        public static void DecodedSizes(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            Span<int> sizes)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (int* os = sizes)
                Check(K4Lz4Native.k4lz4_decoded_size_batch(s, so, sl, os, sizes.Length,
                    K4Lz4Native.MEM_HOST, null, K4Lz4Native.ALL_DEVICES));
        }

        // Whole chained streams in one call (k4lz4_decode_chain_streams): stream s owns entries
        // [entryStarts[s], entryStarts[s+1]) and decodes them back to back at targetBase[targetOffsets[s] ..), behind
        // its prefixLengths[s] bytes of history there; raw[e] != 0 marks a stored block (LZ4ChainDecoder.Inject).
        // lengths[e]: what LZ4ChainDecoder.Decode returns block by block; -1 from a stream's first failing block on.
        // Exact, but today about 4x slower on an H100 than decoding one block per stream per call (DESIGN 4.11).
        public static void DecodeChainStreams(
            ReadOnlySpan<byte> sourceBase, ReadOnlySpan<long> sourceOffsets, ReadOnlySpan<int> sourceLengths,
            ReadOnlySpan<byte> raw, ReadOnlySpan<int> blockSizes, Span<int> lengths, ReadOnlySpan<int> entryStarts,
            Span<byte> targetBase, ReadOnlySpan<long> targetOffsets, ReadOnlySpan<int> prefixLengths)
        {
            fixed (byte* s = sourceBase) fixed (long* so = sourceOffsets) fixed (int* sl = sourceLengths)
            fixed (byte* r = raw) fixed (int* bs = blockSizes) fixed (int* ol = lengths)
            fixed (int* es = entryStarts) fixed (byte* d = targetBase) fixed (long* dof = targetOffsets)
            fixed (int* pl = prefixLengths)
                Check(K4Lz4Native.k4lz4_decode_chain_streams(s, so, sl, raw.IsEmpty ? null : r, bs, ol, lengths.Length,
                    es, d, dof, pl, prefixLengths.Length, K4Lz4Native.MEM_HOST, null, K4Lz4Native.ALL_DEVICES));
        }

        private static void Check(int rc)
        {
            if (rc != 0) throw new InvalidOperationException("libk4lz4: " + K4Lz4Native.LastError());
        }
    }
}
