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

        private static void Check(int rc)
        {
            if (rc != 0) throw new InvalidOperationException("libk4lz4: " + K4Lz4Native.LastError());
        }
    }
}
