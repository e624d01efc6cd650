// K4Lz4Native.cs -- P/Invoke surface of libk4lz4 (include/k4lz4.h) for K4os.Compression.LZ4.
// Drop into src/K4os.Compression.LZ4/Engine/Native/ (see INTEGRATION.md for the two call sites
// in LZ4Codec.cs that change).  Not compiled in this repository: the build image has no .NET SDK.
using System;
using System.Runtime.InteropServices;

namespace K4os.Compression.LZ4.Engine.Native
{
    internal static unsafe class K4Lz4Native
    {
        private const string Lib = "k4lz4";

        public const int R_DELEGATE = -2;      // level not handled natively (HC/OPT stay managed)
        public const int R_CORRUPT = -1000;    // InvalidDataException ("Pickle is corrupted")
        public const int E_NODEVICE = -100;    // <= -100: library-level failure, see k4lz4_last_error()
        public const int MEM_HOST = 0, MEM_DEVICE = 1, ALL_DEVICES = -1;

        [DllImport(Lib)] public static extern int k4lz4_codec_version();
        [DllImport(Lib)] public static extern int k4lz4_device_count();
        [DllImport(Lib)] public static extern sbyte* k4lz4_last_error();
        [DllImport(Lib)] public static extern int k4lz4_max_output_size(int length);
        [DllImport(Lib)] public static extern int k4lz4_pickle_bound(int length);
        [DllImport(Lib)] public static extern int k4lz4_encode(byte* src, int srcLen, byte* dst, int dstCap, int level);
        [DllImport(Lib)] public static extern int k4lz4_decode(byte* src, int srcLen, byte* dst, int dstCap);
        [DllImport(Lib)] public static extern int k4lz4_encode_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* outLen, int nBlocks, int level, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_decode_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* outLen, int nBlocks, int memKind, void* cudaStream, int device);
        // the decoded length of every raw block (no reference counterpart: sizes for blocks stored without them)
        [DllImport(Lib)] public static extern int k4lz4_decoded_size_batch(
            byte* srcBase, long* srcOff, int* srcLen, int* outSize, int nBlocks,
            int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_pickle_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* outLen, int nMessages, int level, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_unpickled_size_batch(
            byte* srcBase, long* srcOff, int* srcLen, int* outSize, int nMessages,
            int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_unpickle_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstLen,
            int* outLen, int nMessages, int memKind, void* cudaStream, int device);

        // decode with an external dictionary / partial decode (LZ4Codec.cs:123-134,144-157)
        [DllImport(Lib)] public static extern int k4lz4_decode_dict(
            byte* src, int srcLen, byte* dst, int dstCap, byte* dict, int dictLen);
        [DllImport(Lib)] public static extern int k4lz4_partial_decode(byte* src, int srcLen, byte* dst, int targetLen);
        [DllImport(Lib)] public static extern int k4lz4_decode_dict_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            byte* dictBase, long* dictOff, int* dictLen, int* outLen, int nBlocks,
            int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_partial_decode_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* targetLen,
            int* outLen, int nBlocks, int memKind, void* cudaStream, int device);
        // LZ4ChainDecoder.DecodeBlock over many streams, one block each (prefix mode of LZ4_decompress_safe_continue)
        [DllImport(Lib)] public static extern int k4lz4_decode_chain_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* prefixLen, int* outLen, int nBlocks, int memKind, void* cudaStream, int device);
        // LZ4FastChainEncoder.Encode (LZ4_compress_fast_continue, prefix mode) for one block of each of many streams;
        // state = K4LZ4_CHAIN_STATE_BYTES (16 400) per stream, all zero for a new one
        [DllImport(Lib)] public static extern int k4lz4_encode_chain_batch(
            byte* srcBase, long* srcOff, int* srcLen, int* prefixLen, byte* dstBase, long* dstOff, int* dstCap,
            byte* stateBase, long* stateOff, int* outLen, int nBlocks, int level, int memKind, void* cudaStream,
            int device);
        // chain groups: S LZ4FastChainEncoder / LZ4ChainDecoder streams whose rings and states stay on one GPU
        // (kind 0 = encoder, 1 = decoder; streams[i] names the stream block i advances; not thread-safe)
        [DllImport(Lib)] public static extern int k4lz4_chain_group_create(
            int kind, int nStreams, int blockSize, int device, void** group);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_destroy(void* group);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_reset(
            void* group, int* streams, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_encode(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* dstCap, int* outLen, int n, int level, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_decode(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* dstCap, int* outLen, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_inject(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_state(void* group, int stream, byte* state);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_history(void* group, int stream, byte* dst, int cap);
        // LL.Enforce32 semantics (LL.tools.cs:29-36) for inputs >= 65 547 bytes
        [DllImport(Lib)] public static extern int k4lz4_encode_x32(byte* src, int srcLen, byte* dst, int dstCap, int level);
        [DllImport(Lib)] public static extern int k4lz4_encode_batch_x32(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* outLen, int nBlocks, int level, int memKind, void* cudaStream, int device);
        // Pickle<TBufferWriter> (LZ4Pickler.pickle.cs:113-148)
        [DllImport(Lib)] public static extern int k4lz4_pickle_writer_bound(int length);
        [DllImport(Lib)] public static extern int k4lz4_pickle_writer_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* outLen, int nMessages, int level, int memKind, void* cudaStream, int device);
        // the other encoders' twins under LZ4Codec.Enforce32: pick the export from LL.Algorithm at each call
        [DllImport(Lib)] public static extern int k4lz4_encode_chain_batch_x32(
            byte* srcBase, long* srcOff, int* srcLen, int* prefixLen, byte* dstBase, long* dstOff, int* dstCap,
            byte* stateBase, long* stateOff, int* outLen, int nBlocks, int level, int memKind, void* cudaStream,
            int device);
        [DllImport(Lib)] public static extern int k4lz4_chain_group_encode_x32(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* dstCap, int* outLen, int n, int level, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_pickle_batch_x32(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* outLen, int nMessages, int level, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_pickle_writer_batch_x32(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* outLen, int nMessages, int level, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_frame_encode_batch_x32(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* outLen, int nFrames, int blockSize, int flags, int level, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_write_x32(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* dstCap, int* outLen, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_close_x32(
            void* group, int* streams, byte* dstBase, long* dstOff, int* dstCap, int* outLen, int n, int memKind,
            void* cudaStream);

        // LZ4Frame.Encode / Decode over whole buffers, batched across frames (k4lz4.h "LZ4 Frame")
        public const int FRAME_INDEPENDENT = 1, FRAME_BLOCK_CHECKSUM = 2, FRAME_CONTENT_CHECKSUM = 4;
        public const int R_DST_SMALL = -1001;
        [DllImport(Lib)] public static extern long k4lz4_frame_bound(long length, int blockSize, int flags);
        [DllImport(Lib)] public static extern int k4lz4_frame_encode_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* outLen, int nFrames, int blockSize, int flags, int level, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_frame_content_size_batch(
            byte* srcBase, long* srcOff, int* srcLen, int* outSize, int nFrames, int memKind, void* cudaStream, int device);
        [DllImport(Lib)] public static extern int k4lz4_frame_decode_batch(
            byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff, int* dstCap,
            int* outLen, int nFrames, int memKind, void* cudaStream, int device);
        // LZ4EncoderStream / LZ4FrameWriter written incrementally, batched across streams (k4lz4.h "frame writer group")
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_create(
            int nStreams, int blockSize, int flags, int level, int device, void** group);
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_destroy(void* group);
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_reset(
            void* group, int* streams, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_write(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, byte* dstBase, long* dstOff,
            int* dstCap, int* outLen, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_frame_writer_group_close(
            void* group, int* streams, byte* dstBase, long* dstOff, int* dstCap, int* outLen, int n, int memKind,
            void* cudaStream);
        [DllImport(Lib)] public static extern long k4lz4_frame_writer_bound(void* group, long length);
        [DllImport(Lib)] public static extern long k4lz4_frame_writer_close_bound(void* group);
        // LZ4DecoderStream / LZ4FrameReader read incrementally, batched across streams (k4lz4.h "frame reader group")
        [DllImport(Lib)] public static extern int k4lz4_frame_reader_group_create(
            int nStreams, int maxBlockSize, int device, void** group);
        [DllImport(Lib)] public static extern int k4lz4_frame_reader_group_destroy(void* group);
        [DllImport(Lib)] public static extern int k4lz4_frame_reader_group_reset(
            void* group, int* streams, int n, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_frame_reader_group_read(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, int* srcUsed, byte* dstBase,
            long* dstOff, int* dstCap, int* outLen, int* frameEnded, int n, int memKind, void* cudaStream);
        // LZ4DecoderStream.Read(buffer, offset, count): dstCap = count (any size); flags = 1 for interactive reads
        [DllImport(Lib)] public static extern int k4lz4_frame_reader_group_read_bytes(
            void* group, int* streams, byte* srcBase, long* srcOff, int* srcLen, int* srcUsed, byte* dstBase,
            long* dstOff, int* dstCap, int* outLen, int* frameEnded, int n, int flags, int memKind, void* cudaStream);
        [DllImport(Lib)] public static extern int k4lz4_frame_reader_group_end(
            void* group, int* streams, int* status, int n, int memKind, void* cudaStream);

        public static string LastError() => new string(k4lz4_last_error());
    }
}
