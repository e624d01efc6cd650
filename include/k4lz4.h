/*
 * k4lz4.h -- C ABI of libk4lz4: an H100-native (sm_90a CUDA) LZ4 *block* codec that is a
 * drop-in for ONE hot path of K4os.Compression.LZ4:
 *     LZ4Codec.Encode(..., LZ4Level.L00_FAST)   LZ4Codec.Decode(...)   LZ4Pickler.Pickle/Unpickle
 * over batches of independent blocks.  Plain C: pointers and sizes only.
 *
 * The reference (pure managed C#) has no FFI seam of its own; the seam sits directly under
 * its public block API.  Each entry point below names the reference call it replaces
 * (paths relative to /root/reference/src/K4os.Compression.LZ4/).  INTEGRATION.md shows the
 * [DllImport] stubs a maintainer adds.
 *
 * Conventions shared by every call
 *   - return values of the per-block functions and the per-block outLen[] entries are
 *     EXACTLY what the reference's LZ4Codec / LZ4Pickler would have returned for that block
 *     (bytes written, 0 for empty input, -1 when it does not fit / is malformed);
 *   - K4LZ4_E_* (<= -100) are library-level failures (no device, CUDA error, bad argument)
 *     and never collide with codec results; k4lz4_last_error() gives the message;
 *   - bytes of a destination block at index >= its returned length are never written
 *     (SpanTests.cs:36-37, PartialDecompressionTests.cs:33-35);
 *   - every batched call checks its arguments before the machine, in this order: an unknown
 *     memKind, a negative block count, a required pointer that is NULL while nBlocks > 0, and the
 *     host-memory contents (a negative prefixLen, a state offset that is not a multiple of 16, a
 *     level outside 0..255) give K4LZ4_E_ARG; then
 *     no device gives K4LZ4_E_NODEVICE; then nBlocks == 0 returns K4LZ4_OK; then a device index
 *     >= k4lz4_device_count() gives K4LZ4_E_ARG and a failed cudaSetDevice K4LZ4_E_CUDA.  So a
 *     caller's mistake gets the same code with or without a GPU;
 *   - the library never falls back to a CPU codec: without a usable CUDA device every
 *     compute call with valid arguments returns K4LZ4_E_NODEVICE.
 */
#ifndef K4LZ4_H
#define K4LZ4_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define K4LZ4_API __declspec(dllexport)
#else
#define K4LZ4_API __attribute__((visibility("default")))
#endif

/* library-level error codes (never produced by the codec itself) */
#define K4LZ4_OK              0
#define K4LZ4_E_NODEVICE   (-100)  /* no CUDA device / driver: the product path refuses to run */
#define K4LZ4_E_CUDA       (-101)  /* a CUDA runtime call failed; see k4lz4_last_error()        */
#define K4LZ4_E_ARG        (-102)  /* null pointer / negative count / unknown memKind           */
#define K4LZ4_E_NOMEM      (-103)  /* device or pinned-host allocation failed                   */

/* per-block result that is not a reference value: "this level is not handled natively"
 * (HC/OPT levels >= 3 keep delegating to the managed engine, LZ4Codec.cs:48-50) */
#define K4LZ4_R_DELEGATE   (-2)
/* per-message result standing for the reference's InvalidDataException
 * (LZ4Pickler.unpickle.cs:131-135,142-143,115-117,126-128) */
#define K4LZ4_R_CORRUPT    (-1000)

/* memKind */
#define K4LZ4_MEM_HOST     0   /* every pointer is host memory; the call is synchronous      */
#define K4LZ4_MEM_DEVICE   1   /* every pointer (incl. offset/length arrays) is device memory
                                  of `device`; the call only enqueues work on `cudaStream`   */

/* ---- information -------------------------------------------------------------------- */

/* LZ4Codec.Version (LZ4Codec.cs:13) -- the lz4 version whose token streams are reproduced. */
K4LZ4_API int32_t k4lz4_codec_version(void);
/* Number of usable CUDA devices (0 => every compute call returns K4LZ4_E_NODEVICE). */
K4LZ4_API int32_t k4lz4_device_count(void);
/* Message of the last library-level failure on the calling thread ("" if none). */
K4LZ4_API const char *k4lz4_last_error(void);

/* ---- single block: mirrors of the reference's pointer overloads ------------------------ */

/* LZ4Codec.MaximumOutputSize(int) -- LZ4Codec.cs:30-31, Engine/LL.tools.cs:38-40. */
K4LZ4_API int32_t k4lz4_max_output_size(int32_t length);

/* LZ4Codec.Encode(byte*,int,byte*,int,LZ4Level) -- LZ4Codec.cs:40-52; replaces the call to
 * LLxx.LZ4_compress_fast (Engine/LLxx.cs:65-75).  Host pointers.  level < 3 is encoded as
 * L00_FAST (acceleration 1); level >= 3 returns K4LZ4_R_DELEGATE. */
K4LZ4_API int32_t k4lz4_encode(const uint8_t *src, int32_t srcLen,
                               uint8_t *dst, int32_t dstCap, int32_t level);

/* LZ4Codec.Decode(byte*,int,byte*,int) -- LZ4Codec.cs:104-115; replaces the call to
 * LLxx.LZ4_decompress_safe (Engine/LLxx.cs:17-26).  Host pointers. */
K4LZ4_API int32_t k4lz4_decode(const uint8_t *src, int32_t srcLen,
                               uint8_t *dst, int32_t dstCap);

/* ---- batches of independent blocks (the fast path) ------------------------------------- */

/*
 * Block i reads srcBase[srcOff[i] .. +srcLen[i]) and writes dstBase[dstOff[i] .. +dstCap[i]).
 * outLen[i] receives exactly what k4lz4_encode / k4lz4_decode would return for block i with
 * the same dstCap[i].  Function result: K4LZ4_OK or K4LZ4_E_*.
 *
 * memKind == K4LZ4_MEM_DEVICE: all seven pointers live on `device`; work is enqueued on
 *   `cudaStream` (a cudaStream_t; NULL = default stream) and the call returns without
 *   synchronising.
 * memKind == K4LZ4_MEM_HOST: pointers are host memory; `device` >= 0 runs on that GPU,
 *   `device` == K4LZ4_ALL_DEVICES splits the block list contiguously (balanced by bytes) over
 *   every visible GPU, one host thread + stream per GPU, no inter-GPU traffic.  Synchronous.
 */
#define K4LZ4_ALL_DEVICES  (-1)

K4LZ4_API int32_t k4lz4_encode_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                     uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                     int32_t *outLen, int32_t nBlocks, int32_t level,
                                     int32_t memKind, void *cudaStream, int32_t device);

/* The same two calls with the reference's global LL.Enforce32 switch set (Engine/LL.tools.cs:29-36,
 * LZ4Codec.cs:21-25): the 32-bit engine LL32.  Its output differs from LL64's only for inputs of
 * >= 65 547 bytes (4 096-entry u32 table with hash4 instead of hash5, LL64.tools.cs:135-143 vs
 * LL32); below that both engines emit identical bytes and these calls equal the plain ones.
 * Every encoder call has such an _x32 twin: the same arguments, checks in the same order and result codes;
 * only the engine differs.  The reference reads the switch at every encode call (Engine/LLxx.cs:65-91), so a
 * caller picks the export per call.  Decoders need no twin: both engines decode alike. */
K4LZ4_API int32_t k4lz4_encode_x32(const uint8_t *src, int32_t srcLen, uint8_t *dst, int32_t dstCap, int32_t level);
K4LZ4_API int32_t k4lz4_encode_batch_x32(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                         uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                         int32_t *outLen, int32_t nBlocks, int32_t level,
                                         int32_t memKind, void *cudaStream, int32_t device);

K4LZ4_API int32_t k4lz4_decode_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                     uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                     int32_t *outLen, int32_t nBlocks,
                                     int32_t memKind, void *cudaStream, int32_t device);

/* The decoded length of every raw LZ4 block, to size the destinations of k4lz4_decode_batch (as
 * k4lz4_unpickled_size_batch does for pickles and k4lz4_frame_content_size_batch for frames).  No reference call
 * corresponds: it is the batch analogue of LZ4Pickler.UnpickledSize for blocks whose sizes were not stored.
 * outSize[i] = 0 for srcLen[i] <= 0; else the sum of the literal runs plus matchlen + 4 of the token chain, or -1
 * where the chain runs past the end of the block or the length exceeds 2^31 - 1.  Offsets and the decoder's
 * end-of-block rules are not checked, so the call runs one way: wherever k4lz4_decode returns r > 0 for some
 * dstCap, outSize[i] == r; where outSize[i] == -1, k4lz4_decode fails for every dstCap.  Argument checks and codes
 * as k4lz4_xxh32_batch.  Device memory only enqueues work on `cudaStream`; host memory is synchronous and runs on
 * one GPU (`device`, K4LZ4_ALL_DEVICES = GPU 0).  One warp walks each block (csrc/size_walk.cuh). */
K4LZ4_API int32_t k4lz4_decoded_size_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           int32_t *outSize, int32_t nBlocks,
                                           int32_t memKind, void *cudaStream, int32_t device);

/* ---- decode with an external dictionary, partial decode (SURVEY 8f rows 3 and 4) ------------ */

/* LZ4Codec.Decode(byte*,int,byte*,int,byte*,int) -- LZ4Codec.cs:144-157; replaces the call to
 * LLxx.LZ4_decompress_safe_usingDict (Engine/LLxx.cs:42-52, Engine/x64/LL64.dec.cs:523-546).
 * Matches may reach back into `dict` (the bytes logically preceding the block).  Host pointers. */
K4LZ4_API int32_t k4lz4_decode_dict(const uint8_t *src, int32_t srcLen, uint8_t *dst, int32_t dstCap,
                                    const uint8_t *dict, int32_t dictLen);

/* LZ4Codec.PartialDecode(byte*,int,byte*,int) -- LZ4Codec.cs:123-134; replaces the call to
 * LLxx.LZ4_decompress_safe_partial (Engine/LLxx.cs:29-39): decoding stops at targetLen bytes. */
K4LZ4_API int32_t k4lz4_partial_decode(const uint8_t *src, int32_t srcLen, uint8_t *dst, int32_t targetLen);

/* Batched forms; block i uses dictBase[dictOff[i] .. +dictLen[i]) (dictBase may be NULL: no
 * dictionaries).  Same memKind / stream / device conventions as k4lz4_decode_batch, except that
 * memKind == K4LZ4_MEM_HOST runs on one GPU (`device`, K4LZ4_ALL_DEVICES = GPU 0).  These are the
 * exact warp-per-block engine (decode_generic.cuh), not the tile kernel. */
K4LZ4_API int32_t k4lz4_decode_dict_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                          uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                          const uint8_t *dictBase, const int64_t *dictOff, const int32_t *dictLen,
                                          int32_t *outLen, int32_t nBlocks,
                                          int32_t memKind, void *cudaStream, int32_t device);
K4LZ4_API int32_t k4lz4_partial_decode_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                             uint8_t *dstBase, const int64_t *dstOff, const int32_t *targetLen,
                                             int32_t *outLen, int32_t nBlocks,
                                             int32_t memKind, void *cudaStream, int32_t device);

/* Encode against an external dictionary: the blocks LZ4Codec.Decode(source, target, dictionary) (and
 * k4lz4_decode_dict) read back.  No reference call corresponds (the reference has no LZ4_loadDict); the result is
 * upstream lz4's 64-bit engine for
 *     LZ4_loadDict(s, dict, dictLen); LZ4_compress_fast_continue(s, src, dst, srcLen, dstCap, 1);
 * with the dictionary in a buffer of its own (the extDict mode).  Only the last 65 536 bytes of a longer dictionary
 * count, and one of fewer than 8 bytes encodes like none.  Result: bytes written; 0 for srcLen <= 0; -1 when the
 * block does not fit dstCap (upstream returns 0).  Nothing is written at or beyond dstCap.  Host pointers; dict may
 * be NULL when dictLen <= 0. */
K4LZ4_API int32_t k4lz4_encode_dict(const uint8_t *src, int32_t srcLen, uint8_t *dst, int32_t dstCap,
                                    const uint8_t *dict, int32_t dictLen);
/* Batched form; block i encodes against dictBase[dictOff[i] .. +dictLen[i]).  Arguments, checks and codes as
 * k4lz4_decode_dict_batch, except that dictBase / dictOff / dictLen are required when nBlocks > 0.  Blocks whose
 * (dictOff, dictLen) are equal share one loaded table; with host memory they also share one staged copy of the
 * dictionary bytes per chunk.  With device memory a block that does not fit may write anything below its dstCap;
 * with host memory exactly outLen[i] > 0 bytes come back.  memKind == K4LZ4_MEM_HOST is synchronous and runs on one
 * GPU (`device`, K4LZ4_ALL_DEVICES = GPU 0); device memory only enqueues work on `cudaStream`.  Blocks are counted in
 * k4lz4_encode_stats out4[3].  There is no _x32 twin: the reference has no dictionary encoder to reproduce. */
K4LZ4_API int32_t k4lz4_encode_dict_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                          uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                          const uint8_t *dictBase, const int64_t *dictOff, const int32_t *dictLen,
                                          int32_t *outLen, int32_t nBlocks,
                                          int32_t memKind, void *cudaStream, int32_t device);

/* ---- encode into fixed-size destinations (upstream's LZ4_compress_destSize) ------------------ */

/* Encode the longest prefix of src whose block fits targetDstSize bytes.  No reference call corresponds (the
 * reference's engine has the fillOutput branch, Engine/x64/LL64.fast.cs, but no public call reaches it); the result
 * is upstream lz4's 64-bit engine for
 *     n = *srcSize; r = LZ4_compress_destSize(src, dst, &n, targetDstSize);
 * at acceleration 1: the return value is r and *srcSize becomes n, the source bytes the block holds.  A target of
 * at least LZ4_compressBound(*srcSize) gives k4lz4_encode's bytes and consumes everything; an empty source with a
 * target of at least 1 gives the one-byte block 0x00.  Nothing is written at or beyond the returned length.
 * Where nothing is written (targetDstSize < 1, *srcSize < 0 or *srcSize > 0x7E000000) the result is 0 and *srcSize
 * becomes 0.  Upstream leaves *srcSize as it was in that case; a loop that packs a source into fixed-size pages and
 * reads it as "consumed" would then drop data.  Host pointers; src may be NULL when *srcSize is 0. */
K4LZ4_API int32_t k4lz4_encode_dest_size(const uint8_t *src, uint8_t *dst, int32_t *srcSize, int32_t targetDstSize);
/* Batched form: block i encodes srcBase[srcOff[i] .. +srcLen[i]) into at most dstCap[i] bytes at dstBase + dstOff[i];
 * outLen[i] is the single call's result and srcUsed[i] what it leaves in *srcSize.  Argument checks and codes as
 * k4lz4_encode_dict_batch, with srcUsed required instead of the dictionary arrays.  memKind == K4LZ4_MEM_HOST is
 * synchronous and runs on one GPU (`device`, K4LZ4_ALL_DEVICES = GPU 0); device memory only enqueues work on
 * `cudaStream`.  Blocks are counted in k4lz4_encode_stats out4[0..2] by the warp kind that encoded them, as
 * k4lz4_encode_batch's are.  There is no _x32 twin and no level: the reference has no destSize call to reproduce. */
K4LZ4_API int32_t k4lz4_encode_dest_size_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                               uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                               int32_t *outLen, int32_t *srcUsed, int32_t nBlocks,
                                               int32_t memKind, void *cudaStream, int32_t device);

/* ---- chained (linked) blocks: LZ4ChainDecoder, one block per stream per call ------------------ */

/* LZ4ChainDecoder.Decode -> LLxx.LZ4_decompress_safe_continue in prefix mode
 * (LZ4ChainDecoder.cs:45-61,142-143; LL64.dec.cs:479-498,558-592).
 * Block i decodes srcBase[srcOff[i] .. +srcLen[i]) to dstBase[dstOff[i] .. +dstCap[i]); the
 * prefixLen[i] bytes directly in front of it, dstBase[dstOff[i]-prefixLen[i] .. dstOff[i]), are the
 * stream's history (what the reference keeps as lz4sd->prefixSize).  Values >= 65535 all mean
 * "withPrefix64k"; only the last 65535 bytes are ever read.  History bytes are read, never written.
 * outLen[i] = bytes decoded, or -1 where LZ4ChainDecoder.Decode would throw (decoded < 0).
 * Like memcpy's buffers, the blocks of one call must not overlap: no block's
 * [dstOff - prefixLen, dstOff + dstCap) may overlap another block's destination in the same call (one
 * block per stream per call meets this).  Clean blocks of at most 64 KiB output take the shared-memory
 * tile kernel; the rest the exact warp-per-block engine.  memKind == K4LZ4_MEM_HOST stages each block's
 * history in front of its device slot and runs on one GPU (`device`, K4LZ4_ALL_DEVICES = GPU 0).
 * A negative prefixLen is K4LZ4_E_ARG with host memory, outLen = -1 with device memory. */
K4LZ4_API int32_t k4lz4_decode_chain_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                           const int32_t *prefixLen, int32_t *outLen, int32_t nBlocks,
                                           int32_t memKind, void *cudaStream, int32_t device);

/* Whole chained streams in one call: nStreams streams, all their blocks in flight at once (DESIGN 4.11).  Exact, but
 * not yet faster: measured on an H100 it is about 4x slower than k4lz4_decode_chain_batch stepped one block per
 * stream per call, at 1 to 64 streams.
 * Stream s owns entries [entryStart[s], entryStart[s+1]), in stream order (entryStart holds nStreams + 1 values,
 * from 0 to nEntries).  Entry e reads srcBase[srcOff[e] .. +srcLen[e]) with capacity dstCap[e] (the blockSize
 * LZ4ChainDecoder.Decode receives).  raw (may be NULL) marks with raw[e] != 0 an entry stored uncompressed: it is
 * copied as-is (LZ4ChainDecoder.Inject, LZ4ChainDecoder.cs:64-93), and is -1 if srcLen[e] < 0 or > dstCap[e].
 * Stream s decodes its entries back to back at dstBase + dstOff[s]; the prefixLen[s] bytes directly in front of it
 * are its history, as in k4lz4_decode_chain_batch (>= 65535 = withPrefix64k; read, never written).  The caller
 * provides sum(max(dstCap[e], 0)) bytes at dstOff[s] for every stream, and no stream's history or region may
 * overlap another stream's region.
 * outLen[e] is what k4lz4_decode_chain_batch returns for the entry when the stream is decoded one block per call,
 * in order, each behind prefixLen[s] + the bytes decoded so far; a stored entry's is its length.  From a stream's
 * first failing entry on (where LZ4ChainDecoder.Decode would throw) every outLen of that stream is -1.  Bytes of
 * a stream's region at or after its failing entry are unspecified; nothing is written outside the stream regions.
 * Arguments, checks and codes as k4lz4_decode_chain_batch: with host memory a malformed entryStart or a negative
 * prefixLen is K4LZ4_E_ARG; with device memory neither can be checked (an entry no stream holds, and every entry
 * of a stream with a negative prefixLen, get -1).  Host memory is synchronous, runs on one GPU (`device`,
 * K4LZ4_ALL_DEVICES = GPU 0) and splits a stream larger than a staging chunk into consecutive pieces; device
 * memory only enqueues work on `cudaStream`.  The call takes 24 KiB of device workspace per entry from the library's
 * private pool (with host memory, per entry of a chunk). */
K4LZ4_API int32_t k4lz4_decode_chain_streams(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                             const uint8_t *raw, const int32_t *dstCap, int32_t *outLen,
                                             int32_t nEntries, const int32_t *entryStart, uint8_t *dstBase,
                                             const int64_t *dstOff, const int32_t *prefixLen, int32_t nStreams,
                                             int32_t memKind, void *cudaStream, int32_t device);

/* LZ4FastChainEncoder.Encode -> LLxx.LZ4_compress_fast_continue(state, src, dst, n, dstCap, 1)
 * (Encoders/LZ4FastChainEncoder.cs:35-41, Engine/x64/LL64.fast.cs:582-667) with the stream's history
 * contiguous in front of the source (the prefix mode the reference's ring buffer sets up).
 * Block i encodes srcBase[srcOff[i] .. +srcLen[i]) into dstBase[dstOff[i] .. +dstCap[i]); the prefixLen[i]
 * bytes directly in front of the source are the stream's history, and the state record at
 * stateBase + stateOff[i] (K4LZ4_CHAIN_STATE_BYTES, 16-aligned) is read and advanced.  The dictionary the
 * block sees is min(state.dictSize, prefixLen[i]) bytes, which is LZ4_saveDict's clamp: a caller that moves
 * its history (a ring buffer) passes the bytes it kept and never writes the state.  At most 65 535 history
 * bytes are read, never written.  Every block size up to 2 GiB uses the same u32 table (hash5; hash4 in the
 * _x32 twin below).
 * outLen[i] = bytes written; 0 for srcLen <= 0 and K4LZ4_R_DELEGATE for level >= 3, both with the state
 * untouched; -1 where LZ4FastChainEncoder.Encode would throw (the engine returned 0: the block does not fit
 * dstCap), with the state advanced exactly as the reference's is.
 * No two blocks of one call may share a state record, and no block's destination or state record may
 * overlap another block's source, history, destination or state (one block per stream per call meets
 * this).  memKind == K4LZ4_MEM_HOST stages [history | source], the state and the destination slot of each
 * block, copies back exactly outLen > 0 bytes and every state record whole, and runs on one GPU (`device`,
 * K4LZ4_ALL_DEVICES = GPU 0).  A negative prefixLen or a misaligned state offset is K4LZ4_E_ARG with host
 * memory, outLen = -1 (state untouched) with device memory.  Counted in k4lz4_encode_stats out4[3]. */
#define K4LZ4_CHAIN_STATE_BYTES 16400  /* uint32 hashTable[4096]; uint32 currentOffset; uint32 dictSize; uint32 reserved[2];
                                          all zero = a new stream (LZ4_createStream / PinnedMemory.Alloc) */
K4LZ4_API int32_t k4lz4_encode_chain_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           const int32_t *prefixLen,
                                           uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                           uint8_t *stateBase, const int64_t *stateOff,
                                           int32_t *outLen, int32_t nBlocks, int32_t level,
                                           int32_t memKind, void *cudaStream, int32_t device);
/* The same under LL.Enforce32 (LL32.LZ4_compress_fast_continue): hash4 over 4 bytes for the u32 table, for every
 * block size.  The state record is the same, so one stream may alternate between the two calls. */
K4LZ4_API int32_t k4lz4_encode_chain_batch_x32(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                               const int32_t *prefixLen,
                                               uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                               uint8_t *stateBase, const int64_t *stateOff,
                                               int32_t *outLen, int32_t nBlocks, int32_t level,
                                               int32_t memKind, void *cudaStream, int32_t device);

/* ---- chain groups: chained streams whose context stays on the GPU ---------------------------- */

/*
 * A chain group holds S chained streams of one direction on one device: per stream a history ring of
 * 128 KiB + max(blockSize, 64 KiB) bytes, its write position and, for encoders, its 16 400-byte state record
 * (an LZ4FastChainEncoder's LZ4_stream_t, Encoders/LZ4FastChainEncoder.cs:14-41) and a "failed" flag.  A call
 * advances any subset of the streams by one block each; only the blocks' own bytes cross PCIe (memKind
 * K4LZ4_MEM_HOST), or nothing does (K4LZ4_MEM_DEVICE: the call only enqueues work on `cudaStream` and never
 * synchronises the host).  A block sees the last min(bytes so far, 65 536) bytes of its stream as history; that
 * gives exactly the bytes the reference's ring buffers give for any blockSize / extraBlocks.
 *
 * streams[i] names the stream block i advances.  Encoder groups: block i is srcBase[srcOff[i] .. +srcLen[i]),
 * srcLen[i] <= blockSize, and outLen[i] is what k4lz4_encode_chain_batch returns for it (0 for an empty block
 * and K4LZ4_R_DELEGATE for level >= 3, both leaving the stream untouched; -1 where Encode would throw, after
 * which the stream returns -1 until it is reset, as the reference's encoder should then be discarded).
 * Decoder groups: block i decodes into dstBase[dstOff[i] .. +dstCap[i]), dstCap[i] <= blockSize, and outLen[i]
 * is what k4lz4_decode_chain_batch returns (a failed block leaves its stream as it was, like
 * LZ4ChainDecoder.Decode).  A block whose stream index is out of range (device memory), whose length exceeds
 * blockSize or whose encoder stream has failed gets -1 and changes nothing.
 *
 * Host memory: sources go up packed in one copy, results and produced bytes come down compacted; bytes of a
 * destination at index >= outLen[i] are never written.  The group's pinned staging buffers grow and never
 * shrink.  Device memory: every array (streams included) lives on the group's device; encoded bytes are written
 * straight into the destination (a block that does not fit may write anything below its dstCap, as
 * k4lz4_encode_chain_batch does), decoded bytes are copied there from the ring.
 *
 * Arguments, in this order, give K4LZ4_E_ARG: a null group or a group of the other kind; an unknown memKind;
 * a negative count; a required pointer that is NULL while n > 0; with host memory a stream index out of range or
 * listed twice in one call; a level outside 0..255.  A group is bound to the device it was created on.  Like the
 * reference's encoder and decoder objects, a group is not thread-safe: calls on one group must not run
 * concurrently, and device-memory calls on different CUDA streams must be ordered by the caller.  With device
 * memory, listing a stream twice in one call is undefined.  Counted in k4lz4_encode_stats out4[3] and
 * k4lz4_decode_stats like the chained batch calls.
 */
typedef struct k4lz4_chain_group k4lz4_chain_group;
#define K4LZ4_CHAIN_ENCODER 0
#define K4LZ4_CHAIN_DECODER 1

/* kind K4LZ4_CHAIN_ENCODER or K4LZ4_CHAIN_DECODER, nStreams > 0, blockSize > 0, device >= 0 (or < 0: the current
 * device).  K4LZ4_E_ARG for bad arguments, then K4LZ4_E_NODEVICE without a device, K4LZ4_E_NOMEM when the rings
 * do not fit; *out is NULL unless K4LZ4_OK is returned.  Every stream starts new. */
K4LZ4_API int32_t k4lz4_chain_group_create(int32_t kind, int32_t nStreams, int32_t blockSize, int32_t device,
                                           k4lz4_chain_group **out);
/* Frees the group after the device has finished its work (NULL is allowed). */
K4LZ4_API int32_t k4lz4_chain_group_destroy(k4lz4_chain_group *g);
/* Streams streams[0 .. n) become new (LZ4_createStream / a new LZ4ChainDecoder). */
K4LZ4_API int32_t k4lz4_chain_group_reset(k4lz4_chain_group *g, const int32_t *streams, int32_t n,
                                          int32_t memKind, void *cudaStream);
K4LZ4_API int32_t k4lz4_chain_group_encode(k4lz4_chain_group *g, const int32_t *streams,
                                           const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                           int32_t *outLen, int32_t n, int32_t level,
                                           int32_t memKind, void *cudaStream);
/* The same with the 32-bit engine (k4lz4_encode_chain_batch_x32).  The engine is chosen per call, not per group. */
K4LZ4_API int32_t k4lz4_chain_group_encode_x32(k4lz4_chain_group *g, const int32_t *streams,
                                               const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                               uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                               int32_t *outLen, int32_t n, int32_t level,
                                               int32_t memKind, void *cudaStream);
K4LZ4_API int32_t k4lz4_chain_group_decode(k4lz4_chain_group *g, const int32_t *streams,
                                           const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                           int32_t *outLen, int32_t n, int32_t memKind, void *cudaStream);
/* LZ4ChainDecoder.Inject (LZ4ChainDecoder.cs:64-93): srcBase[srcOff[i] .. +srcLen[i]) become the end of stream
 * streams[i]'s history (a stored block of a linked frame).  Any length; only the last 65 536 bytes are kept. */
K4LZ4_API int32_t k4lz4_chain_group_inject(k4lz4_chain_group *g, const int32_t *streams,
                                           const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           int32_t n, int32_t memKind, void *cudaStream);
/* Synchronous readers (they wait for the device).  _state: the encoder stream's K4LZ4_CHAIN_STATE_BYTES record
 * into `out`.  Its dictSize may differ from a ring-buffer encoder's where both exceed 65 536: both mean a full
 * window.  _history: copies the last min(history, cap) bytes of the stream's history (its last <= 65 536
 * bytes) to `out` and returns how many, or K4LZ4_E_*. */
K4LZ4_API int32_t k4lz4_chain_group_state(const k4lz4_chain_group *g, int32_t stream, uint8_t *out);
K4LZ4_API int32_t k4lz4_chain_group_history(const k4lz4_chain_group *g, int32_t stream, uint8_t *out, int32_t cap);

/* ---- XXH32: the checksum of the LZ4 Frame container (SURVEY 8f row 2) ------------------------ */

/* XXH32 of one buffer on the host (frame header byte, serial content checksum) --
 * Streams/Frames/LZ4FrameWriter.cs:100,162-181 via K4os.Hash.xxHash; orig/lib/xxhash.c. */
K4LZ4_API uint32_t k4lz4_xxh32(const uint8_t *data, int64_t length, uint32_t seed);
/* XXH32 of every block of a batch on the GPU (per-block checksums, LZ4FrameWriter.cs:169-175):
 * out[i] = XXH32(base[off[i] .. +len[i]), seed). */
K4LZ4_API int32_t k4lz4_xxh32_batch(const uint8_t *base, const int64_t *off, const int32_t *len, uint32_t seed,
                                    uint32_t *out, int32_t nBlocks,
                                    int32_t memKind, void *cudaStream, int32_t device);

/* ---- LZ4 Frame, whole buffers: LZ4Frame.Encode / LZ4Frame.Decode, batched across frames --------- */

/*
 * Frame i reads srcBase[srcOff[i] .. +srcLen[i]) and writes dstBase[dstOff[i] .. +dstCap[i]); frames and contents
 * are at most 2^31 - 1 bytes.  Every array lives in one memory kind.  memKind == K4LZ4_MEM_DEVICE: every pointer is
 * device memory of `device`, the work is enqueued on `cudaStream`, and the call synchronises the host ONCE, to read
 * the number of blocks and steps (the largest block count of a linked frame) it has to launch for.
 * memKind == K4LZ4_MEM_HOST: synchronous; chunks of whole frames go up and come down in one copy each way, and
 * exactly outLen[i] > 0 bytes of each destination are written.  `device` >= 0 names the GPU (K4LZ4_ALL_DEVICES:
 * GPU 0 with host memory, the current device with device memory), as for k4lz4_decode_chain_batch.  Every frame
 * gets its own result; one bad frame does not affect the others.
 */
#define K4LZ4_FRAME_INDEPENDENT      1  /* LZ4EncoderSettings.ChainBlocks = false; linked blocks are the default */
#define K4LZ4_FRAME_BLOCK_CHECKSUM   2  /* XXH32 of every stored block                                           */
#define K4LZ4_FRAME_CONTENT_CHECKSUM 4  /* XXH32 of the content after the end mark                               */
/* per-frame decode result: dstCap[i] is smaller than the frame's content (nothing of it is written) */
#define K4LZ4_R_DST_SMALL  (-1001)

/* The largest frame k4lz4_frame_encode_batch writes for `length` bytes: 7 header bytes, per block 4 bytes of
 * length code + at most the raw length (+ 4 with block checksums), the 4-byte end mark (+ 4 with the content
 * checksum).  blockSize is rounded as LZ4EncoderBase.cs:29 does (max(1024, rounded up to 1 KiB)) and must be
 * 1 .. 4 MiB; a bad blockSize, a negative length or an unknown flag gives K4LZ4_E_ARG. */
K4LZ4_API int64_t k4lz4_frame_bound(int64_t length, int32_t blockSize, int32_t flags);

/* LZ4Frame.Encode(ReadOnlySpan<byte>, Span<byte>, LZ4EncoderSettings) per frame, L00_FAST
 * (Streams/Frames/LZ4FrameWriter.cs:57-189): header (magic, FLG, BD for blockSize, HC), blocks of blockSize bytes
 * (each encoded with capacity LZ4Codec.MaximumOutputSize(blockSize), linked unless K4LZ4_FRAME_INDEPENDENT, stored
 * raw -- bit 31 of its length code -- when it does not shrink), the end mark and the checksums `flags` asks for.
 * No content size and no dictionary id are written.  outLen[i] = the frame's length; -1 when it does not fit
 * dstCap[i] (the frame may then have written anything inside [dstOff, dstOff + dstCap), as the reference's span
 * writer does before it throws); K4LZ4_R_DELEGATE for level >= 3 (chained HC stays managed), nothing written.
 * Nothing is ever written at or beyond dstCap[i].  Argument errors as k4lz4_encode_batch, then blockSize and flags
 * as k4lz4_frame_bound. */
K4LZ4_API int32_t k4lz4_frame_encode_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                           int32_t *outLen, int32_t nFrames, int32_t blockSize, int32_t flags,
                                           int32_t level, int32_t memKind, void *cudaStream, int32_t device);
/* The same with the 32-bit engine: linked blocks as k4lz4_encode_chain_batch_x32, independent blocks as
 * k4lz4_encode_batch_x32 (identical to the plain call below 65 547-byte blocks). */
K4LZ4_API int32_t k4lz4_frame_encode_batch_x32(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                               uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                               int32_t *outLen, int32_t nFrames, int32_t blockSize, int32_t flags,
                                               int32_t level, int32_t memKind, void *cudaStream, int32_t device);

/* The decoded length of every frame, to size the buffers of k4lz4_frame_decode_batch (as k4lz4_unpickled_size_batch
 * does for k4lz4_unpickle_batch).  outSize[i] = the content length from the blocks' length codes and token chains,
 * or the structural verdict decode gives: K4LZ4_R_CORRUPT for a bad magic number, version or header checksum or a
 * frame cut short, K4LZ4_R_DELEGATE for the dictionary-id flag; -1 for a token chain that does not parse.  Checksums
 * and match offsets are not verified.  Wherever decode succeeds it returns exactly this length. */
K4LZ4_API int32_t k4lz4_frame_content_size_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                                 int32_t *outSize, int32_t nFrames,
                                                 int32_t memKind, void *cudaStream, int32_t device);

/* LZ4Frame.Decode(ReadOnlySpan<byte>, TBufferWriter) per frame (LZ4FrameReader.blocking.cs:57-144): linked and
 * independent frames, every block size, stored blocks, both checksums; a content-size field is read and skipped.
 * Each block decodes with the reference's capacity (blockSize + 8 independent, LZ4BlockDecoder.cs:26; blockSize
 * linked, LZ4ChainDecoder.cs:45-53).  outLen[i] = the content length, written to exactly [dstOff, dstOff + outLen);
 * else, for the first problem in stream order: K4LZ4_R_CORRUPT where the reader throws InvalidDataException (magic,
 * version, header checksum, unexpected end, block or content checksum, a stored block larger than the decoder takes:
 * blockSize + 8 independent, max(blockSize, 64 KiB) linked); -1 for a block the block decoder rejects;
 * K4LZ4_R_DELEGATE for the dictionary-id flag (NotImplementedException); K4LZ4_R_DST_SMALL when the content does not
 * fit dstCap[i].  A failed frame may have written inside [dstOff, dstOff + dstCap), never outside. */
K4LZ4_API int32_t k4lz4_frame_decode_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                           uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                           int32_t *outLen, int32_t nFrames,
                                           int32_t memKind, void *cudaStream, int32_t device);

/* ---- LZ4 Frame against a dictionary (upstream's LZ4F_compressBegin_usingCDict / LZ4F_decompress_usingDict,
 * lz4 -D).  No reference call: the reference's frame code throws NotImplementedException for dictionaries. ---- */

/* Frames against a dictionary: byte for byte what upstream writes with
 * LZ4F_compressBegin_usingCDict(LZ4F_createCDict(dict_i)) + LZ4F_compressUpdate(all) + LZ4F_compressEnd,
 * prefs = {blockSizeID of blockSize, linked unless K4LZ4_FRAME_INDEPENDENT, the checksums `flags` asks for,
 * dictID = dictId[i], level 0, autoFlush 0, no content size}.  Frame i's dictionary is
 * dictBase[dictOff[i] .. + dictLen[i]); only its last 64 KiB count, and one of fewer than 8 bytes loads nothing.
 * dictId may be NULL; an ID of 0 writes no dictID field (as lz4 -D).  Every block is encoded with capacity n - 1 and
 * stored raw when it does not fit (lz4frame.c:747-749; not k4lz4_frame_encode_batch's rule).  blockSize must be
 * 65 536, 262 144, 1 048 576 or 4 194 304, flags as k4lz4_frame_bound.  The largest frame is
 * k4lz4_frame_bound(length, blockSize, flags), + 4 when the ID is not 0.  outLen[i] = the frame's length; -1 when it
 * does not fit dstCap[i]; K4LZ4_R_DELEGATE for level >= 3, nothing written.  Nothing is ever written at or beyond
 * dstCap[i].  Argument errors as k4lz4_frame_encode_batch, then the dictionary arrays (required when nFrames > 0). */
K4LZ4_API int32_t k4lz4_frame_encode_dict_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                                uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                                const uint8_t *dictBase, const int64_t *dictOff, const int32_t *dictLen,
                                                const uint32_t *dictId, int32_t *outLen, int32_t nFrames,
                                                int32_t blockSize, int32_t flags, int32_t level,
                                                int32_t memKind, void *cudaStream, int32_t device);
/* k4lz4_frame_decode_batch's results, codes, their order and capacities, except that the dictionary flag is
 * accepted (its 4 ID bytes are covered by the header checksum and otherwise skipped) and every frame, with or without
 * an ID, decodes against its dictionary.  The ID is not checked against the dictionary (as upstream); pick the
 * dictionaries with k4lz4_frame_info_batch.  Linked block k decodes as k4lz4_decode_chain_batch would behind the last
 * 64 KiB of (dictionary | blocks 0 .. k-1); independent blocks each as k4lz4_decode_dict against the dictionary.
 * dictBase may be NULL: no dictionaries (every result then equals k4lz4_frame_decode_batch's, except for the flag). */
K4LZ4_API int32_t k4lz4_frame_decode_dict_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                                uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                                const uint8_t *dictBase, const int64_t *dictOff, const int32_t *dictLen,
                                                int32_t *outLen, int32_t nFrames,
                                                int32_t memKind, void *cudaStream, int32_t device);
/* outSize[i] as k4lz4_frame_content_size_batch, except that the dictionary flag is not a verdict;
 * outDictId[i] = the header's dictID, or -1 when the frame has no dictID field (or no valid header). */
K4LZ4_API int32_t k4lz4_frame_info_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                         int32_t *outSize, int64_t *outDictId, int32_t nFrames,
                                         int32_t memKind, void *cudaStream, int32_t device);

/* ---- LZ4 Frame as upstream lz4 writes it: LZ4F_compressFrame, batched across frames.  No reference call: the
 * reference's writer has no content size and keeps the caller's block size (upstream liblz4, lz4 CLI, python-lz4). */

/* Write the content-size field (FLG bit 3 + 8 bytes): LZ4F_preferences_t.frameInfo.contentSize != 0 */
#define K4LZ4_FRAME_CONTENT_SIZE     8

/* LZ4F_compressFrameBound(length, prefs) for prefs = {blockSizeID of blockSize, the checksums `flags` asks for}:
 * 19 header bytes, per block 4 bytes of length code + at most the raw length (+ 4 with block checksums), the end
 * mark (+ 4 with the content checksum).  blockSize must be 65 536, 262 144, 1 048 576 or 4 194 304; flags are
 * K4LZ4_FRAME_INDEPENDENT, _BLOCK_CHECKSUM, _CONTENT_CHECKSUM and _CONTENT_SIZE.  A bad blockSize, a negative
 * length or an unknown flag gives K4LZ4_E_ARG. */
K4LZ4_API int64_t k4lz4_lz4f_compress_bound(int64_t length, int32_t blockSize, int32_t flags);

/* LZ4F_compressFrame(dst, cap, src_i, n, prefs) per frame, byte for byte, with prefs = {blockSizeID of blockSize,
 * linked unless K4LZ4_FRAME_INDEPENDENT, the checksums `flags` asks for, contentSize != 0 with
 * K4LZ4_FRAME_CONTENT_SIZE, compressionLevel = level}.  As upstream decides each frame on its own size n
 * (lz4frame.c:385-395), one call may mix modes and block sizes:
 *   - the block size shrinks to the smallest of 64 KiB, 256 KiB and 1 MiB that holds n, up to blockSize;
 *   - a frame of one block (n <= block size) is written independent;
 *   - the content-size field is written only when asked for and n > 0.
 * Every block is encoded with capacity n - 1 and stored raw (bit 31 of its length code) when that fails
 * (lz4frame.c:747-749): independent blocks as LZ4_compress_fast, linked blocks as LZ4_compress_fast_continue on one
 * fresh stream per frame.  There is no _x32 twin: this is upstream's call, not LZ4Codec's.
 * Levels 0, 1 and 2 are acceleration 1, as upstream maps them; K4LZ4_R_DELEGATE for level >= 3 (HC) and for a
 * negative level (acceleration > 1), nothing written.  outLen[i] = the frame's length; -1 when it does not fit
 * dstCap[i] (upstream refuses any dstCap below LZ4F_compressFrameBound instead; here a frame is written whenever it
 * fits).  Nothing is ever written at or beyond dstCap[i].  Argument errors, in order: blockSize and flags as
 * k4lz4_lz4f_compress_bound, then as k4lz4_encode_batch (memKind, nFrames, null pointers, device). */
K4LZ4_API int32_t k4lz4_lz4f_compress_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                            uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                            int32_t *outLen, int32_t nFrames, int32_t blockSize, int32_t flags,
                                            int32_t level, int32_t memKind, void *cudaStream, int32_t device);

/* ---- .lz4 streams as upstream `lz4 -d` reads them (programs/lz4io.c over LZ4F_decompress_usingDict) -------- */

/* Stream i is one whole input file, srcBase[srcOff[i] .. +srcLen[i]), read member by member:
 *   - LZ4 frames by LZ4F's rules: version 1, reserved FLG / BD bits clear, block-size IDs 4..7 only, header checksum,
 *     the dictID flag accepted; a block length code above the BD maximum is an error; blocks decode with capacity
 *     maxBlockSize; a non-zero content-size field must equal the content (checked at the end mark, before the content
 *     checksum);
 *   - skippable frames (magic 0x184D2A50..5F) are skipped; a size that reaches past the end ends the stream;
 *   - legacy members (magic 0x184C2102, lz4 -l): blocks with a 4-byte length, each decoded with capacity 8 MiB; a
 *     length above 8 421 520 ends the member and is read as the next member's magic;
 *   - unknown magic: an error on the first member, the end of the stream (success) on any later one.
 * Linked history never crosses a member boundary.  An empty stream decodes to 0 bytes.
 * outLen[i] = the decoded length, written to exactly [dstOff, dstOff + outLen); -1 on an error; K4LZ4_R_DST_SMALL when
 * the content does not fit dstCap[i], unless the stream has an error that needs no decoding (the ones
 * k4lz4_lz4f_decompressed_size_batch gives), which then wins.  Nothing is ever written outside
 * [dstOff, dstOff + dstCap); a failed stream's destination is unspecified (the CLI's partial output is not
 * reproduced).  outErr[i] = 0, or (e << 8) | c for the first error in stream order, where e is the lz4 CLI's error
 * number (its exit code) and c the LZ4F_errorCodes value for e = 66 (0 otherwise):
 *   40 1..3 bytes of a magic number; 42 a skippable size cut short; 44 unknown magic on the first member;
 *   52 a legacy length or block cut short; 53 a legacy block that does not decode (a 0-length one included);
 *   66 an LZ4F error (a failed block gives ERROR_GENERIC with 64 KiB blocks and ERROR_decompressionFailed with larger
 *      ones, as the CLI's 64 KiB output buffer makes LZ4F report it); 68 the input ends inside an LZ4 frame.
 * outEnd[i] = srcLen[i], or the offset of the undecodable data reading stopped at.
 * dictBase may be NULL; otherwise stream i's dictionary is dictBase[dictOff[i] .. + dictLen[i]), of which the last
 * 64 KiB count (lz4 -d -D), used by every LZ4 frame (whatever its dictID flag) and by no legacy member.
 * Argument errors as k4lz4_frame_decode_dict_batch, and outErr / outEnd are required.  Every input gets a verdict
 * here: there is no K4LZ4_R_DELEGATE. */
K4LZ4_API int32_t k4lz4_lz4f_decompress_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                              uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                              const uint8_t *dictBase, const int64_t *dictOff, const int32_t *dictLen,
                                              int32_t *outLen, int32_t *outErr, int32_t *outEnd, int32_t nStreams,
                                              int32_t memKind, void *cudaStream, int32_t device);
/* The decoded length of every stream, from the members' length codes and token chains, to size the buffers of
 * k4lz4_lz4f_decompress_batch: outSize[i] = the length (K4LZ4_R_CORRUPT above 2^31 - 1), or -1 with outErr[i] for the
 * errors that need no decoding (headers, structure, truncation, token chains that do not parse, blocks longer than
 * their capacity); outEnd[i] as k4lz4_lz4f_decompress_batch.  Checksums, match offsets and content-size fields are
 * not checked, so where decompress fails the two may name different errors.  Wherever decompress succeeds it returns
 * exactly this length. */
K4LZ4_API int32_t k4lz4_lz4f_decompressed_size_batch(const uint8_t *srcBase, const int64_t *srcOff,
                                                     const int32_t *srcLen, int32_t *outSize, int32_t *outErr,
                                                     int32_t *outEnd, int32_t nStreams,
                                                     int32_t memKind, void *cudaStream, int32_t device);

/* ---- LZ4 Frame, written incrementally: LZ4EncoderStream / LZ4FrameWriter, batched across streams ------ */

/*
 * A frame writer group holds S frame writers at L00_FAST on one device (Streams/Frames/LZ4FrameWriter.cs and
 * LZ4FrameWriter.blocking.cs): per stream a ring with the chain-group layout (128 KiB + max(B, 64 KiB) bytes for
 * linked frames, B for independent ones, B = blockSize rounded as LZ4EncoderBase.cs:29 does), the partial block,
 * the 16 400-byte chain state (linked frames) and the running XXH32 of the content (content checksum).  Each call
 * takes one write (or one close) for any subset of the streams.
 *
 * Write: the first write of a frame (even of 0 bytes) emits the header k4lz4_frame_encode_batch writes; every block
 * the write completes is emitted in the same call, encoded with capacity MaximumOutputSize(B) and stored raw when
 * it does not shrink, with its XXH32 when K4LZ4_FRAME_BLOCK_CHECKSUM is set; the rest (< B bytes) waits for the
 * next write.  There is no flush: the reference's Flush emits nothing between full blocks.  Close: the partial
 * block, the end mark and, with K4LZ4_FRAME_CONTENT_CHECKSUM, the XXH32 of all the frame's content; a stream that
 * was not written since it was created, reset or closed emits nothing.  After a close the stream is new.  For
 * every way of cutting a stream's content into writes, the bytes it emits equal k4lz4_frame_encode_batch of the
 * whole content with the same blockSize and flags.
 *
 * streams[i] names the stream entry i writes or closes; entry i appends to dstBase[dstOff[i] .. +dstCap[i]) and
 * outLen[i] is the number of bytes appended.  outLen[i] = -1 when dstCap[i] is below the call's bound
 * (k4lz4_frame_writer_bound of srcLen[i], or k4lz4_frame_writer_close_bound); nothing is then consumed or written
 * and the stream is as it was.  With device memory -1 is also the result of a stream index out of range and of a
 * write whose bound exceeds 2^31 - 1.
 *
 * Host memory: synchronous; sources go up packed (in sub-writes of at most 256 MiB of source), produced bytes come
 * down compacted, and exactly outLen[i] > 0 bytes of each destination are written.  Device memory: every array
 * (streams included) lives on the group's device and the work is enqueued on `cudaStream`; a write synchronises the
 * host ONCE, to read the call's number of steps (the most blocks one entry completes), a close never does.
 *
 * Arguments, in this order, give K4LZ4_E_ARG: a null group; an unknown memKind; a negative count; a required
 * pointer that is NULL while n > 0; with host memory a stream index out of range or listed twice in one call, and
 * a write whose bound exceeds 2^31 - 1.  A group is not thread-safe, and device-memory calls on different CUDA
 * streams must be ordered by the caller; with device memory, listing a stream twice in one call is undefined.
 * Blocks are counted in k4lz4_encode_stats like the calls whose codec they use: out4[3] for linked frames, out4[0..2]
 * for independent ones.
 */
typedef struct k4lz4_frame_writer_group k4lz4_frame_writer_group;

/* nStreams > 0; blockSize 1 .. 4 MiB and flags as k4lz4_frame_bound takes them; level 0..255; device >= 0 (or < 0:
 * the current device).  K4LZ4_E_ARG for bad arguments, K4LZ4_R_DELEGATE for level >= 3 (no group: chained HC stays
 * managed), then K4LZ4_E_NODEVICE without a device, K4LZ4_E_NOMEM when the rings do not fit; *out is NULL unless
 * K4LZ4_OK is returned.  Every stream starts new. */
K4LZ4_API int32_t k4lz4_frame_writer_group_create(int32_t nStreams, int32_t blockSize, int32_t flags, int32_t level,
                                                  int32_t device, k4lz4_frame_writer_group **out);
/* Frees the group after the device has finished its work (NULL is allowed). */
K4LZ4_API int32_t k4lz4_frame_writer_group_destroy(k4lz4_frame_writer_group *g);
/* Streams streams[0 .. n) are abandoned: they emit nothing and become new. */
K4LZ4_API int32_t k4lz4_frame_writer_group_reset(k4lz4_frame_writer_group *g, const int32_t *streams, int32_t n,
                                                 int32_t memKind, void *cudaStream);
/* Entry i writes srcBase[srcOff[i] .. +srcLen[i]) to stream streams[i]. */
K4LZ4_API int32_t k4lz4_frame_writer_group_write(k4lz4_frame_writer_group *g, const int32_t *streams,
                                                 const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                                 uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                                 int32_t *outLen, int32_t n, int32_t memKind, void *cudaStream);
/* Entry i closes stream streams[i]. */
K4LZ4_API int32_t k4lz4_frame_writer_group_close(k4lz4_frame_writer_group *g, const int32_t *streams,
                                                 uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                                 int32_t *outLen, int32_t n, int32_t memKind, void *cudaStream);
/* Write and close with the 32-bit engine (the blocks as k4lz4_frame_encode_batch_x32 encodes them).  The engine is
 * chosen per call, not per group: each call's blocks use its own, and streams keep one state layout for both. */
K4LZ4_API int32_t k4lz4_frame_writer_group_write_x32(k4lz4_frame_writer_group *g, const int32_t *streams,
                                                     const uint8_t *srcBase, const int64_t *srcOff,
                                                     const int32_t *srcLen, uint8_t *dstBase, const int64_t *dstOff,
                                                     const int32_t *dstCap, int32_t *outLen, int32_t n,
                                                     int32_t memKind, void *cudaStream);
K4LZ4_API int32_t k4lz4_frame_writer_group_close_x32(k4lz4_frame_writer_group *g, const int32_t *streams,
                                                     uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstCap,
                                                     int32_t *outLen, int32_t n, int32_t memKind, void *cudaStream);
/* The most one write of `length` bytes appends: 7 + floor((B - 1 + length) / B) * (4 + B + 4 with block
 * checksums).  K4LZ4_E_ARG for a null group or a negative length. */
K4LZ4_API int64_t k4lz4_frame_writer_bound(const k4lz4_frame_writer_group *g, int64_t length);
/* The most one close appends: 4 + B (+ 4 with block checksums), the end mark (4), the content checksum (4). */
K4LZ4_API int64_t k4lz4_frame_writer_close_bound(const k4lz4_frame_writer_group *g);

/* ---- LZ4 Frame, read incrementally: LZ4DecoderStream / LZ4FrameReader, batched across streams --------- */

/*
 * A frame reader group holds S frame readers on one device (Streams/Frames/LZ4FrameReader.async.cs): per stream a
 * ring with the chain-group layout (128 KiB + SLOT bytes, SLOT = max(maxBlockSize + 8, 64 KiB)), a stash for a block
 * cut by the end of a chunk (length code, body, checksum), a stash for a cut header or content checksum, the open
 * frame's flags and BD, the running XXH32 of its content, a phase and a sticky error: about 256 KiB per stream at
 * maxBlockSize 64 KiB, 8.3 MB at 4 MiB.  Each call feeds one chunk of compressed bytes (of any size, cut anywhere)
 * to any subset of the streams.  Frames written at any level read alike: the reader has no level.
 *
 * Read: entry i consumes the first srcUsed[i] <= srcLen[i] bytes of srcBase[srcOff[i] ..), in stream order, and
 * appends the content of every block it decodes to dstBase[dstOff[i] ..); outLen[i] is the number of bytes
 * appended.  A call consumes bytes of at most one frame: it stops after the byte that ends a frame (the end mark, or
 * the content checksum when the frame has one), and then frameEnded[i] = 1; the next call starts the next frame, so
 * concatenated frames are read one after another.
 *
 * Room: blockCap is the frame's BD maximum for a linked frame and that maximum + 8 for an independent one (the
 * reference decoder's capacity).  A call decodes at most floor(dstCap[i] / blockCap) blocks, each counted as
 * blockCap whatever it decodes to (decoded bytes are still appended densely).  Once that budget is spent the call
 * stops before the next length code, except that a complete end mark and the content checksum behind it are still
 * consumed.  Header bytes need no room.  A _read block is never drained across calls: dstCap[i] >= blockCap always
 * makes progress.  For destinations of any size, use k4lz4_frame_reader_group_read_bytes.
 *
 * Errors: the first problem in stream order decides, and outLen[i] is then the code k4lz4_frame_decode_batch gives
 * for that frame: K4LZ4_R_CORRUPT for a bad magic (skippable and legacy frames included), version, header checksum,
 * block or content checksum, or a stored block larger than blockCap; -1 for a block the decoder rejects;
 * K4LZ4_R_DELEGATE for the dictionary flag and for a BD above the group's maxBlockSize.  A header is judged when its
 * magic (4 bytes) or all of it (7 or 15 bytes) has arrived.  A compressed block too long for any block the decoder
 * accepts is not stashed but skipped (its body hashed as it passes): its checksum mismatch gives K4LZ4_R_CORRUPT,
 * its truncation K4LZ4_R_CORRUPT from _end, and otherwise -1 once its last byte has arrived.  srcUsed[i] and dstBase[dstOff[i] .. +dstCap[i]) are then unspecified,
 * and the stream has failed: every later read returns the same code and consumes nothing until it is reset or ended.
 *
 * Host memory: synchronous; chunks go up packed, in sub-reads of at most 256 MiB (cutting a read in two changes
 * nothing), decoded bytes come down compacted, and exactly outLen[i] > 0 bytes of each destination are written.
 * Device memory: every array (streams included) lives on the group's device and the work is enqueued on
 * `cudaStream`; a read synchronises the host ONCE, to read the call's row and step counts, an end or reset never
 * does.  A stream index out of range gives outLen[i] (or status[i]) = K4LZ4_E_ARG and consumes nothing.
 *
 * Arguments, in this order, give K4LZ4_E_ARG: a null group; an unknown memKind; a negative count; a required pointer
 * that is NULL while n > 0; with host memory a stream index out of range or listed twice in one call.  A group is not
 * thread-safe; with device memory, listing a stream twice in one call is undefined.  Blocks are counted in
 * k4lz4_decode_stats like the decode calls whose engine they use.
 */
typedef struct k4lz4_frame_reader_group k4lz4_frame_reader_group;

/* nStreams > 0; maxBlockSize 65 536, 262 144, 1 048 576 or 4 194 304; device >= 0 (or < 0: the current device).
 * K4LZ4_E_ARG for bad arguments, then K4LZ4_E_NODEVICE without a device, K4LZ4_E_NOMEM when the rings do not fit;
 * *out is NULL unless K4LZ4_OK is returned.  Every stream starts new. */
K4LZ4_API int32_t k4lz4_frame_reader_group_create(int32_t nStreams, int32_t maxBlockSize, int32_t device,
                                                  k4lz4_frame_reader_group **out);
/* Frees the group after the device has finished its work (NULL is allowed). */
K4LZ4_API int32_t k4lz4_frame_reader_group_destroy(k4lz4_frame_reader_group *g);
/* Streams streams[0 .. n) become new (their input so far is dropped). */
K4LZ4_API int32_t k4lz4_frame_reader_group_reset(k4lz4_frame_reader_group *g, const int32_t *streams, int32_t n,
                                                 int32_t memKind, void *cudaStream);
/* Entry i feeds srcBase[srcOff[i] .. +srcLen[i]) to stream streams[i]. */
K4LZ4_API int32_t k4lz4_frame_reader_group_read(k4lz4_frame_reader_group *g, const int32_t *streams,
                                                const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                                int32_t *srcUsed, uint8_t *dstBase, const int64_t *dstOff,
                                                const int32_t *dstCap, int32_t *outLen, int32_t *frameEnded,
                                                int32_t n, int32_t memKind, void *cudaStream);

/*
 * Byte reads: entry i is one ReadManyBytes(buffer[dstCap[i]], interactive) of the reference
 * (Streams/Frames/LZ4FrameReader.blocking.cs), fed srcBase[srcOff[i] .. +srcLen[i]) instead of pulling.  dstCap[i]
 * may be anything >= 0 and outLen[i] <= dstCap[i].
 *
 * The call first appends min(dstCap[i], undrained) bytes of the stream's current decoded block.  While room is left
 * it then decodes the next complete block of the chunk (or the stashed one) and appends as much of it as fits; the
 * rest stays undrained, on the device, for the next call.  It stops when the destination is full, when the chunk
 * holds no further complete block, at the frame's end, or after a block that decodes to 0 bytes (a raw block
 * 0x80000000, say; the frame stays open).  With K4LZ4_READ_INTERACTIVE it stops after the first drain that appended
 * anything: the leftover of the current block, or else the first new block.  The end mark is consumed only when the
 * call reaches it (nothing undrained and room left), so a call that exactly fills the destination leaves it to the
 * next call, which returns 0 with frameEnded[i] = 1.  Header bytes need no room, as with _read.
 *
 * Otherwise as _read: cut headers and blocks are stashed, at most one frame is consumed per call, and the codes,
 * their order, the sticky failure and the skipped blocks are the same.  A block the call does not reach is neither
 * checksummed nor decoded; the content checksum covers each block as it is decoded.  Host memory: synchronous, and
 * cutting a read into sub-reads changes nothing; device memory: the host waits once per call.
 *
 * Mixing: a _read entry on a stream that holds undrained bytes gives outLen[i] = K4LZ4_E_ARG, consumes nothing and
 * does not fail the stream.  _end and _reset discard undrained bytes; _end then reports K4LZ4_R_CORRUPT, since the
 * frame is still open.  Arguments: _read's, in its order, then flags other than 0 or K4LZ4_READ_INTERACTIVE.
 */
#define K4LZ4_READ_INTERACTIVE 1
K4LZ4_API int32_t k4lz4_frame_reader_group_read_bytes(k4lz4_frame_reader_group *g, const int32_t *streams,
                                                      const uint8_t *srcBase, const int64_t *srcOff,
                                                      const int32_t *srcLen, int32_t *srcUsed, uint8_t *dstBase,
                                                      const int64_t *dstOff, const int32_t *dstCap, int32_t *outLen,
                                                      int32_t *frameEnded, int32_t n, int32_t flags, int32_t memKind,
                                                      void *cudaStream);
/* The input of streams[i] has ended: status[i] = 0 between frames (never fed, or its last read ended a frame),
 * K4LZ4_R_CORRUPT inside a frame (the reference's EndOfStreamException; 1-3 bytes of a magic included), the failed
 * stream's code.  Every stream named becomes new. */
K4LZ4_API int32_t k4lz4_frame_reader_group_end(k4lz4_frame_reader_group *g, const int32_t *streams, int32_t *status,
                                               int32_t n, int32_t memKind, void *cudaStream);

/* ---- LZ4Pickler, byte[] variant, batched ----------------------------------------------- */

/* Upper bound of Pickle() output for an n-byte message: n + 1 (0 for n == 0). */
K4LZ4_API int32_t k4lz4_pickle_bound(int32_t length);

/* LZ4Pickler.Pickle(ReadOnlySpan<byte>, LZ4Level) -- LZ4Pickler.pickle.cs:51-106.
 * Message i -> dstBase[dstOff[i] ..), which must hold k4lz4_pickle_bound(srcLen[i]) bytes;
 * outLen[i] = pickle length (0 for an empty message).  The scratch-capacity rule of the
 * reference (1024 if n <= 1024 else n, pickle.cs:57-67) is applied internally. */
K4LZ4_API int32_t k4lz4_pickle_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                     uint8_t *dstBase, const int64_t *dstOff,
                                     int32_t *outLen, int32_t nMessages, int32_t level,
                                     int32_t memKind, void *cudaStream, int32_t device);
/* The same under LL.Enforce32: messages of >= 65 547 bytes are encoded by the 32-bit engine (LZ4Codec.Encode,
 * k4lz4_encode_x32); shorter ones give the plain call's bytes.  Likewise k4lz4_pickle_writer_batch_x32 below. */
K4LZ4_API int32_t k4lz4_pickle_batch_x32(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                         uint8_t *dstBase, const int64_t *dstOff,
                                         int32_t *outLen, int32_t nMessages, int32_t level,
                                         int32_t memKind, void *cudaStream, int32_t device);

/* LZ4Pickler.Pickle<TBufferWriter>(ReadOnlySpan<byte>, writer, level) -- LZ4Pickler.pickle.cs:113-148.
 * Different bytes than the byte[] variant: the header width is chosen from the full length before
 * encoding (:129,161-165) and the payload is encoded with capacity n (:130-133).  Message i ->
 * dstBase[dstOff[i] ..), which must hold k4lz4_pickle_writer_bound(srcLen[i]) bytes (what the
 * reference asks its writer for); outLen[i] = bytes the reference would Advance() the writer by. */
K4LZ4_API int32_t k4lz4_pickle_writer_bound(int32_t length);
K4LZ4_API int32_t k4lz4_pickle_writer_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                            uint8_t *dstBase, const int64_t *dstOff,
                                            int32_t *outLen, int32_t nMessages, int32_t level,
                                            int32_t memKind, void *cudaStream, int32_t device);
K4LZ4_API int32_t k4lz4_pickle_writer_batch_x32(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                                uint8_t *dstBase, const int64_t *dstOff,
                                                int32_t *outLen, int32_t nMessages, int32_t level,
                                                int32_t memKind, void *cudaStream, int32_t device);

/* LZ4Pickler.UnpickledSize(ReadOnlySpan<byte>) -- LZ4Pickler.unpickle.cs:83-92,131-148.
 * outSize[i] = unpickled size, or K4LZ4_R_CORRUPT where the reference throws. */
K4LZ4_API int32_t k4lz4_unpickled_size_batch(const uint8_t *srcBase, const int64_t *srcOff,
                                             const int32_t *srcLen, int32_t *outSize,
                                             int32_t nMessages,
                                             int32_t memKind, void *cudaStream, int32_t device);

/* LZ4Pickler.Unpickle(ReadOnlySpan<byte>, Span<byte>) -- LZ4Pickler.unpickle.cs:99-129.
 * dstLen[i] must equal the unpickled size (else K4LZ4_R_CORRUPT, unpickle.cs:115-117);
 * outLen[i] = bytes produced or K4LZ4_R_CORRUPT. */
K4LZ4_API int32_t k4lz4_unpickle_batch(const uint8_t *srcBase, const int64_t *srcOff, const int32_t *srcLen,
                                       uint8_t *dstBase, const int64_t *dstOff, const int32_t *dstLen,
                                       int32_t *outLen, int32_t nMessages,
                                       int32_t memKind, void *cudaStream, int32_t device);

/* ---- synthetic workload generator (bench / tests; not part of the reference surface) ---- */

/*
 * Fills nBlocks blocks of blockSize bytes (block i at base + i*blockSize) with LZ-friendly
 * synthetic data: each block independently, a seeded mix of skewed-alphabet literal runs and
 * back-references within the block.  matchPermille steers compressibility (0 = noise only).
 * The host and device variants produce identical bytes for identical arguments.
 */
K4LZ4_API int32_t k4lz4_synth_host(uint8_t *base, int64_t nBlocks, int32_t blockSize,
                                   int32_t matchPermille, uint64_t seed, int64_t firstBlock);
K4LZ4_API int32_t k4lz4_synth_device(uint8_t *base, int64_t nBlocks, int32_t blockSize,
                                     int32_t matchPermille, uint64_t seed, int64_t firstBlock,
                                     void *cudaStream, int32_t device);

/*
 * Batched variable-length copy on the device: block i moves len[i] bytes from
 * srcBase[srcOff[i]..) to dstBase[dstOff[i]..)  (len[i] <= 0 copies nothing).  Used to pack the
 * padded output slots of an encode batch into a dense stream (and by the host path before
 * its single D2H).  Device pointers only; enqueues on `cudaStream`.
 */
K4LZ4_API int32_t k4lz4_copy_blocks_device(const uint8_t *srcBase, const int64_t *srcOff,
                                           uint8_t *dstBase, const int64_t *dstOff,
                                           const int32_t *len, int32_t nBlocks,
                                           void *cudaStream, int32_t device);

/* Counters for bench.py: number of kernels this library has launched since load. */
K4LZ4_API int64_t k4lz4_launch_count(void);

/* Decoder path counters of `device` since the last reset: out4[0] blocks decoded by the
 * shared-memory tile kernel (two CTAs per SM), [1] by its big-stage variant, [2] by the exact
 * warp-per-block decoder (malformed / oversized / unusual blocks), [3] parse repair walks.
 * Synchronises the device.  Diagnostics only (tests assert that clean data stays on the tile path). */
K4LZ4_API int32_t k4lz4_decode_stats(int32_t device, uint64_t *out4, int32_t reset);

/* Encoder path counters of `device` since the last reset: out4[0] blocks encoded by a warp with its
 * hash table in shared memory, [1] by a warp with its table in global memory (only launched when a
 * call has more blocks than the shared-memory warps take in one round), [2] blocks of >= 65 547
 * bytes (the u32-table engine, either warp kind); [0..2] count k4lz4_encode_dest_size_batch's blocks too; [3] chained blocks (k4lz4_encode_chain_batch, any
 * size) and blocks encoded against a dictionary (k4lz4_encode_dict_batch).  Empty blocks, delegated levels and rejected arguments are not counted.
 * Synchronises the device.  Diagnostics only. */
K4LZ4_API int32_t k4lz4_encode_stats(int32_t device, uint64_t *out4, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* K4LZ4_H */
