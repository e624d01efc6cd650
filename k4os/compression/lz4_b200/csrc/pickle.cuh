// pickle.cuh -- LZ4Pickler (byte[] variant) over batches of small messages, one warp per message.
//
// Reference behaviour restated (paths under /root/reference/src/K4os.Compression.LZ4/):
//   Pickle   : LZ4Pickler.pickle.cs:51-106 (scratch capacity 1024 if n <= 1024 else n, :57-67;
//              raw form when encoded <= 0 or >= n, :85-94; header byte/diff width, :203-228)
//   Unpickle : LZ4Pickler.unpickle.cs:99-158 (version bits, diff width, size check, decode)
//
// No scratch buffer is needed: the payload is encoded straight into the message's own output
// slot at dst+2 (the k = 1 layout, the tightest one), with the *reference's* capacity driving
// every limitedOutput test and a physical bound of n-1 bytes -- a stream that would grow to n
// bytes ends up in raw form in the reference as well (encoded >= n), so stopping there yields
// the same pickle.  For diff > 255 the payload is then shifted up by 1 (k = 2) or 3 (k = 4).
#pragma once
#include "common.cuh"
#include "encode_generic.cuh"
#include "encode_tile.cuh"
#include "decode_generic.cuh"

namespace k4 {

constexpr int R_CORRUPT = -1000;   // K4LZ4_R_CORRUPT

__host__ __device__ __forceinline__ int pickle_diff_width(int v) {      // EffectiveSizeOf, pickle.cs:224-225
    return (v > 0xffff || v < 0) ? 4 : (v > 0xff ? 2 : 1);
}

// overlapping move of len bytes up by d (1..3) inside one warp, highest chunk first
__device__ __forceinline__ void warp_shift_up(uint8_t* p, int len, int d, int lane) {
    for (int base = ((len - 1) / 32) * 32; base >= 0; base -= 32) {
        const int i = base + lane;
        uint8_t v = 0;
        if (i < len) v = p[i];
        __syncwarp();
        if (i < len) p[i + d] = v;
        __syncwarp();
    }
}

// LZ4Pickler.Pickle<TBufferWriter> (pickle.cs:113-148): the header width is fixed from the full
// length before encoding (:129,161-165) and the payload is encoded in place with capacity n (:130-133).
// X32 (both variants): LZ4Codec.Enforce32, the 32-bit engine's hash4 for messages of LIMIT_64K bytes or more.
template <bool X32>
__device__ int pickle_writer_message_warp(const uint8_t* __restrict__ src, int n, uint8_t* __restrict__ dst,
                                          int level, void* table) {
    const int lane = lane_id();
    if (n <= 0) return 0;                                        // :122
    if (level >= 3) return -2;
    const int k = pickle_diff_width(n);
    const int hs = 1 + k;
    int enc = (n < LIMIT_64K)
        ? encode_spec_warp<false>(src, nullptr, (uint32_t)n, dst + hs, n, n - 1, reinterpret_cast<uint16_t*>(table))
        : encode_block_warp(src, n, dst + hs, n, n - 1, table, X32);
    __syncwarp();
    if (enc <= 0 || enc >= n) {                                  // :135-140
        if (lane == 0) dst[0] = 0;
        for (int i = lane; i < n; i += 32) dst[1 + i] = __ldg(src + i);
        return 1 + n;
    }
    if (lane == 0) {
        const int diff = n - enc;
        dst[0] = (uint8_t)(((k == 4 ? 3 : k) & 3) << 6);
        for (int i = 0; i < k; i++) dst[1 + i] = (uint8_t)((uint32_t)diff >> (8 * i));
    }
    return hs + enc;                                             // :146
}

template <bool X32>
__device__ int pickle_message_warp(const uint8_t* __restrict__ src, int n, uint8_t* __restrict__ dst,
                                   int level, void* table) {
    const int lane = lane_id();
    if (n <= 0) return 0;                                        // pickle.cs:54
    if (level >= 3) return -2;                                   // delegate HC/OPT
    const int cap = n <= 1024 ? 1024 : n;                        // :57-67
    int enc = (n < LIMIT_64K)                                                 // :83
        ? encode_spec_warp<false>(src, nullptr, (uint32_t)n, dst + 2, cap, n - 1, reinterpret_cast<uint16_t*>(table))
        : encode_block_warp(src, n, dst + 2, cap, n - 1, table, X32);
    __syncwarp();
    if (enc <= 0 || enc >= n) {                                  // :85-94
        if (lane == 0) dst[0] = 0;
        for (int i = lane; i < n; i += 32) dst[1 + i] = __ldg(src + i);
        return 1 + n;
    }
    const int diff = n - enc;                                    // :203-212
    const int k = pickle_diff_width(diff);
    if (k > 1) warp_shift_up(dst + 2, enc, k - 1, lane);
    if (lane == 0) {
        dst[0] = (uint8_t)(((k == 4 ? 3 : k) & 3) << 6);         // :221-228
        for (int i = 0; i < k; i++) dst[1 + i] = (uint8_t)((uint32_t)diff >> (8 * i));
    }
    return 1 + k + enc;
}

// DecodeHeaderV0 (unpickle.cs:137-148): returns size or R_CORRUPT; k and diff by reference.
__device__ __forceinline__ int unpickle_header(const uint8_t* __restrict__ src, int n, int& k, int& diff) {
    const uint8_t h = __ldg(src);
    k = 0; diff = 0;
    if ((h & 7) != 0) return R_CORRUPT;                          // :131-135
    k = (h >> 6) & 3; if (k == 3) k = 4;
    const int datalen = n - 1 - k;
    if (datalen < 0) return R_CORRUPT;                           // :142-143
    uint32_t d = 0;
    for (int i = 0; i < k; i++) d |= (uint32_t)__ldg(src + 1 + i) << (8 * i);
    diff = (int)d;
    const int size = datalen + diff;
    return size < 0 ? R_CORRUPT : size;
}

__device__ int unpickle_message_warp(const uint8_t* __restrict__ src, int n, uint8_t* __restrict__ dst,
                                     int dstLen) {
    const int lane = lane_id();
    if (n <= 0) return 0;                                        // :101-102
    int k, diff;
    const int expected = unpickle_header(src, n, k, diff);
    if (expected < 0) return R_CORRUPT;
    if (dstLen != expected) return R_CORRUPT;                    // :115-117
    if (diff == 0) {                                             // :119-123
        for (int i = lane; i < n - 1 - k; i += 32) dst[i] = __ldg(src + 1 + k + i);
        return expected;
    }
    const int dec = codec_decode_warp(src + 1 + k, n - 1 - k, dst, dstLen);   // :125
    return dec != expected ? R_CORRUPT : expected;               // :126-128
}

template <bool X32>
__global__ void __launch_bounds__(ENC_WARPS_PER_CTA * 32)
pickle_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
              const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
              const int64_t* __restrict__ dstOff, int32_t* __restrict__ outLen,
              int nMessages, int level, int writerVariant) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int wInCta = threadIdx.x >> 5;
    const int b = blockIdx.x * ENC_WARPS_PER_CTA + wInCta;
    if (b >= nMessages) return;
    int r = writerVariant
        ? pickle_writer_message_warp<X32>(srcBase + srcOff[b], srcLen[b], dstBase + dstOff[b], level, smem + wInCta * ENC_SLOT_BYTES)
        : pickle_message_warp<X32>(srcBase + srcOff[b], srcLen[b], dstBase + dstOff[b], level, smem + wInCta * ENC_SLOT_BYTES);
    if (lane_id() == 0) outLen[b] = r;
}

__global__ void __launch_bounds__(128)
unpickle_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstLen,
                int32_t* __restrict__ outLen, int nMessages) {
    const int b = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    if (b >= nMessages) return;
    int r = unpickle_message_warp(srcBase + srcOff[b], srcLen[b], dstBase + dstOff[b], dstLen[b]);
    if (lane_id() == 0) outLen[b] = r;
}

__global__ void unpickled_size_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                                      const int32_t* __restrict__ srcLen, int32_t* __restrict__ outSize,
                                      int nMessages) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nMessages) return;
    const int n = srcLen[b];
    if (n <= 0) { outSize[b] = 0; return; }
    int k, diff;
    outSize[b] = unpickle_header(srcBase + srcOff[b], n, k, diff);
}

}  // namespace k4
