// decode_generic.cuh -- size-agnostic LZ4 block decoder: one warp per block, streams read and
// written in global memory.  It is the path for blocks that do not fit the shared-memory
// tile decoder (decode_tile.cuh) and the warp-level engine behind unpickle.
//
// Semantics = LZ4_decompress_safe as reached from LZ4Codec.Decode:
//   /root/reference/src/K4os.Compression.LZ4/Engine/x64/LL64.dec.cs:124-467 (generic loop,
//   endOnInputSize / full / noDict / lowPrefix = dst) and :469-477; every accept/reject test
//   is evaluated in the reference's order so that the returned value matches for malformed
//   input as well.  Control is warp-uniform: all lanes track (ip, op); the copies are
//   lane-parallel.  A match with offset 0 (accepted by the reference, content unspecified)
//   produces zero bytes.
#pragma once
#include "common.cuh"

namespace k4 {

// dst[op .. op+len) = src bytes; lanes stride by 32.
__device__ __forceinline__ void warp_copy_in(uint8_t* __restrict__ d, const uint8_t* __restrict__ s,
                                             int len, int lane) {
    for (int i = lane; i < len; i += 32) d[i] = __ldg(s + i);
}

// LZ77 match copy inside dst.  For an overlapping match (offset < len) the result is periodic
// with period `offset`, so every byte is fetched from the already-final window
// [match, match+offset): no intra-copy dependency between lanes.
__device__ __forceinline__ void warp_copy_match(uint8_t* dst, int64_t op, int64_t match,
                                                int len, int offset, int lane) {
    __syncwarp();   // earlier stores of other lanes must be visible
    if (offset == 0) {
        for (int i = lane; i < len; i += 32) dst[op + i] = 0;
    } else if (offset >= len) {
        for (int i = lane; i < len; i += 32) dst[op + i] = dst[match + i];
    } else {
        for (int i = lane; i < len; i += 32) dst[op + i] = dst[match + (i % offset)];
    }
}

// Returns bytes written (>= 0) or a negative value on malformed input / insufficient room.
__device__ int decode_block_warp(const uint8_t* __restrict__ src, int n,
                                 uint8_t* __restrict__ dst, int cap) {
    const int lane = lane_id();
    int64_t ip = 0, op = 0;
    const int64_t iend = n, oend = cap;
    const int64_t shortiend = iend - 16;      // LL64.dec.cs:152
    const int64_t shortoend = oend - 32;      // LL64.dec.cs:153

    if (cap == 0) return (n == 1 && __ldg(src) == 0) ? 0 : -1;   // :162-168
    if (n == 0) return -1;                                       // :172

    for (;;) {
        const uint32_t token = __ldg(src + ip); ip++;            // :177
        int64_t len = token >> 4;
        const bool shortcut = (len != 15) && (ip < shortiend) && (op <= shortoend);   // :191-193
        if (!shortcut) {
            if (len == 15) {                                     // :228-243, LL.tools.cs:165-193
                if (ip >= iend - 15) return -1;                  // initial_error
                for (;;) {
                    uint32_t s = __ldg(src + ip); ip++;
                    len += s;
                    if (ip >= iend - 15) break;                  // loop_error: not fatal here
                    if (s != 255) break;
                }
            }
            const int64_t cpy = op + len;                        // :246
            if (cpy > oend - MFLIMIT || ip + len > iend - (2 + 1 + LASTLITERALS)) {
                if (ip + len != iend || cpy > oend) return -1;   // :291-294
                warp_copy_in(dst + op, src + ip, (int)len, lane);
                return (int)(op + len);                          // :304-307, :454-457
            }
        }
        warp_copy_in(dst + op, src + ip, (int)len, lane);        // :196-200 / :311-314
        ip += len; op += len;

        const int offset = (int)__ldg(src + ip) | ((int)__ldg(src + ip + 1) << 8);   // :205 / :318
        ip += 2;
        const int64_t match = op - offset;
        len = token & 15;                                        // :204 / :323

        if (shortcut && len != 15 && offset >= 8 && match >= 0) {   // :211-220
            len += MINMATCH;
            warp_copy_match(dst, op, match, (int)len, offset, lane);
            op += len;
            continue;
        }
        if (len == 15) {                                         // :326-334
            for (;;) {
                uint32_t s = __ldg(src + ip); ip++;
                len += s;
                if (ip >= iend - LASTLITERALS + 1) return -1;    // any overrun is fatal
                if (s != 255) break;
            }
        }
        len += MINMATCH;                                         // :336
        if (match < 0) return -1;                                // :338
        const int64_t cpy = op + len;                            // :383
        if (cpy > oend - LASTLITERALS) return -1;                // :427-433
        warp_copy_match(dst, op, match, (int)len, offset, lane);
        op = cpy;                                                // :450
    }
}

// LZ77 copy through the virtual window [dict | dst]: byte i of the match comes from window position
// match + (i mod offset), which lies in [op - offset, op) -- final bytes of the dictionary (negative
// positions) or of the block; no lane depends on another lane of the same copy.
__device__ __forceinline__ void warp_copy_match_window(uint8_t* dst, int64_t op, int64_t match, int len, int offset,
                                                       const uint8_t* __restrict__ dict, int dictSize, int lane) {
    __syncwarp();
    if (offset == 0) { for (int i = lane; i < len; i += 32) dst[op + i] = 0; return; }
    for (int i = lane; i < len; i += 32) {
        const int64_t j = match + (offset >= len ? i : i % offset);
        dst[op + i] = j < 0 ? __ldg(dict + dictSize + j) : dst[j];
    }
}

// The general form of decode_block_warp: external dictionary (LZ4_decompress_safe_usingDict,
// LL64.dec.cs:523-546 -> forceExtDict :510-521; the prefix variants read the same bytes and reject
// the same offsets) and/or partial decoding (LZ4_decompress_safe_partial :548-556 with
// dstCapacity == targetOutputSize, LLxx.cs:29-39; paths :256-280, :301-307, :387-406), or prefix mode:
// `prefix` bytes of history lie directly in front of dst (LZ4_decompress_safe_withSmallPrefix /
// _withPrefix64k, LL64.dec.cs:479-498, as LZ4_decompress_safe_continue calls them :558-592): lowPrefix =
// dst - prefix, dictSize = 0; prefix >= 65535 is withPrefix64k, whose shortcut test (:213) no offset fails.
__device__ int decode_block_warp_general(const uint8_t* __restrict__ src, int n, uint8_t* __restrict__ dst,
                                         int outputSize, bool partial,
                                         const uint8_t* __restrict__ dict, int dictSize, int prefix = 0) {
    const int lane = lane_id();
    int64_t ip = 0, op = 0;
    const int64_t iend = n, oend = outputSize;
    const int64_t shortiend = iend - 16, shortoend = oend - 32;
    const bool checkOffset = dictSize < 65536;                       // :147
    const bool extDict = dict != nullptr && dictSize > 0;
    if (!extDict) dictSize = 0;
    const int64_t lowPrefix = extDict ? 0 : -(int64_t)(prefix < 65535 ? prefix : 65535);   // relative to dst

    if (outputSize == 0) {                                           // :162-168
        if (partial) return 0;
        return (n == 1 && __ldg(src) == 0) ? 0 : -1;
    }
    if (n == 0) return -1;

    for (;;) {
        const uint32_t token = __ldg(src + ip); ip++;
        int64_t len = token >> 4;
        const bool shortcut = (len != 15) && (ip < shortiend) && (op <= shortoend);
        bool literalsDone = false;
        if (!shortcut) {
            if (len == 15) {
                if (ip >= iend - 15) return -1;
                for (;;) {
                    uint32_t s = __ldg(src + ip); ip++;
                    len += s;
                    if (ip >= iend - 15) break;
                    if (s != 255) break;
                }
            }
            int64_t cpy = op + len;
            if (cpy > oend - MFLIMIT || ip + len > iend - (2 + 1 + LASTLITERALS)) {
                if (partial) {                                       // :256-280
                    if (ip + len > iend - (2 + 1 + LASTLITERALS) && ip + len != iend) return -1;
                    if (cpy > oend) { cpy = oend; len = oend - op; }
                } else if (ip + len != iend || cpy > oend) return -1;   // :291-294
                warp_copy_in(dst + op, src + ip, (int)len, lane);
                ip += len; op += len;
                if (!partial || cpy == oend || ip == iend) return (int)op;   // :304-307
                literalsDone = true;
            }
        }
        if (!literalsDone) {
            warp_copy_in(dst + op, src + ip, (int)len, lane);
            ip += len; op += len;
        }

        const int offset = (int)__ldg(src + ip) | ((int)__ldg(src + ip + 1) << 8);
        ip += 2;
        const int64_t match = op - offset;
        len = token & 15;

        if (shortcut && len != 15 && offset >= 8 && match >= lowPrefix) {   // :211-220
            len += MINMATCH;
            warp_copy_match(dst, op, match, (int)len, offset, lane);
            op += len;
            continue;
        }
        if (len == 15) {
            for (;;) {
                uint32_t s = __ldg(src + ip); ip++;
                len += s;
                if (ip >= iend - LASTLITERALS + 1) return -1;
                if (s != 255) break;
            }
        }
        len += MINMATCH;
        if (checkOffset && match + dictSize < lowPrefix) return -1;  // :338
        if (match < lowPrefix) {
            if (!extDict) return -1;                                  // (unreachable with checkOffset on)
            if (op + len > oend - LASTLITERALS) {                     // :343-347
                if (partial) len = (oend - op) < len ? (oend - op) : len;
                else return -1;
            }
            warp_copy_match_window(dst, op, match, (int)len, offset, dict, dictSize, lane);
            op += len;
            continue;
        }
        const int64_t cpy = op + len;
        if (partial && cpy > oend - 12) {                            // :387-406
            const int64_t mlen = len < oend - op ? len : oend - op;
            warp_copy_match(dst, op, match, (int)mlen, offset, lane);
            op += mlen;
            if (op == oend) return (int)op;
            continue;
        }
        if (cpy > oend - LASTLITERALS) return -1;                    // :427-433
        warp_copy_match(dst, op, match, (int)len, offset, lane);
        op = cpy;
    }
}

// LZ4Codec.Decode post-processing (LZ4Codec.cs:104-115): len <= 0 -> 0 ; result <= 0 -> -1.
__device__ __forceinline__ int codec_decode_warp(const uint8_t* src, int n, uint8_t* dst, int cap) {
    if (n <= 0) return 0;
    int r = decode_block_warp(src, n, dst, cap);
    return r <= 0 ? -1 : r;
}

__global__ void __launch_bounds__(128)
decode_generic_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                      const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                      const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                      int32_t* __restrict__ outLen, int nBlocks,
                      const int32_t* __restrict__ workList /* may be null: identity */, int nWork) {
    const int w = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    if (w >= nWork) return;
    const int b = workList ? workList[w] : w;
    if (b < 0 || b >= nBlocks) return;
    int r = codec_decode_warp(srcBase + srcOff[b], srcLen[b], dstBase + dstOff[b], dstCap[b]);
    if (lane_id() == 0) outLen[b] = r;
}

// LZ4Codec.Decode(src, dst, dict) / LZ4Codec.PartialDecode over a batch: warp per block.
// dictOff/dictLen may be null (no dictionaries); partial != 0 selects PartialDecode semantics
// (dstCap[i] is then the target length).
__global__ void __launch_bounds__(128)
decode_general_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                      const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                      const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                      const uint8_t* __restrict__ dictBase, const int64_t* __restrict__ dictOff,
                      const int32_t* __restrict__ dictLen, int32_t* __restrict__ outLen, int nBlocks,
                      int partial) {
    const int b = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
    if (b >= nBlocks) return;
    const int n = srcLen[b];
    int r;
    if (n <= 0) r = 0;                                               // LZ4Codec.cs:129-130, 150-151
    else {
        const int dl = (dictBase && dictLen) ? dictLen[b] : 0;
        r = decode_block_warp_general(srcBase + srcOff[b], n, dstBase + dstOff[b], dstCap[b] < 0 ? 0 : dstCap[b],
                                      partial != 0, dl > 0 ? dictBase + dictOff[b] : nullptr, dl > 0 ? dl : 0);
        r = r <= 0 ? -1 : r;
    }
    if (lane_id() == 0) outLen[b] = r;
}

}  // namespace k4