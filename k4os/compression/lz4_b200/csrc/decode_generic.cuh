// decode_generic.cuh -- size-agnostic LZ4 block decoder: one warp per block, streams read and
// written in global memory.  It is the path for blocks that do not fit the shared-memory
// tile decoder (decode_tile.cuh), the warp-level engine behind unpickle, the dictionary and
// partial decoder, and the parser of the chained-streams call (decode_stream.cuh).
//
// Semantics = LZ4_decompress_safe as reached from LZ4Codec.Decode:
//   /root/reference/src/K4os.Compression.LZ4/Engine/x64/LL64.dec.cs:124-467 (generic loop,
//   endOnInputSize / full / noDict / lowPrefix = dst) and :469-477; every accept/reject test
//   is evaluated in the reference's order so that the returned value matches for malformed
//   input as well.  Control is warp-uniform: all lanes track (ip, op); the copies are
//   lane-parallel.  A match with offset 0 (accepted by the reference, content unspecified)
//   produces zero bytes.
//
// One engine, decode_block_warp, makes every test; where its writes go is a policy.  DirectOut
// writes each literal run and match copy at once; DeferOut (decode_stream.cuh) records the match
// copies whose source bytes are not final yet.
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

// The engine's writes made at once: a literal run, a match copy inside [dst - prefix, dst) and the block, and a
// match copy through the [dict | dst] window.
struct DirectOut {
    __device__ __forceinline__ void literals(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, int len,
                                             int lane) {
        warp_copy_in(d, s, len, lane);
    }
    __device__ __forceinline__ void match(uint8_t* dst, int64_t op, int64_t match, int len, int offset, int lane) {
        warp_copy_match(dst, op, match, len, offset, lane);
    }
    __device__ __forceinline__ void window(uint8_t* dst, int64_t op, int64_t match, int len, int offset,
                                           const uint8_t* __restrict__ dict, int dictSize, int lane) {
        warp_copy_match_window(dst, op, match, len, offset, dict, dictSize, lane);
    }
    __device__ __forceinline__ int done(int r) { return r; }
};

// Returns bytes written (>= 0) or a negative value on malformed input / insufficient room; every return passes
// through out.done.  With no history (prefix = 0, no dictionary, not partial) it is LZ4_decompress_safe.  The
// other forms: external dictionary (LZ4_decompress_safe_usingDict,
// LL64.dec.cs:523-546 -> forceExtDict :510-521; the prefix variants read the same bytes and reject
// the same offsets) and/or partial decoding (LZ4_decompress_safe_partial :548-556 with
// dstCapacity == targetOutputSize, LLxx.cs:29-39; paths :256-280, :301-307, :387-406), or prefix mode:
// `prefix` bytes of history lie directly in front of dst (LZ4_decompress_safe_withSmallPrefix /
// _withPrefix64k, LL64.dec.cs:479-498, as LZ4_decompress_safe_continue calls them :558-592): lowPrefix =
// dst - prefix, dictSize = 0.  The caller clamps prefix to 65535: every longer history is withPrefix64k, whose
// shortcut test (:213) no offset fails.  Without a dictionary no match reaches out.window.
template <class Out>
__device__ int decode_block_warp(Out&& out, const uint8_t* __restrict__ src, int n, uint8_t* __restrict__ dst,
                                 int outputSize, bool partial,
                                 const uint8_t* __restrict__ dict, int dictSize, int prefix = 0) {
    const int lane = lane_id();
    int64_t ip = 0, op = 0;
    const int64_t iend = n, oend = outputSize;
    const int64_t shortiend = iend - 16, shortoend = oend - 32;      // :152-153
    const bool checkOffset = dictSize < 65536;                       // :147
    const bool extDict = dict != nullptr && dictSize > 0;
    if (!extDict) dictSize = 0;
    const int64_t lowPrefix = extDict ? 0 : -(int64_t)prefix;        // relative to dst

    if (outputSize == 0) {                                           // :162-168
        if (partial) return out.done(0);
        return out.done((n == 1 && __ldg(src) == 0) ? 0 : -1);
    }
    if (n == 0) return out.done(-1);                                 // :172

    for (;;) {
        const uint32_t token = __ldg(src + ip); ip++;                // :177
        int64_t len = token >> 4;
        const bool shortcut = (len != 15) && (ip < shortiend) && (op <= shortoend);   // :191-193
        bool literalsDone = false;
        if (!shortcut) {
            if (len == 15) {                                         // :228-243, LL.tools.cs:165-193
                if (ip >= iend - 15) return out.done(-1);            // initial_error
                for (;;) {
                    uint32_t s = __ldg(src + ip); ip++;
                    len += s;
                    if (ip >= iend - 15) break;                      // loop_error: not fatal here
                    if (s != 255) break;
                }
            }
            int64_t cpy = op + len;                                  // :246
            if (cpy > oend - MFLIMIT || ip + len > iend - (2 + 1 + LASTLITERALS)) {
                if (partial) {                                       // :256-280
                    if (ip + len > iend - (2 + 1 + LASTLITERALS) && ip + len != iend) return out.done(-1);
                    if (cpy > oend) { cpy = oend; len = oend - op; }
                } else if (ip + len != iend || cpy > oend) return out.done(-1);   // :291-294
                out.literals(dst + op, src + ip, (int)len, lane);
                ip += len; op += len;
                if (!partial || cpy == oend || ip == iend) return out.done((int)op);   // :304-307, :454-457
                literalsDone = true;
            }
        }
        if (!literalsDone) {                                         // :196-200 / :311-314
            out.literals(dst + op, src + ip, (int)len, lane);
            ip += len; op += len;
        }

        const int offset = (int)__ldg(src + ip) | ((int)__ldg(src + ip + 1) << 8);   // :205 / :318
        ip += 2;
        const int64_t match = op - offset;
        len = token & 15;                                            // :204 / :323

        if (shortcut && len != 15 && offset >= 8 && match >= lowPrefix) {   // :211-220
            len += MINMATCH;
            out.match(dst, op, match, (int)len, offset, lane);
            op += len;
            continue;
        }
        if (len == 15) {                                             // :326-334
            for (;;) {
                uint32_t s = __ldg(src + ip); ip++;
                len += s;
                if (ip >= iend - LASTLITERALS + 1) return out.done(-1);   // any overrun is fatal
                if (s != 255) break;
            }
        }
        len += MINMATCH;                                             // :336
        if (checkOffset && match + dictSize < lowPrefix) return out.done(-1);   // :338
        if (match < lowPrefix) {
            if (!extDict) return out.done(-1);                       // (unreachable with checkOffset on)
            if (op + len > oend - LASTLITERALS) {                     // :343-347
                if (partial) len = (oend - op) < len ? (oend - op) : len;
                else return out.done(-1);
            }
            out.window(dst, op, match, (int)len, offset, dict, dictSize, lane);
            op += len;
            continue;
        }
        const int64_t cpy = op + len;                                // :383
        if (partial && cpy > oend - 12) {                            // :387-406
            const int64_t mlen = len < oend - op ? len : oend - op;
            out.match(dst, op, match, (int)mlen, offset, lane);
            op += mlen;
            if (op == oend) return out.done((int)op);
            continue;
        }
        if (cpy > oend - LASTLITERALS) return out.done(-1);          // :427-433
        out.match(dst, op, match, (int)len, offset, lane);
        op = cpy;                                                    // :450
    }
}

// LZ4Codec.Decode post-processing (LZ4Codec.cs:104-115): len <= 0 -> 0 ; result <= 0 -> -1.
__device__ __forceinline__ int codec_decode_warp(const uint8_t* src, int n, uint8_t* dst, int cap) {
    if (n <= 0) return 0;
    int r = decode_block_warp(DirectOut{}, src, n, dst, cap, false, nullptr, 0);
    return r <= 0 ? -1 : r;
}

// Block b of LZ4Codec.Decode(src, dst, dict) / LZ4Codec.PartialDecode over a batch (LZ4Codec.cs:129-130, 150-151):
// len <= 0 -> 0 ; result <= 0 -> -1.  A negative capacity decodes as 0; block b's dictionary is
// dictBase[dictOff[b] .. + dictLen[b]) when dictBase and dictLen are not null and dictLen[b] > 0, none otherwise.
__device__ __forceinline__ int codec_decode_general_warp(
        const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff, const int32_t* __restrict__ srcLen,
        uint8_t* __restrict__ dstBase, const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
        bool partial, const uint8_t* __restrict__ dictBase, const int64_t* __restrict__ dictOff,
        const int32_t* __restrict__ dictLen, int b) {
    const int n = srcLen[b];
    if (n <= 0) return 0;
    const int dl = (dictBase && dictLen) ? dictLen[b] : 0;
    const int r = decode_block_warp(DirectOut{}, srcBase + srcOff[b], n, dstBase + dstOff[b],
                                    dstCap[b] < 0 ? 0 : dstCap[b], partial,
                                    dl > 0 ? dictBase + dictOff[b] : nullptr, dl > 0 ? dl : 0);
    return r <= 0 ? -1 : r;
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
    const int r = codec_decode_general_warp(srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, partial != 0, dictBase,
                                            dictOff, dictLen, b);
    if (lane_id() == 0) outLen[b] = r;
}

}  // namespace k4
