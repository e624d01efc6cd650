// encode_chain.cuh -- bit-exact chained (linked-block) LZ4 L00_FAST encoder: one block of each of many
// streams per launch, one warp per block.
//
// Block i of a call is what LZ4_compress_fast_continue(state, src, dst, n, cap, 1) returns when the stream's
// history lies contiguously in front of `src` (the withPrefix64k case, which the reference's ring buffer always
// sets up: LZ4EncoderBase.cs:90-97 with LZ4_saveDict).  That is LZ4_compress_generic with
//   byU32 table (4 096 slots of absolute indices, hash5), limitedOutput, withPrefix64k, dictSmall or
//   noDictIssue (LL64.fast.cs:582-667; upstream orig/lib/lz4.c:851-1240, 1545-1637).
// With H4 = true it is the 32-bit engine's instead (LZ4Codec.Enforce32: LL32.fast.cs, whose only difference is
// hash4 over 4 bytes for the byU32 table, LL32.tools.cs:143-150).  Both engines keep the same state record, so a
// stream may alternate between them.
// The table is the caller's state record (K4LZ4_CHAIN_STATE_BYTES) in global memory, accessed through L2
// (.cg) like the global-table warps of encode_tile.cuh; it is never zeroed.
//
// The match search is encode_spec_warp's (encode_tile.cuh): 32 consecutive probes of a search run at once,
// `__match_any_sync` on the hash substitutes the nearest earlier lane's store, the first hitting lane wins
// and lanes up to it commit their stores.  What differs:
//   * the hash (hash5 over 8 bytes or, with H4, hash4 over 4 bytes, 12 bits) and the slots (absolute index = currentOffset-based, no tag);
//   * an index below startIndex lies in the history at src - (startIndex - index);
//   * the accept tests: index + 65535 >= current, and under dictSmall index >= startIndex - dictSize
//     (lz4.c:1001-1006, 1187-1188);
//   * the catch-up runs down to src - dictSize (lowLimit, lz4.c:907,1019), into the history;
//   * the state update (dictSize += n, currentOffset += n before the search, lz4.c:909-919) and the
//     renormalisation near 2 GiB (LZ4_renormDictT, lz4.c:1545-1562).
// The history a block may read is min(state.dictSize, prefixLen) bytes, and never more than 65 535 of them.
//
// The search itself (chain_search_warp) reads positions below 0 through a window: PrefixWindow here, whose
// history lies directly in front of `src`, and ExtWindow (encode_dict.cuh), whose dictionary is a buffer of its own.
#pragma once
#include "common.cuh"
#include "encode_generic.cuh"
#include "encode_tile.cuh"

namespace k4 {

// LZ4_stream_t_internal's hash table, currentOffset and dictSize (orig/lib/lz4.h:596-603) in a fixed layout
struct ChainState {
    uint32_t table[4096];
    uint32_t currentOffset;
    uint32_t dictSize;
    uint32_t reserved[2];
};
static_assert(sizeof(ChainState) == 16400, "K4LZ4_CHAIN_STATE_BYTES");

#ifndef K4_ENC_CHAIN_WARPS
#define K4_ENC_CHAIN_WARPS 32   // resident one-warp CTAs per SM (the hardware limit; the register budget allows it)
#endif
constexpr int ENC_CHAIN_WARPS = K4_ENC_CHAIN_WARPS;

// Reads in the prefix layout: position p < 0 is src[p], the `d` bytes of history directly in front of the source.
// The catch-up's byte compare (same8) and its floor (floor/above) are window members rather than expressions over
// rd8 and an int: a compare of the two bytes widened to uint32_t, or a floor hoisted into an int, changes the
// chained kernels' SASS.  So same8 compares the bytes as uint8_t, and floor is an empty tag that keeps -d in the test.
struct PrefixWindow {
    uint32_t d;
    struct Floor {};
    __device__ __forceinline__ uint32_t rd8(const uint8_t* __restrict__ src, int p) const {
        return (uint32_t)__ldg(src + p);
    }
    __device__ __forceinline__ uint32_t rd32(const uint8_t* __restrict__ src, int p) const { return ldg_u32u(src + p); }
    __device__ __forceinline__ bool same8(const uint8_t* __restrict__ src, int a, int b) const {
        return __ldg(src + a) == __ldg(src + b);
    }
    __device__ __forceinline__ Floor floor(int) const { return {}; }
    __device__ __forceinline__ bool above(int x, Floor) const { return x > -(int)d; }         // lowLimit, :907
};

// The search of one block, from position 0 through the last literals: the table's slots hold absolute indices,
// position 0 is `startIndex`, and the window `w` reads the `d` bytes of history below it.  Under dictSmall no index
// below startIndex - d is accepted.  Returns the engine's value: bytes written, or 0 when a limitedOutput check fails.
template <bool H4, class W>
__device__ __forceinline__ int chain_search_warp(const W w, const uint8_t* __restrict__ src, const uint32_t n,
                                                 const uint32_t startIndex, const uint32_t d, const bool dictSmall,
                                                 uint32_t* table, uint8_t* __restrict__ dst, const int cap) {
    const int lane = lane_id();
    const uint32_t prefixIdxLimit = startIndex - d;
    // a candidate index passes the reference's tests (and lies below the probe, as every valid state's do)
    auto accept = [&](uint32_t idx, uint32_t cur) {
        return idx < cur && !(dictSmall && idx < prefixIdxLimit) && !(idx + (uint32_t)MAX_DISTANCE < cur);
    };
#define RD32(p) w.rd32(src, (int)(p))
#define RD8(p) w.rd8(src, (int)(p))
#define HASH(p) (H4 ? hash4(ldg_u32u(src + (p)), 12) : hash5(ldg_u64u(src + (p)), 12))
    const int64_t olimit = cap;                                               // limitedOutput, always
    uint32_t ip = 0, anchor = 0, op = 0;

    if (n >= (uint32_t)MINLENGTH) {
        const uint32_t mfl1 = n - MFLIMIT + 1, mlim = n - LASTLITERALS;
        if (lane == 0) __stcg(table + HASH(0), startIndex);                   // :924
        __syncwarp();
        ip = 1;
        bool post = false;              // lane 0 of the next batch is the post-match probe at ip
        uint32_t q0 = 0;                // first search-probe index of the next batch
        uint32_t base = 1;              // position of search probe 0 of the current run
        for (;;) {
            uint32_t h2 = 0xFFFFFFFFu;
            if (post) h2 = HASH(ip - 2);                                      // put(ip-2), :1146
            const bool isPost = post && lane == 0;
            const uint32_t q = q0 + (uint32_t)lane - (post ? 1u : 0u);
            const uint32_t pos = isPost ? ip : base + probe_advance(q);
            const bool valid = isPost || (base + probe_advance(q + 1) <= mfl1);   // :969
            uint32_t v, h;
            if constexpr (H4) {                                               // one word: all the compare needs
                v = valid ? ldg_u32u(src + pos) : 0u;
                h = valid ? hash4(v, 12) : (0x10000u + (uint32_t)lane);
            } else {
                const uint64_t v64 = valid ? ldg_u64u(src + pos) : 0ull;
                v = (uint32_t)v64;
                h = valid ? hash5(v64, 12) : (0x10000u + (uint32_t)lane);
            }
            uint32_t cand = valid ? __ldcg(table + h) : 0u;
            if (h == h2) cand = startIndex + ip - 2;                          // sees the put(ip-2)
            const unsigned peers = __match_any_sync(FULL, h);
            const unsigned earlier = peers & ((1u << lane) - 1u);
            const int fromLane = earlier ? 31 - __clz(earlier) : lane;
            const uint32_t fwdPos = __shfl_sync(FULL, pos, fromLane);
            if (earlier) cand = startIndex + fwdPos;                          // sees the nearest earlier store
            const uint32_t cur = startIndex + pos;
            bool hit = false;
            if (valid && accept(cand, cur)) hit = RD32(cand - startIndex) == v;   // :1009, :1189
            const unsigned hits = __ballot_sync(FULL, hit);
            const unsigned ends = __ballot_sync(FULL, !valid);
            const int f = hits ? __ffs(hits) - 1 : 32;
            const int e = ends ? __ffs(ends) - 1 : 32;
            {   // commit the slot stores of the probes that ran (0..f, or 0..e-1 when the search ran into the
                // end first) in serial order: last writer per hash wins.  Unlike an independent block's, this
                // table outlives the block, so the stores before the end count too.
                const int last = e < f ? e - 1 : f;
                const unsigned upto = (last >= 31) ? 0xffffffffu : ((1u << (last + 1)) - 1u);
                const unsigned later = peers & ~((2u << lane) - 1u) & upto;
                const bool doStore = valid && ((1u << lane) & upto) && !(lane < 31 ? later : 0u);
                if (post) {
                    const unsigned same2 = __ballot_sync(FULL, valid && h == h2) & upto;
                    if (lane == 0 && !same2) __stcg(table + h2, startIndex + ip - 2);
                }
                if (doStore) __stcg(table + h, cur);
                __syncwarp();
            }
            if (e < f) break;                                                 // ran into the end: last literals
            if (f == 32) {
                if (post) { post = false; base = ip + 1; q0 = 31; }
                else q0 += 32;
                continue;
            }
            const bool zeroLit = post && f == 0;
            int m = (int)(__shfl_sync(FULL, cand, f) - startIndex);           // may be < 0: in the history
            ip = __shfl_sync(FULL, pos, f);
            const uint32_t a0h = ip + MINMATCH;
            const int b0h = m + MINMATCH;
            uint32_t x1 = 0u;
            {
                const uint32_t a = a0h + 4u * lane;
                if (lane < 8 && (int)mlim - (int)a > 0) x1 = RD32(a) ^ RD32(b0h + 4 * lane);
            }
            uint32_t caught = 0;
            if (!zeroLit) {                                                   // catch-up down to lowLimit, :1019
                const auto low = w.floor(m);
                for (int width = 8;; width = 32) {
                    const bool part = lane < width;
                    const bool ok = !part || ((ip > anchor + lane) && w.above(m - lane, low) &&
                                              w.same8(src, ip - 1 - lane, m - 1 - lane));
                    const unsigned bad = __ballot_sync(FULL, !ok);
                    const int c = bad ? __ffs(bad) - 1 : width;
                    ip -= c; m -= c; caught += (uint32_t)c;
                    if (bad) break;
                }
            }
            const uint32_t lit = ip - anchor;
            if (!zeroLit && (int64_t)op + 1 + lit + 8 + lit / 255 > olimit) return 0;   // :1024-1027
            uint32_t mc = caught;
            {   // LZ4_count(ip+4, m+4, matchlimit) over one contiguous window, 4 bytes per lane
                uint32_t a0 = a0h;
                int b0 = b0h;
                for (int width = 8;; width = 32) {
                    const uint32_t a = a0 + 4u * lane;
                    const int bb = b0 + 4 * lane;
                    const bool part = lane < width;
                    const int room = (int)mlim - (int)a;
                    const uint32_t x = width == 8 ? x1 : ((part && room > 0) ? (RD32(a) ^ RD32(bb)) : 0u);
                    int eq = x ? ((__ffs(x) - 1) >> 3) : 4;
                    if (eq > room) eq = room < 0 ? 0 : room;
                    if (!part) eq = 4;
                    const unsigned stop = __ballot_sync(FULL, eq < 4);
                    if (stop) {
                        const int s = __ffs(stop) - 1;
                        mc += 4u * s + (uint32_t)__shfl_sync(FULL, eq, s);
                        break;
                    }
                    mc += 4u * width; a0 += 4u * width; b0 += 4 * width;
                }
            }
            const uint32_t hdr = run_header_size(lit);
            const uint32_t afterOff = op + hdr + lit + 2;
            if ((int64_t)afterOff + 6 + (mc + 240) / 255 > olimit) return 0;   // :1097-1121
            {
                const uint32_t mlTok = mc >= 15 ? 15u : mc;
                const uint32_t off = (uint32_t)((int)ip - m);
                if (lane == 0) {
                    if (lit >= 15) {
                        uint32_t o = op, rest = lit - 15;
                        dst[o++] = (uint8_t)(0xF0 | mlTok);
                        for (; rest >= 255; rest -= 255) dst[o++] = 255;
                        dst[o] = (uint8_t)rest;
                    } else dst[op] = (uint8_t)((lit << 4) | mlTok);
                    dst[afterOff - 2] = (uint8_t)off;
                    dst[afterOff - 1] = (uint8_t)(off >> 8);
                }
                for (uint32_t i = lane; i < lit; i += 32) dst[op + hdr + i] = (uint8_t)RD8(anchor + i);
                op = afterOff;
                if (mc >= 15) {
                    const uint32_t rest = mc - 15, nff = rest / 255;
                    for (uint32_t i = lane; i < nff; i += 32) dst[op + i] = 0xFF;
                    if (lane == 0) dst[op + nff] = (uint8_t)(rest % 255);
                    op += nff + 1;
                }
            }
            ip += mc + MINMATCH;
            anchor = ip;                                                      // :1140
            if (ip >= mfl1) break;                                            // :1143
            post = true; q0 = 0; base = ip + 1;                               // :1146-1200 ride with the next batch
        }
    }
    {   // last literals, :1204-1231
        const uint32_t run = n - anchor;
        if ((int64_t)op + run + 1 + (run + 255 - 15) / 255 > olimit) return 0;
        const uint32_t hdr = run_header_size(run);
        if (lane == 0) write_run_header(dst, op, run);
        op += hdr;
        for (uint32_t i = lane; i < run; i += 32) dst[op + i] = (uint8_t)RD8(anchor + i);
        op += run;
        return (int)op;
    }
#undef RD32
#undef RD8
#undef HASH
}

// Returns the engine's value: bytes written, or 0 when a limitedOutput check fails (the state has then
// advanced as far as upstream's has).  `P` is the caller's prefixLen (>= 0).  H4: hash4 (the 32-bit engine).
template <bool H4>
__device__ int encode_chain_warp(const uint8_t* __restrict__ src, const uint32_t n, const uint32_t P,
                                 uint8_t* __restrict__ dst, const int cap, ChainState* st) {
    const int lane = lane_id();
    uint32_t* const table = st->table;
    uint32_t startIndex = __ldcg(&st->currentOffset), dsz = __ldcg(&st->dictSize);
    if (startIndex + n > 0x80000000u) {                                       // LZ4_renormDictT
        const uint32_t delta = startIndex - 65536u;
        for (int i = lane; i < 4096; i += 32) {
            const uint32_t t = __ldcg(table + i);
            __stcg(table + i, t < delta ? 0u : t - delta);
        }
        startIndex = 65536u;
        if (dsz > 65536u) dsz = 65536u;
    }
    if (n > (uint32_t)MAX_INPUT_SIZE) {                                       // lz4.c: before any state update
        if (lane == 0) { __stcg(&st->currentOffset, startIndex); __stcg(&st->dictSize, dsz); }
        __syncwarp();
        return 0;
    }
    const uint32_t d = dsz < P ? dsz : P;                                     // LZ4_saveDict's clamp
    const bool dictSmall = d < 65536u && d < startIndex;                      // lz4.c:1601
    if (lane == 0) { __stcg(&st->currentOffset, startIndex + n); __stcg(&st->dictSize, d + n); }
    return chain_search_warp<H4>(PrefixWindow{d}, src, n, startIndex, d, dictSmall, table, dst, cap);
}

// Persistent: one-warp CTAs pull blocks from a device counter.  Block b's result: 0 for n == 0 and -2
// (K4LZ4_R_DELEGATE) for level >= 3, both without touching the state; -1 for a negative prefix length or a
// state record not 16-aligned (state untouched) and where the engine returns 0 (state advanced); otherwise
// the bytes written.  H4: the 32-bit engine (k4lz4_*_x32).
template <bool H4>
__global__ void __launch_bounds__(32, ENC_CHAIN_WARPS)
encode_chain_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                    const int32_t* __restrict__ srcLen, const int32_t* __restrict__ prefixLen,
                    uint8_t* __restrict__ dstBase, const int64_t* __restrict__ dstOff,
                    const int32_t* __restrict__ dstCap, uint8_t* __restrict__ stateBase,
                    const int64_t* __restrict__ stateOff, int32_t* __restrict__ outLen, int nBlocks, int level,
                    uint32_t* __restrict__ nextBlock) {
    const int lane = lane_id();
    for (;;) {
        int b = 0;
        if (lane == 0) b = (int)atomicAdd(nextBlock, 1u);
        b = __shfl_sync(FULL, b, 0);
        if (b >= nBlocks) return;
        const int n = srcLen[b];
        if (n <= 0) { if (lane == 0) outLen[b] = 0; continue; }
        if (level >= 3) { if (lane == 0) outLen[b] = -2; continue; }
        const int P = prefixLen[b];
        uint8_t* const sp = stateBase + stateOff[b];
        if (P < 0 || (reinterpret_cast<uintptr_t>(sp) & 15)) { if (lane == 0) outLen[b] = -1; continue; }
        const int r = encode_chain_warp<H4>(srcBase + srcOff[b], (uint32_t)n, (uint32_t)P, dstBase + dstOff[b],
                                        dstCap[b], reinterpret_cast<ChainState*>(sp));
        if (lane == 0) {
            outLen[b] = r <= 0 ? -1 : r;
            atomicAdd(&g_encode_stats[3], 1ull);
        }
        __syncwarp();
    }
}

}  // namespace k4
