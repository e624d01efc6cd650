// size_walk.cuh -- the decoded length of a raw LZ4 block from its token chain, one warp per block.
//
// The length is the sum of the literal runs plus matchlen + 4 of every match; offsets are never read.  For every
// block LZ4_decompress_safe accepts it equals the decoder's result; -1 where the chain runs past the end of the
// block (tests/test_frame_model.py's `walk` is the serial restatement).
//
// The chain is serial, but it is confluent: a walk started at an arbitrary byte soon lands on the true chain (the
// tile decoder's parse uses the same property, DESIGN 4.1).  So the warp covers the block in windows of 32
// segments of SW_SEG bytes, one segment per lane.  Lane t starts SW_WARM bytes before its segment (or at the
// window's exact entry, `carry`, when that is later), walks up to its segment and records its entry (the first
// token position inside the segment), its exit (the first position past it) and the output bytes between the two.
// Lane t is right iff entry[t] == exit[t-1]; wrong lanes re-walk from exit[t-1] until every link agrees (the first
// wrong lane is exact after one round, so a window takes at most 31 rounds).  A warp sum gives the window's
// output, and the exact exit of lane 31 is the next window's carry: the work is linear in the block's length.
// A speculative lane reads extension bytes only up to one segment past its own, so a long run of 0xFF costs only
// the exact lane that owns it.
//
// Plain C++ apart from the warp loop, so that tests/native/size_walk_check.cpp runs the same lanes and links on
// the host, lane by lane, against the serial walk.
#pragma once
#include <stdint.h>

#if !defined(K4_HD)
#if defined(__CUDACC__)
#define K4_HD __host__ __device__ __forceinline__
#else
#define K4_HD inline
#endif
#endif

#ifndef K4_SW_SEG
#define K4_SW_SEG 128       // bytes per lane (DESIGN 4.9: measured against 32 and 64)
#endif
#ifndef K4_SW_WARM
#define K4_SW_WARM 64       // warm-up bytes in front of a lane's segment
#endif

namespace k4 {

constexpr int SW_SEG = K4_SW_SEG, SW_WARM = K4_SW_WARM;

// the outcome of a sequence or of a lane
constexpr int SW_NEXT = 0;   // another sequence follows at *q (< n)
constexpr int SW_END = 1;    // the terminal literal run ends exactly at n: the chain is complete
constexpr int SW_FAIL = 2;   // the chain runs past the end: the walk is -1
constexpr int SW_CUT = 3;    // not known: a speculative walk stopped at its read limit or before its segment

// The sequence whose token is at p (0 <= p < n).  Extension bytes are read only below lim (<= n): a sequence that
// needs one at or beyond lim < n is SW_CUT.  *v = its output bytes (SW_NEXT, SW_END).
template <class LD8>
K4_HD int sw_seq(LD8 ld8, const int64_t n, const int64_t lim, int64_t p, int64_t* q, int64_t* v) {
    const uint32_t tok = ld8(p++);
    int64_t lit = tok >> 4;
    if (lit == 15) {
        uint32_t x;
        do {
            if (p >= lim) return p >= n ? SW_FAIL : SW_CUT;
            x = ld8(p++);
            lit += x;
        } while (x == 255);
    }
    p += lit;
    if (p == n) { *v = lit; return SW_END; }
    if (p + 2 > n) return SW_FAIL;
    p += 2;
    int64_t ml = tok & 15;
    if (ml == 15) {
        uint32_t x;
        do {
            if (p >= lim) return p >= n ? SW_FAIL : SW_CUT;
            x = ld8(p++);
            ml += x;
        } while (x == 255);
    }
    if (p >= n) return SW_FAIL;              // a chain that ends on a match has no terminal literal run
    *q = p;
    *v = lit + ml + 4;
    return SW_NEXT;
}

// One lane: walk from `start` (< n) up to the segment [a, b), then through it.  -> SW_NEXT with *e = entry,
// *x = exit, *o = output bytes of the sequences whose tokens lie in [*e, b); SW_END with the terminal run counted;
// SW_FAIL; SW_CUT (*e = -1 when the warm-up stopped).
template <class LD8>
K4_HD int sw_lane(LD8 ld8, const int64_t n, const int64_t start, const int64_t a, const int64_t b,
                  const int64_t lim, int64_t* e, int64_t* x, int64_t* o) {
    int64_t p = start, q = 0, v = 0, out = 0;
    *o = 0;
    while (p < a) {
        if (sw_seq(ld8, n, lim, p, &q, &v) != SW_NEXT) { *e = -1; *x = -1; return SW_CUT; }
        p = q;
    }
    *e = p;
    int r = SW_NEXT;
    while (p < b) {
        r = sw_seq(ld8, n, lim, p, &q, &v);
        if (r == SW_FAIL || r == SW_CUT) break;
        out += v;
        if (r == SW_END) break;
        p = q;
    }
    *x = p;
    *o = out;
    return r;
}

// Where lane t of the window at `base` starts, and how far it may read.  Lane 0 (base <= carry) starts exactly at
// carry and may read to the end; a lane whose warm-up would begin before carry starts there too, but like every
// other speculative lane reads at most one segment past its own, so that it never repeats lane 0's long runs.
K4_HD void sw_lane_start(const int64_t n, const int64_t base, const int64_t carry, const int t, const int seg,
                         const int warm, int64_t* a, int64_t* b, int64_t* start, int64_t* lim) {
    *a = base + (int64_t)t * seg;
    *b = *a + seg;
    *start = *a - warm > carry ? *a - warm : carry;
    *lim = t == 0 ? n : (*b + seg < n ? *b + seg : n);
}

// Lane t (> 0) is not yet known right: its predecessor (status ps, exit px) may continue the chain and t was not
// entered exactly where the predecessor left.
K4_HD bool sw_broken(const int t, const int64_t e, const int s, const int64_t px, const int ps) {
    return t > 0 && (ps != SW_NEXT || s == SW_CUT || e != px);
}

// the segment grid point at or below the carry: the next window's base
K4_HD int64_t sw_base(const int64_t carry, const int seg) { return carry / seg * seg; }

#if defined(__CUDACC__)
// The walk of s[0 .. n) by the whole warp (every lane calls it with the same block; every lane gets the result).
__device__ __forceinline__ int64_t sw_walk_warp(const uint8_t* __restrict__ s, const int64_t n, const int lane) {
    if (n <= 0) return -1;
    auto ld8 = [s](int64_t q) -> uint32_t { return __ldg(s + q); };
    constexpr unsigned ALL = 0xffffffffu;
    int64_t carry = 0, acc = 0;
    for (;;) {
        const int64_t base = sw_base(carry, SW_SEG);
        int64_t a, b, start, lim, e = -1, x = -1, o = 0;
        sw_lane_start(n, base, carry, lane, SW_SEG, SW_WARM, &a, &b, &start, &lim);
        int s = SW_CUT, live = 32;
        bool walk = a < n;                    // lanes past the end never matter: a lane before them ends the chain
        for (;;) {
            if (walk) s = sw_lane(ld8, n, start, a, b, lim, &e, &x, &o);
            const int64_t px = __shfl_up_sync(ALL, x, 1);
            const int ps = __shfl_up_sync(ALL, s, 1);
            const bool bad = sw_broken(lane, e, s, px, ps);
            const unsigned brk = __ballot_sync(ALL, bad);
            if (!brk) break;
            const int k = __ffs(brk) - 1;     // lanes < k are right
            if (__shfl_sync(ALL, ps, k) != SW_NEXT) { live = k; break; }   // lane k - 1 ends the chain
            // lane k re-walks exactly; the wrong lanes behind it re-walk from their predecessors' exits meanwhile
            walk = bad && lane >= k && ps == SW_NEXT;
            start = px;
            if (lane == k) lim = n;
        }
        int64_t sum = lane < live ? o : 0;
        for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(ALL, sum, d);
        acc += sum;
        const int sl = __shfl_sync(ALL, s, live - 1);
        if (sl != SW_NEXT) return sl == SW_END ? acc : -1;
        carry = __shfl_sync(ALL, x, 31);
    }
}

// k4lz4_decoded_size_batch: one warp per block.  outSize[i] = 0 for srcLen <= 0, else the walk, or -1 where the
// chain does not parse or its length exceeds 2^31 - 1.
__global__ void decoded_size_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                                    const int32_t* __restrict__ srcLen, int32_t* __restrict__ outSize, int n) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const int32_t L = srcLen[i];
    const int64_t w = L > 0 ? sw_walk_warp(srcBase + srcOff[i], L, lane) : 0;
    if (lane == 0) outSize[i] = (w < 0 || w > 0x7FFFFFFF) ? -1 : (int32_t)w;
}
#endif

}  // namespace k4
