// lane_copy.cuh -- per-lane copies of short runs inside shared memory in 4-byte words.
//
// Every lane of a warp owns one short run (a literal run or a match of at most LC_MAX bytes) at
// arbitrary byte alignment on both sides.  Copying it byte by byte costs one load and one store
// instruction (and one shared-memory wavefront each) per byte of the LONGEST run of the warp; the
// shared-memory pipe and the issue slots are what the tile decoder runs out of.  Here a lane copies
//     up to 3 head bytes until its destination is word aligned,
//     whole destination words, each built from two aligned source words by a funnel shift,
//     up to 3 tail bytes,
// all lanes in lock step (predicated), loads issued ahead of the stores that need them.
//
// A lane reads only aligned words that contain at least one byte of its source run -- plus, when the
// source is word aligned itself, the word right behind it (never used, but always inside the tile /
// stage padding) -- and writes only bytes of its own destination run, so runs of different lanes may
// touch at any byte boundary.  The memory accessors are a template parameter: the kernel passes
// ld.shared / st.shared wrappers, tests/native/lane_copy_check.cpp a byte array.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define K4_LC_HD __device__ __forceinline__
#else
#define K4_LC_HD inline
#endif

namespace k4 {

constexpr int LC_MAX = 32;               // longest run a lane copies on its own
constexpr int LC_WORDS = LC_MAX / 4;     // whole destination words of such a run: at most 8

K4_LC_HD uint32_t lc_funnel(uint32_t lo, uint32_t hi, uint32_t shBits) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, shBits);
#else
    return shBits ? (lo >> shBits) | (hi << (32u - shBits)) : lo;
#endif
}

// One lane's part.  `nwTop` is the largest whole-word count among the lanes that run in lock step
// (warp-uniform: __reduce_max_sync of lc_words(...)); len <= LC_MAX; source and destination do not overlap.
K4_LC_HD int lc_words(const uint32_t d, const int len) {
    const int h0 = (int)((4u - (d & 3u)) & 3u);
    const int h = h0 < len ? h0 : len;
    return (len - h) >> 2;
}

template <class M>
K4_LC_HD void lc_copy(M& m, const uint32_t d, const uint32_t s, const int len, const int nwTop) {
    const int h0 = (int)((4u - (d & 3u)) & 3u);
    const int h = h0 < len ? h0 : len;
    const int nw = (len - h) >> 2;
    const int t = len - h - 4 * nw;
    const uint32_t dw = d + (uint32_t)h, sw = s + (uint32_t)h;           // dw is word aligned when nw > 0
    const uint32_t sa = sw & ~3u, sh = (sw & 3u) * 8u;
    const uint32_t dt = dw + 4u * (uint32_t)nw, st = sw + 4u * (uint32_t)nw;
    // head and tail bytes: all loads, then all stores
    uint32_t hb0 = 0, hb1 = 0, hb2 = 0, tb0 = 0, tb1 = 0, tb2 = 0;
    if (h > 0) hb0 = m.ld8(s);
    if (h > 1) hb1 = m.ld8(s + 1u);
    if (h > 2) hb2 = m.ld8(s + 2u);
    if (t > 0) tb0 = m.ld8(st);
    if (t > 1) tb1 = m.ld8(st + 1u);
    if (t > 2) tb2 = m.ld8(st + 2u);
    uint32_t lo = nw > 0 ? m.ld32(sa) : 0u;
    if (h > 0) m.st8(d, hb0);
    if (h > 1) m.st8(d + 1u, hb1);
    if (h > 2) m.st8(d + 2u, hb2);
    if (t > 0) m.st8(dt, tb0);
    if (t > 1) m.st8(dt + 1u, tb1);
    if (t > 2) m.st8(dt + 2u, tb2);
    // whole words, four at a time
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int base = 0; base < LC_WORDS; base += 4) {
        if (base >= nwTop) break;
        uint32_t w[4];
#if defined(__CUDACC__)
#pragma unroll
#endif
        for (int j = 0; j < 4; j++) if (base + j < nw) w[j] = m.ld32(sa + 4u * (uint32_t)(base + j) + 4u);
#if defined(__CUDACC__)
#pragma unroll
#endif
        for (int j = 0; j < 4; j++) {
            if (base + j < nw) {
                m.st32(dw + 4u * (uint32_t)(base + j), lc_funnel(lo, w[j], sh));
                lo = w[j];
            }
        }
    }
}

}  // namespace k4
