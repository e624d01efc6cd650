// decode_tile.cuh -- the batched LZ4 block decoder for H100: ONE kernel, ONE CTA per block.
//
// A CTA (512 threads) owns one block.  Everything a block needs lives in shared memory: the
// compressed stream (pulled in by one TMA bulk copy), the 64 KiB output tile (left through one
// TMA bulk store) and a few KiB of bookkeeping; the compressed stream is read from HBM once, the
// raw block is written once, nothing else moves.
//
//   1. JUMP TABLE + SEGMENTED SPECULATIVE PARSE.  The token chain is the only serial part of LZ4
//      decoding.  First every thread computes, for four stream positions at a time, the distance to
//      the next token IF a token started there (parse_table.cuh; one byte per position, kept in the
//      still unused output tile).  Then the stream is cut into 80-byte segments, one lane each.  A
//      lane starts walking some hundred bytes BEFORE its segment at an arbitrary byte (LZ4 chains are
//      confluent: a walk started anywhere falls onto the true chain within a few sequences) -- a
//      hop is one byte load and an add --, notes the first position it reaches inside its segment
//      (entry) and the first one past it (exit), and counts the sequences and output bytes in
//      between.  Lane 0 is exact; lane t is right iff entry[t] == exit[t-1]; wrong lanes re-walk
//      from exit[t-1] until every link agrees.
//   2. BLOCK-WIDE EXCLUSIVE SCAN of the per-segment sequence counts and output sizes gives every
//      segment its first sequence index and output position; a second walk (same table) writes one 32-bit
//      descriptor (tokenPos | outPos << 16) per sequence into the still unused TAIL of the output
//      tile.  (A sequence produces >= 4 output bytes and its descriptor is 4 bytes, so the output
//      front never overtakes the descriptors of sequences that have not been decoded yet.)
//   3. STEPS of 512 consecutive sequences, one per thread: literals and every match whose source
//      lies entirely before the step's first output byte ("far") are copied at once, lane-parallel
//      for short runs, by the whole warp in 4-byte words for long ones.  The remaining "near"
//      matches (source reaches into the step's own output) are compacted into a sorted interval
//      list; a near match is copied as soon as no still-pending interval intersects its source
//      (binary search once, then a flag scan per round); rounds are separated by CTA barriers,
//      chains inside one warp resolve without a barrier.
//
// The fast path accepts a block only when every sequence satisfies the reference decoder's
// accept tests with room to spare (so the shortcut and the general path of the reference agree);
// anything else -- malformed input, decoded size > 64 KiB or > dstCap, offset 0, > 16384
// sequences, compressed size > 65535 -- is handed UNTOUCHED to the exact warp-per-block decoder
// (decode_generic.cuh), which reproduces LL64.dec.cs test by test.  Nothing reaches global memory
// before a block is known to be clean.
//
// Reference semantics: /root/reference/src/K4os.Compression.LZ4/Engine/x64/LL64.dec.cs:124-477,
// Engine/LL.tools.cs:165-193 (LZ4_readVLE), LZ4Codec.cs:104-115.
#pragma once
#include <mutex>

#include "common.cuh"
#include "decode_generic.cuh"
#include "parse_table.cuh"
#include "lane_copy.cuh"

namespace k4 {

constexpr int TILE_BYTES = 65536;
constexpr int TILE_PAD = 32;             // slack behind the tile: output shift (<= 15) + descriptor safety
#ifndef K4_DT_THREADS
#define K4_DT_THREADS 512
#endif
constexpr int DT_THREADS = K4_DT_THREADS;
constexpr int DT_WARPS = DT_THREADS / 32;
constexpr int DT_K = DT_THREADS;         // sequences per step
#ifndef K4_DT_WARM
#define K4_DT_WARM 256
#endif
constexpr int DT_WARM = K4_DT_WARM;      // speculative warm-up before the segment
#ifndef K4_DT_NEARSPIN
#define K4_DT_NEARSPIN 1
#endif
#ifndef K4_DT_LATEBAR
#define K4_DT_LATEBAR 1                    // the barrier that ends a step sits behind the NEXT step's literal copies
#endif
#ifndef K4_DT_LSHORT
#define K4_DT_LSHORT 32
#endif
constexpr int DT_LSHORT = K4_DT_LSHORT;  // runs up to this length are copied by the owning lane, longer ones by the warp
constexpr int STAGE_SMALL = 40 * 1024;   // two CTAs per SM
constexpr int STAGE_BIG = 65536 + 32;    // one CTA per SM: every block the tile path can take
constexpr int DT_NMAX = 16384;           // sequences per block the tile tail can describe
constexpr int DT_MAX_SRC = 65535;        // token positions are 16-bit
constexpr uint32_t DT_NONE = 0xFFFFFFFFu;
constexpr int SQ_LAST = 1, SQ_BAD = 2;

// counters (per device): [0] blocks decoded by the small-stage tile path, [1] by the big-stage
// tile path, [2] by the exact generic decoder, [3] parse repair walks
__device__ unsigned long long g_decode_stats[4];

// -DK4_DT_PROFILE (tools only, never the shipped build): per-phase cycle sums of thread 0 of every CTA
#ifdef K4_DT_PROFILE
__device__ unsigned long long g_decode_prof[32];
#define DT_PROF_DECL long long pfT = clock64();
#define DT_PROF(slot) do { if (threadIdx.x == 0) { const long long t_ = clock64(); atomicAdd(&g_decode_prof[slot], (unsigned long long)(t_ - pfT)); pfT = t_; } } while (0)
#define DT_PROF_COUNT(slot, v) do { if (threadIdx.x == 0) atomicAdd(&g_decode_prof[slot], (unsigned long long)(v)); } while (0)
#else
#define DT_PROF_DECL
#define DT_PROF(slot) do {} while (0)
#define DT_PROF_COUNT(slot, v) do {} while (0)
#endif

// Parse-lane granularity: every one of the 512 threads parses, so the serial chain per lane is as
// short as the stage allows (40 KiB / 512 = 80 bytes; 64 KiB / 512 = 128 bytes).
#ifndef K4_DT_SEG
#define K4_DT_SEG 80
#endif
template <int STAGE> struct TileCfg { static constexpr int SEG = STAGE <= 40 * 1024 ? K4_DT_SEG : 128; };
static_assert(K4_DT_SEG * K4_DT_THREADS >= 40 * 1024 && K4_DT_SEG <= 128, "one lane per segment of the small stage");

template <int STAGE>
struct TileSmem {
    alignas(128) uint8_t tile[TILE_BYTES + TILE_PAD];
    alignas(16) uint8_t stage[STAGE];
    uint32_t nearIv[DT_K];               // destFirst | destLast << 16, sorted
    uint16_t nearOff[DT_K];              // match distance of the entry
    uint8_t nearFlag[DT_K];              // 1 = still pending
    uint32_t warpA[DT_WARPS];
    uint32_t warpB[DT_WARPS];
    uint32_t nearCnt[2][DT_WARPS];       // per-warp near-match counts, double-buffered by step parity
    alignas(8) unsigned long long bar;
};
// While a block is parsed the output tile is empty: it holds the jump table (parse_table.cuh), one byte
// per stream position at the stage's own alignment; the descriptors later grow down from the tile's end.
// The per-segment exits of the parse live in nearIv (unused until the steps begin).
static_assert(sizeof(uint32_t) * DT_K >= sizeof(uint16_t) * DT_THREADS, "exit array fits nearIv");

static_assert(sizeof(TileSmem<STAGE_SMALL>) <= 115712, "two CTAs per SM: (228 KiB - 2 x 1 KiB) / 2");
static_assert(sizeof(TileSmem<STAGE_BIG>) <= 232448, "one CTA per SM: 227 KiB");

// ---- small PTX helpers ----------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(a), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(a), "r"(parity) : "memory");
    } while (!ok);
}
// global -> shared bulk copy (TMA), completion on an mbarrier; all three of dst/src/bytes 16-aligned
__device__ __forceinline__ void tma_load(void* sdst, const void* gsrc, int bytes, unsigned long long* bar) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(sdst);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(a), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(d), "l"(gsrc), "r"(bytes), "r"(a) : "memory");
}
// shared -> global bulk copy (TMA); returns when the shared source has been read
__device__ __forceinline__ void tma_store(void* gdst, const void* ssrc, int bytes) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(ssrc);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 :: "l"(gdst), "r"(s), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- shared memory by 32-bit shared-space address -----------------------------------------------
// Every hot access goes through these: with generic pointers into the dynamic shared array nvcc
// re-materialises the shared-window base (S2R SR_CgaCtaId, MOV, LEA, IADD) in front of EVERY
// predicated byte access (4-5 extra instructions per byte moved in the SASS).  A shared address
// computed once costs nothing.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t lds8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t lds16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void sts8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
// the compressed stream is read-only while it is parsed: no memory clobber (ordinary memory operations
// may move across these loads); still volatile, so they stay behind the barrier that publishes the stage
__device__ __forceinline__ uint32_t lds32_ro(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds8_ro(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }

// ---- sequence header ------------------------------------------------------------------------
// Header of the sequence whose token sits at stream position p; sStg = shared address of stream
// byte 0.  Two unaligned 4-byte windows -- token + first length byte, offset + first match-length
// byte -- decode the common case without a branch; only 255-chains take the byte loop.  ml includes
// MINMATCH and is 0 for the terminal (literal-only) sequence.  flags: SQ_LAST terminal, SQ_BAD the
// stream cannot be a clean block, SQ_EDGE (EXACT only) one of the reference's length-overrun tests
// would fire (LL.tools.cs:165-193, LL64.dec.cs:231-232,329-331).  Every access stays below stream
// position n + 8.
constexpr int SQ_EDGE = 4;
__device__ __forceinline__ uint32_t stage_load4(const uint32_t sStg, const int p) {
    const uint32_t a = sStg + (uint32_t)p;
    const uint32_t w0 = lds32_ro(a & ~3u), w1 = lds32_ro((a & ~3u) + 4u);
    return __funnelshift_r(w0, w1, (a & 3u) * 8u);
}
template <bool EXACT>
__device__ __forceinline__ void seq_header(const uint32_t sStg, const int p, const int n, int& lit,
                                           int& litPos, int& ml, int& off, int& next, uint32_t& flags) {
    // literal length: token nibble + up to three extension bytes straight from the first window
    const uint32_t w = stage_load4(sStg, p);
    const uint32_t tok = w & 0xFFu, e1 = (w >> 8) & 0xFFu, e2 = (w >> 16) & 0xFFu, e3 = w >> 24;
    const bool l15 = (tok >> 4) == 15u;
    const bool l2 = l15 && e1 == 255u, l3 = l2 && e2 == 255u;
    lit = (int)(tok >> 4) + (l15 ? (int)e1 : 0) + (l2 ? (int)e2 : 0) + (l3 ? (int)e3 : 0);
    int q = p + 1 + (l15 ? 1 : 0) + (l2 ? 1 : 0) + (l3 ? 1 : 0);
    if (l3 && e3 == 255u) {                                     // rare: >= 780 literals, byte loop
        while (q < n) { const uint32_t s = lds8_ro(sStg + q); q++; lit += (int)s; if (s != 255u) break; }
    }
    flags = 0;
    // LZ4_readVLE (LL.tools.cs:165-193): fatal if the first extension byte sits at >= iend-15; stops early
    // (the walker does not) if a 255 byte ends at >= iend-15.  With k bytes consumed at p+1 .. p+k = q-1
    // both reduce to q-1 >= n-15 (the last byte, which is not 255, may sit anywhere).
    if (EXACT && l15 && q - 1 >= n - 15) flags |= SQ_EDGE;
    litPos = q;
    const int litEnd = q + lit;
    const bool last = litEnd + 2 > n;                           // no room for an offset: terminal sequence
    // match length: second window at the offset (at p again for the terminal sequence: always in range)
    const uint32_t w2 = stage_load4(sStg, last ? p : litEnd);
    const uint32_t m1 = (w2 >> 16) & 0xFFu, m2 = w2 >> 24;
    const bool m15 = (tok & 15u) == 15u;
    const bool mm2 = m15 && m1 == 255u;
    int mlen = (int)(tok & 15u) + (m15 ? (int)m1 : 0) + (mm2 ? (int)m2 : 0);
    int q2 = litEnd + 2 + (m15 ? 1 : 0) + (mm2 ? 1 : 0);
    if (mm2 && m2 == 255u && !last) {                           // rare: match of >= 529 bytes, byte loop
        while (q2 < n) { const uint32_t s = lds8_ro(sStg + q2); q2++; mlen += (int)s; if (s != 255u) break; }
    }
    // any overrun is fatal in the reference (:326-334); the terminal sequence's match nibble is never read (:247-294)
    if (EXACT && m15 && !last && q2 >= n - 4) flags |= SQ_EDGE;
    off = last ? 0 : (int)(w2 & 0xFFFFu);
    ml = last ? 0 : mlen + MINMATCH;
    next = last ? n : (q2 < n ? q2 : n);
    flags |= last ? (uint32_t)(SQ_LAST | (litEnd != n ? SQ_BAD : 0)) : (q2 >= n ? (uint32_t)SQ_BAD : 0u);   // a block never ends with a match
}

// The walker's view of the same header: only where the next token sits and how many bytes the
// sequence produces (the parse runs tens of these hops back to back per lane; every instruction on
// that path costs latency).  Must agree with seq_header on `next` and lit + ml for every input.
__device__ __forceinline__ void seq_next(const uint32_t sStg, const int p, const int n, int& next, int& outb, uint32_t& bad) {
    const uint32_t w = stage_load4(sStg, p);
    const uint32_t tok = w & 0xFFu, e1 = (w >> 8) & 0xFFu, e2 = (w >> 16) & 0xFFu, e3 = w >> 24;
    const bool l15 = (tok >> 4) == 15u;
    const bool l2 = l15 && e1 == 255u, l3 = l2 && e2 == 255u;
    int lit = (int)(tok >> 4) + (l15 ? (int)e1 : 0) + (l2 ? (int)e2 : 0) + (l3 ? (int)e3 : 0);
    int q = p + 1 + (l15 ? 1 : 0) + (l2 ? 1 : 0) + (l3 ? 1 : 0);
    if (l3 && e3 == 255u) {
        while (q < n) { const uint32_t s = lds8_ro(sStg + q); q++; lit += (int)s; if (s != 255u) break; }
    }
    const int litEnd = q + lit;
    const bool last = litEnd + 2 > n;
    const uint32_t w2 = stage_load4(sStg, last ? p : litEnd);
    const uint32_t m1 = (w2 >> 16) & 0xFFu, m2 = w2 >> 24;
    const bool m15 = (tok & 15u) == 15u;
    const bool mm2 = m15 && m1 == 255u;
    int mlen = (int)(tok & 15u) + (m15 ? (int)m1 : 0) + (mm2 ? (int)m2 : 0);
    int q2 = litEnd + 2 + (m15 ? 1 : 0) + (mm2 ? 1 : 0);
    if (mm2 && m2 == 255u && !last) {
        while (q2 < n) { const uint32_t s = lds8_ro(sStg + q2); q2++; mlen += (int)s; if (s != 255u) break; }
    }
    next = last ? n : (q2 < n ? q2 : n);
    outb = lit + (last ? 0 : mlen + MINMATCH);
    bad = last ? (litEnd != n ? 1u : 0u) : (q2 >= n ? 1u : 0u);
}

// One hop of a walk through the jump table: sJ = shared address of table byte 0 (position 0).  The
// escape value sends the (rare) exotic sequence through the exact header code.
__device__ __forceinline__ int jt_hop(const uint32_t sJ, const uint32_t sStg, const int p, const int n) {
    const uint32_t j = lds8_ro(sJ + (uint32_t)p);
    if (j != JT_ESC) return p + (int)j;
    int nx, o; uint32_t b;
    seq_next(sStg, p, n, nx, o, b);
    return nx;
}
// Walks the sequences whose tokens sit in [p, end) and calls f(position, decoded size) for each; returns the
// first token position >= end and ORs `bad`.  The only serial dependency is table byte -> next position
// -> table byte: the loads that give a sequence's decoded size are issued BEHIND the next table load and
// consumed one hop later, so a hop costs one shared-memory round trip (the kernel keeps the LSU queue
// busy: a dependent load can take hundreds of cycles there).
template <class F>
__device__ __forceinline__ int jt_walk(const uint32_t sJ, const uint32_t sStg, int p, const int end, const int n,
                                       uint32_t& bad, F f) {
    uint32_t j = p < end ? lds8_ro(sJ + (uint32_t)p) : 0u;
    while (p < end) {
        int nx, o;
        uint32_t jn;
        if (j != JT_ESC) {
            nx = p + (int)j;
            const uint32_t tok = lds8_ro(sStg + (uint32_t)p), e1 = lds8_ro(sStg + (uint32_t)p + 1u);
            const uint32_t m1 = lds8_ro(sStg + (uint32_t)nx - 1u);
            jn = nx < end ? lds8_ro(sJ + (uint32_t)nx) : 0u;
            const uint32_t L = tok >> 4, M = tok & 15u;
            o = (int)(L + M + 4u + (L == 15u ? e1 : 0u) + (M == 15u ? m1 : 0u));      // == jt_outbytes(p, j)
        } else {
            uint32_t b;
            seq_next(sStg, p, n, nx, o, b);
            bad |= b;
            jn = nx < end ? lds8_ro(sJ + (uint32_t)nx) : 0u;
        }
        f(p, o);
        p = nx; j = jn;
    }
    return p;
}

// ---- copies inside shared memory (all addresses are 32-bit shared addresses) -------------------
// whole warp, uniform arguments, source and destination do not overlap: destination-aligned
// 4-byte words built from two aligned source words
__device__ __forceinline__ void warp_copy(uint32_t d, uint32_t s, int len, const int lane) {
    const int h0 = (int)((4u - (d & 3u)) & 3u);
    const int h = h0 < len ? h0 : len;
    if (lane < h) sts8(d + lane, lds8(s + lane));
    d += h; s += h; len -= h;
    const int nw = len >> 2;
    const uint32_t sh = (s & 3u) * 8u;
    const uint32_t sa = s & ~3u;
    for (int w = lane; w < nw; w += 32) {
        const uint32_t lo = lds32(sa + 4u * w);
        const uint32_t hi = sh ? lds32(sa + 4u * w + 4u) : 0u;
        sts32(d + 4u * w, __funnelshift_r(lo, hi, sh));
    }
    const int t = len & 3;
    if (lane < t) sts8(d + 4u * nw + lane, lds8(s + 4u * nw + lane));
}
// whole warp, LZ77 match of `len` bytes at d with distance off (uniform arguments)
__device__ __forceinline__ void warp_copy_match_smem(uint32_t d, const int off, const int len, const int lane) {
    if (off >= len) { warp_copy(d, d - off, len, lane); return; }
    if (off >= 160) {
        // overlapping but far enough apart: 128-byte slices, each one reads only bytes that earlier
        // slices (or the time before the copy) made final
        for (int i = 0; i < len; i += 128) {
            const int c = len - i < 128 ? len - i : 128;
            warp_copy(d + i, d + i - off, c, lane);
            __syncwarp();
        }
        return;
    }
    const uint32_t s = d - off;                 // periodic: every byte comes from the final window [d-off, d)
    for (int i = lane; i < len; i += 32) sts8(d + i, lds8(s + (i % off)));
}

// Lane-parallel copies of short runs, called by ALL lanes of a warp (len = 0 for lanes without work).
// The warp walks the runs in tiers of eight bytes; inside a tier every lane issues its (predicated)
// loads back to back and only then its stores, so a tier costs one shared-memory round trip instead of
// one per group of bytes (measured: the byte-group loop was the longest serial chain of a step).
// `ovl` lanes (LZ77 copy whose source runs into its destination) are done byte by byte afterwards.
#ifndef K4_DT_WORDCOPY
#define K4_DT_WORDCOPY 0                   // 1: lane_copy.cuh (4-byte words) instead of byte tiers
#endif
struct SmemOps {
    __device__ __forceinline__ uint32_t ld8(uint32_t a) const { return lds8(a); }
    __device__ __forceinline__ uint32_t ld32(uint32_t a) const { return lds32(a); }
    __device__ __forceinline__ void st8(uint32_t a, uint32_t v) const { sts8(a, v); }
    __device__ __forceinline__ void st32(uint32_t a, uint32_t v) const { sts32(a, v); }
};
__device__ __forceinline__ void lanes_copy(const uint32_t d, const uint32_t s, const int len, const bool ovl) {
    const int plain = ovl ? 0 : len;
#if K4_DT_WORDCOPY
    static_assert(DT_LSHORT <= LC_MAX, "lane copies are bounded by LC_MAX");
    SmemOps m;
    lc_copy(m, d, s, plain, __reduce_max_sync(FULL, lc_words(d, plain)));
    if (ovl) for (int j = 0; j < len; j++) sts8(d + j, lds8(s + j));
    return;
#endif
    const int top = __reduce_max_sync(FULL, plain);
    for (int base = 0; base < top; base += 8) {
        const int left = plain - base;
        uint32_t v[8];
#pragma unroll
        for (int j = 0; j < 8; j++) if (j < left) v[j] = lds8(s + base + j);
#pragma unroll
        for (int j = 0; j < 8; j++) if (j < left) sts8(d + base + j, v[j]);
    }
    if (ovl) for (int j = 0; j < len; j++) sts8(d + j, lds8(s + j));
}

// ---- copies from the stream's history (global memory in front of the block's destination) ---------
// Same shapes as lanes_copy / warp_copy, source in global memory: the history of a chained block is read
// where it lies (at most 64 KiB per stream, read-only during the call), never staged.
__device__ __forceinline__ void lanes_copy_hist(const uint32_t d, const uint8_t* __restrict__ s, const int len) {
    const int top = __reduce_max_sync(FULL, len);
    for (int base = 0; base < top; base += 8) {
        const int left = len - base;
        uint32_t v[8];
#pragma unroll
        for (int j = 0; j < 8; j++) if (j < left) v[j] = __ldg(s + base + j);
#pragma unroll
        for (int j = 0; j < 8; j++) if (j < left) sts8(d + base + j, v[j]);
    }
}
__device__ __forceinline__ void warp_copy_hist(const uint32_t d, const uint8_t* __restrict__ s, const int len, const int lane) {
    for (int i = lane; i < len; i += 32) sts8(d + (uint32_t)i, __ldg(s + i));
}

// ---- the tile decoder ---------------------------------------------------------------------------
// All DT_THREADS threads of the CTA call it with the same arguments.  Requires 1 <= n <= DT_MAX_SRC,
// (src & 15) + n + 16 <= STAGE, cap >= 1, 0 <= P <= 65535.  Returns the decoded size (> 0) after the
// bytes have been written to gdst, or -1 -- nothing written -- when the block has to go to the exact decoder.
// P is the length of the stream's history, gdst[-P .. 0) (prefix mode of LZ4_decompress_safe_continue,
// LL64.dec.cs:479-498: lowPrefix = dst - P; 65535 stands for every P >= 65535, withPrefix64k).  A match
// whose source starts before the block is split the way the reference splits an external-dictionary match
// (LL64.dec.cs:359-374): the history part is copied from global memory in the far phase, the remainder is
// a match at d' = off with source 0 and is scheduled like any other.  With P = 0 nothing changes.
template <int STAGE>
__device__ int tile_decode_block(TileSmem<STAGE>& S, const uint8_t* __restrict__ src, const int n,
                                 uint8_t* __restrict__ gdst, const int cap, const int P, uint32_t& barParity) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int shift = (int)(reinterpret_cast<uintptr_t>(src) & 15);
    uint8_t* const stg = S.stage + shift;                       // stg[p] == src[p]
    const uint32_t sStg = smem_u32(S.stage) + (uint32_t)shift;  // shared address of stream byte 0
    DT_PROF_DECL

    // ---- compressed block -> shared memory: aligned middle by TMA, ragged ends by plain loads ----
    {
        const int headRaw = (16 - shift) & 15;
        const int head = headRaw < n ? headRaw : n;
        const int mid = (n - head) & ~15;
        const int tail = n - head - mid;
        if (tid == 0 && mid > 0) {
            fence_async_smem();
            tma_load(stg + head, src + head, mid, &S.bar);
        }
        if (tid >= 32 && tid < 32 + head) stg[tid - 32] = src[tid - 32];
        if (tid >= 64 && tid < 64 + tail) stg[head + mid + tid - 64] = src[head + mid + tid - 64];
        if (mid > 0) { mbar_wait(&S.bar, barParity); barParity ^= 1u; }
    }
    __syncthreads();
    DT_PROF(0);

    // ---- 1a. jump table: distance to the next token for EVERY stream position (parse_table.cuh) --------
    const uint32_t sJ = smem_u32(S.tile) + (uint32_t)shift;     // J[p] sits at the stage's alignment: word k <-> word k
    {
        const uint32_t sStage0 = smem_u32(S.stage), sTile0 = smem_u32(S.tile);
        const int nWords = (shift + n + 3) >> 2;
        auto ld8 = [&](int q) { return lds8_ro(sStg + (uint32_t)q); };
        for (int k = tid; k < nWords; k += DT_THREADS) {
            const uint32_t w0 = lds32_ro(sStage0 + 4u * (uint32_t)k), w1 = lds32_ro(sStage0 + 4u * (uint32_t)k + 4u);
            sts32(sTile0 + 4u * (uint32_t)k, jt_word(w0, w1, 4 * k - shift, n, ld8));
        }
    }
    __syncthreads();
    DT_PROF(14);

    // ---- 1b. segmented speculative parse ---------------------------------------------------------------
    constexpr int SEG = TileCfg<STAGE>::SEG;
    const int NS = (n + SEG - 1) / SEG;                          // <= DT_THREADS by the caller's size test
    const int segStart = tid * SEG;
    const int segEnd = segStart + SEG < n ? segStart + SEG : n;
    const uint32_t sExit = smem_u32(S.nearIv);                    // u16 per segment, read across warps only
    uint32_t myEntry = 0, myExit = 0, myCnt = 0, myOut = 0, myBad = 0;
    // walks from p to the end of the lane's segment; counts what starts inside the segment
    auto walk = [&](int p) {
        uint32_t cnt = 0, ob = 0, bad = 0;
        while (p < segStart) p = jt_hop(sJ, sStg, p, n);         // warm-up: only the position matters
        myEntry = (uint32_t)p;                                   // first position >= segStart
        p = jt_walk(sJ, sStg, p, segEnd, n, bad, [&](int, int o) { cnt++; ob += (uint32_t)o; });
        myExit = (uint32_t)p; myCnt = cnt; myOut = ob; myBad = bad;
    };
    const bool parses = tid < NS;
    if (parses) { walk(segStart > DT_WARM ? segStart - DT_WARM : 0); sts16(sExit + 2u * tid, myExit); }
    // Lane t is right iff entry[t] == exit[t-1].  Inside a warp the exits travel by shuffle and a chain of
    // wrong lanes (a literal run that covers several whole segments makes every one of them wrong) is
    // repaired without leaving the warp; across warps through the exit array, one CTA round per hop.
    for (int round = 0;; round++) {
        if (round == 0) { __syncthreads(); DT_PROF(1); }         // later rounds: the barrier that ended the previous round
        bool walked = false;
        for (int it = 0; it < 34; it++) {
            uint32_t e = __shfl_up_sync(FULL, myExit, 1);
            if (lane == 0) e = tid > 0 && parses ? lds16(sExit + 2u * (tid - 1)) : 0u;
            const bool wrong = parses && tid >= 1 && myEntry != e;
            if (!__any_sync(FULL, wrong)) break;
            if (wrong) {
                walk((int)e);
#ifdef K4_DT_PROFILE
                atomicAdd(&g_decode_stats[3], 1ull);
#endif
            }
            walked = true;
        }
        if (walked && parses) sts16(sExit + 2u * tid, myExit);
        DT_PROF_COUNT(16, 1);
        if (!__syncthreads_or(walked)) break;                   // a full round without a single re-walk: all links agree
        if (round > NS + 1) return -1;                          // cannot happen: lane t is final after round t
    }
    DT_PROF(2);

    // ---- 2. block-wide exclusive scan of (sequence count, output bytes) per segment ----------------
    const uint32_t cIn = parses ? myCnt : 0u, oIn = parses ? myOut : 0u, badSeg = parses ? myBad : 0u;
    uint32_t cInc = cIn, oInc = oIn;
#pragma unroll
    for (int dlt = 1; dlt < 32; dlt <<= 1) {
        const uint32_t c2 = __shfl_up_sync(FULL, cInc, dlt), o2 = __shfl_up_sync(FULL, oInc, dlt);
        if (lane >= dlt) { cInc += c2; oInc += o2; }
    }
    if (lane == 31) { S.warpA[warp] = cInc; S.warpB[warp] = oInc; }
    const bool anyBad = __syncthreads_or(badSeg != 0);
    uint32_t wc = lane < DT_WARPS ? S.warpA[lane] : 0u, wo = lane < DT_WARPS ? S.warpB[lane] : 0u;
#pragma unroll
    for (int dlt = 1; dlt < DT_WARPS; dlt <<= 1) {
        const uint32_t c2 = __shfl_up_sync(FULL, wc, dlt), o2 = __shfl_up_sync(FULL, wo, dlt);
        if (lane >= dlt) { wc += c2; wo += o2; }
    }
    const int N = (int)__shfl_sync(FULL, wc, DT_WARPS - 1);     // sequences in the block
    const int O = (int)__shfl_sync(FULL, wo, DT_WARPS - 1);     // decoded size
    const uint32_t cBase = warp ? __shfl_sync(FULL, wc, warp - 1) : 0u;
    const uint32_t oBase = warp ? __shfl_sync(FULL, wo, warp - 1) : 0u;
    if (anyBad || N <= 0 || N > DT_NMAX || O <= 0 || O > TILE_BYTES || O > cap) return -1;
    DT_PROF(3);

    // descriptors: desc[i] = tokenPos | outPos << 16, in the tail of the tile
    const uint32_t sDesc = smem_u32(S.tile) + (uint32_t)(TILE_BYTES + TILE_PAD) - 4u * (uint32_t)N;   // &desc[0]
    // pass 2 walks the jump table again; it stays intact as long as the descriptors do not reach down to it
    const bool tableIntact = (uint32_t)(shift + n + 4) + 4u * (uint32_t)N <= (uint32_t)(TILE_BYTES + TILE_PAD);
    if (tid < NS) {
        int p = (int)myEntry;
        uint32_t idx = cBase + cInc - cIn;
        int op = (int)(oBase + oInc - oIn);
        if (tableIntact) {
            uint32_t b = 0;
            jt_walk(sJ, sStg, p, segEnd, n, b, [&](int q, int o) {
                sts32(sDesc + 4u * idx, (uint32_t)q | ((uint32_t)(op < 65535 ? op : 65535) << 16));
                idx++;
                op += o;
            });
        } else {
            while (p < segEnd) {
                int nx, o; uint32_t b;
                seq_next(sStg, p, n, nx, o, b);
                sts32(sDesc + 4u * idx, (uint32_t)p | ((uint32_t)(op < 65535 ? op : 65535) << 16));
                idx++;
                op += o;
                p = nx;
            }
        }
    }
    __syncthreads();
    DT_PROF(4);

    // ---- 3. steps of DT_K sequences ----------------------------------------------------------------
    const int tshift = (int)(reinterpret_cast<uintptr_t>(gdst) & 15);
    uint8_t* const T = S.tile + tshift;                          // T[op] is output byte op
    const uint32_t sT = smem_u32(S.tile) + (uint32_t)tshift;     // shared address of output byte 0
    const uint32_t sNearIv = smem_u32(S.nearIv), sNearOff = smem_u32(S.nearOff), sNearFlag = smem_u32(S.nearFlag);
    const int nsteps = (N + DT_K - 1) / DT_K;
    uint32_t dCur = tid < N ? lds32(sDesc + 4u * tid) : 0u;
    int Sr = 0;                                                  // output position where the step begins
    for (int r = 0; r < nsteps; r++) {
        const int i = r * DT_K + tid;
        const bool valid = i < N;
        const uint32_t dNext = i + DT_K < N ? lds32(sDesc + 4u * (i + DT_K)) : 0u;   // intact until the next step writes
        const int SrNext = (r + 1) * DT_K < N ? (int)(lds32(sDesc + 4u * ((r + 1) * DT_K)) >> 16) : O;

        // sequence header, with the reference's accept tests (conservative: see file header)
        int lit = 0, ml = 0, off = 0, litPos = 0, op = 0;
        bool bad = false;
        if (valid) {
            const int tp = (int)(dCur & 0xFFFFu);
            op = (int)(dCur >> 16);
            int nx; uint32_t fl;
            seq_header<true>(sStg, tp, n, lit, litPos, ml, off, nx, fl);
            bad = (fl & (SQ_EDGE | SQ_BAD)) != 0;
            if (i == N - 1) {                                    // terminal: LL64.dec.cs:247-294
                if (!(fl & SQ_LAST) || op + lit > cap) bad = true;
            } else {
                if ((fl & SQ_LAST) || litPos + lit > n - 8 || op + lit > cap - MFLIMIT) bad = true;   // :247
                if (off == 0 || off > op + lit + P || op + lit + ml > cap - LASTLITERALS) bad = true;   // :338, :427-433
            }
            if (bad) { lit = 0; ml = 0; }
        }
        DT_PROF(5);

        // history part of a match whose source starts before the block: hl bytes from gdst + d - off
        int d = op + lit;                                        // match destination
        const int hl = P > 0 && off > d ? (off - d < ml ? off - d : ml) : 0;
        const int hd = d;
        d += hl;                                                 // the remainder: at d = off, source 0
        ml -= hl;

        // classification of the match
        const int a = d - off;                                   // match source
        const int srcEnd = a + ml < d ? a + ml : d;              // bytes read from outside the match itself: [a, srcEnd)
        const bool nearM = ml > 0 && srcEnd > Sr;
        const bool farM = ml > 0 && !nearM;

        // literals, then far matches: short runs by the owning lane, long ones by the whole warp
        lanes_copy(sT + (uint32_t)op, sStg + (uint32_t)litPos, lit <= DT_LSHORT ? lit : 0, false);
        for (unsigned m = __ballot_sync(FULL, lit > DT_LSHORT); m; m &= m - 1) {
            const int l = __ffs(m) - 1;
            warp_copy(sT + (uint32_t)__shfl_sync(FULL, op, l), sStg + (uint32_t)__shfl_sync(FULL, litPos, l), __shfl_sync(FULL, lit, l), lane);
        }
        if (P > 0) {
            // history parts: nothing else of this step reads or writes [hd, hd + hl) before barrier #1, and a
            // near remainder that reads it (off < its length) runs behind that barrier
            lanes_copy_hist(sT + (uint32_t)hd, gdst + (hd - off), hl <= DT_LSHORT ? hl : 0);
            for (unsigned m = __ballot_sync(FULL, hl > DT_LSHORT); m; m &= m - 1) {
                const int l = __ffs(m) - 1;
                const int ld = __shfl_sync(FULL, hd, l);
                warp_copy_hist(sT + (uint32_t)ld, gdst + (ld - __shfl_sync(FULL, off, l)), __shfl_sync(FULL, hl, l), lane);
            }
        }
        DT_PROF(6);
#if K4_DT_LATEBAR
        // The previous step's near matches must be final before a far match may read them -- but not before this
        // step's headers and literals (stage -> bytes beyond everything earlier steps write): warps that are
        // done with the near phase early do those instead of waiting (the step-end barrier was 17 % of all
        // warp stall samples).  The near arrays are first touched behind barrier #1 below.
        if (r > 0) __syncthreads();
        DT_PROF(11);
#endif
        lanes_copy(sT + (uint32_t)d, sT + (uint32_t)a, farM && ml <= DT_LSHORT ? ml : 0, off < ml);
        for (unsigned m = __ballot_sync(FULL, farM && ml > DT_LSHORT); m; m &= m - 1) {
            const int l = __ffs(m) - 1;
            warp_copy_match_smem(sT + (uint32_t)__shfl_sync(FULL, d, l), __shfl_sync(FULL, off, l), __shfl_sync(FULL, ml, l), lane);
        }
        const unsigned nearBallot = __ballot_sync(FULL, nearM);
        if (lane == 0) S.nearCnt[r & 1][warp] = (uint32_t)__popc(nearBallot);
        DT_PROF(7);
        if (__syncthreads_or(bad)) return -1;                    // barrier #1: literals and far matches are final
        DT_PROF(8);
        DT_PROF_COUNT(17, 1);

        // near matches: sorted interval list, one thread per entry, rounds
        uint32_t nc = lane < DT_WARPS ? S.nearCnt[r & 1][lane] : 0u;
#pragma unroll
        for (int dlt = 1; dlt < DT_WARPS; dlt <<= 1) {
            const uint32_t c2 = __shfl_up_sync(FULL, nc, dlt);
            if (lane >= dlt) nc += c2;
        }
        const int nearTotal = (int)__shfl_sync(FULL, nc, DT_WARPS - 1);
        if (nearTotal > 0) {
            const int nearBase = warp ? (int)__shfl_sync(FULL, nc, warp - 1) : 0;   // all lanes: no shuffle under divergence
            if (nearM) {
                const int me = nearBase + __popc(nearBallot & ((1u << lane) - 1u));
                sts32(sNearIv + 4u * me, (uint32_t)d | ((uint32_t)(d + ml - 1) << 16));
                sts16(sNearOff + 2u * me, (uint32_t)off);
                sts8(sNearFlag + me, 1u);
            }
            __syncthreads();                                     // barrier #2: list complete
            // entry `tid` of the list is mine from here on
            const bool mine = tid < nearTotal;
            int nd = 0, nml = 0, noff = 1, lo = 0, hi = 0;
            if (mine) {
                const uint32_t iv = lds32(sNearIv + 4u * tid);
                nd = (int)(iv & 0xFFFFu); nml = (int)(iv >> 16) - nd + 1; noff = (int)lds16(sNearOff + 2u * tid);
                const int na = nd - noff;
                const int nSrcEnd = na + nml < nd ? na + nml : nd;
                // pending intervals before mine that intersect my source [na, nSrcEnd)
                int x = 0, y = tid;
                while (x < y) { const int mid = (x + y) >> 1; if ((int)(lds32(sNearIv + 4u * mid) >> 16) >= na) y = mid; else x = mid + 1; }
                lo = x; hi = lo;
                while (hi < tid && (int)(lds32(sNearIv + 4u * hi) & 0xFFFFu) < nSrcEnd) hi++;
            }
            bool pend = mine;
            DT_PROF(9);
            const bool warpHasWork = warp * 32 < nearTotal;
            for (int round = 0;; round++) {
                if (warpHasWork) {
                    bool progress;
                    do {
                        bool go = pend;
                        if (go) {
                            while (lo < hi && !lds8(sNearFlag + lo)) lo++;
                            go = lo >= hi;
                        }
                        __threadfence_block();                   // bytes behind the cleared flags
                        lanes_copy(sT + (uint32_t)nd, sT + (uint32_t)(nd - noff), go && nml <= DT_LSHORT ? nml : 0, noff < nml);
                        for (unsigned m = __ballot_sync(FULL, go && nml > DT_LSHORT); m; m &= m - 1) {
                            const int l = __ffs(m) - 1;
                            warp_copy_match_smem(sT + (uint32_t)__shfl_sync(FULL, nd, l), __shfl_sync(FULL, noff, l), __shfl_sync(FULL, nml, l), lane);
                        }
                        __threadfence_block();
                        __syncwarp();
                        if (go) { sts8(sNearFlag + tid, 0u); pend = false; }
                        __syncwarp();
                        progress = __any_sync(FULL, go);
                        DT_PROF_COUNT(19, 1);
                    } while (progress && __any_sync(FULL, pend));
                }
                DT_PROF(10);
#if K4_DT_NEARSPIN
                // no CTA barrier between rounds: a pending entry only ever waits for entries with a LOWER
                // index (same warp, lower lane, or an earlier warp), entry 0 waits for nothing, so polling
                // the flags terminates; one barrier after the loop publishes the step
                if (!warpHasWork || !__any_sync(FULL, pend)) break;
#ifndef K4_DT_SPINNS
#define K4_DT_SPINNS 40
#endif
                __nanosleep(K4_DT_SPINNS);
                DT_PROF_COUNT(18, 1);
                if (round > (1 << 20)) break;                     // (bounded for safety; never reached)
#else
                const bool more = __syncthreads_or(pend);
                DT_PROF(11);
                DT_PROF_COUNT(18, 1);
                if (!more) break;
                if (round > DT_K + 2) return -1;                 // cannot happen: each round retires the first pending match
#endif
            }
#if K4_DT_NEARSPIN && !K4_DT_LATEBAR
            __syncthreads();
            DT_PROF(11);
#endif
        }
        dCur = dNext;
        Sr = SrNext;
    }

    // ---- tile -> global: ragged head and tail by threads, the aligned middle by one TMA bulk store ----
    fence_async_smem();
    __syncthreads();
    DT_PROF(12);
    {
        const int hRaw = (16 - tshift) & 15;
        const int h = hRaw < O ? hRaw : O;
        const int bulk = (O - h) & ~15;
        if (tid < h) gdst[tid] = T[tid];
        const int tail = O - h - bulk;
        if (tid >= 32 && tid < 32 + tail) gdst[h + bulk + tid - 32] = T[h + bulk + tid - 32];
        if (tid == 0 && bulk > 0) tma_store(gdst + h, T + h, bulk);
    }
    DT_PROF(13);
    DT_PROF_COUNT(20, 1);
    return O;
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
// Work-list entry of the second and third launch: block index, bit 31 = "exact decoder only".
constexpr uint32_t WL_GENERIC = 0x80000000u;

struct DecodeLists {
    uint32_t* big;      // blocks for the big-stage tile kernel
    uint32_t* gen;      // blocks for the exact generic decoder
    uint32_t* counts;   // [0] = entries in big, [1] = entries in gen
};

__device__ __forceinline__ void wl_push(uint32_t* list, uint32_t* count, uint32_t b) {
    list[atomicAdd(count, 1u)] = b;
}

// LZ4Codec.Decode argument handling (LZ4Codec.cs:104-115, LL64.dec.cs:162-172); true when done
__device__ __forceinline__ bool decode_trivial(int n, int cap, int32_t* outLen) {
    if (n <= 0) { *outLen = 0; return true; }
    if (cap <= 0) { *outLen = -1; return true; }
    return false;
}

// LZ4ChainDecoder.Decode has no LZ4Codec post-processing: the engine's own special cases (LL64.dec.cs:162-172)
__device__ __forceinline__ int chain_trivial(int n, int cap, const uint8_t* src) {
    if (n <= 0 || cap < 0) return -1;
    return (n == 1 && src[0] == 0) ? 0 : -1;                       // cap == 0
}
// the block's history length (prefix mode); every value >= 65535 reads the same bytes (withPrefix64k)
__device__ __forceinline__ int chain_prefix(const int32_t* prefixLen, int b) {
    if (!prefixLen) return 0;
    const int p = prefixLen[b];
    return p < 65535 ? p : 65535;
}

// launch 1: one CTA per block, small stage, two CTAs per SM
__global__ void __launch_bounds__(DT_THREADS, 2)
decode_tile_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                   const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                   const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                   const int32_t* __restrict__ prefixLen, int32_t* __restrict__ outLen, DecodeLists wl) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    TileSmem<STAGE_SMALL>& S = *reinterpret_cast<TileSmem<STAGE_SMALL>*>(smem_raw);
    const int b = blockIdx.x;
    const int n = srcLen[b], cap = dstCap[b];
    const int P = chain_prefix(prefixLen, b);
    if (n <= 0 || cap <= 0 || P < 0) {
        if (threadIdx.x == 0) {
            if (!prefixLen) decode_trivial(n, cap, &outLen[b]);
            else outLen[b] = P < 0 ? -1 : chain_trivial(n, cap, srcBase + srcOff[b]);
        }
        return;
    }
    const uint8_t* src = srcBase + srcOff[b];
    const int shift = (int)(reinterpret_cast<uintptr_t>(src) & 15);
    if (n > DT_MAX_SRC) { if (threadIdx.x == 0) wl_push(wl.gen, &wl.counts[1], (uint32_t)b); return; }
    if (shift + n + 16 > STAGE_SMALL) { if (threadIdx.x == 0) wl_push(wl.big, &wl.counts[0], (uint32_t)b); return; }
    if (threadIdx.x == 0) mbar_init(&S.bar, 1);
    __syncthreads();
    uint32_t parity = 0;
    const int r = tile_decode_block<STAGE_SMALL>(S, src, n, dstBase + dstOff[b], cap, P, parity);
    if (threadIdx.x == 0) {
        if (r > 0) { outLen[b] = r; atomicAdd(&g_decode_stats[0], 1ull); }
        else wl_push(wl.gen, &wl.counts[1], (uint32_t)b);
    }
}

// launch 2: persistent, one CTA per SM, big stage: blocks whose compressed size needs it
__global__ void __launch_bounds__(DT_THREADS, 1)
decode_tile_big_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                       const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                       const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                       const int32_t* __restrict__ prefixLen, int32_t* __restrict__ outLen, DecodeLists wl) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    TileSmem<STAGE_BIG>& S = *reinterpret_cast<TileSmem<STAGE_BIG>*>(smem_raw);
    const uint32_t count = wl.counts[0];
    if (blockIdx.x >= count) return;
    if (threadIdx.x == 0) mbar_init(&S.bar, 1);
    __syncthreads();
    uint32_t parity = 0;
    for (uint32_t e = blockIdx.x; e < count; e += gridDim.x) {
        const int b = (int)wl.big[e];
        const uint8_t* src = srcBase + srcOff[b];
        const int r = tile_decode_block<STAGE_BIG>(S, src, srcLen[b], dstBase + dstOff[b], dstCap[b],
                                                   chain_prefix(prefixLen, b), parity);
        if (threadIdx.x == 0) {
            if (r > 0) { outLen[b] = r; atomicAdd(&g_decode_stats[1], 1ull); }
            else wl_push(wl.gen, &wl.counts[1], (uint32_t)b);
        }
        __syncthreads();            // the tile and the stage are reused
    }
}

// launch 3: persistent, warp per block: the exact decoder for everything the tile path declined
__global__ void __launch_bounds__(128)
decode_rest_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                   const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                   const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                   const int32_t* __restrict__ prefixLen, int32_t* __restrict__ outLen, DecodeLists wl) {
    const uint32_t count = wl.counts[1];
    const uint32_t nwarps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); e < count; e += nwarps) {
        const int b = (int)wl.gen[e];
        int r;
        if (!prefixLen) r = codec_decode_warp(srcBase + srcOff[b], srcLen[b], dstBase + dstOff[b], dstCap[b]);
        else {                                   // LZ4_decompress_safe_continue in prefix mode, raw engine result
            r = decode_block_warp_general(srcBase + srcOff[b], srcLen[b], dstBase + dstOff[b], dstCap[b], false,
                                          nullptr, 0, chain_prefix(prefixLen, b));
            r = r < 0 ? -1 : r;
        }
        if (lane_id() == 0) { outLen[b] = r; atomicAdd(&g_decode_stats[2], 1ull); }
    }
}

// ------------------------------------------------------------------------------------------------
// launcher (host)
// ------------------------------------------------------------------------------------------------
// Enqueues the decode of n blocks on `st` (current device).  prefixLen (device array, may be null:
// independent blocks) gives each block's history length, the bytes in front of its destination; with it the
// results are those of LZ4_decompress_safe_continue in prefix mode (bytes decoded or -1).  On success
// DECODE_LAUNCHES kernels were launched.  The work lists come from `pool`, a private stream-ordered
// pool of the current device (the process-wide default pool is never touched); `sms` is its SM count.  The
// tile kernels must have been granted their dynamic shared memory (sizeof(TileSmem<...>)).
constexpr int DECODE_LAUNCHES = 3;
inline cudaError_t decode_launch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                 uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                                 const int32_t* prefixLen, int32_t* outLen, int n, cudaStream_t st,
                                 cudaMemPool_t pool, int sms) {
    uint32_t* scratch = nullptr;
    cudaError_t e = cudaMallocFromPoolAsync((void**)&scratch, ((size_t)2 * n + 4) * sizeof(uint32_t), pool, st);
    if (e != cudaSuccess) return e;
    DecodeLists wl;
    wl.counts = scratch;
    wl.big = scratch + 4;
    wl.gen = scratch + 4 + n;
    e = cudaMemsetAsync(wl.counts, 0, 4 * sizeof(uint32_t), st);
    if (e == cudaSuccess) {
        decode_tile_kernel<<<n, DT_THREADS, sizeof(TileSmem<STAGE_SMALL>), st>>>(
            srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, prefixLen, outLen, wl);
        const int gridBig = n < sms ? n : sms;
        decode_tile_big_kernel<<<gridBig, DT_THREADS, sizeof(TileSmem<STAGE_BIG>), st>>>(
            srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, prefixLen, outLen, wl);
        const int want = (n + 3) / 4;
        const int gridRest = want < sms * 8 ? want : sms * 8;
        decode_rest_kernel<<<gridRest, 128, 0, st>>>(srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, prefixLen,
                                                      outLen, wl);
        e = cudaGetLastError();
    }
    cudaFreeAsync(scratch, st);
    return e;
}

}  // namespace k4
