// encode_tile.cuh -- bit-exact LZ4 L00_FAST encoder for blocks below the 64 KiB table limit
// (n < 65 547: the reference's byU16 case, LL64.fast.cs:526,548), one warp per block.  The block is
// read where it lies, from global memory through L1.
//
// The reference's match search is a serial chain per probe (hash -> slot load -> slot store ->
// 4-byte compare, LL64.fast.cs:158-234).  Inside one search run the probe POSITIONS do not depend on
// the data (step = searchMatchNb++ >> 6, :159-170), only the table contents do -- and the only table
// writes between two probes of a run are the run's own earlier probes.  So a warp evaluates 32
// consecutive probes at once: every lane hashes its position, loads the slot, and `__match_any_sync`
// on the hash substitutes the position of the nearest earlier lane with the same hash (= the store
// the serial code would have done in between).  The first hitting lane wins; lanes up to it commit
// their slot stores (last writer per hash), later lanes are discarded -- exactly the serial history.
// The probe right after a match (put ip-2, test ip, LL64.fast.cs:394-466) rides as lane 0 of the
// next batch.  Common-prefix counting and the backward catch-up are lane-parallel.  The hash table
// is either 16 KiB of u16 slots in shared memory (the shared-memory warps and the pickler) or 32 KiB
// of 32-bit tagged slots in an L2-resident global workspace (the global-table warps, see GTAB below).
//
// Reference: /root/reference/src/K4os.Compression.LZ4/Engine/x64/LL64.fast.cs:35-576,
// Engine/LL.tools.cs:38-51, Engine/x64/LL64.tools.cs:87-133; step numbers = SURVEY.md App. A.
#pragma once
#include "common.cuh"
#include "encode_generic.cuh"

namespace k4 {

// K4_ENC_WIN (tools/build_variant.py): lanes of the FIRST batch of a search run in the persistent encoder (0 or
// 32: all 32).  Only lanes below it hash, load a slot and load candidate bytes; when none of them hits, their slot
// stores are committed and the run goes on 32 lanes wide.  Most runs hit within a few probes, so the scattered
// loads of the lanes behind the hit (discarded anyway) are mostly not issued, at the price of one more batch for
// the longer runs.
#ifndef K4_ENC_WIN
#define K4_ENC_WIN 16
#endif
static_assert(K4_ENC_WIN >= 0 && K4_ENC_WIN <= 32, "K4_ENC_WIN: lanes of a run's first batch, 1..32 (0 = 32)");

// Distance of search probe q from probe 0 of its run.  The reference advances by `step`, then
// sets step = searchMatchNb++ >> 6 with searchMatchNb starting at 64 (LL64.fast.cs:159-170): the
// first advance is 1, advance i >= 1 is (63 + i) >> 6, so the first 65 advances are 1, the next 64 are 2, ...
__device__ __forceinline__ uint32_t probe_advance(uint32_t q) {
    if (q <= 64u) return q;                       // the common case: a run shorter than 65 probes
    if (q == 0) return 0;
    const uint32_t c = 63u + q, k = c >> 6;
    return 1u + 32u * k * (k - 1u) + (c - 64u * k) * k;
}

// The encoder proper.  Positions are read from global memory through L1.
// Returns the engine's value: bytes written, 0 when the reference's limitedOutput checks fail.
// HARD: stop at `hardCap`, the pickler's physical write bound (see pickle.cuh).
// GTAB: the global-table warps.  `table` is a global workspace of 32-bit slots (position | 16-bit tag << 16),
// accessed through L2 (.cg) so that the little L1 left beside 224 KiB of shared memory keeps the input
// windows of all warps of the SM.  Otherwise it holds plain u16 slots (shared memory) and every candidate is fetched.
// WIN: lanes of the first batch of every search run (32 = all; K4_ENC_WIN).
// FILL: upstream's fillOutput directive (LZ4_compress_destSize, lz4.c:1382-1396): with cap below the bound, encode
// the longest prefix whose block fits `cap` instead of failing; lane 0 stores the input bytes it took at *used.
// The search never reads the output limit, so the sequences are the plain encoder's up to the cut (DESIGN 4.12).
template <bool HARD = true, bool GTAB = false, int WIN = 32, bool FILL = false>
__device__ int encode_spec_warp(const uint8_t* __restrict__ src, const uint32_t n,
                                uint8_t* __restrict__ dst, const int cap, const int hardCap, uint16_t* table,
                                int32_t* used = nullptr) {
    const int lane = lane_id();
    const int64_t hard = hardCap;       // physical write bound (pickler, see pickle.cuh); 0x7fffffff otherwise
#define RD32(p) ldg_u32u(src + (p))
#define RD8(p) ((uint32_t)__ldg(src + (p)))
    // Tag filter (GTAB).  Beside every position sits a tag: the 16 bits below the hash of the same product
    // whose bits 19..31 are the hash, taken from the 4 bytes AT the stored position.  Equal 4-byte values
    // have equal tags, so a probe only has to fetch its candidate's bytes (a scattered global load into
    // the 64 KiB window, 32 of them per batch otherwise) when the tags agree -- one probe in 65 536
    // by chance, plus the true hits.
    constexpr uint32_t TAG_SHIFT = 3u, TAG_MASK = 0xFFFFu;
    uint32_t* const table32 = reinterpret_cast<uint32_t*>(table);
    auto slotPut = [&](uint32_t h, uint32_t pos, uint32_t tg) {
        if (GTAB) __stcg(table32 + h, pos | (tg << 16)); else table[h] = (uint16_t)pos;
    };
    {   // LZ4_initStream: zero the table (LL.tools.cs:235-239); every slot then "holds" position 0
        const uint32_t t0 = (GTAB && n >= 4) ? (((RD32(0) * 2654435761u) >> TAG_SHIFT) & TAG_MASK) : 0u;
        const uint32_t fillT = GTAB ? (t0 << 16) : 0u;
        uint4* t = reinterpret_cast<uint4*>(table);
        constexpr int TBYTES = GTAB ? 2 * ENC_TABLE_BYTES : ENC_TABLE_BYTES;
        for (int i = lane; i < TBYTES / 16; i += 32) {
            if (GTAB) __stcg(t + i, make_uint4(fillT, fillT, fillT, fillT)); else t[i] = make_uint4(fillT, fillT, fillT, fillT);
        }
        __syncwarp();
    }
    const bool limited = !FILL && !(cap >= max_output_size((int)n));                  // LL64.fast.cs:524
    const bool fill = FILL && !(cap >= max_output_size((int)n));                      // lz4.c:1387
    const int64_t olimit = cap;
    uint32_t ip = 0, anchor = 0, op = 0;

    if (n >= (uint32_t)MINLENGTH) {                                               // :117
        const uint32_t mfl1 = n - MFLIMIT + 1, mlim = n - LASTLITERALS;           // :70-71
        if (lane == 0) { const uint32_t p0 = RD32(0) * 2654435761u; slotPut(p0 >> 19, 0u, (p0 >> TAG_SHIFT) & TAG_MASK); }   // :120
        __syncwarp();
        ip = 1;
        bool post = false;              // lane 0 of the next batch is the post-match probe at ip
        uint32_t q0 = 0;                // first search-probe index of the next batch
        uint32_t base = 1;              // position of search probe 0 of the current run
        constexpr uint32_t WIN0 = (WIN <= 0 || WIN > 32) ? 32u : (uint32_t)WIN;
        constexpr bool NARROW = WIN0 < 32u;
        uint32_t width = WIN0;          // lanes of the current batch: WIN0 for a run's first batch, then 32
        for (;;) {
            // ---- one batch of up to 32 probes (App. A step 3, and step 8 as lane 0) -----------------
            uint32_t h2 = 0xFFFFFFFFu, tag2 = 0;
            if (post) { const uint32_t p2 = RD32(ip - 2) * 2654435761u; h2 = p2 >> 19; tag2 = (p2 >> TAG_SHIFT) & TAG_MASK; }   // put(ip-2), :394
            const bool isPost = post && lane == 0;
            const uint32_t q = q0 + (uint32_t)lane - (post ? 1u : 0u);            // search-probe index (lanes >= 1 if post)
            const uint32_t pos = isPost ? ip : base + probe_advance(q);
            // a search probe executes only if the NEXT probe position stays <= mflimitPlusOne (:172); lanes beyond
            // the batch's width are neither probes nor the end of the run
            const bool inWin = !NARROW || (uint32_t)lane < width;
            const bool valid = inWin && (isPost || (base + probe_advance(q + 1) <= mfl1));
            const uint32_t v = valid ? RD32(pos) : 0u;
            const uint32_t prod = v * 2654435761u;
            const uint32_t h = valid ? prod >> 19 : (0x10000u + (uint32_t)lane);
            const uint32_t tg = (prod >> TAG_SHIFT) & TAG_MASK;
            uint32_t cand = 0u, ctag = tg;                                        // !GTAB: no filter, every candidate is fetched
            if (GTAB) {
                const uint32_t e32 = valid ? __ldcg(table32 + h) : 0xFFFF0000u;
                cand = e32 & 0xFFFFu; ctag = e32 >> 16;
                if (!valid) ctag = 0x10000u;
            } else {
                cand = valid ? (uint32_t)table[h] : 0u;
            }
            if (h == h2) { cand = ip - 2; ctag = tag2; }                           // sees the put(ip-2)
            const unsigned peers = __match_any_sync(FULL, h);
            const unsigned earlier = peers & ((1u << lane) - 1u);
            const int fromLane = earlier ? 31 - __clz(earlier) : lane;
            const uint32_t fwdPos = __shfl_sync(FULL, pos, fromLane);
            const uint32_t fwdTag = __shfl_sync(FULL, tg, fromLane);
            if (earlier) { cand = fwdPos; ctag = fwdTag; }                        // sees the nearest earlier store
            // GTAB: equal 4-byte words have equal tags, so only a lane whose tag agrees can hit -- and with 16-bit
            // tags nearly every such lane does.  So the first agreeing lane is taken as the hit, and the load that
            // checks its candidate word (lane 8) goes out together with the first round of the catch-up and of
            // LZ4_count (lanes 0..7), which only need the candidate's position: one memory round trip where
            // checking first takes two.  A failed check moves on to the next agreeing lane, so `f` is exactly the
            // first lane whose candidate word equals its own.
            bool hit = false;
            if (!GTAB && valid) hit = RD32(cand) == v;                            // :228 (byU16: no distance test)
            const unsigned ends = __ballot_sync(FULL, inWin && !valid);
            const int e = ends ? __ffs(ends) - 1 : 32;
            int f = 32;
            uint32_t sm = 0u, sip = 0u, sx1 = 0u;                                 // GTAB: the hit's candidate, position,
            bool sok = true;                                                      // first count round and catch-up round
            if (GTAB) {
                for (unsigned agree = __ballot_sync(FULL, valid && ctag == tg); agree; agree &= agree - 1u) {
                    const int c = __ffs(agree) - 1;
                    if (e < c) break;
                    sm = __shfl_sync(FULL, cand, c);
                    sip = __shfl_sync(FULL, pos, c);
                    const uint32_t vc = __shfl_sync(FULL, v, c);
                    bool same = true;
                    sx1 = 0u; sok = true;
                    if (lane < 8) {
                        const uint32_t a = sip + MINMATCH + 4u * lane;
                        if ((int)mlim - (int)a > 0) sx1 = RD32(a) ^ RD32(sm + MINMATCH + 4u * lane);
                        sok = (sip > anchor + lane) && (sm > (uint32_t)lane) && (RD8(sip - 1 - lane) == RD8(sm - 1 - lane));
                    } else if (lane == 8) {
                        same = RD32(sm) == vc;
                    }
                    if (__all_sync(FULL, same)) { f = c; break; }
                }
            } else {
                const unsigned hits = __ballot_sync(FULL, hit);
                f = hits ? __ffs(hits) - 1 : 32;
            }
            if (e < f) break;                                                     // ran into the end: last literals
            // commit the slot stores of probes 0..f in serial order: last writer per hash wins
            {
                const unsigned upto = (f >= 31) ? 0xffffffffu : ((2u << f) - 1u);
                const unsigned later = peers & ~((2u << lane) - 1u) & upto;       // lanes in (lane, f] with my hash
                const bool doStore = valid && ((1u << lane) & upto) && !(lane < 31 ? later : 0u);
                if (post) {
                    const unsigned same2 = __ballot_sync(FULL, valid && h == h2) & upto;
                    if (lane == 0 && !same2) {                                    // nobody overwrote the put(ip-2)
                        slotPut(h2, ip - 2, tag2);
                    }
                }
                if (doStore) slotPut(h, pos, tg);
                __syncwarp();
            }
            if (f == 32) {                                                        // no hit: keep searching
                const uint32_t w = NARROW ? width : 32u;
                if (post) { post = false; base = ip + 1; q0 = w - 1; }
                else q0 += w;
                width = 32;
                continue;
            }
            const bool zeroLit = post && f == 0;                                  // :459-463
            uint32_t m = GTAB ? sm : __shfl_sync(FULL, cand, f);
            ip = GTAB ? sip : __shfl_sync(FULL, pos, f);
            // LZ4_count does not depend on the catch-up: [ip-c, ip+4) is known equal, so counting from the hit's
            // ip+4 and adding c gives the reference's value (ip+4 <= mflimit+4 < matchlimit).  Its first round of
            // loads is issued before the catch-up loop so that both wait for memory at the same time.
            const uint32_t a0h = ip + MINMATCH, b0h = m + MINMATCH;
            uint32_t x1 = sx1;
            if (!GTAB) {
                const uint32_t a = a0h + 4u * lane;
                if (lane < 8 && (int)mlim - (int)a > 0) x1 = RD32(a) ^ RD32(b0h + 4u * lane);
            }
            uint32_t caught = 0;
            if (!zeroLit) {                                                       // step 4: catch-up, :237-242
                // eight lanes first: a catch-up is rarely longer, and lanes that do not take part issue no load
                for (int width = 8;; width = 32) {
                    const bool part = lane < width;
                    const bool ok = (GTAB && width == 8) ? sok
                                  : (!part || ((ip > anchor + lane) && (m > (uint32_t)lane) &&
                                               (RD8(ip - 1 - lane) == RD8(m - 1 - lane))));
                    const unsigned bad = __ballot_sync(FULL, !ok);
                    const int c = bad ? __ffs(bad) - 1 : width;
                    ip -= c; m -= c; caught += (uint32_t)c;
                    if (bad) break;
                }
            }
            // ---- step 5/6: literal run, offset, match length -----------------------------------------
            const uint32_t lit = ip - anchor;
            if (!zeroLit && limited && (int64_t)op + 1 + lit + 8 + lit / 255 > olimit) return 0;   // :246-251
            // fill rules 1 and 2 (lz4.c:1028-1032, 1057-1062): token, literal run, offset and MFLIMIT - MINMATCH would
            // pass the target.  (lit + 240) / 255 is the run header's extra bytes, so both tests read the same; the
            // sequence is dropped before any byte of it is written and the rest goes to last literals.
            if (fill && (int64_t)op + run_header_size(lit) + lit + 2 + 1 + (MFLIMIT - MINMATCH) > olimit) break;
            uint32_t mc = caught;
            {   // LZ4_count(ip+4, m+4, matchlimit), 4 bytes per lane, :328; the first round looks at 32 bytes
                // (eight lanes: half of all matches end there and the other lanes' lines are not fetched)
                uint32_t a0 = a0h, b0 = b0h;
                for (int width = 8;; width = 32) {
                    const uint32_t a = a0 + 4u * lane, bb = b0 + 4u * lane;
                    const bool part = lane < width;
                    const int room = (int)mlim - (int)a;                          // bytes of this lane below matchlimit
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
                    mc += 4u * width; a0 += 4u * width; b0 += 4u * width;
                }
            }
            const uint32_t hdr = run_header_size(lit);
            const uint32_t afterOff = op + hdr + lit + 2;
            if (limited && (int64_t)afterOff + 6 + (mc + 240) / 255 > olimit) return 0;   // :332-362
            // fill rule 3 (lz4.c:1097-1104): the match-length bytes would pass the target, so the match is shortened
            // to what fits; op then ends at olimit - 6, where rules 1 and 2 stop every later sequence, so the block
            // goes straight to last literals.  Upstream's hash clearing after the cut (:1105-1116) only matters to a
            // table that is used again, and this one is not.
            bool cut = false;
            if (fill && (int64_t)afterOff + 6 + (mc + 240) / 255 > olimit) {
                mc = 14u + (uint32_t)(olimit - afterOff - 6) * 255u;
                cut = true;
            }
            if (HARD && (int64_t)afterOff + (mc >= 15 ? (mc - 15) / 255 + 1 : 0) > hard) return 0;
            // emit: token, literal length bytes, literals, offset, match length bytes
            {
                const uint32_t mlTok = mc >= 15 ? 15u : mc;
                if (lane == 0) {
                    if (lit >= 15) {
                        uint32_t o = op, rest = lit - 15;
                        dst[o++] = (uint8_t)(0xF0 | mlTok);
                        for (; rest >= 255; rest -= 255) dst[o++] = 255;
                        dst[o] = (uint8_t)rest;
                    } else dst[op] = (uint8_t)((lit << 4) | mlTok);
                    dst[afterOff - 2] = (uint8_t)(ip - m);
                    dst[afterOff - 1] = (uint8_t)((ip - m) >> 8);
                }
                for (uint32_t i = lane; i < lit; i += 32) dst[op + hdr + i] = RD8(anchor + i);
                op = afterOff;
                if (mc >= 15) {                                                   // :365-379
                    const uint32_t rest = mc - 15, nff = rest / 255;
                    for (uint32_t i = lane; i < nff; i += 32) dst[op + i] = 0xFF;
                    if (lane == 0) dst[op + nff] = (uint8_t)(rest % 255);
                    op += nff + 1;
                }
            }
            ip += mc + MINMATCH;
            anchor = ip;                                                          // :388
            if (ip >= mfl1 || cut) break;                                         // :391
            post = true; q0 = 0; base = ip + 1; width = WIN0;                     // step 8 rides with the next batch
        }
    }
    {   // ---- step 9: last literals, :469-503 -----------------------------------------------------------
        uint32_t run = n - anchor;
        if (limited && (int64_t)op + run + 1 + (run + 255 - 15) / 255 > olimit) return 0;
        if (fill && (int64_t)op + run + 1 + (run + 255 - 15) / 255 > olimit) {     // fill rule 4, lz4.c:1209-1213
            run = (uint32_t)(olimit - op) - 1;
            run -= (run + 256 - 15) / 256;
        }
        const uint32_t hdr = run_header_size(run);
        if (HARD && (int64_t)op + hdr + run > hard) return 0;
        if (lane == 0) write_run_header(dst, op, run);
        op += hdr;
        for (uint32_t i = lane; i < run; i += 32) dst[op + i] = RD8(anchor + i);
        op += run;
        if (FILL && lane == 0) *used = (int32_t)(anchor + run);
        return (int)op;
    }
#undef RD32
#undef RD8
}

// counters (per device): blocks encoded by [0] a shared-memory-table warp, [1] a global-table warp (both
// n < 65 547), [2] the generic engine (n >= 65 547, either warp kind); [3] unused.  One atomic per block.
__device__ unsigned long long g_encode_stats[4];

// Persistent encoder, one warp per block at a time, one warp per CTA (a CTA leaves as soon as ITS warp
// runs out of blocks, so the CTAs of the next launch on another stream move in without a gap).  Blocks
// are handed out by a device counter.  Input and output stay in global memory.  Two kernels pull from
// the same counter and run concurrently: `encode_spec_kernel` keeps its 16 KiB hash table in shared
// memory (ENC_SM_WARPS of them fill an SM), `encode_spec_gtab_kernel` keeps it in an L2-resident
// workspace -- slower per block, but those warps use issue slots and registers the others leave idle.
// FILL: the destSize kernels (k4lz4_encode_dest_size_batch): dstCap is the target, outLen gets upstream's
// LZ4_compress_destSize result and srcUsed the input bytes it consumed; no level, no 32-bit engine.
template <bool GTAB, bool FILL = false>
__device__ __forceinline__ void encode_persistent_warp(
        const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
        const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
        const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
        int32_t* __restrict__ outLen, const int nBlocks, int level,
        uint32_t* __restrict__ nextBlock, uint16_t* const table, const int reserve,
        int32_t* __restrict__ srcUsed = nullptr) {
    const int lane = lane_id();
    const bool enforce32 = (level & ENC_FLAG_X32) != 0;   // LL.Enforce32 (LL.tools.cs:29): hash4 for the byU32 table
    level &= 0xFF;
    for (;;) {
        int b = 0;
        if (lane == 0) {
            // the slower global-table warps leave the last `reserve` blocks to the shared-memory warps
            if (GTAB && (int)*(volatile uint32_t*)nextBlock >= nBlocks - reserve) b = nBlocks;
            else b = (int)atomicAdd(nextBlock, 1u);
        }
        b = __shfl_sync(FULL, b, 0);
        if (b >= nBlocks) return;
        const int n_ = srcLen[b];
        const uint8_t* __restrict__ src = srcBase + srcOff[b];
        uint8_t* __restrict__ dst = dstBase + dstOff[b];
        const int cap = dstCap[b];
        if (FILL) {
            // nothing to encode: upstream's one-byte empty block where the target holds it (lz4.c:1263-1273), else
            // nothing written and nothing consumed
            if (n_ <= 0 || n_ > MAX_INPUT_SIZE || cap < 1) {
                if (lane == 0) {
                    const bool empty = n_ == 0 && cap >= 1;
                    if (empty) dst[0] = 0;
                    outLen[b] = empty ? 1 : 0;
                    srcUsed[b] = 0;
                }
                continue;
            }
        } else {
            if (n_ <= 0) { if (lane == 0) outLen[b] = 0; continue; }
            if (level >= 3) { if (lane == 0) outLen[b] = -2; continue; }
        }
        int r;
        if (n_ >= LIMIT_64K) r = encode_block_warp<FILL>(src, n_, dst, cap, 0x7fffffff, table, enforce32, srcUsed + b);
        else r = encode_spec_warp<false, GTAB, K4_ENC_WIN, FILL>(src, (uint32_t)n_, dst, cap, 0x7fffffff, table,
                                                                 srcUsed + b);
        if (lane == 0) {
            outLen[b] = FILL ? r : (r <= 0 ? -1 : r);
            atomicAdd(&g_encode_stats[n_ >= LIMIT_64K ? 2 : (GTAB ? 1 : 0)], 1ull);
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(32)
encode_spec_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                   const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                   const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                   int32_t* __restrict__ outLen, int nBlocks, int level, uint32_t* __restrict__ nextBlock) {
    extern __shared__ __align__(128) uint8_t smem_encs[];
    encode_persistent_warp<false>(srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, level,
                                  nextBlock, reinterpret_cast<uint16_t*>(smem_encs), 0);
}

__global__ void __launch_bounds__(32)
encode_spec_gtab_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                        const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                        const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                        int32_t* __restrict__ outLen, int nBlocks, int level, uint32_t* __restrict__ nextBlock,
                        uint8_t* __restrict__ gtab, int reserve) {
    encode_persistent_warp<true>(srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, level, nextBlock,
                                 reinterpret_cast<uint16_t*>(gtab + (size_t)blockIdx.x * ENC_GSLOT_BYTES), reserve);
}

// The destSize pair (k4lz4_encode_dest_size_batch): the two kernels above with the fill policy on, launched the same
// way and pulling from one counter.  A block whose target reaches compressBound(n) runs the plain path.
__global__ void __launch_bounds__(32)
encode_fill_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                   const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                   const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                   int32_t* __restrict__ outLen, int32_t* __restrict__ srcUsed, int nBlocks,
                   uint32_t* __restrict__ nextBlock) {
    extern __shared__ __align__(128) uint8_t smem_encf[];
    encode_persistent_warp<false, true>(srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, 0,
                                        nextBlock, reinterpret_cast<uint16_t*>(smem_encf), 0, srcUsed);
}

__global__ void __launch_bounds__(32)
encode_fill_gtab_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                        const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                        const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                        int32_t* __restrict__ outLen, int32_t* __restrict__ srcUsed, int nBlocks,
                        uint32_t* __restrict__ nextBlock, uint8_t* __restrict__ gtab, int reserve) {
    encode_persistent_warp<true, true>(srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, 0, nextBlock,
                                       reinterpret_cast<uint16_t*>(gtab + (size_t)blockIdx.x * ENC_GSLOT_BYTES),
                                       reserve, srcUsed);
}

}  // namespace k4
