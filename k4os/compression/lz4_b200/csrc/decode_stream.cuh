// decode_stream.cuh -- whole chained LZ4 streams in one call, every block of every stream in flight at once
// (k4lz4_decode_chain_streams, DESIGN 4.11).
//
// A chained block's accept / reject decisions read its token stream, its capacity and its history length P as a
// number, never a decoded byte (LL64.dec.cs:124-467: every test compares ip, op, lengths and offsets against bounds
// and lowPrefix).  Block k's P is the stream's history plus the bytes the blocks before it decode, and those are
// known up front from the size walk (size_walk.cuh).  So every block is parsed, judged and mostly written in
// parallel; only the match copies that read bytes this call writes in earlier blocks wait for them:
//
//   1. place    one warp per entry: decoded size (the walk, or srcLen for a stored entry), clamped to the capacity
//               so that a failing block cannot move a later one out of its stream's region; the stream of each
//               entry.  Then one CTA scans the sizes over all entries; an entry's offset in its stream is its scan
//               value minus that of the stream's first entry.
//   2. decode   persistent warps, one entry each: the exact engine (decode_block_warp) in prefix mode, so the
//               verdict is final here, with its writes going through DeferOut.  Literals and the matches whose
//               source is final (the caller's history, or bytes of this block that are not deferred) are written.
//               A match that reads bytes of an earlier block of this call, or a deferred interval of its own block,
//               is recorded as (op, len, offset) on the block's deferred list; the list's destinations are the
//               block's deferred intervals (increasing and disjoint, so membership is a binary search over the
//               list).  A block with more than DS_BUDGET deferred matches is marked "whole".
//   3. verdicts and
//   4. replay   one warp per stream, streams handed out by a counter: the stream's entries in order, -1 from its
//               first failing entry on; each block's deferred records replayed with the exact engine's copy
//               semantics (the records that read only earlier blocks 32 at a time, then the rest in order, in runs
//               of independent records), or a "whole" block decoded again by the engine with DirectOut, whose
//               history is final by then.  Every stream's chain runs on its own warp, so all resident streams
//               advance side by side, and no warp ever waits on another.
//
// Why the replay is exact: LZ4 writes every output byte once, in order.  Pass 2 wrote every byte that depends only
// on final bytes; pass 4 writes the rest in stream order, after everything they read is final.  A replay warp reads
// only bytes written by an earlier kernel or by itself.
#pragma once
#include "common.cuh"
#include "decode_generic.cuh"
#include "decode_tile.cuh"
#include "size_walk.cuh"

#ifndef K4_DS_BUDGET
#define K4_DS_BUDGET 2048    // deferred matches per entry before it is decoded whole (DESIGN 4.11)
#endif

namespace k4 {

constexpr int DS_BUDGET = K4_DS_BUDGET;
constexpr int DS_SCAN_THREADS = 1024;
constexpr int DS_LAUNCHES = 4;

struct DeferCopy { int32_t op, len, off; };

// The call's workspace (from the private pool).  ndef[e] = deferred copies of entry e, -1 = decode whole.
struct StreamWork {
    int64_t* gex;        // n + 1: exclusive scan of the placed sizes over all entries
    int32_t* sid;        // n: the stream of each entry, -1 where no stream holds it
    int32_t* ndef;       // n
    DeferCopy* copies;   // n * DS_BUDGET
    uint32_t* ticket;    // the replay's stream counter
};

// Where entry e sits: its stream s, its output offset in the stream and its history length (-1: negative prefix).
struct Place { int s; int64_t off; int P; };

__device__ __forceinline__ Place ds_place(const StreamWork& w, const int32_t* entryStart, const int32_t* prefixLen,
                                          int e) {
    Place p{w.sid[e], 0, -1};
    if (p.s < 0) return p;
    p.off = w.gex[e] - w.gex[entryStart[p.s]];
    const int64_t P = prefixLen[p.s] < 0 ? -1 : prefixLen[p.s] + p.off;
    p.P = P < 0 ? -1 : (P < 65535 ? (int)P : 65535);
    return p;
}

// pass 1: one warp per entry
__global__ void stream_place_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                                    const int32_t* __restrict__ srcLen, const uint8_t* __restrict__ raw,
                                    const int32_t* __restrict__ dstCap, const int32_t* __restrict__ entryStart,
                                    int nStreams, StreamWork w, int n) {
    const int64_t e = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (e >= n) return;
    int lo = 0, hi = nStreams;                       // the last s with entryStart[s] <= e
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (entryStart[mid] <= e) lo = mid; else hi = mid - 1; }
    const int s = (lo < nStreams && entryStart[lo] >= 0 && entryStart[lo] <= e && e < entryStart[lo + 1]) ? lo : -1;
    const int32_t L = srcLen[e], cap = dstCap[e];
    int64_t sz = 0;
    if (raw && raw[e]) sz = (L >= 0 && L <= cap) ? L : 0;
    else if (L > 0 && cap > 0) {
        sz = sw_walk_warp(srcBase + srcOff[e], L, lane);
        sz = sz < 0 ? 0 : (sz < cap ? sz : cap);
    }
    if (lane == 0) { w.gex[e + 1] = sz; w.sid[e] = s; }
}

// pass 1, scan: gex[0] = 0, gex[1 .. n] = inclusive sums (one CTA)
__global__ void __launch_bounds__(DS_SCAN_THREADS) stream_scan_kernel(StreamWork w, int n) {
    __shared__ int64_t part[DS_SCAN_THREADS / 32];
    __shared__ int64_t carry;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    if (t == 0) { carry = 0; w.gex[0] = 0; *w.ticket = 0; }
    __syncthreads();
    for (int64_t b = 0; b < n; b += DS_SCAN_THREADS) {
        const int64_t i = b + t;
        int64_t v = i < n ? w.gex[i + 1] : 0;
        for (int d = 1; d < 32; d <<= 1) { const int64_t u = __shfl_up_sync(FULL, v, d); if (lane >= d) v += u; }
        if (lane == 31) part[wid] = v;
        __syncthreads();
        if (wid == 0) {
            int64_t p = part[lane];
            for (int d = 1; d < 32; d <<= 1) { const int64_t u = __shfl_up_sync(FULL, p, d); if (lane >= d) p += u; }
            part[lane] = p;
        }
        __syncthreads();
        const int64_t c = carry;
        if (i < n) w.gex[i + 1] = c + v + (wid ? part[wid - 1] : 0);
        __syncthreads();
        if (t == DS_SCAN_THREADS - 1) carry = c + part[31];
        __syncthreads();
    }
}

// The engine's output in pass 2 (prefix mode, outputSize = cap, no dictionary, not partial).  `off` = the block's
// offset in its stream: bytes in [-off, 0) are this call's earlier blocks.  Literals and the match copies whose
// source is final are written; a match that touches [-off, 0) or a deferred interval of this block is recorded on
// `copies` instead.  The block's deferred intervals increase and are disjoint, so membership is a binary search over
// the earlier records.  Past DS_BUDGET records the block is "whole": nothing more is written.  After the engine
// returns, nd = the deferred copies or -1 (whole).
struct DeferOut {
    int64_t off;
    DeferCopy* copies;
    int ndef = 0;
    bool whole = false;
    int64_t lastLo = 0, lastHi = -1;                 // the last deferred interval (in registers)
    int nd = 0;

    __device__ __forceinline__ void literals(uint8_t* d, const uint8_t* __restrict__ s, int len, int lane) {
        if (!whole) warp_copy_in(d, s, len, lane);
    }
    __device__ __forceinline__ void match(uint8_t* dst, int64_t op, int64_t match, int len, int offset, int lane) {
        if (whole) return;
        if (offset == 0) { warp_copy_match(dst, op, match, len, offset, lane); return; }
        const int64_t lo = match, hi = match + (offset < len ? offset : len);
        bool dep = (lo > -off ? lo : -off) < (hi < 0 ? hi : 0);
        if (!dep && hi > 0) {
            const int64_t qlo = lo > 0 ? lo : 0;
            dep = lastLo < hi && lastHi > qlo;
            if (!dep && ndef > 1 && qlo < lastLo) {  // the last earlier deferred copy that starts below hi
                __syncwarp();
                int a = 0, b = ndef - 2;
                while (a < b) { const int m = (a + b + 1) >> 1; if (copies[m].op < hi) a = m; else b = m - 1; }
                const DeferCopy c = copies[a];
                dep = c.op < hi && c.op + c.len > qlo;
            }
        }
        if (!dep) { warp_copy_match(dst, op, match, len, offset, lane); return; }
        if (ndef == DS_BUDGET) { whole = true; return; }
        if (lane == 0) copies[ndef] = DeferCopy{(int32_t)op, len, offset};
        ndef++;
        lastLo = op; lastHi = op + len;
    }
    // never reached: a chained stream has no dictionary
    __device__ __forceinline__ void window(uint8_t*, int64_t, int64_t, int, int, const uint8_t*, int, int) {}
    __device__ __forceinline__ int done(int r) { nd = whole ? -1 : ndef; return r; }
};

// pass 2: persistent warps, one entry at a time
__global__ void stream_decode_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                     const int32_t* __restrict__ srcLen, const uint8_t* __restrict__ raw,
                     const int32_t* __restrict__ dstCap, const int32_t* __restrict__ entryStart,
                     uint8_t* dstBase, const int64_t* __restrict__ dstOff, const int32_t* __restrict__ prefixLen,
                     int32_t* __restrict__ outLen, StreamWork w, int n) {
    const int lane = lane_id();
    const int nwarps = (int)(gridDim.x * (blockDim.x >> 5));
    for (int e = (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)); e < n; e += nwarps) {
        const Place p = ds_place(w, entryStart, prefixLen, e);
        const int32_t L = srcLen[e], cap = dstCap[e];
        const uint8_t* src = srcBase + srcOff[e];
        int r = -1, nd = 0;
        if (p.s >= 0 && p.P >= 0) {
            uint8_t* dst = dstBase + dstOff[p.s] + p.off;
            if (raw && raw[e]) {                                     // LZ4ChainDecoder.Inject of a stored block
                if (L >= 0 && L <= cap) { warp_copy_in(dst, src, L, lane); r = L; }
            } else if (L <= 0 || cap <= 0) {
                r = chain_trivial(L, cap, src);
            } else {
                DeferOut out{p.off, w.copies + (int64_t)e * DS_BUDGET};
                r = decode_block_warp(out, src, L, dst, cap, false, nullptr, 0, p.P);
                r = r < 0 ? -1 : r;
                nd = out.nd;
            }
        }
        if (lane == 0) { outLen[e] = r; w.ndef[e] = nd; }
    }
}

constexpr int DS_LANE_COPY = 64;     // records up to this long are replayed one per lane

// Every source byte of a deferred record lies in [op - offset, op), in front of its own destination, so its loads
// may run ahead of its stores.  The result is the exact engine's (warp_copy_match).
__device__ __forceinline__ int64_t rec_src(const DeferCopy& d, int i) {
    return (int64_t)d.op - d.off + (d.off >= d.len ? i : i % d.off);
}

// one record by the whole warp
__device__ __forceinline__ void replay_copy(uint8_t* dst, const DeferCopy d, int lane) {
    constexpr int U = 16;
    __syncwarp();
    for (int b = 0; b < d.len; b += 32 * U) {
        uint8_t v[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int i = b + u * 32 + lane;
            if (i < d.len) v[u] = dst[rec_src(d, i)];
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int i = b + u * 32 + lane;
            if (i < d.len) dst[d.op + i] = v[u];
        }
    }
}

// one record (at most DS_LANE_COPY bytes) by one lane, 16 bytes of loads ahead of their stores
__device__ __forceinline__ void lane_copy(uint8_t* dst, const DeferCopy d) {
    for (int b = 0; b < d.len; b += 16) {
        uint8_t v[16];
#pragma unroll
        for (int u = 0; u < 16; u++)
            if (b + u < d.len) v[u] = dst[rec_src(d, b + u)];
#pragma unroll
        for (int u = 0; u < 16; u++)
            if (b + u < d.len) dst[d.op + b + u] = v[u];
    }
}

// A block's deferred records, exactly as if copied one after another.  Phase A: the records whose source lies wholly
// in front of the block (in earlier blocks, all final now) read no byte any record writes, so they go 32 at a time,
// one per lane.  Phase B: the rest, in order, in runs of records none of which reads an earlier one's destination
// (one per lane); a record that does, or a long one, goes alone with the whole warp once the run before it is done.
__device__ void replay_block(uint8_t* dst, const DeferCopy* c, int nd, int lane) {
    for (int k0 = 0; k0 < nd; k0 += 32) {
        DeferCopy d{0, 0, 1};
        const bool valid = k0 + lane < nd;
        if (valid) d = c[k0 + lane];
        const bool a = valid && (int64_t)d.op - d.off + min(d.len, d.off) <= 0;
        __syncwarp();
        if (a && d.len <= DS_LANE_COPY) lane_copy(dst, d);
        for (unsigned big = __ballot_sync(FULL, a && d.len > DS_LANE_COPY); big; big &= big - 1) {
            const int j = __ffs(big) - 1;
            replay_copy(dst, DeferCopy{__shfl_sync(FULL, d.op, j), __shfl_sync(FULL, d.len, j),
                                       __shfl_sync(FULL, d.off, j)}, lane);
        }
    }
    for (int k = 0; k < nd;) {
        DeferCopy d{0, 0, 1};
        const bool valid = k + lane < nd;
        if (valid) d = c[k + lane];
        const int64_t lo = (int64_t)d.op - d.off, hi = lo + min(d.len, d.off);
        const bool b = valid && hi > 0;
        bool dep = false;
        for (int i = 0; i < 31; i++) {            // an earlier phase-B record of the window writes my source
            const int iop = __shfl_sync(FULL, d.op, i), ilen = __shfl_sync(FULL, d.len, i);
            const bool ib = __shfl_sync(FULL, b, i);
            dep |= i < lane && ib && iop < hi && iop + ilen > lo;
        }
        const unsigned stop = __ballot_sync(FULL, b && (dep || d.len > DS_LANE_COPY));
        const int m = stop ? __ffs(stop) - 1 : 32;
        __syncwarp();
        if (lane < m && b) lane_copy(dst, d);
        if (m < 32) {
            replay_copy(dst, DeferCopy{__shfl_sync(FULL, d.op, m), __shfl_sync(FULL, d.len, m),
                                       __shfl_sync(FULL, d.off, m)}, lane);
            k += m + 1;
        } else {
            k += 32;
        }
    }
    __syncwarp();
}

// passes 3 and 4: one warp per stream at a time (streams handed out by a counter), its chain in order: from the
// stream's first failing entry on every entry is -1; a deferred list is replayed, a "whole" block decoded again
// by the engine with DirectOut (its history is final by then).  A warp reads only bytes it wrote itself or that
// an earlier kernel wrote, so no warp ever waits on another and the chains of all resident streams run side by side.
__global__ void __launch_bounds__(128)
stream_replay_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                     const int32_t* __restrict__ srcLen, const int32_t* __restrict__ dstCap,
                     const int32_t* __restrict__ entryStart, uint8_t* dstBase, const int64_t* __restrict__ dstOff,
                     const int32_t* __restrict__ prefixLen, int32_t* outLen, StreamWork w, int n, int nStreams) {
    const int lane = lane_id();
    for (;;) {
        int s = 0;
        if (lane == 0) s = (int)atomicAdd(w.ticket, 1u);
        s = __shfl_sync(FULL, s, 0);
        if (s >= nStreams) return;
        const int e0 = max(entryStart[s], 0), e1 = min(entryStart[s + 1], n);
        bool failed = false;
        for (int e = e0; e < e1; e++) {
            if (w.sid[e] != s) continue;
            const int r = outLen[e], nd = w.ndef[e];
            if (failed || r < 0) {
                failed = true;
                if (lane == 0 && r >= 0) outLen[e] = -1;
                continue;
            }
            if (nd == 0) continue;
            const Place p = ds_place(w, entryStart, prefixLen, e);
            uint8_t* dst = dstBase + dstOff[s] + p.off;
            __syncwarp();
            if (nd < 0) decode_block_warp(DirectOut{}, srcBase + srcOff[e], srcLen[e], dst, dstCap[e], false, nullptr, 0,
                                          p.P);
            else replay_block(dst, w.copies + (int64_t)e * DS_BUDGET, nd, lane);
        }
    }
}

// Enqueues the decode of n entries of nStreams chained streams on `st` (current device); every pointer is a device
// pointer.  The workspace comes from `pool`, a private stream-ordered pool of the current device; `sms` is its SM
// count.  On success DS_LAUNCHES kernels were launched.
inline cudaError_t stream_decode_launch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                        const uint8_t* raw, const int32_t* dstCap, int32_t* outLen, int n,
                                        const int32_t* entryStart, uint8_t* dstBase, const int64_t* dstOff,
                                        const int32_t* prefixLen, int nStreams, cudaStream_t st,
                                        cudaMemPool_t pool, int sms) {
    auto a256 = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t N = (size_t)n;
    const size_t gexAt = 256, sidAt = gexAt + a256((N + 1) * 8), ndefAt = sidAt + a256(N * 4);
    const size_t copyAt = ndefAt + a256(N * 4), total = copyAt + N * DS_BUDGET * sizeof(DeferCopy);
    uint8_t* ws = nullptr;
    cudaError_t e = cudaMallocFromPoolAsync((void**)&ws, total, pool, st);
    if (e != cudaSuccess) return e;
    StreamWork w{reinterpret_cast<int64_t*>(ws + gexAt), reinterpret_cast<int32_t*>(ws + sidAt),
                 reinterpret_cast<int32_t*>(ws + ndefAt),
                 reinterpret_cast<DeferCopy*>(ws + copyAt), reinterpret_cast<uint32_t*>(ws)};
    stream_place_kernel<<<(unsigned)((N * 32 + 127) / 128), 128, 0, st>>>(srcBase, srcOff, srcLen, raw, dstCap,
                                                                         entryStart, nStreams, w, n);
    stream_scan_kernel<<<1, DS_SCAN_THREADS, 0, st>>>(w, n);
    const int want = (n + 3) / 4;
    const int gridDec = want < sms * 8 ? want : sms * 8;
    stream_decode_kernel<<<gridDec, 128, 0, st>>>(srcBase, srcOff, srcLen, raw, dstCap, entryStart, dstBase, dstOff,
                                                  prefixLen, outLen, w, n);
    // one warp per stream, as many as the streams or as fit on the device (32 per SM) if fewer
    const int64_t warps = std::min<int64_t>((int64_t)nStreams, (int64_t)sms * 32);
    stream_replay_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, st>>>(srcBase, srcOff, srcLen, dstCap, entryStart,
                                                                      dstBase, dstOff, prefixLen, outLen, w, n,
                                                                      nStreams);
    e = cudaGetLastError();
    cudaFreeAsync(ws, st);
    return e;
}

}  // namespace k4
