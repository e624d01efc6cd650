// encode_dict.cuh -- LZ4 L00_FAST blocks against an external dictionary, bit-exact with upstream's
//   LZ4_loadDict(s, dict, dictLen); LZ4_compress_fast_continue(s, src, dst, n, cap, 1)
// (orig/lib/lz4.c:1475-1514, 1565-1637) with the dictionary in a buffer of its own: the usingExtDict branch
// (lz4.c:1626-1631).  What LZ4Codec.Decode(source, target, dictionary) reads back.
//
// The load (LZ4_loadDict, 64-bit HASH_UNIT = 8): currentOffset = 65 536; only the last 65 536 bytes count
// (dictSize = min(dictLen, 65 536)); positions p = start + 3k with p <= dictEnd - 8 go into slot hash5(8 bytes at p)
// with value 65 536 - (dictEnd - p), the last writer per slot winning; a dictionary of fewer than 8 bytes loads
// nothing and leaves dictSize = 0 (lz4.c:1499-1501), so it encodes exactly like an empty one.
//
// The search (encode_dict_warp) is the chained encoder's, chain_search_warp, through ExtWindow: startIndex = 65 536,
// dictSmall for dictSize < 65 536, and the extDict addressing and catch-up floor.
//
// Blocks whose dictionaries are the same bytes range share one loaded table: dict_key_kernel gives every block
// the first block that claimed its (start, size) key, and each distinct key one record, up to DICT_RECORDS;
// dict_load_kernel fills the records; every block then starts from a private copy of its record in a per-warp
// workspace slot (16 KiB through L2, the chained encoder's table access), or loads its table itself when its
// dictionary got no record.
#pragma once
#include "common.cuh"
#include "encode_chain.cuh"

namespace k4 {

constexpr int DICT_WINDOW = 65536;
constexpr int DICT_HASH_UNIT = 8;
constexpr int DICT_RECORDS = 1024;    // loaded tables per launch (16 MiB); blocks of further dictionaries load their own

// The bytes of a dictionary of `len` bytes that LZ4_loadDict keeps: the last min(len, 65 536), none below 8.
__host__ __device__ inline int dict_kept(int len) {
    return len < DICT_HASH_UNIT ? 0 : (len > DICT_WINDOW ? DICT_WINDOW : len);
}

// LZ4_loadDict into `st` by one warp, 32 positions per step in increasing order: within a step the last lane of
// each slot stores, and __syncwarp orders the steps, so the largest position per slot wins.
__device__ void load_dict_warp(const uint8_t* __restrict__ dict, int len, ChainState* st) {
    const int lane = lane_id();
    const int dsz = dict_kept(len);
    uint4* const t4 = reinterpret_cast<uint4*>(st);
    for (int i = lane; i < (int)(sizeof(ChainState) / 16); i += 32) __stcg(t4 + i, make_uint4(0u, 0u, 0u, 0u));
    __syncwarp();
    if (lane == 0) { __stcg(&st->currentOffset, (uint32_t)DICT_WINDOW); __stcg(&st->dictSize, (uint32_t)dsz); }
    if (dsz == 0) { __syncwarp(); return; }
    const uint8_t* const p0 = dict + (len - dsz);
    const int npos = (dsz - DICT_HASH_UNIT) / 3 + 1;
    const uint32_t base = (uint32_t)(DICT_WINDOW - dsz);
    constexpr int U = 8;                                  // steps whose loads are issued together
    for (int k0 = 0; k0 < npos; k0 += 32 * U) {
        uint32_t h[U];
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int k = k0 + 32 * j + lane;
            h[j] = k < npos ? hash5(ldg_u64u(p0 + 3 * k), 12) : 0x10000u + (uint32_t)lane;
        }
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int k = k0 + 32 * j + lane;
            const unsigned peers = __match_any_sync(FULL, h[j]);
            if (k < npos && !((peers >> lane) >> 1)) __stcg(st->table + h[j], base + 3u * (uint32_t)k);
            __syncwarp();
        }
    }
}

// Reads in the extDict layout: position p < 0 is dictEnd[p], the `d` kept dictionary bytes that logically precede
// the source in a buffer of its own.  A word may straddle the two buffers.  same8 and floor/above keep the forms
// PrefixWindow (encode_chain.cuh) explains: a byte compare of the widened reads, and the floor hoisted into an int.
struct ExtWindow {
    const uint8_t* dictEnd;
    uint32_t d;
    __device__ __forceinline__ uint32_t rd8(const uint8_t* __restrict__ src, int p) const {
        return p < 0 ? (uint32_t)__ldg(dictEnd + p) : (uint32_t)__ldg(src + p);
    }
    __device__ __forceinline__ uint32_t rd32(const uint8_t* __restrict__ src, int p) const {
        if (p >= 0) return ldg_u32u(src + p);
        if (p <= -4) return ldg_u32u(dictEnd + p);
        uint32_t v = 0;
        for (int i = 0; i < 4; i++) v |= rd8(src, p + i) << (8 * i);
        return v;
    }
    __device__ __forceinline__ bool same8(const uint8_t* __restrict__ src, int a, int b) const {
        return rd8(src, a) == rd8(src, b);
    }
    __device__ __forceinline__ int floor(int m) const { return m < 0 ? -(int)d : 0; }
    __device__ __forceinline__ bool above(int x, int low) const { return x > low; }
};

// One block against its loaded table `table` (a private copy: the block's stores go into it) and the `d` kept
// dictionary bytes that end at dictEnd.  Returns the engine's value: bytes written, or 0 when a limitedOutput check
// fails.  This is chain_search_warp<false> (encode_chain.cuh, whose comments give the upstream lines) with
// startIndex = 65 536, dictSmall for d < 65 536 (lz4.c:1626-1629), and the usingExtDict mode's reads and catch-up:
//   * an index below startIndex lies in the dictionary at dictEnd - (startIndex - index), and reads that run past
//     the dictionary's end continue at src[0], as upstream's match count does (lz4.c:1078-1089);
//   * a match found in the source catches up no further than the source's start (lz4.c:992, 1180); one found in
//     the dictionary down to the dictionary's start (lz4.c:989, 1177).
__device__ int encode_dict_warp(const uint8_t* __restrict__ src, const uint32_t n, const uint8_t* __restrict__ dictEnd,
                                const uint32_t d, uint8_t* __restrict__ dst, const int cap, uint32_t* table) {
    if (n > (uint32_t)MAX_INPUT_SIZE) return 0;
    return chain_search_warp<false>(ExtWindow{dictEnd, d}, src, n, (uint32_t)DICT_WINDOW, d,
                                    d < (uint32_t)DICT_WINDOW, table, dst, cap);
}

// The key of a block's dictionary: the (start, size) of the bytes the load keeps.  An empty one is (0, 0).
struct DictKey { int64_t at; int32_t size; };
__device__ __forceinline__ DictKey dict_key(const int64_t* dictOff, const int32_t* dictLen, int b) {
    const int len = dictLen[b];
    const int dsz = dict_kept(len);
    return dsz == 0 ? DictKey{0, 0} : DictKey{dictOff[b] + (len - dsz), dsz};
}

// One thread per block: claims the block's key in an open-addressing map of mask + 1 >= 2n slots (block + 1, 0 =
// free) or finds the block that did.  rep[b] = that block; a claiming block numbers its key's record in
// recId[b] (-1 beyond DICT_RECORDS) and names itself in recBlock[] for the load.  Empty sources need no table.
__global__ void dict_key_kernel(const int64_t* __restrict__ dictOff, const int32_t* __restrict__ dictLen,
                                const int32_t* __restrict__ srcLen, int n, int32_t* __restrict__ map, uint32_t mask,
                                int32_t* __restrict__ rep, int32_t* __restrict__ recId,
                                int32_t* __restrict__ recBlock, uint32_t* __restrict__ nRec) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n || srcLen[b] <= 0) return;
    const DictKey k = dict_key(dictOff, dictLen, b);
    uint64_t x = (uint64_t)k.at * 0x9E3779B97F4A7C15ull ^ ((uint64_t)(uint32_t)k.size * 0xC2B2AE3D27D4EB4Full);
    uint32_t s = (uint32_t)(x >> 32) & mask;
    for (;;) {
        const int32_t v = atomicCAS(map + s, 0, b + 1);
        if (v == 0) break;
        const DictKey o = dict_key(dictOff, dictLen, v - 1);
        if (o.at == k.at && o.size == k.size) { rep[b] = v - 1; return; }
        s = (s + 1) & mask;
    }
    rep[b] = b;
    const uint32_t id = atomicAdd(nRec, 1u);
    recId[b] = id < (uint32_t)DICT_RECORDS ? (int32_t)id : -1;
    if (id < (uint32_t)DICT_RECORDS) recBlock[id] = b;
}

// One warp per record: LZ4_loadDict of the record's dictionary.
__global__ void __launch_bounds__(32)
dict_load_kernel(const uint8_t* __restrict__ dictBase, const int64_t* __restrict__ dictOff,
                 const int32_t* __restrict__ dictLen, const int32_t* __restrict__ recBlock,
                 const uint32_t* __restrict__ nRec, ChainState* __restrict__ recs) {
    const int r = blockIdx.x;
    if ((uint32_t)r >= *nRec) return;
    const int b = recBlock[r];
    load_dict_warp(dictBase + dictOff[b], dictLen[b], recs + r);
}

// Persistent: one-warp CTAs pull blocks from a device counter; CTA c encodes in workspace slot work[c].
// Block b's result: 0 for n <= 0; -1 where the engine returns 0 (does not fit dstCap); otherwise the bytes written.
__global__ void __launch_bounds__(32, ENC_CHAIN_WARPS)
encode_dict_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                   const int32_t* __restrict__ srcLen, uint8_t* __restrict__ dstBase,
                   const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                   const uint8_t* __restrict__ dictBase, const int64_t* __restrict__ dictOff,
                   const int32_t* __restrict__ dictLen, const int32_t* __restrict__ rep,
                   const int32_t* __restrict__ recId, const ChainState* __restrict__ recs,
                   ChainState* __restrict__ work, int32_t* __restrict__ outLen, int nBlocks,
                   uint32_t* __restrict__ nextBlock) {
    const int lane = lane_id();
    ChainState* const ws = work + blockIdx.x;
    for (;;) {
        int b = 0;
        if (lane == 0) b = (int)atomicAdd(nextBlock, 1u);
        b = __shfl_sync(FULL, b, 0);
        if (b >= nBlocks) return;
        const int n = srcLen[b];
        if (n <= 0) { if (lane == 0) outLen[b] = 0; continue; }
        const uint8_t* const dict = dictBase + dictOff[b];
        const int len = dictLen[b];
        const int r = recId[rep[b]];
        if (r >= 0) {
            const uint4* const from = reinterpret_cast<const uint4*>(recs + r);
            uint4* const to = reinterpret_cast<uint4*>(ws);
            for (int i = lane; i < (int)(sizeof(ChainState) / 16); i += 32) __stcg(to + i, __ldcg(from + i));
            __syncwarp();
        } else {
            load_dict_warp(dict, len, ws);
        }
        const int res = encode_dict_warp(srcBase + srcOff[b], (uint32_t)n, dict + (len > 0 ? len : 0),
                                         (uint32_t)dict_kept(len), dstBase + dstOff[b], dstCap[b], ws->table);
        if (lane == 0) {
            outLen[b] = res <= 0 ? -1 : res;
            atomicAdd(&g_encode_stats[3], 1ull);
        }
        __syncwarp();
    }
}

}  // namespace k4
