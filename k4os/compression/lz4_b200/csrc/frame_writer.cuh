// frame_writer.cuh -- the bookkeeping kernels of a frame writer group (k4lz4_frame_writer_group_*): S LZ4 frames
// written incrementally, each stream's partial block, chain state and running content checksum kept on one GPU
// between calls (LZ4EncoderStream over LZ4FrameWriter, Streams/Frames/LZ4FrameWriter.cs and .blocking.cs).
//
// Stream s owns ring s with the chain-group layout (chain_group.cuh): [history | slot] for linked frames, the slot
// alone (pos stays 0) for independent ones.  Its ChainGroupHdr holds the write position `pos`; its FwState holds
// the `pending` bytes of the partial block at ring + pos, the "open" flag (a header has been written) and the
// streaming XXH32 of the content.  A write of L bytes emits floor((pending + L) / B) blocks, one per step: the
// step moves the next B - pending bytes of the source behind the pending ones, the codec encodes the slot, the
// place kernel lays the block out at the entry's cursor, and for linked frames chain_group_commit_kernel advances
// `pos` and slides the ring.  What is left (< B bytes) becomes the new partial block.  Close encodes the partial
// block (one step with length `pending`), then writes the end mark and the content checksum.
//
// The bytes are moved by copy_blocks_kernel, encoded by the codec kernels and hashed by xxh32_batch_kernel, all
// unchanged; these kernels only write tables, headers and length codes.  One thread per entry unless noted.
#pragma once
#include "common.cuh"
#include "chain_group.cuh"
#include "frame.cuh"
#include "xxh32.cuh"

namespace k4 {

struct FwState {             // per stream, on the device
    uint32_t v[4];           // XXH32 accumulators (seed 0)
    uint64_t total;          // content bytes so far
    uint8_t carry[16];       // content bytes not yet in a 16-byte stripe
    int32_t carryLen;
    int32_t pending;         // bytes of the partial block at ring + pos
    int32_t open;            // the frame's header has been written
    int32_t reserved;
};

struct FwEntry {             // per entry of one call
    int64_t srcOff;          // the entry's source
    int64_t start, cursor;   // where its output starts / goes next
    int64_t used;            // source bytes moved into the ring so far
    int32_t stream;          // -1: the entry does nothing (rejected, or a close of a stream that is not open)
    int32_t len;             // source length (0 for close)
    int32_t steps;           // blocks the call emits for it
    int32_t reserved;
};

// The most one write of `len` bytes or one close appends (k4lz4_frame_writer_bound / _close_bound).
__host__ __device__ inline int64_t fw_write_bound(int64_t len, int32_t B, bool bc) {
    return 7 + (B - 1 + len) / B * (4 + (int64_t)B + (bc ? 4 : 0));
}
__host__ __device__ inline int64_t fw_close_bound(int32_t B, bool bc, bool cc) {
    return 4 + (int64_t)B + (bc ? 4 : 0) + 4 + (cc ? 4 : 0);
}

// Write (len != null) or close (len == null): checks range and capacity (rejected: outLen = -1, nothing changes),
// opens the frame on its first write (header at the cursor, fresh checksum state), and counts the steps.  A close
// of a stream that is not open appends nothing (outLen = 0).  maxSteps: the call's largest step count.
__global__ void frame_writer_plan_kernel(const int32_t* __restrict__ streams, const int64_t* __restrict__ srcOff,
                                         const int32_t* __restrict__ len, const int64_t* __restrict__ dstOff,
                                         const int32_t* __restrict__ dstCap, int n, int nStreams, int32_t B, int flags,
                                         uint64_t header, uint8_t* __restrict__ dstBase, FwState* __restrict__ fw,
                                         FwEntry* __restrict__ ent, int32_t* __restrict__ outLen,
                                         int32_t* __restrict__ maxSteps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool bc = flags & FR_BLOCK_SUM, cc = flags & FR_CONTENT_SUM;
    const int s = streams[i];
    const int64_t L = len ? (len[i] > 0 ? len[i] : 0) : 0;
    const int64_t bound = len ? fw_write_bound(L, B, bc) : fw_close_bound(B, bc, cc);
    FwEntry e = {};
    e.stream = -1;
    e.srcOff = len ? srcOff[i] : 0;
    e.start = e.cursor = dstOff[i];
    e.len = (int32_t)L;
    if (s < 0 || s >= nStreams || bound > 0x7FFFFFFF || dstCap[i] < bound) {
        outLen[i] = -1;
    } else if (!len) {
        if (fw[s].open) { e.stream = s; e.steps = fw[s].pending > 0 ? 1 : 0; }
        else outLen[i] = 0;
    } else {
        FwState& f = fw[s];
        if (!f.open) {
            uint8_t* d = dstBase + e.cursor;
            for (int j = 0; j < 7; j++) d[j] = (uint8_t)(header >> (8 * j));
            e.cursor += 7;
            f.open = 1;
            f.v[0] = XXP1 + XXP2; f.v[1] = XXP2; f.v[2] = 0; f.v[3] = 0u - XXP1;
            f.total = 0; f.carryLen = 0;
        }
        e.stream = s;
        e.steps = (int32_t)((f.pending + L) / B);
        if (e.steps > 0) atomicMax(maxSteps, e.steps);
    }
    ent[i] = e;
}

// Content checksum: advances each written stream's XXH32 state over the entry's source, as XXH32_update does
// (orig/lib/xxhash.c): the carried bytes complete a first stripe, whole stripes follow, the rest is carried.
// Four consecutive lanes per entry, lane g owns accumulator g, as in xxh32_batch_kernel.
__global__ void __launch_bounds__(128)
frame_writer_xxh_kernel(const uint8_t* __restrict__ srcBase, const FwEntry* __restrict__ ent, int n,
                        FwState* __restrict__ fw) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = t >> 2, g = t & 3;
    const unsigned quad = 0xFu << (threadIdx.x & 28);
    const int s = i < n ? ent[i].stream : -1;
    const int64_t L = s >= 0 ? ent[i].len : 0;
    const uint8_t* p = srcBase + (s >= 0 ? ent[i].srcOff : 0);
    FwState* f = fw + (s >= 0 ? s : 0);
    const int c = s >= 0 ? f->carryLen : 0;
    int64_t q = 0;
    uint32_t v = 0;
    if (s >= 0 && c + L >= 16) {
        v = f->v[g];
        if (c > 0) {
            uint32_t w = 0;
            for (int j = 3; j >= 0; j--) {
                const int k = 4 * g + j;
                w = (w << 8) | (k < c ? f->carry[k] : p[k - c]);
            }
            v = xx_round(v, w);
            q = 16 - c;
        }
        const int64_t stripes = (L - q) >> 4;
        for (int64_t k = 0; k < stripes; k++) v = xx_round(v, ldg_u32u(p + q + 16 * k + 4 * g));
        q += 16 * stripes;
    }
    __syncwarp(quad);                 // every lane has read the carry before lane 0 replaces it
    if (s < 0) return;
    if (c + L >= 16) {
        f->v[g] = v;
        if (g == 0) {
            for (int64_t k = q; k < L; k++) f->carry[k - q] = p[k];
            f->carryLen = (int32_t)(L - q);
        }
    } else if (g == 0) {
        for (int64_t k = 0; k < L; k++) f->carry[c + k] = p[k];
        f->carryLen = (int32_t)(c + L);
    }
    if (g == 0) f->total += (uint64_t)L;
}

// Step k of entries [e0, e0 + m) (table index x = i - e0): an entry with k < steps gets its block -- the slot at
// ring + pos, B bytes when writing (the next B - pending source bytes move in behind the pending ones: copyOff ->
// copyDst), `pending` bytes when closing.  The others get an empty block (the codec returns 0 and touches nothing)
// and stream -1 (the commit skips them).
__global__ void frame_writer_step_kernel(int k, int e0, int m, int closing, FwEntry* __restrict__ ent,
                                         const FwState* __restrict__ fw, const ChainGroupHdr* __restrict__ hdr,
                                         int32_t B, int64_t ring, int linked, ChainGroupTable t,
                                         int64_t* __restrict__ copyDst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= m) return;
    FwEntry& e = ent[e0 + x];
    const int s = e.stream;
    int32_t blen = 0, take = 0, pre = 0;
    int64_t at = 0, from = 0;
    if (s >= 0 && k < e.steps) {
        const int64_t pos = linked ? hdr[s].pos : 0;
        const int32_t pending = fw[s].pending;
        at = (int64_t)s * ring + pos;
        blen = closing ? pending : B;
        take = closing ? 0 : B - pending;
        from = e.srcOff + e.used;
        e.used += take;
        pre = linked ? (int32_t)(pos < CG_WINDOW ? pos : CG_WINDOW) : 0;
        copyDst[x] = at + pending;
    } else {
        copyDst[x] = 0;
    }
    t.ringOff[x] = at;
    t.len[x] = blen;
    t.prefix[x] = pre;
    t.stateOff[x] = blen > 0 ? (int64_t)s * (int64_t)sizeof(ChainState) : 0;
    t.stream[x] = blen > 0 ? s : -1;
    t.copyOff[x] = from;
    t.copyLen[x] = take;
}

// After the codec: each block goes to its entry's cursor -- length code, then the encoded body (from the scratch
// slot x * bound) or, when it does not shrink, the raw bytes from the ring (LZ4EncoderBase.cs:79-83), then room
// for the block checksum -- and the stream's partial block is gone.
__global__ void frame_writer_place_kernel(int e0, int m, FwEntry* __restrict__ ent, FwState* __restrict__ fw,
                                          ChainGroupTable t, FrameEnc e, uint8_t* __restrict__ dstBase, int32_t bound,
                                          int bc) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= m) return;
    const int s = t.stream[x];
    int32_t cl = 0, rl = 0, ck = 0;
    int64_t cd = 0;
    if (s >= 0) {
        FwEntry& en = ent[e0 + x];
        const int32_t L = t.len[x], res = e.res[x];
        const bool raw = res <= 0 || res >= L;
        const int32_t stored = raw ? L : res;
        fr_wr32(dstBase + en.cursor, (uint32_t)stored | (raw ? 0x80000000u : 0u));
        cd = en.cursor + 4;
        if (raw) rl = L; else cl = res;
        ck = bc ? stored : 0;
        en.cursor += 4 + (int64_t)stored + (bc ? 4 : 0);
        fw[s].pending = 0;
    }
    e.cSrc[x] = (int64_t)x * bound; e.cDst[x] = cd; e.cLen[x] = cl;
    e.rSrc[x] = t.ringOff[x]; e.rLen[x] = rl;
    e.ckOff[x] = cd; e.ckLen[x] = ck;
}

// The end of a call.  Write: the rest of the source (< B bytes) joins the partial block (copyOff -> copyDst,
// copyLen).  Close: the end mark and the content checksum; the stream is no longer open, and reset[i] names it so
// that chain_group_reset_kernel empties its ring and state record (-1 elsewhere).  outLen = the bytes appended.
__global__ void frame_writer_finish_kernel(int closing, const FwEntry* __restrict__ ent, int n,
                                           FwState* __restrict__ fw, const ChainGroupHdr* __restrict__ hdr,
                                           int64_t ring, int linked, int cc, uint8_t* __restrict__ dstBase,
                                           int64_t* __restrict__ copyOff, int64_t* __restrict__ copyDst,
                                           int32_t* __restrict__ copyLen, int32_t* __restrict__ reset,
                                           int32_t* __restrict__ outLen) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FwEntry e = ent[i];
    const int s = e.stream;
    int64_t from = 0, to = 0;
    int32_t rest = 0, rs = -1;
    if (s >= 0) {
        FwState& f = fw[s];
        int64_t cur = e.cursor;
        if (!closing) {
            rest = (int32_t)(e.len - e.used);
            from = e.srcOff + e.used;
            to = (int64_t)s * ring + (linked ? hdr[s].pos : 0) + f.pending;
            f.pending += rest;
        } else {
            fr_wr32(dstBase + cur, 0);
            cur += 4;
            if (cc) {
                uint32_t h = f.total >= 16 ? xx_rotl(f.v[0], 1) + xx_rotl(f.v[1], 7) + xx_rotl(f.v[2], 12) +
                                             xx_rotl(f.v[3], 18)
                                           : f.v[2] + XXP5;
                h += (uint32_t)f.total;
                fr_wr32(dstBase + cur, xx_finish(h, f.carry, (size_t)f.carryLen));
                cur += 4;
            }
            f.open = 0;
            f.pending = 0;
            rs = s;
        }
        outLen[i] = (int32_t)(cur - e.start);
    }
    if (copyOff) { copyOff[i] = from; copyDst[i] = to; copyLen[i] = rest; }
    if (reset) reset[i] = rs;
}

// Reset (abandon): the streams are no longer open and hold no partial block; chain_group_reset_kernel empties
// their rings and state records.  An index out of range is skipped.
__global__ void frame_writer_reset_kernel(const int32_t* __restrict__ streams, int n, int nStreams,
                                          FwState* __restrict__ fw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    if (s < 0 || s >= nStreams) return;
    fw[s].open = 0;
    fw[s].pending = 0;
}

}  // namespace k4
