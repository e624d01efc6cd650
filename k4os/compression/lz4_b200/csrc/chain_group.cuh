// chain_group.cuh -- the bookkeeping kernels of a chain group (k4lz4_chain_group_*): S chained streams whose
// history rings, encoder states and write positions stay on one GPU between calls.
//
// Stream s owns ring s, RING bytes at ringBase + s * RING, laid out [history | slot].  Its header holds the write
// position `pos`: ring[0 .. pos) are the stream's last pos bytes, and the next block is read or written at
// ring + pos.  The history a block sees is the last min(pos, 65 536) bytes; `pos` only falls below 65 536 before
// the stream's first slide, when it is the whole stream.  After a block, when the next one might not fit
// (pos + SLOT > RING, SLOT = max(blockSize, 65 536)), the last 65 536 bytes slide to the front.  RING = 128 KiB +
// SLOT, so a slide starts beyond 64 KiB and never overlaps its own destination.
//
// These kernels only write block tables and headers: the bytes move with copy_blocks_kernel (copy_blocks.cuh) and
// the codec kernels run unchanged on tables that point into the rings.  One thread per block of the call.
#pragma once
#include "common.cuh"
#include "encode_chain.cuh"

namespace k4 {

struct ChainGroupHdr {       // per stream, on the device
    int64_t pos;             // bytes in the ring in front of the slot
    int32_t failed;          // encoder: a block did not fit; the stream returns -1 until it is reset
    int32_t reserved;
};

enum ChainGroupKind { CG_ENCODE = 0, CG_DECODE = 1, CG_INJECT = 2 };

constexpr int64_t CG_WINDOW = 65536;

// The block table of one call.  Every array has n entries.
struct ChainGroupTable {
    int64_t* ringOff;        // codec: the block's slot in the ring; after the commit: a slide's destination
    int32_t* len;            // encode: the codec's srcLen; decode: its dstCap; inject: the bytes kept
    int32_t* prefix;         // codec: the history length, -1 for a block that must not run
    int64_t* stateOff;       // encode: the state record
    int32_t* stream;         // the stream the block advances, -1 for none
    int64_t* copyOff;        // source of the copy into the ring, then of the slide
    int32_t* copyLen;        // bytes of that copy (0: none)
};

// Block i of stream streams[i].  `len` is srcLen (encode, inject) or dstCap (decode), `srcOff` the caller's
// source offsets (encode, inject).  A block whose stream index is out of range, whose stream failed (encode) or
// whose length exceeds `blockSize` (encode: srcLen, decode: dstCap) gets prefix -1, so that the codec returns -1
// for it without reading anything, and advances no stream.  An empty encode block runs as it is (result 0).
__global__ void chain_group_prepare_kernel(int kind, const int32_t* __restrict__ streams,
                                           const int32_t* __restrict__ len, const int64_t* __restrict__ srcOff,
                                           int n, int nStreams, int32_t blockSize, int64_t ring,
                                           const ChainGroupHdr* __restrict__ hdr, ChainGroupTable t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    const int32_t L = len[i];
    const bool inRange = s >= 0 && s < nStreams;
    const int64_t pos = inRange ? hdr[s].pos : 0;
    bool ok = inRange;
    if (kind == CG_ENCODE) ok = ok && !hdr[s].failed && L <= blockSize;
    if (kind == CG_DECODE) ok = ok && L <= blockSize;
    const int64_t at = ok ? (int64_t)s * ring + pos : 0;
    t.ringOff[i] = at;
    t.prefix[i] = ok ? (int32_t)(pos < CG_WINDOW ? pos : CG_WINDOW) : -1;
    t.stateOff[i] = ok ? (int64_t)s * (int64_t)sizeof(ChainState) : 0;
    t.stream[i] = ok ? s : -1;
    int32_t keep = 0;
    if (kind == CG_INJECT) keep = !ok || L <= 0 ? 0 : (L < CG_WINDOW ? L : (int32_t)CG_WINDOW);
    else if (kind == CG_ENCODE) keep = ok && L > 0 ? L : 0;
    t.len[i] = kind == CG_INJECT ? keep : (ok ? L : (kind == CG_ENCODE ? 1 : 0));
    t.copyOff[i] = keep > 0 ? srcOff[i] + (L - keep) : 0;
    t.copyLen[i] = keep;
}

// After the codec (and the gather of its output): advances each block's stream by what the block added -- the
// source length of an encoded block, the bytes decoded, the bytes injected -- marks an encoder stream failed
// where the codec returned -1, and writes the slide of every stream whose next block might not fit.  A failed
// decode and an empty, delegated or rejected block leave the stream as it was.
__global__ void chain_group_commit_kernel(int kind, const int32_t* __restrict__ outLen, int n, int64_t ring,
                                          int64_t slot, ChainGroupHdr* __restrict__ hdr, ChainGroupTable t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = t.stream[i];
    int64_t add = 0;
    if (s >= 0) {
        if (kind == CG_INJECT) add = t.len[i];
        else {
            const int32_t r = outLen[i];
            if (r > 0) add = kind == CG_ENCODE ? t.len[i] : r;
            else if (r == -1 && kind == CG_ENCODE) hdr[s].failed = 1;
        }
    }
    int32_t slide = 0;
    if (add > 0) {
        int64_t pos = hdr[s].pos + add;
        if (pos + slot > ring) {
            t.copyOff[i] = (int64_t)s * ring + pos - CG_WINDOW;
            t.ringOff[i] = (int64_t)s * ring;
            slide = (int32_t)CG_WINDOW;
            pos = CG_WINDOW;
        }
        hdr[s].pos = pos;
    }
    t.copyLen[i] = slide;
}

// Reset: stream streams[i] becomes a new stream (empty ring, zero state record, not failed).  One CTA per entry;
// an index out of range is skipped.
__global__ void chain_group_reset_kernel(const int32_t* __restrict__ streams, int n, int nStreams,
                                         ChainGroupHdr* __restrict__ hdr, uint8_t* __restrict__ stateBase) {
    const int i = blockIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    if (s < 0 || s >= nStreams) return;
    if (threadIdx.x == 0) { hdr[s].pos = 0; hdr[s].failed = 0; }
    if (!stateBase) return;
    uint4* st = reinterpret_cast<uint4*>(stateBase + (int64_t)s * (int64_t)sizeof(ChainState));
    for (int k = threadIdx.x; k < (int)(sizeof(ChainState) / 16); k += blockDim.x) st[k] = make_uint4(0, 0, 0, 0);
}

}  // namespace k4
