// frame.cuh -- the per-frame bookkeeping kernels of the LZ4 Frame calls (k4lz4_frame_*): header parse, block
// table, token-chain size walk, layout, encode placement and the per-frame verdicts.  The bytes are coded by the
// existing codec kernels (launch_op in k4lz4_api.cu) on block tables these kernels write, moved by
// copy_blocks_kernel and hashed by xxh32_batch_kernel.
//
// Format: orig/doc/lz4_Frame_format.md; the reference's writer and reader: Streams/Frames/LZ4FrameWriter.cs:57-189,
// LZ4FrameReader.cs:55-59, LZ4FrameReader.blocking.cs:57-144.  The CPU restatement of the parse is frame.py's
// _Frame; of the walk (size_walk.cuh), tests/test_frame_model.py.
//
// Decode keeps one error KEY per frame: (block index << 4) | kind, the smallest one wins, because the reference
// reads a frame in order and throws at the first problem.  Kinds: FK_TRUNC (the block's length code, body or
// checksum, or the content checksum, is cut off), FK_SUM (block or content checksum mismatch), FK_RAW (a stored
// block larger than the reader takes), FK_BLOCK (the block decoder rejects the block: -1).
#pragma once
#include "common.cuh"
#include "xxh32.cuh"
#include "size_walk.cuh"

namespace k4 {

constexpr uint32_t FRAME_MAGIC = 0x184D2204u;
constexpr int FR_INDEPENDENT = 1, FR_BLOCK_SUM = 2, FR_CONTENT_SUM = 4;   // K4LZ4_FRAME_* (and the parsed FLG bits)
constexpr int FR_CORRUPT = -1000, FR_DELEGATE = -2, FR_DST_SMALL = -1001;   // K4LZ4_R_*
constexpr unsigned long long FK_NONE = ~0ull;
constexpr int FK_TRUNC = 0, FK_SUM = 1, FK_RAW = 2, FK_BLOCK = 3;
constexpr int64_t FR_HIST = 65536;           // history room in front of a decode scratch slot

// row kinds of the decode block table
constexpr int RK_RAW = 1, RK_SCRATCH = 2, RK_SKIP = 4, RK_LINKED = 8;

struct FrameRec {            // per frame, on the device
    int64_t first;           // first row of the frame in the block table
    int64_t slot;            // decode: first scratch slot
    int64_t pos;             // decode: content size (sum of the walks); encode: bytes laid out so far
    unsigned long long err;  // decode: smallest error key
    int32_t nb;              // decode: complete blocks; encode: blocks
    int32_t nslot;           // decode: scratch slots
    int32_t status;          // 0, or the frame's verdict before any block (R_CORRUPT / R_DELEGATE); encode: -1
    int32_t flags;           // FR_* as parsed (decode)
    int32_t maxBlock;        // BD maximum
    int32_t k0;              // decode: first block that may need a scratch slot
    uint32_t expect;         // decode: stored content checksum
    int32_t reserved;
};

struct FrameTotals { int64_t blocks, slots; int32_t maxSteps, maxCap; };

// The decode block table: one row per block of every frame.
struct FrameTable {
    int64_t* srcOff;         // the stored bytes, in srcBase
    int32_t* len;            // stored length
    int32_t* kind;           // RK_*
    uint32_t* sum;           // stored block checksum
    int32_t* frame; int32_t* idx;
    int32_t* size;           // decoded length (the walk) or the raw length
    int64_t* fin;            // final position, relative to dstBase
    int64_t* dst;            // where the block is decoded, relative to dstBase (in place or a scratch slot)
    int32_t* cap;            // the reference's capacity
    int32_t* ilen;           // OP_DECODE source length (independent compressed blocks; 0 elsewhere)
    int32_t* res;            // decoder result
    int32_t* ckLen;          // bytes to checksum (block checksums on)
    uint32_t* got;           // their XXH32
    int64_t* cpySrc;         // raw copy (source in srcBase), then scratch copy-back (source relative to dstBase)
    int32_t* cpyLen;
};
constexpr int64_t FRAME_ROW_BYTES = 8 * 5 + 4 * 11;

__device__ __forceinline__ uint32_t fr_rd32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ void fr_wr32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}
__host__ __device__ inline int32_t frame_max_block(int code) {   // LZ4FrameReader.cs:55-59
    return code == 7 ? (1 << 22) : code == 6 ? (1 << 20) : code == 5 ? (1 << 18) : (1 << 16);
}
// A lower bound of the decoded length of any stored block the reader accepts: a raw block is its length; an LZ4
// block of L bytes decodes to at least (L - 2) * 255 / 256 (every byte is output except a token, the offset and
// length-extension bytes, and each extension byte but the first of a literal run stands for 255 literals).
__device__ __forceinline__ int64_t frame_lb(int64_t L, bool raw) {
    return raw ? L : (L > 2 ? (L - 2) * 255 / 256 : 0);
}

// ---- decode ---------------------------------------------------------------------------------------------------

// The header checks on the first L bytes of a frame, in frame.py's _Frame order: magic, version with the
// reference's 0x11 mask, dictionary flag, HC.  -> 0 or the verdict (R_CORRUPT / R_DELEGATE); *p = the offset of the
// HC byte (6 or 14); *flg, *bd = the FLG and BD bytes (0 when L < 7).
__device__ __forceinline__ int frame_header_check(const uint8_t* f, int64_t L, int64_t* p, int* flg, int* bd) {
    int status = 0;
    if (L < 7 || fr_rd32(f) != FRAME_MAGIC) status = FR_CORRUPT;
    *flg = L >= 7 ? f[4] : 0;
    *bd = L >= 7 ? f[5] : 0;
    if (!status && ((*flg >> 6) & 0x11) != 1) status = FR_CORRUPT;
    if (!status && (*flg & 1)) status = FR_DELEGATE;
    const bool hasSize = (*flg >> 3) & 1;
    *p = 6 + (hasSize ? 8 : 0);
    if (!status) {
        if (L < *p + 1) status = FR_CORRUPT;
        else {
            const uint32_t h = xx_finish(XXP5 + (uint32_t)(*p - 4), f + 4, (size_t)(*p - 4));
            if (((h >> 8) & 0xFF) != f[*p]) status = FR_CORRUPT;
        }
    }
    return status;
}
__device__ __forceinline__ int frame_flags_of(int flg) {
    return (((flg >> 5) & 1) ? FR_INDEPENDENT : 0) | (((flg >> 4) & 1) ? FR_BLOCK_SUM : 0) |
           (((flg >> 2) & 1) ? FR_CONTENT_SUM : 0);
}

// One thread per frame.  Pass 0: header (frame.py's _Frame order: magic, version with the reference's 0x11 mask,
// dictionary flag, HC), the block length codes, the first block that may need a scratch slot, and the frame's
// counts.  Pass 1: the table rows.
__global__ void frame_parse_kernel(int pass, const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                                   const int32_t* __restrict__ srcLen, int n, FrameRec* __restrict__ fr,
                                   FrameTable t, FrameTotals* __restrict__ tot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    FrameRec r = fr[i];
    if (pass == 1 && r.status) return;
    const int64_t L = srcLen[i] > 0 ? srcLen[i] : 0;
    const uint8_t* f = srcBase + srcOff[i];
    int64_t p = 0;
    if (pass == 0) {
        r.status = 0; r.err = FK_NONE; r.nb = 0; r.nslot = 0; r.flags = 0; r.maxBlock = 1 << 16; r.k0 = 0; r.expect = 0;
        r.pos = 0;
        int flg, bd;
        r.status = frame_header_check(f, L, &p, &flg, &bd);
        if (r.status) { r.nb = 0; fr[i] = r; return; }
        r.flags = frame_flags_of(flg);
        r.maxBlock = frame_max_block((bd >> 4) & 7);
        p += 1;
        r.pos = p;               // where the first length code is, for pass 1
    } else {
        p = r.pos;
    }
    const bool bc = r.flags & FR_BLOCK_SUM, linked = !(r.flags & FR_INDEPENDENT);
    const int64_t cap = linked ? r.maxBlock : (int64_t)r.maxBlock + 8;
    if (pass == 0) {
        int64_t lbTotal = 0, q = p;
        int nb = 0;
        bool done = false;
        while (true) {
            if (q + 4 > L) break;
            const uint32_t code = fr_rd32(f + q);
            q += 4;
            if (code == 0) { done = true; break; }
            const int64_t blen = code & 0x7FFFFFFFu;
            if (q + blen + (bc ? 4 : 0) > L) break;
            lbTotal += frame_lb(blen, code >> 31);
            q += blen + (bc ? 4 : 0);
            nb++;
        }
        if (done && (r.flags & FR_CONTENT_SUM)) {
            if (q + 4 > L) done = false;
            else r.expect = fr_rd32(f + q);
        }
        if (!done) r.err = ((unsigned long long)nb << 4) | FK_TRUNC;
        // blocks k with less than `cap` bytes of lower bound behind them: only they can reach past dstCap
        int64_t acc = 0;
        int k0 = nb;
        q = p;
        for (int k = 0; k < nb; k++) {
            const uint32_t code = fr_rd32(f + q);
            const int64_t blen = code & 0x7FFFFFFFu;
            acc += frame_lb(blen, code >> 31);
            if (lbTotal - acc < cap) { k0 = k; break; }
            q += 4 + blen + (bc ? 4 : 0);
        }
        r.nb = nb; r.k0 = k0;
        r.nslot = nb == 0 ? 0 : linked ? (k0 < nb ? 1 : 0) : nb - k0;
        fr[i] = r;
        if (tot) {
            if (linked) atomicMax(&tot->maxSteps, nb);
            atomicMax(&tot->maxCap, (int)cap);
        }
        return;
    }
    for (int k = 0; k < r.nb; k++) {
        const int64_t b = r.first + k;
        const uint32_t code = fr_rd32(f + p);
        p += 4;
        const int32_t blen = (int32_t)(code & 0x7FFFFFFFu);
        t.srcOff[b] = srcOff[i] + p;
        t.len[b] = blen;
        t.kind[b] = (code >> 31 ? RK_RAW : 0) | (linked ? RK_LINKED : 0);
        t.frame[b] = i; t.idx[b] = k;
        p += blen;
        t.sum[b] = bc ? fr_rd32(f + p) : 0;
        p += bc ? 4 : 0;
    }
}

// Single CTA: exclusive scan of the frames' block and slot counts -> first row and first slot; totals.
__global__ void __launch_bounds__(1024) frame_scan_kernel(FrameRec* __restrict__ fr, int n, FrameTotals* __restrict__ tot,
                                                          int slots) {
    __shared__ int64_t wa[32], wb[32];
    __shared__ int64_t carry[2];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry[0] = 0; carry[1] = 0; }
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const int64_t a = i < n ? fr[i].nb : 0, b = i < n && slots ? fr[i].nslot : 0;
        int64_t xa = a, xb = b;
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t ya = __shfl_up_sync(FULL, xa, d), yb = __shfl_up_sync(FULL, xb, d);
            if (lane >= d) { xa += ya; xb += yb; }
        }
        if (lane == 31) { wa[w] = xa; wb[w] = xb; }
        __syncthreads();
        if (w == 0) {
            int64_t va = wa[lane], vb = wb[lane];
            for (int d = 1; d < 32; d <<= 1) {
                const int64_t ya = __shfl_up_sync(FULL, va, d), yb = __shfl_up_sync(FULL, vb, d);
                if (lane >= d) { va += ya; vb += yb; }
            }
            wa[lane] = va; wb[lane] = vb;
        }
        __syncthreads();
        const int64_t oa = carry[0] + (w ? wa[w - 1] : 0) + xa - a, ob = carry[1] + (w ? wb[w - 1] : 0) + xb - b;
        if (i < n) { fr[i].first = oa; fr[i].slot = ob; }
        __syncthreads();
        if (threadIdx.x == 1023) { carry[0] = oa + a; carry[1] = ob + b; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { tot->blocks = carry[0]; tot->slots = carry[1]; }
}

// One warp per row: the decoded length of a compressed block (a raw block's is its length), by the warp walk of
// size_walk.cuh.  A chain that does not parse is an error of its block (the decoder rejects it too); its size is
// then the lower bound, so that the layout's scratch rule still holds.  Launch with 32 * nB threads.
__global__ void block_size_walk_kernel(const uint8_t* __restrict__ srcBase, FrameTable t, int64_t nB,
                                       FrameRec* __restrict__ fr) {
    const int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= nB) return;
    const int32_t L = t.len[b];
    const bool raw = t.kind[b] & RK_RAW;
    int64_t s = raw ? L : sw_walk_warp(srcBase + t.srcOff[b], L, threadIdx.x & 31);
    if (threadIdx.x & 31) return;
    if (s < 0) {
        atomicMin(&fr[t.frame[b]].err, ((unsigned long long)t.idx[b] << 4) | FK_BLOCK);
        s = frame_lb(L, false);
    }
    t.size[b] = (int32_t)(s < frame_lb(L, raw) ? frame_lb(L, raw) : (s > 0x7FFFFFFF ? 0x7FFFFFFF : s));
}

// One thread per frame: content size, positions, where each block decodes (in place when the reference's capacity
// stays inside dstCap, else in a scratch slot), raw copies, checksum lengths.  dstCap null: sizes only.  A frame
// with a header verdict or a content larger than dstCap is skipped: nothing of it is written.
__global__ void frame_layout_kernel(FrameRec* __restrict__ fr, int n, FrameTable t, const int64_t* __restrict__ dstOff,
                                    const int32_t* __restrict__ dstCap, int64_t scratchRel, int64_t slotBytes,
                                    int32_t* __restrict__ ccLen) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    FrameRec r = fr[i];
    int64_t total = 0;
    for (int k = 0; k < r.nb; k++) total += t.size[r.first + k];
    r.pos = total;
    const int64_t room = dstCap ? (dstCap[i] > 0 ? dstCap[i] : 0) : INT64_MAX;
    const bool skip = r.status != 0 || total > room;
    const bool linked = !(r.flags & FR_INDEPENDENT), bc = r.flags & FR_BLOCK_SUM;
    const int32_t cap = linked ? r.maxBlock : r.maxBlock + 8;
    const int64_t rawLimit = linked ? (r.maxBlock > 65536 ? r.maxBlock : 65536) : (int64_t)r.maxBlock + 8;
    if (ccLen) ccLen[i] = (!skip && (r.flags & FR_CONTENT_SUM)) ? (int32_t)total : 0;
    int64_t pos = 0;
    for (int k = 0; k < r.nb; k++) {
        const int64_t b = r.first + k;
        const int32_t L = t.len[b], sz = t.size[b];
        const bool raw = t.kind[b] & RK_RAW;
        const int64_t fin = (dstOff ? dstOff[i] : 0) + pos;
        const unsigned long long rawKey = ((unsigned long long)k << 4) | FK_RAW;
        if (raw && L > rawLimit && rawKey < r.err) r.err = rawKey;
        const bool scratch = dstCap && !skip && !raw && pos + cap > room;
        int64_t at = fin;
        if (scratch) at = scratchRel + (r.slot + (linked ? 0 : k - r.k0)) * slotBytes + FR_HIST;
        t.fin[b] = fin;
        t.dst[b] = at;
        t.cap[b] = cap;
        t.kind[b] = (t.kind[b] & (RK_RAW | RK_LINKED)) | (scratch ? RK_SCRATCH : 0) | (skip ? RK_SKIP : 0);
        t.ilen[b] = (!skip && !raw && !linked) ? L : 0;
        t.cpyLen[b] = (!skip && raw && L <= rawLimit) ? L : 0;
        t.cpySrc[b] = t.srcOff[b];
        t.ckLen[b] = (!skip && bc) ? L : 0;
        t.res[b] = 0;
        pos += sz;
    }
    fr[i].pos = r.pos;
    fr[i].err = r.err;
}

// Linked frames, step k: block k of every frame that has one (a compressed, not skipped block) decodes behind the
// frame's output so far.  One entry per frame; the others get an empty source (no work).  A block in a scratch
// slot gets the last <= 64 KiB of the output copied in front of it.
struct FrameStep {
    int64_t* srcOff; int32_t* srcLen; int64_t* dstOff; int32_t* cap; int32_t* prefix; int32_t* res;
    int64_t* hSrc; int64_t* hDst; int32_t* hLen;     // history copy, then copy-back
};
__global__ void frame_step_prepare_kernel(int k, const FrameRec* __restrict__ fr, int n, FrameTable t, FrameStep s,
                                          const int64_t* __restrict__ dstOff) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FrameRec& r = fr[i];
    int32_t len = 0, hl = 0, pre = 0, cap = 0;
    int64_t so = 0, dof = 0, hs = 0, hd = 0;
    if (!(r.flags & FR_INDEPENDENT) && k < r.nb) {
        const int64_t b = r.first + k;
        const int kind = t.kind[b];
        if (!(kind & (RK_RAW | RK_SKIP))) {
            len = t.len[b]; so = t.srcOff[b]; dof = t.dst[b]; cap = t.cap[b];
            const int64_t produced = t.fin[b] - dstOff[i];
            pre = (int32_t)(produced < 65535 ? produced : 65535);
            if (kind & RK_SCRATCH) {
                hl = (int32_t)(produced < FR_HIST ? produced : FR_HIST);
                hs = t.fin[b] - hl; hd = dof - hl;
            }
        }
    }
    s.srcOff[i] = so; s.srcLen[i] = len; s.dstOff[i] = dof; s.cap[i] = cap; s.prefix[i] = pre;
    s.hSrc[i] = hs; s.hDst[i] = hd; s.hLen[i] = hl;
}

// After the step's decode: the result goes to the row, an accepted block in a scratch slot is copied back.
__global__ void frame_step_commit_kernel(int k, const FrameRec* __restrict__ fr, int n, FrameTable t, FrameStep s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FrameRec& r = fr[i];
    int32_t back = 0;
    int64_t bs = 0, bd = 0;
    if (s.srcLen[i] > 0) {
        const int64_t b = r.first + k;
        const int32_t res = s.res[i];
        t.res[b] = res;
        if ((t.kind[b] & RK_SCRATCH) && res == t.size[b]) { back = res; bs = t.dst[b]; bd = t.fin[b]; }
    }
    s.hSrc[i] = bs; s.hDst[i] = bd; s.hLen[i] = back;
}

// One thread per row, after every decode: block checksums, decoder results against the walk, and the copy-back of
// independent blocks decoded in a scratch slot (cpySrc / fin / cpyLen).
__global__ void frame_verdict_kernel(FrameRec* __restrict__ fr, FrameTable t, int64_t nB) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nB) return;
    const int kind = t.kind[b];
    const int k = t.idx[b];
    unsigned long long* err = &fr[t.frame[b]].err;
    int32_t back = 0;
    if (!(kind & RK_SKIP)) {
        if (t.ckLen[b] > 0 && t.got[b] != t.sum[b]) atomicMin(err, ((unsigned long long)k << 4) | FK_SUM);
        if (!(kind & RK_RAW)) {
            const int32_t res = t.res[b];
            if (res != t.size[b]) atomicMin(err, ((unsigned long long)k << 4) | FK_BLOCK);
            else if ((kind & RK_SCRATCH) && !(kind & RK_LINKED)) back = res;
        }
    }
    t.cpySrc[b] = t.dst[b];
    t.cpyLen[b] = back;
}

// One thread per frame: the frame's result.  sizeOnly: the content-size call (no checksums, no decoder results).
__global__ void frame_decode_finish_kernel(const FrameRec* __restrict__ fr, int n, const int32_t* __restrict__ dstCap,
                                           const uint32_t* __restrict__ ccGot, const int32_t* __restrict__ ccLen,
                                           int32_t* __restrict__ outLen) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FrameRec& r = fr[i];
    unsigned long long err = r.err;
    int32_t out;
    if (r.status) out = r.status;
    else if (dstCap && r.pos > (dstCap[i] > 0 ? dstCap[i] : 0))
        out = (err != FK_NONE && (err & 15) == FK_TRUNC) ? FR_CORRUPT : FR_DST_SMALL;
    else {
        if (ccGot && (r.flags & FR_CONTENT_SUM) && ccLen[i] == r.pos && ccGot[i] != r.expect) {
            const unsigned long long key = ((unsigned long long)r.nb << 4) | FK_SUM;
            if (key < err) err = key;
        }
        if (err != FK_NONE) out = (err & 15) == FK_BLOCK ? -1 : FR_CORRUPT;
        else out = r.pos > 0x7FFFFFFF ? FR_CORRUPT : (int32_t)r.pos;
    }
    outLen[i] = out;
}

// ---- encode ---------------------------------------------------------------------------------------------------

// One thread per frame.  Pass 0: block counts (and the number of steps).  Pass 1: the rows (source offset and
// length of every block; in FrameTable's srcOff / len) and the frame's starting layout.
__global__ void frame_enc_plan_kernel(int pass, const int64_t* __restrict__ srcOff, const int32_t* __restrict__ srcLen,
                                      int n, int32_t bs, FrameRec* __restrict__ fr, FrameTable t,
                                      FrameTotals* __restrict__ tot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t L = srcLen[i] > 0 ? srcLen[i] : 0;
    const int nb = (int)((L + bs - 1) / bs);
    if (pass == 0) {
        FrameRec r = {};
        r.nb = nb; r.pos = 7; r.err = FK_NONE;
        fr[i] = r;
        atomicMax(&tot->maxSteps, nb);
        return;
    }
    const int64_t first = fr[i].first;
    for (int k = 0; k < nb; k++) {
        t.srcOff[first + k] = srcOff[i] + (int64_t)k * bs;
        t.len[first + k] = (int32_t)((L - (int64_t)k * bs) < bs ? (L - (int64_t)k * bs) : bs);
    }
}

// Entries of one encode launch, as laid out into the frames.
struct FrameEnc {
    int64_t* cSrc; int64_t* cDst; int32_t* cLen;     // encoded body: scratch -> destination
    int64_t* rSrc; int32_t* rLen;                    // raw body: source -> destination (at cDst)
    int64_t* ckOff; int32_t* ckLen; uint32_t* ckSum; // block checksum of the stored bytes
    int32_t* res;                                    // the encoder's results, by entry
};

// One thread per frame: lays out the frame's blocks of this launch -- rows [b0, b1) (independent: entry = row - b0)
// or, with k >= 0, its block k (linked: entry = frame - f0).  Stored = the encoded bytes when they shrink the block,
// else the raw bytes (LZ4EncoderBase.cs:79-83).  A block that does not fit dstCap fails the frame (-1); nothing is
// written at or beyond dstCap.
__global__ void frame_enc_place_kernel(int k, int64_t b0, int64_t b1, int f0, int f1, FrameRec* __restrict__ fr,
                                       FrameTable t, FrameEnc e, uint8_t* __restrict__ dstBase,
                                       const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                                       int32_t bound, int bc) {
    const int i = f0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f1) return;
    FrameRec r = fr[i];
    int64_t lo, hi;
    if (k >= 0 && k >= r.nb) {            // no block k: the frame's entry copies and hashes nothing
        const int x = i - f0;
        e.cLen[x] = 0; e.rLen[x] = 0; e.ckLen[x] = 0;
        e.cSrc[x] = 0; e.cDst[x] = 0; e.rSrc[x] = 0; e.ckOff[x] = 0;
        return;
    }
    if (k >= 0) { lo = r.first + k; hi = lo + 1; }
    else { lo = r.first > b0 ? r.first : b0; hi = r.first + r.nb < b1 ? r.first + r.nb : b1; }
    const int64_t room = dstCap[i] > 0 ? dstCap[i] : 0;
    for (int64_t b = lo; b < hi; b++) {
        const int64_t x = k >= 0 ? i - f0 : b - b0;
        const int32_t L = t.len[b], res = e.res[x];
        int32_t cl = 0, rl = 0, ck = 0;
        int64_t cd = 0;
        if (!r.status) {
            const bool raw = res >= L;
            const int32_t stored = raw ? L : res;
            const int64_t need = 4 + (int64_t)stored + (bc ? 4 : 0);
            if (res <= 0 || r.pos + need > room) r.status = -1;
            else {
                fr_wr32(dstBase + dstOff[i] + r.pos, (uint32_t)stored | (raw ? 0x80000000u : 0u));
                cd = dstOff[i] + r.pos + 4;
                if (raw) rl = L; else cl = res;
                ck = bc ? stored : 0;
                r.pos += need;
            }
        }
        e.cSrc[x] = x * (int64_t)bound; e.cDst[x] = cd; e.cLen[x] = cl;
        e.rSrc[x] = t.srcOff[b]; e.rLen[x] = rl;
        e.ckOff[x] = cd; e.ckLen[x] = ck;
    }
    fr[i].pos = r.pos;
    fr[i].status = r.status;
}

// Linked step k: block k of frame i (entry i - f0) behind the frame's own source; other entries are empty.
__global__ void frame_enc_step_kernel(int k, int f0, int f1, const FrameRec* __restrict__ fr, FrameTable t,
                                      int64_t* __restrict__ so, int32_t* __restrict__ sl, int32_t* __restrict__ pre,
                                      int32_t bs) {
    const int i = f0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f1) return;
    const int x = i - f0;
    const FrameRec& r = fr[i];
    const bool on = k < r.nb && !r.status;
    so[x] = on ? t.srcOff[r.first + k] : 0;
    sl[x] = on ? t.len[r.first + k] : 0;
    const int64_t p = (int64_t)k * bs;
    pre[x] = (int32_t)(p < 0x7FFFFFFF ? p : 0x7FFFFFFF);
}

// Block checksums into place, after the bodies.
__global__ void frame_put_sum_kernel(uint8_t* __restrict__ dstBase, FrameEnc e, int n) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= n || e.ckLen[x] <= 0) return;
    fr_wr32(dstBase + e.ckOff[x] + e.ckLen[x], e.ckSum[x]);
}

// One thread per frame: header, end mark, content checksum, result.
__global__ void frame_enc_finish_kernel(const FrameRec* __restrict__ fr, int n, uint8_t* __restrict__ dstBase,
                                        const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                                        uint64_t header, int cc, const uint32_t* __restrict__ csum,
                                        int32_t* __restrict__ outLen) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FrameRec& r = fr[i];
    const int64_t total = r.pos + 4 + (cc ? 4 : 0);
    if (r.status || total > (dstCap[i] > 0 ? dstCap[i] : 0) || total > 0x7FFFFFFF) { outLen[i] = -1; return; }
    uint8_t* d = dstBase + dstOff[i];
    for (int j = 0; j < 7; j++) d[j] = (uint8_t)(header >> (8 * j));
    fr_wr32(d + r.pos, 0);
    if (cc) fr_wr32(d + r.pos + 4, csum[i]);
    outLen[i] = (int32_t)total;
}

// off[x] = x * stride and, when cap is given, cap[x] = capValue: the fixed slots of a launch.
__global__ void frame_slots_kernel(int64_t* __restrict__ off, int32_t* __restrict__ cap, int n, int64_t stride,
                                   int32_t capValue) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= n) return;
    off[x] = x * stride;
    if (cap) cap[x] = capValue;
}

__global__ void frame_fill_kernel(int32_t* __restrict__ out, int n, int32_t v) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v;
}

}  // namespace k4
