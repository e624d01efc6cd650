// frame_reader.cuh -- the bookkeeping kernels of a frame reader group (k4lz4_frame_reader_group_*): S LZ4 frame
// streams read incrementally, each stream's partial header or block, history and running content checksum kept on
// one GPU between calls (LZ4DecoderStream over LZ4FrameReader, Streams/Frames/LZ4FrameReader.async.cs:46-172).
//
// Stream s owns ring s with the chain-group layout (chain_group.cuh; SLOT = max(maxBlockSize + 8, 64 KiB)): blocks
// decode into the slot at ring + pos, linked frames with the last min(pos, 64 KiB) bytes as their history,
// independent ones at pos 0.  Its stash holds a block cut by the end of a chunk ([length code | body | checksum],
// the first `have` bytes of it), its FrState a cut header or content checksum (hbuf), the frame's flags and BD, a
// phase and a sticky error, and its FwState the content XXH32 (frame_writer.cuh's layout, so that
// frame_writer_xxh_kernel updates it unchanged).  A compressed block longer than the stash (no such block decodes
// within blockCap) is skipped instead: its body is hashed in a second FwState as it passes, so that its verdict
// keeps the whole-frame order -- truncated (end) or a block checksum mismatch: R_CORRUPT; otherwise -1.
//
// A read plans every entry first (one thread per entry, a count pass, frame_scan_kernel, a fill pass): it
// continues the stream's phase over the chunk, hops over the length codes under the room rule (at most
// floor(dstCap / blockCap) blocks per call, blockCap = the reference decoder's capacity) and writes one row per
// block it completes -- stored bytes in the chunk, or in the stash for the one block a previous chunk began.  The
// rows' checksums are verified by xxh32_batch_kernel before anything decodes; then step k decodes block k of every
// entry into its slot, gathers it to the entry's cursor, advances the content XXH32 and commits the ring
// (chain_group_commit_kernel).  The finish kernel gives the verdicts, and the unconsumed tail of a cut block is
// copied into the stash last.
#pragma once
#include "common.cuh"
#include "chain_group.cuh"
#include "frame.cuh"
#include "frame_writer.cuh"
#include "xxh32.cuh"

namespace k4 {

enum FrPhase { FP_IDLE = 0, FP_HEADER = 1, FP_BLOCK = 2, FP_TAIL = 3, FP_SKIP = 4 };
constexpr int FR_ARG = -102;                   // K4LZ4_E_ARG: a device-memory entry's stream index is out of range
constexpr int FRK_LINKED = 1, FRK_INDEP = 2, FRK_BLOCK_SUM = 4, FRK_CONTENT_SUM = 8;   // kinds of rows a call has
constexpr int FRK_SKIP = 16;                   // ... and a skipped block's bytes to hash

struct FrState {             // per stream, on the device
    int32_t phase;           // FrPhase: between frames, in a header, at or in a block, in the content checksum
    int32_t have;            // bytes of the current item held: in hbuf (header, checksum) or in the stash (block)
    int32_t err;             // 0, or the result every read returns until the stream is reset
    int32_t flags;           // FR_* of the open frame
    int32_t maxBlock;        // its BD maximum
    int32_t skip;            // FP_SKIP: body bytes of the skipped block still to come (then its checksum, in hbuf)
    uint8_t hbuf[24];
};

struct FrEntry {             // per entry of one read; the rest is in its FrameRec
    int64_t start;           // where its output starts (relative to dstBase)
    int64_t used;            // chunk bytes consumed
    int32_t stream;          // -1: out of range
    int32_t ended;           // the call ended a frame
    int32_t check;           // FrameRec.expect to verify: 1 the content checksum, 2 the skipped block's checksum
    int32_t reserved;
};

// Copies the plan orders from the chunk into the stash: the rest of a block a previous chunk began (before the
// checksums) and the tail of the chunk when it ends inside a block (after every decode).
struct FrCopies { int64_t* upOff; int64_t* upDst; int32_t* upLen; int64_t* tailOff; int64_t* tailDst; int32_t* tailLen; };

// Byte j of the current item: the `have` stashed bytes, then the chunk from q on.
__device__ __forceinline__ uint32_t fr_vbyte(const uint8_t* stash, int have, const uint8_t* p, int64_t q, int64_t j) {
    return j < have ? stash[j] : p[q + j - have];
}
// xxhash.c's XXH32_digest of a streaming state (seed 0).
__device__ __forceinline__ uint32_t fr_digest(const FwState& f) {
    uint32_t h = f.total >= 16 ? xx_rotl(f.v[0], 1) + xx_rotl(f.v[1], 7) + xx_rotl(f.v[2], 12) + xx_rotl(f.v[3], 18)
                               : f.v[2] + XXP5;
    h += (uint32_t)f.total;
    return xx_finish(h, f.carry, (size_t)f.carryLen);
}
__device__ __forceinline__ void fr_xxh_reset(FwState& x) {
    x.v[0] = XXP1 + XXP2; x.v[1] = XXP2; x.v[2] = 0; x.v[3] = 0u - XXP1;
    x.total = 0; x.carryLen = 0;
}
__device__ __forceinline__ uint32_t fr_vrd32(const uint8_t* stash, int have, const uint8_t* p, int64_t q, int64_t j) {
    return fr_vbyte(stash, have, p, q, j) | (fr_vbyte(stash, have, p, q, j + 1) << 8) |
           (fr_vbyte(stash, have, p, q, j + 2) << 16) | (fr_vbyte(stash, have, p, q, j + 3) << 24);
}

// One thread per entry.  Pass 0 counts the rows (FrameRec.nb; nslot = nb when the output is staged densely);
// pass 1, after frame_scan_kernel, walks again and writes the rows, the copies, the stream's new phase and, for a
// frame it opens, a fresh content checksum state.  spent (nullable): blocks earlier sub-reads of the same read
// decoded.  stageOff (nullable): the output goes to stageOff[i] = FrameRec.slot * stageSlot instead of dstOff[i].
// A verdict before any row is FrameRec.status (header, sticky error, stream out of range); one at row k is the
// error key (k << 4) | kind in FrameRec.err, as frame.cuh keeps it.  skipEnt[i]: the skipped block's bytes in the
// chunk, for frame_writer_xxh_kernel over bxs (stream -1: none).
__global__ void frame_reader_plan_kernel(int pass, const int32_t* __restrict__ streams, const uint8_t* __restrict__ srcBase,
                                         const int64_t* __restrict__ srcOff, const int32_t* __restrict__ srcLen,
                                         const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                                         const int32_t* __restrict__ spent, int n, int nStreams, int32_t maxBlockSize,
                                         int32_t stashBody, int64_t stashStride, int64_t stashRel,
                                         const uint8_t* __restrict__ stash, FrState* __restrict__ st,
                                         FwState* __restrict__ xs, FwState* __restrict__ bxs, FwEntry* __restrict__ skipEnt,
                                         FrameRec* __restrict__ fr, FrEntry* __restrict__ ent,
                                         FrameTable t, FrCopies c, int64_t* __restrict__ stageOff, int64_t stageSlot,
                                         FrameTotals* __restrict__ tot, int32_t* __restrict__ kinds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    FrameRec r = {};
    r.err = FK_NONE;
    if (pass == 1) { r.first = fr[i].first; r.slot = fr[i].slot; }
    FrEntry e = {};
    e.stream = s >= 0 && s < nStreams ? s : -1;
    e.start = stageOff ? r.slot * stageSlot : dstOff[i];
    int64_t q = 0, tailFrom = -1, tailAt = 0;
    int rows = 0;
    bool opened = false, skipStart = false;
    FwEntry sk = {};
    sk.stream = -1;
    FrState S = {};
    if (e.stream < 0) r.status = FR_ARG;
    else {
        S = st[s];
        r.status = S.err;
    }
    if (!r.status) {
        const uint8_t* p = srcBase + srcOff[i];
        const uint8_t* sp = stash + (int64_t)s * stashStride;
        const int64_t L = srcLen[i] > 0 ? srcLen[i] : 0;
        int64_t budget = -1;
        for (;;) {
            if (S.phase == FP_IDLE) {
                if (q >= L) break;
                S.phase = FP_HEADER;
                S.have = 0;
            }
            if (S.phase == FP_HEADER) {
                // the magic is judged at 4 bytes, the rest once the header (7 or 15 bytes) is complete
                int v = 0;
                bool done = false;
                for (;;) {
                    const int need = S.have < 4 ? 4 : S.have < 7 ? 7 : (S.hbuf[4] & 8) ? 15 : 7;
                    while (S.have < need && q < L) S.hbuf[S.have++] = p[q++];
                    if (S.have < need) break;
                    if (need == 4) {
                        if (fr_rd32(S.hbuf) != FRAME_MAGIC) { v = FR_CORRUPT; break; }
                        continue;
                    }
                    int64_t hp;
                    int flg, bd;
                    v = frame_header_check(S.hbuf, S.have, &hp, &flg, &bd);
                    if (v == FR_CORRUPT && hp + 1 > S.have) { v = 0; continue; }
                    if (!v && frame_max_block((bd >> 4) & 7) > maxBlockSize) v = FR_DELEGATE;
                    if (!v) { S.flags = frame_flags_of(flg); S.maxBlock = frame_max_block((bd >> 4) & 7); done = true; }
                    break;
                }
                if (v) { r.status = v; break; }
                if (!done) break;
                S.phase = FP_BLOCK;
                S.have = 0;
                opened = true;
            }
            if (S.phase == FP_BLOCK) {
                const bool linked = !(S.flags & FR_INDEPENDENT), bc = S.flags & FR_BLOCK_SUM;
                const int64_t cap = linked ? S.maxBlock : (int64_t)S.maxBlock + 8;
                if (budget < 0) budget = (dstCap[i] > 0 ? dstCap[i] : 0) / cap - (spent ? spent[i] : 0);
                const int64_t avail = S.have + (L - q);
                if (avail < 4) {
                    if (rows >= budget) break;          // stops before the length code
                    tailFrom = q; tailAt = S.have; S.have = (int32_t)avail; q = L;
                    break;
                }
                const uint32_t code = fr_vrd32(sp, S.have, p, q, 0);
                if (code == 0) {                        // the end mark: consumed whatever the budget
                    q += 4 - S.have;
                    S.have = 0;
                    if (!(S.flags & FR_CONTENT_SUM)) { S.phase = FP_IDLE; e.ended = 1; break; }
                    S.phase = FP_TAIL;
                } else {
                    if (rows >= budget) break;
                    const int64_t blen = code & 0x7FFFFFFFu;
                    const bool raw = code >> 31;
                    // a stored block larger than the decoder takes: R_CORRUPT whatever follows (a truncation or a
                    // checksum mismatch in it is R_CORRUPT too)
                    if (raw && blen > cap) {
                        r.err = ((unsigned long long)rows << 4) | FK_RAW;
                        break;
                    }
                    // a compressed block too long to decode within blockCap (frame_lb(stashBody + 1) >
                    // maxBlockSize + 8): its body is skipped and hashed, its checksum then decides
                    if (!raw && blen > stashBody) {
                        q += 4 - S.have;
                        S.have = 0;
                        S.skip = (int32_t)blen;
                        S.phase = FP_SKIP;
                        skipStart = true;
                        continue;
                    }
                    const int64_t total = 4 + blen + (bc ? 4 : 0);
                    if (avail < total) {
                        tailFrom = q; tailAt = S.have; S.have = (int32_t)avail; q = L;
                        break;
                    }
                    if (pass == 1) {
                        const int64_t b = r.first + rows;
                        t.srcOff[b] = S.have ? stashRel + (int64_t)s * stashStride + 4 : srcOff[i] + q + 4;
                        t.len[b] = (int32_t)blen;
                        t.kind[b] = raw ? RK_RAW : 0;
                        t.sum[b] = bc ? fr_vrd32(sp, S.have, p, q, 4 + blen) : 0;
                        t.ckLen[b] = bc ? (int32_t)blen : 0;
                        if (S.have) {
                            c.upOff[i] = srcOff[i] + q;
                            c.upDst[i] = (int64_t)s * stashStride + S.have;
                            c.upLen[i] = (int32_t)(total - S.have);
                        }
                    }
                    q += total - S.have;
                    S.have = 0;
                    rows++;
                    continue;
                }
            }
            if (S.phase == FP_SKIP) {
                const bool bc = S.flags & FR_BLOCK_SUM;
                const int64_t take = S.skip < L - q ? S.skip : L - q;
                if (bc && take > 0) { sk.srcOff = srcOff[i] + q; sk.len = (int32_t)take; sk.stream = s; }
                q += take;
                S.skip -= (int32_t)take;
                if (S.skip > 0) break;
                if (!bc) { r.err = ((unsigned long long)rows << 4) | FK_BLOCK; break; }
                while (S.have < 4 && q < L) S.hbuf[S.have++] = p[q++];
                if (S.have < 4) break;
                r.expect = fr_rd32(S.hbuf);
                e.check = 2;
                break;
            }
            if (S.phase == FP_TAIL) {
                while (S.have < 4 && q < L) S.hbuf[S.have++] = p[q++];
                if (S.have < 4) break;
                r.expect = fr_rd32(S.hbuf);
                e.check = 1; e.ended = 1;
                S.phase = FP_IDLE; S.have = 0;
                break;
            }
        }
    }
    r.nb = rows;
    r.flags = S.flags;
    r.maxBlock = S.maxBlock;
    e.used = r.status ? 0 : q;
    if (pass == 0) {
        r.nslot = stageOff ? rows : 0;
        fr[i] = r;
        if (sk.stream >= 0) atomicOr(kinds, FRK_SKIP);
        if (rows > 0) {
            atomicMax(&tot->maxSteps, rows);
            atomicOr(kinds, ((S.flags & FR_INDEPENDENT) ? FRK_INDEP : FRK_LINKED) |
                                ((S.flags & FR_BLOCK_SUM) ? FRK_BLOCK_SUM : 0) |
                                ((S.flags & FR_CONTENT_SUM) ? FRK_CONTENT_SUM : 0));
        }
        return;
    }
    r.pos = e.start;
    fr[i] = r;
    ent[i] = e;
    if (stageOff) stageOff[i] = e.start;
    const bool tail = !r.status && tailFrom >= 0;
    c.tailOff[i] = tail ? srcOff[i] + tailFrom : 0;
    c.tailDst[i] = tail ? (int64_t)s * stashStride + tailAt : 0;
    c.tailLen[i] = tail ? (int32_t)(q - tailFrom) : 0;
    skipEnt[i] = sk;
    if (e.stream < 0 || S.err) return;
    st[s] = S;
    if (opened) fr_xxh_reset(xs[s]);
    if (skipStart) fr_xxh_reset(bxs[s]);
}

// The arrays of one step, n entries each.
struct FrStep {
    int64_t* srcOff;         // the stored bytes, relative to the chunks' base
    int32_t* lenC; int32_t* lenD;   // compressed length for OP_CHAIN (linked) / OP_DECODE (independent), else 0
    int32_t* resC; int32_t* resD;   // their results
    int32_t* kind;           // 0: no block; 1: raw; 2: compressed
    int32_t* res;            // the bytes the block added (the commit's outLen)
    int64_t* gDst; int32_t* gLen;   // gather: slot -> cursor
    FwEntry* xe;             // content checksum: the slot's bytes (frame_writer_xxh_kernel)
};

// Step k, before the codec: block k of every entry that has one and no verdict at or before it.  Its checksum
// (verified by xxh32_batch_kernel over all rows) is checked first, then the block goes to the codec table -- the
// slot at ring + pos (pos 0 for independent frames), the reference's capacity, the history min(pos, 64 KiB) --
// or, raw, to the copy into the slot (t.copyOff / copyLen).
__global__ void frame_reader_step_kernel(int k, FrameRec* __restrict__ fr, const FrEntry* __restrict__ ent, int n,
                                         FrameTable rows, const ChainGroupHdr* __restrict__ hdr, int64_t ring,
                                         ChainGroupTable t, FrStep s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FrameRec& r = fr[i];
    int32_t kind = 0, len = 0, cap = 0, pre = 0;
    int64_t at = 0, src = 0;
    const bool linked = !(r.flags & FR_INDEPENDENT);
    if (k < r.nb && !r.status && (r.err >> 4) > (unsigned long long)k) {
        const int64_t b = r.first + k;
        if (rows.ckLen[b] > 0 && rows.got[b] != rows.sum[b]) {
            fr[i].err = ((unsigned long long)k << 4) | FK_SUM;
        } else {
            const int sm = ent[i].stream;
            const int64_t pos = linked ? hdr[sm].pos : 0;
            at = (int64_t)sm * ring + pos;
            src = rows.srcOff[b];
            len = rows.len[b];
            kind = (rows.kind[b] & RK_RAW) ? 1 : 2;
            cap = linked ? r.maxBlock : r.maxBlock + 8;
            pre = (int32_t)(pos < CG_WINDOW ? pos : CG_WINDOW);
        }
    }
    s.srcOff[i] = src;
    s.kind[i] = kind;
    s.lenC[i] = kind == 2 && linked ? len : 0;
    s.lenD[i] = kind == 2 && !linked ? len : 0;
    t.ringOff[i] = at;
    t.len[i] = kind == 2 ? cap : 0;
    t.prefix[i] = kind == 2 && linked ? pre : 0;
    t.copyOff[i] = src;
    t.copyLen[i] = kind == 1 ? len : 0;
}

// Step k, after the codec: a rejected block is the verdict -1 at row k; an accepted one is gathered to the cursor,
// hashed into the content checksum and, in a linked frame, committed to the ring.
__global__ void frame_reader_post_kernel(int k, FrameRec* __restrict__ fr, const FrEntry* __restrict__ ent, int n,
                                         ChainGroupTable t, FrStep s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int kind = s.kind[i];
    const int flags = fr[i].flags;
    int32_t res = 0;
    if (kind == 1) res = t.copyLen[i];
    else if (kind == 2) res = (flags & FR_INDEPENDENT) ? s.resD[i] : s.resC[i];
    const bool ok = kind != 0 && res >= 0;
    if (kind == 2 && res < 0) fr[i].err = ((unsigned long long)k << 4) | FK_BLOCK;
    int64_t cur = fr[i].pos;
    s.gDst[i] = cur;
    s.gLen[i] = ok ? res : 0;
    if (ok) fr[i].pos = cur + res;
    s.res[i] = ok ? res : 0;
    t.stream[i] = ok && !(flags & FR_INDEPENDENT) ? ent[i].stream : -1;
    FwEntry x = {};
    x.srcOff = t.ringOff[i];
    x.len = ok ? res : 0;
    x.stream = ok && (flags & FR_CONTENT_SUM) ? ent[i].stream : -1;
    s.xe[i] = x;
}

// The end of a read: the content checksum of a frame it ended, the verdict (the smallest key; frame.cuh's codes),
// outLen = the bytes appended or the verdict, srcUsed, frameEnded, and the stream's state: failed (sticky), or,
// after a frame's end, an empty ring.  rowsOut (nullable): the blocks decoded, for the next sub-read.
__global__ void frame_reader_finish_kernel(const FrameRec* __restrict__ fr, const FrEntry* __restrict__ ent, int n,
                                           FrState* __restrict__ st, const FwState* __restrict__ xs,
                                           const FwState* __restrict__ bxs,
                                           ChainGroupHdr* __restrict__ hdr, int32_t* __restrict__ outLen,
                                           int32_t* __restrict__ srcUsed, int32_t* __restrict__ frameEnded,
                                           int32_t* __restrict__ rowsOut) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const FrameRec r = fr[i];
    const FrEntry e = ent[i];
    const int s = e.stream;
    int32_t out;
    if (r.status) out = r.status;
    else {
        unsigned long long key = r.err;
        const unsigned long long at = (unsigned long long)r.nb << 4;
        if (e.check == 1 && fr_digest(xs[s]) != r.expect && (at | FK_SUM) < key) key = at | FK_SUM;
        if (e.check == 2) {              // the skipped block: its checksum, else the decoder's verdict
            const unsigned long long k2 = at | (fr_digest(bxs[s]) != r.expect ? FK_SUM : FK_BLOCK);
            if (k2 < key) key = k2;
        }
        if (key != FK_NONE) out = (key & 15) == FK_BLOCK ? -1 : FR_CORRUPT;
        else out = (int32_t)(r.pos - e.start);
    }
    if (s >= 0) {
        if (out < 0) st[s].err = out;
        else if (e.ended) hdr[s].pos = 0;
    }
    outLen[i] = out;
    srcUsed[i] = out < 0 ? 0 : (int32_t)e.used;
    frameEnded[i] = out < 0 ? 0 : e.ended;
    if (rowsOut) rowsOut[i] = r.nb;
}

// End (status non-null) or reset: the stream's verdict -- 0 between frames, R_CORRUPT inside one, its sticky
// error when failed, K4LZ4_E_ARG for an index out of range -- and it becomes new.
__global__ void frame_reader_end_kernel(const int32_t* __restrict__ streams, int n, int nStreams,
                                        FrState* __restrict__ st, ChainGroupHdr* __restrict__ hdr,
                                        int32_t* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    if (s < 0 || s >= nStreams) {
        if (status) status[i] = FR_ARG;
        return;
    }
    FrState& S = st[s];
    if (status) status[i] = S.err ? S.err : S.phase == FP_IDLE ? 0 : FR_CORRUPT;
    S.phase = FP_IDLE;
    S.have = 0;
    S.err = 0;
    hdr[s].pos = 0;
}

// ---- byte-granular reads (k4lz4_frame_reader_group_read_bytes) -------------------------------------------------
//
// ReadManyBytes (Streams/Frames/LZ4FrameReader.blocking.cs:157-179) for the push contract: a read first drains the
// rest of the stream's current decoded block, then decodes blocks while room is left, appending as much of each as
// fits; what does not fit stays undrained in the ring for the next read.  The room a block takes is its decoded
// size, so a read plans in two steps, both before anything decodes:
//
// * The plan (one thread per entry, count and fill passes around frame_scan_kernel) continues the stream's phase
//   like frame_reader_plan_kernel, but takes candidate rows until the lower bounds frame_lb of their sizes cover
//   the room left after the drain (one row in interactive mode).  Its stops and the stream's state at the first
//   length code of the call go to an FrCut; the stream's state itself is not written.
// * block_size_walk_kernel gives each candidate's exact size (the lower bound for a chain that does not parse: the
//   decoder rejects that block wherever the cut falls), and the cut kernel replays the reference's loop over the
//   sizes: the rows that decode, whether the plan's last step (end mark, cut block, skipped block, raw block above
//   its limit) is reached, the stream's new phase, `have`, stash tail and undrained length.  Rows it does not reach
//   are neither checksummed nor decoded.
//
// The undrained bytes are the last FrDrain.len bytes in front of FrDrain.end in the stream's ring.  While a stream
// holds any, its FrState.err is FR_ARG: frame_reader_plan_kernel then answers a plain read K4LZ4_E_ARG and consumes
// nothing, and only byte reads, end and reset clear it.  Slides: a linked block that leaves at most 64 KiB
// undrained slides at once (its undrained bytes stay the last ones in front of pos); one that leaves more keeps
// pos beyond RING - SLOT and slides when a later read has drained it, before anything else decodes.

struct FrDrain {             // per stream: the undrained rest of its current block, ring[end - len, end)
    int64_t end;
    int32_t len;
    int32_t reserved;
};

struct FrCut {               // per entry of a byte read: what its plan found, for the cut kernel
    FrState at;              // the stream at its first length code of the call (its phase is FP_BLOCK)
    FrState fin;             // the stream after the plan's last step
    FwEntry sk;              // the skipped block's bytes in the chunk, if the last step skips one
    unsigned long long err;  // the plan's error key (a raw block above its limit)
    int64_t q0, qFin;        // chunk bytes consumed before the first length code / by the whole plan
    int64_t tailFrom;        // the plan's tail copy: source in srcBase (-1: none), stash offset, length
    int32_t tailAt, tailLen;
    int32_t drain, take;     // undrained bytes at the start, and how many of them this read appends
    int32_t room;            // dstCap - take
    int32_t gated;           // the plan met a length code, so the loop must reach its last step
    int32_t go;              // the loop reaches the first length code (room left, nothing appended interactively)
    int32_t opened, skipStart, check, ended;
};

// The copies a byte read makes before its first step: the drain (ring -> the entry's output) and a pending slide.
struct FrPre { int64_t* dOff; int64_t* dDst; int32_t* dLen; int64_t* sOff; int64_t* sDst; int32_t* sLen; };

// One thread per entry; pass 0 counts candidate rows (FrameRec.nb); pass 1 writes the rows (t.frame / t.idx for
// the walk, rowEnd = chunk bytes consumed up to the end of each), the stash top-up, the FrCut and, for a frame it
// opens, a fresh content checksum.  staged: the output is placed in a staging buffer once the cut knows its size
// (frame_reader_bytes_place_kernel), so it starts at 0 here instead of dstOff[i].
__global__ void frame_reader_bytes_plan_kernel(int pass, int interactive, const int32_t* __restrict__ streams,
                                               const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                                               const int32_t* __restrict__ srcLen, const int64_t* __restrict__ dstOff,
                                               const int32_t* __restrict__ dstCap, int n, int nStreams,
                                               int32_t maxBlockSize, int32_t stashBody, int64_t stashStride,
                                               int64_t stashRel, const uint8_t* __restrict__ stash,
                                               const FrState* __restrict__ st, const FrDrain* __restrict__ drain,
                                               FwState* __restrict__ xs, FrameRec* __restrict__ fr,
                                               FrEntry* __restrict__ ent, FrCut* __restrict__ cut, FrameTable t,
                                               int64_t* __restrict__ rowEnd, FrCopies c, int staged,
                                               FrameTotals* __restrict__ tot, int32_t* __restrict__ kinds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    FrameRec r = {};
    r.err = FK_NONE;
    if (pass == 1) { r.first = fr[i].first; r.slot = fr[i].slot; }
    FrEntry e = {};
    e.stream = s >= 0 && s < nStreams ? s : -1;
    e.start = staged ? 0 : dstOff[i];
    FrCut u = {};
    u.tailFrom = -1;
    u.sk.stream = -1;
    int64_t q = 0, lbSum = 0;
    int rows = 0;
    FrState S = {};
    if (e.stream < 0) r.status = FR_ARG;
    else {
        S = st[s];
        r.status = S.err == FR_ARG ? 0 : S.err;
    }
    const int64_t cap0 = dstCap[i] > 0 ? dstCap[i] : 0;
    u.drain = !r.status && S.err == FR_ARG ? drain[s].len : 0;
    u.take = (int32_t)(cap0 < u.drain ? cap0 : u.drain);
    const int64_t room = cap0 - u.take;
    if (!r.status) {
        const uint8_t* p = srcBase + srcOff[i];
        const uint8_t* sp = stash + (int64_t)s * stashStride;
        const int64_t L = srcLen[i] > 0 ? srcLen[i] : 0;
        for (;;) {
            if (S.phase == FP_IDLE) {
                if (q >= L) break;
                S.phase = FP_HEADER;
                S.have = 0;
            }
            if (S.phase == FP_HEADER) {             // EnsureHeader: before the loop, whatever the room
                int v = 0;
                bool done = false;
                for (;;) {
                    const int need = S.have < 4 ? 4 : S.have < 7 ? 7 : (S.hbuf[4] & 8) ? 15 : 7;
                    while (S.have < need && q < L) S.hbuf[S.have++] = p[q++];
                    if (S.have < need) break;
                    if (need == 4) {
                        if (fr_rd32(S.hbuf) != FRAME_MAGIC) { v = FR_CORRUPT; break; }
                        continue;
                    }
                    int64_t hp;
                    int flg, bd;
                    v = frame_header_check(S.hbuf, S.have, &hp, &flg, &bd);
                    if (v == FR_CORRUPT && hp + 1 > S.have) { v = 0; continue; }
                    if (!v && frame_max_block((bd >> 4) & 7) > maxBlockSize) v = FR_DELEGATE;
                    if (!v) { S.flags = frame_flags_of(flg); S.maxBlock = frame_max_block((bd >> 4) & 7); done = true; }
                    break;
                }
                if (v) { r.status = v; break; }
                if (!done) break;
                S.phase = FP_BLOCK;
                S.have = 0;
                u.opened = 1;
            }
            if (S.phase == FP_BLOCK) {
                if (!u.gated) {
                    u.gated = 1;
                    u.at = S;
                    u.q0 = q;
                    u.go = room > 0 && !(interactive && u.take > 0);
                }
                // the candidates: the loop can reach this length code only if the rows before it may leave room
                if (rows == 0 ? !u.go : (interactive || lbSum >= room)) break;
                const bool bc = S.flags & FR_BLOCK_SUM;
                const int64_t cap = (S.flags & FR_INDEPENDENT) ? (int64_t)S.maxBlock + 8 : S.maxBlock;
                const int64_t avail = S.have + (L - q);
                if (avail < 4) {
                    u.tailFrom = q; u.tailAt = S.have; S.have = (int32_t)avail; q = L;
                    break;
                }
                const uint32_t code = fr_vrd32(sp, S.have, p, q, 0);
                if (code == 0) {
                    q += 4 - S.have;
                    S.have = 0;
                    if (!(S.flags & FR_CONTENT_SUM)) { S.phase = FP_IDLE; u.ended = 1; break; }
                    S.phase = FP_TAIL;
                } else {
                    const int64_t blen = code & 0x7FFFFFFFu;
                    const bool raw = code >> 31;
                    if (raw && blen > cap) {
                        r.err = ((unsigned long long)rows << 4) | FK_RAW;
                        break;
                    }
                    if (!raw && blen > stashBody) {
                        q += 4 - S.have;
                        S.have = 0;
                        S.skip = (int32_t)blen;
                        S.phase = FP_SKIP;
                        u.skipStart = 1;
                        continue;
                    }
                    const int64_t total = 4 + blen + (bc ? 4 : 0);
                    if (avail < total) {
                        u.tailFrom = q; u.tailAt = S.have; S.have = (int32_t)avail; q = L;
                        break;
                    }
                    if (pass == 1) {
                        const int64_t b = r.first + rows;
                        t.srcOff[b] = S.have ? stashRel + (int64_t)s * stashStride + 4 : srcOff[i] + q + 4;
                        t.len[b] = (int32_t)blen;
                        t.kind[b] = raw ? RK_RAW : 0;
                        t.sum[b] = bc ? fr_vrd32(sp, S.have, p, q, 4 + blen) : 0;
                        t.ckLen[b] = bc ? (int32_t)blen : 0;
                        t.frame[b] = i;
                        t.idx[b] = rows;
                        rowEnd[b] = q + total - S.have;
                        if (S.have) {
                            c.upOff[i] = srcOff[i] + q;
                            c.upDst[i] = (int64_t)s * stashStride + S.have;
                            c.upLen[i] = (int32_t)(total - S.have);
                        }
                    }
                    lbSum += frame_lb(blen, raw);
                    q += total - S.have;
                    S.have = 0;
                    rows++;
                    continue;
                }
            }
            if (S.phase == FP_SKIP) {
                const bool bc = S.flags & FR_BLOCK_SUM;
                const int64_t take = S.skip < L - q ? S.skip : L - q;
                if (bc && take > 0) { u.sk.srcOff = srcOff[i] + q; u.sk.len = (int32_t)take; u.sk.stream = s; }
                q += take;
                S.skip -= (int32_t)take;
                if (S.skip > 0) break;
                if (!bc) { r.err = ((unsigned long long)rows << 4) | FK_BLOCK; break; }
                while (S.have < 4 && q < L) S.hbuf[S.have++] = p[q++];
                if (S.have < 4) break;
                r.expect = fr_rd32(S.hbuf);
                u.check = 2;
                break;
            }
            if (S.phase == FP_TAIL) {
                while (S.have < 4 && q < L) S.hbuf[S.have++] = p[q++];
                if (S.have < 4) break;
                r.expect = fr_rd32(S.hbuf);
                u.check = 1; u.ended = 1;
                S.phase = FP_IDLE; S.have = 0;
                break;
            }
        }
    }
    r.nb = rows;
    r.flags = S.flags;
    r.maxBlock = S.maxBlock;
    if (pass == 0) {
        fr[i] = r;
        if (u.sk.stream >= 0) atomicOr(kinds, FRK_SKIP);
        if (rows > 0) {
            atomicMax(&tot->maxSteps, rows);
            atomicOr(kinds, ((S.flags & FR_INDEPENDENT) ? FRK_INDEP : FRK_LINKED) |
                                ((S.flags & FR_BLOCK_SUM) ? FRK_BLOCK_SUM : 0) |
                                ((S.flags & FR_CONTENT_SUM) ? FRK_CONTENT_SUM : 0));
        }
        return;
    }
    r.pos = e.start;
    u.fin = S;
    u.qFin = q;
    u.err = r.err;
    u.room = (int32_t)room;
    if (u.tailFrom >= 0) { u.tailLen = (int32_t)(q - u.tailFrom); u.tailFrom += srcOff[i]; }
    if (!u.gated) u.at = S;
    fr[i] = r;
    ent[i] = e;
    cut[i] = u;
    if (u.opened && !r.status) fr_xxh_reset(xs[s]);
}

// One thread per entry, after the walk: the reference's loop over the candidates' sizes -- a row decodes while
// the rows before it left room (and, interactively, appended nothing), and none of them decoded to 0 bytes.  The
// plan's last step counts only when the loop reaches it (always, when the call met no length code).  Writes the
// rows to decode (FrameRec.nb), srcUsed, the stream's state, the tail copy, the skipped bytes to hash, the drain
// copy, a pending slide, `stopped` (the loop stopped on room, interactive mode or an empty block) and zeroes the
// checksum lengths of the rows left over.  place (nullable, staged output): FrameRec.nslot = the bytes the entry
// appends (the rows' walked sizes; a row the decoder rejects appends less) in 16-byte units, nb = 0, for
// frame_scan_kernel.
__global__ void frame_reader_bytes_cut_kernel(int interactive, FrameRec* __restrict__ fr, FrEntry* __restrict__ ent,
                                              const FrCut* __restrict__ cut, int n, FrameTable t,
                                              const int64_t* __restrict__ rowEnd, FrState* __restrict__ st,
                                              FwState* __restrict__ bxs, FwEntry* __restrict__ skipEnt,
                                              FrDrain* __restrict__ drain, ChainGroupHdr* __restrict__ hdr,
                                              int64_t ring, int64_t slot, int64_t stashStride, FrCopies c, FrPre pre,
                                              int32_t* __restrict__ stopped, FrameRec* __restrict__ place) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (place) place[i] = FrameRec{};
    FrameRec r = fr[i];
    FrEntry e = ent[i];
    const FrCut& u = cut[i];
    const int s = e.stream;
    FwEntry sk = {};
    sk.stream = -1;
    c.tailOff[i] = 0; c.tailDst[i] = 0; c.tailLen[i] = 0;
    pre.dOff[i] = 0; pre.dDst[i] = 0; pre.dLen[i] = 0;
    pre.sOff[i] = 0; pre.sDst[i] = 0; pre.sLen[i] = 0;
    if (r.status) {
        skipEnt[i] = sk;
        stopped[i] = 1;
        return;
    }
    int nb = 0;
    bool go = u.gated ? u.go : true;
    int64_t room = u.room;
    for (; nb < r.nb && go; nb++) {
        const int64_t size = t.size[r.first + nb];
        room -= size;
        go = room > 0 && !interactive && size > 0;
    }
    for (int k = nb; k < r.nb; k++) t.ckLen[r.first + k] = 0;
    const bool reached = nb == r.nb && go;
    FrState S;
    if (reached) {
        S = u.fin;
        e.used = u.qFin;
        e.ended = u.ended;
        e.check = u.check;
        r.err = u.err;
        if (u.tailFrom >= 0) {
            c.tailOff[i] = u.tailFrom;
            c.tailDst[i] = (int64_t)s * stashStride + u.tailAt;
            c.tailLen[i] = u.tailLen;
        }
        sk = u.sk;
        if (u.skipStart) fr_xxh_reset(bxs[s]);
    } else {
        S = u.at;
        if (nb > 0) S.have = 0;
        e.used = nb > 0 ? rowEnd[r.first + nb - 1] : u.q0;
        e.ended = 0;
        e.check = 0;
        r.err = FK_NONE;
    }
    skipEnt[i] = sk;
    stopped[i] = !reached;
    if (place) {
        const int64_t out = u.take + (nb > 0 ? u.room - (room > 0 ? room : 0) : 0);
        place[i].nslot = (int32_t)((out + 15) >> 4);
    }
    // the undrained bytes after the call: the last row's rest, or what the drain left
    const int32_t left = nb > 0 ? (int32_t)(room < 0 ? -room : 0) : u.drain - u.take;
    if (u.take > 0) {
        const FrDrain d = drain[s];
        pre.dOff[i] = (int64_t)s * ring + d.end - u.drain;
        pre.dDst[i] = e.start;
        pre.dLen[i] = u.take;
    }
    if (nb == 0) drain[s].len = left;      // else each row's commit sets it
    // a slide deferred while more than 64 KiB were undrained: once they are drained, before anything decodes
    if (u.drain > 0 && u.drain == u.take && !(r.flags & FR_INDEPENDENT) && hdr[s].pos + slot > ring) {
        pre.sOff[i] = (int64_t)s * ring + hdr[s].pos - CG_WINDOW;
        pre.sDst[i] = (int64_t)s * ring;
        pre.sLen[i] = (int32_t)CG_WINDOW;
        hdr[s].pos = CG_WINDOW;
    }
    S.err = left > 0 ? FR_ARG : 0;
    st[s] = S;
    r.nb = nb;
    r.pos = e.start + u.take;
    fr[i] = r;
    ent[i] = e;
}

// Staged output, after frame_scan_kernel over `place`: entry i's output starts at byte 16 * place[i].slot of the
// staging buffer; its cursor, its drain copy's destination and stageOff[i] move there.
__global__ void frame_reader_bytes_place_kernel(const FrameRec* __restrict__ place, FrameRec* __restrict__ fr,
                                                FrEntry* __restrict__ ent, FrPre pre, int64_t* __restrict__ stageOff,
                                                int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t at = place[i].slot * 16;
    fr[i].pos += at;
    ent[i].start += at;
    pre.dDst[i] += at;
    stageOff[i] = at;
}

// Step k of a byte read, after the codec: as frame_reader_post_kernel, but the gather takes only what fits in the
// room left (dstCap here is the entry's), and every accepted block -- linked or independent -- goes to the commit.
__global__ void frame_reader_bytes_post_kernel(int k, FrameRec* __restrict__ fr, const FrEntry* __restrict__ ent,
                                               const int32_t* __restrict__ dstCap, int n, ChainGroupTable t, FrStep s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int kind = s.kind[i];
    const int flags = fr[i].flags;
    int32_t res = 0;
    if (kind == 1) res = t.copyLen[i];
    else if (kind == 2) res = (flags & FR_INDEPENDENT) ? s.resD[i] : s.resC[i];
    const bool ok = kind != 0 && res >= 0;
    if (kind == 2 && res < 0) fr[i].err = ((unsigned long long)k << 4) | FK_BLOCK;
    const int64_t cur = fr[i].pos;
    const int64_t left = (int64_t)(dstCap[i] > 0 ? dstCap[i] : 0) - (cur - ent[i].start);
    const int32_t take = !ok ? 0 : (int64_t)res < left ? res : (int32_t)(left > 0 ? left : 0);
    s.gDst[i] = cur;
    s.gLen[i] = take;
    fr[i].pos = cur + take;
    s.res[i] = ok ? res : 0;
    t.stream[i] = ok ? ent[i].stream : -1;
    FwEntry x = {};
    x.srcOff = t.ringOff[i];
    x.len = ok ? res : 0;
    x.stream = ok && (flags & FR_CONTENT_SUM) ? ent[i].stream : -1;
    s.xe[i] = x;
}

// Step k of a byte read, after the gather and the content checksum: the stream's undrained rest of the block
// and, in a linked frame, pos += the block and the slide -- unless more than 64 KiB stay undrained, whose slide
// the cut kernel makes once they are drained.  t.copyOff / ringOff / copyLen: the slide, for copy_blocks_kernel.
__global__ void frame_reader_bytes_commit_kernel(const FrameRec* __restrict__ fr, int n, int64_t ring, int64_t slot,
                                                 ChainGroupHdr* __restrict__ hdr, FrDrain* __restrict__ drain,
                                                 ChainGroupTable t, FrStep s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int sm = t.stream[i];
    int32_t slide = 0;
    if (sm >= 0) {
        const int32_t res = s.res[i], left = res - s.gLen[i];
        int64_t end;
        if (fr[i].flags & FR_INDEPENDENT) end = t.ringOff[i] - (int64_t)sm * ring + res;
        else {
            end = hdr[sm].pos + res;
            if (end + slot > ring && left <= CG_WINDOW) {
                t.copyOff[i] = (int64_t)sm * ring + end - CG_WINDOW;
                t.ringOff[i] = (int64_t)sm * ring;
                slide = (int32_t)CG_WINDOW;
                end = CG_WINDOW;
            }
            hdr[sm].pos = end;
        }
        drain[sm].end = end;
        drain[sm].len = left;
    }
    t.copyLen[i] = slide;
}

// Before frame_reader_end_kernel in an end or reset: the stream's undrained bytes go, and with them the FR_ARG
// mark, so that an end inside a frame reports R_CORRUPT.
__global__ void frame_reader_bytes_end_kernel(const int32_t* __restrict__ streams, int n, int nStreams,
                                              FrState* __restrict__ st, FrDrain* __restrict__ drain) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    if (s < 0 || s >= nStreams) return;
    if (st[s].err == FR_ARG) st[s].err = 0;
    drain[s].len = 0;
}

}  // namespace k4
