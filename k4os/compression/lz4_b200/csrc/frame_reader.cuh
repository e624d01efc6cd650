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
// continues the stream's phase over the chunk, hops over the length codes under the read's room rule and writes
// one row per block it completes -- stored bytes in the chunk, or in the stash for the one block a previous chunk
// began.  The rows' checksums are verified by xxh32_batch_kernel before anything decodes; then step k decodes
// block k of every entry into its slot, gathers it to the entry's cursor, advances the content XXH32 and commits
// the ring.  The finish kernel gives the verdicts, and the unconsumed tail of a cut block is copied into the stash
// last.
//
// Two kinds of reads share all of this and differ in their room rule:
//
// * A plain read (k4lz4_frame_reader_group_read) decodes whole blocks only, at most floor(dstCap / blockCap) of
//   them per call (blockCap = the reference decoder's capacity).
// * A byte read (k4lz4_frame_reader_group_read_bytes) is ReadManyBytes (Streams/Frames/LZ4FrameReader.blocking.cs:
//   157-179) for the push contract: it first drains the rest of the stream's current decoded block, then decodes
//   blocks while room is left, appending as much of each as fits; what does not fit stays undrained in the ring
//   for the next read.  The room a block takes is its decoded size, so its plan takes candidate rows until the
//   lower bounds frame_lb of their sizes cover the room left after the drain (one row in interactive mode); its
//   stops and the stream's state at the first length code of the call go to an FrCut, and the stream's state
//   itself is not written.  block_size_walk_kernel then gives each candidate's exact size (the lower bound for a
//   chain that does not parse: the decoder rejects that block wherever the cut falls), and the cut kernel replays
//   the reference's loop over the sizes: the rows that decode, whether the plan's last step (end mark, cut block,
//   skipped block, raw block above its limit) is reached, the stream's new phase, `have`, stash tail and
//   undrained length.  Rows it does not reach are neither checksummed nor decoded.
//
// The undrained bytes are the last FrDrain.len bytes in front of FrDrain.end in the stream's ring.  While a stream
// holds any, its FrState.err is FR_ARG: a plain read then gets K4LZ4_E_ARG and consumes nothing, and only byte
// reads, end and reset clear it.  Slides: a linked block that leaves at most 64 KiB undrained slides at once (its
// undrained bytes stay the last ones in front of pos); one that leaves more keeps pos beyond RING - SLOT and slides
// when a later read has drained it, before anything else decodes.
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

// Copies the plan orders from the chunk into the stash: the rest of a block a previous chunk began (before the
// checksums) and the tail of the chunk when it ends inside a block (after every decode).
struct FrCopies { int64_t* upOff; int64_t* upDst; int32_t* upLen; int64_t* tailOff; int64_t* tailDst; int32_t* tailLen; };

// The copies a byte read makes before its first step: the drain (ring -> the entry's output) and a pending slide.
struct FrPre { int64_t* dOff; int64_t* dDst; int32_t* dLen; int64_t* sOff; int64_t* sDst; int32_t* sLen; };

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

// The arguments of both plan passes.  t is empty in pass 0.
struct FrPlan {
    const int32_t* streams; const uint8_t* srcBase; const int64_t* srcOff; const int32_t* srcLen;
    const int64_t* dstOff; const int32_t* dstCap;
    int n, nStreams;
    int32_t maxBlockSize, stashBody;
    int64_t stashStride, stashRel;   // stash s is at stash + s * stashStride = srcBase + stashRel + s * stashStride
    const uint8_t* stash;
    FrState* st; FwState* xs; FwState* bxs;
    FrameRec* fr; FrEntry* ent; FrameTable t; FrCopies c;
    FrameTotals* tot; int32_t* kinds;
    int64_t* stageOff;       // nullable: the output is staged (host memory), b.dstOff is not used
    // plain reads
    const int32_t* spent;    // nullable: blocks earlier sub-reads of the same read decoded
    int64_t stageSlot;       // staged: entry i's output at FrameRec.slot * stageSlot
    FwEntry* skipEnt;        // the skipped block's bytes in the chunk, for frame_writer_xxh_kernel over bxs
    // byte reads
    int interactive;
    const FrDrain* drain;
    FrCut* cut;
    int64_t* rowEnd;         // per row: chunk bytes consumed up to its end
};

// One thread per entry.  Pass 0 counts the rows (FrameRec.nb; for a staged plain read nslot = nb, the output
// placed densely by rows); pass 1, after frame_scan_kernel, walks again and writes the rows, the stash top-up and,
// for a frame it opens, a fresh content checksum state.  A verdict before any row is FrameRec.status (header,
// sticky error, stream out of range); one at row k is the error key (k << 4) | kind in FrameRec.err, as frame.cuh
// keeps it.  The room rule and what the walk leaves behind depend on the read:
//
// * Plain (Bytes = false): the room is a budget of floor(dstCap / blockCap) - spent rows, checked before a
//   non-zero length code and before stashing a partial one; an end mark is consumed whatever the budget.  Pass 1
//   writes the stream's new state, the tail copy and skipEnt itself.  A stream with undrained bytes (FR_ARG) gets
//   K4LZ4_E_ARG.
// * Bytes: the room left after the drain gates every length code, the end mark included; rows are taken while
//   their lower bounds are below it.  The rows also carry t.frame / t.idx (for block_size_walk_kernel) and rowEnd;
//   pass 1 writes an FrCut and leaves the stream to the cut kernel.  A staged byte read is placed once the cut
//   knows its size (frame_reader_place_kernel), so its output starts at 0 here.
template <bool Bytes>
__global__ void frame_reader_plan_kernel(int pass, FrPlan a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const int s = a.streams[i];
    FrameRec r = {};
    r.err = FK_NONE;
    if (pass == 1) { r.first = a.fr[i].first; r.slot = a.fr[i].slot; }
    FrEntry e = {};
    e.stream = s >= 0 && s < a.nStreams ? s : -1;
    if (Bytes) e.start = a.stageOff ? 0 : a.dstOff[i];
    else e.start = a.stageOff ? r.slot * a.stageSlot : a.dstOff[i];
    FrState S = {};
    if (e.stream < 0) r.status = FR_ARG;
    else {
        S = a.st[s];
        r.status = Bytes && S.err == FR_ARG ? 0 : S.err;
    }
    const int64_t cap0 = a.dstCap[i] > 0 ? a.dstCap[i] : 0;
    FrCut u = {};
    int64_t room = 0, lbSum = 0, budget = -1;
    if (Bytes) {
        u.drain = !r.status && S.err == FR_ARG ? a.drain[s].len : 0;
        u.take = (int32_t)(cap0 < u.drain ? cap0 : u.drain);
        room = cap0 - u.take;
    }
    int64_t q = 0, tailFrom = -1;
    int32_t tailAt = 0, check = 0, ended = 0;
    int rows = 0;
    bool opened = false, skipStart = false;
    FwEntry sk = {};
    sk.stream = -1;
    if (!r.status) {
        const uint8_t* p = a.srcBase + a.srcOff[i];
        const uint8_t* sp = a.stash + (int64_t)s * a.stashStride;
        const int64_t L = a.srcLen[i] > 0 ? a.srcLen[i] : 0;
        for (;;) {
            if (S.phase == FP_IDLE) {
                if (q >= L) break;
                S.phase = FP_HEADER;
                S.have = 0;
            }
            if (S.phase == FP_HEADER) {
                // the magic is judged at 4 bytes, the rest once the header (7 or 15 bytes) is complete; a byte read
                // (EnsureHeader) reads it before its loop, whatever the room
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
                    if (!v && frame_max_block((bd >> 4) & 7) > a.maxBlockSize) v = FR_DELEGATE;
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
                const bool bc = S.flags & FR_BLOCK_SUM;
                const int64_t cap = (S.flags & FR_INDEPENDENT) ? (int64_t)S.maxBlock + 8 : S.maxBlock;
                bool full = false;
                if (Bytes) {
                    if (!u.gated) {
                        u.gated = 1;
                        u.at = S;
                        u.q0 = q;
                        u.go = room > 0 && !(a.interactive && u.take > 0);
                    }
                    // the candidates: the loop can reach this length code only if the rows before it may leave room
                    if (rows == 0 ? !u.go : (a.interactive || lbSum >= room)) break;
                } else {
                    if (budget < 0) budget = cap0 / cap - (a.spent ? a.spent[i] : 0);
                    full = rows >= budget;
                }
                const int64_t avail = S.have + (L - q);
                if (avail < 4) {
                    if (full) break;                    // stops before the length code
                    tailFrom = q; tailAt = S.have; S.have = (int32_t)avail; q = L;
                    break;
                }
                const uint32_t code = fr_vrd32(sp, S.have, p, q, 0);
                if (code == 0) {                        // the end mark: a plain read consumes it whatever the budget
                    q += 4 - S.have;
                    S.have = 0;
                    if (!(S.flags & FR_CONTENT_SUM)) { S.phase = FP_IDLE; ended = 1; break; }
                    S.phase = FP_TAIL;
                } else {
                    if (full) break;
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
                    if (!raw && blen > a.stashBody) {
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
                        a.t.srcOff[b] = S.have ? a.stashRel + (int64_t)s * a.stashStride + 4 : a.srcOff[i] + q + 4;
                        a.t.len[b] = (int32_t)blen;
                        a.t.kind[b] = raw ? RK_RAW : 0;
                        a.t.sum[b] = bc ? fr_vrd32(sp, S.have, p, q, 4 + blen) : 0;
                        a.t.ckLen[b] = bc ? (int32_t)blen : 0;
                        if (Bytes) {
                            a.t.frame[b] = i;
                            a.t.idx[b] = rows;
                            a.rowEnd[b] = q + total - S.have;
                        }
                        if (S.have) {
                            a.c.upOff[i] = a.srcOff[i] + q;
                            a.c.upDst[i] = (int64_t)s * a.stashStride + S.have;
                            a.c.upLen[i] = (int32_t)(total - S.have);
                        }
                    }
                    if (Bytes) lbSum += frame_lb(blen, raw);
                    q += total - S.have;
                    S.have = 0;
                    rows++;
                    continue;
                }
            }
            if (S.phase == FP_SKIP) {
                const bool bc = S.flags & FR_BLOCK_SUM;
                const int64_t take = S.skip < L - q ? S.skip : L - q;
                if (bc && take > 0) { sk.srcOff = a.srcOff[i] + q; sk.len = (int32_t)take; sk.stream = s; }
                q += take;
                S.skip -= (int32_t)take;
                if (S.skip > 0) break;
                if (!bc) { r.err = ((unsigned long long)rows << 4) | FK_BLOCK; break; }
                while (S.have < 4 && q < L) S.hbuf[S.have++] = p[q++];
                if (S.have < 4) break;
                r.expect = fr_rd32(S.hbuf);
                check = 2;
                break;
            }
            if (S.phase == FP_TAIL) {
                while (S.have < 4 && q < L) S.hbuf[S.have++] = p[q++];
                if (S.have < 4) break;
                r.expect = fr_rd32(S.hbuf);
                check = 1; ended = 1;
                S.phase = FP_IDLE; S.have = 0;
                break;
            }
        }
    }
    r.nb = rows;
    r.flags = S.flags;
    r.maxBlock = S.maxBlock;
    if (pass == 0) {
        if (!Bytes) r.nslot = a.stageOff ? rows : 0;
        a.fr[i] = r;
        if (sk.stream >= 0) atomicOr(a.kinds, FRK_SKIP);
        if (rows > 0) {
            atomicMax(&a.tot->maxSteps, rows);
            atomicOr(a.kinds, ((S.flags & FR_INDEPENDENT) ? FRK_INDEP : FRK_LINKED) |
                                  ((S.flags & FR_BLOCK_SUM) ? FRK_BLOCK_SUM : 0) |
                                  ((S.flags & FR_CONTENT_SUM) ? FRK_CONTENT_SUM : 0));
        }
        return;
    }
    r.pos = e.start;
    a.fr[i] = r;
    if (Bytes) {
        u.fin = S;
        u.qFin = q;
        u.err = r.err;
        u.room = (int32_t)room;
        u.sk = sk;
        u.opened = opened; u.skipStart = skipStart; u.check = check; u.ended = ended;
        u.tailFrom = tailFrom; u.tailAt = tailAt;
        if (tailFrom >= 0) { u.tailLen = (int32_t)(q - tailFrom); u.tailFrom += a.srcOff[i]; }
        if (!u.gated) u.at = S;
        a.ent[i] = e;
        a.cut[i] = u;
        if (opened && !r.status) fr_xxh_reset(a.xs[s]);
        return;
    }
    e.used = r.status ? 0 : q;
    e.check = check;
    e.ended = ended;
    a.ent[i] = e;
    if (a.stageOff) a.stageOff[i] = e.start;
    const bool tail = !r.status && tailFrom >= 0;
    a.c.tailOff[i] = tail ? a.srcOff[i] + tailFrom : 0;
    a.c.tailDst[i] = tail ? (int64_t)s * a.stashStride + tailAt : 0;
    a.c.tailLen[i] = tail ? (int32_t)(q - tailFrom) : 0;
    a.skipEnt[i] = sk;
    if (e.stream < 0 || S.err) return;
    a.st[s] = S;
    if (opened) fr_xxh_reset(a.xs[s]);
    if (skipStart) fr_xxh_reset(a.bxs[s]);
}

// One thread per entry of a byte read, after the walk: the reference's loop over the candidates' sizes -- a row
// decodes while the rows before it left room (and, interactively, appended nothing), and none of them decoded to
// 0 bytes.  The plan's last step counts only when the loop reaches it (always, when the call met no length code).
// Writes the rows to decode (FrameRec.nb), srcUsed, the stream's state, the tail copy, the skipped bytes to hash,
// the drain copy, a pending slide, `stopped` (the loop stopped on room, interactive mode or an empty block) and
// zeroes the checksum lengths of the rows left over.  place (nullable, staged output): FrameRec.nslot = the bytes
// the entry appends (the rows' walked sizes; a row the decoder rejects appends less) in 16-byte units, nb = 0, for
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

// Staged byte read, after frame_scan_kernel over `place`: entry i's output starts at byte 16 * place[i].slot of
// the staging buffer; its cursor, its drain copy's destination and stageOff[i] move there.
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

// Step k, after the codec: a rejected block is the verdict -1 at row k; an accepted one is gathered to the cursor
// -- only what fits in the room left (dstCap here is the entry's); in a plain read the room rule leaves room for
// every accepted block -- hashed into the content checksum and goes to the commit.
__global__ void frame_reader_post_kernel(int k, FrameRec* __restrict__ fr, const FrEntry* __restrict__ ent,
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

// Step k, after the gather and the content checksum: the stream's undrained rest of the block and, in a linked
// frame, pos += the block and the slide -- unless more than 64 KiB stay undrained, whose slide the cut kernel
// makes once they are drained.  t.copyOff / ringOff / copyLen: the slide, for copy_blocks_kernel.
//
// A plain read commits here too, by chain_group_commit_kernel's decode rule: it leaves nothing undrained (left =
// 0), so a linked block slides when pos + res + SLOT > RING.  The one difference, a block of 0 bytes that slides
// where the chain kernel would leave pos alone, cannot arise: a plain read always starts with pos + SLOT <= RING,
// because every commit that leaves pos beyond RING - SLOT leaves undrained bytes, a stream holding them refuses
// plain reads (FR_ARG), and the cut kernel makes the deferred slide before anything else decodes.
__global__ void frame_reader_commit_kernel(const FrameRec* __restrict__ fr, int n, int64_t ring, int64_t slot,
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

// End (status non-null) or reset: the stream's undrained bytes go, and with them the FR_ARG mark; then its verdict
// -- 0 between frames, R_CORRUPT inside one, its sticky error when failed, K4LZ4_E_ARG for an index out of range
// -- and it becomes new.
__global__ void frame_reader_end_kernel(const int32_t* __restrict__ streams, int n, int nStreams,
                                        FrState* __restrict__ st, ChainGroupHdr* __restrict__ hdr,
                                        FrDrain* __restrict__ drain, int32_t* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = streams[i];
    if (s < 0 || s >= nStreams) {
        if (status) status[i] = FR_ARG;
        return;
    }
    FrState& S = st[s];
    const int32_t err = S.err == FR_ARG ? 0 : S.err;
    if (status) status[i] = err ? err : S.phase == FP_IDLE ? 0 : FR_CORRUPT;
    S.phase = FP_IDLE;
    S.have = 0;
    S.err = 0;
    hdr[s].pos = 0;
    drain[s].len = 0;
}

}  // namespace k4
