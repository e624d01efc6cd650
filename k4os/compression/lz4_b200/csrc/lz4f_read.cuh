// lz4f_read.cuh -- reading .lz4 streams as upstream's `lz4 -d` does (k4lz4_lz4f_decompress_batch,
// k4lz4_lz4f_decompressed_size_batch): the front end of the whole-frame decode for upstream's rules -- the member
// walk, the layout over a stream's members and the per-stream finish.  The blocks themselves go through
// block_size_walk_kernel and the block pass that the reference's frames use too (frame_decode_blocks in
// k4lz4_api.cu: the stored copies, block XXH32, OP_DECODE, the linked steps, frame_verdict_kernel), with one FrameRec
// per decodable member.
//
// The rules are upstream's: selectDecoder / LZ4IO_decompressLZ4F / LZ4IO_decodeLegacyStream (programs/lz4io.c) over
// LZ4F_decompress_usingDict (lib/lz4frame.c).  A stream is read member by member:
//   - an LZ4 frame (0x184D2204) by LZ4F's header and block rules: version 1, reserved bits clear, block-size ID 4..7,
//     header checksum; a block length code above the BD maximum is an error; blocks decode with capacity maxBlockSize;
//     a non-zero content-size field must equal the content at the end mark;
//   - a skippable frame (0x184D2A5?) is skipped; a size past the end ends the stream successfully;
//   - a legacy member (0x184C2102) is a run of blocks with a 4-byte length, each LZ4_decompress_safe with capacity
//     8 MiB; a length above LZ4_COMPRESSBOUND(8 MiB) ends the member and is the next member's magic;
//   - unknown magic is an error on the first member and ends the stream successfully on a later one.
// The first error in stream order wins: (member, block, kind), and within a block: length check, truncation,
// checksum, decode; at the end mark: frameSize_wrong, truncation, content checksum.
//
// Errors are (cliError << 8) | LZ4F_errorCodes, cliError being the lz4 CLI's EXM_THROW number.
#pragma once
#include "frame.cuh"

namespace k4 {

constexpr uint32_t LZ4F_LEGACY_MAGIC = 0x184C2102u;
constexpr uint32_t LZ4F_LEGACY_BOUND = 8421520u;      // LZ4_COMPRESSBOUND(LEGACY_BLOCKSIZE)
constexpr int32_t LZ4F_LEGACY_CAP = 8 << 20;          // LEGACY_BLOCKSIZE
constexpr int64_t LZ4F_SLOT_UNIT = 65536;             // scratch slots are whole units of this many bytes

// LZ4F_errorCodes (lz4frame.h) that the reader can raise, and the CLI's error numbers
constexpr int LE_GENERIC = 1, LE_MAX_BLOCK = 2, LE_VERSION = 6, LE_BLOCK_SUM = 7, LE_RESERVED = 8,
              LE_FRAME_SIZE = 14, LE_DECOMPRESS = 16, LE_HEADER_SUM = 17, LE_CONTENT_SUM = 18;
constexpr int CE_MAGIC = 40 << 8, CE_SKIP_SIZE = 42 << 8, CE_UNKNOWN = 44 << 8, CE_LEGACY_READ = 52 << 8,
              CE_LEGACY_DECODE = 53 << 8, CE_LZ4F = 66 << 8, CE_UNFINISHED = 68 << 8;

// member flags beside FR_*: the end mark was read; the member is a legacy run
constexpr int LF_END_READ = 32, LF_LEGACY = 64;

// The rules a member is read by, per member.
__host__ __device__ inline int32_t lz4f_member_cap(int flags, int32_t maxBlock) {
    return (flags & LF_LEGACY) ? LZ4F_LEGACY_CAP : maxBlock;
}
__host__ __device__ inline int64_t lz4f_slot_units(int32_t cap) {
    return (FR_HIST + cap + LZ4F_SLOT_UNIT - 1) / LZ4F_SLOT_UNIT;
}
// The code of a block that fails to decode.  The CLI's 64 KiB output buffer decides which one LZ4F reports: with a
// 64 KiB maximum the block decodes straight into it (ERROR_GENERIC), with a larger one through tmpOut
// (ERROR_decompressionFailed), lz4frame.c:1654-1713.
__host__ __device__ inline int lz4f_decode_error(int flags, int32_t maxBlock) {
    return (flags & LF_LEGACY) ? CE_LEGACY_DECODE : CE_LZ4F | (maxBlock <= 65536 ? LE_GENERIC : LE_DECOMPRESS);
}

// What the walk reports, member by member: begin(flags, maxBlock, contentSize, dictFlag), block(at, len, raw, sum),
// end(walkKey, walkCode, expect) -- walkKey FK_NONE or the (block << 4) | kind of the walk's error in this member,
// which then ends the stream -- and once stop(code, end): the stream-level verdict (0 or an error no member holds)
// and the offset where reading stopped.
template <class V>
__device__ void lz4f_walk(const uint8_t* __restrict__ f, const int64_t L, V& v) {
    int64_t q = 0, at = 0;
    bool first = true, pending = false;
    uint32_t magic = 0;
    while (true) {
        if (!pending) {
            if (q >= L) { v.stop(0, L); return; }
            if (L - q < 4) { v.stop(CE_MAGIC, L); return; }
            at = q; magic = fr_rd32(f + q); q += 4;
        }
        pending = false;
        if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {
            if (L - q < 4) { v.stop(CE_SKIP_SIZE, L); return; }
            const uint32_t size = fr_rd32(f + q);
            q += 4;
            q = L - q < (int64_t)size ? L : q + size;      // fseek past the end succeeds; the next read is EOF
        } else if (magic == FRAME_MAGIC) {
            const int64_t avail = L - at;
            if (avail < 7) { v.stop(CE_UNFINISHED, L); return; }
            const int flg = f[at + 4], bd = f[at + 5];
            if ((flg >> 1) & 1) { v.stop(CE_LZ4F | LE_RESERVED, L); return; }
            if (((flg >> 6) & 3) != 1) { v.stop(CE_LZ4F | LE_VERSION, L); return; }
            const int64_t fhs = 7 + ((flg & 8) ? 8 : 0) + ((flg & 1) ? 4 : 0);
            if (avail < fhs) { v.stop(CE_UNFINISHED, L); return; }
            if (bd & 0x80) { v.stop(CE_LZ4F | LE_RESERVED, L); return; }
            if (((bd >> 4) & 7) < 4) { v.stop(CE_LZ4F | LE_MAX_BLOCK, L); return; }
            if (bd & 0x0F) { v.stop(CE_LZ4F | LE_RESERVED, L); return; }
            if (((xx_finish(XXP5 + (uint32_t)(fhs - 5), f + at + 4, (size_t)(fhs - 5)) >> 8) & 0xFF) != f[at + fhs - 1]) {
                v.stop(CE_LZ4F | LE_HEADER_SUM, L);
                return;
            }
            const int32_t maxBlock = 1 << (8 + 2 * ((bd >> 4) & 7));
            const uint64_t cs = (flg & 8) ? ((uint64_t)fr_rd32(f + at + 6) | ((uint64_t)fr_rd32(f + at + 10) << 32)) : 0;
            int flags = frame_flags_of(flg);
            const bool bc = flags & FR_BLOCK_SUM;
            v.begin(flags, maxBlock, cs, flg & 1);
            q = at + fhs;
            int k = 0;
            unsigned long long key = FK_NONE;
            int code = 0;
            while (true) {
                if (L - q < 4) { key = ((unsigned long long)k << 4) | FK_TRUNC; code = CE_UNFINISHED; break; }
                const uint32_t c = fr_rd32(f + q);
                q += 4;
                if (c == 0) { flags |= LF_END_READ; break; }
                const int64_t blen = c & 0x7FFFFFFFu;
                if (blen > maxBlock) { key = ((unsigned long long)k << 4) | FK_TRUNC; code = CE_LZ4F | LE_MAX_BLOCK; break; }
                if (L - q < blen + (bc ? 4 : 0)) { key = ((unsigned long long)k << 4) | FK_TRUNC; code = CE_UNFINISHED; break; }
                v.block(q, (int32_t)blen, c >> 31, bc ? fr_rd32(f + q + blen) : 0u);
                q += blen + (bc ? 4 : 0);
                k++;
            }
            uint32_t expect = 0;
            if (!code && (flags & FR_CONTENT_SUM)) {
                if (L - q < 4) { key = ((unsigned long long)k << 4) | FK_TRUNC; code = CE_UNFINISHED; }
                else { expect = fr_rd32(f + q); q += 4; }
            }
            v.end(flags, key, code, expect);
            if (code) { v.stop(0, L); return; }
        } else if (magic == LZ4F_LEGACY_MAGIC) {
            v.begin(FR_INDEPENDENT | LF_LEGACY, LZ4F_LEGACY_CAP, 0, 0);
            int k = 0;
            unsigned long long key = FK_NONE;
            int code = 0;
            while (q < L) {
                if (L - q < 4) { key = ((unsigned long long)k << 4) | FK_TRUNC; code = CE_LEGACY_READ; break; }
                const uint32_t len = fr_rd32(f + q);
                if (len > LZ4F_LEGACY_BOUND) { at = q; magic = len; q += 4; pending = true; break; }
                q += 4;
                if (L - q < (int64_t)len) { key = ((unsigned long long)k << 4) | FK_TRUNC; code = CE_LEGACY_READ; break; }
                if (len == 0) { key = ((unsigned long long)k << 4) | FK_BLOCK; code = CE_LEGACY_DECODE; break; }
                v.block(q, (int32_t)len, 0, 0u);
                q += len;
                k++;
            }
            v.end(FR_INDEPENDENT | LF_LEGACY, key, code, 0u);
            if (code) { v.stop(0, L); return; }
        } else {
            v.stop(first ? CE_UNKNOWN : 0, first ? L : at);
            return;
        }
        first = false;
    }
}

// The per-stream and per-member arrays of one call.
struct Lz4fStreams {
    FrameRec* rows;          // per stream: nb = its blocks, nslot = its scratch units (first / slot after the scan)
    FrameRec* mems;          // per stream: nb = its members (first after the scan)
    int32_t* code;           // per stream: the walk's stream-level verdict
    int32_t* end;            // per stream: where reading stopped
    int64_t* total;          // per stream: the content (layout)
    uint64_t* lb;            // per stream: the lower bound of the content (pass 0)
};
struct Lz4fMembers {
    int32_t* stream;         // the member's stream
    int32_t* code;           // the code of the walk's error in this member, with its key in `key`
    unsigned long long* key;
    uint64_t* size;          // the content-size field (0: none)
    int64_t* dst;            // where the member's content starts, relative to dstBase
    int64_t* dictOff; int32_t* dictLen;   // the member's dictionary (dictionary calls; none for legacy members)
};

// Pass 0 visitor: counts, the lower bound of the content, the verdict and the end.
struct Lz4fCount {
    int64_t blocks = 0, lb = 0; int members = 0, maxLinked = 0, nb = 0, flags = 0;
    int code = 0, stopAt = 0;
    __device__ void begin(int fl, int32_t, uint64_t, int) { nb = 0; flags = fl; }
    __device__ void block(int64_t, int32_t len, uint32_t raw, uint32_t) { blocks++; nb++; lb += frame_lb(len, raw); }
    __device__ void end(int, unsigned long long, int, uint32_t) {
        members++;
        if (!(flags & FR_INDEPENDENT) && nb > maxLinked) maxLinked = nb;
    }
    __device__ void stop(int c, int64_t e) { code = c; stopAt = (int)e; }
};

// Pass 0b / 1 visitor: which blocks may need a scratch slot (the content behind them, by its lower bound, is less
// than their capacity: only they can reach past dstCap), and with `write`, the member records and the rows.
struct Lz4fPlace {
    bool write, dict;
    int64_t lbTotal, acc = 0, units = 0, row = 0, slot = 0;
    int s = 0, m = 0;
    FrameRec r;
    int64_t base;            // srcOff of the stream
    FrameRec* fr; FrameTable t; Lz4fMembers mb;
    const int64_t* dictOff; const int32_t* dictLen;
    __device__ void begin(int fl, int32_t maxBlock, uint64_t cs, int) {
        r = FrameRec{};
        r.first = row; r.slot = slot; r.flags = fl; r.maxBlock = maxBlock; r.err = FK_NONE;
        r.k0 = -1;
        if (write) mb.size[m] = cs;
    }
    __device__ void block(int64_t at, int32_t len, uint32_t raw, uint32_t sum) {
        const int k = r.nb++;
        acc += frame_lb(len, raw);
        if (r.k0 < 0 && lbTotal - acc < lz4f_member_cap(r.flags, r.maxBlock)) r.k0 = k;
        if (write) {
            const int64_t b = row;
            t.srcOff[b] = base + at; t.len[b] = len;
            t.kind[b] = (raw ? RK_RAW : 0) | ((r.flags & FR_INDEPENDENT) ? 0 : RK_LINKED);
            t.frame[b] = m; t.idx[b] = k; t.sum[b] = sum;
        }
        row++;
    }
    __device__ void end(int fl, unsigned long long key, int code, uint32_t expect) {
        r.flags = fl;
        if (r.k0 < 0) r.k0 = r.nb;
        const bool linked = !(r.flags & FR_INDEPENDENT);
        const int64_t u = lz4f_slot_units(lz4f_member_cap(r.flags, r.maxBlock));
        const int64_t n = r.nb == 0 ? 0 : linked ? ((r.k0 < r.nb || dict) ? 1 : 0) : r.nb - r.k0;
        r.nslot = (int32_t)(n * u);
        slot += n * u; units += n * u;
        if (write) {
            r.err = key; r.expect = expect;
            fr[m] = r;
            mb.stream[m] = s; mb.code[m] = code; mb.key[m] = key;
            if (mb.dictLen) {
                const bool on = dictLen && !(r.flags & LF_LEGACY);
                mb.dictOff[m] = on ? dictOff[s] : 0;
                mb.dictLen[m] = on && dictLen[s] > 0 ? dictLen[s] : 0;
            }
        }
        m++;
    }
    __device__ void stop(int, int64_t) {}
};

// One thread per stream.  Pass 0: the stream's blocks, scratch units and members (into ss.rows / ss.mems for
// frame_scan_kernel), its verdict and end, and the largest block count of a linked member.  Pass 1, after the scans:
// the member records (first row, first scratch unit, blocks, k0, flags, BD maximum, walk key, stored checksum) and
// the rows.  dict: a linked member with blocks always gets its slot (frame_dict_layout_kernel puts the dictionary's
// tail in front of its early blocks there).
__global__ void lz4f_walk_kernel(int pass, const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                                 const int32_t* __restrict__ srcLen, int n, Lz4fStreams ss, FrameRec* __restrict__ fr,
                                 Lz4fMembers mb, FrameTable t, const int64_t* __restrict__ dictOff,
                                 const int32_t* __restrict__ dictLen, int dict, FrameTotals* __restrict__ tot) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int64_t L = srcLen[s] > 0 ? srcLen[s] : 0;
    const uint8_t* f = srcBase + srcOff[s];
    if (pass == 0) {
        Lz4fCount c;
        lz4f_walk(f, L, c);
        Lz4fPlace p{false, dict != 0, c.lb};
        lz4f_walk(f, L, p);
        FrameRec a{}, b{};
        a.nb = (int32_t)c.blocks; a.nslot = (int32_t)p.units;
        b.nb = c.members;
        ss.rows[s] = a; ss.mems[s] = b;
        ss.code[s] = c.code; ss.end[s] = c.stopAt; ss.lb[s] = (uint64_t)c.lb;
        if (tot && c.maxLinked) atomicMax(&tot->maxSteps, c.maxLinked);
        return;
    }
    Lz4fPlace p{true, dict != 0, (int64_t)ss.lb[s]};
    p.row = ss.rows[s].first; p.slot = ss.rows[s].slot; p.m = (int)ss.mems[s].first; p.s = s;
    p.base = srcOff[s]; p.fr = fr; p.t = t; p.mb = mb; p.dictOff = dictOff; p.dictLen = dictLen;
    lz4f_walk(f, L, p);
}

// One thread per stream, after block_size_walk_kernel: each member's place in the stream's destination (behind the
// members before it), then its blocks' placement (frame_place_row) with the member's capacity (maxBlockSize, or
// 8 MiB for legacy runs) and its own scratch units.  A block whose walk gives more than that capacity fails as the
// decoder would.  A stream whose content exceeds dstCap is skipped: nothing of it is written.  dstCap null: sizes.
__global__ void lz4f_layout_kernel(int n, Lz4fStreams ss, FrameRec* __restrict__ fr, Lz4fMembers mb, FrameTable t,
                                   const int64_t* __restrict__ dstOff, const int32_t* __restrict__ dstCap,
                                   int64_t scratchRel, int32_t* __restrict__ ccLen) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int64_t m0 = ss.mems[s].first, m1 = m0 + ss.mems[s].nb;
    const int64_t b0 = ss.rows[s].first, b1 = b0 + ss.rows[s].nb;
    int64_t total = 0;
    for (int64_t b = b0; b < b1; b++) total += t.size[b];
    ss.total[s] = total;
    const int64_t room = dstCap ? (dstCap[s] > 0 ? dstCap[s] : 0) : INT64_MAX;
    const bool skip = total > room;
    const int64_t base = dstOff ? dstOff[s] : 0;
    int64_t pos = 0;
    for (int64_t m = m0; m < m1; m++) {
        FrameRec r = fr[m];
        const bool linked = !(r.flags & FR_INDEPENDENT), bc = r.flags & FR_BLOCK_SUM;
        const int32_t cap = lz4f_member_cap(r.flags, r.maxBlock);
        const int64_t unit = lz4f_slot_units(cap) * LZ4F_SLOT_UNIT;
        mb.dst[m] = base + pos;
        const int64_t start = pos;
        for (int k = 0; k < r.nb; k++) {
            const int64_t b = r.first + k;
            const int32_t L = t.len[b], sz = t.size[b];
            const bool raw = t.kind[b] & RK_RAW;
            const unsigned long long blockKey = ((unsigned long long)k << 4) | FK_BLOCK;
            if (!raw && sz > cap && blockKey < r.err) r.err = blockKey;
            const bool scratch = dstCap && !skip && !raw && pos + cap > room;
            int64_t at = base + pos;
            if (scratch) at = scratchRel + r.slot * LZ4F_SLOT_UNIT + (linked ? 0 : k - r.k0) * unit + FR_HIST;
            // the block checksum also when skipped: it needs no decoding, and lz4f_finish_kernel reports its mismatch
            frame_place_row(t, b, L, raw, linked, skip, scratch, base + pos, at, cap, (!skip && raw) ? L : 0,
                            bc ? L : 0);
            pos += sz;
        }
        fr[m].pos = pos - start;
        fr[m].err = r.err;
        if (ccLen) ccLen[m] = (!skip && (r.flags & FR_CONTENT_SUM) && mb.key[m] == FK_NONE) ? (int32_t)(pos - start) : 0;
    }
}

// One thread per stream: the first error in stream order, member by member (a block's error from the walk or the
// decode, then at the end mark frameSize_wrong, truncation, the content checksum), else the walk's stream-level
// verdict.  A stream that does not fit dstCap gets the verdicts that need no decoding (the block checksums, which
// come before a block's decode, among them), else K4LZ4_R_DST_SMALL.
// ccGot null: the size call.  The content-size field is checked only where the blocks were decoded: a block that
// fails to decode may walk to any size.
__global__ void lz4f_finish_kernel(int n, Lz4fStreams ss, const FrameRec* __restrict__ fr, Lz4fMembers mb,
                                   FrameTable t, const int32_t* __restrict__ dstCap, const uint32_t* __restrict__ ccGot,
                                   const int32_t* __restrict__ ccLen, int32_t* __restrict__ outLen,
                                   int32_t* __restrict__ outErr, int32_t* __restrict__ outEnd) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int64_t m0 = ss.mems[s].first, m1 = m0 + ss.mems[s].nb;
    const int64_t total = ss.total[s];
    const bool small = dstCap && total > (dstCap[s] > 0 ? dstCap[s] : 0);
    const bool sums = ccGot && !small;
    int code = 0;
    for (int64_t m = m0; m < m1 && !code; m++) {
        const FrameRec& r = fr[m];
        // the walk's own error sits at block nb (the block it could not take), so below that key only the blocks'
        // checksums and decodes can fail
        unsigned long long err = r.err;
        const unsigned long long endKey = (unsigned long long)r.nb << 4;
        if (small && ccGot)                            // skipped: frame_verdict_kernel did not compare the checksums
            for (int k = 0; k < r.nb && ((unsigned long long)k << 4) < err; k++) {
                const int64_t b = r.first + k;
                if (t.ckLen[b] > 0 && t.got[b] != t.sum[b]) { err = ((unsigned long long)k << 4) | FK_SUM; break; }
            }
        if (err < endKey) {
            code = (err & 15) == FK_SUM ? CE_LZ4F | LE_BLOCK_SUM : lz4f_decode_error(r.flags, r.maxBlock);
        } else if (sums && (r.flags & LF_END_READ) && mb.size[m] && mb.size[m] != (uint64_t)r.pos) {
            code = CE_LZ4F | LE_FRAME_SIZE;
        } else if (err != FK_NONE) {
            code = mb.code[m];
        } else if (sums && (r.flags & FR_CONTENT_SUM) && ccLen[m] == r.pos && ccGot[m] != r.expect) {
            code = CE_LZ4F | LE_CONTENT_SUM;
        }
    }
    if (!code) code = ss.code[s];
    int32_t out;
    if (code) out = -1;
    else if (small) out = FR_DST_SMALL;
    else out = total > 0x7FFFFFFF ? FR_CORRUPT : (int32_t)total;
    outLen[s] = out;
    outErr[s] = code;
    outEnd[s] = ss.end[s];
}

}  // namespace k4
