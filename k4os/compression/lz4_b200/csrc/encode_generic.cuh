// encode_generic.cuh -- bit-exact LZ4 L00_FAST block encoder, one warp per block.
//
// Reproduces the token stream of LZ4_compress_fast as reached from LZ4Codec.Encode
// (acceleration 1, fresh zeroed table, noDict):
//   /root/reference/src/K4os.Compression.LZ4/Engine/x64/LL64.fast.cs:35-513 (generic loop),
//   :517-568 (table/limit selection), Engine/LL.tools.cs:46-58 (hash4/hash5),
//   Engine/x64/LL64.tools.cs:87-133 (LZ4_count).  Step numbers in comments = SURVEY.md App. A.
//
// Bit-exactness forces the reference's serial table history, so the match *search*
// (hash -> slot load -> slot store -> 4-byte compare, App. A step 3/8) is a serial chain
// executed by lane 0 against a 16 KiB shared-memory table; everything that is not on that
// chain -- common-prefix counting, literal copies, LSIC fills, table zeroing -- is done by
// all 32 lanes.  Output bytes are written once, exactly; nothing beyond the returned length
// is touched.
#pragma once
#include "common.cuh"

namespace k4 {

constexpr int ENC_TABLE_BYTES = 16384;   // LZ4_stream_t hash table, LL.types.cs:18-39
constexpr int ENC_FLAG_X32 = 0x100;      // `level` bit: reproduce the 32-bit engine (LL32) for inputs >= 65 547 bytes
// the global-table encoder warps (encode_tile.cuh, GTAB) keep 32-bit slots: position | 16-bit tag
constexpr int ENC_GSLOT_BYTES = 2 * ENC_TABLE_BYTES;

struct EncCtx {
    const uint8_t* src;
    uint32_t n;
    bool by16;
    bool use5;
    uint16_t* t16;
    uint32_t* t32;
    __device__ __forceinline__ uint32_t hash_at(uint32_t p) const {
        if (by16) return hash4(ldg_u32u(src + p), 13);
        return use5 ? hash5(ldg_u64u(src + p), 12) : hash4(ldg_u32u(src + p), 12);
    }
    __device__ __forceinline__ uint32_t tget(uint32_t h) const { return by16 ? (uint32_t)t16[h] : t32[h]; }
    __device__ __forceinline__ void tput(uint32_t h, uint32_t v) const {
        if (by16) t16[h] = (uint16_t)v; else t32[h] = v;
    }
};

// lane 0 writes token + LSIC bytes of a literal run; returns new op (uniform via caller)
__device__ __forceinline__ uint32_t run_header_size(uint32_t run) {
    return run >= 15 ? 2 + (run - 15) / 255 : 1;
}
__device__ __forceinline__ void write_run_header(uint8_t* dst, uint32_t op, uint32_t run) {
    if (run >= 15) {
        uint32_t rest = run - 15;
        dst[op++] = 0xF0;
        for (; rest >= 255; rest -= 255) dst[op++] = 255;
        dst[op++] = (uint8_t)rest;
    } else {
        dst[op] = (uint8_t)(run << 4);
    }
}

/*
 * Returns the engine's value: bytes written (> 0) or 0 when the reference's limitedOutput
 * checks fail.  `cap` is the capacity the reference would have been given (drives the
 * notLimited/limitedOutput choice and every olimit test).  `hardCap` is a physical write
 * bound used only by the pickler (see pickle.cuh): as soon as the stream would grow past it
 * the function returns 0; pass 0x7fffffff otherwise.
 * FILL: upstream's fillOutput directive, as in encode_spec_warp (encode_tile.cuh): with cap below the bound the
 * longest prefix whose block fits cap is encoded, and lane 0 stores the input bytes it took at *used.
 */
template <bool FILL = false>
__device__ int encode_block_warp(const uint8_t* __restrict__ src, int n_, uint8_t* __restrict__ dst,
                                 int cap, int hardCap, void* tableSmem, bool enforce32, int32_t* used = nullptr) {
    const int lane = lane_id();
    if ((uint32_t)n_ > (uint32_t)MAX_INPUT_SIZE) return 0;                     // LL64.fast.cs:90
    EncCtx c;
    c.src = src; c.n = (uint32_t)n_;
    c.by16 = n_ < LIMIT_64K;                                              // :526,548
    c.use5 = !c.by16 && !enforce32;                                       // LL64.tools.cs:135-143
    c.t16 = reinterpret_cast<uint16_t*>(tableSmem);
    c.t32 = reinterpret_cast<uint32_t*>(tableSmem);
    const bool limited = !FILL && !(cap >= max_output_size(n_));          // :524
    const bool fill = FILL && !(cap >= max_output_size(n_));              // lz4.c:1387
    const int64_t olimit = cap;
    const int64_t hard = hardCap;
    const uint32_t n = c.n;

    // LZ4_initStream: zero the table (LL.tools.cs:235-239)
    {
        uint4* t = reinterpret_cast<uint4*>(tableSmem);
        for (int i = lane; i < ENC_TABLE_BYTES / 16; i += 32) t[i] = make_uint4(0, 0, 0, 0);
        __syncwarp();
    }

    uint32_t ip = 0, anchor = 0, op = 0;

    if (n >= (uint32_t)MINLENGTH) {                                       // :117
        const uint32_t mfl1 = n - MFLIMIT + 1;                            // :70
        const uint32_t mlim = n - LASTLITERALS;                           // :71
        uint32_t fh = 0, m = 0, tokpos = 0;
        if (lane == 0) {
            c.tput(c.hash_at(0), 0);                                      // :120
            fh = c.hash_at(1);                                            // :122
        }
        ip = 1;
        for (;;) {
            // ---- step 3 (search) + step 4 (catch-up): the serial chain, lane 0 ----------
            uint32_t status = 0;   // 1 = match found at (ip, m); 0 = ran into the end
            if (lane == 0) {
                uint32_t fwd = ip, step = 1, cnt = 1u << SKIP_TRIGGER;
                for (;;) {
                    const uint32_t hh = fh, cur = fwd;
                    m = c.tget(hh);
                    ip = fwd;
                    fwd += step;
                    step = cnt++ >> SKIP_TRIGGER;
                    if (fwd > mfl1) { status = 0; break; }                // :172
                    fh = c.hash_at(fwd);                                  // :212
                    c.tput(hh, cur);                                      // :213
                    if (!c.by16 && m + MAX_DISTANCE < cur) continue;      // :219-224
                    if (ldg_u32u(src + m) == ldg_u32u(src + ip)) { status = 1; break; }   // :228
                }
                if (status) {                                             // :237-242
                    while (ip > anchor && m > 0 && __ldg(src + ip - 1) == __ldg(src + m - 1)) { ip--; m--; }
                }
            }
            status = __shfl_sync(FULL, status, 0);
            if (!status) break;                                           // -> last literals
            ip = __shfl_sync(FULL, ip, 0);
            m = __shfl_sync(FULL, m, 0);

            // ---- step 5: literal run ----------------------------------------------------
            {
                const uint32_t lit = ip - anchor;
                if (limited && (int64_t)op + 1 + lit + 8 + lit / 255 > olimit) return 0;   // :246-251
                const uint32_t hdr = run_header_size(lit);
                // fill rule 1 (lz4.c:1028-1032): the sequence would pass the target; drop it unwritten
                if (fill && (int64_t)op + hdr + lit + 2 + 1 + (MFLIMIT - MINMATCH) > olimit) goto last_literals;
                if ((int64_t)op + hdr + lit > hard) return 0;
                tokpos = op;
                if (lane == 0) write_run_header(dst, op, lit);
                op += hdr;
                for (uint32_t i = lane; i < lit; i += 32) dst[op + i] = __ldg(src + anchor + i);
                op += lit;
            }

            for (;;) {   // _next_match
                // ---- step 6: offset + match length -------------------------------------
                if ((int64_t)op + 2 > hard) return 0;
                if (lane == 0) { dst[op] = (uint8_t)(ip - m); dst[op + 1] = (uint8_t)((ip - m) >> 8); }
                op += 2;
                uint32_t mc = 0;
                {   // LZ4_count(ip+4, m+4, matchlimit): lane-parallel common prefix, :328
                    uint32_t a = ip + MINMATCH, b = m + MINMATCH;
                    for (;;) {
                        const bool in = a + lane < mlim;
                        const bool eq = in && (__ldg(src + a + lane) == __ldg(src + b + lane));
                        const unsigned miss = __ballot_sync(FULL, !eq);
                        if (miss) { mc += __ffs(miss) - 1; break; }
                        mc += 32; a += 32; b += 32;
                    }
                }
                ip += mc + MINMATCH;
                if (limited && (int64_t)op + 6 + (mc + 240) / 255 > olimit) return 0;   // :332-362
                // fill rule 3 (lz4.c:1097-1104): shorten the match to what fits; no later sequence can pass rules
                // 1 and 2 from here, so the block goes to last literals (encode_spec_warp says why)
                bool cut = false;
                if (fill && (int64_t)op + 6 + (mc + 240) / 255 > olimit) {
                    const uint32_t mc2 = 14u + (uint32_t)(olimit - op - 6) * 255u;
                    ip -= mc - mc2;
                    mc = mc2;
                    cut = true;
                }
                if (mc >= 15) {                                           // :365-379
                    const uint32_t rest = mc - 15;
                    const uint32_t nff = rest / 255;
                    if ((int64_t)op + nff + 1 > hard) return 0;
                    for (uint32_t i = lane; i < nff; i += 32) dst[op + i] = 0xFF;
                    if (lane == 0) {
                        dst[tokpos] = (uint8_t)(dst[tokpos] + 15);
                        dst[op + nff] = (uint8_t)(rest % 255);
                    }
                    op += nff + 1;
                } else if (lane == 0) {
                    dst[tokpos] = (uint8_t)(dst[tokpos] + mc);
                }
                __syncwarp();
                anchor = ip;                                              // :388
                if (ip >= mfl1 || cut) goto last_literals;                // :391

                // ---- step 8: post-match insert + immediate probe, lane 0 ---------------
                uint32_t hit = 0;
                if (lane == 0) {
                    c.tput(c.hash_at(ip - 2), ip - 2);                    // :394
                    const uint32_t hh = c.hash_at(ip);
                    m = c.tget(hh);
                    c.tput(hh, ip);
                    if ((c.by16 || m + MAX_DISTANCE >= ip) && ldg_u32u(src + m) == ldg_u32u(src + ip))
                        hit = 1;                                          // :452-463
                    else
                        fh = c.hash_at(ip + 1);                           // :466
                }
                hit = __shfl_sync(FULL, hit, 0);
                if (!hit) { ip++; break; }
                m = __shfl_sync(FULL, m, 0);
                // fill rule 2 (lz4.c:1057-1062): the zero-literal sequence would pass the target; drop it unwritten
                if (fill && (int64_t)op + 1 + 2 + 1 + (MFLIMIT - MINMATCH) > olimit) goto last_literals;
                if ((int64_t)op + 1 > hard) return 0;
                tokpos = op;
                if (lane == 0) dst[op] = 0;                               // :459-460
                op++;
                __syncwarp();
            }
        }
    }

last_literals:
    {   // ---- step 9, :469-503 ----------------------------------------------------------
        uint32_t run = n - anchor;
        if (limited && (int64_t)op + run + 1 + (run + 255 - 15) / 255 > olimit) return 0;
        if (fill && (int64_t)op + run + 1 + (run + 255 - 15) / 255 > olimit) {     // fill rule 4, lz4.c:1209-1213
            run = (uint32_t)(olimit - op) - 1;
            run -= (run + 256 - 15) / 256;
        }
        const uint32_t hdr = run_header_size(run);
        if ((int64_t)op + hdr + run > hard) return 0;
        if (lane == 0) write_run_header(dst, op, run);
        op += hdr;
        for (uint32_t i = lane; i < run; i += 32) dst[op + i] = __ldg(src + anchor + i);
        op += run;
        if (FILL && lane == 0) *used = (int32_t)(anchor + run);
    }
    return (int)op;
}

constexpr int ENC_WARPS_PER_CTA = 7;   // pickle_kernel: 2 CTAs x 7 warps x 16 KiB of tables fill the SM
// encode_spec_kernel / encode_spec_gtab_kernel (one warp per CTA, see encode_tile.cuh): resident warps per SM
#ifndef K4_ENC_SM_WARPS
#define K4_ENC_SM_WARPS 10      // shared-memory tables: 10 x (16 KiB + 1 KiB the hardware reserves per CTA); the rest of the 256 KiB stays L1
#endif
#ifndef K4_ENC_GM_WARPS
#define K4_ENC_GM_WARPS 20      // global-memory tables (H100 sweep in DESIGN.md 7.2)
#endif
constexpr int ENC_SM_WARPS = K4_ENC_SM_WARPS;
constexpr int ENC_GM_WARPS = K4_ENC_GM_WARPS;

}  // namespace k4
