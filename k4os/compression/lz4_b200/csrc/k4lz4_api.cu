// k4lz4_api.cu -- the C ABI of libk4lz4 (include/k4lz4.h): argument handling, the
// device-resident launch path, the host-buffer staging paths (chunked, double-buffered,
// NCCL-free multi-GPU split of the block list for the codec; one synchronous routine for the
// rest) and the synthetic workload generator.
//
// There is deliberately NO CPU codec in this library: without a usable CUDA device every
// compute call with valid arguments fails with K4LZ4_E_NODEVICE.
#include "../../../../include/k4lz4.h"

#include <cuda_runtime.h>
#if defined(__linux__)
#include <sched.h>
#endif

#include <algorithm>
#include <cctype>
#include <cstdlib>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"
#include "decode_generic.cuh"
#include "decode_tile.cuh"
#include "encode_generic.cuh"
#include "encode_tile.cuh"
#include "encode_chain.cuh"
#include "chain_group.cuh"
#include "pickle.cuh"
#include "synth.cuh"
#include "copy_blocks.cuh"
#include "xxh32.cuh"
#include "frame.cuh"
#include "frame_writer.cuh"
#include "frame_reader.cuh"

namespace {

std::atomic<int64_t> g_launches{0};
thread_local std::string t_err;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    t_err = buf;
    return code;
}

#define CU_TRY(expr)                                                                         \
    do {                                                                                     \
        cudaError_t e__ = (expr);                                                            \
        if (e__ != cudaSuccess)                                                              \
            return fail(K4LZ4_E_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__));      \
    } while (0)

int device_count_cached() {
    static int n = [] {
        int c = 0;
        cudaError_t e = cudaGetDeviceCount(&c);
        if (e != cudaSuccess) { (void)cudaGetLastError(); return 0; }
        return c;
    }();
    return n;
}

// ---- one batch description, one argument check ------------------------------------------------

enum Op {
    OP_ENCODE, OP_DECODE, OP_CHAIN, OP_GENERAL, OP_PICKLE, OP_PICKLEW, OP_UNPICKLE, OP_USIZE, OP_XXH32, OP_COPY,
    OP_ENCCHAIN, OP_DSIZE
};

// Block i reads srcBase[srcOff[i] .. +srcLen[i]) and writes dstBase[dstOff[i] .. +dstCap[i]) and outLen[i].
// The optional parts are null / 0 unless the op reads them.
struct Batch {
    const uint8_t* srcBase; const int64_t* srcOff; const int32_t* srcLen;
    uint8_t* dstBase; const int64_t* dstOff; const int32_t* dstCap;
    int32_t* outLen;                  // OP_XXH32: the uint32 checksums
    int64_t n;
    int level = 0;                    // OP_ENCODE: 0..255; OP_PICKLE(W): passed through
    bool x32 = false;                 // OP_ENCODE, OP_ENCCHAIN, OP_PICKLE(W): the 32-bit engine (k4lz4_*_x32)
    const uint8_t* dictBase = nullptr; const int64_t* dictOff = nullptr; const int32_t* dictLen = nullptr;
    const int32_t* prefixLen = nullptr;   // OP_CHAIN: history in front of each destination; OP_ENCCHAIN: of each source
    uint8_t* stateBase = nullptr; const int64_t* stateOff = nullptr;   // OP_ENCCHAIN: K4LZ4_CHAIN_STATE_BYTES per block
    bool partial = false;             // OP_GENERAL: PartialDecode semantics (dstCap = target length)
    uint32_t seed = 0;                // OP_XXH32
};

// The pointers each op needs when n > 0, besides srcBase / srcOff / srcLen.  A dictionary is optional
// wherever it is read: with dictBase set, dictOff and dictLen are required too.
struct Needs { bool dst, cap, out, prefix, level, state; };
constexpr Needs NEEDS[] = {
    /* OP_ENCODE   */ {true,  true,  true,  false, true,  false},
    /* OP_DECODE   */ {true,  true,  true,  false, false, false},
    /* OP_CHAIN    */ {true,  true,  true,  true,  false, false},
    /* OP_GENERAL  */ {true,  true,  true,  false, false, false},
    /* OP_PICKLE   */ {true,  false, true,  false, false, false},
    /* OP_PICKLEW  */ {true,  false, true,  false, false, false},
    /* OP_UNPICKLE */ {true,  true,  true,  false, false, false},
    /* OP_USIZE    */ {false, false, true,  false, false, false},
    /* OP_XXH32    */ {false, false, true,  false, false, false},
    /* OP_COPY     */ {true,  false, false, false, false, false},
    /* OP_ENCCHAIN */ {true,  true,  true,  true,  true,  true},
    /* OP_DSIZE    */ {false, false, true,  false, false, false},
};
static_assert(sizeof(NEEDS) / sizeof(NEEDS[0]) == OP_DSIZE + 1, "one row per op");

// The machine part of check(): a device must exist, an empty batch is then done (the caller returns OK for
// n == 0), and `device` (K4LZ4_ALL_DEVICES or the current device when negative) must name a visible GPU.
int check_device(int device, int64_t n) {
    const int ndev = device_count_cached();
    if (ndev <= 0) return fail(K4LZ4_E_NODEVICE, "no CUDA device available");
    if (n == 0) return K4LZ4_OK;
    if (device >= ndev) return fail(K4LZ4_E_ARG, "device %d out of range (%d visible)", device, ndev);
    return K4LZ4_OK;
}

// Every batched export: the arguments first, then the machine, so that a caller's mistake gets the same
// code with or without a GPU.
int check(Op op, const Batch& b, int memKind, int device) {
    const Needs& w = NEEDS[op];
    if (memKind != K4LZ4_MEM_HOST && memKind != K4LZ4_MEM_DEVICE) return fail(K4LZ4_E_ARG, "unknown memKind %d", memKind);
    if (b.n < 0 || b.n > INT32_MAX) return fail(K4LZ4_E_ARG, "bad block count %lld", (long long)b.n);
    if (b.n > 0 && (!b.srcBase || !b.srcOff || !b.srcLen || (w.out && !b.outLen) || (w.dst && (!b.dstBase || !b.dstOff)) ||
                    (w.cap && !b.dstCap) || (w.prefix && !b.prefixLen) || (b.dictBase && (!b.dictOff || !b.dictLen)) ||
                    (w.state && (!b.stateBase || !b.stateOff))))
        return fail(K4LZ4_E_ARG, "null pointer argument");
    if (w.prefix && memKind == K4LZ4_MEM_HOST)       // device arrays cannot be checked here: there a negative prefix gives -1
        for (int64_t i = 0; i < b.n; i++)
            if (b.prefixLen[i] < 0) return fail(K4LZ4_E_ARG, "negative prefix length at block %lld", (long long)i);
    if (w.state && memKind == K4LZ4_MEM_HOST)        // likewise: on the device a misaligned state record gives -1
        for (int64_t i = 0; i < b.n; i++)
            if (b.stateOff[i] & 15) return fail(K4LZ4_E_ARG, "state offset not a multiple of 16 at block %lld", (long long)i);
    if (w.level && (b.level < 0 || b.level > 0xFF)) return fail(K4LZ4_E_ARG, "bad level %d", b.level);
    return check_device(device, b.n);
}

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (dev >= 0) {
            cudaGetDevice(&prev);
            if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess; else prev = -1;
        }
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// ---- per-device state ---------------------------------------------------------------------------

struct Buf {           // grows, never shrinks: device memory, or pinned host memory
    bool pinned = false;
    void* p = nullptr; size_t cap = 0;
    cudaError_t alloc(size_t n) { return pinned ? cudaHostAlloc(&p, n, cudaHostAllocDefault) : cudaMalloc(&p, n); }
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) { if (pinned) cudaFreeHost(p); else cudaFree(p); }
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 4096;
        cudaError_t e = alloc(want);
        if (e != cudaSuccess) { e = alloc(n); want = n; }
        if (e == cudaSuccess) cap = want; else p = nullptr;
        return e;
    }
    void release() {
        if (p) { if (pinned) cudaFreeHost(p); else cudaFree(p); }
        p = nullptr; cap = 0;
    }
};

struct Slot {          // one in-flight chunk of the pipelined host path
    cudaStream_t stream = nullptr;
    Buf dSrc, dDst, dMeta, dPack, dPackOff;
    Buf hSrc{true}, hDst{true}, hMeta{true}, hPackOff{true};
    const int64_t* dDstOffArr = nullptr;   // device copies of the chunk's dst offsets / results (inside dMeta)
    const int32_t* dOutLenArr = nullptr;
    bool compact = false;             // stage 2 gathered the produced bytes on the device first
    std::vector<int64_t> compactOff;  // ... and this is where block k starts in the staging buffer
    // description of the chunk that is in flight
    int64_t b0 = 0, b1 = 0;           // block range
    int64_t dLo = 0;                  // dst extent origin (direct mode) or 0 (packed mode)
    bool dstPacked = false;
    std::vector<int64_t> packedDstOff;
    int64_t dstBytes = 0;             // device-side extent of the destination region of the chunk
    bool direct = false;              // stage 2 copied straight into the caller's buffer
    int state = 0;                    // 0 idle, 3 inputs on their way, 1 kernel + outLen enqueued, 2 data D2H enqueued
    Batch launch{};                   // the chunk's kernel arguments (state 3 -> 1)
};

constexpr int ENC_BIG_WAVES = 6;        // encode chunks in the middle of a batch: this many waves of blocks
constexpr int NSLOT = 4;                // chunks in flight per device (see run_host_slice)

// Everything the library keeps per GPU, set up once on first use with that GPU current: its SM count, a
// PRIVATE stream-ordered memory pool for the decoder's work lists and the encoder's tables (the process-wide
// default pool is never touched), the encoder's helper stream, the kernels' function attributes and the
// slots of the pipelined host path (guarded by `mu`).
struct Dev {
    std::once_flag once;
    cudaError_t err = cudaSuccess;
    int sms = 0;
    cudaMemPool_t pool = nullptr;
    cudaStream_t helper = nullptr;    // side stream of the encoder (encode_launch)
    std::mutex mu;
    Slot slot[NSLOT];
};

Dev* dev_state(int dev) {
    static Dev devs[64];
    if (dev < 0 || dev >= 64) return nullptr;
    Dev* d = &devs[dev];
    std::call_once(d->once, [d, dev] {
        // best effort, as their results never decide anything: the pickler's shared memory, and the split of
        // shared memory / L1 both encoder kernels ask for (they share SMs): just enough for the shared-memory
        // tables (+1 KiB the hardware reserves per CTA), the rest stays L1 for the input windows
        for (auto* pk : {k4::pickle_kernel<false>, k4::pickle_kernel<true>})
            cudaFuncSetAttribute(pk, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 k4::ENC_WARPS_PER_CTA * k4::ENC_SLOT_BYTES);
        const int carve = (k4::ENC_SM_WARPS * (k4::ENC_SLOT_BYTES + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024);
        cudaFuncSetAttribute(k4::encode_spec_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carve > 100 ? 100 : carve);
        cudaFuncSetAttribute(k4::encode_spec_gtab_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carve > 100 ? 100 : carve);
        cudaError_t e = cudaDeviceGetAttribute(&d->sms, cudaDevAttrMultiProcessorCount, dev);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(k4::decode_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(k4::TileSmem<k4::STAGE_SMALL>));
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(k4::decode_tile_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(k4::TileSmem<k4::STAGE_BIG>));
        if (e == cudaSuccess) {
            cudaMemPoolProps props = {};
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = dev;
            e = cudaMemPoolCreate(&d->pool, &props);
            if (e == cudaSuccess) {
                unsigned long long keep = 256ull << 20;         // cache up to 256 MiB of work lists and encoder tables
                cudaMemPoolSetAttribute(d->pool, cudaMemPoolAttrReleaseThreshold, &keep);
            }
        }
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&d->helper, cudaStreamNonBlocking);
        for (auto& s : d->slot)
            if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking);
        d->err = e;
    });
    return d;
}

// ---- kernel launchers (device pointers, current device) ------------------------------------------

// Enqueues the block encoder: a shared-memory-table kernel on `st` and, when the batch is big enough for
// it to pay, a global-memory-table kernel on a helper stream that runs beside it (fork / join by events).
// Both are persistent and pull blocks from one device counter.  The workspace (counter + the global
// tables) comes from the private stream-ordered pool.
cudaError_t encode_launch(const Batch& a, int level, const Dev& D, cudaStream_t st, int* launches) {
    const int n = (int)a.n;
    const int wave = D.sms * k4::ENC_SM_WARPS;
    const int gridS = n < wave ? n : wave;
    // The global-table warps need longer per block than the shared-memory warps: a batch that the latter
    // finish in one round goes to them alone.
    const bool useG = k4::ENC_GM_WARPS > 0 && n > wave;
    const int gridG = useG ? D.sms * k4::ENC_GM_WARPS : 0;
    const size_t tabBytes = (size_t)gridG * k4::ENC_GSLOT_BYTES;
    uint8_t* ws = nullptr;
    cudaError_t e = cudaMallocFromPoolAsync((void**)&ws, 256 + tabBytes, D.pool, st);
    if (e != cudaSuccess) return e;
    uint32_t* counter = reinterpret_cast<uint32_t*>(ws);
    e = cudaMemsetAsync(ws, 0, 4, st);
    cudaEvent_t fork = nullptr, join = nullptr;
    if (e == cudaSuccess && useG) {
        // ONE side stream per device: the global-table kernels of consecutive chunks run one after the other, so an
        // SM never holds more than ENC_GM_WARPS of them (CTAs of a queued launch would otherwise fill the SM's spare
        // CTA slots and crowd out the mix; measured slower)
        cudaStream_t hs = D.helper;
        e = cudaEventCreateWithFlags(&fork, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&join, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(fork, st);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(hs, fork, 0);
        if (e == cudaSuccess) {
            k4::encode_spec_gtab_kernel<<<gridG, 32, 0, hs>>>(a.srcBase, a.srcOff, a.srcLen, a.dstBase, a.dstOff,
                                                             a.dstCap, a.outLen, n, level, counter, ws + 256, wave);
            e = cudaGetLastError();
            (*launches)++;
        }
        if (e == cudaSuccess) e = cudaEventRecord(join, hs);
    }
    if (e == cudaSuccess && gridS > 0) {
        k4::encode_spec_kernel<<<gridS, 32, k4::ENC_SLOT_BYTES, st>>>(a.srcBase, a.srcOff, a.srcLen, a.dstBase,
                                                                      a.dstOff, a.dstCap, a.outLen, n, level, counter);
        e = cudaGetLastError();
        (*launches)++;
    }
    if (join && e == cudaSuccess) e = cudaStreamWaitEvent(st, join, 0);
    if (fork) cudaEventDestroy(fork);
    if (join) cudaEventDestroy(join);
    cudaFreeAsync(ws, st);
    return e;
}

// Every kernel of the codec is launched here, on `st` of the current device.
cudaError_t launch_op(Op op, const Batch& a, cudaStream_t st) {
    if (a.n <= 0) return cudaSuccess;
    int dev = 0;
    cudaGetDevice(&dev);
    const Dev* D = dev_state(dev);
    if (!D || D->err != cudaSuccess) return D ? D->err : cudaErrorInvalidDevice;
    const int n = (int)a.n;
    switch (op) {
    case OP_ENCODE: {
        int nl = 0;
        const cudaError_t ee = encode_launch(a, a.level | (a.x32 ? k4::ENC_FLAG_X32 : 0), *D, st, &nl);
        g_launches += nl;
        if (ee != cudaSuccess) { (void)cudaGetLastError(); return ee; }
        break;
    }
    case OP_DECODE:
    case OP_CHAIN: {
        const cudaError_t de = k4::decode_launch(a.srcBase, a.srcOff, a.srcLen, a.dstBase, a.dstOff, a.dstCap,
                                                 op == OP_CHAIN ? a.prefixLen : nullptr, a.outLen, n, st, D->pool, D->sms);
        if (de != cudaSuccess) { (void)cudaGetLastError(); return de; }
        g_launches += k4::DECODE_LAUNCHES;
        break;
    }
    case OP_GENERAL:
        k4::decode_general_kernel<<<(n + 3) / 4, 128, 0, st>>>(a.srcBase, a.srcOff, a.srcLen, a.dstBase, a.dstOff,
                                                               a.dstCap, a.dictBase, a.dictOff, a.dictLen, a.outLen,
                                                               n, a.partial ? 1 : 0);
        g_launches++;
        break;
    case OP_PICKLE:
    case OP_PICKLEW: {
        const int ctas = (n + k4::ENC_WARPS_PER_CTA - 1) / k4::ENC_WARPS_PER_CTA;
        (a.x32 ? k4::pickle_kernel<true> : k4::pickle_kernel<false>)<<<ctas, k4::ENC_WARPS_PER_CTA * 32,
                                                                        k4::ENC_WARPS_PER_CTA * k4::ENC_SLOT_BYTES, st>>>(
            a.srcBase, a.srcOff, a.srcLen, a.dstBase, a.dstOff, a.outLen, n, a.level, op == OP_PICKLEW ? 1 : 0);
        g_launches++;
        break;
    }
    case OP_UNPICKLE:
        k4::unpickle_kernel<<<(n + 3) / 4, 128, 0, st>>>(a.srcBase, a.srcOff, a.srcLen, a.dstBase, a.dstOff,
                                                         a.dstCap, a.outLen, n);
        g_launches++;
        break;
    case OP_USIZE:
        k4::unpickled_size_kernel<<<(n + 255) / 256, 256, 0, st>>>(a.srcBase, a.srcOff, a.srcLen, a.outLen, n);
        g_launches++;
        break;
    case OP_XXH32:
        k4::xxh32_batch_kernel<<<(unsigned)(((int64_t)n * 4 + 127) / 128), 128, 0, st>>>(
            a.srcBase, a.srcOff, a.srcLen, a.seed, reinterpret_cast<uint32_t*>(a.outLen), n);
        g_launches++;
        break;
    case OP_COPY:      // srcLen[i] bytes of block i
        k4::copy_blocks_kernel<<<n, 256, 0, st>>>(a.srcBase, a.srcOff, a.dstBase, a.dstOff, a.srcLen, n);
        g_launches++;
        break;
    case OP_ENCCHAIN: {   // one persistent warp kind; its counter comes from the private pool
        uint32_t* counter = nullptr;
        cudaError_t e = cudaMallocFromPoolAsync((void**)&counter, 256, D->pool, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(counter, 0, 4, st);
        if (e != cudaSuccess) { (void)cudaGetLastError(); return e; }
        const int wave = D->sms * k4::ENC_CHAIN_WARPS;
        (a.x32 ? k4::encode_chain_kernel<true> : k4::encode_chain_kernel<false>)<<<n < wave ? n : wave, 32, 0, st>>>(
            a.srcBase, a.srcOff, a.srcLen, a.prefixLen, a.dstBase, a.dstOff, a.dstCap, a.stateBase, a.stateOff,
            a.outLen, n, a.level, counter);
        g_launches++;
        cudaFreeAsync(counter, st);
        break;
    }
    case OP_DSIZE:     // one warp per block
        k4::decoded_size_kernel<<<(unsigned)(((int64_t)n * 32 + 127) / 128), 128, 0, st>>>(a.srcBase, a.srcOff,
                                                                                       a.srcLen, a.outLen, n);
        g_launches++;
        break;
    }
    return cudaGetLastError();
}

// ---- pipelined host path: encode / decode / pickle / unpickle --------------------------------------

inline int64_t dst_room(Op op, const Batch& a, int64_t i) {
    switch (op) {
    case OP_PICKLE: return a.srcLen[i] <= 0 ? 0 : (int64_t)a.srcLen[i] + 1;
    case OP_PICKLEW: return a.srcLen[i] <= 0 ? 0 : (int64_t)a.srcLen[i] + 1 + k4::pickle_diff_width(a.srcLen[i]);
    case OP_USIZE: return 0;
    case OP_ENCODE: {      // a capacity beyond compressBound(srcLen) behaves like compressBound (notLimited)
        const int64_t cap = a.dstCap[i] < 0 ? 0 : a.dstCap[i];
        const int64_t bound = a.srcLen[i] > 0 ? k4::max_output_size(a.srcLen[i]) : 0;
        return cap < bound ? cap : bound;
    }
    default: return a.dstCap[i] < 0 ? 0 : a.dstCap[i];
    }
}
inline int64_t src_size(const Batch& a, int64_t i) { return a.srcLen[i] < 0 ? 0 : a.srcLen[i]; }

void parallel_for_blocks(int64_t b0, int64_t b1, int64_t bytesHint, const std::function<void(int64_t, int64_t)>& fn);
int launch_chunk(Op op, Slot& s);

constexpr int64_t CHUNK_BYTES = 192ll << 20;   // src + dst payload per in-flight chunk

// Copies every produced byte of chunk [b0,b1) from the pinned staging buffer into the
// caller's destination; bytes at index >= outLen[i] are never touched.
void scatter_chunk(Op op, const Batch& a, Slot& s) {
    if (op == OP_USIZE) return;
    const uint8_t* stage = (const uint8_t*)s.hDst.p;
    int64_t total = 0;
    for (int64_t i = s.b0; i < s.b1; i++) total += std::max<int32_t>(a.outLen[i], 0);
    parallel_for_blocks(s.b0, s.b1, total, [&](int64_t lo, int64_t hi) {
        for (int64_t i = lo; i < hi; i++) {
            const int32_t r = a.outLen[i];
            if (r <= 0) continue;
            const int64_t off = s.compact ? s.compactOff[i - s.b0]
                                : (s.dstPacked ? s.packedDstOff[i - s.b0] : a.dstOff[i] - s.dLo);
            memcpy(a.dstBase + a.dstOff[i], stage + off, (size_t)r);
        }
    });
}

// stage 2: the kernel of the chunk has finished -> per-block results to the caller, then the
// data D2H.  When every block filled its whole slot and the slots are contiguous (the decode
// case) the bytes go straight into the caller's buffer in one copy; otherwise through the pinned
// staging buffer and a host-side scatter (stage 3) that leaves bytes >= outLen[i] untouched.
int stage2_slot(Op op, const Batch& a, Slot& s) {
    if (s.state == 3) { int rc = launch_chunk(op, s); if (rc != K4LZ4_OK) return rc; }
    if (s.state != 1) return K4LZ4_OK;
    CU_TRY(cudaStreamSynchronize(s.stream));
    memcpy(a.outLen + s.b0, (const int32_t*)s.hMeta.p, sizeof(int32_t) * (size_t)(s.b1 - s.b0));
    s.state = 2;
    s.direct = false;
    s.compact = false;
    if (op == OP_USIZE || s.dstBytes <= 0) return K4LZ4_OK;
    bool full = !s.dstPacked;
    int64_t sum = 0;
    for (int64_t i = s.b0; i < s.b1 && full; i++) {
        const int64_t room = dst_room(op, a, i);
        full = (int64_t)a.outLen[i] == room;
        sum += room;
    }
    full = full && sum == s.dstBytes;                 // slots tile the extent exactly: no gaps
    if (full) {
        s.direct = true;
        CU_TRY(cudaMemcpyAsync(a.dstBase + s.dLo, s.dDst.p, (size_t)s.dstBytes, cudaMemcpyDeviceToHost, s.stream));
    } else {
        // variable-length results (encode, pickle, short decodes): gather the produced bytes on the
        // device (copy_blocks_kernel) so that only they cross PCIe, not the slots' slack
        const int64_t nb = s.b1 - s.b0;
        s.compactOff.resize((size_t)nb);
        int64_t total = 0;
        for (int64_t k = 0; k < nb; k++) {
            s.compactOff[(size_t)k] = total;
            const int32_t r = a.outLen[s.b0 + k];
            if (r > 0) total += ((int64_t)r + 15) & ~int64_t(15);
        }
        s.compact = true;
        s.dstBytes = total;
        if (total == 0) return K4LZ4_OK;
        CU_TRY(s.hPackOff.ensure((size_t)nb * 8));
        CU_TRY(s.dPackOff.ensure((size_t)nb * 8));
        CU_TRY(s.dPack.ensure((size_t)total + 16));
        CU_TRY(s.hDst.ensure((size_t)total + 16));
        memcpy(s.hPackOff.p, s.compactOff.data(), (size_t)nb * 8);
        CU_TRY(cudaMemcpyAsync(s.dPackOff.p, s.hPackOff.p, (size_t)nb * 8, cudaMemcpyHostToDevice, s.stream));
        Batch g{(const uint8_t*)s.dDst.p, s.dDstOffArr, s.dOutLenArr, (uint8_t*)s.dPack.p,
                (const int64_t*)s.dPackOff.p, nullptr, nullptr, nb};
        CU_TRY(launch_op(OP_COPY, g, s.stream));
        CU_TRY(cudaMemcpyAsync(s.hDst.p, s.dPack.p, (size_t)total, cudaMemcpyDeviceToHost, s.stream));
    }
    return K4LZ4_OK;
}

// stage 3: data has landed
int stage3_slot(Op op, const Batch& a, Slot& s) {
    if (s.state == 1 || s.state == 3) { int rc = stage2_slot(op, a, s); if (rc != K4LZ4_OK) return rc; }
    if (s.state != 2) return K4LZ4_OK;
    s.state = 0;
    CU_TRY(cudaStreamSynchronize(s.stream));
    if (!s.direct) scatter_chunk(op, a, s);
    return K4LZ4_OK;
}

// stage 1a: stage the chunk's inputs and block table on the device (asynchronous copies on the slot's stream)
int enqueue_chunk(Op op, const Batch& a, Slot& s, int64_t b0, int64_t b1) {
    const int64_t nb = b1 - b0;
    s.b0 = b0; s.b1 = b1;
    // extents
    int64_t sLo = INT64_MAX, sHi = INT64_MIN, dLo = INT64_MAX, dHi = INT64_MIN, sSum = 0, dSum = 0;
    for (int64_t i = b0; i < b1; i++) {
        const int64_t sl = src_size(a, i), dl = dst_room(op, a, i);
        if (sl > 0) { sLo = std::min(sLo, a.srcOff[i]); sHi = std::max(sHi, a.srcOff[i] + sl); sSum += sl; }
        if (dl > 0) { dLo = std::min(dLo, a.dstOff[i]); dHi = std::max(dHi, a.dstOff[i] + dl); dSum += dl; }
    }
    if (sSum == 0) { sLo = 0; sHi = 0; }
    if (dSum == 0) { dLo = 0; dHi = 0; }
    const bool srcPacked = (sHi - sLo) > sSum + sSum / 4 + 65536;
    const bool dstPacked = (dHi - dLo) > dSum + dSum / 4 + 65536;
    s.dstPacked = dstPacked;
    s.dLo = dLo;

    // meta layout (device): srcOff[nb] dstOff[nb] (int64) | srcLen[nb] dstCap[nb] outLen[nb] (int32)
    const size_t metaBytes = (size_t)nb * (8 + 8 + 4 + 4 + 4);
    CU_TRY(s.dMeta.ensure(metaBytes));
    CU_TRY(s.hMeta.ensure(metaBytes));
    int64_t* hSrcOff = (int64_t*)s.hMeta.p;
    int64_t* hDstOff = hSrcOff + nb;
    int32_t* hSrcLen = (int32_t*)(hDstOff + nb);
    int32_t* hDstCap = hSrcLen + nb;
    // (outLen comes back into the front of hMeta after the kernel; see below)
    int64_t* dSrcOff = (int64_t*)s.dMeta.p;
    int64_t* dDstOff = dSrcOff + nb;
    int32_t* dSrcLen = (int32_t*)(dDstOff + nb);
    int32_t* dDstCap = dSrcLen + nb;
    int32_t* dOutLen = dDstCap + nb;

    const int64_t srcBytes = srcPacked ? sSum : (sHi - sLo);
    const int64_t dstBytes = dstPacked ? dSum : (dHi - dLo);
    CU_TRY(s.dSrc.ensure((size_t)srcBytes + 16));
    if (op != OP_USIZE) CU_TRY(s.dDst.ensure((size_t)dstBytes + 16));
    s.dstBytes = (op == OP_USIZE) ? 0 : dstBytes;
    if (dstPacked) s.packedDstOff.resize((size_t)nb);

    int64_t sp = 0, dp = 0;
    if (srcPacked) CU_TRY(s.hSrc.ensure((size_t)sSum + 16));
    for (int64_t i = b0; i < b1; i++) {
        const int64_t k = i - b0;
        const int64_t sl = src_size(a, i), dl = dst_room(op, a, i);
        hSrcLen[k] = a.srcLen[i];
        hDstCap[k] = (op == OP_PICKLE || op == OP_PICKLEW || op == OP_USIZE) ? 0 : (op == OP_ENCODE ? (int32_t)dl : a.dstCap[i]);
        if (srcPacked) {
            hSrcOff[k] = sp;
            if (sl > 0) memcpy((uint8_t*)s.hSrc.p + sp, a.srcBase + a.srcOff[i], (size_t)sl);
            sp += sl;
        } else {
            hSrcOff[k] = sl > 0 ? a.srcOff[i] - sLo : 0;
        }
        if (dstPacked) { hDstOff[k] = dp; s.packedDstOff[(size_t)k] = dp; dp += dl; }
        else hDstOff[k] = dl > 0 ? a.dstOff[i] - dLo : 0;
    }

    cudaStream_t st = s.stream;
    if (srcBytes > 0)
        CU_TRY(cudaMemcpyAsync(s.dSrc.p, srcPacked ? (const void*)s.hSrc.p : (const void*)(a.srcBase + sLo),
                               (size_t)srcBytes, cudaMemcpyHostToDevice, st));
    CU_TRY(cudaMemcpyAsync(s.dMeta.p, s.hMeta.p, (size_t)nb * 24, cudaMemcpyHostToDevice, st));
    s.launch = a;
    s.launch.srcBase = (const uint8_t*)s.dSrc.p; s.launch.srcOff = dSrcOff; s.launch.srcLen = dSrcLen;
    s.launch.dstBase = (uint8_t*)s.dDst.p; s.launch.dstOff = dDstOff; s.launch.dstCap = dDstCap;
    s.launch.outLen = dOutLen; s.launch.n = nb;
    s.dDstOffArr = dDstOff;
    s.dOutLenArr = dOutLen;
    s.state = 3;
    return K4LZ4_OK;
}

// stage 1b: the kernel of a chunk whose inputs are on their way (same stream), then its per-block results
int launch_chunk(Op op, Slot& s) {
    if (s.state != 3) return K4LZ4_OK;
    CU_TRY(launch_op(op, s.launch, s.stream));
    // outLen lands at the front of hMeta (offset arrays there are no longer needed once the
    // H2D of the chunk has been issued *and completed*; stream order guarantees that)
    CU_TRY(cudaMemcpyAsync(s.hMeta.p, s.launch.outLen, (size_t)s.launch.n * 4, cudaMemcpyDeviceToHost, s.stream));
    s.state = 1;
    return K4LZ4_OK;
}

// One device, blocks [b0, b1): chunked + double-buffered (H2D/kernel/D2H of chunk c overlap
// the host-side scatter of chunk c-1 and the copies of chunk c+1 on the other stream).
int run_host_slice(Op op, const Batch& a, int64_t b0, int64_t b1, int dev) {
    if (b1 <= b0) return K4LZ4_OK;
    DeviceGuard g(dev);
    if (!g.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", dev);
    Dev* ctx = dev_state(dev);
    if (!ctx) return fail(K4LZ4_E_CUDA, "device %d: no state", dev);
    if (ctx->err != cudaSuccess) return fail(K4LZ4_E_CUDA, "device %d setup failed: %s", dev, cudaGetErrorString(ctx->err));
    std::lock_guard<std::mutex> lk(ctx->mu);
    // blocks the encoder finishes in about one shared-memory-warp block time (a global-table warp counts half)
    const int64_t W = (int64_t)ctx->sms * (k4::ENC_SM_WARPS + (k4::ENC_GM_WARPS + 1) / 2);
    int rc = K4LZ4_OK;
    // Chunk boundaries.  Encode: a warp works on one block for milliseconds; consecutive chunks' kernels
    // overlap (one-warp CTAs leave individually and the next launch, on another stream, moves in), so a
    // chunk only has to be long enough to hide its copies and the host's work behind the previous kernel:
    // ENC_BIG_WAVES waves in the middle of a batch, one and two waves at both ends so that the pipeline
    // fills and drains fast.
    auto chunk_end = [&](int64_t i, int c) {
        int64_t bytes = 0, j = i;
        int64_t limit = CHUNK_BYTES, maxBlocks = INT64_MAX;
        if (op == OP_ENCODE) {
            const int64_t rem = b1 - i;
            limit = 2560ll << 20;
            if (c == 0) maxBlocks = W;
            else if (c == 1) maxBlocks = 2 * W;
            else if (2 * rem <= 3 * W) maxBlocks = rem;
            else if (2 * rem <= 7 * W) maxBlocks = std::min<int64_t>(2 * W, rem - W);
            else maxBlocks = std::max<int64_t>(std::min<int64_t>(ENC_BIG_WAVES * W, rem - 3 * W), W);
        } else if (op == OP_PICKLE || op == OP_PICKLEW) {
            limit = 4 * CHUNK_BYTES;
        }
        while (j < b1 && j - i < maxBlocks && (j == i || bytes + src_size(a, j) + dst_room(op, a, j) <= limit)) {
            bytes += src_size(a, j) + dst_room(op, a, j);
            j++;
        }
        return j;
    };
    // Four chunks in flight, copies issued two chunks ahead, kernels one:
    //   inputs(c+1) -> wait kernel(c-1), its results, gather + data D2H (stage 2) -> kernel(c+1) -> scatter(c-2)
    // so while kernel c runs, chunk c+1 is queued behind it with its inputs already on the device, the data
    // of chunk c-1 crosses PCIe and the host scatters chunk c-2: the GPU never waits for PCIe or for the host.
    // No more than two kernels are queued at any time (a third one would crowd the SMs with the CTAs of
    // three launches; measured slower).
    auto slot_of = [&](int c) -> Slot& { return ctx->slot[((c % NSLOT) + NSLOT) % NSLOT]; };
    int64_t next = b0;                                     // first block not yet staged
    int staged = 0;                                        // chunks whose inputs have been issued
    auto stage_next = [&]() -> int {
        if (next >= b1) return K4LZ4_OK;
        Slot& s = slot_of(staged);
        int r = stage3_slot(op, a, s);                     // chunk staged-4: long done
        if (r != K4LZ4_OK) return r;
        const int64_t j = chunk_end(next, staged);
        r = enqueue_chunk(op, a, s, next, j);
        next = j; staged++;
        return r;
    };
    rc = stage_next();
    if (rc == K4LZ4_OK) rc = launch_chunk(op, slot_of(0));
    for (int c = 0; rc == K4LZ4_OK && c < staged; c++) {
        if ((rc = stage_next()) != K4LZ4_OK) break;                                       // inputs of chunk c+1
        if (c >= 1 && (rc = stage2_slot(op, a, slot_of(c - 1))) != K4LZ4_OK) break;       // kernel c-1 done
        if (c + 1 < staged && (rc = launch_chunk(op, slot_of(c + 1))) != K4LZ4_OK) break; // kernel c+1 queued
        if (c >= 2 && (rc = stage3_slot(op, a, slot_of(c - 2))) != K4LZ4_OK) break;       // scatter c-2
    }
    if (rc != K4LZ4_OK) { for (auto& s : ctx->slot) s.state = 0; cudaDeviceSynchronize(); return rc; }
    // drain in issue order: results + data D2H of everything still on the device first, then the scatters
    for (int k = staged - NSLOT; k < staged && rc == K4LZ4_OK; k++) if (k >= 0) rc = stage2_slot(op, a, slot_of(k));
    for (int k = staged - NSLOT; k < staged && rc == K4LZ4_OK; k++) if (k >= 0) rc = stage3_slot(op, a, slot_of(k));
    if (rc != K4LZ4_OK) { for (auto& s : ctx->slot) s.state = 0; cudaDeviceSynchronize(); }
    return rc;
}

void parallel_for_blocks(int64_t b0, int64_t b1, int64_t bytesHint,
                         const std::function<void(int64_t, int64_t)>& fn) {
    unsigned hw = std::thread::hardware_concurrency();
    int T = (int)std::min<unsigned>(hw ? hw : 1, 16);
    if (bytesHint < (8 << 20) || b1 - b0 < 2 * T) T = 1;
    if (T <= 1) { fn(b0, b1); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++) {
        int64_t lo = b0 + (b1 - b0) * t / T, hi = b0 + (b1 - b0) * (t + 1) / T;
        th.emplace_back([=, &fn] { fn(lo, hi); });
    }
    for (auto& t : th) t.join();
}

// Best effort: run the calling thread on the CPUs of the NUMA node GPU `dev` is attached to, so that
// the pinned staging buffers it allocates (first touch) and its memcpy traffic stay node-local.
// (HGX boards hang GPUs 0-3 and 4-7 off different sockets; staging through the far socket halves the
// aggregate PCIe rate of an all-devices call.)
void bind_thread_near_gpu(int dev) {
#if defined(__linux__)
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), dev) != cudaSuccess) { (void)cudaGetLastError(); return; }
    for (char* c = bus; *c; c++) *c = (char)tolower(*c);
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return;
    char list[4096] = {0};
    const size_t got = fread(list, 1, sizeof(list) - 1, f);
    fclose(f);
    if (got == 0) return;
    cpu_set_t want, have;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof(have), &have) != 0) return;
    int any = 0;
    for (char* p = list; *p;) {
        char* e;
        long lo = strtol(p, &e, 10), hi = lo;
        if (e == p) break;
        if (*e == '-') { p = e + 1; hi = strtol(p, &e, 10); }
        for (long c = lo; c <= hi && c < CPU_SETSIZE; c++) if (CPU_ISSET((int)c, &have)) { CPU_SET((int)c, &want); any = 1; }
        p = (*e == ',') ? e + 1 : e;
        if (*e != ',' ) break;
    }
    if (any) sched_setaffinity(0, sizeof(want), &want);
#else
    (void)dev;
#endif
}

int run_host(Op op, const Batch& a, int device) {
    const int64_t n = a.n;
    const int ndev = device_count_cached();
    if (device >= 0 || ndev == 1) return run_host_slice(op, a, 0, n, device >= 0 ? device : 0);

    // K4LZ4_ALL_DEVICES: contiguous split balanced by bytes, one host thread per GPU
    std::vector<int64_t> cut(ndev + 1, n);
    cut[0] = 0;
    int64_t total = 0;
    for (int64_t i = 0; i < n; i++) total += src_size(a, i) + dst_room(op, a, i) + 64;
    int64_t acc = 0; int g = 1;
    for (int64_t i = 0; i < n && g < ndev; i++) {
        acc += src_size(a, i) + dst_room(op, a, i) + 64;
        while (g < ndev && acc >= total * g / ndev) cut[g++] = i + 1;
    }
    std::vector<int> rcs(ndev, K4LZ4_OK);
    std::vector<std::string> errs(ndev);
    std::vector<std::thread> th;
    for (int d = 0; d < ndev; d++)
        th.emplace_back([&, d] {
            bind_thread_near_gpu(d);
            rcs[d] = run_host_slice(op, a, cut[d], cut[d + 1], d);
            if (rcs[d] != K4LZ4_OK) errs[d] = t_err;
        });
    for (auto& t : th) t.join();
    for (int d = 0; d < ndev; d++) if (rcs[d] != K4LZ4_OK) { t_err = errs[d]; return rcs[d]; }
    return K4LZ4_OK;
}

// ---- synchronous host path: dictionary / partial / chained decode and XXH32 ------------------------

struct DevMem {         // the call's device buffer: grows with the chunks, freed when the call returns
    void* p = nullptr; size_t cap = 0;
    ~DevMem() { if (p) cudaFree(p); }
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        cap = 0;
        const cudaError_t e = cudaMalloc(&p, n);
        if (e == cudaSuccess) cap = n; else p = nullptr;
        return e;
    }
};

constexpr int64_t STAGE_BYTES = 256ll << 20;   // staged payload per chunk

// One GPU, no pipelining: per chunk of at most STAGE_BYTES, everything the kernel reads is packed into one
// host buffer -- the block table, the sources, the dictionaries (when the batch has them) and, with a
// prefix, the destination slots [history | capacity] (16-aligned, history filled in: all the decoder reads
// of a stream is its last <= 65535 bytes) -- and goes up in one copy.  The chained encoder's history goes in
// front of its source instead ([history | source], 16-aligned) and its state records (16-aligned) go up and
// come back whole.  The results and the destination region come back, and exactly outLen[i] > 0 bytes of
// each block are copied to the caller.  A batch without dstCap (XXH32) has no destination: its per-block
// result is the whole output.
int run_staged(Op op, const Batch& b, int dev) {
    DeviceGuard guard(dev);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", dev);
    const bool dict = b.dictBase != nullptr, prefix = b.prefixLen != nullptr, dst = b.dstCap != nullptr;
    const bool enc = op == OP_ENCCHAIN;
    constexpr int64_t SB = K4LZ4_CHAIN_STATE_BYTES;
    auto hist = [&](int64_t i) -> int64_t { return prefix ? std::min<int32_t>(b.prefixLen[i], 65535) : 0; };
    auto cap = [&](int64_t i) -> int64_t {      // the encoder never writes more than compressBound(srcLen)
        const int64_t c = dst ? std::max<int32_t>(b.dstCap[i], 0) : 0;
        return enc ? std::min<int64_t>(c, b.srcLen[i] > 0 ? k4::max_output_size(b.srcLen[i]) : 0) : c;
    };
    auto dlen = [&](int64_t i) -> int64_t { return dict ? std::max<int32_t>(b.dictLen[i], 0) : 0; };
    auto up = [](int64_t x) { return (x + 255) & ~int64_t(255); };
    auto a16 = [](int64_t x) { return (x + 15) & ~int64_t(15); };
    std::vector<uint8_t> h;          // reused by every chunk: the kernel reads only bytes the chunk has written
    DevMem d;
    for (int64_t i = 0, j; i < b.n; i = j) {
        int64_t bytes = 0;
        for (j = i; j < b.n; j++) {
            const int64_t add = src_size(b, j) + dlen(j) + cap(j) + (prefix ? hist(j) + 16 : 0) + (enc ? SB : 0);
            if (j > i && bytes + add > STAGE_BYTES) break;
            bytes += add;
        }
        const int64_t nb = j - i;
        // block table: srcOff dstOff dictOff stateOff (int64) | srcLen dstCap dictLen prefixLen outLen (int32)
        int64_t sTot = 0, diTot = 0, dTot = 0;
        for (int64_t k = 0; k < nb; k++) {
            sTot = (enc ? a16(sTot + hist(i + k)) : sTot) + src_size(b, i + k);
            diTot += dlen(i + k);
            dTot = (prefix && !enc ? a16(dTot + hist(i + k)) : dTot) + cap(i + k);
        }
        const int64_t stTot = enc ? nb * SB : 0;
        const int64_t srcAt = up(nb * (4 * 8 + 5 * 4)), dictAt = up(srcAt + sTot), stateAt = up(dictAt + diTot);
        const int64_t dstAt = up(stateAt + stTot);
        const int64_t total = dstAt + dTot;
        if (h.size() < (size_t)total + 16) h.resize((size_t)total + 16);
        int64_t* so = (int64_t*)h.data(); int64_t* doff = so + nb; int64_t* dio = doff + nb; int64_t* sto = dio + nb;
        int32_t* sl = (int32_t*)(sto + nb); int32_t* dc = sl + nb; int32_t* dl = dc + nb; int32_t* pl = dl + nb;
        int32_t* res = pl + nb;
        for (int64_t k = 0, sp = 0, dip = 0, dp = 0; k < nb; k++) {
            const int64_t x = i + k, hl = hist(x);
            sl[k] = b.srcLen[x]; dc[k] = dst ? b.dstCap[x] : 0; dl[k] = (int32_t)dlen(x);
            pl[k] = enc ? b.prefixLen[x] : (int32_t)hl;   // the encoder's dictSize clamp needs the caller's value
            so[k] = enc ? a16(sp + hl) : sp; dio[k] = dip; sto[k] = k * SB;
            doff[k] = prefix && !enc ? a16(dp + hl) : dp;
            if (enc && hl > 0) memcpy(h.data() + srcAt + so[k] - hl, b.srcBase + b.srcOff[x] - hl, (size_t)hl);
            if (sl[k] > 0) memcpy(h.data() + srcAt + so[k], b.srcBase + b.srcOff[x], (size_t)sl[k]);
            if (dl[k] > 0) memcpy(h.data() + dictAt + dip, b.dictBase + b.dictOff[x], (size_t)dl[k]);
            if (enc) memcpy(h.data() + stateAt + sto[k], b.stateBase + b.stateOff[x], (size_t)SB);
            else if (prefix && hl > 0) memcpy(h.data() + dstAt + doff[k] - hl, b.dstBase + b.dstOff[x] - hl, (size_t)hl);
            sp = so[k] + src_size(b, x); dip += dl[k]; dp = doff[k] + cap(x);
        }
        CU_TRY(d.ensure((size_t)total + 16));
        uint8_t* D = (uint8_t*)d.p;
        CU_TRY(cudaMemcpy(D, h.data(), (size_t)(prefix && !enc ? total : dstAt), cudaMemcpyHostToDevice));
        int32_t* dRes = (int32_t*)(D + ((uint8_t*)res - h.data()));
        Batch kb = b;                                // the same batch, on the device
        kb.srcBase = D + srcAt; kb.srcOff = (int64_t*)D; kb.srcLen = (int32_t*)(D + ((uint8_t*)sl - h.data()));
        kb.dstBase = D + dstAt; kb.dstOff = kb.srcOff + nb; kb.dstCap = dst ? kb.srcLen + nb : nullptr;
        kb.dictBase = dict ? D + dictAt : nullptr; kb.dictOff = kb.srcOff + 2 * nb; kb.dictLen = kb.srcLen + 2 * nb;
        kb.prefixLen = prefix ? kb.srcLen + 3 * nb : nullptr;
        kb.stateBase = enc ? D + stateAt : nullptr; kb.stateOff = enc ? kb.srcOff + 3 * nb : nullptr;
        kb.outLen = dRes; kb.n = nb;
        CU_TRY(launch_op(op, kb, nullptr));
        CU_TRY(cudaMemcpy(b.outLen + i, dRes, (size_t)nb * 4, cudaMemcpyDeviceToHost));
        if (enc) {
            CU_TRY(cudaMemcpy(h.data() + stateAt, D + stateAt, (size_t)stTot, cudaMemcpyDeviceToHost));
            for (int64_t k = 0; k < nb; k++)
                memcpy(b.stateBase + b.stateOff[i + k], h.data() + stateAt + sto[k], (size_t)SB);
        }
        if (!dst || dTot == 0) continue;
        CU_TRY(cudaMemcpy(h.data() + dstAt, D + dstAt, (size_t)dTot, cudaMemcpyDeviceToHost));
        for (int64_t k = 0; k < nb; k++) {
            const int32_t r = b.outLen[i + k];
            if (r > 0) memcpy(b.dstBase + b.dstOff[i + k], h.data() + dstAt + doff[k], (size_t)r);
        }
    }
    return K4LZ4_OK;
}

int run(Op op, const Batch& b, int memKind, void* stream, int device) {
    const int rc = check(op, b, memKind, device);
    if (rc != K4LZ4_OK || b.n == 0) return rc;
    if (memKind == K4LZ4_MEM_HOST)
        return (op == OP_GENERAL || op == OP_CHAIN || op == OP_XXH32 || op == OP_ENCCHAIN || op == OP_DSIZE)
                   ? run_staged(op, b, device < 0 ? 0 : device) : run_host(op, b, device);
    DeviceGuard g(device);
    if (!g.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", device);
    CU_TRY(launch_op(op, b, (cudaStream_t)stream));
    return K4LZ4_OK;
}

// One block in host memory through the batched path, after the reference's answers that need no device.
int32_t run_one(Op op, const uint8_t* src, int32_t srcLen, uint8_t* dst, int32_t dstCap, int level = 0,
                bool x32 = false, const uint8_t* dict = nullptr, int32_t dictLen = 0, bool partial = false) {
    if (srcLen <= 0) return 0;                       // LZ4Codec.cs:45-46,108-109,129-130,150-151
    if (op == OP_ENCODE && level >= 3) return K4LZ4_R_DELEGATE;
    if (!src || (!dst && dstCap > 0) || (!dict && dictLen > 0)) return fail(K4LZ4_E_ARG, "null pointer argument");
    if (dstCap <= 0) return -1;                      // nothing fits in an empty target (LL64.dec.cs:162-168; LZ4Codec.cs:135)
    int64_t zero = 0; int32_t out = -1;
    Batch b{src, &zero, &srcLen, dst, &zero, &dstCap, &out, 1};
    // the encoder reads bits 0-7 of its level word as the level and bit 8 as the 32-bit switch: a level
    // below 0 reaches it as that word
    const int word = level | (x32 ? k4::ENC_FLAG_X32 : 0);
    b.level = word & 0xFF; b.x32 = (word & k4::ENC_FLAG_X32) != 0;
    if (dictLen > 0) { b.dictBase = dict; b.dictOff = &zero; b.dictLen = &dictLen; }
    b.partial = partial;
    const int rc = run(op, b, K4LZ4_MEM_HOST, nullptr, 0);
    return rc != K4LZ4_OK ? rc : out;
}

// Counter array `sym` (4 x u64) of `device`, after the device is idle.
int read_stats(const void* sym, int32_t device, uint64_t* out4, int32_t reset) {
    if (!out4) return fail(K4LZ4_E_ARG, "null pointer argument");
    const int rc = check_device(device, 1);
    if (rc != K4LZ4_OK) return rc;
    DeviceGuard g(device);
    if (!g.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", device);
    unsigned long long v[4] = {0, 0, 0, 0};
    CU_TRY(cudaDeviceSynchronize());
    CU_TRY(cudaMemcpyFromSymbol(v, sym, sizeof(v)));
    for (int i = 0; i < 4; i++) out4[i] = v[i];
    if (reset) { unsigned long long z[4] = {0, 0, 0, 0}; CU_TRY(cudaMemcpyToSymbol(sym, z, sizeof(z))); }
    return K4LZ4_OK;
}

// ---- LZ4 frames (frame.cuh) ---------------------------------------------------------------------------------

constexpr int FRAME_FLAGS = K4LZ4_FRAME_INDEPENDENT | K4LZ4_FRAME_BLOCK_CHECKSUM | K4LZ4_FRAME_CONTENT_CHECKSUM;
static_assert(K4LZ4_FRAME_INDEPENDENT == k4::FR_INDEPENDENT && K4LZ4_FRAME_BLOCK_CHECKSUM == k4::FR_BLOCK_SUM &&
              K4LZ4_FRAME_CONTENT_CHECKSUM == k4::FR_CONTENT_SUM && K4LZ4_R_CORRUPT == k4::FR_CORRUPT &&
              K4LZ4_R_DELEGATE == k4::FR_DELEGATE && K4LZ4_R_DST_SMALL == k4::FR_DST_SMALL, "frame codes");
constexpr int64_t FRAME_SCRATCH = 512ll << 20;   // encoder output slots per launch

// LZ4EncoderBase.cs:29: max(1024, blockSize rounded up to 1 KiB); 0 for a block size a frame cannot declare.
int32_t frame_block_size(int32_t blockSize) {
    if (blockSize <= 0 || blockSize > (4 << 20)) return 0;
    return std::max<int32_t>(1024, (blockSize + 1023) / 1024 * 1024);
}

int64_t frame_bound_of(int64_t length, int32_t bs, int flags) {
    const int64_t nb = (length + bs - 1) / bs;
    return 7 + nb * (4 + ((flags & K4LZ4_FRAME_BLOCK_CHECKSUM) ? 4 : 0)) + length + 4 +
           ((flags & K4LZ4_FRAME_CONTENT_CHECKSUM) ? 4 : 0);
}

// Magic, FLG, BD (LZ4FrameWriter.cs:183-188: the code of the caller's block size) and HC, little-endian.
uint64_t frame_header(int32_t blockSize, int flags) {
    const int code = blockSize <= (1 << 16) ? 4 : blockSize <= (1 << 18) ? 5 : blockSize <= (1 << 20) ? 6 : 7;
    const uint8_t fb[2] = {(uint8_t)((1 << 6) | ((flags & K4LZ4_FRAME_INDEPENDENT) ? 1 << 5 : 0) |
                                     ((flags & K4LZ4_FRAME_BLOCK_CHECKSUM) ? 1 << 4 : 0) |
                                     ((flags & K4LZ4_FRAME_CONTENT_CHECKSUM) ? 1 << 2 : 0)),
                           (uint8_t)(code << 4)};
    const uint8_t hc = (uint8_t)(k4::xxh32_host(fb, 2, 0) >> 8);
    return (uint64_t)k4::FRAME_MAGIC | ((uint64_t)fb[0] << 32) | ((uint64_t)fb[1] << 40) | ((uint64_t)hc << 48);
}

// Stream-ordered allocations of one frame call, from the device's private pool; freed (in stream order) at the end.
struct FramePool {
    cudaMemPool_t pool; cudaStream_t st;
    std::vector<void*> ps;
    cudaError_t err = cudaSuccess;
    FramePool(cudaMemPool_t p, cudaStream_t s) : pool(p), st(s) {}
    ~FramePool() { for (void* p : ps) cudaFreeAsync(p, st); }
    template <class T> T* get(int64_t count) {
        void* p = nullptr;
        if (err == cudaSuccess) err = cudaMallocFromPoolAsync(&p, (size_t)std::max<int64_t>(count, 1) * sizeof(T) + 16, pool, st);
        if (err != cudaSuccess) return nullptr;
        ps.push_back(p);
        return (T*)p;
    }
};

inline unsigned grid_of(int64_t n, int t = 128) { return (unsigned)std::max<int64_t>((n + t - 1) / t, 1); }

#define FR_TRY(expr) do { const cudaError_t e__ = (expr); if (e__ != cudaSuccess) return e__; } while (0)
#define FR_LAUNCH() FR_TRY(cudaGetLastError())

// Decode (or, with sizeOnly, only the content sizes of) b.n frames in device memory on `st`: parse, scan, one
// host synchronisation for the block and step counts, then everything else enqueued.  b.dstCap may be null
// (sizeOnly).
cudaError_t frame_decode_dev(const Batch& b, bool sizeOnly, cudaStream_t st) {
    int dev = 0;
    cudaGetDevice(&dev);
    const Dev* D = dev_state(dev);
    if (!D || D->err != cudaSuccess) return D ? D->err : cudaErrorInvalidDevice;
    const int n = (int)b.n;
    FramePool P(D->pool, st);
    k4::FrameRec* fr = P.get<k4::FrameRec>(n);
    k4::FrameTotals* tot = P.get<k4::FrameTotals>(1);
    FR_TRY(P.err);
    FR_TRY(cudaMemsetAsync(tot, 0, sizeof(k4::FrameTotals), st));
    k4::frame_parse_kernel<<<grid_of(n), 128, 0, st>>>(0, b.srcBase, b.srcOff, b.srcLen, n, fr, k4::FrameTable{}, tot);
    FR_LAUNCH();
    k4::frame_scan_kernel<<<1, 1024, 0, st>>>(fr, n, tot, sizeOnly ? 0 : 1);
    FR_LAUNCH();
    g_launches += 2;
    k4::FrameTotals h{};
    FR_TRY(cudaMemcpyAsync(&h, tot, sizeof(h), cudaMemcpyDeviceToHost, st));
    FR_TRY(cudaStreamSynchronize(st));                 // the one wait: the table's size and the number of steps
    const int64_t nB = h.blocks;
    uint8_t* rows = P.get<uint8_t>(nB * k4::FRAME_ROW_BYTES + 16 * 16);
    FR_TRY(P.err);
    k4::FrameTable t;
    {
        uint8_t* p = rows;
        auto take = [&](int64_t bytes) { uint8_t* q = p; p += (bytes + 15) & ~int64_t(15); return q; };
        t.srcOff = (int64_t*)take(nB * 8); t.fin = (int64_t*)take(nB * 8); t.dst = (int64_t*)take(nB * 8);
        t.cpySrc = (int64_t*)take(nB * 8);
        t.len = (int32_t*)take(nB * 4); t.kind = (int32_t*)take(nB * 4); t.sum = (uint32_t*)take(nB * 4);
        t.frame = (int32_t*)take(nB * 4); t.idx = (int32_t*)take(nB * 4); t.size = (int32_t*)take(nB * 4);
        t.cap = (int32_t*)take(nB * 4); t.ilen = (int32_t*)take(nB * 4); t.res = (int32_t*)take(nB * 4);
        t.ckLen = (int32_t*)take(nB * 4); t.got = (uint32_t*)take(nB * 4); t.cpyLen = (int32_t*)take(nB * 4);
    }
    k4::frame_parse_kernel<<<grid_of(n), 128, 0, st>>>(1, b.srcBase, b.srcOff, b.srcLen, n, fr, t, nullptr);
    FR_LAUNCH();
    g_launches++;
    if (nB > 0) {
        k4::block_size_walk_kernel<<<grid_of(nB * 32), 128, 0, st>>>(b.srcBase, t, nB, fr);
        FR_LAUNCH();
        g_launches++;
    }
    const int64_t slotBytes = (k4::FR_HIST + std::max(h.maxCap, 0) + 15) & ~int64_t(15);
    uint8_t* scratch = sizeOnly ? nullptr : P.get<uint8_t>(h.slots * slotBytes);
    int32_t* ccLen = P.get<int32_t>(n);
    uint32_t* ccGot = P.get<uint32_t>(n);
    FR_TRY(P.err);
    const int64_t scratchRel = sizeOnly ? 0 : (int64_t)((uintptr_t)scratch - (uintptr_t)b.dstBase);
    k4::frame_layout_kernel<<<grid_of(n), 128, 0, st>>>(fr, n, t, sizeOnly ? nullptr : b.dstOff,
                                                       sizeOnly ? nullptr : b.dstCap, scratchRel, slotBytes, ccLen);
    FR_LAUNCH();
    g_launches++;
    if (!sizeOnly && nB > 0) {
        const int nb = (int)nB;
        // stored blocks first: they are history for the linked blocks after them
        FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, t.cpySrc, t.cpyLen, b.dstBase, t.fin, nullptr, nullptr, nb}, st));
        FR_TRY(launch_op(OP_XXH32, Batch{b.srcBase, t.srcOff, t.ckLen, nullptr, nullptr, nullptr, (int32_t*)t.got, nb}, st));
        FR_TRY(launch_op(OP_DECODE, Batch{b.srcBase, t.srcOff, t.ilen, b.dstBase, t.dst, t.cap, t.res, nb}, st));
        if (h.maxSteps > 0) {
            k4::FrameStep s;
            s.srcOff = P.get<int64_t>(n); s.dstOff = P.get<int64_t>(n); s.hSrc = P.get<int64_t>(n); s.hDst = P.get<int64_t>(n);
            s.srcLen = P.get<int32_t>(n); s.cap = P.get<int32_t>(n); s.prefix = P.get<int32_t>(n); s.res = P.get<int32_t>(n);
            s.hLen = P.get<int32_t>(n);
            FR_TRY(P.err);
            for (int k = 0; k < h.maxSteps; k++) {
                k4::frame_step_prepare_kernel<<<grid_of(n), 128, 0, st>>>(k, fr, n, t, s, b.dstOff);
                FR_LAUNCH();
                g_launches++;
                FR_TRY(launch_op(OP_COPY, Batch{b.dstBase, s.hSrc, s.hLen, b.dstBase, s.hDst, nullptr, nullptr, n}, st));
                Batch cb{b.srcBase, s.srcOff, s.srcLen, b.dstBase, s.dstOff, s.cap, s.res, n};
                cb.prefixLen = s.prefix;
                FR_TRY(launch_op(OP_CHAIN, cb, st));
                k4::frame_step_commit_kernel<<<grid_of(n), 128, 0, st>>>(k, fr, n, t, s);
                FR_LAUNCH();
                g_launches++;
                FR_TRY(launch_op(OP_COPY, Batch{b.dstBase, s.hSrc, s.hLen, b.dstBase, s.hDst, nullptr, nullptr, n}, st));
            }
        }
        k4::frame_verdict_kernel<<<grid_of(nB), 128, 0, st>>>(fr, t, nB);
        FR_LAUNCH();
        g_launches++;
        FR_TRY(launch_op(OP_COPY, Batch{b.dstBase, t.cpySrc, t.cpyLen, b.dstBase, t.fin, nullptr, nullptr, nb}, st));
    }
    if (!sizeOnly)
        FR_TRY(launch_op(OP_XXH32, Batch{b.dstBase, b.dstOff, ccLen, nullptr, nullptr, nullptr, (int32_t*)ccGot, n}, st));
    k4::frame_decode_finish_kernel<<<grid_of(n), 128, 0, st>>>(fr, n, sizeOnly ? nullptr : b.dstCap,
                                                              sizeOnly ? nullptr : ccGot, ccLen, b.outLen);
    FR_LAUNCH();
    g_launches++;
    return cudaSuccess;
}

// Encode b.n frames in device memory on `st` (level < 3): plan, scan, one host synchronisation for the block and
// step counts, then everything else enqueued.  Independent frames: the blocks of all frames in launches of at most
// FRAME_SCRATCH bytes of encoder output; linked frames: one launch per step over chunks of frames.
cudaError_t frame_encode_dev(const Batch& b, int32_t bs, int flags, uint64_t header, cudaStream_t st) {
    int dev = 0;
    cudaGetDevice(&dev);
    const Dev* D = dev_state(dev);
    if (!D || D->err != cudaSuccess) return D ? D->err : cudaErrorInvalidDevice;
    const int n = (int)b.n;
    const bool bc = flags & K4LZ4_FRAME_BLOCK_CHECKSUM, cc = flags & K4LZ4_FRAME_CONTENT_CHECKSUM;
    FramePool P(D->pool, st);
    k4::FrameRec* fr = P.get<k4::FrameRec>(n);
    k4::FrameTotals* tot = P.get<k4::FrameTotals>(1);
    FR_TRY(P.err);
    FR_TRY(cudaMemsetAsync(tot, 0, sizeof(k4::FrameTotals), st));
    k4::FrameTable t{};
    k4::frame_enc_plan_kernel<<<grid_of(n), 128, 0, st>>>(0, b.srcOff, b.srcLen, n, bs, fr, t, tot);
    FR_LAUNCH();
    k4::frame_scan_kernel<<<1, 1024, 0, st>>>(fr, n, tot, 0);
    FR_LAUNCH();
    g_launches += 2;
    k4::FrameTotals h{};
    FR_TRY(cudaMemcpyAsync(&h, tot, sizeof(h), cudaMemcpyDeviceToHost, st));
    FR_TRY(cudaStreamSynchronize(st));                 // the one wait: the table's size and the number of steps
    const int64_t nB = h.blocks;
    t.srcOff = P.get<int64_t>(nB);
    t.len = P.get<int32_t>(nB);
    uint32_t* csum = P.get<uint32_t>(n);
    FR_TRY(P.err);
    k4::frame_enc_plan_kernel<<<grid_of(n), 128, 0, st>>>(1, b.srcOff, b.srcLen, n, bs, fr, t, tot);
    FR_LAUNCH();
    g_launches++;
    if (cc) FR_TRY(launch_op(OP_XXH32, Batch{b.srcBase, b.srcOff, b.srcLen, nullptr, nullptr, nullptr, (int32_t*)csum, n}, st));
    const int32_t bound = k4::max_output_size(bs);
    const bool linked = !(flags & K4LZ4_FRAME_INDEPENDENT);
    const int64_t per = std::max<int64_t>(FRAME_SCRATCH / bound, 1);
    const int64_t E = std::max<int64_t>(std::min<int64_t>(per, linked ? n : nB), 1);
    if (nB > 0) {
        uint8_t* scratch = P.get<uint8_t>(E * bound);
        int64_t* eDst = P.get<int64_t>(E);
        int32_t* eCap = P.get<int32_t>(E);
        k4::FrameEnc e;
        e.cSrc = P.get<int64_t>(E); e.cDst = P.get<int64_t>(E); e.rSrc = P.get<int64_t>(E); e.ckOff = P.get<int64_t>(E);
        e.cLen = P.get<int32_t>(E); e.rLen = P.get<int32_t>(E); e.ckLen = P.get<int32_t>(E); e.ckSum = P.get<uint32_t>(E);
        e.res = P.get<int32_t>(E);
        FR_TRY(P.err);
        k4::frame_slots_kernel<<<grid_of(E), 128, 0, st>>>(eDst, eCap, (int)E, bound, bound);
        FR_LAUNCH();
        g_launches++;
        // the bodies into place, then the block checksums over them
        auto place = [&](int k, int64_t b0, int64_t b1, int f0, int f1, int64_t m) -> cudaError_t {
            k4::frame_enc_place_kernel<<<grid_of(f1 - f0), 128, 0, st>>>(k, b0, b1, f0, f1, fr, t, e, b.dstBase, b.dstOff,
                                                                         b.dstCap, bound, bc ? 1 : 0);
            FR_LAUNCH();
            g_launches++;
            const int mm = (int)m;
            FR_TRY(launch_op(OP_COPY, Batch{scratch, e.cSrc, e.cLen, b.dstBase, e.cDst, nullptr, nullptr, mm}, st));
            FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, e.rSrc, e.rLen, b.dstBase, e.cDst, nullptr, nullptr, mm}, st));
            if (bc) {
                FR_TRY(launch_op(OP_XXH32, Batch{b.dstBase, e.ckOff, e.ckLen, nullptr, nullptr, nullptr, (int32_t*)e.ckSum, mm}, st));
                k4::frame_put_sum_kernel<<<grid_of(m), 128, 0, st>>>(b.dstBase, e, mm);
                FR_LAUNCH();
                g_launches++;
            }
            return cudaSuccess;
        };
        if (!linked) {
            for (int64_t b0 = 0; b0 < nB; b0 += E) {
                const int64_t m = std::min<int64_t>(E, nB - b0);
                Batch kb{b.srcBase, t.srcOff + b0, t.len + b0, scratch, eDst, eCap, e.res, m, b.level, b.x32};
                FR_TRY(launch_op(OP_ENCODE, kb, st));
                FR_TRY(place(-1, b0, b0 + m, 0, n, m));
            }
        } else {
            uint8_t* state = P.get<uint8_t>(E * K4LZ4_CHAIN_STATE_BYTES);
            int64_t* stOff = P.get<int64_t>(E);
            int64_t* so = P.get<int64_t>(E);
            int32_t* sl = P.get<int32_t>(E);
            int32_t* pre = P.get<int32_t>(E);
            FR_TRY(P.err);
            k4::frame_slots_kernel<<<grid_of(E), 128, 0, st>>>(stOff, nullptr, (int)E, K4LZ4_CHAIN_STATE_BYTES, 0);
            FR_LAUNCH();
            g_launches++;
            for (int f0 = 0; f0 < n; f0 += (int)E) {
                const int m = (int)std::min<int64_t>(E, n - f0);
                FR_TRY(cudaMemsetAsync(state, 0, (size_t)m * K4LZ4_CHAIN_STATE_BYTES, st));
                for (int k = 0; k < h.maxSteps; k++) {
                    k4::frame_enc_step_kernel<<<grid_of(m), 128, 0, st>>>(k, f0, f0 + m, fr, t, so, sl, pre, bs);
                    FR_LAUNCH();
                    g_launches++;
                    Batch kb{b.srcBase, so, sl, scratch, eDst, eCap, e.res, m, b.level, b.x32};
                    kb.prefixLen = pre; kb.stateBase = state; kb.stateOff = stOff;
                    FR_TRY(launch_op(OP_ENCCHAIN, kb, st));
                    FR_TRY(place(k, 0, 0, f0, f0 + m, m));
                }
            }
        }
    }
    k4::frame_enc_finish_kernel<<<grid_of(n), 128, 0, st>>>(fr, n, b.dstBase, b.dstOff, b.dstCap, header, cc ? 1 : 0,
                                                           csum, b.outLen);
    FR_LAUNCH();
    g_launches++;
    return cudaSuccess;
}

enum FrameOp { FO_ENCODE, FO_DECODE, FO_SIZE };

cudaError_t frame_dev(FrameOp fo, const Batch& b, int32_t bs, int flags, uint64_t header, cudaStream_t st) {
    if (fo == FO_ENCODE && b.level >= 3) {
        k4::frame_fill_kernel<<<grid_of(b.n), 128, 0, st>>>(b.outLen, (int)b.n, K4LZ4_R_DELEGATE);
        g_launches++;
        return cudaGetLastError();
    }
    return fo == FO_ENCODE ? frame_encode_dev(b, bs, flags, header, st) : frame_decode_dev(b, fo == FO_SIZE, st);
}

// Host memory, one GPU, synchronous: chunks of whole frames (a frame is never split: its linked blocks and its
// content checksum need all of it).  Per chunk, the offsets, lengths and packed frames go up in one copy; the
// device path runs on them; the results come down, the produced bytes are gathered on the device and come down in
// one copy, and exactly outLen[i] > 0 bytes of each frame go to the caller.  The device region of a frame is
// min(dstCap, frame bound) when encoding (a frame never needs more) and dstCap when decoding.
int frame_host(FrameOp fo, const Batch& b, int32_t bs, int flags, uint64_t header, int dev) {
    DeviceGuard guard(dev);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", dev);
    if (fo == FO_ENCODE && b.level >= 3) {
        for (int64_t i = 0; i < b.n; i++) b.outLen[i] = K4LZ4_R_DELEGATE;
        return K4LZ4_OK;
    }
    auto a16 = [](int64_t x) { return (x + 15) & ~int64_t(15); };
    auto room = [&](int64_t i) -> int64_t {
        if (fo == FO_SIZE) return 0;
        const int64_t c = std::max<int32_t>(b.dstCap[i], 0);
        return fo == FO_ENCODE ? std::min<int64_t>(c, frame_bound_of(src_size(b, i), bs, flags)) : c;
    };
    std::vector<uint8_t> h;
    std::vector<int64_t> pack;
    DevMem d;
    for (int64_t i = 0, j; i < b.n; i = j) {
        int64_t bytes = 0;
        for (j = i; j < b.n; j++) {
            const int64_t add = a16(src_size(b, j)) + 2 * a16(room(j)) + 64;
            if (j > i && bytes + add > STAGE_BYTES) break;
            bytes += add;
        }
        const int64_t nb = j - i;
        // up: srcOff dstOff packOff (int64) | srcLen dstCap outLen (int32) | frames; then the regions and the pack
        const int64_t srcAt = a16(nb * (3 * 8 + 3 * 4));
        int64_t sTot = 0, dTot = 0;
        for (int64_t k = 0; k < nb; k++) { sTot += a16(src_size(b, i + k)); dTot += a16(room(i + k)); }
        const int64_t dstAt = a16(srcAt + sTot), packAt = a16(dstAt + dTot), total = packAt + dTot;
        if (h.size() < (size_t)srcAt + (size_t)sTot + 16) h.resize((size_t)srcAt + (size_t)sTot + 16);
        int64_t* so = (int64_t*)h.data(); int64_t* doff = so + nb; int64_t* po = doff + nb;
        int32_t* sl = (int32_t*)(po + nb); int32_t* dc = sl + nb; int32_t* res = dc + nb;
        for (int64_t k = 0, sp = 0, dp = 0; k < nb; k++) {
            const int64_t x = i + k, s = src_size(b, x), r = room(x);
            so[k] = sp; doff[k] = dp; sl[k] = (int32_t)s; dc[k] = (int32_t)r; po[k] = 0;
            sp += a16(s); dp += a16(r);
        }
        parallel_for_blocks(0, nb, sTot, [&](int64_t lo, int64_t hi) {
            for (int64_t k = lo; k < hi; k++)
                if (sl[k] > 0) memcpy(h.data() + srcAt + so[k], b.srcBase + b.srcOff[i + k], (size_t)sl[k]);
        });
        CU_TRY(d.ensure((size_t)total + 16));
        uint8_t* Dp = (uint8_t*)d.p;
        CU_TRY(cudaMemcpy(Dp, h.data(), (size_t)(srcAt + sTot), cudaMemcpyHostToDevice));
        Batch kb = b;
        kb.srcBase = Dp + srcAt; kb.srcOff = (int64_t*)Dp; kb.srcLen = (int32_t*)(Dp + ((uint8_t*)sl - h.data()));
        kb.dstBase = Dp + dstAt; kb.dstOff = kb.srcOff + nb; kb.dstCap = fo == FO_SIZE ? nullptr : kb.srcLen + nb;
        kb.outLen = (int32_t*)(Dp + ((uint8_t*)res - h.data())); kb.n = nb;
        const cudaError_t e = frame_dev(fo, kb, bs, flags, header, nullptr);
        if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "frame call: %s", cudaGetErrorString(e)); }
        CU_TRY(cudaMemcpy(b.outLen + i, kb.outLen, (size_t)nb * 4, cudaMemcpyDeviceToHost));
        if (fo == FO_SIZE) continue;
        pack.resize((size_t)nb);
        int64_t got = 0;
        for (int64_t k = 0; k < nb; k++) { pack[(size_t)k] = got; if (b.outLen[i + k] > 0) got = a16(got + b.outLen[i + k]); }
        if (got == 0) continue;
        CU_TRY(cudaMemcpy(Dp + ((uint8_t*)po - h.data()), pack.data(), (size_t)nb * 8, cudaMemcpyHostToDevice));
        CU_TRY(launch_op(OP_COPY, Batch{kb.dstBase, kb.dstOff, kb.outLen, Dp + packAt, (int64_t*)(Dp + ((uint8_t*)po - h.data())),
                                        nullptr, nullptr, nb}, nullptr));
        if (h.size() < (size_t)got + 16) { h.resize((size_t)got + 16); }
        CU_TRY(cudaMemcpy(h.data(), Dp + packAt, (size_t)got, cudaMemcpyDeviceToHost));
        parallel_for_blocks(0, nb, got, [&](int64_t lo, int64_t hi) {
            for (int64_t k = lo; k < hi; k++) {
                const int32_t r = b.outLen[i + k];
                if (r > 0) memcpy(b.dstBase + b.dstOff[i + k], h.data() + pack[(size_t)k], (size_t)r);
            }
        });
    }
    return K4LZ4_OK;
}

// Every frame export: its own arguments, then the batch's (check()), then host or device.
int frame_run(FrameOp fo, const Batch& b, int32_t blockSize, int flags, int memKind, void* stream, int device) {
    int32_t bs = 0;
    if (fo == FO_ENCODE) {
        bs = frame_block_size(blockSize);
        if (!bs) return fail(K4LZ4_E_ARG, "bad frame block size %d (1 .. 4 MiB)", blockSize);
        if (flags & ~FRAME_FLAGS) return fail(K4LZ4_E_ARG, "unknown frame flags 0x%x", flags);
    }
    const int rc = check(fo == FO_ENCODE ? OP_ENCODE : fo == FO_SIZE ? OP_USIZE : OP_DECODE, b, memKind, device);
    if (rc != K4LZ4_OK || b.n == 0) return rc;
    const uint64_t header = fo == FO_ENCODE ? frame_header(blockSize, flags) : 0;
    if (memKind == K4LZ4_MEM_HOST) return frame_host(fo, b, bs, flags, header, device < 0 ? 0 : device);
    DeviceGuard g(device);
    if (!g.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", device);
    const cudaError_t e = frame_dev(fo, b, bs, flags, header, (cudaStream_t)stream);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "frame call: %s", cudaGetErrorString(e)); }
    return K4LZ4_OK;
}

// ---- resident groups: what chain, frame writer and frame reader groups share ---------------------------------

// S streams on one device, each with a ring in the chain-group layout (chain_group.cuh) and its header; the kind's
// own per-stream arrays; the staging buffers of host-memory calls, which grow and never shrink.  Every device array
// comes from alloc() and is freed with the group.
struct GroupCore {
    int32_t nStreams = 0;
    int device = 0;
    int64_t ring = 0, slot = 0;       // bytes per ring; the room a block or an injection may need at the write position
    uint8_t* rings = nullptr;
    k4::ChainGroupHdr* hdr = nullptr;
    Buf dStage, dDown, hUp{true}, hDown{true};
    std::vector<void*> owned;
    cudaError_t allocErr = cudaSuccess;   // the first failure of alloc(), after which it allocates nothing

    // nStreams * per bytes on the current device, zeroed when `zero`
    template <class T> T* alloc(size_t per, bool zero) {
        void* p = nullptr;
        if (allocErr == cudaSuccess) allocErr = cudaMalloc(&p, (size_t)nStreams * per);
        if (allocErr != cudaSuccess) return nullptr;
        owned.push_back(p);
        if (zero) allocErr = cudaMemset(p, 0, (size_t)nStreams * per);
        return (T*)p;
    }
    ~GroupCore() {
        for (void* p : owned) cudaFree(p);
        for (Buf* b : {&dStage, &dDown, &hUp, &hDown}) b->release();
    }
};

}  // namespace

// S streams of one direction (k4lz4.h, chain_group.cuh): encoder groups also keep each stream's state record.
struct k4lz4_chain_group : GroupCore {
    int kind = 0;
    int32_t blockSize = 0;
    uint8_t* states = nullptr;        // encoder groups: K4LZ4_CHAIN_STATE_BYTES per stream
};

namespace {

// The chain-group ring layout: 128 KiB of history in front of a slot of max(x, 64 KiB) bytes.
void chain_layout(GroupCore& g, int64_t x) {
    g.slot = std::max<int64_t>(x, k4::CG_WINDOW);
    g.ring = 2 * k4::CG_WINDOW + g.slot;
}

// Every group's create after the kind's own argument check: the device (the current one when negative), then on
// it a new group of nStreams streams that `setup` sizes (ring, slot) and gives its kind's arrays through alloc(),
// and a ring and a zeroed header per stream.  On failure everything is freed again and *out stays null.
template <class G, class Setup>
int group_create(int32_t nStreams, int device, const char* what, G** out, Setup setup) {
    const int rc = check_device(device, 1);
    if (rc != K4LZ4_OK) return rc;
    if (device < 0 && cudaGetDevice(&device) != cudaSuccess) return fail(K4LZ4_E_CUDA, "cudaGetDevice failed");
    DeviceGuard guard(device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", device);
    G* g = new G;
    g->nStreams = nStreams; g->device = device;
    setup(*g);
    g->rings = g->template alloc<uint8_t>((size_t)g->ring, false);
    g->hdr = g->template alloc<k4::ChainGroupHdr>(sizeof(k4::ChainGroupHdr), true);
    cudaError_t e = g->allocErr;
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        const long long ring = g->ring;
        delete g;
        return fail(e == cudaErrorMemoryAllocation ? K4LZ4_E_NOMEM : K4LZ4_E_CUDA, "%s of %d streams x %lld-byte rings: %s",
                    what, nStreams, ring, cudaGetErrorString(e));
    }
    *out = g;
    return K4LZ4_OK;
}

// Every group's destroy, after the device has finished its work.
template <class G>
int32_t group_destroy(G* g) {
    if (!g) return K4LZ4_OK;
    DeviceGuard guard(g->device);
    cudaDeviceSynchronize();
    delete g;
    return K4LZ4_OK;
}

// The work of a reset or an end on the group's device: with host memory the stream list goes up through the staging
// buffers first (dStage has room for an int32 result per stream behind it), and the call waits for the device after
// `enqueue(ds, st)` has launched the kind's kernels over the list `ds`.
template <class Enqueue>
int group_streams_run(GroupCore* g, const int32_t* streams, int32_t n, int memKind, void* stream, Enqueue enqueue) {
    DeviceGuard guard(g->device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", g->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int32_t* ds = streams;
    if (memKind == K4LZ4_MEM_HOST) {
        CU_TRY(g->hUp.ensure((size_t)n * 4));
        CU_TRY(g->dStage.ensure((size_t)n * 8));
        memcpy(g->hUp.p, streams, (size_t)n * 4);
        CU_TRY(cudaMemcpyAsync(g->dStage.p, g->hUp.p, (size_t)n * 4, cudaMemcpyHostToDevice, st));
        ds = (const int32_t*)g->dStage.p;
    }
    CU_TRY(enqueue(ds, st));
    if (memKind == K4LZ4_MEM_HOST) CU_TRY(cudaStreamSynchronize(st));
    return K4LZ4_OK;
}

// Every group's reset, in k4lz4.h's order: the group, memKind, the count, the pointer, with host memory the stream
// range (a stream listed twice is reset twice, and no device is needed to get here), then n == 0 is done.
template <class Enqueue>
int group_reset(GroupCore* g, const int32_t* streams, int32_t n, int32_t memKind, void* stream, Enqueue enqueue) {
    if (!g) return fail(K4LZ4_E_ARG, "null group");
    if (memKind != K4LZ4_MEM_HOST && memKind != K4LZ4_MEM_DEVICE) return fail(K4LZ4_E_ARG, "unknown memKind %d", memKind);
    if (n < 0) return fail(K4LZ4_E_ARG, "bad stream count %d", n);
    if (n > 0 && !streams) return fail(K4LZ4_E_ARG, "null pointer argument");
    if (memKind == K4LZ4_MEM_HOST)
        for (int32_t i = 0; i < n; i++)
            if (streams[i] < 0 || streams[i] >= g->nStreams) return fail(K4LZ4_E_ARG, "stream %d out of range", streams[i]);
    if (n == 0) return K4LZ4_OK;
    return group_streams_run(g, streams, n, memKind, stream, enqueue);
}

// Every group's step-call check, in k4lz4.h's order: the group, memKind, the count, the pointers (`pointers`: the
// call's required ones besides `streams` are set), with host memory each entry's stream (in range, listed once) and
// then `entry(i)`, the level (b.level is 0 but in a chain encoder's calls), then the machine.  A group exists only on
// a device, so no check here meets "no device" before an argument error.
template <class Entry>
int check_step(const GroupCore* g, const Batch& b, const int32_t* streams, bool pointers, int memKind, Entry entry) {
    if (!g) return fail(K4LZ4_E_ARG, "null group");
    if (memKind != K4LZ4_MEM_HOST && memKind != K4LZ4_MEM_DEVICE) return fail(K4LZ4_E_ARG, "unknown memKind %d", memKind);
    if (b.n < 0 || b.n > INT32_MAX) return fail(K4LZ4_E_ARG, "bad stream count %lld", (long long)b.n);
    if (b.n > 0 && (!streams || !pointers)) return fail(K4LZ4_E_ARG, "null pointer argument");
    if (memKind == K4LZ4_MEM_HOST && b.n > 0) {
        std::vector<uint8_t> seen((size_t)g->nStreams, 0);
        for (int64_t i = 0; i < b.n; i++) {
            const int32_t s = streams[i];
            if (s < 0 || s >= g->nStreams) return fail(K4LZ4_E_ARG, "stream %d out of range at entry %lld", s, (long long)i);
            if (seen[(size_t)s]++) return fail(K4LZ4_E_ARG, "stream %d listed twice", s);
            const int rc = entry(i);
            if (rc != K4LZ4_OK) return rc;
        }
    }
    if (b.level < 0 || b.level > 0xFF) return fail(K4LZ4_E_ARG, "bad level %d", b.level);
    return check_device(g->device, b.n);
}

const auto no_entry_check = [](int64_t) { return K4LZ4_OK; };

// One host-memory step's upload, in one copy into dStage: the table srcOff dstOff (int64) | stream len cap aux
// (int32) of the m entries row(k) describes, then their `send` source bytes packed 16-aligned.  Behind it in dStage:
// resInts * m int32 results, m compact offsets (stage_down), `extra` bytes for the caller, and the entries'
// destination slots, `room` bytes each at dstOff (16-aligned).
struct UpRow { const uint8_t* src; int64_t send, room; int32_t stream, len, cap, aux; };
struct StageUp {                      // device pointers into dStage
    const uint8_t* src; const int64_t* srcOff; const int64_t* dstOff;
    const int32_t* stream; const int32_t* len; const int32_t* cap; const int32_t* aux;
    int32_t* res; int64_t* coff; uint8_t* extra; uint8_t* dst;
};

template <class Row>
int stage_up(GroupCore* g, int64_t m, int64_t resInts, int64_t extra, Row row, StageUp& up, cudaStream_t st) {
    auto a16 = [](int64_t x) { return (x + 15) & ~int64_t(15); };
    std::vector<UpRow> r((size_t)m);
    int64_t srcBytes = 0, dstBytes = 0;
    for (int64_t k = 0; k < m; k++) {
        r[(size_t)k] = row(k);
        srcBytes += a16(r[(size_t)k].send); dstBytes += a16(r[(size_t)k].room);
    }
    const int64_t sendAt = a16(m * (8 * 2 + 4 * 4)), upBytes = sendAt + srcBytes;
    const int64_t resAt = a16(upBytes), coffAt = resAt + a16(m * 4 * resInts), extraAt = coffAt + a16(m * 8);
    const int64_t dstAt = extraAt + a16(extra);
    CU_TRY(g->hUp.ensure((size_t)std::max(upBytes, m * 8) + 16));   // stage_down sends the compact offsets through it
    CU_TRY(g->dStage.ensure((size_t)(dstAt + dstBytes) + 16));
    uint8_t* H = (uint8_t*)g->hUp.p;
    int64_t* hso = (int64_t*)H; int64_t* hdo = hso + m;
    int32_t* hs = (int32_t*)(hdo + m); int32_t* hl = hs + m; int32_t* hc = hl + m; int32_t* ha = hc + m;
    for (int64_t k = 0, sp = 0, dp = 0; k < m; k++) {
        const UpRow& x = r[(size_t)k];
        hs[k] = x.stream; hl[k] = x.len; hc[k] = x.cap; ha[k] = x.aux;
        hso[k] = sp; hdo[k] = dp;
        sp += a16(x.send); dp += a16(x.room);
    }
    parallel_for_blocks(0, m, srcBytes, [&](int64_t lo, int64_t hi) {
        for (int64_t k = lo; k < hi; k++)
            if (r[(size_t)k].send > 0) memcpy(H + sendAt + hso[k], r[(size_t)k].src, (size_t)r[(size_t)k].send);
    });
    uint8_t* D = (uint8_t*)g->dStage.p;
    CU_TRY(cudaMemcpyAsync(D, H, (size_t)upBytes, cudaMemcpyHostToDevice, st));
    const int32_t* ds = (const int32_t*)(D + m * 16);
    up = StageUp{D + sendAt, (const int64_t*)D, (const int64_t*)D + m, ds, ds + m, ds + 2 * m, ds + 3 * m,
                 (int32_t*)(D + resAt), (int64_t*)(D + coffAt), D + extraAt, D + dstAt};
    return K4LZ4_OK;
}

// One host-memory step's download, behind the device work on `st`: the resInts * m results come back into hRes (the
// first m are the entries' lengths) and, where any is positive, entry k's hRes[k] bytes at from + fromOff[k] on the
// device are gathered into dDown and come down in one copy, then go to to(k), exactly hRes[k] > 0 bytes each.
// `after` (may be empty) is enqueued behind the gather, or alone when nothing was produced, and the call waits for it.
template <class To>
int stage_down(GroupCore* g, const StageUp& up, int64_t m, int32_t* hRes, int64_t resInts, const uint8_t* from,
               const int64_t* fromOff, const std::function<cudaError_t()>& after, To to, cudaStream_t st) {
    auto a16 = [](int64_t x) { return (x + 15) & ~int64_t(15); };
    CU_TRY(cudaMemcpyAsync(hRes, up.res, (size_t)(m * 4 * resInts), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    std::vector<int64_t> co((size_t)m);
    int64_t total = 0;
    for (int64_t k = 0; k < m; k++) { co[(size_t)k] = total; if (hRes[k] > 0) total = a16(total + hRes[k]); }
    if (total == 0) {
        if (after) { CU_TRY(after()); CU_TRY(cudaStreamSynchronize(st)); }
        return K4LZ4_OK;
    }
    CU_TRY(g->dDown.ensure((size_t)total + 16));
    CU_TRY(g->hDown.ensure((size_t)total + 16));
    memcpy(g->hUp.p, co.data(), (size_t)m * 8);     // the upload buffer is free again
    CU_TRY(cudaMemcpyAsync(up.coff, g->hUp.p, (size_t)m * 8, cudaMemcpyHostToDevice, st));
    CU_TRY(launch_op(OP_COPY, Batch{from, fromOff, up.res, (uint8_t*)g->dDown.p, up.coff, nullptr, nullptr, m}, st));
    if (after) CU_TRY(after());
    CU_TRY(cudaMemcpyAsync(g->hDown.p, g->dDown.p, (size_t)total, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    const uint8_t* stage = (const uint8_t*)g->hDown.p;
    parallel_for_blocks(0, m, total, [&](int64_t lo, int64_t hi) {
        for (int64_t k = lo; k < hi; k++)
            if (hRes[k] > 0) memcpy(to(k), stage + co[(size_t)k], (size_t)hRes[k]);
    });
    return K4LZ4_OK;
}

// ---- chain groups -----------------------------------------------------------------------------------

// Table of n blocks (chain_group.cuh) carved from `p`: 40 bytes per block.
k4::ChainGroupTable carve_table(uint8_t* p, int64_t n) {
    k4::ChainGroupTable t;
    t.ringOff = (int64_t*)p; t.stateOff = t.ringOff + n; t.copyOff = t.stateOff + n;
    t.len = (int32_t*)(t.copyOff + n); t.prefix = t.len + n; t.stream = t.prefix + n; t.copyLen = t.stream + n;
    return t;
}
constexpr int64_t TABLE_BYTES = 3 * 8 + 4 * 4;

// The first half of a step on the device, current device = the group's: prepare, the copy into the rings, the
// codec and, when `gather`, the copy of decoded bytes to the destination.  `b` holds device pointers; for
// encoding its destination is where the codec writes.
cudaError_t group_codec(k4lz4_chain_group* g, int cg, const Batch& b, const int32_t* streams, const k4::ChainGroupTable& t,
                        bool gather, cudaStream_t st) {
    const int n = (int)b.n, thr = 128, grid = (n + thr - 1) / thr;
    k4::chain_group_prepare_kernel<<<grid, thr, 0, st>>>(cg, streams, cg == k4::CG_DECODE ? b.dstCap : b.srcLen,
                                                         b.srcOff, n, g->nStreams, g->blockSize, g->ring, g->hdr, t);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && cg != k4::CG_DECODE)
        e = launch_op(OP_COPY, Batch{b.srcBase, t.copyOff, t.copyLen, g->rings, t.ringOff, nullptr, nullptr, n}, st);
    if (e == cudaSuccess && cg == k4::CG_ENCODE) {
        Batch kb{g->rings, t.ringOff, t.len, b.dstBase, b.dstOff, b.dstCap, b.outLen, n, b.level, b.x32};
        kb.prefixLen = t.prefix; kb.stateBase = g->states; kb.stateOff = t.stateOff;
        e = launch_op(OP_ENCCHAIN, kb, st);
    }
    if (e == cudaSuccess && cg == k4::CG_DECODE) {
        Batch kb{b.srcBase, b.srcOff, b.srcLen, g->rings, t.ringOff, t.len, b.outLen, n};
        kb.prefixLen = t.prefix;
        e = launch_op(OP_CHAIN, kb, st);
        if (e == cudaSuccess && gather)
            e = launch_op(OP_COPY, Batch{g->rings, t.ringOff, b.outLen, b.dstBase, b.dstOff, nullptr, nullptr, n}, st);
    }
    return e;
}

// The second half, after every read of the block's slot: the commit and the slides (a slide may overwrite the
// front of a block that started below 64 KiB).
cudaError_t group_commit(const GroupCore* g, int cg, const int32_t* outLen, int64_t n64, const k4::ChainGroupTable& t,
                         cudaStream_t st) {
    const int n = (int)n64, thr = 128, grid = (n + thr - 1) / thr;
    k4::chain_group_commit_kernel<<<grid, thr, 0, st>>>(cg, outLen, n, g->ring, g->slot, g->hdr, t);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess)
        e = launch_op(OP_COPY, Batch{g->rings, t.copyOff, t.copyLen, g->rings, t.ringOff, nullptr, nullptr, n}, st);
    return e;
}

// Device memory: the table comes from the device's stream-ordered pool, so nothing here waits for the device.
int group_device(k4lz4_chain_group* g, int cg, const Batch& b, const int32_t* streams, cudaStream_t st) {
    const Dev* D = dev_state(g->device);
    if (!D || D->err != cudaSuccess) return fail(K4LZ4_E_CUDA, "device %d setup failed", g->device);
    FramePool P(D->pool, st);
    uint8_t* tab = P.get<uint8_t>(b.n * TABLE_BYTES);
    cudaError_t e = P.err;
    if (e == cudaSuccess) {
        const k4::ChainGroupTable t = carve_table(tab, b.n);
        e = group_codec(g, cg, b, streams, t, cg == k4::CG_DECODE, st);
        if (e == cudaSuccess) e = group_commit(g, cg, b.outLen, b.n, t, st);
    }
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "chain group step: %s", cudaGetErrorString(e)); }
    return K4LZ4_OK;
}

// Host memory, synchronous: stage_up (an injection sends only the bytes it keeps; an encoder's destination slot is
// where the codec writes), the codec, stage_down with the commit and the slides behind the gather.  An injection
// commits right after the codec and brings nothing down.
int group_host(k4lz4_chain_group* g, int cg, const Batch& b, const int32_t* streams, cudaStream_t st) {
    const int64_t n = b.n;
    const bool enc = cg == k4::CG_ENCODE, inj = cg == k4::CG_INJECT;
    StageUp up;
    const int rc = stage_up(g, n, 1, n * TABLE_BYTES, [&](int64_t i) {
        const int32_t L = b.srcLen[i];
        const bool fits = L > 0 && L <= g->blockSize;
        const int64_t send = L <= 0 ? 0 : inj ? std::min<int64_t>(L, k4::CG_WINDOW) : enc && !fits ? 0 : L;
        const int64_t room = enc && fits ? std::min<int64_t>(std::max<int32_t>(b.dstCap[i], 0), k4::max_output_size(L)) : 0;
        return UpRow{send > 0 ? b.srcBase + b.srcOff[i] + (L - send) : nullptr, send, room, streams[i],
                     inj ? (int32_t)send : L, inj ? 0 : b.dstCap[i], 0};
    }, up, st);
    if (rc != K4LZ4_OK) return rc;
    Batch kb = b;
    kb.srcBase = up.src; kb.srcOff = up.srcOff; kb.srcLen = up.len;
    kb.dstBase = up.dst; kb.dstOff = up.dstOff; kb.dstCap = up.cap;
    kb.outLen = up.res;
    const k4::ChainGroupTable t = carve_table(up.extra, n);
    auto commit = [&] { return group_commit(g, cg, up.res, n, t, st); };
    cudaError_t e = group_codec(g, cg, kb, up.stream, t, false, st);
    if (e == cudaSuccess && inj) e = commit();
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "chain group step: %s", cudaGetErrorString(e)); }
    if (inj) { CU_TRY(cudaStreamSynchronize(st)); return K4LZ4_OK; }
    return stage_down(g, up, n, b.outLen, 1, enc ? up.dst : g->rings, enc ? up.dstOff : t.ringOff, commit,
                      [&](int64_t i) { return b.dstBase + b.dstOff[i]; }, st);
}

int group_run(k4lz4_chain_group* g, int kind, int cg, const Batch& b, const int32_t* streams, int memKind, void* stream) {
    if (g && g->kind != kind) return fail(K4LZ4_E_ARG, "chain group of the other kind");
    const bool io = cg != k4::CG_INJECT;
    const int rc = check_step(g, b, streams, b.srcBase && b.srcOff && b.srcLen &&
                                                 (!io || (b.dstBase && b.dstOff && b.dstCap && b.outLen)),
                              memKind, no_entry_check);
    if (rc != K4LZ4_OK || b.n == 0) return rc;
    DeviceGuard guard(g->device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", g->device);
    return memKind == K4LZ4_MEM_HOST ? group_host(g, cg, b, streams, (cudaStream_t)stream)
                                     : group_device(g, cg, b, streams, (cudaStream_t)stream);
}

}  // namespace

// ---- frame writer groups ----------------------------------------------------------------------------

// S incrementally written LZ4 frames (k4lz4.h, frame_writer.cuh): each stream also keeps its FwState (partial block,
// content checksum) and, in linked frames, its chain state.
struct k4lz4_frame_writer_group : GroupCore {
    int32_t blockSize = 0, B = 0;     // the caller's block size (BD) and the encoder's (blocks)
    int flags = 0, level = 0;
    uint64_t header = 0;
    uint8_t* states = nullptr;        // linked frames: K4LZ4_CHAIN_STATE_BYTES per stream
    k4::FwState* fw = nullptr;
    bool linked() const { return !(flags & K4LZ4_FRAME_INDEPENDENT); }
    bool bc() const { return flags & K4LZ4_FRAME_BLOCK_CHECKSUM; }
    bool cc() const { return flags & K4LZ4_FRAME_CONTENT_CHECKSUM; }
};

namespace {

constexpr int64_t FW_STAGE_BYTES = 256ll << 20;   // source bytes of one host-memory sub-write

// One write (or close) of b.n entries in device memory on `st`: plan, the content checksum, one host
// synchronisation for the number of steps (a close has at most one and does not wait), the steps over chunks of at
// most FRAME_SCRATCH bytes of encoder output, then the rest of each source into its ring (or the end marks).
cudaError_t fw_device(k4lz4_frame_writer_group* g, bool closing, const Batch& b, const int32_t* streams, cudaStream_t st) {
    const Dev* D = dev_state(g->device);
    if (!D || D->err != cudaSuccess) return D ? D->err : cudaErrorInvalidDevice;
    const int n = (int)b.n;
    const bool linked = g->linked(), bc = g->bc(), cc = g->cc();
    FramePool P(D->pool, st);
    k4::FwEntry* ent = P.get<k4::FwEntry>(n);
    int32_t* mx = P.get<int32_t>(1);
    FR_TRY(P.err);
    FR_TRY(cudaMemsetAsync(mx, 0, 4, st));
    k4::frame_writer_plan_kernel<<<grid_of(n), 128, 0, st>>>(streams, b.srcOff, closing ? nullptr : b.srcLen, b.dstOff,
                                                            b.dstCap, n, g->nStreams, g->B, g->flags, g->header,
                                                            b.dstBase, g->fw, ent, b.outLen, mx);
    FR_LAUNCH();
    g_launches++;
    int32_t steps = 1;
    if (!closing) {
        if (cc) {
            k4::frame_writer_xxh_kernel<<<grid_of((int64_t)n * 4), 128, 0, st>>>(b.srcBase, ent, n, g->fw);
            FR_LAUNCH();
            g_launches++;
        }
        FR_TRY(cudaMemcpyAsync(&steps, mx, 4, cudaMemcpyDeviceToHost, st));
        FR_TRY(cudaStreamSynchronize(st));             // the one wait: the number of steps
    }
    if (steps > 0) {
        const int32_t bound = k4::max_output_size(g->B);
        const int E = (int)std::max<int64_t>(std::min<int64_t>(FRAME_SCRATCH / bound, n), 1);
        uint8_t* scratch = P.get<uint8_t>((int64_t)E * bound);
        uint8_t* tab = P.get<uint8_t>((int64_t)E * TABLE_BYTES);
        int64_t* copyDst = P.get<int64_t>(E);
        int64_t* eDst = P.get<int64_t>(E);
        int32_t* eCap = P.get<int32_t>(E);
        k4::FrameEnc e;
        e.cSrc = P.get<int64_t>(E); e.cDst = P.get<int64_t>(E); e.rSrc = P.get<int64_t>(E); e.ckOff = P.get<int64_t>(E);
        e.cLen = P.get<int32_t>(E); e.rLen = P.get<int32_t>(E); e.ckLen = P.get<int32_t>(E); e.ckSum = P.get<uint32_t>(E);
        e.res = P.get<int32_t>(E);
        FR_TRY(P.err);
        const k4::ChainGroupTable t = carve_table(tab, E);
        k4::frame_slots_kernel<<<grid_of(E), 128, 0, st>>>(eDst, eCap, E, bound, bound);
        FR_LAUNCH();
        g_launches++;
        for (int k = 0; k < steps; k++) {
            for (int e0 = 0; e0 < n; e0 += E) {
                const int m = std::min(E, n - e0);
                k4::frame_writer_step_kernel<<<grid_of(m), 128, 0, st>>>(k, e0, m, closing ? 1 : 0, ent, g->fw, g->hdr,
                                                                        g->B, g->ring, linked ? 1 : 0, t, copyDst);
                FR_LAUNCH();
                g_launches++;
                if (!closing)
                    FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, t.copyOff, t.copyLen, g->rings, copyDst, nullptr, nullptr, m}, st));
                Batch kb{g->rings, t.ringOff, t.len, scratch, eDst, eCap, e.res, m, g->level, b.x32};
                if (linked) { kb.prefixLen = t.prefix; kb.stateBase = g->states; kb.stateOff = t.stateOff; }
                FR_TRY(launch_op(linked ? OP_ENCCHAIN : OP_ENCODE, kb, st));
                k4::frame_writer_place_kernel<<<grid_of(m), 128, 0, st>>>(e0, m, ent, g->fw, t, e, b.dstBase, bound,
                                                                         bc ? 1 : 0);
                FR_LAUNCH();
                g_launches++;
                FR_TRY(launch_op(OP_COPY, Batch{scratch, e.cSrc, e.cLen, b.dstBase, e.cDst, nullptr, nullptr, m}, st));
                FR_TRY(launch_op(OP_COPY, Batch{g->rings, e.rSrc, e.rLen, b.dstBase, e.cDst, nullptr, nullptr, m}, st));
                if (bc) {
                    FR_TRY(launch_op(OP_XXH32, Batch{b.dstBase, e.ckOff, e.ckLen, nullptr, nullptr, nullptr, (int32_t*)e.ckSum, m}, st));
                    k4::frame_put_sum_kernel<<<grid_of(m), 128, 0, st>>>(b.dstBase, e, m);
                    FR_LAUNCH();
                    g_launches++;
                }
                if (linked) FR_TRY(group_commit(g, k4::CG_ENCODE, e.res, m, t, st));   // pos += B and the slide
            }
        }
    }
    int64_t* rOff = closing ? nullptr : P.get<int64_t>(n);
    int64_t* rDst = closing ? nullptr : P.get<int64_t>(n);
    int32_t* rLen = closing ? nullptr : P.get<int32_t>(n);
    int32_t* reset = closing ? P.get<int32_t>(n) : nullptr;
    FR_TRY(P.err);
    k4::frame_writer_finish_kernel<<<grid_of(n), 128, 0, st>>>(closing ? 1 : 0, ent, n, g->fw, g->hdr, g->ring,
                                                              linked ? 1 : 0, cc ? 1 : 0, b.dstBase, rOff, rDst, rLen,
                                                              reset, b.outLen);
    FR_LAUNCH();
    g_launches++;
    if (!closing) {
        FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, rOff, rLen, g->rings, rDst, nullptr, nullptr, n}, st));
    } else {
        k4::chain_group_reset_kernel<<<n, 256, 0, st>>>(reset, n, g->nStreams, g->hdr, linked ? g->states : nullptr);
        FR_LAUNCH();
        g_launches++;
    }
    return cudaSuccess;
}

// Host memory, synchronous.  One sub-write (or the close) of entries idx[k] with piece[k] source bytes starting
// at srcAt[k] of theirs: stage_up with a destination slot of the piece's bound per entry, the device path, and
// stage_down to the caller at dstOff + wrote[k].
int fw_host_part(k4lz4_frame_writer_group* g, bool closing, const Batch& b, const int32_t* streams,
                 const std::vector<int64_t>& idx, const std::vector<int64_t>& srcAt, const std::vector<int64_t>& piece,
                 std::vector<int64_t>& wrote, std::vector<int32_t>& res, cudaStream_t st) {
    const int64_t m = (int64_t)idx.size();
    const int64_t cb = k4::fw_close_bound(g->B, g->bc(), g->cc());
    StageUp up;
    const int rc = stage_up(g, m, 1, 0, [&](int64_t k) {
        const int64_t room = closing ? std::min<int64_t>(std::max<int32_t>(b.dstCap[idx[k]], 0), cb)
                                     : k4::fw_write_bound(piece[k], g->B, g->bc());
        return UpRow{piece[k] > 0 ? b.srcBase + b.srcOff[idx[k]] + srcAt[k] : nullptr, piece[k], room,
                     streams[idx[k]], (int32_t)piece[k], (int32_t)room, 0};
    }, up, st);
    if (rc != K4LZ4_OK) return rc;
    const Batch kb{up.src, up.srcOff, up.len, up.dst, up.dstOff, up.cap, up.res, m, g->level, b.x32};
    const cudaError_t e = fw_device(g, closing, kb, up.stream, st);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "frame writer step: %s", cudaGetErrorString(e)); }
    res.resize((size_t)m);
    const int rd = stage_down(g, up, m, res.data(), 1, up.dst, up.dstOff, nullptr,
                              [&](int64_t k) { return b.dstBase + b.dstOff[idx[k]] + wrote[(size_t)k]; }, st);
    if (rd != K4LZ4_OK) return rd;
    for (int64_t k = 0; k < m; k++) if (res[(size_t)k] > 0) wrote[(size_t)k] += res[(size_t)k];
    return K4LZ4_OK;
}

// Host memory: entries whose capacity is below their bound get -1 and are left out; the others are written in
// sub-writes of at most FW_STAGE_BYTES source bytes, in entry order (cutting a write in two changes nothing of what
// a stream emits).  The first sub-write lists every such entry, so that a 0-byte write still opens its frame.
int fw_host(k4lz4_frame_writer_group* g, bool closing, const Batch& b, const int32_t* streams, cudaStream_t st) {
    std::vector<int32_t> res;
    if (closing) {                   // the device checks the capacities
        std::vector<int64_t> idx((size_t)b.n), zero((size_t)b.n, 0), wrote((size_t)b.n, 0);
        for (int64_t i = 0; i < b.n; i++) idx[(size_t)i] = i;
        const int rc = fw_host_part(g, true, b, streams, idx, zero, zero, wrote, res, st);
        if (rc != K4LZ4_OK) return rc;
        for (int64_t i = 0; i < b.n; i++) b.outLen[i] = res[(size_t)i];
        return K4LZ4_OK;
    }
    std::vector<int64_t> all;
    for (int64_t i = 0; i < b.n; i++) {
        if (b.dstCap[i] < k4::fw_write_bound(src_size(b, i), g->B, g->bc())) b.outLen[i] = -1;
        else all.push_back(i);
    }
    std::vector<int64_t> used(all.size(), 0), total(all.size(), 0);
    for (bool first = true;; first = false) {
        std::vector<int64_t> idx, at, piece, wrote, which;
        int64_t budget = FW_STAGE_BYTES;
        for (size_t k = 0; k < all.size(); k++) {
            const int64_t take = std::min(src_size(b, all[k]) - used[k], budget);
            if (!first && take == 0) continue;
            idx.push_back(all[k]); at.push_back(used[k]); piece.push_back(take); wrote.push_back(total[k]);
            which.push_back((int64_t)k);
            used[k] += take;
            budget -= take;
        }
        if (idx.empty()) break;
        const int rc = fw_host_part(g, false, b, streams, idx, at, piece, wrote, res, st);
        if (rc != K4LZ4_OK) return rc;
        for (size_t k = 0; k < idx.size(); k++) total[(size_t)which[k]] = wrote[k];
    }
    for (size_t k = 0; k < all.size(); k++) b.outLen[all[k]] = (int32_t)total[k];
    return K4LZ4_OK;
}

int fw_run(k4lz4_frame_writer_group* g, bool closing, const Batch& b, const int32_t* streams, int memKind, void* stream) {
    const int rc = check_step(g, b, streams, b.dstBase && b.dstOff && b.dstCap && b.outLen &&
                                                 (closing || (b.srcBase && b.srcOff && b.srcLen)),
                              memKind, [&](int64_t i) {
        if (closing || k4::fw_write_bound(src_size(b, i), g->B, g->bc()) <= INT32_MAX) return K4LZ4_OK;
        return fail(K4LZ4_E_ARG, "write of %d bytes at entry %lld: its bound exceeds 2^31 - 1", b.srcLen[i], (long long)i);
    });
    if (rc != K4LZ4_OK || b.n == 0) return rc;
    DeviceGuard guard(g->device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", g->device);
    if (memKind == K4LZ4_MEM_HOST) return fw_host(g, closing, b, streams, (cudaStream_t)stream);
    const cudaError_t e = fw_device(g, closing, b, streams, (cudaStream_t)stream);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "frame writer step: %s", cudaGetErrorString(e)); }
    return K4LZ4_OK;
}

}  // namespace

// ---- frame reader groups ----------------------------------------------------------------------------

// S incrementally read LZ4 frame streams (k4lz4.h, frame_reader.cuh): each stream also keeps a stash for a cut
// block, its FrState and the checksum states of its content and of a block being skipped.
struct k4lz4_frame_reader_group : GroupCore {
    int32_t maxBlockSize = 0, stashBody = 0;
    int64_t stashStride = 0;
    uint8_t* stash = nullptr;
    k4::FwState* xs = nullptr;
    k4::FwState* bxs = nullptr;       // the XXH32 of a block being skipped
    k4::FrState* st = nullptr;
    k4::FrDrain* drain = nullptr;     // the undrained rest of each stream's current block (byte reads)
};

namespace {

enum FrMode { FR_END = 0, FR_READ = 1, FR_BYTES = 2, FR_BYTES_INTERACTIVE = 3 };

// One read (FR_READ) or byte read (FR_BYTES*) of b.n entries on `st` with every array on the device: the plan
// (count, scan, the one host synchronisation for the rows and steps, fill), the top-up copies into the stashes;
// for a byte read the walk of the candidate rows, the cut, the drain and pending slides; the skipped blocks' and
// the block checksums, the steps (each: step, copy, codec, post, gather, content checksum, commit, slide), the
// finish, the tail copies.  Host staging (stageOff non-null; b.dstOff is ignored): a plain read places its output
// densely in a pool buffer (*stage) by rows x (maxBlockSize + 8); a byte read waits a second time, once the cut
// knows each entry's output size, and places it 16-aligned in a buffer of the bytes the read appends.  spent (plain
// reads, nullable): the blocks earlier sub-reads decoded.  more (nullable): per entry, for the next sub-read --
// plain: the blocks decoded; byte read: 1 when it stopped on room, interactive mode or an empty block.
cudaError_t fr_device(k4lz4_frame_reader_group* g, int mode, const Batch& b, const int32_t* streams, int32_t* used,
                      int32_t* ended, const int32_t* spent, int32_t* more, int64_t* stageOff, uint8_t** stage,
                      FramePool& P, cudaStream_t st) {
    const int n = (int)b.n;
    const bool bytes = mode != FR_READ;
    const int interactive = mode == FR_BYTES_INTERACTIVE;
    struct Tot { k4::FrameTotals t; int32_t kinds; };
    k4::FrPlan a{};
    a.streams = streams; a.srcBase = b.srcBase; a.srcOff = b.srcOff; a.srcLen = b.srcLen;
    a.dstOff = b.dstOff; a.dstCap = b.dstCap; a.n = n; a.nStreams = g->nStreams;
    a.maxBlockSize = g->maxBlockSize; a.stashBody = g->stashBody; a.stashStride = g->stashStride;
    a.stashRel = (int64_t)((uintptr_t)g->stash - (uintptr_t)b.srcBase);
    a.stash = g->stash; a.st = g->st; a.xs = g->xs; a.bxs = g->bxs; a.stageOff = stageOff;
    a.spent = spent; a.stageSlot = (int64_t)g->maxBlockSize + 8;
    a.interactive = interactive; a.drain = g->drain;
    a.fr = P.get<k4::FrameRec>(n);
    a.ent = P.get<k4::FrEntry>(n);
    a.skipEnt = P.get<k4::FwEntry>(n);
    Tot* tot = P.get<Tot>(1);
    a.tot = &tot->t; a.kinds = &tot->kinds;
    k4::FrCopies& c = a.c;
    c.upOff = P.get<int64_t>(n); c.upDst = P.get<int64_t>(n); c.upLen = P.get<int32_t>(n);
    c.tailOff = P.get<int64_t>(n); c.tailDst = P.get<int64_t>(n); c.tailLen = P.get<int32_t>(n);
    k4::FrameRec* walkFr = nullptr;                    // the walk's error keys: the cut and the decoder decide
    k4::FrPre pre{};
    if (bytes) {
        walkFr = P.get<k4::FrameRec>(n);
        a.cut = P.get<k4::FrCut>(n);
        pre.dOff = P.get<int64_t>(n); pre.dDst = P.get<int64_t>(n); pre.dLen = P.get<int32_t>(n);
        pre.sOff = P.get<int64_t>(n); pre.sDst = P.get<int64_t>(n); pre.sLen = P.get<int32_t>(n);
        if (!more) more = P.get<int32_t>(n);
    }
    FR_TRY(P.err);
    FR_TRY(cudaMemsetAsync(tot, 0, sizeof(Tot), st));
    FR_TRY(cudaMemsetAsync(c.upLen, 0, (size_t)n * 4, st));
    auto plan = [&](int pass) {
        if (bytes) k4::frame_reader_plan_kernel<true><<<grid_of(n), 128, 0, st>>>(pass, a);
        else k4::frame_reader_plan_kernel<false><<<grid_of(n), 128, 0, st>>>(pass, a);
        g_launches++;
    };
    plan(0);
    FR_LAUNCH();
    k4::frame_scan_kernel<<<1, 1024, 0, st>>>(a.fr, n, &tot->t, !bytes && stageOff ? 1 : 0);
    FR_LAUNCH();
    g_launches++;
    Tot h{};
    FR_TRY(cudaMemcpyAsync(&h, tot, sizeof(h), cudaMemcpyDeviceToHost, st));
    FR_TRY(cudaStreamSynchronize(st));                 // the one wait: the rows, the steps, a plain read's staging
    const int64_t nB = h.t.blocks;
    k4::FrameTable& t = a.t;
    t.srcOff = P.get<int64_t>(nB); t.len = P.get<int32_t>(nB); t.kind = P.get<int32_t>(nB);
    t.sum = P.get<uint32_t>(nB); t.ckLen = P.get<int32_t>(nB); t.got = P.get<uint32_t>(nB);
    k4::FrameRec* place = nullptr;
    k4::FrameTotals* placeTot = nullptr;
    if (bytes) {
        t.frame = P.get<int32_t>(nB); t.idx = P.get<int32_t>(nB); t.size = P.get<int32_t>(nB);
        a.rowEnd = P.get<int64_t>(nB);
        if (stageOff) { place = P.get<k4::FrameRec>(n); placeTot = P.get<k4::FrameTotals>(1); }
    }
    uint8_t* dstBase = b.dstBase;
    if (stageOff && !bytes) *stage = dstBase = P.get<uint8_t>(h.t.slots * a.stageSlot);
    FR_TRY(P.err);
    plan(1);
    FR_LAUNCH();
    FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, c.upOff, c.upLen, g->stash, c.upDst, nullptr, nullptr, n}, st));
    if (bytes) {
        if (nB > 0) {
            k4::block_size_walk_kernel<<<grid_of(nB * 32), 128, 0, st>>>(b.srcBase, t, nB, walkFr);
            FR_LAUNCH();
            g_launches++;
        }
        k4::frame_reader_bytes_cut_kernel<<<grid_of(n), 128, 0, st>>>(interactive, a.fr, a.ent, a.cut, n, t, a.rowEnd,
                                                                       g->st, g->bxs, a.skipEnt, g->drain, g->hdr,
                                                                       g->ring, g->slot, g->stashStride, c, pre, more,
                                                                       place);
        FR_LAUNCH();
        g_launches++;
        if (stageOff) {          // host staging only: a second wait, for the bytes the read appends
            k4::frame_scan_kernel<<<1, 1024, 0, st>>>(place, n, placeTot, 1);
            FR_LAUNCH();
            k4::FrameTotals pt{};
            FR_TRY(cudaMemcpyAsync(&pt, placeTot, sizeof(pt), cudaMemcpyDeviceToHost, st));
            FR_TRY(cudaStreamSynchronize(st));
            *stage = dstBase = P.get<uint8_t>(pt.slots * 16);
            FR_TRY(P.err);
            k4::frame_reader_bytes_place_kernel<<<grid_of(n), 128, 0, st>>>(place, a.fr, a.ent, pre, stageOff, n);
            FR_LAUNCH();
            g_launches += 2;
        }
        FR_TRY(launch_op(OP_COPY, Batch{g->rings, pre.dOff, pre.dLen, dstBase, pre.dDst, nullptr, nullptr, n}, st));
        FR_TRY(launch_op(OP_COPY, Batch{g->rings, pre.sOff, pre.sLen, g->rings, pre.sDst, nullptr, nullptr, n}, st));
    }
    if (h.kinds & k4::FRK_SKIP) {
        k4::frame_writer_xxh_kernel<<<grid_of((int64_t)n * 4), 128, 0, st>>>(b.srcBase, a.skipEnt, n, g->bxs);
        FR_LAUNCH();
        g_launches++;
    }
    if (nB > 0 && (h.kinds & k4::FRK_BLOCK_SUM))
        FR_TRY(launch_op(OP_XXH32, Batch{b.srcBase, t.srcOff, t.ckLen, nullptr, nullptr, nullptr, (int32_t*)t.got, nB}, st));
    if (h.t.maxSteps > 0) {
        uint8_t* tab = P.get<uint8_t>((int64_t)n * TABLE_BYTES);
        k4::FrStep s;
        s.srcOff = P.get<int64_t>(n); s.gDst = P.get<int64_t>(n);
        s.lenC = P.get<int32_t>(n); s.lenD = P.get<int32_t>(n); s.resC = P.get<int32_t>(n); s.resD = P.get<int32_t>(n);
        s.kind = P.get<int32_t>(n); s.res = P.get<int32_t>(n); s.gLen = P.get<int32_t>(n);
        s.xe = P.get<k4::FwEntry>(n);
        FR_TRY(P.err);
        const k4::ChainGroupTable ct = carve_table(tab, n);
        const bool linked = h.kinds & k4::FRK_LINKED, indep = h.kinds & k4::FRK_INDEP;
        for (int k = 0; k < h.t.maxSteps; k++) {
            k4::frame_reader_step_kernel<<<grid_of(n), 128, 0, st>>>(k, a.fr, a.ent, n, t, g->hdr, g->ring, ct, s);
            FR_LAUNCH();
            g_launches++;
            FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, ct.copyOff, ct.copyLen, g->rings, ct.ringOff, nullptr, nullptr, n}, st));
            if (linked) {
                Batch kb{b.srcBase, s.srcOff, s.lenC, g->rings, ct.ringOff, ct.len, s.resC, n};
                kb.prefixLen = ct.prefix;
                FR_TRY(launch_op(OP_CHAIN, kb, st));
            }
            if (indep) FR_TRY(launch_op(OP_DECODE, Batch{b.srcBase, s.srcOff, s.lenD, g->rings, ct.ringOff, ct.len, s.resD, n}, st));
            k4::frame_reader_post_kernel<<<grid_of(n), 128, 0, st>>>(k, a.fr, a.ent, b.dstCap, n, ct, s);
            FR_LAUNCH();
            g_launches++;
            FR_TRY(launch_op(OP_COPY, Batch{g->rings, ct.ringOff, s.gLen, dstBase, s.gDst, nullptr, nullptr, n}, st));
            if (h.kinds & k4::FRK_CONTENT_SUM) {
                k4::frame_writer_xxh_kernel<<<grid_of((int64_t)n * 4), 128, 0, st>>>(g->rings, s.xe, n, g->xs);
                FR_LAUNCH();
                g_launches++;
            }
            // a plain read of independent blocks only has nothing to commit: it leaves neither history nor
            // undrained bytes
            if (bytes || linked) {
                k4::frame_reader_commit_kernel<<<grid_of(n), 128, 0, st>>>(a.fr, n, g->ring, g->slot, g->hdr, g->drain,
                                                                           ct, s);
                FR_LAUNCH();
                g_launches++;
            }
            if (linked)
                FR_TRY(launch_op(OP_COPY, Batch{g->rings, ct.copyOff, ct.copyLen, g->rings, ct.ringOff, nullptr, nullptr, n}, st));
        }
    }
    k4::frame_reader_finish_kernel<<<grid_of(n), 128, 0, st>>>(a.fr, a.ent, n, g->st, g->xs, g->bxs, g->hdr, b.outLen,
                                                              used, ended, bytes ? nullptr : more);
    FR_LAUNCH();
    g_launches++;
    FR_TRY(launch_op(OP_COPY, Batch{b.srcBase, c.tailOff, c.tailLen, g->stash, c.tailDst, nullptr, nullptr, n}, st));
    return cudaSuccess;
}

// Host memory, synchronous: sub-reads of at most FW_STAGE_BYTES chunk bytes, in entry order.  Each sub-read is
// one fr_device call on stage_up's table -- cap / aux: a plain read's dstCap and the blocks earlier sub-reads
// decoded, or the room a byte read has left (dstCap minus the bytes earlier sub-reads appended) -- and its output
// comes down behind it, exactly outLen bytes per entry.  The first sub-read lists every entry, so that a byte read
// of an empty chunk still drains.  An entry goes on from where it stopped while it ended no frame, failed nothing
// and has bytes left, and:
// * plain: it consumed its whole piece, or stopped less than 4 bytes before the piece's end inside its chunk.  A
//   sub-read that stopped short of its piece stopped at the room rule, but it consumes an end mark without room, so
//   a length code cut by the piece must be seen whole in the next sub-read.
// * bytes: it did not stop on room, interactive mode or an empty block (a byte read never reads a code once it is
//   out of room) and, interactively, appended nothing yet.
// So cutting a read in two changes nothing.
int fr_host(k4lz4_frame_reader_group* g, int mode, const Batch& b, const int32_t* streams, int32_t* srcUsed,
            int32_t* frameEnded, cudaStream_t st) {
    const Dev* D = dev_state(g->device);
    if (!D || D->err != cudaSuccess) return fail(K4LZ4_E_CUDA, "device %d setup failed", g->device);
    const bool bytes = mode != FR_READ;
    const int64_t n = b.n;
    std::vector<int64_t> usedTot((size_t)n, 0), outTot((size_t)n, 0);
    std::vector<int32_t> spentTot((size_t)n, 0);
    std::vector<uint8_t> active((size_t)n, 1);
    for (int64_t i = 0; i < n; i++) { b.outLen[i] = 0; srcUsed[i] = 0; frameEnded[i] = 0; }
    for (bool first = true;; first = false) {
        std::vector<int64_t> idx, at, piece;
        int64_t budget = FW_STAGE_BYTES;
        for (int64_t i = 0; i < n; i++) {
            if (!active[(size_t)i]) continue;
            if (!first && budget == 0) break;
            const int64_t take = std::min(src_size(b, i) - usedTot[(size_t)i], budget);
            if (!first && take <= 0) { active[(size_t)i] = 0; continue; }
            idx.push_back(i); at.push_back(usedTot[(size_t)i]); piece.push_back(take);
            budget -= take;
        }
        if (idx.empty()) break;
        const int64_t m = (int64_t)idx.size();
        StageUp up;
        const int rc = stage_up(g, m, 4, m * 8, [&](int64_t k) {
            const int64_t i = idx[(size_t)k];
            const int64_t room = std::max<int64_t>(b.dstCap[i], 0) - outTot[(size_t)i];
            return UpRow{piece[k] > 0 ? b.srcBase + b.srcOff[i] + at[k] : nullptr, piece[k], 0, streams[i],
                         (int32_t)piece[k], bytes ? (int32_t)room : b.dstCap[i], bytes ? 0 : spentTot[(size_t)i]};
        }, up, st);
        if (rc != K4LZ4_OK) return rc;
        int64_t* dOff = (int64_t*)up.extra;
        uint8_t* stage = nullptr;
        cudaError_t e;
        {
            FramePool P(D->pool, st);
            const Batch kb{up.src, up.srcOff, up.len, nullptr, nullptr, up.cap, up.res, m};
            e = fr_device(g, mode, kb, up.stream, up.res + m, up.res + 2 * m, up.aux, up.res + 3 * m, dOff, &stage, P, st);
            if (e == cudaSuccess) {
                std::vector<int32_t> down((size_t)m * 4);
                const int rd = stage_down(g, up, m, down.data(), 4, stage, dOff, nullptr, [&](int64_t k) {
                    return b.dstBase + b.dstOff[idx[(size_t)k]] + outTot[(size_t)idx[(size_t)k]];
                }, st);
                if (rd != K4LZ4_OK) return rd;
                for (int64_t k = 0; k < m; k++) {
                    const int64_t i = idx[(size_t)k];
                    const int32_t res = down[(size_t)k], used = down[(size_t)(m + k)];
                    const int32_t ended = down[(size_t)(2 * m + k)], more = down[(size_t)(3 * m + k)];
                    if (res < 0) { b.outLen[i] = res; active[(size_t)i] = 0; continue; }
                    outTot[(size_t)i] += res;
                    usedTot[(size_t)i] += used;
                    b.outLen[i] = (int32_t)outTot[(size_t)i];
                    srcUsed[i] = (int32_t)usedTot[(size_t)i];
                    frameEnded[i] = ended;
                    bool stop;
                    if (bytes) {
                        stop = more || (mode == FR_BYTES_INTERACTIVE && outTot[(size_t)i] > 0);
                    } else {
                        spentTot[(size_t)i] += more;
                        const int64_t end = at[(size_t)k] + piece[(size_t)k];
                        stop = used != piece[(size_t)k] && (end >= src_size(b, i) || end - usedTot[(size_t)i] >= 4);
                    }
                    if (stop || ended || usedTot[(size_t)i] >= src_size(b, i)) active[(size_t)i] = 0;
                }
            }
        }
        if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "frame reader step: %s", cudaGetErrorString(e)); }
    }
    return K4LZ4_OK;
}

// A read, a byte read, or an end (b.outLen = the statuses).  Device memory: enqueued on `stream`; a read waits
// once.  mode -1: a byte read with unknown flags (K4LZ4_E_ARG after the pointer and stream checks).
int fr_run(k4lz4_frame_reader_group* g, int mode, const Batch& b, const int32_t* streams, int32_t* srcUsed,
           int32_t* frameEnded, int memKind, void* stream) {
    const bool reading = mode != FR_END;
    const int rc = check_step(g, b, streams, b.outLen && (!reading || (b.srcBase && b.srcOff && b.srcLen && srcUsed &&
                                                                        b.dstBase && b.dstOff && b.dstCap && frameEnded)),
                              memKind, no_entry_check);
    if (rc != K4LZ4_OK) return rc;
    if (mode < 0) return fail(K4LZ4_E_ARG, "unknown read flags");
    if (b.n == 0) return rc;
    const int n = (int)b.n;
    if (!reading)             // with host memory the statuses come back from behind the stream list in dStage
        return group_streams_run(g, streams, n, memKind, stream, [&](const int32_t* ds, cudaStream_t st) {
            const bool host = memKind == K4LZ4_MEM_HOST;
            int32_t* dStatus = host ? (int32_t*)g->dStage.p + n : b.outLen;
            k4::frame_reader_end_kernel<<<grid_of(n), 128, 0, st>>>(ds, n, g->nStreams, g->st, g->hdr, g->drain, dStatus);
            g_launches++;
            cudaError_t e = cudaGetLastError();
            if (e == cudaSuccess && host) e = cudaMemcpyAsync(b.outLen, dStatus, (size_t)n * 4, cudaMemcpyDeviceToHost, st);
            return e;
        });
    DeviceGuard guard(g->device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", g->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (memKind == K4LZ4_MEM_HOST) return fr_host(g, mode, b, streams, srcUsed, frameEnded, st);
    const Dev* D = dev_state(g->device);
    if (!D || D->err != cudaSuccess) return fail(K4LZ4_E_CUDA, "device %d setup failed", g->device);
    cudaError_t e;
    {
        FramePool P(D->pool, st);
        e = fr_device(g, mode, b, streams, srcUsed, frameEnded, nullptr, nullptr, nullptr, nullptr, P, st);
    }
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(K4LZ4_E_CUDA, "frame reader step: %s", cudaGetErrorString(e)); }
    return K4LZ4_OK;
}

}  // namespace

// ---- exported C ABI ------------------------------------------------------------------------

extern "C" {

int32_t k4lz4_codec_version(void) { return 192; }
int32_t k4lz4_device_count(void) { return device_count_cached(); }
const char* k4lz4_last_error(void) { return t_err.c_str(); }
int64_t k4lz4_launch_count(void) { return g_launches.load(); }

int32_t k4lz4_decode_stats(int32_t device, uint64_t* out4, int32_t reset) {
    return read_stats((const void*)&k4::g_decode_stats, device, out4, reset);
}

int32_t k4lz4_encode_stats(int32_t device, uint64_t* out4, int32_t reset) {
    return read_stats((const void*)&k4::g_encode_stats, device, out4, reset);
}

#ifdef K4_DT_PROFILE
// tools-only build: per-phase cycle sums of the tile decoder (scratch/, never shipped)
__attribute__((visibility("default"))) int32_t k4lz4_debug_prof(uint64_t* out32, int32_t reset) {
    unsigned long long v[32];
    CU_TRY(cudaDeviceSynchronize());
    CU_TRY(cudaMemcpyFromSymbol(v, k4::g_decode_prof, sizeof(v)));
    for (int i = 0; i < 32; i++) out32[i] = v[i];
    if (reset) { unsigned long long z[32] = {0}; CU_TRY(cudaMemcpyToSymbol(k4::g_decode_prof, z, sizeof(z))); }
    return K4LZ4_OK;
}
#endif

int32_t k4lz4_max_output_size(int32_t length) { return k4::max_output_size(length); }
int32_t k4lz4_pickle_bound(int32_t length) { return length <= 0 ? 0 : length + 1; }

int32_t k4lz4_encode(const uint8_t* src, int32_t srcLen, uint8_t* dst, int32_t dstCap, int32_t level) {
    return run_one(OP_ENCODE, src, srcLen, dst, dstCap, level);
}

int32_t k4lz4_encode_x32(const uint8_t* src, int32_t srcLen, uint8_t* dst, int32_t dstCap, int32_t level) {
    return run_one(OP_ENCODE, src, srcLen, dst, dstCap, level, true);
}

int32_t k4lz4_decode(const uint8_t* src, int32_t srcLen, uint8_t* dst, int32_t dstCap) {
    return run_one(OP_DECODE, src, srcLen, dst, dstCap);
}

int32_t k4lz4_decode_dict(const uint8_t* src, int32_t srcLen, uint8_t* dst, int32_t dstCap,
                          const uint8_t* dict, int32_t dictLen) {
    return run_one(OP_GENERAL, src, srcLen, dst, dstCap, 0, false, dict, dictLen);
}

int32_t k4lz4_partial_decode(const uint8_t* src, int32_t srcLen, uint8_t* dst, int32_t targetLen) {
    return run_one(OP_GENERAL, src, srcLen, dst, targetLen, 0, false, nullptr, 0, true);
}

int32_t k4lz4_decode_dict_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                                const uint8_t* dictBase, const int64_t* dictOff, const int32_t* dictLen,
                                int32_t* outLen, int32_t nBlocks, int32_t memKind, void* cudaStream,
                                int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks};
    b.dictBase = dictBase; b.dictOff = dictOff; b.dictLen = dictLen;
    return run(OP_GENERAL, b, memKind, cudaStream, device);
}

int32_t k4lz4_decode_chain_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                 uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                                 const int32_t* prefixLen, int32_t* outLen, int32_t nBlocks,
                                 int32_t memKind, void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks};
    b.prefixLen = prefixLen;
    return run(OP_CHAIN, b, memKind, cudaStream, device);
}

namespace {
int encode_chain_batch(bool x32, const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                       const int32_t* prefixLen, uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                       uint8_t* stateBase, const int64_t* stateOff, int32_t* outLen, int32_t nBlocks, int32_t level,
                       int32_t memKind, void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, level, x32};
    b.prefixLen = prefixLen; b.stateBase = stateBase; b.stateOff = stateOff;
    return run(OP_ENCCHAIN, b, memKind, cudaStream, device);
}
}  // namespace

int32_t k4lz4_encode_chain_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                 const int32_t* prefixLen, uint8_t* dstBase, const int64_t* dstOff,
                                 const int32_t* dstCap, uint8_t* stateBase, const int64_t* stateOff,
                                 int32_t* outLen, int32_t nBlocks, int32_t level, int32_t memKind, void* cudaStream,
                                 int32_t device) {
    return encode_chain_batch(false, srcBase, srcOff, srcLen, prefixLen, dstBase, dstOff, dstCap, stateBase, stateOff,
                              outLen, nBlocks, level, memKind, cudaStream, device);
}

int32_t k4lz4_encode_chain_batch_x32(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                     const int32_t* prefixLen, uint8_t* dstBase, const int64_t* dstOff,
                                     const int32_t* dstCap, uint8_t* stateBase, const int64_t* stateOff,
                                     int32_t* outLen, int32_t nBlocks, int32_t level, int32_t memKind,
                                     void* cudaStream, int32_t device) {
    return encode_chain_batch(true, srcBase, srcOff, srcLen, prefixLen, dstBase, dstOff, dstCap, stateBase, stateOff,
                              outLen, nBlocks, level, memKind, cudaStream, device);
}

int32_t k4lz4_chain_group_create(int32_t kind, int32_t nStreams, int32_t blockSize, int32_t device,
                                 k4lz4_chain_group** out) {
    if (out) *out = nullptr;
    if (!out || (kind != K4LZ4_CHAIN_ENCODER && kind != K4LZ4_CHAIN_DECODER) || nStreams <= 0 || blockSize <= 0)
        return fail(K4LZ4_E_ARG, "bad chain group arguments (kind %d, %d streams, block size %d)", kind, nStreams, blockSize);
    return group_create(nStreams, device, "chain group", out, [&](k4lz4_chain_group& g) {
        g.kind = kind; g.blockSize = blockSize;
        chain_layout(g, (blockSize + 15) & ~int64_t(15));
        if (kind == K4LZ4_CHAIN_ENCODER) g.states = g.alloc<uint8_t>(K4LZ4_CHAIN_STATE_BYTES, true);
    });
}

int32_t k4lz4_chain_group_destroy(k4lz4_chain_group* g) { return group_destroy(g); }

int32_t k4lz4_chain_group_reset(k4lz4_chain_group* g, const int32_t* streams, int32_t n, int32_t memKind,
                                void* cudaStream) {
    return group_reset(g, streams, n, memKind, cudaStream, [&](const int32_t* ds, cudaStream_t st) {
        k4::chain_group_reset_kernel<<<n, 256, 0, st>>>(ds, n, g->nStreams, g->hdr, g->states);
        g_launches++;
        return cudaGetLastError();
    });
}

int32_t k4lz4_chain_group_encode(k4lz4_chain_group* g, const int32_t* streams, const uint8_t* srcBase,
                                 const int64_t* srcOff, const int32_t* srcLen, uint8_t* dstBase, const int64_t* dstOff,
                                 const int32_t* dstCap, int32_t* outLen, int32_t n, int32_t level, int32_t memKind,
                                 void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n, level};
    return group_run(g, K4LZ4_CHAIN_ENCODER, k4::CG_ENCODE, b, streams, memKind, cudaStream);
}

int32_t k4lz4_chain_group_encode_x32(k4lz4_chain_group* g, const int32_t* streams, const uint8_t* srcBase,
                                     const int64_t* srcOff, const int32_t* srcLen, uint8_t* dstBase,
                                     const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int32_t n,
                                     int32_t level, int32_t memKind, void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n, level, true};
    return group_run(g, K4LZ4_CHAIN_ENCODER, k4::CG_ENCODE, b, streams, memKind, cudaStream);
}

int32_t k4lz4_chain_group_decode(k4lz4_chain_group* g, const int32_t* streams, const uint8_t* srcBase,
                                 const int64_t* srcOff, const int32_t* srcLen, uint8_t* dstBase, const int64_t* dstOff,
                                 const int32_t* dstCap, int32_t* outLen, int32_t n, int32_t memKind, void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n};
    return group_run(g, K4LZ4_CHAIN_DECODER, k4::CG_DECODE, b, streams, memKind, cudaStream);
}

int32_t k4lz4_chain_group_inject(k4lz4_chain_group* g, const int32_t* streams, const uint8_t* srcBase,
                                 const int64_t* srcOff, const int32_t* srcLen, int32_t n, int32_t memKind,
                                 void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, nullptr, nullptr, nullptr, nullptr, n};
    return group_run(g, K4LZ4_CHAIN_DECODER, k4::CG_INJECT, b, streams, memKind, cudaStream);
}

int32_t k4lz4_chain_group_state(const k4lz4_chain_group* g, int32_t stream, uint8_t* out) {
    if (!g || g->kind != K4LZ4_CHAIN_ENCODER || !out || stream < 0 || stream >= g->nStreams)
        return fail(K4LZ4_E_ARG, "bad chain group state arguments");
    DeviceGuard guard(g->device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", g->device);
    CU_TRY(cudaDeviceSynchronize());
    CU_TRY(cudaMemcpy(out, g->states + (size_t)stream * K4LZ4_CHAIN_STATE_BYTES, K4LZ4_CHAIN_STATE_BYTES,
                      cudaMemcpyDeviceToHost));
    return K4LZ4_OK;
}

int32_t k4lz4_chain_group_history(const k4lz4_chain_group* g, int32_t stream, uint8_t* out, int32_t cap) {
    if (!g || (!out && cap > 0) || cap < 0 || stream < 0 || stream >= g->nStreams)
        return fail(K4LZ4_E_ARG, "bad chain group history arguments");
    DeviceGuard guard(g->device);
    if (!guard.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", g->device);
    CU_TRY(cudaDeviceSynchronize());
    k4::ChainGroupHdr h;
    CU_TRY(cudaMemcpy(&h, g->hdr + stream, sizeof(h), cudaMemcpyDeviceToHost));
    const int64_t k = std::min<int64_t>(std::min<int64_t>(h.pos, k4::CG_WINDOW), cap);
    if (k > 0)
        CU_TRY(cudaMemcpy(out, g->rings + (size_t)stream * (size_t)g->ring + (size_t)(h.pos - k), (size_t)k,
                          cudaMemcpyDeviceToHost));
    return (int32_t)k;
}

int32_t k4lz4_partial_decode_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                   uint8_t* dstBase, const int64_t* dstOff, const int32_t* targetLen,
                                   int32_t* outLen, int32_t nBlocks, int32_t memKind, void* cudaStream,
                                   int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, targetLen, outLen, nBlocks};
    b.partial = true;
    return run(OP_GENERAL, b, memKind, cudaStream, device);
}

int32_t k4lz4_encode_batch_x32(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                               uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                               int32_t* outLen, int32_t nBlocks, int32_t level, int32_t memKind,
                               void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, level, true};
    return run(OP_ENCODE, b, memKind, cudaStream, device);
}

int32_t k4lz4_encode_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                           uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                           int32_t* outLen, int32_t nBlocks, int32_t level, int32_t memKind,
                           void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks, level};
    return run(OP_ENCODE, b, memKind, cudaStream, device);
}

int32_t k4lz4_decode_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                           uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                           int32_t* outLen, int32_t nBlocks, int32_t memKind, void* cudaStream,
                           int32_t device) {
    return run(OP_DECODE, Batch{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nBlocks},
               memKind, cudaStream, device);
}

int32_t k4lz4_pickle_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                           uint8_t* dstBase, const int64_t* dstOff, int32_t* outLen,
                           int32_t nMessages, int32_t level, int32_t memKind, void* cudaStream,
                           int32_t device) {
    return run(OP_PICKLE, Batch{srcBase, srcOff, srcLen, dstBase, dstOff, nullptr, outLen, nMessages, level},
               memKind, cudaStream, device);
}

int32_t k4lz4_pickle_batch_x32(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                               uint8_t* dstBase, const int64_t* dstOff, int32_t* outLen,
                               int32_t nMessages, int32_t level, int32_t memKind, void* cudaStream,
                               int32_t device) {
    return run(OP_PICKLE, Batch{srcBase, srcOff, srcLen, dstBase, dstOff, nullptr, outLen, nMessages, level, true},
               memKind, cudaStream, device);
}

int32_t k4lz4_pickle_writer_bound(int32_t length) { return length <= 0 ? 0 : length + 1 + k4::pickle_diff_width(length); }

int32_t k4lz4_pickle_writer_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                  uint8_t* dstBase, const int64_t* dstOff, int32_t* outLen,
                                  int32_t nMessages, int32_t level, int32_t memKind, void* cudaStream,
                                  int32_t device) {
    return run(OP_PICKLEW, Batch{srcBase, srcOff, srcLen, dstBase, dstOff, nullptr, outLen, nMessages, level},
               memKind, cudaStream, device);
}

int32_t k4lz4_pickle_writer_batch_x32(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                      uint8_t* dstBase, const int64_t* dstOff, int32_t* outLen,
                                      int32_t nMessages, int32_t level, int32_t memKind, void* cudaStream,
                                      int32_t device) {
    return run(OP_PICKLEW, Batch{srcBase, srcOff, srcLen, dstBase, dstOff, nullptr, outLen, nMessages, level, true},
               memKind, cudaStream, device);
}

int32_t k4lz4_unpickled_size_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                   int32_t* outSize, int32_t nMessages, int32_t memKind,
                                   void* cudaStream, int32_t device) {
    return run(OP_USIZE, Batch{srcBase, srcOff, srcLen, nullptr, nullptr, nullptr, outSize, nMessages},
               memKind, cudaStream, device);
}

int32_t k4lz4_unpickle_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                             uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstLen,
                             int32_t* outLen, int32_t nMessages, int32_t memKind, void* cudaStream,
                             int32_t device) {
    return run(OP_UNPICKLE, Batch{srcBase, srcOff, srcLen, dstBase, dstOff, dstLen, outLen, nMessages},
               memKind, cudaStream, device);
}

int32_t k4lz4_decoded_size_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                 int32_t* outSize, int32_t nBlocks, int32_t memKind, void* cudaStream,
                                 int32_t device) {
    return run(OP_DSIZE, Batch{srcBase, srcOff, srcLen, nullptr, nullptr, nullptr, outSize, nBlocks},
               memKind, cudaStream, device);
}

uint32_t k4lz4_xxh32(const uint8_t* data, int64_t length, uint32_t seed) {
    return k4::xxh32_host(data, length > 0 && data ? (size_t)length : 0, seed);
}

int32_t k4lz4_xxh32_batch(const uint8_t* base, const int64_t* off, const int32_t* len, uint32_t seed,
                          uint32_t* out, int32_t nBlocks, int32_t memKind, void* cudaStream, int32_t device) {
    Batch b{base, off, len, nullptr, nullptr, nullptr, reinterpret_cast<int32_t*>(out), nBlocks};
    b.seed = seed;
    return run(OP_XXH32, b, memKind, cudaStream, device);
}

int32_t k4lz4_synth_host(uint8_t* base, int64_t nBlocks, int32_t blockSize, int32_t matchPermille,
                         uint64_t seed, int64_t firstBlock) {
    if (!base || nBlocks < 0 || blockSize <= 0) return fail(K4LZ4_E_ARG, "bad synth arguments");
    unsigned hw = std::thread::hardware_concurrency();
    int T = (int)std::min<int64_t>(std::min<unsigned>(hw ? hw : 1, 64), std::max<int64_t>(nBlocks, 1));
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([=] {
            for (int64_t b = nBlocks * t / T; b < nBlocks * (t + 1) / T; b++)
                k4::synth_block(base + b * (int64_t)blockSize, blockSize, (uint32_t)matchPermille, seed,
                                (uint64_t)(firstBlock + b));
        });
    for (auto& t : th) t.join();
    return K4LZ4_OK;
}

int32_t k4lz4_synth_device(uint8_t* base, int64_t nBlocks, int32_t blockSize, int32_t matchPermille,
                           uint64_t seed, int64_t firstBlock, void* cudaStream, int32_t device) {
    if (!base || nBlocks < 0 || blockSize <= 0) return fail(K4LZ4_E_ARG, "bad synth arguments");
    const int rc = check_device(device, nBlocks);
    if (rc != K4LZ4_OK || nBlocks == 0) return rc;
    DeviceGuard g(device);
    if (!g.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", device);
    const int threads = 64;
    const long long ctas = (nBlocks + threads - 1) / threads;
    k4::synth_kernel<<<(unsigned)ctas, threads, 0, (cudaStream_t)cudaStream>>>(
        base, nBlocks, blockSize, (uint32_t)matchPermille, seed, firstBlock);
    g_launches++;
    CU_TRY(cudaGetLastError());
    return K4LZ4_OK;
}

int32_t k4lz4_copy_blocks_device(const uint8_t* srcBase, const int64_t* srcOff, uint8_t* dstBase,
                                 const int64_t* dstOff, const int32_t* len, int32_t nBlocks,
                                 void* cudaStream, int32_t device) {
    if (nBlocks < 0 || !srcBase || !srcOff || !dstBase || !dstOff || !len)
        return fail(K4LZ4_E_ARG, "bad copy_blocks arguments");
    const int rc = check_device(device, nBlocks);
    if (rc != K4LZ4_OK || nBlocks == 0) return rc;
    DeviceGuard g(device);
    if (!g.ok) return fail(K4LZ4_E_CUDA, "cudaSetDevice(%d) failed", device);
    CU_TRY(launch_op(OP_COPY, Batch{srcBase, srcOff, len, dstBase, dstOff, nullptr, nullptr, nBlocks},
                     (cudaStream_t)cudaStream));
    return K4LZ4_OK;
}

int64_t k4lz4_frame_bound(int64_t length, int32_t blockSize, int32_t flags) {
    const int32_t bs = frame_block_size(blockSize);
    if (!bs || length < 0 || (flags & ~FRAME_FLAGS)) return fail(K4LZ4_E_ARG, "bad frame bound arguments");
    return frame_bound_of(length, bs, flags);
}

int32_t k4lz4_frame_encode_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                 uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
                                 int32_t nFrames, int32_t blockSize, int32_t flags, int32_t level, int32_t memKind,
                                 void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nFrames, level};
    return frame_run(FO_ENCODE, b, blockSize, flags, memKind, cudaStream, device);
}

int32_t k4lz4_frame_encode_batch_x32(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                     uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
                                     int32_t nFrames, int32_t blockSize, int32_t flags, int32_t level,
                                     int32_t memKind, void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nFrames, level, true};
    return frame_run(FO_ENCODE, b, blockSize, flags, memKind, cudaStream, device);
}

int32_t k4lz4_frame_content_size_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                       int32_t* outSize, int32_t nFrames, int32_t memKind, void* cudaStream,
                                       int32_t device) {
    Batch b{srcBase, srcOff, srcLen, nullptr, nullptr, nullptr, outSize, nFrames};
    return frame_run(FO_SIZE, b, 0, 0, memKind, cudaStream, device);
}

int32_t k4lz4_frame_decode_batch(const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                 uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
                                 int32_t nFrames, int32_t memKind, void* cudaStream, int32_t device) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, nFrames};
    return frame_run(FO_DECODE, b, 0, 0, memKind, cudaStream, device);
}

int32_t k4lz4_frame_writer_group_create(int32_t nStreams, int32_t blockSize, int32_t flags, int32_t level,
                                        int32_t device, k4lz4_frame_writer_group** out) {
    if (out) *out = nullptr;
    const int32_t B = frame_block_size(blockSize);
    if (!out || nStreams <= 0 || !B || (flags & ~FRAME_FLAGS) || level < 0 || level > 0xFF)
        return fail(K4LZ4_E_ARG, "bad frame writer group arguments (%d streams, block size %d, flags 0x%x, level %d)",
                    nStreams, blockSize, flags, level);
    if (level >= 3) return K4LZ4_R_DELEGATE;
    return group_create(nStreams, device, "frame writer group", out, [&](k4lz4_frame_writer_group& g) {
        g.blockSize = blockSize; g.B = B; g.flags = flags; g.level = level;
        g.header = frame_header(blockSize, flags);
        if (g.linked()) chain_layout(g, B);
        else g.ring = g.slot = B;     // independent blocks: the slot alone, pos stays 0
        g.fw = g.alloc<k4::FwState>(sizeof(k4::FwState), true);
        if (g.linked()) g.states = g.alloc<uint8_t>(K4LZ4_CHAIN_STATE_BYTES, true);
    });
}

int32_t k4lz4_frame_writer_group_destroy(k4lz4_frame_writer_group* g) { return group_destroy(g); }

int32_t k4lz4_frame_writer_group_reset(k4lz4_frame_writer_group* g, const int32_t* streams, int32_t n, int32_t memKind,
                                       void* cudaStream) {
    return group_reset(g, streams, n, memKind, cudaStream, [&](const int32_t* ds, cudaStream_t st) {
        k4::frame_writer_reset_kernel<<<grid_of(n), 128, 0, st>>>(ds, n, g->nStreams, g->fw);
        k4::chain_group_reset_kernel<<<n, 256, 0, st>>>(ds, n, g->nStreams, g->hdr, g->states);
        g_launches += 2;
        return cudaGetLastError();
    });
}

int32_t k4lz4_frame_writer_group_write(k4lz4_frame_writer_group* g, const int32_t* streams, const uint8_t* srcBase,
                                       const int64_t* srcOff, const int32_t* srcLen, uint8_t* dstBase,
                                       const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int32_t n,
                                       int32_t memKind, void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n};
    return fw_run(g, false, b, streams, memKind, cudaStream);
}

int32_t k4lz4_frame_writer_group_write_x32(k4lz4_frame_writer_group* g, const int32_t* streams,
                                           const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                           uint8_t* dstBase, const int64_t* dstOff, const int32_t* dstCap,
                                           int32_t* outLen, int32_t n, int32_t memKind, void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n};
    b.x32 = true;
    return fw_run(g, false, b, streams, memKind, cudaStream);
}

int32_t k4lz4_frame_writer_group_close(k4lz4_frame_writer_group* g, const int32_t* streams, uint8_t* dstBase,
                                       const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int32_t n,
                                       int32_t memKind, void* cudaStream) {
    Batch b{nullptr, nullptr, nullptr, dstBase, dstOff, dstCap, outLen, n};
    return fw_run(g, true, b, streams, memKind, cudaStream);
}

int32_t k4lz4_frame_writer_group_close_x32(k4lz4_frame_writer_group* g, const int32_t* streams, uint8_t* dstBase,
                                           const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen, int32_t n,
                                           int32_t memKind, void* cudaStream) {
    Batch b{nullptr, nullptr, nullptr, dstBase, dstOff, dstCap, outLen, n};
    b.x32 = true;
    return fw_run(g, true, b, streams, memKind, cudaStream);
}

int64_t k4lz4_frame_writer_bound(const k4lz4_frame_writer_group* g, int64_t length) {
    if (!g || length < 0) return fail(K4LZ4_E_ARG, "bad frame writer bound arguments");
    return k4::fw_write_bound(length, g->B, g->bc());
}

int64_t k4lz4_frame_writer_close_bound(const k4lz4_frame_writer_group* g) {
    if (!g) return fail(K4LZ4_E_ARG, "null frame writer group");
    return k4::fw_close_bound(g->B, g->bc(), g->cc());
}

int32_t k4lz4_frame_reader_group_create(int32_t nStreams, int32_t maxBlockSize, int32_t device,
                                        k4lz4_frame_reader_group** out) {
    if (out) *out = nullptr;
    const bool bd = maxBlockSize == (1 << 16) || maxBlockSize == (1 << 18) || maxBlockSize == (1 << 20) ||
                    maxBlockSize == (1 << 22);
    if (!out || nStreams <= 0 || !bd)
        return fail(K4LZ4_E_ARG, "bad frame reader group arguments (%d streams, max block size %d)", nStreams,
                    maxBlockSize);
    return group_create(nStreams, device, "frame reader group", out, [&](k4lz4_frame_reader_group& g) {
        g.maxBlockSize = maxBlockSize;
        chain_layout(g, (int64_t)maxBlockSize + 8);
        // a compressed block longer than this decodes to more than maxBlockSize + 8 bytes (frame_lb), so every block
        // a reader can accept fits: [length code | body | checksum]; a longer one is skipped (frame_reader.cuh)
        const int32_t M = maxBlockSize + 8;
        g.stashBody = M + M / 255 + 4;
        g.stashStride = (4 + (int64_t)g.stashBody + 4 + 15) & ~int64_t(15);
        g.stash = g.alloc<uint8_t>((size_t)g.stashStride, false);
        g.xs = g.alloc<k4::FwState>(sizeof(k4::FwState), true);
        g.bxs = g.alloc<k4::FwState>(sizeof(k4::FwState), false);
        g.st = g.alloc<k4::FrState>(sizeof(k4::FrState), true);
        g.drain = g.alloc<k4::FrDrain>(sizeof(k4::FrDrain), true);
    });
}

int32_t k4lz4_frame_reader_group_destroy(k4lz4_frame_reader_group* g) { return group_destroy(g); }

int32_t k4lz4_frame_reader_group_reset(k4lz4_frame_reader_group* g, const int32_t* streams, int32_t n, int32_t memKind,
                                       void* cudaStream) {
    return group_reset(g, streams, n, memKind, cudaStream, [&](const int32_t* ds, cudaStream_t st) {
        k4::frame_reader_end_kernel<<<grid_of(n), 128, 0, st>>>(ds, n, g->nStreams, g->st, g->hdr, g->drain, nullptr);
        g_launches++;
        return cudaGetLastError();
    });
}

int32_t k4lz4_frame_reader_group_read(k4lz4_frame_reader_group* g, const int32_t* streams, const uint8_t* srcBase,
                                      const int64_t* srcOff, const int32_t* srcLen, int32_t* srcUsed, uint8_t* dstBase,
                                      const int64_t* dstOff, const int32_t* dstCap, int32_t* outLen,
                                      int32_t* frameEnded, int32_t n, int32_t memKind, void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n};
    return fr_run(g, FR_READ, b, streams, srcUsed, frameEnded, memKind, cudaStream);
}

int32_t k4lz4_frame_reader_group_read_bytes(k4lz4_frame_reader_group* g, const int32_t* streams,
                                            const uint8_t* srcBase, const int64_t* srcOff, const int32_t* srcLen,
                                            int32_t* srcUsed, uint8_t* dstBase, const int64_t* dstOff,
                                            const int32_t* dstCap, int32_t* outLen, int32_t* frameEnded, int32_t n,
                                            int32_t flags, int32_t memKind, void* cudaStream) {
    Batch b{srcBase, srcOff, srcLen, dstBase, dstOff, dstCap, outLen, n};
    return fr_run(g, flags == 0 ? FR_BYTES : flags == K4LZ4_READ_INTERACTIVE ? FR_BYTES_INTERACTIVE : -1, b, streams,
                  srcUsed, frameEnded, memKind, cudaStream);
}

int32_t k4lz4_frame_reader_group_end(k4lz4_frame_reader_group* g, const int32_t* streams, int32_t* status, int32_t n,
                                     int32_t memKind, void* cudaStream) {
    Batch b{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, status, n};
    return fr_run(g, FR_END, b, streams, nullptr, nullptr, memKind, cudaStream);
}

}  // extern "C"
