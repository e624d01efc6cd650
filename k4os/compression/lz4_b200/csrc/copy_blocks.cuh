// copy_blocks.cuh -- batched variable-length device copy (one CTA per block): 16-byte vector
// body when source and destination are mutually aligned, byte head/tail otherwise.
#pragma once
#include "common.cuh"

namespace k4 {

__global__ void __launch_bounds__(256)
copy_blocks_kernel(const uint8_t* __restrict__ srcBase, const int64_t* __restrict__ srcOff,
                   uint8_t* __restrict__ dstBase, const int64_t* __restrict__ dstOff,
                   const int32_t* __restrict__ len, int n) {
    const int b = blockIdx.x;
    if (b >= n) return;
    const int L = len[b];
    if (L <= 0) return;
    const uint8_t* s = srcBase + srcOff[b];
    uint8_t* d = dstBase + dstOff[b];
    const uintptr_t sa = reinterpret_cast<uintptr_t>(s), da = reinterpret_cast<uintptr_t>(d);
    if (((sa ^ da) & 15) == 0 && L >= 64) {
        int head = (int)((16 - (da & 15)) & 15);
        for (int i = threadIdx.x; i < head; i += blockDim.x) d[i] = s[i];
        const int body = (L - head) >> 4;
        const uint4* s4 = reinterpret_cast<const uint4*>(s + head);
        uint4* d4 = reinterpret_cast<uint4*>(d + head);
        for (int i = threadIdx.x; i < body; i += blockDim.x) d4[i] = __ldg(s4 + i);
        // the tails count in 64 bits: head + body * 16 + threadIdx.x passes INT32_MAX when L is near it
#pragma unroll 1
        for (int64_t i = head + ((int64_t)body << 4) + threadIdx.x; i < L; i += blockDim.x) d[i] = s[i];
    } else {
        // mutually misaligned: 4-byte destination words assembled from two source words
        int head = (int)((4 - (da & 3)) & 3);
        if (head > L) head = L;
        for (int i = threadIdx.x; i < head; i += blockDim.x) d[i] = s[i];
        const int body = (L - head) >> 2;
        uint32_t* d4 = reinterpret_cast<uint32_t*>(d + head);
        for (int i = threadIdx.x; i < body; i += blockDim.x) d4[i] = ldg_u32u(s + head + 4 * i);
#pragma unroll 1
        for (int64_t i = head + ((int64_t)body << 2) + threadIdx.x; i < L; i += blockDim.x) d[i] = s[i];
    }
}

}  // namespace k4
