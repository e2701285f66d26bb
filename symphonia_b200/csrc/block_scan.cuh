// Exclusive sums within one thread block, and the one-block kernel that runs them over a table of records, shared by the device
// indexes (ogg_index_kernel.cu, adts_index_kernel.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace symgpu_detail {

// Inclusive sum over a warp.
__device__ inline uint64_t warp_sum(uint64_t v) {
    const uint32_t lane = threadIdx.x & 31;
    for (int o = 1; o < 32; o *= 2) {
        const uint64_t u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= uint32_t(o)) v += u;
    }
    return v;
}

// For each of N values per thread: before[k] = v[k] summed over the block's lower threads, total[k] over all of them.  Every
// thread of the block calls it; blockDim.x is a multiple of 32, at most 1024.
template <int N>
__device__ inline void block_exclusive_sums(const uint64_t (&v)[N], uint64_t (&before)[N], uint64_t (&total)[N]) {
    __shared__ uint64_t warp_tot[N][32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    uint64_t s[N];
    for (int k = 0; k < N; ++k) {
        s[k] = warp_sum(v[k]);
        if (lane == 31) warp_tot[k][warp] = s[k];
    }
    __syncthreads();
    if (warp == 0)
        for (int k = 0; k < N; ++k) warp_tot[k][lane] = warp_sum(lane < n_warps ? warp_tot[k][lane] : 0);  // inclusive over the warps
    __syncthreads();
    for (int k = 0; k < N; ++k) before[k] = (warp ? warp_tot[k][warp - 1] : 0) + s[k] - v[k], total[k] = warp_tot[k][n_warps - 1];
    __syncthreads();  // warp_tot may be reused by the next call
}

// Exclusive sums over records rec[0 .. n) in one block of 1024 threads: for every field k < Fields::kN, f.put(rec[i], k, x) with
// x = f.get(rec[j], k) summed over j < i.  get and put may name the same member: each record is read before it is written.
template <class Fields, class Rec>
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(Rec* rec, uint64_t n, Fields f) {
    constexpr int N = Fields::kN;
    uint64_t carry[N] = {};
    for (uint64_t base = 0; base < n; base += 1024) {
        const uint64_t i = base + threadIdx.x;
        uint64_t v[N], before[N], total[N];
        for (int k = 0; k < N; ++k) v[k] = i < n ? f.get(rec[i], k) : 0;
        block_exclusive_sums<N>(v, before, total);
        if (i < n)
            for (int k = 0; k < N; ++k) f.put(rec[i], k, carry[k] + before[k]);
        for (int k = 0; k < N; ++k) carry[k] += total[k];
    }
}

}  // namespace symgpu_detail
