// scan.cuh -- the block-wide integer scans of libpysteps_b200.so (sm_90a).  Every sum runs in a fixed
// order (no atomics), so the offsets they give are the same on every call.
//   block_exclusive_scan  one value per thread of a CTA: a warp scan by __shfl_up_sync, then warp 0
//                         scans the warp sums
//   single_cta_scan       one CTA scans a whole count array, THREADS values at a time, carrying the
//                         sum of the chunks before
#pragma once
#include "common.cuh"

namespace b200 {

// exclusive prefix of v over the CTA; *total = the CTA's sum.  sh: THREADS / 32 values of shared
// memory, free for reuse when this returns
template <int THREADS, typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T *sh, T *total) {
    static_assert(THREADS % 32 == 0 && THREADS <= 1024, "THREADS: whole warps, at most 32 of them");
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    T x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[w] = x;
    __syncthreads();
    if (w == 0) {
        T s = lane < THREADS / 32 ? sh[lane] : T(0);
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < THREADS / 32) sh[lane] = s;
    }
    __syncthreads();
    const T before = w ? sh[w - 1] : T(0);
    *total = sh[THREADS / 32 - 1];
    __syncthreads();  // sh may be reused by the caller
    return before + x - v;
}

// Run by every thread of one CTA of THREADS threads: offset[i] = count[0] + ... + count[i - 1] for
// i < n, summed as T; returns the sum of all n counts to every thread.  offset may be count (the scan
// is then in place).
template <int THREADS, typename C, typename T>
__device__ __forceinline__ T single_cta_scan(const C *count, int64_t n, T *offset) {
    __shared__ T sh[THREADS / 32];
    T carry = 0;
    for (int64_t i0 = 0; i0 < n; i0 += THREADS) {
        const int64_t i = i0 + threadIdx.x;
        const T v = i < n ? (T)count[i] : T(0);
        T total;
        const T e = block_exclusive_scan<THREADS>(v, sh, &total);
        if (i < n) offset[i] = carry + e;
        carry += total;
    }
    return carry;
}

}  // namespace b200
