// util.cu -- field statistics (validation of semilagrangian.py:112-123,171-172)
// and a float64 fill.  Pure streaming, HBM-bound: 16-byte loads, grid sized
// to a multiple of the SM count, deterministic two-stage reduction.
#include <math_constants.h>

#include "common.cuh"

namespace {

struct Stats {
    unsigned long long nonfinite, nan;
    double mn, mx;
};

__device__ __forceinline__ void stats_acc(Stats &s, double v) {
    if (!isfinite(v)) s.nonfinite++;
    if (isnan(v)) {
        s.nan++;
    } else {
        s.mn = fmin(s.mn, v);
        s.mx = fmax(s.mx, v);
    }
}

__device__ __forceinline__ Stats stats_merge(Stats a, const Stats &b) {
    a.nonfinite += b.nonfinite;
    a.nan += b.nan;
    a.mn = fmin(a.mn, b.mn);
    a.mx = fmax(a.mx, b.mx);
    return a;
}

__device__ __forceinline__ Stats warp_reduce(Stats s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Stats t;
        t.nonfinite = __shfl_xor_sync(0xffffffffu, s.nonfinite, o);
        t.nan = __shfl_xor_sync(0xffffffffu, s.nan, o);
        t.mn = __shfl_xor_sync(0xffffffffu, s.mn, o);
        t.mx = __shfl_xor_sync(0xffffffffu, s.mx, o);
        s = stats_merge(s, t);
    }
    return s;
}

__device__ __forceinline__ Stats block_reduce(Stats s) {
    __shared__ Stats sm[32];
    s = warp_reduce(s);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) sm[w] = s;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    if (w == 0) {
        Stats t;
        t.nonfinite = 0; t.nan = 0; t.mn = CUDART_INF; t.mx = -CUDART_INF;
        if (l < nw) t = sm[l];
        s = warp_reduce(t);
    }
    return s;
}

template <typename F>
__global__ void __launch_bounds__(256) stats_partial_kernel(const F *__restrict__ a, int64_t count,
                                                            Stats *__restrict__ partial) {
    Stats s;
    s.nonfinite = 0; s.nan = 0; s.mn = CUDART_INF; s.mx = -CUDART_INF;
    constexpr int VEC = 16 / sizeof(F);
    const int64_t nvec = count / VEC;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ((reinterpret_cast<uintptr_t>(a) & 15) == 0) {
        const int4 *a4 = reinterpret_cast<const int4 *>(a);
        for (int64_t i = tid; i < nvec; i += stride) {
            int4 raw = __ldg(a4 + i);
            const F *v = reinterpret_cast<const F *>(&raw);
#pragma unroll
            for (int k = 0; k < VEC; k++) stats_acc(s, (double)v[k]);
        }
        for (int64_t i = nvec * VEC + tid; i < count; i += stride) stats_acc(s, (double)a[i]);
    } else {
        for (int64_t i = tid; i < count; i += stride) stats_acc(s, (double)a[i]);
    }
    s = block_reduce(s);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(256) stats_final_kernel(const Stats *__restrict__ partial, int nparts,
                                                          double *__restrict__ stats) {
    Stats s;
    s.nonfinite = 0; s.nan = 0; s.mn = CUDART_INF; s.mx = -CUDART_INF;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) s = stats_merge(s, partial[i]);
    s = block_reduce(s);
    if (threadIdx.x == 0) {
        stats[0] = (double)s.nonfinite;
        stats[3] = (double)s.nan;
        // np.nanmin / np.nanmax: NaN when every element is NaN
        const bool any = s.mn <= s.mx;
        stats[1] = any ? s.mn : CUDART_NAN;
        stats[2] = any ? s.mx : CUDART_NAN;
    }
}

__global__ void __launch_bounds__(256) fill_kernel(double *__restrict__ dst, int64_t count, double v) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) dst[i] = v;
}

}  // namespace

extern "C" int b200_fill_f64(double *dst, int64_t count, double value, void *stream) {
    B200_REQUIRE(dst != nullptr && count >= 0, "bad arguments");
    const int blocks = (int)std::max<int64_t>(
        1, std::min<int64_t>(b200::ceil_div64(count, 256), (int64_t)b200::num_sms() * 16));
    fill_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dst, count, value);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_field_stats(const void *a, int field_dtype, int64_t count, double *stats,
                                void *stream) {
    B200_REQUIRE(a != nullptr && stats != nullptr && count >= 0, "bad arguments");
    return b200::with_dtype("field", field_dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        cudaStream_t s = (cudaStream_t)stream;
        const int blocks = (int)std::max<int64_t>(
            1, std::min<int64_t>(b200::ceil_div64(count, 256 * 4), (int64_t)b200::num_sms() * 8));
        b200::Scratch part;
        B200_CUDA(part.alloc(sizeof(Stats) * blocks, s));
        stats_partial_kernel<F><<<blocks, 256, 0, s>>>((const F *)a, count, (Stats *)part.p);
        B200_LAUNCH_CHECK();
        stats_final_kernel<<<1, 256, 0, s>>>((const Stats *)part.p, blocks, stats);
        B200_LAUNCH_CHECK();
        return 0;
    });
}
