// ensemblestats.cu -- the ensemble statistics of pysteps/postprocessing/ensemblestats.py on the
// device (sm_90a).  Every kernel reads the (k, N) ensemble in member order, one thread per pixel,
// coalesced across pixels:
//   mean     NumPy's sequential sum over the member axis in X's dtype (no FMA), divided by k; the
//            nanmean form sums the members that are not NaN (and not below X_thr) and divides
//            float64(sum) by the integer count
//   excprob  per pixel the exact member counts of X >= thr for up to EXC_CHUNK thresholds a pass,
//            divided by k (NaN when a member is not finite) or by the number of finite members
//   band     a mask kernel (all members finite, some member >= thr) with an exclusive scan of the
//            mask in C order, so that every masked pixel knows its column of the random tie-breaks
//            b; then every member's rank 1 + #{j : (X_j, b_j) < (X_i, b_i)} (the lower member wins a
//            full tie) and the int64 sums of (k - rank) (rank - 1) over the masked pixels
// Floating-point warnings that NumPy would raise are reported as flag bits that the host turns into
// the same warnings.  No atomics touch floating-point values: repeated calls are bit-identical.
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int EXC_CHUNK = 8;        // thresholds counted per pass over X
constexpr int MASK_THREADS = 1024;  // pixels per block of the mask scan
constexpr int SCAN_THREADS = 1024;

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float to_f(double v, float) { return __double2float_rn(v); }
__device__ __forceinline__ double to_f(double v, double) { return v; }

// OR of v over the warp, then one integer atomic per warp that has a bit to report
__device__ __forceinline__ void report(int v, int *flags) {
    v = __reduce_or_sync(0xffffffffu, v);
    if (v && (threadIdx.x & 31) == 0) atomicOr(flags, v);
}

template <typename F>
__global__ void __launch_bounds__(THREADS)
    mean_kernel(const F *__restrict__ X, int k, int64_t N, int nan_mode, int use_thr, double thr,
                F *__restrict__ out, int *__restrict__ flags) {
    const int64_t pix = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    int fl = 0;
    if (pix < N) {
        F acc = F(0);
        int cnt = 0;
#pragma unroll 4
        for (int i = 0; i < k; i++) {
            F v = __ldg(X + (int64_t)i * N + pix);
            if (nan_mode) {
                // X[X < X_thr] = nan, then nanmean adds 0 for every NaN and counts the rest
                if (isnan(v) || (use_thr && (double)v < thr)) v = F(0);
                else cnt++;
            }
            const F s = add_rn(acc, v);
            if (isnan(s) && !isnan(acc) && !isnan(v)) fl |= B200_ENSEMBLE_INVALID;  // inf + -inf
            else if (isinf(s) && !isinf(acc) && !isinf(v)) fl |= B200_ENSEMBLE_OVERFLOW;
            acc = s;
        }
        if (nan_mode) {
            if (cnt == 0) fl |= B200_ENSEMBLE_EMPTY;
            out[pix] = to_f(__ddiv_rn((double)acc, (double)cnt), F(0));
        } else {
            out[pix] = div_rn(acc, (F)k);
        }
    }
    report(fl, flags);
}

struct Thresholds {
    double t[EXC_CHUNK];
    int count;
};

template <typename F>
__global__ void __launch_bounds__(THREADS)
    excprob_kernel(const F *__restrict__ X, int k, int64_t N, const Thresholds th, int ignore_nan,
                   double *__restrict__ out, int *__restrict__ flags) {
    const int64_t pix = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    int fl = 0;
    if (pix < N) {
        int cnt[EXC_CHUNK] = {};
        int finite = 0;
#pragma unroll 4
        for (int i = 0; i < k; i++) {
            const double v = (double)__ldg(X + (int64_t)i * N + pix);
            const bool f = isfinite(v);
            finite += f;
#pragma unroll
            for (int c = 0; c < EXC_CHUNK; c++) cnt[c] += (f && v >= th.t[c]) ? 1 : 0;
        }
        // np.mean: NaN as soon as one member is not finite; np.nanmean: count / finite members
        const bool nan_out = !ignore_nan && finite < k;
        const double den = (double)(ignore_nan ? finite : k);
        if (ignore_nan && finite == 0) fl |= B200_ENSEMBLE_EMPTY;
#pragma unroll
        for (int c = 0; c < EXC_CHUNK; c++)
            if (c < th.count) out[c * N + pix] = nan_out ? b200::quiet_nan() : __ddiv_rn((double)cnt[c], den);
    }
    report(fl, flags);
}

// mask = all members finite and some member >= thr; one byte per pixel and the block's count
template <typename F>
__global__ void __launch_bounds__(MASK_THREADS)
    band_mask_kernel(const F *__restrict__ X, int k, int64_t N, double thr, unsigned char *__restrict__ mask,
                     int *__restrict__ block_count) {
    const int64_t pix = (int64_t)blockIdx.x * MASK_THREADS + threadIdx.x;
    int in = 0;
    if (pix < N) {
        bool finite = true, above = false;
        for (int i = 0; i < k; i++) {
            const double v = (double)__ldg(X + (int64_t)i * N + pix);
            finite = finite && isfinite(v);
            above = above || v >= thr;
        }
        in = finite && above;
        mask[pix] = (unsigned char)in;
    }
    const int c = __syncthreads_count(in);
    if (threadIdx.x == 0) block_count[blockIdx.x] = c;
}

// one block: offset[b] = sum of block_count[0..b), offset[nblocks] = p
__global__ void __launch_bounds__(SCAN_THREADS)
    band_offsets_kernel(const int *__restrict__ block_count, int nblocks, int64_t *__restrict__ offset) {
    const int64_t p = b200::single_cta_scan<SCAN_THREADS>(block_count, nblocks, offset);
    if (threadIdx.x == 0) offset[nblocks] = p;
}

// col[pix] = the pixel's column among the masked pixels in C order, -1 where it is not masked
__global__ void __launch_bounds__(MASK_THREADS)
    band_columns_kernel(const unsigned char *__restrict__ mask, int64_t N, const int64_t *__restrict__ offset,
                        int *__restrict__ col) {
    __shared__ int64_t sh[MASK_THREADS / 32];
    const int64_t pix = (int64_t)blockIdx.x * MASK_THREADS + threadIdx.x;
    const int64_t in = pix < N ? mask[pix] : 0;
    int64_t total;
    const int64_t excl = b200::block_exclusive_scan<MASK_THREADS>(in, sh, &total);
    if (pix < N) col[pix] = in ? (int)(offset[blockIdx.x] + excl) : -1;
}

// every member's rank at every masked pixel, 1 + #{j : (X_j, b_j) < (X_i, b_i)}, ties of both keys
// to the lower member index (np.lexsort((b, X)).argsort() + 1); partial[blockIdx.x * k + i] += the
// block's sum of (k - rank_i) (rank_i - 1), one integer atomic per warp and member
template <typename F>
__global__ void __launch_bounds__(THREADS)
    band_match_kernel(const F *__restrict__ X, int k, int64_t N, const int *__restrict__ col,
                      const double *__restrict__ b, int64_t p, unsigned long long *__restrict__ partial) {
    const int64_t stride = (int64_t)gridDim.x * THREADS;
    unsigned long long *acc = partial + (int64_t)blockIdx.x * k;
    for (int64_t base = (int64_t)blockIdx.x * THREADS; base < N; base += stride) {
        const int64_t pix = base + threadIdx.x;
        const int c = pix < N ? __ldg(col + pix) : -1;
        if (!__any_sync(0xffffffffu, c >= 0)) continue;
        for (int i = 0; i < k; i++) {
            long long m = 0;
            if (c >= 0) {
                const F xi = __ldg(X + (int64_t)i * N + pix);
                const double bi = __ldg(b + (int64_t)i * p + c);
                int r = 1;
                for (int j = 0; j < k; j++) {
                    const F xj = __ldg(X + (int64_t)j * N + pix);
                    const double bj = __ldg(b + (int64_t)j * p + c);
                    r += (xj < xi || (xj == xi && (bj < bi || (bj == bi && j < i)))) ? 1 : 0;
                }
                m = (long long)(k - r) * (long long)(r - 1);
            }
            for (int o = 16; o; o >>= 1) m += __shfl_down_sync(0xffffffffu, m, o);
            if ((threadIdx.x & 31) == 0 && m) atomicAdd(acc + i, (unsigned long long)m);
        }
    }
}

// match[i] = sum over blocks of partial[blk * k + i], one thread per member
__global__ void __launch_bounds__(THREADS)
    band_sum_kernel(const unsigned long long *__restrict__ partial, int blocks, int k, int64_t *__restrict__ match) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    if (i >= k) return;
    unsigned long long s = 0ull;
    for (int blk = 0; blk < blocks; blk++) s += partial[(int64_t)blk * k + i];
    match[i] = (int64_t)s;
}

unsigned grid_for(int64_t N, int threads) { return (unsigned)b200::ceil_div64(N, threads); }

template <typename F>
int mean_run(const F *X, int k, int64_t N, int nan_mode, int use_thr, double thr, F *out, int *flags,
             cudaStream_t s) {
    mean_kernel<F><<<grid_for(N, THREADS), THREADS, 0, s>>>(X, k, N, nan_mode, use_thr, thr, out, flags);
    B200_LAUNCH_CHECK();
    return 0;
}

template <typename F>
int excprob_run(const F *X, int k, int64_t N, const double *thr, int n_thr, int ignore_nan, double *out,
                int *flags, cudaStream_t s) {
    for (int t0 = 0; t0 < n_thr; t0 += EXC_CHUNK) {
        Thresholds th{};
        th.count = n_thr - t0 < EXC_CHUNK ? n_thr - t0 : EXC_CHUNK;
        for (int c = 0; c < EXC_CHUNK; c++) th.t[c] = c < th.count ? thr[t0 + c] : 0.0;
        excprob_kernel<F><<<grid_for(N, THREADS), THREADS, 0, s>>>(X, k, N, th, ignore_nan, out + t0 * N, flags);
        B200_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace

extern "C" int b200_ensemble_mean(const void *X, int dtype, int k, int64_t N, int nan_mode, int use_thr, double thr,
                                  void *out, int *flags, void *stream) {
    B200_REQUIRE(k >= 0 && N >= 0 && N < ((int64_t)1 << 31) && flags != nullptr, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        B200_CUDA(cudaMemsetAsync(flags, 0, sizeof(int), s));
        if (N == 0) return 0;
        B200_REQUIRE(out != nullptr && (k == 0 || X != nullptr), "bad arguments");
        return mean_run<F>((const F *)X, k, N, nan_mode, use_thr, thr, (F *)out, flags, s);
    });
}

extern "C" int b200_ensemble_excprob(const void *X, int dtype, int k, int64_t N, const double *thr, int n_thr,
                                     int ignore_nan, double *out, int *flags, void *stream) {
    B200_REQUIRE(k >= 0 && N >= 0 && N < ((int64_t)1 << 31) && n_thr >= 0 && flags != nullptr, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        B200_CUDA(cudaMemsetAsync(flags, 0, sizeof(int), s));
        if (N == 0 || n_thr == 0) return 0;
        B200_REQUIRE(thr != nullptr && out != nullptr && (k == 0 || X != nullptr), "bad arguments");
        return excprob_run<F>((const F *)X, k, N, thr, n_thr, ignore_nan, out, flags, s);
    });
}

extern "C" int b200_ensemble_band_mask(const void *X, int dtype, int k, int64_t N, double thr, int *col, int64_t *p,
                                       void *stream) {
    B200_REQUIRE(k >= 0 && N >= 0 && N < ((int64_t)1 << 31) && p != nullptr, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (N == 0) {
            B200_CUDA(cudaMemsetAsync(p, 0, sizeof(int64_t), s));
            return 0;
        }
        B200_REQUIRE(col != nullptr && (k == 0 || X != nullptr), "bad arguments");
        const int nblocks = (int)b200::ceil_div64(N, MASK_THREADS);
        b200::Scratch mask, counts, offsets;
        B200_CUDA(mask.alloc((size_t)N, s));
        B200_CUDA(counts.alloc(sizeof(int) * nblocks, s));
        B200_CUDA(offsets.alloc(sizeof(int64_t) * (nblocks + 1), s));
        unsigned char *m = (unsigned char *)mask.p;
        band_mask_kernel<F><<<nblocks, MASK_THREADS, 0, s>>>((const F *)X, k, N, thr, m, (int *)counts.p);
        B200_LAUNCH_CHECK();
        int64_t *off = (int64_t *)offsets.p;
        band_offsets_kernel<<<1, SCAN_THREADS, 0, s>>>((const int *)counts.p, nblocks, off);
        B200_LAUNCH_CHECK();
        band_columns_kernel<<<nblocks, MASK_THREADS, 0, s>>>(m, N, off, col);
        B200_LAUNCH_CHECK();
        B200_CUDA(cudaMemcpyAsync(p, off + nblocks, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
        return 0;
    });
}

extern "C" int b200_ensemble_band_match(const void *X, int dtype, int k, int64_t N, const int *col, const double *b,
                                        int64_t p, int64_t *match, void *stream) {
    B200_REQUIRE(k >= 0 && N >= 0 && N < ((int64_t)1 << 31) && p >= 0 && p <= N, "bad arguments");
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (k == 0) return 0;
        B200_REQUIRE(match != nullptr, "bad arguments");
        cudaStream_t s = (cudaStream_t)stream;
        B200_CUDA(cudaMemsetAsync(match, 0, sizeof(int64_t) * k, s));
        if (p == 0) return 0;
        B200_REQUIRE(X != nullptr && col != nullptr && b != nullptr, "bad arguments");
        const int blocks = (int)std::min<int64_t>(b200::ceil_div64(N, THREADS), (int64_t)b200::num_sms() * 8);
        b200::Scratch partial;
        B200_CUDA(partial.alloc(sizeof(unsigned long long) * blocks * k, s));
        B200_CUDA(cudaMemsetAsync(partial.p, 0, sizeof(unsigned long long) * blocks * k, s));
        unsigned long long *part = (unsigned long long *)partial.p;
        band_match_kernel<F><<<blocks, THREADS, 0, s>>>((const F *)X, k, N, col, b, p, part);
        B200_LAUNCH_CHECK();
        band_sum_kernel<<<b200::ceil_div(k, THREADS), THREADS, 0, s>>>(part, blocks, k, match);
        B200_LAUNCH_CHECK();
        return 0;
    });
}
