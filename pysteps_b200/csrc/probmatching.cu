// probmatching.cu -- probability matching of pysteps/postprocessing/probmatching.py on the device
// (sm_90a), on the radix sort of radix_sort.cuh.
//   stats     the record the host checks before matching: nanmin and counts of both arrays, in two
//             passes (minima by integer atomics on order keys, then counts relative to them).
//   match     nonparam_match_empirical_cdf, sorting only the wet values.  The initial values above
//             their minimum (outside the ignore mask) and the target values above theirs are
//             compacted stably with their indices by a scan, and both lists are sorted.  Initial
//             pixel j with wet position q holds rank r = n - n_xwet + q; ranked(r) is the target's
//             minimum below its dry count n - n_twet and the sorted wet target value after it, and
//             values below the percentile p become the minimum.  Ties are ranked in pixel order,
//             which is argsort(kind="stable").  Every output value is read from an input by index,
//             so -0.0 survives.
//   resample  resample_distributions: the values that are NaN in neither array are compacted and
//             sorted, the 0/1 draws pick between the two descending lists, the picks are sorted
//             again and written, descending, behind the NaN prefix.
// No atomics touch floating-point values and every scan runs in a fixed order, so repeated calls
// are bit-identical.
#include "radix_sort.cuh"

namespace {

// order-preserving 64-bit image of a double with -0.0 below +0.0; NaN is never passed in.  ~0 (no
// double maps there) stands for "no value".
__device__ __forceinline__ unsigned long long signed_key(double d) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(d);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double signed_value(unsigned long long k) {
    if (k == ~0ull) return quiet_nan();
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

template <typename T> __device__ __forceinline__ double ld(const void *p, int64_t i) {
    return (double)((const T *)p)[i];
}
__device__ __forceinline__ double load(const void *p, int dtype, int64_t i) {
    return dtype == B200_F32 ? ld<float>(p, i) : ld<double>(p, i);
}

enum { X_NOTNAN, X_NONFINITE, X_MASKED, X_WET, T_NOTNAN, T_WET, N_COUNTS };

struct Head {
    unsigned long long xmin, tmin;  // signed_key of the minima
    unsigned long long cnt[N_COUNTS];
};

struct PmScratch {
    Head *head;
    SortBuffers a, b;  // initial / target (match), first / second (resample)
    double *picks;     // resample: the picked values in descending position order
};

static int64_t carve(PmScratch *s, char *base, int64_t n) {
    Carver c{base};
    s->head = (Head *)c.take(sizeof(Head));
    carve_sort(&s->a, c, n);
    carve_sort(&s->b, c, n);
    s->picks = (double *)c.take(8 * n);
    return c.off;
}

__device__ __forceinline__ void warp_add(unsigned long long *dst, unsigned v) {
    v = __reduce_add_sync(FULL, v);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(dst, (unsigned long long)v);
}

// ---------------------------------------------------------------- match: the statistics
__global__ void __launch_bounds__(THREADS)
    stats_min(const void *x, int xd, int64_t nx, const void *t, int td, int64_t nt, Head *h) {
    unsigned long long mx = ~0ull, mt = ~0ull;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < max(nx, nt); j += (int64_t)gridDim.x * THREADS) {
        if (j < nx) {
            const double v = load(x, xd, j);
            if (!isnan(v)) mx = min(mx, signed_key(v));
        }
        if (j < nt) {
            const double v = load(t, td, j);
            if (!isnan(v)) mt = min(mt, signed_key(v));
        }
    }
    for (int o = 16; o; o >>= 1) {
        mx = min(mx, (unsigned long long)__shfl_xor_sync(FULL, mx, o));
        mt = min(mt, (unsigned long long)__shfl_xor_sync(FULL, mt, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (mx != ~0ull) atomicMin(&h->xmin, mx);
        if (mt != ~0ull) atomicMin(&h->tmin, mt);
    }
}

__global__ void __launch_bounds__(THREADS)
    stats_count(const void *x, int xd, const unsigned char *ignore, int64_t nx, const void *t, int td, int64_t nt,
                Head *h) {
    const double zx = signed_value(h->xmin), zt = signed_value(h->tmin);
    unsigned c[N_COUNTS] = {};
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < max(nx, nt); j += (int64_t)gridDim.x * THREADS) {
        if (j < nx) {
            const double v = load(x, xd, j);
            c[X_NOTNAN] += !isnan(v);
            if (ignore && ignore[j]) {
                c[X_MASKED]++;
            } else {
                c[X_NONFINITE] += !isfinite(v);
                c[X_WET] += v > zx;
            }
        }
        if (j < nt) {
            const double v = load(t, td, j);
            c[T_NOTNAN] += !isnan(v);
            c[T_WET] += v > zt;
        }
    }
#pragma unroll
    for (int k = 0; k < N_COUNTS; k++) warp_add(&h->cnt[k], c[k]);
}

__global__ void stats_record(const Head *h, double *stats) {
    if (threadIdx.x != 0) return;
    stats[0] = signed_value(h->xmin);
    stats[1] = (double)h->cnt[X_NOTNAN];
    stats[2] = (double)h->cnt[X_NONFINITE];
    stats[3] = (double)h->cnt[X_MASKED];
    stats[4] = (double)h->cnt[X_WET];
    stats[5] = signed_value(h->tmin);
    stats[6] = (double)h->cnt[T_NOTNAN];
    stats[7] = (double)h->cnt[T_WET];
}

// ---------------------------------------------------------------- compaction of the wet values
// value i is kept when keep(i); the kept values go, in index order, to key[0] / idx[0] of the sort
struct WetInitial {
    const void *x;
    int dtype;
    const unsigned char *ignore;
    const double *stats;
    __device__ bool keep(int64_t i) const { return !(ignore && ignore[i]) && load(x, dtype, i) > stats[0]; }
    __device__ double value(int64_t i) const { return load(x, dtype, i); }
};
struct WetTarget {
    const void *t;
    int dtype;
    const double *stats;
    __device__ bool keep(int64_t i) const { return load(t, dtype, i) > stats[5]; }
    __device__ double value(int64_t i) const { return load(t, dtype, i); }
};
struct NotNan {  // resample: NaN in neither array; the values of array `a`
    const void *a;
    int ad;
    const void *b;
    int bd;
    __device__ bool keep(int64_t i) const { return !isnan(load(a, ad, i)) && !isnan(load(b, bd, i)); }
    __device__ double value(int64_t i) const { return load(a, ad, i); }
};

template <typename Sel> struct Compact {
    Sel sel;
    SortBuffers s;
    __device__ bool skip() const { return false; }
    __device__ unsigned load(int64_t i) const { return sel.keep(i); }
    __device__ void store(int64_t i, unsigned excl, unsigned v) const {
        if (v) {
            s.key[0][excl] = order_key(sel.value(i));
            s.idx[0][excl] = (unsigned)i;
        }
    }
};

template <typename Sel> int compact_sort(const Sel &sel, const SortBuffers &s, int64_t n, int64_t kept, cudaStream_t st) {
    if (int rc = scan(Compact<Sel>{sel, s}, n, s.bsum, st)) return rc;
    return radix_sort(s, kept, st);
}

__device__ __forceinline__ const unsigned *sorted_idx(const SortBuffers &s) { return s.idx[s.src[PASSES]]; }

// ---------------------------------------------------------------- match: the output
struct Ranked {
    const void *t;
    int td;
    const unsigned *tidx;  // the sorted wet target values' indices
    int64_t dry;           // n - n_twet
    double zt;
    __device__ double at(int64_t r) const { return r < dry ? zt : load(t, td, tidx[r - dry]); }
};

// the pixels outside the wet list: ignored ones keep the initial value, the others are dry
__global__ void __launch_bounds__(THREADS)
    match_dry(const void *x, int xd, const unsigned char *ignore, int64_t n, const double *stats, double *out) {
    const double zx = stats[0], zt = stats[5];
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS) {
        const double v = load(x, xd, j);
        if (ignore && ignore[j]) out[j] = v;
        else if (!(v > zx)) out[j] = zt;
    }
}

// the wet pixels: ranked(r) at rank r = n - n_xwet + q for sorted wet position q.  clip: values below
// np.percentile's p = _lerp(ranked(i0), ranked(i1), gamma) become zt.
__global__ void __launch_bounds__(THREADS)
    match_wet(const void *t, int td, SortBuffers sx, SortBuffers sw, int64_t n, int64_t n_xwet, int64_t n_twet,
              const double *stats, int clip, int64_t i0, int64_t i1, double gamma, double *out) {
    const Ranked rk{t, td, n_twet ? sorted_idx(sw) : nullptr, n - n_twet, stats[5]};
    double p = 0.0;
    if (clip) {  // numpy/lib/_function_base_impl.py:_lerp, its two forms, no FMA (--fmad=false)
        const double a = rk.at(i0), b = rk.at(i1);
        const double diff = b - a;
        p = gamma >= 0.5 ? b - diff * (1.0 - gamma) : a + diff * gamma;
    }
    const unsigned *xidx = sorted_idx(sx);
    for (int64_t q = (int64_t)blockIdx.x * THREADS + threadIdx.x; q < n_xwet; q += (int64_t)gridDim.x * THREADS) {
        double v = rk.at(n - n_xwet + q);
        if (clip && v < p) v = rk.zt;
        out[xidx[q]] = v;
    }
}

// ---------------------------------------------------------------- resample
__global__ void __launch_bounds__(THREADS)
    count_nan(const void *a, int ad, const void *b, int bd, int64_t n, unsigned long long *nnan) {
    unsigned c = 0;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS)
        c += isnan(load(a, ad, j)) || isnan(load(b, bd, j));
    warp_add(nnan, c);
}

// picks[q] (descending position q of the m values that are NaN in neither array) = draw ? a : b
__global__ void __launch_bounds__(THREADS)
    pick(const void *a, int ad, const void *b, int bd, SortBuffers sa, SortBuffers sb, int64_t m, int64_t n_nan,
         const unsigned char *draws, double *picks) {
    const unsigned *ia = sorted_idx(sa), *ib = sorted_idx(sb);
    for (int64_t q = (int64_t)blockIdx.x * THREADS + threadIdx.x; q < m; q += (int64_t)gridDim.x * THREADS)
        picks[q] = draws[n_nan + q] ? load(a, ad, ia[m - 1 - q]) : load(b, bd, ib[m - 1 - q]);
}

__global__ void __launch_bounds__(THREADS) pick_keys(const double *picks, int64_t m, SortBuffers s) {
    for (int64_t q = (int64_t)blockIdx.x * THREADS + threadIdx.x; q < m; q += (int64_t)gridDim.x * THREADS) {
        s.key[0][q] = order_key(picks[q]);
        s.idx[0][q] = (unsigned)q;
    }
}

// out[0 .. n_nan) = NaN, then the sorted picks in descending order
template <typename T>
__global__ void __launch_bounds__(THREADS)
    resample_out(const double *picks, SortBuffers s, int64_t m, int64_t n_nan, T *out) {
    const unsigned *idx = m ? sorted_idx(s) : nullptr;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n_nan + m; j += (int64_t)gridDim.x * THREADS)
        out[j] = j < n_nan ? (T)quiet_nan() : (T)picks[idx[m - 1 - (j - n_nan)]];
}

// the kernels here load either dtype at run time, so the entry points take only the visitor's check
int check_dtypes(int a, int b) {
    return b200::with_dtypes(a, b, [](auto, auto) { return 0; });
}

}  // namespace

extern "C" int b200_pm_scratch_bytes(int64_t n, int64_t *bytes) {
    B200_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) && bytes != nullptr, "bad arguments");
    PmScratch s;
    *bytes = carve(&s, nullptr, n);
    return 0;
}

extern "C" int b200_pm_match_stats(const void *x, int x_dtype, const unsigned char *ignore, int64_t n_x, const void *t,
                                   int t_dtype, int64_t n_t, double *stats, void *scratch, int64_t scratch_bytes,
                                   void *stream) {
    const int64_t n = std::max(n_x, n_t);
    PmScratch s;
    B200_REQUIRE(n_x >= 0 && n_t >= 0 && n < ((int64_t)1 << 31) && stats && scratch &&
                     scratch_bytes >= carve(&s, nullptr, 0) && (n_x == 0 || x) && (n_t == 0 || t),
                 "bad arguments");
    if (int rc = check_dtypes(x_dtype, t_dtype)) return rc;
    carve(&s, (char *)scratch, 0);
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaMemsetAsync(s.head, 0, sizeof(Head), st));
    B200_CUDA(cudaMemsetAsync(s.head, 0xff, 2 * sizeof(unsigned long long), st));
    if (n) {
        stats_min<<<grid_for(n), THREADS, 0, st>>>(x, x_dtype, n_x, t, t_dtype, n_t, s.head);
        B200_LAUNCH_CHECK();
        stats_count<<<grid_for(n), THREADS, 0, st>>>(x, x_dtype, ignore, n_x, t, t_dtype, n_t, s.head);
        B200_LAUNCH_CHECK();
    }
    stats_record<<<1, 32, 0, st>>>(s.head, stats);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_pm_match(const void *x, int x_dtype, const unsigned char *ignore, const void *t, int t_dtype,
                             int64_t n, const double *stats, int64_t n_xwet, int64_t n_twet, int clip, int64_t i0,
                             int64_t i1, double gamma, double *out, void *scratch, int64_t scratch_bytes,
                             void *stream) {
    PmScratch s;
    B200_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) && n_xwet >= 0 && n_xwet <= n && n_twet >= 0 && n_twet <= n &&
                     (!clip || (i0 >= 0 && i0 < n && i1 >= 0 && i1 < n)),
                 "bad arguments");
    if (int rc = check_dtypes(x_dtype, t_dtype)) return rc;
    if (n == 0) return 0;
    B200_REQUIRE(x && t && stats && out && scratch && scratch_bytes >= carve(&s, nullptr, n), "bad arguments");
    carve(&s, (char *)scratch, n);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = compact_sort(WetInitial{x, x_dtype, ignore, stats}, s.a, n, n_xwet, st)) return rc;
    if (int rc = compact_sort(WetTarget{t, t_dtype, stats}, s.b, n, n_twet, st)) return rc;
    match_dry<<<grid_for(n), THREADS, 0, st>>>(x, x_dtype, ignore, n, stats, out);
    B200_LAUNCH_CHECK();
    if (n_xwet) {
        match_wet<<<grid_for(n_xwet), THREADS, 0, st>>>(t, t_dtype, s.a, s.b, n, n_xwet, n_twet, stats, clip, i0, i1,
                                                        gamma, out);
        B200_LAUNCH_CHECK();
    }
    return 0;
}

extern "C" int b200_pm_resample_nan(const void *a, int a_dtype, const void *b, int b_dtype, int64_t n,
                                    int64_t *n_nan, void *stream) {
    B200_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) && n_nan, "bad arguments");
    if (int rc = check_dtypes(a_dtype, b_dtype)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaMemsetAsync(n_nan, 0, sizeof(int64_t), st));
    if (n == 0) return 0;
    B200_REQUIRE(a && b, "bad arguments");
    count_nan<<<grid_for(n), THREADS, 0, st>>>(a, a_dtype, b, b_dtype, n, (unsigned long long *)n_nan);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_pm_resample(const void *a, int a_dtype, const void *b, int b_dtype, int64_t n, int64_t n_nan,
                                const unsigned char *draws, void *out, int out_dtype, void *scratch,
                                int64_t scratch_bytes, void *stream) {
    PmScratch s;
    B200_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) && n_nan >= 0 && n_nan <= n, "bad arguments");
    if (int rc = check_dtypes(a_dtype, b_dtype)) return rc;
    return b200::with_dtype("output", out_dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        if (n == 0) return 0;
        B200_REQUIRE(a && b && draws && out && scratch && scratch_bytes >= carve(&s, nullptr, n), "bad arguments");
        carve(&s, (char *)scratch, n);
        cudaStream_t st = (cudaStream_t)stream;
        const int64_t m = n - n_nan;
        if (m) {
            if (int rc = compact_sort(NotNan{a, a_dtype, b, b_dtype}, s.a, n, m, st)) return rc;
            if (int rc = compact_sort(NotNan{b, b_dtype, a, a_dtype}, s.b, n, m, st)) return rc;
            pick<<<grid_for(m), THREADS, 0, st>>>(a, a_dtype, b, b_dtype, s.a, s.b, m, n_nan, draws, s.picks);
            B200_LAUNCH_CHECK();
            pick_keys<<<grid_for(m), THREADS, 0, st>>>(s.picks, m, s.a);
            B200_LAUNCH_CHECK();
            if (int rc = radix_sort(s.a, m, st)) return rc;
        }
        resample_out<T><<<grid_for(n), THREADS, 0, st>>>(s.picks, s.a, m, n_nan, (T *)out);
        B200_LAUNCH_CHECK();
        return 0;
    });
}
