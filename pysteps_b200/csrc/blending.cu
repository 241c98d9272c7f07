// blending.cu -- linear and salient blending of pysteps/blending/linear_blending.py on the device
// (sm_90a).
//   transform  the inverse transforms of utils/conversion.py:to_rainrate in the field's dtype; the
//              exact ones (copy, square) bit for bit, the transcendental ones (10**(x/10), exp, the
//              Box-Cox inverse) within a few ulp.  Every pixel whose value lies within the error
//              bound of the threshold goes to a list (index, input value) that the host settles
//              with NumPy's own expression; every other pixel is decided here.
//   unit       mm -> mm/h (x / a * b, exact) and dBZ -> mm/h ((x / a) ** b) in place.
//   linear     one launch for all leads and output members: the nowcast and NWP values are read
//              through the member maps, the NWP is nan_to_num'd, the nowcast's NaN filled per output
//              member, and each lead copied or blended in the dtypes the host passes (no FMA).
//   salient    per lead: maxima of both slabs (integer atomics on order-preserving keys), diff and
//              its 64-bit keys, the LSD radix sort of radix_sort.cuh (8-bit digits, every digit all
//              keys share skipped), a dense rank from an inclusive scan of key changes
//              scattered back to pixel order, then the salience weight and the blended value.
// No atomics touch floating-point values and every scan runs in a fixed order, so repeated calls
// are bit-identical.
#include "radix_sort.cuh"

namespace {

template <typename T> __device__ __forceinline__ T max_finite();
template <> __device__ __forceinline__ float max_finite<float>() { return 3.4028234663852886e38f; }
template <> __device__ __forceinline__ double max_finite<double>() { return 1.7976931348623157e308; }

// np.nan_to_num: NaN -> 0, +-inf -> +-max finite of the dtype
template <typename T> __device__ __forceinline__ T nan_to_num(T v) {
    if (isnan(v)) return T(0);
    if (isinf(v)) return v > T(0) ? max_finite<T>() : -max_finite<T>();
    return v;
}

// ---------------------------------------------------------------- conversion to rain rate
template <typename T>
__global__ void __launch_bounds__(THREADS)
    transform_kernel(const T *__restrict__ x, T *__restrict__ y, int64_t n, int kind, double lam, double thr,
                     double zero, double eps, long long *__restrict__ fix_idx, double *__restrict__ fix_x,
                     long long cap, unsigned long long *__restrict__ nfix) {
    for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * THREADS) {
        const T v = x[i];
        T r;
        double rel = 0.0;
        if (kind == B200_BLEND_COPY) {
            r = v;
        } else if (kind == B200_BLEND_SQUARE) {
            r = v * v;
        } else if (kind == B200_BLEND_DB) {
            r = pow(T(10), v / T(10));
            rel = 16.0 * eps;
        } else if (kind == B200_BLEND_EXP) {
            r = exp(v);
            rel = 16.0 * eps;
        } else {  // Box-Cox, lambda != 0: exp(log(lambda x + 1) / lambda), the error grows with the exponent
            const T z = log(T(lam) * v + T(1)) / T(lam);
            r = exp(z);
            rel = 16.0 * eps * (2.0 + fabs((double)z));
        }
        if (rel > 0.0) {
            const double d = (double)r;
            // a non-finite value is never within the bound of a finite threshold
            if (isfinite(d) && fabs(d - thr) <= rel * fmax(fabs(d), fabs(thr)) + 1e-300) {
                const unsigned long long slot = atomicAdd(nfix, 1ull);
                if ((long long)slot < cap) {
                    fix_idx[slot] = i;
                    fix_x[slot] = (double)v;
                }
            } else if (d < thr) {
                r = (T)zero;
            }
        }
        y[i] = r;
    }
}

template <typename T>
__global__ void __launch_bounds__(THREADS) unit_kernel(const T *x, T *y, int64_t n, int kind, double a, double b) {
    for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * THREADS) {
        const T v = x[i];
        y[i] = kind == B200_BLEND_MM ? v / T(a) * T(b) : pow(v / T(a), T(b));
    }
}

template <typename T>
__global__ void __launch_bounds__(THREADS)
    scatter_kernel(T *__restrict__ y, const long long *__restrict__ idx, const double *__restrict__ val, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (i < n) y[idx[i]] = (T)val[i];
}

// ---------------------------------------------------------------- the member-mapped fields
struct Fields {
    const void *now;
    const int *now_map;
    int64_t now_member;
    const void *nwp;
    const int *nwp_map;
    int64_t nwp_member;
    int64_t P;
    int fill_nwp;
};

// the nowcast value of output member e at lead i, pixel p, its NaN filled as the reference does
template <typename Tc, typename Tn>
__device__ __forceinline__ Tc now_value(const Fields &f, int e, int i, int64_t p) {
    Tc v = ((const Tc *)f.now)[(int64_t)f.now_map[e] * f.now_member + (int64_t)i * f.P + p];
    if (isnan(v)) {
        const Tn w = ((const Tn *)f.nwp)[(int64_t)f.nwp_map[e] * f.nwp_member + (int64_t)i * f.P + p];
        v = f.fill_nwp ? (Tc)nan_to_num(w) : Tc(0);
    }
    return v;
}
template <typename Tn>
__device__ __forceinline__ Tn nwp_value(const Fields &f, int e, int i, int64_t p) {
    return nan_to_num(((const Tn *)f.nwp)[(int64_t)f.nwp_map[e] * f.nwp_member + (int64_t)i * f.P + p]);
}

template <typename T> __device__ __forceinline__ T mul(double w, T v) { return T(w) * v; }

// modes: B200_BLEND_NOWCAST, B200_BLEND_NWP, B200_BLEND_LINEAR (dtype bits: 1 w_nwp * nwp in float64,
// 2 w_now * now in float64, 4 their sum in float64), B200_BLEND_SKIP
template <typename Tc, typename Tn>
__global__ void __launch_bounds__(THREADS)
    linear_kernel(Fields f, Tn *__restrict__ out, int n_out, int T, const int *__restrict__ mode,
                  const int *__restrict__ bits, const double *__restrict__ w_nwp, const double *__restrict__ w_now) {
    for (int y = blockIdx.y; y < n_out * T; y += gridDim.y) {
        const int e = y / T, i = y % T, md = mode[i];
        if (md == B200_BLEND_SKIP) continue;
        const int bt = bits[i];
        const double wn = w_nwp[i], wc = w_now[i];
        Tn *o = out + (int64_t)y * f.P;
        for (int64_t p = (int64_t)blockIdx.x * THREADS + threadIdx.x; p < f.P; p += (int64_t)gridDim.x * THREADS) {
            if (md == B200_BLEND_NOWCAST) {
                o[p] = (Tn)now_value<Tc, Tn>(f, e, i, p);
            } else if (md == B200_BLEND_NWP) {
                o[p] = nwp_value<Tn>(f, e, i, p);
            } else {
                const Tn g = nwp_value<Tn>(f, e, i, p);
                const Tc c = now_value<Tc, Tn>(f, e, i, p);
                const double a = (bt & 1) ? wn * (double)g : (double)mul<Tn>(wn, g);
                const double b = (bt & 2) ? wc * (double)c : (double)mul<Tc>(wc, c);
                o[p] = (bt & 4) ? (Tn)(a + b) : (Tn)((float)a + (float)b);
            }
        }
    }
}

// ---------------------------------------------------------------- salience: maxima, diff, keys
struct SortScratch {
    SortBuffers sort;
    unsigned *rank;              // dense rank of every pixel
    unsigned long long *maxkey;  // 2: maxima of the two slabs
    int *nan_flag;
    unsigned *max_rank;
};

static int64_t carve(SortScratch *s, char *base, int64_t n) {
    Carver c{base};
    carve_sort(&s->sort, c, n);
    s->rank = (unsigned *)c.take(4 * n);
    s->maxkey = (unsigned long long *)c.take(16);
    s->nan_flag = (int *)c.take(4);
    s->max_rank = (unsigned *)c.take(4);
    return c.off;
}

// warp max of 64-bit values (no 64-bit redux instruction)
__device__ __forceinline__ unsigned long long warp_max64(unsigned long long v) {
    for (int o = 16; o; o >>= 1) v = max(v, (unsigned long long)__shfl_xor_sync(FULL, v, o));
    return v;
}

template <typename Tc, typename Tn>
__global__ void __launch_bounds__(THREADS) slab_max(Fields f, int n_out, int lead, unsigned long long *maxkey) {
    unsigned long long mc = 0, mn = 0;
    const int64_t n = (int64_t)n_out * f.P;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS) {
        const int e = (int)(j / f.P);
        const int64_t p = j - (int64_t)e * f.P;
        const Tc c = now_value<Tc, Tn>(f, e, lead, p);
        const Tn g = nwp_value<Tn>(f, e, lead, p);
        mc = max(mc, isnan(c) ? ~0ull : order_key((double)c));  // NaN propagates: the largest key
        mn = max(mn, isnan(g) ? ~0ull : order_key((double)g));
    }
    mc = warp_max64(mc);
    mn = warp_max64(mn);
    if ((threadIdx.x & 31) == 0) {
        atomicMax(maxkey, mc);
        atomicMax(maxkey + 1, mn);
    }
}

// diff = nowcast / max - nwp / max (zeros for a slab whose max == 0) in the reference's dtypes
template <typename Tc, typename Tn, typename Td>
__global__ void __launch_bounds__(THREADS)
    diff_keys(Fields f, int n_out, int lead, const unsigned long long *__restrict__ maxkey,
              unsigned long long *__restrict__ key, unsigned *__restrict__ idx, int *__restrict__ nan_flag) {
    const Tc mc = (Tc)key_value(maxkey[0]);
    const Tn mn = (Tn)key_value(maxkey[1]);
    const int64_t n = (int64_t)n_out * f.P;
    int nan_seen = 0;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS) {
        const int e = (int)(j / f.P);
        const int64_t p = j - (int64_t)e * f.P;
        const Tc c = mc == Tc(0) ? Tc(0) : now_value<Tc, Tn>(f, e, lead, p) / mc;
        const Tn g = mn == Tn(0) ? Tn(0) : nwp_value<Tn>(f, e, lead, p) / mn;
        const Td d = (Td)c - (Td)g;
        nan_seen |= isnan(d);
        key[j] = order_key((double)d);
        idx[j] = (unsigned)j;
    }
    if (__any_sync(FULL, nan_seen) && (threadIdx.x & 31) == 0) atomicOr(nan_flag, 1);
}

template <typename T>
__global__ void __launch_bounds__(THREADS)
    array_keys(const T *__restrict__ x, int64_t n, unsigned long long *__restrict__ key, unsigned *__restrict__ idx,
               int *__restrict__ nan_flag) {
    int nan_seen = 0;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS) {
        const double d = (double)x[j];
        nan_seen |= isnan(d);
        key[j] = order_key(d);
        idx[j] = (unsigned)j;
    }
    if (__any_sync(FULL, nan_seen) && (threadIdx.x & 31) == 0) atomicOr(nan_flag, 1);
}

// ---------------------------------------------------------------- dense rank
// the inclusive scan of the key changes of the sorted keys: the dense rank, scattered to pixel order
struct RankScan {
    SortScratch s;
    int64_t n;
    __device__ bool skip() const { return false; }
    __device__ unsigned load(int64_t i) const {
        const unsigned long long *k = s.sort.key[s.sort.src[PASSES]];
        return i == 0 || k[i] != k[i - 1];
    }
    __device__ void store(int64_t i, unsigned excl, unsigned v) const {
        const unsigned incl = excl + v;
        s.rank[s.sort.idx[s.sort.src[PASSES]][i]] = incl;
        if (i == n - 1) *s.max_rank = incl;
    }
};

// sort the n keys in s.sort.key[0] / s.sort.idx[0] and rank them densely into s.rank, s.max_rank
int dense_rank(SortScratch &s, int64_t n, cudaStream_t st) {
    if (int rc = radix_sort(s.sort, n, st)) return rc;
    return scan(RankScan{s, n}, n, s.sort.bsum, st);
}

// linear_blending.py:_get_ws on the dense rank, then ws * nowcast + (1 - ws) * nwp in float64;
// w = weight, w1 = 1 - weight, w2 = weight**2, w12 = (1 - weight)**2 as the host computed them
template <typename Tc, typename Tn>
__global__ void __launch_bounds__(THREADS)
    salient_kernel(Fields f, Tn *__restrict__ out, int n_out, int T, int lead, SortScratch s, double w, double w1,
                   double w2, double w12) {
    const int64_t n = (int64_t)n_out * f.P;
    const bool all_nan = *s.nan_flag != 0;  // scipy's rankdata: one NaN makes every rank NaN
    const double max_rank = (double)*s.max_rank;
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS) {
        const int e = (int)(j / f.P);
        const int64_t p = j - (int64_t)e * f.P;
        double ws = quiet_nan();
        if (!all_nan) {
            const double r = (double)s.rank[j] / max_rank;
            const double a = w * r;
            const double q = 1.0 - r;
            const double s1 = sqrt(r * r + w2);
            const double s2 = sqrt(q * q + w12);
            ws = 0.5 * (a / (a + w1 * q) + s1 / (s1 + s2));
        }
        const double v = ws * (double)now_value<Tc, Tn>(f, e, lead, p) + (1.0 - ws) * (double)nwp_value<Tn>(f, e, lead, p);
        out[((int64_t)e * T + lead) * f.P + p] = (Tn)v;
    }
}

template <typename T> int transform_run(const void *x, void *y, int64_t n, int kind, double lam, double thr,
                                        double zero, long long *fix_idx, double *fix_x, long long cap,
                                        unsigned long long *nfix, cudaStream_t st) {
    const double eps = sizeof(T) == 4 ? 1.1920928955078125e-07 : 2.220446049250313e-16;
    transform_kernel<T><<<grid_for(n), THREADS, 0, st>>>((const T *)x, (T *)y, n, kind, lam, thr, zero, eps, fix_idx,
                                                        fix_x, cap, nfix);
    B200_LAUNCH_CHECK();
    return 0;
}

template <typename Tc, typename Tn>
int linear_run(const Fields &f, void *out, int n_out, int T, const int *mode, const int *bits, const double *w_nwp,
               const double *w_now, cudaStream_t st) {
    const dim3 grid((unsigned)std::max<int64_t>(1, std::min<int64_t>(b200::ceil_div64(f.P, THREADS), 1024)),
                    (unsigned)std::min(n_out * T, 65535));
    linear_kernel<Tc, Tn><<<grid, THREADS, 0, st>>>(f, (Tn *)out, n_out, T, mode, bits, w_nwp, w_now);
    B200_LAUNCH_CHECK();
    return 0;
}

template <typename Tc, typename Tn, typename Td>
int salient_run(const Fields &f, void *out, int n_out, int T, int lead, double w, double w1, double w2, double w12,
                void *scratch, cudaStream_t st) {
    const int64_t n = (int64_t)n_out * f.P;
    SortScratch s;
    carve(&s, (char *)scratch, n);
    B200_CUDA(cudaMemsetAsync(s.maxkey, 0, 16, st));
    B200_CUDA(cudaMemsetAsync(s.nan_flag, 0, 4, st));
    slab_max<Tc, Tn><<<grid_for(n), THREADS, 0, st>>>(f, n_out, lead, s.maxkey);
    B200_LAUNCH_CHECK();
    diff_keys<Tc, Tn, Td><<<grid_for(n), THREADS, 0, st>>>(f, n_out, lead, s.maxkey, s.sort.key[0], s.sort.idx[0], s.nan_flag);
    B200_LAUNCH_CHECK();
    if (int rc = dense_rank(s, n, st)) return rc;
    salient_kernel<Tc, Tn><<<grid_for(n), THREADS, 0, st>>>(f, (Tn *)out, n_out, T, lead, s, w, w1, w2, w12);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int b200_blend_scratch_bytes(int64_t n, int64_t *bytes) {
    B200_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) && bytes != nullptr, "bad arguments");
    SortScratch s;
    *bytes = carve(&s, nullptr, n);
    return 0;
}

extern "C" int b200_blend_transform(const void *x, void *y, int dtype, int64_t n, int kind, double lam, double thr,
                                    double zero, long long *fix_idx, double *fix_x, int64_t cap,
                                    unsigned long long *nfix, void *stream) {
    B200_REQUIRE(n >= 0 && cap >= 0 && kind >= B200_BLEND_COPY && kind <= B200_BLEND_BOXCOX &&
                     (kind < B200_BLEND_DB || nfix != nullptr),
                 "bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (nfix) B200_CUDA(cudaMemsetAsync(nfix, 0, sizeof(unsigned long long), st));
        if (n == 0) return 0;
        B200_REQUIRE(x != nullptr && y != nullptr && (cap == 0 || (fix_idx != nullptr && fix_x != nullptr)),
                     "bad arguments");
        return transform_run<F>(x, y, n, kind, lam, thr, zero, fix_idx, fix_x, cap, nfix, st);
    });
}

extern "C" int b200_blend_unit(const void *x, void *y, int dtype, int64_t n, int kind, double a, double b,
                               void *stream) {
    B200_REQUIRE(n >= 0 && (kind == B200_BLEND_MM || kind == B200_BLEND_DBZ), "bad arguments");
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (n == 0) return 0;
        B200_REQUIRE(x != nullptr && y != nullptr, "bad arguments");
        unit_kernel<F><<<grid_for(n), THREADS, 0, (cudaStream_t)stream>>>((const F *)x, (F *)y, n, kind, a, b);
        B200_LAUNCH_CHECK();
        return 0;
    });
}

extern "C" int b200_blend_scatter(void *y, int dtype, const long long *idx, const double *val, int64_t n,
                                  void *stream) {
    B200_REQUIRE(n >= 0, "bad arguments");
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (n == 0) return 0;
        B200_REQUIRE(y != nullptr && idx != nullptr && val != nullptr, "bad arguments");
        const unsigned g = (unsigned)b200::ceil_div64(n, THREADS);
        scatter_kernel<F><<<g, THREADS, 0, (cudaStream_t)stream>>>((F *)y, idx, val, n);
        B200_LAUNCH_CHECK();
        return 0;
    });
}

static bool fields_ok(const void *now, const int *now_map, const void *nwp, const int *nwp_map, const void *out) {
    return now && now_map && nwp && nwp_map && out;
}

extern "C" int b200_blend_linear(const void *now, int now_dtype, const int *now_map, int64_t now_member,
                                 const void *nwp, int nwp_dtype, const int *nwp_map, int64_t nwp_member, void *out,
                                 int n_out, int T, int64_t P, const int *mode, const int *bits, const double *w_nwp,
                                 const double *w_now, int fill_nwp, void *stream) {
    B200_REQUIRE(n_out >= 0 && T >= 0 && P >= 0 && (int64_t)n_out * T <= INT32_MAX, "bad arguments");
    return b200::with_dtypes(now_dtype, nwp_dtype, [&](auto tc, auto tn) {
        using Tc = typename decltype(tc)::type;
        using Tn = typename decltype(tn)::type;
        if ((int64_t)n_out * T * P == 0) return 0;
        // now may be NULL when the nowcast has no lead (every lead is then B200_BLEND_NWP)
        B200_REQUIRE(now_map && nwp && nwp_map && out && mode && bits && w_nwp && w_now, "bad arguments");
        const Fields f{now, now_map, now_member, nwp, nwp_map, nwp_member, P, fill_nwp};
        return linear_run<Tc, Tn>(f, out, n_out, T, mode, bits, w_nwp, w_now, (cudaStream_t)stream);
    });
}

extern "C" int b200_blend_salient(const void *now, int now_dtype, const int *now_map, int64_t now_member,
                                  const void *nwp, int nwp_dtype, const int *nwp_map, int64_t nwp_member, void *out,
                                  int n_out, int T, int64_t P, int lead, double w, double w1, double w2, double w12,
                                  int fill_nwp, void *scratch, int64_t scratch_bytes, void *stream) {
    const int64_t n = (int64_t)n_out * P;
    B200_REQUIRE(n_out >= 0 && P >= 0 && n < ((int64_t)1 << 31) && lead >= 0 && lead < T, "bad arguments");
    return b200::with_dtypes(now_dtype, nwp_dtype, [&](auto tc, auto tn) {
        using Tc = typename decltype(tc)::type;
        using Tn = typename decltype(tn)::type;
        if (n == 0) return 0;
        SortScratch s;
        B200_REQUIRE(fields_ok(now, now_map, nwp, nwp_map, out) && scratch && scratch_bytes >= carve(&s, nullptr, n),
                     "bad arguments");
        const Fields f{now, now_map, now_member, nwp, nwp_map, nwp_member, P, fill_nwp};
        return salient_run<Tc, Tn, typename b200::Promote<Tc, Tn>::T>(f, out, n_out, T, lead, w, w1, w2, w12, scratch,
                                                                      (cudaStream_t)stream);
    });
}

extern "C" int b200_dense_rank(const void *x, int dtype, int64_t n, unsigned *rank, unsigned *max_rank, int *nan_flag,
                               void *scratch, int64_t scratch_bytes, void *stream) {
    B200_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "bad arguments");
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (n == 0) return 0;
        SortScratch s;
        B200_REQUIRE(x && rank && max_rank && nan_flag && scratch && scratch_bytes >= carve(&s, nullptr, n),
                     "bad arguments");
        carve(&s, (char *)scratch, n);
        cudaStream_t st = (cudaStream_t)stream;
        B200_CUDA(cudaMemsetAsync(s.nan_flag, 0, 4, st));
        array_keys<F><<<grid_for(n), THREADS, 0, st>>>((const F *)x, n, s.sort.key[0], s.sort.idx[0], s.nan_flag);
        B200_LAUNCH_CHECK();
        if (int rc = dense_rank(s, n, st)) return rc;
        B200_CUDA(cudaMemcpyAsync(rank, s.rank, 4 * n, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaMemcpyAsync(max_rank, s.max_rank, 4, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaMemcpyAsync(nan_flag, s.nan_flag, 4, cudaMemcpyDeviceToDevice, st));
        return 0;
    });
}
