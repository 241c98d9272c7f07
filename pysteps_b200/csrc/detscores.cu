// detscores.cu -- the contingency table of pysteps/verification/detcatscores.py and the moments of
// detcontscores.py on the device (sm_90a).
//
// det_cat_fct_accum counts, per output element, the pairs with pred > thr and obs > thr (hits), pred
// only (false alarms), obs only (misses) and neither (correct negatives), summed over the reduced
// axes.  The input is read in place through the strides of the kept and the reduced axes: no permuted
// copy.  The counts are integers, so their order is free:
//   R <= SMALL_R  one thread per output element walks its R pairs
//   otherwise     one block per (output element, chunk of its pairs), reduced in the block and added
//                 to the output with one 64-bit integer atomic per count
// NaN compares false on both sides, so a NaN pair counts as a "no", as in the reference.
//
// det_cont_fct_accum takes nine np.nanmean over the reduced axes, each of them np.sum of the summand
// with NaN replaced by 0 over its own non-NaN count.  Every sum follows NumPy's order on C-contiguous
// data, which the host hands over as a plan: per output element m, the outer reduced axes o (those
// left of a kept axis, in C order) are added one after the other onto 0, each adding the pairwise sum
// (pairwise_body.cuh) of a contiguous run of L elements (the trailing reduced axes, merged):
//   L <= 128 (one leaf)  one thread per output element runs both phases
//   otherwise            one thread per leaf of every (m, o) run, a block per run combining its tree
//                        level by level, and one thread per output element adding the runs
// Phase 1 sums obs, pred, res = pred - obs, res^2, (pred + obs)^2 and |res|, and counts the finite
// residuals; its means (float64(total) / float64(count), rounded to the summand's dtype, as NumPy
// divides) are broadcast into phase 2, which sums (obs - mobs)(pred - mpred), |obs - mobs|^2 and
// |pred - mpred|^2.  The kernels also report what NumPy's floating-point warnings need: which
// element-wise operations overflowed or made a NaN, and per output element and sum whether +inf and
// -inf were summed.
#include "common.cuh"
#include "pairwise_body.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int64_t SMALL_R = 32;
constexpr int64_t CHUNK = THREADS * 16;  // pairs per block in the block mode
constexpr int MAXD = 4;

// up to four axes of a C-contiguous array: sizes and element strides, slowest first
struct Axes {
    int n;
    int64_t size[MAXD], stride[MAXD];
};

__device__ __forceinline__ int64_t offset(const Axes &a, int64_t i) {
    int64_t off = 0;
#pragma unroll
    for (int d = MAXD - 1; d >= 0; d--) {
        if (d >= a.n) continue;
        const int64_t q = i / a.size[d];
        off += (i - q * a.size[d]) * a.stride[d];
        i = q;
    }
    return off;
}

// 0: hit, 1: false alarm, 2: miss, 3: correct negative
template <typename P, typename O>
__device__ __forceinline__ int category(const P *pred, const O *obs, int64_t off, double thr_p, double thr_o) {
    const bool p = (double)pred[off] > thr_p, o = (double)obs[off] > thr_o;
    return p ? (o ? 0 : 1) : (o ? 2 : 3);
}

template <typename P, typename O>
__global__ void __launch_bounds__(THREADS)
    contab_small_kernel(const P *__restrict__ pred, const O *__restrict__ obs, double thr_p, double thr_o, Axes kept,
                        Axes red, int64_t M, int64_t R, long long *__restrict__ counts) {
    const int64_t m = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (m >= M) return;
    const int64_t base = offset(kept, m);
    long long c0 = 0, c1 = 0, c2 = 0;
    for (int64_t r = 0; r < R; r++) {
        const int k = category(pred, obs, base + offset(red, r), thr_p, thr_o);
        c0 += k == 0;
        c1 += k == 1;
        c2 += k == 2;
    }
    counts[m] = c0;
    counts[M + m] = c1;
    counts[2 * M + m] = c2;
    counts[3 * M + m] = R - c0 - c1 - c2;
}

template <typename P, typename O>
__global__ void __launch_bounds__(THREADS)
    contab_block_kernel(const P *__restrict__ pred, const O *__restrict__ obs, double thr_p, double thr_o, Axes kept,
                        Axes red, int64_t M, int64_t R, int64_t chunks, unsigned long long *__restrict__ counts) {
    __shared__ unsigned sh[3][THREADS / 32];
    const int64_t m = blockIdx.x / chunks, r0 = (blockIdx.x % chunks) * CHUNK;
    const int64_t r1 = r0 + CHUNK < R ? r0 + CHUNK : R;
    const int64_t base = offset(kept, m);
    unsigned c[3] = {0, 0, 0};
    for (int64_t r = r0 + threadIdx.x; r < r1; r += THREADS) {
        const int k = category(pred, obs, base + offset(red, r), thr_p, thr_o);
        c[0] += k == 0;
        c[1] += k == 1;
        c[2] += k == 2;
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int j = 0; j < 3; j++) {
        const unsigned v = __reduce_add_sync(0xffffffffu, c[j]);
        if (lane == 0) sh[j][w] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t[3] = {0, 0, 0};
        for (int j = 0; j < 3; j++)
            for (int i = 0; i < THREADS / 32; i++) t[j] += sh[j][i];
        for (int j = 0; j < 3; j++) atomicAdd(counts + j * M + m, t[j]);
        atomicAdd(counts + 3 * M + m, (unsigned long long)(r1 - r0) - t[0] - t[1] - t[2]);
    }
}

int axes_from(const int64_t *size, const int64_t *stride, int n, Axes *a) {
    B200_REQUIRE(n >= 0 && n <= MAXD && (n == 0 || (size != nullptr && stride != nullptr)), "verif_contab: bad axes");
    a->n = n;
    for (int d = 0; d < n; d++) {
        B200_REQUIRE(size[d] >= 1 && stride[d] >= 0, "verif_contab: bad axes");
        a->size[d] = size[d];
        a->stride[d] = stride[d];
    }
    return 0;
}

int64_t count_of(const Axes &a) {
    int64_t c = 1;
    for (int d = 0; d < a.n; d++) c *= a.size[d];
    return c;
}

template <typename P, typename O>
int contab_run(const P *pred, const O *obs, double thr_p, double thr_o, const Axes &kept, const Axes &red, int64_t M,
               int64_t R, int64_t *counts, cudaStream_t s) {
    if (R <= SMALL_R) {
        contab_small_kernel<P, O><<<(unsigned)b200::ceil_div64(M, THREADS), THREADS, 0, s>>>(
            pred, obs, thr_p, thr_o, kept, red, M, R, (long long *)counts);
        B200_LAUNCH_CHECK();
        return 0;
    }
    const int64_t chunks = b200::ceil_div64(R, CHUNK);
    B200_REQUIRE(M * chunks < ((int64_t)1 << 31), "verif_contab: too many blocks");
    B200_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * 4 * M, s));
    contab_block_kernel<P, O><<<(unsigned)(M * chunks), THREADS, 0, s>>>(pred, obs, thr_p, thr_o, kept, red, M, R,
                                                                          chunks, (unsigned long long *)counts);
    B200_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// moments

constexpr int NSUM = 9;
constexpr int MOM_THREADS = 128;  // the per-element kernels hold nine sums and ten counts  // obs, pred, res, res^2, sum^2, |res|; cov, |obs - mobs|^2, |pred - mpred|^2

template <typename P, typename Q>
struct Mom {
    using R = typename b200::Promote<P, Q>::T;
    const P *pred;
    const Q *obs;
    int cond;  // 0: all pairs, 1: pred > thr or obs > thr, 2: both
    double thr_p, thr_o;
    Axes kept, outer;
    int64_t M, O, L, H;  // H: heap nodes per run
    int depth;
    double *heap;        // runs * H * (6 or 3)
    double *tot;         // NSUM * M, each in its summand's dtype
    long long *cnt;      // (1 + NSUM) * M: the finite residuals, then the non-NaN summands
    int *infs;           // M: bit 2k / 2k + 1 when sum k saw +inf / -inf
    int *flags;          // one word of B200_MOM_* bits

    __device__ __forceinline__ void load(int64_t a, P &p, Q &q) const {
        p = pred[a];
        q = obs[a];
        if (cond) {
            const bool sp = (double)p > thr_p, so = (double)q > thr_o;
            if (!(cond == 1 ? (sp || so) : (sp && so))) {
                p = P(NAN);
                q = Q(NAN);
            }
        }
    }
    __device__ __forceinline__ int64_t run_base(int64_t m, int64_t o) const { return offset(kept, m) + offset(outer, o); }
};

template <typename T> __device__ __forceinline__ T nz(T v) { return isnan(v) ? T(0) : v; }

template <typename T> __device__ __forceinline__ int inf_bits(T v, int k) {
    return isinf(v) ? (1 << (2 * k + (v < T(0)))) : 0;
}

// over / inv: the flags of an operation with result r from operands a, b (NumPy: overflow is a
// finite result rounded to inf, invalid a NaN from non-NaN operands)
template <typename T, typename U, typename V>
__device__ __forceinline__ int op_flags(T r, U a, V b, int over, int inv) {
    int f = 0;
    if (isinf(r) && isfinite(a) && isfinite(b)) f |= over;
    if (isnan(r) && !isnan(a) && !isnan(b)) f |= inv;
    return f;
}

// phase 1 over the leaf [lo, lo + len) of the run at base: the six pairwise leaf sums, and the counts,
// inf bits and flags of its elements added into cnt6 / n / infs / flags
template <typename P, typename Q>
__device__ void phase1_leaf(const Mom<P, Q> &a, int64_t base, int64_t lo, int64_t len, double out[6], long long c[7],
                            int &infs, int &flags) {
    using R = typename Mom<P, Q>::R;
    auto pq = [&](int64_t i, P &p, Q &q) { a.load(base + i, p, q); };
    auto res = [&](int64_t i) { P p; Q q; pq(i, p, q); return (R)p - (R)q; };
    auto sum = [&](int64_t i) { P p; Q q; pq(i, p, q); return (R)p + (R)q; };
    out[0] = pw::leaf<Q>([&](int64_t i) { P p; Q q; pq(i, p, q); return nz(q); }, lo, len);
    out[1] = pw::leaf<P>([&](int64_t i) { P p; Q q; pq(i, p, q); return nz(p); }, lo, len);
    out[2] = pw::leaf<R>([&](int64_t i) { return nz(res(i)); }, lo, len);
    out[3] = pw::leaf<R>([&](int64_t i) { const R r = res(i); return nz(r * r); }, lo, len);
    out[4] = pw::leaf<R>([&](int64_t i) { const R s = sum(i); return nz(s * s); }, lo, len);
    out[5] = pw::leaf<R>([&](int64_t i) { return nz(fabs(res(i))); }, lo, len);
    for (int64_t i = lo; i < lo + len; i++) {
        P p;
        Q q;
        pq(i, p, q);
        const R rp = p, rq = q, r = rp - rq, s = rp + rq, r2 = r * r, s2 = s * s, ar = fabs(r);
        c[0] += isfinite(r);
        c[1] += !isnan(q);
        c[2] += !isnan(p);
        c[3] += !isnan(r);
        c[4] += !isnan(r2);
        c[5] += !isnan(s2);
        c[6] += !isnan(ar);
        infs |= inf_bits(q, 0) | inf_bits(p, 1) | inf_bits(r, 2) | inf_bits(r2, 3) | inf_bits(s2, 4) | inf_bits(ar, 5);
        flags |= op_flags(r, rp, rq, B200_MOM_SUB_RES_OVER, B200_MOM_SUB_RES_INV) | op_flags(s, rp, rq, B200_MOM_ADD_SUM_OVER, B200_MOM_ADD_SUM_INV);
        if (isinf(r2) && isfinite(r)) flags |= B200_MOM_SQ_RES_OVER;
        if (isinf(s2) && isfinite(s)) flags |= B200_MOM_SQ_SUM_OVER;
    }
}

// phase 2 with the output element's means mo (obs) and mp (pred)
template <typename P, typename Q>
__device__ void phase2_leaf(const Mom<P, Q> &a, int64_t base, int64_t lo, int64_t len, Q mo, P mp, double out[3],
                            long long c[3], int &infs, int &flags) {
    using R = typename Mom<P, Q>::R;
    auto dq = [&](int64_t i) { P p; Q q; a.load(base + i, p, q); return (Q)(q - mo); };
    auto dp = [&](int64_t i) { P p; Q q; a.load(base + i, p, q); return (P)(p - mp); };
    out[0] = pw::leaf<R>([&](int64_t i) { return nz((R)dq(i) * (R)dp(i)); }, lo, len);
    out[1] = pw::leaf<Q>([&](int64_t i) { const Q d = fabs(dq(i)); return nz((Q)(d * d)); }, lo, len);
    out[2] = pw::leaf<P>([&](int64_t i) { const P d = fabs(dp(i)); return nz((P)(d * d)); }, lo, len);
    for (int64_t i = lo; i < lo + len; i++) {
        P p;
        Q q;
        a.load(base + i, p, q);
        const Q x = q - mo;
        const P y = p - mp;
        const R cv = (R)x * (R)y;
        const Q vx = fabs(x) * fabs(x);
        const P vy = fabs(y) * fabs(y);
        c[0] += !isnan(cv);
        c[1] += !isnan(vx);
        c[2] += !isnan(vy);
        infs |= inf_bits(cv, 6) | inf_bits(vx, 7) | inf_bits(vy, 8);
        flags |= op_flags(x, q, mo, B200_MOM_SUB_OBS_OVER, B200_MOM_SUB_OBS_INV) | op_flags(y, p, mp, B200_MOM_SUB_PRED_OVER, B200_MOM_SUB_PRED_INV) |
                 op_flags(cv, x, y, B200_MOM_MUL_OVER, B200_MOM_MUL_INV);
        if (isinf(vx) && isfinite(x)) flags |= B200_MOM_SQ_VOBS_OVER;
        if (isinf(vy) && isfinite(y)) flags |= B200_MOM_SQ_VPRED_OVER;
    }
}

// x + y in T, for values of T held in doubles
template <typename T> __device__ __forceinline__ double add_as(double x, double y) { return (double)((T)x + (T)y); }

template <typename P, typename Q>
__device__ __forceinline__ double add_slot(int k, double x, double y) {
    using R = typename Mom<P, Q>::R;
    switch (k) {
        case 0: return add_as<Q>(x, y);
        case 1: return add_as<P>(x, y);
        case 7: return add_as<Q>(x, y);
        case 8: return add_as<P>(x, y);
        default: return add_as<R>(x, y);
    }
}

template <typename T> __device__ __forceinline__ double mean_of(double tot, long long n) {
    return (double)(T)(tot / (double)n);
}

// L <= LEAF: one thread per output element runs both phases over its O runs
template <typename P, typename Q>
__global__ void __launch_bounds__(MOM_THREADS) moments_small_kernel(Mom<P, Q> a) {
    const int64_t m = (int64_t)blockIdx.x * MOM_THREADS + threadIdx.x;
    if (m >= a.M) return;
    double t[NSUM];
#pragma unroll
    for (int k = 0; k < NSUM; k++) t[k] = 0.0;
    long long c[1 + NSUM] = {0};
    int infs = 0, flags = 0;
    for (int64_t o = 0; o < a.O; o++) {
        double s[6];
        phase1_leaf(a, a.run_base(m, o), 0, a.L, s, c, infs, flags);
#pragma unroll
        for (int k = 0; k < 6; k++) t[k] = add_slot<P, Q>(k, t[k], s[k]);
    }
    const Q mo = (Q)mean_of<Q>(t[0], c[1]);
    const P mp = (P)mean_of<P>(t[1], c[2]);
    for (int64_t o = 0; o < a.O; o++) {
        double s[3];
        phase2_leaf(a, a.run_base(m, o), 0, a.L, mo, mp, s, c + 7, infs, flags);
#pragma unroll
        for (int k = 0; k < 3; k++) t[6 + k] = add_slot<P, Q>(6 + k, t[6 + k], s[k]);
    }
#pragma unroll
    for (int k = 0; k < NSUM; k++) a.tot[k * a.M + m] = t[k];
#pragma unroll
    for (int k = 0; k <= NSUM; k++) a.cnt[k * a.M + m] = c[k];
    a.infs[m] = infs;
    if (flags) atomicOr(a.flags, flags);
}

// L > LEAF, phase `ph` (1 or 2): one thread per leaf slot of every run; the leftmost slot below a
// leaf sums it into the run's heap (node-major, K sums per node)
template <typename P, typename Q>
__global__ void __launch_bounds__(MOM_THREADS) moments_leaf_kernel(Mom<P, Q> a, int ph, const double *means) {
    const int64_t t = (int64_t)blockIdx.x * MOM_THREADS + threadIdx.x;
    const int64_t slots = (int64_t)1 << a.depth;
    if (t >= a.M * a.O * slots) return;
    const int64_t run = t / slots, u = t % slots, m = run / a.O, o = run % a.O;
    int64_t lo = 0, len = a.L;
    int level = 0;
    while (len > pw::LEAF) {
        const int64_t h = pw::left_len(len);
        if ((u >> (a.depth - 1 - level)) & 1) {
            lo += h;
            len -= h;
        } else {
            len = h;
        }
        level++;
    }
    const int below = a.depth - level;
    if (u & (((int64_t)1 << below) - 1)) return;
    const int64_t node = ((int64_t)1 << level) - 1 + (u >> below);
    const int K = ph == 1 ? 6 : 3;
    double *h = a.heap + (run * a.H + node) * K;
    int infs = 0, flags = 0;
    if (ph == 1) {
        long long c[7] = {0};
        phase1_leaf(a, a.run_base(m, o), lo, len, h, c, infs, flags);
#pragma unroll
        for (int k = 0; k < 7; k++)
            if (c[k]) atomicAdd((unsigned long long *)a.cnt + k * a.M + m, (unsigned long long)c[k]);
    } else {
        long long c[3] = {0};
        phase2_leaf(a, a.run_base(m, o), lo, len, (Q)means[m], (P)means[a.M + m], h, c, infs, flags);
#pragma unroll
        for (int k = 0; k < 3; k++)
            if (c[k]) atomicAdd((unsigned long long *)a.cnt + (7 + k) * a.M + m, (unsigned long long)c[k]);
    }
    if (infs) atomicOr(a.infs + m, infs);
    if (flags) atomicOr(a.flags, flags);
}

// one block per run: every internal node = left child + right child, deepest level first
template <typename P, typename Q>
__global__ void __launch_bounds__(THREADS) moments_combine_kernel(Mom<P, Q> a, int ph) {
    const int64_t run = blockIdx.x;
    const int K = ph == 1 ? 6 : 3, k0 = ph == 1 ? 0 : 6;
    double *h = a.heap + run * a.H * K;
    for (int L = a.depth - 1; L >= 0; L--) {
        for (int64_t v = threadIdx.x; v < ((int64_t)K << L); v += THREADS) {
            const int64_t u = v / K;
            const int k = (int)(v % K);
            int64_t lo, len;
            if (!pw::node(a.L, L, u, &lo, &len) || len <= pw::LEAF) continue;
            const int64_t c = ((int64_t)1 << (L + 1)) - 1 + 2 * u;
            h[(((int64_t)1 << L) - 1 + u) * K + k] = add_slot<P, Q>(k0 + k, h[c * K + k], h[(c + 1) * K + k]);
        }
        __syncthreads();
    }
}

// one thread per output element: the runs added onto 0 in C order; after phase 1 also the means
template <typename P, typename Q>
__global__ void __launch_bounds__(THREADS) moments_finish_kernel(Mom<P, Q> a, int ph, double *means) {
    const int64_t m = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (m >= a.M) return;
    const int K = ph == 1 ? 6 : 3, k0 = ph == 1 ? 0 : 6;
    for (int k = 0; k < K; k++) {
        double t = 0.0;
        for (int64_t o = 0; o < a.O; o++) t = add_slot<P, Q>(k0 + k, t, a.heap[((m * a.O + o) * a.H) * K + k]);
        a.tot[(k0 + k) * a.M + m] = t;
    }
    if (ph == 1) {
        means[m] = mean_of<Q>(a.tot[m], a.cnt[a.M + m]);
        means[a.M + m] = mean_of<P>(a.tot[a.M + m], a.cnt[2 * a.M + m]);
    }
}

template <typename P, typename Q>
int moments_run(Mom<P, Q> a, cudaStream_t s) {
    B200_CUDA(cudaMemsetAsync(a.flags, 0, sizeof(int), s));
    if (a.L <= pw::LEAF) {
        moments_small_kernel<P, Q><<<(unsigned)b200::ceil_div64(a.M, MOM_THREADS), MOM_THREADS, 0, s>>>(a);
        B200_LAUNCH_CHECK();
        return 0;
    }
    a.depth = pw::depth_bound(a.L);
    a.H = ((int64_t)2 << a.depth) - 1;
    const int64_t runs = a.M * a.O;
    B200_REQUIRE(runs < ((int64_t)1 << 31), "verif_cont_moments: too many runs");
    b200::Scratch heap, means;
    B200_CUDA(heap.alloc(sizeof(double) * runs * a.H * 6, s));
    B200_CUDA(means.alloc(sizeof(double) * 2 * a.M, s));
    B200_CUDA(cudaMemsetAsync(a.cnt, 0, sizeof(long long) * (1 + NSUM) * a.M, s));
    B200_CUDA(cudaMemsetAsync(a.infs, 0, sizeof(int) * a.M, s));
    a.heap = (double *)heap.p;
    const unsigned leaf_blocks = (unsigned)b200::ceil_div64(runs << a.depth, MOM_THREADS);
    const unsigned out_blocks = (unsigned)b200::ceil_div64(a.M, THREADS);
    for (int ph = 1; ph <= 2; ph++) {
        moments_leaf_kernel<P, Q><<<leaf_blocks, MOM_THREADS, 0, s>>>(a, ph, (const double *)means.p);
        B200_LAUNCH_CHECK();
        moments_combine_kernel<P, Q><<<(unsigned)runs, THREADS, 0, s>>>(a, ph);
        B200_LAUNCH_CHECK();
        moments_finish_kernel<P, Q><<<out_blocks, THREADS, 0, s>>>(a, ph, (double *)means.p);
        B200_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace

extern "C" int b200_verif_contab(const void *pred, int p_dtype, const void *obs, int o_dtype, double thr_p,
                                 double thr_o, const int64_t *kept_size, const int64_t *kept_stride, int n_kept,
                                 const int64_t *red_size, const int64_t *red_stride, int n_red, int64_t *counts,
                                 void *stream) {
    return b200::with_dtypes(p_dtype, o_dtype, [&](auto tp, auto to) {
        using P = typename decltype(tp)::type;
        using O = typename decltype(to)::type;
        Axes kept, red;
        if (int rc = axes_from(kept_size, kept_stride, n_kept, &kept)) return rc;
        if (int rc = axes_from(red_size, red_stride, n_red, &red)) return rc;
        const int64_t M = count_of(kept), R = count_of(red);
        B200_REQUIRE(M * R < ((int64_t)1 << 31) && counts != nullptr && pred != nullptr && obs != nullptr,
                     "verif_contab: bad arguments");
        return contab_run<P, O>((const P *)pred, (const O *)obs, thr_p, thr_o, kept, red, M, R, counts,
                                (cudaStream_t)stream);
    });
}

extern "C" int b200_verif_cont_moments(const void *pred, int p_dtype, const void *obs, int o_dtype, int conditioning,
                                       double thr_p, double thr_o, const int64_t *kept_size,
                                       const int64_t *kept_stride, int n_kept, const int64_t *outer_size,
                                       const int64_t *outer_stride, int n_outer, int64_t L, double *tot,
                                       int64_t *cnt, int *infs, int *flags, void *stream) {
    return b200::with_dtypes(p_dtype, o_dtype, [&](auto tp, auto tq) {
        using P = typename decltype(tp)::type;
        using Q = typename decltype(tq)::type;
        B200_REQUIRE(conditioning >= 0 && conditioning <= 2 && L >= 1, "verif_cont_moments: bad arguments");
        Axes kept, outer;
        if (int rc = axes_from(kept_size, kept_stride, n_kept, &kept)) return rc;
        if (int rc = axes_from(outer_size, outer_stride, n_outer, &outer)) return rc;
        const int64_t M = count_of(kept), O = count_of(outer);
        B200_REQUIRE(M * O * L < ((int64_t)1 << 31) && pred != nullptr && obs != nullptr && tot != nullptr &&
                         cnt != nullptr && infs != nullptr && flags != nullptr,
                     "verif_cont_moments: bad arguments");
        return moments_run<P, Q>(Mom<P, Q>{(const P *)pred, (const Q *)obs, conditioning, thr_p, thr_o, kept, outer, M,
                                           O, L, 1, 0, nullptr, tot, (long long *)cnt, infs, flags},
                                 (cudaStream_t)stream);
    });
}
