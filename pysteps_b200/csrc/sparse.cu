// sparse.cu -- the sparse-vector cleansing stages of dense_lucaskanade on the device
// (sm_90a): compaction of the kept vectors and grid-cell declustering (the outlier test itself
// needs scipy.spatial.cKDTree's neighbour order and lives in knn.cu).
//
// Reference: pysteps/utils/cleansing.py:21-121 (decluster), a Python loop over <= a few thousand
// vectors around np.unique / np.median; here one small kernel (float64, deterministic order) so
// the vectors never leave the device.
#include <math_constants.h>

#include "common.cuh"

namespace {

// keep rows whose flag is 0, preserving order (xy[~outliers], uv[~outliers])
__global__ void __launch_bounds__(1024)
compact_rows_kernel(const double *__restrict__ xy, const double *__restrict__ uv, const uint8_t *__restrict__ drop,
                    const int *__restrict__ n_dev, int n_cap, double *__restrict__ oxy, double *__restrict__ ouv,
                    int *__restrict__ out_count) {
    __shared__ int warp_tot[32];
    __shared__ int s_base;
    const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int start = 0; start < n; start += blockDim.x) {
        const int i = start + tid;
        const bool keep = i < n && !drop[i];
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[wid] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int q = 0; q < 32; q++) {
            if (q < wid) before += warp_tot[q];
            total += warp_tot[q];
        }
        if (keep) {
            const int o = s_base + before + __popc(bal & ((1u << lane) - 1u));
            oxy[2 * o] = xy[2 * i]; oxy[2 * o + 1] = xy[2 * i + 1];
            ouv[2 * o] = uv[2 * i]; ouv[2 * o + 1] = uv[2 * i + 1];
        }
        __syncthreads();
        if (tid == 0) s_base += total;
        __syncthreads();
    }
    if (tid == 0) *out_count = s_base;
}

// ---- decluster ---------------------------------------------------------------------------
constexpr int DC_MAX = 16384;  // vectors (12 B of shared memory each)
// key = cell_x code (25 bits) | cell_y code (25 bits) | index (14 bits: DC_MAX - 1 fits).  A finite
// cell c in [1 - DC_BIAS, DC_BIAS - 2] has code c + DC_BIAS; -inf is code 0 and +inf the largest
// code, so infinite cells sort where np.unique puts them.
constexpr int DC_IBITS = 14, DC_CBITS = 25;
constexpr long long DC_BIAS = 1ll << (DC_CBITS - 1);
constexpr unsigned long long DC_IMASK = (1ull << DC_IBITS) - 1;

// floor(c / scale) as a key code: -1 for NaN (the row matches no cell), -2 for a finite cell the
// key cannot hold
__device__ __forceinline__ long long cell_code(double c, double scale) {
    const double f = floor(__ddiv_rn(c, scale));
    if (isnan(f)) return -1;
    if (f == -CUDART_INF) return 0;
    if (f == CUDART_INF) return 2 * DC_BIAS - 1;
    if (f < (double)(1 - DC_BIAS) || f > (double)(DC_BIAS - 2)) return -2;
    return (long long)f + DC_BIAS;
}

__device__ __forceinline__ double median_of(const double *__restrict__ a, int stride,
                                            const unsigned long long *__restrict__ keys, int s) {
    // rank selection (s is small): the elements of rank (s-1)/2 and s/2, averaged
    double lo = 0.0, hi = 0.0;
    const int rlo = (s - 1) / 2, rhi = s / 2;
    for (int p = 0; p < s; p++) {
        const double v = a[(size_t)(keys[p] & DC_IMASK) * stride];
        int rank = 0;
        for (int q = 0; q < s; q++) {
            const double u = a[(size_t)(keys[q] & DC_IMASK) * stride];
            rank += (u < v) || (u == v && q < p);
        }
        if (rank == rlo) lo = v;
        if (rank == rhi) hi = v;
    }
    return (rlo == rhi) ? lo : __ddiv_rn(__dadd_rn(lo, hi), 2.0);
}

__global__ void __launch_bounds__(1024)
decluster_kernel(const double *__restrict__ xy, const double *__restrict__ uv, const int *__restrict__ n_dev,
                 int n_cap, int cap_pad, double scale, int min_samples, double *__restrict__ oxy,
                 double *__restrict__ ouv, int *__restrict__ out_count) {
    extern __shared__ __align__(16) unsigned char dc_smem[];
    __shared__ int s_nseg;
    const int ncap = n_dev ? min(*n_dev, n_cap) : n_cap;
    const int tid = threadIdx.x;
    int npad = 1;
    while (npad < ncap) npad <<= 1;
    if (npad < 2) npad = 2;
    unsigned long long *key = reinterpret_cast<unsigned long long *>(dc_smem);  // cap_pad entries
    int *seg_start = reinterpret_cast<int *>(key + cap_pad);                    // cap_pad + 1
    // key = (cell_x, cell_y, index): np.unique(axis=0) orders cells lexicographically by x then y.
    // A row with a NaN cell matches no cell of the reference (coord_ == ucoord_ is false): it sorts
    // last, past the n rows that count.
    __shared__ int s_nan;
    if (tid == 0) s_nan = 0;
    __syncthreads();
    int refuse = 0;
    for (int i = tid; i < npad; i += blockDim.x) {
        unsigned long long kv = ~0ull;
        if (i < ncap) {
            const long long cx = cell_code(xy[2 * i], scale), cy = cell_code(xy[2 * i + 1], scale);
            if (cx == -2 || cy == -2) refuse = 1;
            else if (cx == -1 || cy == -1) atomicAdd(&s_nan, 1);
            else kv = ((unsigned long long)cx << (DC_CBITS + DC_IBITS)) | ((unsigned long long)cy << DC_IBITS) |
                      (unsigned long long)i;
        }
        key[i] = kv;
    }
    // a cell beyond the key, or NaN rows where the reference appends a NaN median for each of them
    // (min_samples < 1): refused with *out_count = -1, nothing else written
    if (__syncthreads_or(refuse) || (s_nan > 0 && min_samples < 1)) {
        if (tid == 0) *out_count = -1;
        return;
    }
    const int n = ncap - s_nan;
    for (int k = 2; k <= npad; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = tid; t < npad / 2; t += blockDim.x) {
                const int lo = 2 * t - (t & (j - 1)), hi = lo + j;
                const bool asc = (lo & k) == 0;
                const unsigned long long a = key[lo], b = key[hi];
                if ((a > b) == asc) { key[lo] = b; key[hi] = a; }
            }
            __syncthreads();
        }
    // segment heads (first vector of every occupied cell) by a block-wide exclusive scan
    {
        __shared__ int warp_sum[32];
        const int per = (npad + (int)blockDim.x - 1) / (int)blockDim.x;  // consecutive elements per thread
        const int i0 = tid * per;
        int local = 0;
        for (int q = 0; q < per; q++) {
            const int i = i0 + q;
            if (i < n && (i == 0 || (key[i] >> DC_IBITS) != (key[i - 1] >> DC_IBITS))) local++;
        }
        int incl = local;
        const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) warp_sum[wid] = incl;
        __syncthreads();
        int base = 0;
        for (int w = 0; w < wid; w++) base += warp_sum[w];
        int pos = base + incl - local;  // number of heads before this thread's elements
        for (int q = 0; q < per; q++) {
            const int i = i0 + q;
            if (i < n && (i == 0 || (key[i] >> DC_IBITS) != (key[i - 1] >> DC_IBITS))) seg_start[pos++] = i;
        }
        if (tid == (int)blockDim.x - 1) {
            s_nseg = base + incl;
            seg_start[base + incl] = n;
        }
    }
    __syncthreads();
    const int nseg = s_nseg;
    // kept segments keep their sorted order; with min_samples > 1 the output index is the
    // number of kept segments before this one
    for (int sgi = tid; sgi < nseg; sgi += blockDim.x) {
        const int s0 = seg_start[sgi], s = seg_start[sgi + 1] - s0;
        if (s < min_samples) continue;
        int o = sgi;  // every cell is kept when min_samples <= 1 (what dense_lucaskanade passes)
        if (min_samples > 1) {
            o = 0;
            for (int q = 0; q < sgi; q++) o += (seg_start[q + 1] - seg_start[q]) >= min_samples;
        }
        ouv[2 * o] = median_of(uv, 2, key + s0, s);
        ouv[2 * o + 1] = median_of(uv + 1, 2, key + s0, s);
        oxy[2 * o] = median_of(xy, 2, key + s0, s);
        oxy[2 * o + 1] = median_of(xy + 1, 2, key + s0, s);
    }
    __syncthreads();
    if (tid == 0) {
        int o = 0;
        for (int q = 0; q < nseg; q++) o += (seg_start[q + 1] - seg_start[q]) >= min_samples;
        *out_count = o;
    }
}

// ---- global Mahalanobis outlier test (cleansing.py:201-214, k is None) --------------------------
// MD_i = sqrt(z_i VI z_i^T) with z = uv - mean(uv), V = np.cov(z.T), VI = inv(V); out = MD > thr.
// One CTA; float64 sums by a fixed tree (NumPy reduces through BLAS here, so the last bits of V are
// not defined by the reference either: decisions agree unless MD is within ~1e-13 of thr).
__global__ void __launch_bounds__(256)
outliers_global_kernel(const double *__restrict__ uv, const int *__restrict__ n_dev, int n_cap, double thr,
                       uint8_t *__restrict__ out) {
    __shared__ double red[5][256];
    __shared__ double s_mu, s_mv, s_vi[4];
    __shared__ int s_ok;
    const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
    const int tid = threadIdx.x;
    if (n < 2) {  // :177-178
        for (int i = tid; i < n; i += 256) out[i] = 0;
        return;
    }
    auto reduce = [&](int nv) {
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if (tid < o)
                for (int v = 0; v < nv; v++) red[v][tid] += red[v][tid + o];
            __syncthreads();
        }
    };
    double a = 0.0, b = 0.0;
    for (int i = tid; i < n; i += 256) { a += uv[2 * i]; b += uv[2 * i + 1]; }
    red[0][tid] = a; red[1][tid] = b;
    reduce(2);
    if (tid == 0) { s_mu = red[0][0] / (double)n; s_mv = red[1][0] / (double)n; }
    __syncthreads();
    const double mu = s_mu, mv = s_mv;
    // np.cov subtracts the (tiny) mean of the centred data again
    a = b = 0.0;
    for (int i = tid; i < n; i += 256) { a += uv[2 * i] - mu; b += uv[2 * i + 1] - mv; }
    red[0][tid] = a; red[1][tid] = b;
    reduce(2);
    const double au = red[0][0] / (double)n, av = red[1][0] / (double)n;
    __syncthreads();
    double suu = 0.0, suv = 0.0, svv = 0.0;
    for (int i = tid; i < n; i += 256) {
        const double x = (uv[2 * i] - mu) - au, y = (uv[2 * i + 1] - mv) - av;
        suu += x * x; suv += x * y; svv += y * y;
    }
    red[0][tid] = suu; red[1][tid] = suv; red[2][tid] = svv;
    reduce(3);
    if (tid == 0) {
        const double fact = 1.0 / (double)(n - 1);
        const double va = red[0][0] * fact, vb = red[1][0] * fact, vd = red[2][0] * fact;
        // np.linalg.inv: LU with partial pivoting; exactly singular -> LinAlgError -> MD = 0
        const bool swap = fabs(vb) > fabs(va);
        const double p0 = swap ? vb : va, p1 = swap ? vd : vb, q0 = swap ? va : vb, q1 = swap ? vb : vd;
        int ok = 0;
        if (p0 != 0.0 && !isnan(p0)) {
            const double l = q0 * (1.0 / p0), u22 = q1 - l * p1;
            if (u22 != 0.0) {
                const double r00 = swap ? 0.0 : 1.0, r10 = swap ? 1.0 : 0.0, r01 = swap ? 1.0 : 0.0, r11 = swap ? 0.0 : 1.0;
                const double x10 = (r10 - l * r00) / u22, x11 = (r11 - l * r01) / u22;
                s_vi[0] = (r00 - p1 * x10) / p0; s_vi[1] = (r01 - p1 * x11) / p0; s_vi[2] = x10; s_vi[3] = x11;
                ok = 1;
            }
        }
        s_ok = ok;
    }
    __syncthreads();
    for (int i = tid; i < n; i += 256) {
        double MD = 0.0;
        if (s_ok) {
            const double zu = uv[2 * i] - mu, zv = uv[2 * i + 1] - mv;
            const double t0 = zu * s_vi[0] + zv * s_vi[2], t1 = zu * s_vi[1] + zv * s_vi[3];
            MD = sqrt(t0 * zu + t1 * zv);
        }
        out[i] = (MD > thr) ? 1 : 0;
    }
}

}  // namespace

extern "C" int b200_detect_outliers_global(const double *uv, const int *n_dev, int n_cap, double thr,
                                           uint8_t *out, void *stream) {
    B200_REQUIRE(uv && out && n_cap >= 0, "bad arguments");
    if (n_cap == 0) return 0;
    outliers_global_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(uv, n_dev, n_cap, thr, out);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_compact_rows(const double *xy, const double *uv, const uint8_t *drop, const int *n_dev,
                                 int n_cap, double *out_xy, double *out_uv, int *out_count, void *stream) {
    B200_REQUIRE(xy && uv && drop && out_xy && out_uv && out_count && n_cap >= 0, "bad arguments");
    compact_rows_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(xy, uv, drop, n_dev, n_cap, out_xy, out_uv, out_count);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_decluster(const double *xy, const double *uv, const int *n_dev, int n_cap, double scale,
                              int min_samples, double *out_xy, double *out_uv, int *out_count, void *stream) {
    B200_REQUIRE(xy && uv && out_xy && out_uv && out_count && n_cap >= 0 && scale > 0.0, "bad arguments");
    if (n_cap > DC_MAX) {
        b200::set_error("decluster: at most %d vectors are supported", DC_MAX);
        return B200_ENOTSUP;
    }
    int cap_pad = 2;
    while (cap_pad < n_cap) cap_pad <<= 1;
    const size_t smem = (size_t)cap_pad * 8 + ((size_t)cap_pad + 1) * 4;
    B200_CUDA(cudaFuncSetAttribute(decluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    decluster_kernel<<<1, 1024, smem, (cudaStream_t)stream>>>(xy, uv, n_dev, n_cap, cap_pad, scale, min_samples,
                                                             out_xy, out_uv, out_count);
    B200_LAUNCH_CHECK();
    return 0;
}
