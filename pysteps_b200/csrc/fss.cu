// fss.cu -- the fractions skill score of pysteps/verification/spatialscores.py on the device (sm_90a).
//
// fss_accum thresholds a field (non-finite values replaced by thr - 1 first), smooths the 0/1
// indicator with scipy.ndimage.uniform_filter(size=s, mode="constant") and adds three sums of
// products of the smoothed planes.  uniform_filter runs one 1-D pass per axis, axis 0 first; each
// pass is scipy's running sum along a line padded with s // 2 zeros in front:
//   tmp = in[0] + ... + in[s - 1] (sequentially), out[0] = tmp / s,
//   tmp += (in[l + s - 1] - in[l - 1]), out[l] = tmp / s.
//   pass 0 (axis 0)  the input is 0/1, so tmp is an exact integer count and out = count / s in any
//                    order: one thread per (field, column, chunk of rows), coalesced across columns
//   pass 1 (axis 1)  the input is not integral, so the chain runs as scipy runs it: one thread per
//                    (field, row), all rows of all fields of a call in one launch
// The sums are NumPy's pairwise sums (pairwise_body.cuh) of S_a * S_b over the flattened plane.  For
// a group of fields every pair (a <= b) is summed in one launch: each block stages one leaf (at most
// 128 values) of every field of the group in shared memory and forms the leaves of all pairs from
// it; a second kernel combines each pair's leaves along the same tree.  No floating-point atomics.
#include "common.cuh"
#include "pairwise_body.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ROW_CHUNK = 128;

template <typename T>
__device__ __forceinline__ int indicator(T v, double thr, double sub) {
    const double x = isfinite((double)v) ? (double)v : sub;
    return x >= thr;
}

// s <= 1: out = the indicator; otherwise out = the axis-0 pass of the indicator
template <typename T>
__global__ void __launch_bounds__(THREADS)
    fss_pass0_kernel(const T *__restrict__ X, int nf, int m, int n, double thr, double sub, int s,
                     double *__restrict__ out) {
    const int col = blockIdx.x * THREADS + threadIdx.x;
    const int chunks = (m + ROW_CHUNK - 1) / ROW_CHUNK;
    const int f = blockIdx.y / chunks, r0 = (blockIdx.y % chunks) * ROW_CHUNK;
    if (col >= n) return;
    const int r1 = r0 + ROW_CHUNK < m ? r0 + ROW_CHUNK : m;
    const T *x = X + (int64_t)f * m * n + col;
    double *o = out + (int64_t)f * m * n + col;
    if (s <= 1) {
        for (int r = r0; r < r1; r++) o[(int64_t)r * n] = indicator(x[(int64_t)r * n], thr, sub);
        return;
    }
    // the window of output row r covers input rows r - s/2 .. r - s/2 + s - 1
    const int s1 = s / 2;
    auto at = [&](int r) { return (r >= 0 && r < m) ? indicator(x[(int64_t)r * n], thr, sub) : 0; };
    int c = 0;
    for (int r = r0 - s1; r < r0 - s1 + s; r++) c += at(r);
    for (int r = r0; r < r1; r++) {
        if (r > r0) c += at(r - s1 + s - 1) - at(r - 1 - s1);
        o[(int64_t)r * n] = (double)c / (double)s;
    }
}

// scipy's axis-1 chain, one thread per (field, row)
__global__ void __launch_bounds__(THREADS)
    fss_pass1_kernel(const double *__restrict__ in, int64_t rows, int n, int s, double *__restrict__ out) {
    const int64_t row = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (row >= rows) return;
    const double *x = in + row * n;
    double *o = out + row * n;
    const int s1 = s / 2;
    auto pad = [&](int j) { return (j >= s1 && j - s1 < n) ? x[j - s1] : 0.0; };
    const double fs = (double)s;
    double tmp = 0.0;
    for (int j = 0; j < s; j++) tmp = tmp + pad(j);
    o[0] = tmp / fs;
    for (int l = 1; l < n; l++) {
        tmp = tmp + (pad(l + s - 1) - pad(l - 1));
        o[l] = tmp / fs;
    }
}

template <typename T>
int fractions_run(const T *X, int nf, int m, int n, double thr, double sub, int s, double *S, cudaStream_t st) {
    const int chunks = (m + ROW_CHUNK - 1) / ROW_CHUNK;
    B200_REQUIRE((int64_t)nf * chunks < 65536, "fss_fractions: too many fields");
    const dim3 grid((unsigned)b200::ceil_div64(n, THREADS), (unsigned)(nf * chunks));
    if (s <= 1) {
        fss_pass0_kernel<T><<<grid, THREADS, 0, st>>>(X, nf, m, n, thr, sub, s, S);
        B200_LAUNCH_CHECK();
        return 0;
    }
    b200::Scratch tmp;
    B200_CUDA(tmp.alloc(sizeof(double) * nf * (size_t)m * n, st));
    fss_pass0_kernel<T><<<grid, THREADS, 0, st>>>(X, nf, m, n, thr, sub, s, (double *)tmp.p);
    B200_LAUNCH_CHECK();
    const int64_t rows = (int64_t)nf * m;
    fss_pass1_kernel<<<(unsigned)b200::ceil_div64(rows, THREADS), THREADS, 0, st>>>((const double *)tmp.p, rows, n, s,
                                                                                   S);
    B200_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// the sums of products: one block per leaf slot of the pairwise tree of P values, every pair of the
// two groups of fields A = [a0, a0 + na), B = [b0, b0 + nb); pair (i, j) at heap + (i * nb + j) * H

__device__ __forceinline__ bool pair_wanted(int a0, int b0, int i, int j) { return a0 + i <= b0 + j; }

__global__ void __launch_bounds__(THREADS)
    fss_leaf_kernel(const double *__restrict__ S, int64_t P, int depth, int a0, int na, int b0, int nb, int64_t H,
                    double *__restrict__ heap) {
    __shared__ double sa[B200_FSS_GROUP][pw::LEAF], sb[B200_FSS_GROUP][pw::LEAF];
    const int64_t u = blockIdx.x;
    int64_t lo = 0, len = P;
    int level = 0;
    while (len > pw::LEAF) {
        const int64_t h = pw::left_len(len);
        if ((u >> (depth - 1 - level)) & 1) {
            lo += h;
            len -= h;
        } else {
            len = h;
        }
        level++;
    }
    const int below = depth - level;
    if (u & (((int64_t)1 << below) - 1)) return;  // the leftmost slot below a leaf sums it
    for (int t = threadIdx.x; t < na * pw::LEAF; t += THREADS) {
        const int i = t / pw::LEAF, e = t % pw::LEAF;
        if (e < len) sa[i][e] = S[(int64_t)(a0 + i) * P + lo + e];
    }
    for (int t = threadIdx.x; t < nb * pw::LEAF; t += THREADS) {
        const int j = t / pw::LEAF, e = t % pw::LEAF;
        if (e < len) sb[j][e] = S[(int64_t)(b0 + j) * P + lo + e];
    }
    __syncthreads();
    const int64_t node = ((int64_t)1 << level) - 1 + (u >> below);
    for (int p = threadIdx.x; p < na * nb; p += THREADS) {
        const int i = p / nb, j = p % nb;
        if (!pair_wanted(a0, b0, i, j)) continue;
        const double *x = sa[i], *y = sb[j];
        auto get = [x, y](int64_t e) { return x[e] * y[e]; };
        heap[p * H + node] = pw::leaf<double>(get, 0, len);
    }
}

// one block per pair: every internal node = left child + right child, deepest level first
__global__ void __launch_bounds__(THREADS)
    fss_combine_kernel(int64_t P, int depth, int a0, int b0, int nb, int64_t H, double *__restrict__ heap,
                       double *__restrict__ out) {
    const int p = blockIdx.x, i = p / nb, j = p % nb;
    if (!pair_wanted(a0, b0, i, j)) return;
    double *h = heap + p * H;
    for (int L = depth - 1; L >= 0; L--) {
        for (int64_t u = threadIdx.x; u < ((int64_t)1 << L); u += THREADS) {
            int64_t lo, len;
            if (!pw::node(P, L, u, &lo, &len) || len <= pw::LEAF) continue;
            const int64_t c = ((int64_t)1 << (L + 1)) - 1 + 2 * u;
            h[((int64_t)1 << L) - 1 + u] = h[c] + h[c + 1];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) out[p] = 0.0 + h[0];
}

}  // namespace

extern "C" int b200_fss_fractions(const void *X, int dtype, int nf, int m, int n, double thr, double sub, int s,
                                  double *S, void *stream) {
    B200_REQUIRE(nf >= 0 && m >= 0 && n >= 0 && s >= 0 && (int64_t)nf * m * n < ((int64_t)1 << 31),
                 "fss_fractions: bad arguments");
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if ((int64_t)nf * m * n == 0) return 0;
        B200_REQUIRE(X != nullptr && S != nullptr, "fss_fractions: bad arguments");
        return fractions_run<F>((const F *)X, nf, m, n, thr, sub, s, S, (cudaStream_t)stream);
    });
}

extern "C" int b200_fss_sums(const double *S, int64_t P, int a0, int na, int b0, int nb, double *out, void *stream) {
    B200_REQUIRE(P >= 0 && P < ((int64_t)1 << 31) && a0 >= 0 && b0 >= 0 && na >= 1 && nb >= 1 &&
                     na <= B200_FSS_GROUP && nb <= B200_FSS_GROUP && out != nullptr,
                 "fss_sums: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (P == 0) {
        B200_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * na * nb, st));
        return 0;
    }
    B200_REQUIRE(S != nullptr, "fss_sums: bad arguments");
    const int depth = pw::depth_bound(P);
    const int64_t H = ((int64_t)2 << depth) - 1;
    b200::Scratch heap;
    B200_CUDA(heap.alloc(sizeof(double) * H * na * nb, st));
    fss_leaf_kernel<<<(unsigned)((int64_t)1 << depth), THREADS, 0, st>>>(S, P, depth, a0, na, b0, nb, H,
                                                                         (double *)heap.p);
    B200_LAUNCH_CHECK();
    fss_combine_kernel<<<na * nb, THREADS, 0, st>>>(P, depth, a0, b0, nb, H, (double *)heap.p, out);
    B200_LAUNCH_CHECK();
    return 0;
}
