// verification.cu -- the ensemble and probability scores of pysteps/verification/probscores.py and
// ensscores.py on the device (sm_90a): the accumulation steps of CRPS, the rank histogram, the
// reliability diagram and the ROC curve.  One thread per pixel reads the (k, N) ensemble once in
// member order, coalesced across pixels:
//   crps      the masked pixel's k members sorted (in a local array up to 32 members, in an HBM scratch
//             plane above), its k + 1 alpha / beta terms
//             weighted by p^2 and (1 - p)^2 and summed pairwise (pairwise_body.cuh), then the
//             per-pixel sums compacted in pixel order for the pairwise sum over pixels
//   rankhist  the counts b1 = #{members < obs} and b2 = k - #{members > obs} after the X_min
//             substitution; an untied pixel counts in bin b1, a tied one is compacted in pixel order
//             so that the host's uniform draws reach it in the reference's order (rankhist_ties)
//   reldiag   np.digitize(P, edges, right=True) as a left binary search over the float64 edges, the
//             per-bin counts of obs >= X_min, and a stable counting sort of P by bin that the
//             pairwise sum then reduces bin by bin in P's dtype
//   roc       per pixel the number of thresholds <= P, histogrammed apart for events and
//             non-events; the host's suffix sums give the four counts of every threshold
// The compactions are stable block-chunked counting sorts: every block owns a contiguous chunk of
// pixels, counts its keys in shared memory, and scatters after one scan of the (key, block) counts.
// Counts are integers and no atomics touch floating-point values: repeated calls are bit-identical.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "pairwise_body.cuh"
#include "scan.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int SCAN_THREADS = 1024;

__device__ __forceinline__ bool finite(double v) { return isfinite(v); }

// ---------------------------------------------------------------------------------------------------
// stable partition of the pixels by key (-1: dropped), block-chunked

struct Chunks {
    int blocks;
    int64_t chunk;  // pixels per block, a multiple of THREADS
};

Chunks chunks_for(int64_t N) {
    const int64_t tiles = std::max<int64_t>(1, b200::ceil_div64(N, THREADS));
    const int blocks = (int)std::min<int64_t>(tiles, (int64_t)b200::num_sms() * 2);
    return {blocks, b200::ceil_div64(tiles, blocks) * THREADS};
}

// counts[key * gridDim.x + blockIdx.x] = the keys of the block's chunk
__global__ void __launch_bounds__(THREADS)
    part_count_kernel(const int *__restrict__ key, int64_t N, int nkeys, int64_t chunk, int *__restrict__ counts) {
    extern __shared__ int hist[];
    for (int i = threadIdx.x; i < nkeys; i += THREADS) hist[i] = 0;
    __syncthreads();
    const int64_t b0 = (int64_t)blockIdx.x * chunk, b1 = b0 + chunk < N ? b0 + chunk : N;
    for (int64_t pix = b0 + threadIdx.x; pix < b1; pix += THREADS) {
        const int c = key[pix];
        if (c >= 0) atomicAdd(hist + c, 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nkeys; i += THREADS) counts[(int64_t)i * gridDim.x + blockIdx.x] = hist[i];
}

// one block: offset[i] = the exclusive sum of counts[0..i); seg[key] = offset[key * blocks],
// seg[nkeys] = the total
__global__ void __launch_bounds__(SCAN_THREADS)
    part_scan_kernel(const int *__restrict__ counts, int64_t n, int blocks, int nkeys, int64_t *__restrict__ offset,
                     int64_t *__restrict__ seg) {
    const int64_t total = b200::single_cta_scan<SCAN_THREADS>(counts, n, offset);
    __syncthreads();  // seg is read from offsets that other threads wrote
    for (int key = threadIdx.x; key < nkeys; key += SCAN_THREADS) seg[key] = offset[(int64_t)key * blocks];
    if (threadIdx.x == 0) seg[nkeys] = total;
}

// out[offset of (key, block) + the pixel's rank among the earlier pixels of its key] = val[pix]
template <typename V>
__global__ void __launch_bounds__(THREADS)
    part_scatter_kernel(const int *__restrict__ key, const V *__restrict__ val, int64_t N, int nkeys, int64_t chunk,
                        const int64_t *__restrict__ offset, V *__restrict__ out) {
    extern __shared__ int run[];  // nkeys running counts, then THREADS keys of the tile
    int *tile = run + nkeys;
    for (int i = threadIdx.x; i < nkeys; i += THREADS) run[i] = 0;
    const int64_t b0 = (int64_t)blockIdx.x * chunk, b1 = b0 + chunk < N ? b0 + chunk : N;
    for (int64_t base = b0; base < b1; base += THREADS) {
        const int64_t pix = base + threadIdx.x;
        const int c = pix < b1 ? key[pix] : -1;
        tile[threadIdx.x] = c;
        __syncthreads();
        if (c >= 0) {
            int r = 0;
            for (int j = 0; j < (int)threadIdx.x; j++) r += tile[j] == c;
            out[offset[(int64_t)c * gridDim.x + blockIdx.x] + run[c] + r] = val[pix];
        }
        __syncthreads();
        if (c >= 0) atomicAdd(run + c, 1);
        __syncthreads();
    }
}

// seg[0..nkeys]: where every key's pixels start in out (seg[nkeys] = their total)
template <typename V>
int partition(const int *key, const V *val, int64_t N, int nkeys, V *out, int64_t *seg, cudaStream_t s) {
    const Chunks ch = chunks_for(N);
    const int64_t n = (int64_t)nkeys * ch.blocks;
    b200::Scratch counts, offsets;
    B200_CUDA(counts.alloc(sizeof(int) * n, s));
    B200_CUDA(offsets.alloc(sizeof(int64_t) * n, s));
    part_count_kernel<<<ch.blocks, THREADS, sizeof(int) * nkeys, s>>>(key, N, nkeys, ch.chunk, (int *)counts.p);
    B200_LAUNCH_CHECK();
    part_scan_kernel<<<1, SCAN_THREADS, 0, s>>>((const int *)counts.p, n, ch.blocks, nkeys, (int64_t *)offsets.p, seg);
    B200_LAUNCH_CHECK();
    part_scatter_kernel<V><<<ch.blocks, THREADS, sizeof(int) * (nkeys + THREADS), s>>>(
        key, val, N, nkeys, ch.chunk, (const int64_t *)offsets.p, out);
    B200_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// the pairwise sum of many segments: one thread per leaf, then the levels of every segment's tree

struct Segment {
    int64_t off, len;  // of the values
    int64_t thread0;   // the first of its 2^depth leaf threads
    int64_t heap;      // its nodes: level L, index u at heap + 2^L - 1 + u
    int depth;         // pw::depth_bound(len)
};

template <typename F>
__global__ void __launch_bounds__(THREADS)
    pw_leaf_kernel(const F *__restrict__ x, const Segment *__restrict__ seg, int nseg, int64_t threads,
                   F *__restrict__ heap) {
    const int64_t t = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (t >= threads) return;
    int a = 0, b = nseg - 1;  // the last segment whose thread0 <= t
    while (a < b) {
        const int m = (a + b + 1) / 2;
        if (seg[m].thread0 <= t) a = m;
        else b = m - 1;
    }
    const Segment sg = seg[a];
    const int64_t u = t - sg.thread0;
    // descend along u's bits until a leaf; the leftmost thread below a leaf sums it
    int64_t lo = 0, len = sg.len;
    int level = 0;
    while (len > pw::LEAF) {
        const int64_t h = pw::left_len(len);
        if ((u >> (sg.depth - 1 - level)) & 1) {
            lo += h;
            len -= h;
        } else {
            len = h;
        }
        level++;
    }
    const int below = sg.depth - level;
    if (u & (((int64_t)1 << below) - 1)) return;
    const F *v = x + sg.off;
    auto get = [v](int64_t i) { return v[i]; };
    heap[sg.heap + ((int64_t)1 << level) - 1 + (u >> below)] = pw::leaf<F>(get, lo, len);
}

// one block per segment: every internal node = left child + right child, deepest level first
template <typename F>
__global__ void __launch_bounds__(THREADS)
    pw_combine_kernel(const Segment *__restrict__ seg, F *__restrict__ heap, F *__restrict__ out) {
    const Segment sg = seg[blockIdx.x];
    F *h = heap + sg.heap;
    for (int L = sg.depth - 1; L >= 0; L--) {
        for (int64_t u = threadIdx.x; u < ((int64_t)1 << L); u += THREADS) {
            int64_t lo, len;
            if (!pw::node(sg.len, L, u, &lo, &len) || len <= pw::LEAF) continue;
            const int64_t c = ((int64_t)1 << (L + 1)) - 1 + 2 * u;
            h[((int64_t)1 << L) - 1 + u] = h[c] + h[c + 1];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) out[blockIdx.x] = F(0) + h[0];
}

template <typename F>
int pairwise_run(const F *x, const int64_t *off, const int64_t *len, int nseg, F *out, cudaStream_t s) {
    std::vector<Segment> tab(nseg);
    int64_t threads = 0, heap = 0;
    for (int i = 0; i < nseg; i++) {
        B200_REQUIRE(off[i] >= 0 && len[i] >= 0, "pairwise_sum: bad segment");
        const int d = pw::depth_bound(len[i]);
        tab[i] = {off[i], len[i], threads, heap, d};
        threads += (int64_t)1 << d;
        heap += ((int64_t)2 << d) - 1;
    }
    b200::Scratch d_tab, d_heap;
    B200_CUDA(d_tab.alloc(sizeof(Segment) * nseg, s));
    B200_CUDA(d_heap.alloc(sizeof(F) * heap, s));
    B200_CUDA(cudaMemcpyAsync(d_tab.p, tab.data(), sizeof(Segment) * nseg, cudaMemcpyHostToDevice, s));
    const Segment *t = (const Segment *)d_tab.p;
    pw_leaf_kernel<F><<<(unsigned)b200::ceil_div64(threads, THREADS), THREADS, 0, s>>>(x, t, nseg, threads,
                                                                                       (F *)d_heap.p);
    B200_LAUNCH_CHECK();
    pw_combine_kernel<F><<<nseg, THREADS, 0, s>>>(t, (F *)d_heap.p, out);
    B200_LAUNCH_CHECK();
    // the host table must outlive the copy: it was staged before cudaMemcpyAsync returned (pageable)
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// CRPS

// the sorted members of a pixel: a local array of at most LOCAL_MEMBERS values, or for larger k the
// pixel's column of a (k, N) scratch plane in HBM, coalesced across pixels like X (a local array of
// B200_VERIF_MAX_MEMBERS doubles would need 4 KB of local memory for every resident thread)
constexpr int LOCAL_MEMBERS = 32;

template <typename F>
struct LocalMembers {
    F v[LOCAL_MEMBERS];
    __device__ LocalMembers(F *, int64_t, int64_t) {}
    __device__ F &operator[](int i) { return v[i]; }
};

template <typename F>
struct ScratchMembers {
    F *p;
    int64_t stride;
    __device__ ScratchMembers(F *scratch, int64_t pix, int64_t N) : p(scratch + pix), stride(N) {}
    __device__ F &operator[](int i) { return p[(int64_t)i * stride]; }
};

// key[pix] = 0 where every member and the observation are finite (res[pix] = the pixel's sum of
// alpha p^2 + beta (1 - p)^2 over the k + 1 columns), -1 elsewhere
template <typename F, typename O, typename Members>
__global__ void __launch_bounds__(THREADS)
    crps_kernel(const F *__restrict__ X, const O *__restrict__ obs, int k, int64_t N, F *scratch,
                double *__restrict__ res, int *__restrict__ key) {
    using P = typename b200::Promote<F, O>::T;
    const int64_t pix = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (pix >= N) return;
    const O o = obs[pix];
    bool in = finite((double)o);
    Members x(scratch, pix, N);
    for (int i = 0; i < k; i++) {
        const F v = __ldg(X + (int64_t)i * N + pix);
        in = in && finite((double)v);
        // insertion sort; equal values (+0 and -0 included) give the same differences in any order
        int j = i;
        while (j > 0 && x[j - 1] > v) {
            x[j] = x[j - 1];
            j--;
        }
        x[j] = v;
    }
    key[pix] = in ? 0 : -1;
    if (!in) return;
    const double od = (double)o;
    auto term = [&](int64_t c) -> double {
        double alpha = 0.0, beta = 0.0;
        const int i = (int)c;
        if (i >= 1 && i < k) {
            const double xi = (double)x[i], xm = (double)x[i - 1];
            if (od > xi) {
                alpha = (double)(F)(x[i] - x[i - 1]);
                beta = 0.0;
            }
            if (xi > od && od > xm) {
                alpha = (double)((P)o - (P)x[i - 1]);
                beta = (double)((P)x[i] - (P)o);
            }
            if (od < xm) {
                alpha = 0.0;
                beta = (double)(F)(x[i] - x[i - 1]);
            }
        }
        if (i == 0 && od < (double)x[0]) {
            alpha = 0.0;
            beta = (double)((P)x[0] - (P)o);
        }
        if (i == k && (double)x[k - 1] < od) {
            alpha = (double)((P)o - (P)x[k - 1]);
            beta = 0.0;
        }
        const double p = (double)i / (double)k, q = 1.0 - p;
        return alpha * (p * p) + beta * (q * q);
    };
    res[pix] = pw::pairwise_sum<double, 4>(term, (int64_t)k + 1);
}

template <typename F, typename O>
int crps_run(const F *X, const O *obs, int k, int64_t N, double *res, int64_t *n, cudaStream_t s) {
    b200::Scratch keys, vals, seg;
    B200_CUDA(keys.alloc(sizeof(int) * N, s));
    B200_CUDA(vals.alloc(sizeof(double) * N, s));
    B200_CUDA(seg.alloc(sizeof(int64_t) * 2, s));
    const unsigned grid = (unsigned)b200::ceil_div64(N, THREADS);
    int *key = (int *)keys.p;
    double *v = (double *)vals.p;
    b200::Scratch members;
    if (k <= LOCAL_MEMBERS) {
        crps_kernel<F, O, LocalMembers<F>><<<grid, THREADS, 0, s>>>(X, obs, k, N, nullptr, v, key);
    } else {
        B200_CUDA(members.alloc(sizeof(F) * k * N, s));
        crps_kernel<F, O, ScratchMembers<F>><<<grid, THREADS, 0, s>>>(X, obs, k, N, (F *)members.p, v, key);
    }
    B200_LAUNCH_CHECK();
    if (int rc = partition<double>(key, v, N, 1, res, (int64_t *)seg.p, s)) return rc;
    B200_CUDA(cudaMemcpyAsync(n, (int64_t *)seg.p + 1, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// rank histogram

// untied masked pixels counted into hist[b1]; a tied one gets key 0 and (b1, b2) for the compaction
template <typename F, typename O>
__global__ void __launch_bounds__(THREADS)
    rankhist_kernel(const F *__restrict__ X, const O *__restrict__ obs, int k, int64_t N, int use_min, double thr_f,
                    F sub_f, double thr_o, O sub_o, unsigned long long *__restrict__ hist, int2 *__restrict__ pair,
                    int *__restrict__ key) {
    extern __shared__ int h[];  // k + 1 bins
    for (int i = threadIdx.x; i <= k; i += THREADS) h[i] = 0;
    __syncthreads();
    const int64_t pix = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (pix < N) {
        O o = obs[pix];
        bool in = finite((double)o), nz = !use_min || (double)o >= thr_o;
        for (int i = 0; i < k; i++) {
            const double v = (double)__ldg(X + (int64_t)i * N + pix);
            in = in && finite(v);
            nz = nz || v >= thr_f;
        }
        int c = -1;
        if (in && nz) {
            if (use_min && (double)o < thr_o) o = sub_o;
            const double od = (double)o;
            int below = 0, above = 0;
            for (int i = 0; i < k; i++) {
                F v = __ldg(X + (int64_t)i * N + pix);
                if (use_min && (double)v < thr_f) v = sub_f;
                below += (double)v < od;
                above += (double)v > od;
            }
            if (below + above == k) {
                atomicAdd(h + below, 1);
            } else {
                c = 0;
                pair[pix] = make_int2(below, k - above);
            }
        }
        key[pix] = c;
    }
    __syncthreads();
    for (int i = threadIdx.x; i <= k; i += THREADS)
        if (h[i]) atomicAdd(hist + i, (unsigned long long)h[i]);
}

// the tied pixel j goes to bin int(b1 + u[j] * (b2 + 1 - b1))
__global__ void __launch_bounds__(THREADS)
    rankhist_ties_kernel(const int2 *__restrict__ pair, int64_t n, const double *__restrict__ u,
                         unsigned long long *__restrict__ hist) {
    const int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (j >= n) return;
    const int2 b = pair[j];
    const double r = (double)b.x + u[j] * (double)(b.y + 1 - b.x);
    atomicAdd(hist + (int64_t)r, 1ull);
}

template <typename F, typename O>
int rankhist_run(const F *X, const O *obs, int k, int64_t N, int use_min, double thr_f, double sub_f, double thr_o,
                 double sub_o, int64_t *hist, void *ties, int64_t *n_ties, cudaStream_t s) {
    b200::Scratch keys, pairs, seg;
    B200_CUDA(keys.alloc(sizeof(int) * N, s));
    B200_CUDA(pairs.alloc(sizeof(int2) * N, s));
    B200_CUDA(seg.alloc(sizeof(int64_t) * 2, s));
    B200_CUDA(cudaMemsetAsync(hist, 0, sizeof(int64_t) * (k + 1), s));
    rankhist_kernel<F, O><<<(unsigned)b200::ceil_div64(N, THREADS), THREADS, sizeof(int) * (k + 1), s>>>(
        X, obs, k, N, use_min, thr_f, (F)sub_f, thr_o, (O)sub_o, (unsigned long long *)hist, (int2 *)pairs.p,
        (int *)keys.p);
    B200_LAUNCH_CHECK();
    if (int rc = partition<int2>((const int *)keys.p, (const int2 *)pairs.p, N, 1, (int2 *)ties, (int64_t *)seg.p, s))
        return rc;
    B200_CUDA(cudaMemcpyAsync(n_ties, (int64_t *)seg.p + 1, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// reliability diagram and ROC curve

// the number of the n sorted values t[] that are < v (side "left") or <= v (side "right")
__device__ __forceinline__ int count_below(const double *t, int n, double v, bool or_equal) {
    int a = 0, b = n;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (or_equal ? t[m] <= v : t[m] < v) a = m + 1;
        else b = m;
    }
    return a;
}

// key[pix] = bin - 1 for the finite pairs whose bin is in 1..n_edges - 1, else -1; above[bin - 1] +=
// obs >= thr_o
template <typename F, typename O>
__global__ void __launch_bounds__(THREADS)
    reldiag_kernel(const F *__restrict__ P, const O *__restrict__ obs, int64_t N, const double *__restrict__ edges,
                   int n_edges, double thr_o, unsigned long long *__restrict__ above, int *__restrict__ key) {
    extern __shared__ double e[];  // n_edges edges, then n_edges - 1 counts
    int *cnt = (int *)(e + n_edges);
    for (int i = threadIdx.x; i < n_edges; i += THREADS) e[i] = edges[i];
    for (int i = threadIdx.x; i < n_edges - 1; i += THREADS) cnt[i] = 0;
    __syncthreads();
    const int64_t pix = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (pix < N) {
        const double p = (double)P[pix], o = (double)obs[pix];
        int c = -1;
        if (finite(p) && finite(o)) {
            const int bin = count_below(e, n_edges, p, false);
            if (bin >= 1 && bin < n_edges) {
                c = bin - 1;
                if (o >= thr_o) atomicAdd(cnt + c, 1);
            }
        }
        key[pix] = c;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_edges - 1; i += THREADS)
        if (cnt[i]) atomicAdd(above + i, (unsigned long long)cnt[i]);
}

template <typename F, typename O>
int reldiag_run(const F *P, const O *obs, int64_t N, const double *edges, int n_edges, double thr_o, F *sorted,
                int64_t *seg, int64_t *above, cudaStream_t s) {
    const int nb = n_edges - 1;
    B200_CUDA(cudaMemsetAsync(above, 0, sizeof(int64_t) * std::max(nb, 1), s));
    b200::Scratch d_edges, keys;
    B200_CUDA(d_edges.alloc(sizeof(double) * n_edges, s));
    B200_CUDA(keys.alloc(sizeof(int) * N, s));
    B200_CUDA(cudaMemcpyAsync(d_edges.p, edges, sizeof(double) * n_edges, cudaMemcpyHostToDevice, s));
    const size_t shm = sizeof(double) * n_edges + sizeof(int) * std::max(nb, 1);
    reldiag_kernel<F, O><<<(unsigned)b200::ceil_div64(N, THREADS), THREADS, shm, s>>>(
        P, obs, N, (const double *)d_edges.p, n_edges, thr_o, (unsigned long long *)above, (int *)keys.p);
    B200_LAUNCH_CHECK();
    if (nb == 0) {
        B200_CUDA(cudaMemsetAsync(seg, 0, sizeof(int64_t), s));
        return 0;
    }
    return partition<F>((const int *)keys.p, P, N, nb, sorted, seg, s);
}

// counts[c] (events) and counts[n_thr + 1 + c] (non-events) += the finite pairs with c thresholds <= P
template <typename F, typename O>
__global__ void __launch_bounds__(THREADS)
    roc_kernel(const F *__restrict__ P, const O *__restrict__ obs, int64_t N, const double *__restrict__ thr, int n_thr,
               double thr_o, unsigned long long *__restrict__ counts) {
    extern __shared__ double t[];  // n_thr thresholds, then 2 (n_thr + 1) counts
    int *cnt = (int *)(t + n_thr);
    for (int i = threadIdx.x; i < n_thr; i += THREADS) t[i] = thr[i];
    for (int i = threadIdx.x; i < 2 * (n_thr + 1); i += THREADS) cnt[i] = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * THREADS;
    for (int64_t pix = (int64_t)blockIdx.x * THREADS + threadIdx.x; pix < N; pix += stride) {
        const double p = (double)P[pix], o = (double)obs[pix];
        if (finite(p) && finite(o)) {
            const int c = count_below(t, n_thr, p, true);
            atomicAdd(cnt + (o >= thr_o ? 0 : n_thr + 1) + c, 1);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * (n_thr + 1); i += THREADS)
        if (cnt[i]) atomicAdd(counts + i, (unsigned long long)cnt[i]);
}

template <typename F, typename O>
int roc_run(const F *P, const O *obs, int64_t N, const double *thr, int n_thr, double thr_o, int64_t *counts,
            cudaStream_t s) {
    B200_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * 2 * (n_thr + 1), s));
    b200::Scratch d_thr;
    B200_CUDA(d_thr.alloc(sizeof(double) * std::max(n_thr, 1), s));
    if (n_thr) B200_CUDA(cudaMemcpyAsync(d_thr.p, thr, sizeof(double) * n_thr, cudaMemcpyHostToDevice, s));
    const int blocks = (int)std::min<int64_t>(b200::ceil_div64(N, THREADS), (int64_t)b200::num_sms() * 8);
    const size_t shm = sizeof(double) * n_thr + sizeof(int) * 2 * (n_thr + 1);
    roc_kernel<F, O><<<blocks, THREADS, shm, s>>>(P, obs, N, (const double *)d_thr.p, n_thr, thr_o,
                                                  (unsigned long long *)counts);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int b200_pairwise_sum(const void *x, int dtype, const int64_t *seg_off, const int64_t *seg_len, int nseg,
                                 void *out, void *stream) {
    B200_REQUIRE(nseg >= 0, "pairwise_sum: bad arguments");
    return b200::with_dtype("field", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        if (nseg == 0) return 0;
        B200_REQUIRE(seg_off != nullptr && seg_len != nullptr && out != nullptr, "pairwise_sum: bad arguments");
        return pairwise_run<F>((const F *)x, seg_off, seg_len, nseg, (F *)out, (cudaStream_t)stream);
    });
}

extern "C" int b200_verif_crps(const void *Xf, int f_dtype, const void *Xo, int o_dtype, int k, int64_t N,
                               double *res, int64_t *n, void *stream) {
    B200_REQUIRE(k >= 1 && k <= B200_VERIF_MAX_MEMBERS && N >= 0 && N < ((int64_t)1 << 31) && n != nullptr,
                 "verif_crps: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(f_dtype, o_dtype, [&](auto tf, auto to) {
        using F = typename decltype(tf)::type;
        using O = typename decltype(to)::type;
        if (N == 0) {
            B200_CUDA(cudaMemsetAsync(n, 0, sizeof(int64_t), s));
            return 0;
        }
        B200_REQUIRE(Xf != nullptr && Xo != nullptr && res != nullptr, "verif_crps: bad arguments");
        return crps_run<F, O>((const F *)Xf, (const O *)Xo, k, N, res, n, s);
    });
}

extern "C" int b200_verif_rankhist(const void *Xf, int f_dtype, const void *Xo, int o_dtype, int k, int64_t N,
                                   int use_min, double thr_f, double sub_f, double thr_o, double sub_o,
                                   int64_t *hist, void *ties, int64_t *n_ties, void *stream) {
    B200_REQUIRE(k >= 1 && k <= B200_VERIF_MAX_MEMBERS && N >= 0 && N < ((int64_t)1 << 31) && hist != nullptr &&
                     n_ties != nullptr,
                 "verif_rankhist: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(f_dtype, o_dtype, [&](auto tf, auto to) {
        using F = typename decltype(tf)::type;
        using O = typename decltype(to)::type;
        if (N == 0) {
            B200_CUDA(cudaMemsetAsync(hist, 0, sizeof(int64_t) * (k + 1), s));
            B200_CUDA(cudaMemsetAsync(n_ties, 0, sizeof(int64_t), s));
            return 0;
        }
        B200_REQUIRE(Xf != nullptr && Xo != nullptr && ties != nullptr, "verif_rankhist: bad arguments");
        return rankhist_run<F, O>((const F *)Xf, (const O *)Xo, k, N, use_min, thr_f, sub_f, thr_o, sub_o, hist, ties,
                                  n_ties, s);
    });
}

extern "C" int b200_verif_rankhist_ties(const void *ties, int64_t n_ties, const double *u, int k, int64_t *hist,
                                        void *stream) {
    B200_REQUIRE(n_ties >= 0 && k >= 1 && hist != nullptr, "verif_rankhist_ties: bad arguments");
    if (n_ties == 0) return 0;
    B200_REQUIRE(ties != nullptr && u != nullptr, "verif_rankhist_ties: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    rankhist_ties_kernel<<<(unsigned)b200::ceil_div64(n_ties, THREADS), THREADS, 0, s>>>(
        (const int2 *)ties, n_ties, u, (unsigned long long *)hist);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_verif_reldiag(const void *P, int p_dtype, const void *Xo, int o_dtype, int64_t N,
                                  const double *edges, int n_edges, double thr_o, void *sorted, int64_t *seg,
                                  int64_t *above, void *stream) {
    B200_REQUIRE(N >= 0 && N < ((int64_t)1 << 31) && n_edges >= 1 && n_edges <= B200_VERIF_MAX_BINS + 1 &&
                     edges != nullptr && seg != nullptr && above != nullptr,
                 "verif_reldiag: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(p_dtype, o_dtype, [&](auto tp, auto to) {
        using F = typename decltype(tp)::type;
        using O = typename decltype(to)::type;
        if (N == 0) {
            B200_CUDA(cudaMemsetAsync(seg, 0, sizeof(int64_t) * n_edges, s));
            B200_CUDA(cudaMemsetAsync(above, 0, sizeof(int64_t) * std::max(n_edges - 1, 1), s));
            return 0;
        }
        B200_REQUIRE(P != nullptr && Xo != nullptr && sorted != nullptr, "verif_reldiag: bad arguments");
        return reldiag_run<F, O>((const F *)P, (const O *)Xo, N, edges, n_edges, thr_o, (F *)sorted, seg, above, s);
    });
}

extern "C" int b200_verif_roc(const void *P, int p_dtype, const void *Xo, int o_dtype, int64_t N, const double *thr,
                              int n_thr, double thr_o, int64_t *counts, void *stream) {
    B200_REQUIRE(N >= 0 && N < ((int64_t)1 << 31) && n_thr >= 0 && n_thr <= B200_VERIF_MAX_BINS &&
                     counts != nullptr && (n_thr == 0 || thr != nullptr),
                 "verif_roc: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(p_dtype, o_dtype, [&](auto tp, auto to) {
        using F = typename decltype(tp)::type;
        using O = typename decltype(to)::type;
        if (N == 0) {
            B200_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * 2 * (n_thr + 1), s));
            return 0;
        }
        B200_REQUIRE(P != nullptr && Xo != nullptr, "verif_roc: bad arguments");
        return roc_run<F, O>((const F *)P, (const O *)Xo, N, thr, n_thr, thr_o, counts, s);
    });
}
