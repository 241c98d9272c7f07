// knn.cu -- scipy.spatial.cKDTree's neighbour order on the device, for the two k-NN stages of
// dense_lucaskanade: the local outlier test (pysteps/utils/cleansing.py:216-245) and the
// inverse-distance grid fill (pysteps/utils/interpolate.py:67-114).
//
// Corner coordinates are integers (declustered ones multiples of 1/2), so equidistant and
// coincident vectors are common, and WHICH of the tied vectors cKDTree returns is a property of
// its tree: median splits by libstdc++'s std::nth_element, best-first search with scipy's own
// binary heaps (knn_body.cuh restates both; DESIGN.md section 4).  The reference's results depend
// on that order, so the tree is rebuilt here exactly:
//
//   kd_build_kernel    one CTA, the whole point set in shared memory as position-aligned
//                      (x, y, index) triples.  Tree levels are processed breadth-first, one WARP
//                      per node: bounds by shuffle reductions, and the two sequential partition
//                      loops of the build (introselect's unguarded partition, scipy's
//                      partition_below) executed as ballot-ranked PAIR SWAPS -- the i-th position
//                      where the left scan stops trades places with the i-th position where the
//                      right scan stops, for every i before the scans cross.  That is the same
//                      permutation the sequential loops produce (knn_body.cuh: build_pairs is the
//                      serial statement of it, pinned against scipy on the host), at ~n/32 steps per
//                      pass instead of n.
//   outliers_warp_kernel  one warp per vector: scipy's query for its k+1 nearest, then the
//                      Mahalanobis test on them.
//   idw_fix_kernel     the grid fill's exhaustive tile search (idw.cu) is order-free except where
//                      the k-th and (k+1)-th neighbour are exactly equidistant; those grid points
//                      (~0.1 %) are listed by idw.cu and recomputed here from scipy's query.
#include "common.cuh"
#include "knn_body.cuh"
#include "knn_device.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;

struct BuildSmem {
    double kx[kdp::NMAX], ky[kdp::NMAX];
    int idx[kdp::NMAX];
    unsigned short posA[kdp::NMAX], posB[kdp::NMAX];
    int queue[2][kdp::QCAP];  // node ids of the level being split / the next one
    int qn[2];
    int nnodes;
};

__device__ __forceinline__ void swap3(BuildSmem &s, int p, int q) {
    const double x = s.kx[p], y = s.ky[p];
    const int i = s.idx[p];
    s.kx[p] = s.kx[q]; s.ky[p] = s.ky[q]; s.idx[p] = s.idx[q];
    s.kx[q] = x; s.ky[q] = y; s.idx[q] = i;
}

// knn_body.cuh pair_partition_serial, one warp: ranks by ballot, swaps in parallel.
template <int MODE>
__device__ int warp_pair_partition(BuildSmem &s, const double *K, int lo, int hi, double piv, int lane) {
    const unsigned lt = (1u << lane) - 1u;
    int cntA = 0, cntB = 0;
    for (int c = lo; c < hi; c += 32) {
        const int p = c + lane;
        const bool a = p < hi && !(K[p] < piv);
        const unsigned bal = __ballot_sync(FULL, a);
        if (a) s.posA[lo + cntA + __popc(bal & lt)] = (unsigned short)p;
        cntA += __popc(bal);
    }
    for (int c = hi - 1; c >= lo; c -= 32) {
        const int p = c - lane;
        const bool b = p >= lo && (MODE == 0 ? !(piv < K[p]) : !(K[p] >= piv));
        const unsigned bal = __ballot_sync(FULL, b);
        if (b) s.posB[lo + cntB + __popc(bal & lt)] = (unsigned short)p;
        cntB += __popc(bal);
    }
    __syncwarp();
    const int npair = min(cntA, cntB);
    int j = 0;
    for (int c = 0; c < npair; c += 32) {
        const int i = c + lane;
        const bool ok = i < npair && s.posA[lo + i] < s.posB[lo + i];
        const unsigned bal = __ballot_sync(FULL, ok);
        if (ok) swap3(s, s.posA[lo + i], s.posB[lo + i]);
        j += __popc(bal);
        if (bal != FULL) break;  // A ascends, B descends: the first failure is final
    }
    __syncwarp();
    if (MODE == 1) return hi - cntA;
    const int fa = j < cntA ? (int)s.posA[lo + j] : hi, fb = j > 0 ? (int)s.posB[lo + j - 1] : hi;
    return min(fa, fb);
}

// std::nth_element(first, nth, last) on the triples, comparing dimension d (libstdc++ introselect)
__device__ void warp_nth_element(BuildSmem &s, int d, int first, int nth, int last, int lane) {
    const double *K = d ? s.ky : s.kx;
    kd::Tri tri;
    tri.kx = s.kx; tri.ky = s.ky; tri.idx = s.idx;
    int depth = 0;
    for (int m = last - first; m > 1; m >>= 1) depth++;
    depth *= 2;
    while (last - first > 3) {
        if (depth == 0) {  // introselect gives up on quickselect: heap-select, sequential
            if (lane == 0) {
                kd::tri_heap_select(tri, first, nth + 1, last, d);
                kd::tri_swap(tri, first, nth);
            }
            __syncwarp();
            return;
        }
        depth--;
        const int mid = first + (last - first) / 2;
        if (lane == 0) swap3(s, first, kd::tri_median_pick(K, first, mid, last));
        __syncwarp();
        const int cut = warp_pair_partition<0>(s, K, first + 1, last, K[first], lane);
        if (cut <= nth) first = cut; else last = cut;
    }
    if (lane == 0) kd::tri_insertion_sort(tri, first, last, d);
    __syncwarp();
}

__device__ __forceinline__ void write_leaf(kd::Node *nodes, int id, int start, int end) {
    kd::Node nd;
    nd.split_dim = -1; nd.less = -1; nd.greater = -1; nd.start = start; nd.end = end; nd.split = 0.0;
    nodes[id] = nd;
}

__global__ void __launch_bounds__(32 * kdp::WARPS)
kd_build_kernel(const double *__restrict__ xy, const int *__restrict__ n_dev, int n_cap, kdp::TreeBuf tb) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    BuildSmem &s = *reinterpret_cast<BuildSmem *>(smem_raw);
    const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < n; i += blockDim.x) {
        s.kx[i] = xy[2 * (size_t)i];
        s.ky[i] = xy[2 * (size_t)i + 1];
        s.idx[i] = i;
    }
    if (tid == 0) {
        s.nnodes = 1;
        s.qn[0] = n > kd::LEAFSIZE ? 1 : 0;
        s.qn[1] = 0;
        s.queue[0][0] = 0;
        write_leaf(tb.nodes, 0, 0, n);
    }
    __syncthreads();
    if (wid == 0) {  // bounds of the whole set (tree.maxes / tree.mins)
        double mx0 = n ? s.kx[0] : 0.0, mn0 = mx0, mx1 = n ? s.ky[0] : 0.0, mn1 = mx1;
        for (int i = lane; i < n; i += 32) {
            mx0 = fmax(mx0, s.kx[i]); mn0 = fmin(mn0, s.kx[i]);
            mx1 = fmax(mx1, s.ky[i]); mn1 = fmin(mn1, s.ky[i]);
        }
        for (int o = 16; o > 0; o >>= 1) {
            mx0 = fmax(mx0, __shfl_xor_sync(FULL, mx0, o)); mn0 = fmin(mn0, __shfl_xor_sync(FULL, mn0, o));
            mx1 = fmax(mx1, __shfl_xor_sync(FULL, mx1, o)); mn1 = fmin(mn1, __shfl_xor_sync(FULL, mn1, o));
        }
        if (lane == 0) { tb.bounds[0] = mx0; tb.bounds[1] = mx1; tb.bounds[2] = mn0; tb.bounds[3] = mn1; }
    }
    int cur = 0;
    for (;;) {
        const int cnt = s.qn[cur];
        if (cnt == 0) break;
        for (int w = wid; w < cnt; w += kdp::WARPS) {
            const int me = s.queue[cur][w];
            const int start = tb.nodes[me].start, end = tb.nodes[me].end;
            double mx0 = s.kx[start], mn0 = mx0, mx1 = s.ky[start], mn1 = mx1;
            for (int i = start + lane; i < end; i += 32) {
                mx0 = fmax(mx0, s.kx[i]); mn0 = fmin(mn0, s.kx[i]);
                mx1 = fmax(mx1, s.ky[i]); mn1 = fmin(mn1, s.ky[i]);
            }
            for (int o = 16; o > 0; o >>= 1) {
                mx0 = fmax(mx0, __shfl_xor_sync(FULL, mx0, o)); mn0 = fmin(mn0, __shfl_xor_sync(FULL, mn0, o));
                mx1 = fmax(mx1, __shfl_xor_sync(FULL, mx1, o)); mn1 = fmin(mn1, __shfl_xor_sync(FULL, mn1, o));
            }
            // split dimension: the larger extent, the first on a tie; no extent: the node stays a leaf
            int d = 0;
            double size = 0.0;
            if (mx0 - mn0 > size) { d = 0; size = mx0 - mn0; }
            if (mx1 - mn1 > size) { d = 1; size = mx1 - mn1; }
            if ((d ? mx1 : mx0) == (d ? mn1 : mn0)) continue;
            const double *K = d ? s.ky : s.kx;
            const int nth = start + (end - start) / 2;
            warp_nth_element(s, d, start, nth, end, lane);
            double split = K[nth];
            int p = warp_pair_partition<1>(s, K, start, end, split, lane);
            if (p == start) {  // the median is the minimum: the split moves just above it
                split = nextafter(split, (double)INFINITY);
                p = warp_pair_partition<1>(s, K, start, end, split, lane);
            }
            if (lane == 0) {
                const int lo = atomicAdd(&s.nnodes, 2), hi = lo + 1;
                write_leaf(tb.nodes, lo, start, p);
                write_leaf(tb.nodes, hi, p, end);
                kd::Node nd;
                nd.split_dim = d; nd.less = lo; nd.greater = hi; nd.start = start; nd.end = end; nd.split = split;
                tb.nodes[me] = nd;
                if (p - start > kd::LEAFSIZE) s.queue[cur ^ 1][atomicAdd(&s.qn[cur ^ 1], 1)] = lo;
                if (end - p > kd::LEAFSIZE) s.queue[cur ^ 1][atomicAdd(&s.qn[cur ^ 1], 1)] = hi;
            }
        }
        __syncthreads();
        if (tid == 0) s.qn[cur] = 0;
        cur ^= 1;
        __syncthreads();
    }
    for (int i = tid; i < n; i += blockDim.x) tb.idx[i] = s.idx[i];
    if (tid == 0) {
        tb.meta[0] = s.nnodes;
        tb.meta[1] = n;
        tb.meta[2] = 0;  // next free entry of the overflow arena
    }
}

// more than NMAX points: the sequential restatement, one thread (slow; not a dense_lucaskanade size)
__global__ void kd_build_serial_kernel(const double *__restrict__ xy, const int *__restrict__ n_dev, int n_cap,
                                       kdp::TreeBuf tb) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const int n = n_dev ? min(*n_dev, n_cap) : n_cap;
    int stack[128];
    kd::Tree t;
    t.data = xy;
    t.n = n;
    t.idx = tb.idx;
    t.nodes = tb.nodes;
    kd::build(t, stack);
    tb.meta[0] = t.nnodes;
    tb.meta[1] = n;
    tb.meta[2] = 0;
    for (int c = 0; c < 2; c++) {
        tb.bounds[c] = t.maxes[c];
        tb.bounds[2 + c] = t.mins[c];
    }
}

// ---- one WARP per query -----------------------------------------------------------------------
// A best-first search is one long dependent chain (heap sifts); threads of a warp running 32
// different searches diverge at every branch and each pays for all (measured: 380 us for 1000
// searches).  Here a warp runs ONE search: every lane executes the scalar control flow on the same
// values (uniform, no divergence), lane 0 alone writes the heaps in shared memory, and the lanes
// share the one data-parallel part -- the distances of a leaf's points.  The order of every
// comparison, push and pop is scipy's (knn_body.cuh: query states it serially; the GPU tests pin
// both against the oracle); the heap sifts carry the moving element in a register instead of
// swapping, which visits the same positions with the same comparisons.
constexpr int QW = 4;  // warps (queries in flight) per CTA

struct WarpScratch {
    kd::NodeInfo q[kdp::QHEAP];
    kd::Item nb[kdp::NBSMEM];
    double w[kdp::NBSMEM];
    int inds[kdp::NBSMEM];
};

template <class T>
__device__ __forceinline__ void wheap_push(T *h, int &n, const T &it, int lane) {
    int i = n++;
    while (i > 0 && kd::prio(it) < kd::prio(h[(i - 1) / 2])) {
        if (lane == 0) h[i] = h[(i - 1) / 2];
        i = (i - 1) / 2;
    }
    if (lane == 0) h[i] = it;
    __syncwarp();
}

template <class T>
__device__ __forceinline__ void wheap_remove(T *h, int &n, int lane) {
    const T it = h[n - 1];
    n--;
    int i = 0, j = 1, k = 2;
    while ((j < n && kd::prio(it) > kd::prio(h[j])) || (k < n && kd::prio(it) > kd::prio(h[k]))) {
        const int l = (k < n && kd::prio(h[j]) > kd::prio(h[k])) ? k : j;
        if (lane == 0) h[i] = h[l];
        i = l;
        j = 2 * i + 1;
        k = 2 * i + 2;
    }
    if (lane == 0 && n > 0) h[i] = it;
    __syncwarp();
}

// kd::query for one warp; out_idx / out_dist in shared memory.  Returns with the results visible
// to every lane.
__device__ void warp_query(const kd::Tree &t, const kdp::TreeBuf &tb, double x0, double x1, int kmax,
                           WarpScratch &ws, bool want_dist, int lane) {
    kd::NodeInfo *q = ws.q;
    kd::Item *nb = ws.nb;
    int qcap = kdp::QHEAP;
    const double x[2] = {x0, x1};
    int nbn = 0, qn = 0;
    kd::NodeInfo cur;
    cur.node = 0;
    cur.min_distance = 0.0;
    for (int c = 0; c < 2; c++) {
        double s = x[c] - t.maxes[c];
        const double s2 = t.mins[c] - x[c];
        if (s2 > s) s = s2;
        if (s < 0.0) s = 0.0;
        cur.side[c] = s * s;
        cur.min_distance += cur.side[c];
    }
    double dub = (double)INFINITY;
    for (;;) {
        const kd::Node node = t.nodes[cur.node];
        if (node.split_dim == -1) {
            for (int base = node.start; base < node.end; base += 32) {
                const int i = base + lane;
                const bool valid = i < node.end;
                int pi = 0;
                double d = (double)INFINITY;
                if (valid) {
                    pi = t.idx[i];
                    const double dx = t.data[2 * (size_t)pi] - x[0], dy = t.data[2 * (size_t)pi + 1] - x[1];
                    d = 0.0;
                    d += dx * dx;
                    d += dy * dy;
                }
                // candidates against the bound as it stands; each is re-tested in index order
                // against the bound as the sequential loop would have it by then
                unsigned m = __ballot_sync(FULL, valid && d < dub);
                while (m) {
                    const int l = __ffs(m) - 1;
                    m &= m - 1;
                    const double dl = __shfl_sync(FULL, d, l);
                    const int pl = __shfl_sync(FULL, pi, l);
                    if (dl < dub) {
                        if (nbn == kmax) wheap_remove(nb, nbn, lane);
                        kd::Item it;
                        it.priority = -dl;
                        it.payload = pl;
                        wheap_push(nb, nbn, it, lane);
                        if (nbn == kmax) dub = -nb[0].priority;
                    }
                }
            }
            if (qn == 0) break;
            cur = q[0];
            wheap_remove(q, qn, lane);
        } else {
            if (cur.min_distance > dub) break;
            const int sd = node.split_dim;
            kd::NodeInfo far = cur;
            double s;
            if (x[sd] < node.split) {
                cur.node = node.less;
                far.node = node.greater;
                s = node.split - x[sd];
            } else {
                cur.node = node.greater;
                far.node = node.less;
                s = x[sd] - node.split;
            }
            s = s * s;
            far.min_distance += s - far.side[sd];
            far.side[sd] = s;
            if (cur.min_distance > far.min_distance) {
                const kd::NodeInfo tmp = cur;
                cur = far;
                far = tmp;
            }
            if (far.min_distance <= dub) {
                if (qn == qcap) {  // rare: move the pending nodes to a node-count sized piece of the arena
                    const int need = tb.meta[0];
                    int off = 0;
                    if (lane == 0) off = atomicAdd(&tb.meta[2], need);
                    off = __shfl_sync(FULL, off, 0);
                    if (qcap >= need || off + need > kdp::ARENA) __trap();
                    kd::NodeInfo *big = tb.arena + off;
                    for (int e = lane; e < qn; e += 32) big[e] = q[e];
                    __syncwarp();
                    q = big;
                    qcap = need;
                }
                wheap_push(q, qn, far, lane);
            }
        }
    }
    const int found = nbn;
    for (int i = found - 1; i >= 0; i--) {
        const kd::Item top = nb[0];
        if (lane == 0) {
            ws.inds[i] = top.payload;
            if (want_dist) ws.w[i] = sqrt(-top.priority);
        }
        wheap_remove(nb, nbn, lane);
    }
    if (lane == 0)
        for (int i = found; i < kmax; i++) {
            ws.inds[i] = t.n;
            if (want_dist) ws.w[i] = (double)INFINITY;
        }
    __syncwarp();
}

struct OutlierParams {
    const double *xy, *uv;
    int k;
    double thr;
    kdp::TreeBuf tb;
    int *inds;         // nthreads * (k+1)   (k + 1 > NBSMEM only)
    kd::Item *nb;      // nthreads * (k+1)   (k + 1 > NBSMEM only)
    kd::NodeInfo *q;   // nthreads * QHEAP   (k + 1 > NBSMEM only)
    uint8_t *out;
};

// one warp per vector: scipy's query for its k+1 nearest, Mahalanobis test on them
__global__ void __launch_bounds__(32 * QW)
outliers_warp_kernel(const __grid_constant__ OutlierParams p) {
    __shared__ WarpScratch scratch[QW];
    const int n = p.tb.meta[1];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int v = blockIdx.x * QW + wid;
    if (v >= n) return;
    if (n < 2) {  // cleansing.py:178-179
        if (lane == 0) p.out[v] = 0;
        return;
    }
    const int kk = min(p.k + 1, n);  // :197
    const kd::Tree t = kdp::tree_of(p.tb, p.xy);
    WarpScratch &ws = scratch[wid];
    warp_query(t, p.tb, p.xy[2 * (size_t)v], p.xy[2 * (size_t)v + 1], kk, ws, false, lane);
    if (lane == 0) p.out[v] = kd::mahalanobis_outlier(p.uv, v, ws.inds, kk - 1, p.thr) ? 1 : 0;
}

// general neighbour count: one thread per vector, heaps in global scratch
__global__ void __launch_bounds__(kdp::QTHREADS)
outliers_kernel(const __grid_constant__ OutlierParams p) {
    const int n = p.tb.meta[1];
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= n) return;
    if (n < 2) {
        p.out[tid] = 0;
        return;
    }
    const int kk = min(p.k + 1, n);
    const kd::Tree t = kdp::tree_of(p.tb, p.xy);
    int *inds = p.inds + (size_t)tid * (p.k + 1);
    kd::Strided<kd::Item> nb{p.nb + (size_t)tid * (p.k + 1), 1};
    kd::Strided<kd::NodeInfo> q{p.q + (size_t)tid * kdp::QHEAP, 1};
    kdp::ArenaGrow grow(p.tb);
    kd::query(t, p.xy[2 * (size_t)tid], p.xy[2 * (size_t)tid + 1], kk, inds, nb, q, kdp::QHEAP, grow);
    p.out[tid] = kd::mahalanobis_outlier(p.uv, tid, inds, kk - 1, p.thr) ? 1 : 0;
}

struct IdwFixParams {
    const double *xy, *vals, *xgrid, *ygrid;
    int nvar, k, nx, ny;
    double power, offset, mean_res;
    kdp::TreeBuf tb;
    const int *list;       // grid points to recompute (row * nx + column)
    const int *list_count; // null: every grid point
    int *inds;             // nthreads * k       (k > NBSMEM only)
    double *w;             // nthreads * k       (k > NBSMEM only)
    kd::Item *nb;          // nthreads * k       (k > NBSMEM only)
    kd::NodeInfo *q;       // nthreads * QHEAP   (k > NBSMEM only)
    double *out;           // (nvar, ny, nx)
    double2 *twin;         // (ny, nx) pairs of out's two variables, or null
};

// scipy's query and numpy's weighting (knn_body.cuh: idw_point) for the listed grid points, one
// warp per grid point at a time
__global__ void __launch_bounds__(32 * QW)
idw_fix_warp_kernel(const __grid_constant__ IdwFixParams p) {
    __shared__ WarpScratch scratch[QW];
    const int n = p.tb.meta[1];
    const int k = min(p.k, n);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t warp = (size_t)blockIdx.x * QW + wid, nwarps = (size_t)gridDim.x * QW;
    const size_t N = (size_t)p.ny * p.nx;
    const size_t count = p.list_count ? (size_t)min(*p.list_count, (int)min(N, (size_t)0x7fffffff)) : N;
    if (k < 1) return;
    const kd::Tree t = kdp::tree_of(p.tb, p.xy);
    WarpScratch &ws = scratch[wid];
    for (size_t e = warp; e < count; e += nwarps) {
        const size_t g = p.list_count ? (size_t)p.list[e] : e;
        const int i = (int)(g / p.nx), j = (int)(g % p.nx);
        warp_query(t, p.tb, p.xgrid[j], p.ygrid[i], k, ws, true, lane);
        if (lane == 0) {
            kd::idw_point(p.vals, p.nvar, ws.inds, ws.w, k, p.power, p.offset, p.mean_res, p.out + g, N);
            if (p.twin) p.twin[g] = make_double2(p.out[g], p.out[N + g]);
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(kdp::QTHREADS)
idw_fix_kernel(const __grid_constant__ IdwFixParams p) {
    const int n = p.tb.meta[1];
    const int k = min(p.k, n);
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    const size_t N = (size_t)p.ny * p.nx;
    const size_t count = p.list_count ? (size_t)min(*p.list_count, (int)min(N, (size_t)0x7fffffff)) : N;
    if (k < 1) return;
    const kd::Tree t = kdp::tree_of(p.tb, p.xy);
    int *inds = p.inds + tid * p.k;
    double *w = p.w + tid * p.k;
    for (size_t e = tid; e < count; e += nthreads) {
        const size_t g = p.list_count ? (size_t)p.list[e] : e;
        const int i = (int)(g / p.nx), j = (int)(g % p.nx);
        kd::Strided<kd::Item> nb{p.nb + tid * p.k, 1};
        kd::Strided<kd::NodeInfo> q{p.q + tid * kdp::QHEAP, 1};
        kdp::ArenaGrow grow(p.tb);
        kd::query(t, p.xgrid[j], p.ygrid[i], k, inds, nb, q, kdp::QHEAP, grow, w);
        kd::idw_point(p.vals, p.nvar, inds, w, k, p.power, p.offset, p.mean_res, p.out + g, N);
        if (p.twin) p.twin[g] = make_double2(p.out[g], p.out[N + g]);
    }
}

}  // namespace

namespace kdp {

int tree_alloc(TreeScratch &ts, int n_cap, cudaStream_t s) {
    B200_CUDA(ts.idx.alloc(sizeof(int) * (size_t)std::max(n_cap, 1), s));
    B200_CUDA(ts.nodes.alloc(sizeof(kd::Node) * (size_t)kd::max_nodes(n_cap), s));
    B200_CUDA(ts.meta.alloc(sizeof(int) * 4, s));
    B200_CUDA(ts.bounds.alloc(sizeof(double) * 4, s));
    B200_CUDA(ts.arena.alloc(sizeof(kd::NodeInfo) * (size_t)ARENA, s));
    ts.tb.idx = (int *)ts.idx.p;
    ts.tb.nodes = (kd::Node *)ts.nodes.p;
    ts.tb.meta = (int *)ts.meta.p;
    ts.tb.bounds = (double *)ts.bounds.p;
    ts.tb.arena = (kd::NodeInfo *)ts.arena.p;
    return 0;
}

int tree_build(const double *xy, const int *n_dev, int n_cap, const TreeBuf &tb, cudaStream_t s) {
    if (n_cap <= NMAX) {
        static bool attr_set = false;
        if (!attr_set) {
            B200_CUDA(cudaFuncSetAttribute(kd_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)sizeof(BuildSmem)));
            attr_set = true;
        }
        kd_build_kernel<<<1, 32 * WARPS, sizeof(BuildSmem), s>>>(xy, n_dev, n_cap, tb);
    } else {
        kd_build_serial_kernel<<<1, 1, 0, s>>>(xy, n_dev, n_cap, tb);
    }
    B200_LAUNCH_CHECK();
    return 0;
}

int idw_fix(const double *xy, const double *vals, int nvar, int k, double power, double dist_offset,
            double mean_res, const double *xgrid, int nx, const double *ygrid, int ny, const TreeBuf &tb,
            const int *list, const int *list_count, double *out, double2 *twin, cudaStream_t s) {
    IdwFixParams p;
    memset(&p, 0, sizeof(p));
    p.xy = xy; p.vals = vals; p.xgrid = xgrid; p.ygrid = ygrid; p.nvar = nvar; p.k = k; p.nx = nx; p.ny = ny;
    p.power = power; p.offset = dist_offset; p.mean_res = mean_res; p.tb = tb;
    p.list = list; p.list_count = list_count; p.out = out; p.twin = nvar == 2 ? twin : nullptr;
    const size_t N = (size_t)ny * nx;
    if (k <= NBSMEM) {
        // as many warps as the chip holds (one search each); the list is usually shorter
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((N + QW - 1) / QW, (size_t)b200::num_sms() * 16));  // 16 CTAs of 4 warps fill an SM
        idw_fix_warp_kernel<<<blocks, 32 * QW, 0, s>>>(p);
        B200_LAUNCH_CHECK();
        return 0;
    }
    const int T = QTHREADS;
    const int blocks = (int)std::max<size_t>(1, std::min<size_t>((N + T - 1) / T, (size_t)b200::num_sms() * 2));
    const size_t nthreads = (size_t)blocks * T;
    b200::Scratch inds, w, nb, q;
    B200_CUDA(inds.alloc(sizeof(int) * nthreads * k, s));
    B200_CUDA(w.alloc(sizeof(double) * nthreads * k, s));
    B200_CUDA(nb.alloc(sizeof(kd::Item) * nthreads * k, s));
    B200_CUDA(q.alloc(sizeof(kd::NodeInfo) * nthreads * QHEAP, s));
    p.inds = (int *)inds.p; p.w = (double *)w.p; p.nb = (kd::Item *)nb.p; p.q = (kd::NodeInfo *)q.p;
    idw_fix_kernel<<<blocks, T, 0, s>>>(p);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace kdp

extern "C" int b200_kdtree_build(const double *xy, const int *n_dev, int n_cap, int *tree_indices,
                                 int *node_count, void *stream) {
    B200_REQUIRE(xy != nullptr && tree_indices != nullptr && n_cap >= 0, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    kdp::TreeScratch ts;
    if (int rc = kdp::tree_alloc(ts, n_cap, s)) return rc;
    if (int rc = kdp::tree_build(xy, n_dev, n_cap, ts.tb, s)) return rc;
    B200_CUDA(cudaMemcpyAsync(tree_indices, ts.tb.idx, sizeof(int) * (size_t)n_cap, cudaMemcpyDeviceToDevice, s));
    if (node_count) B200_CUDA(cudaMemcpyAsync(node_count, ts.tb.meta, sizeof(int), cudaMemcpyDeviceToDevice, s));
    return 0;
}

extern "C" int b200_idw_fill_ckdtree(const double *xy, const double *vals, const int *npts_dev, int npts_cap,
                                     int nvar, int k, double power, double dist_offset, double mean_res,
                                     const double *xgrid, int nx, const double *ygrid, int ny, double *out,
                                     void *stream) {
    B200_REQUIRE(xy && vals && xgrid && ygrid && out && npts_cap >= 1 && nvar >= 1 && nx >= 1 && ny >= 1,
                 "bad arguments");
    B200_REQUIRE(k >= 1 && k <= 128, "k must be 1..128");
    cudaStream_t s = (cudaStream_t)stream;
    kdp::TreeScratch ts;
    if (int rc = kdp::tree_alloc(ts, npts_cap, s)) return rc;
    if (int rc = kdp::tree_build(xy, npts_dev, npts_cap, ts.tb, s)) return rc;
    return kdp::idw_fix(xy, vals, nvar, k, power, dist_offset, mean_res, xgrid, nx, ygrid, ny, ts.tb, nullptr,
                        nullptr, out, nullptr, s);
}

extern "C" int b200_detect_outliers(const double *uv, const double *xy, const int *n_dev, int n_cap,
                                    double thr, int k, uint8_t *out, void *stream) {
    B200_REQUIRE(uv != nullptr && xy != nullptr && out != nullptr && n_cap >= 0, "bad arguments");
    B200_REQUIRE(k >= 1 && k <= 4096, "k out of range");
    if (n_cap == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    kdp::TreeScratch ts;
    if (int rc = kdp::tree_alloc(ts, n_cap, s)) return rc;
    if (int rc = kdp::tree_build(xy, n_dev, n_cap, ts.tb, s)) return rc;
    OutlierParams p;
    memset(&p, 0, sizeof(p));
    p.xy = xy; p.uv = uv; p.k = k; p.thr = thr; p.tb = ts.tb; p.out = out;
    if (k + 1 <= kdp::NBSMEM) {
        outliers_warp_kernel<<<b200::ceil_div(n_cap, QW), 32 * QW, 0, s>>>(p);
        B200_LAUNCH_CHECK();
        return 0;
    }
    const int T = kdp::QTHREADS;
    b200::Scratch inds, nb, q;
    B200_CUDA(inds.alloc(sizeof(int) * (size_t)n_cap * (k + 1), s));
    B200_CUDA(nb.alloc(sizeof(kd::Item) * (size_t)n_cap * (k + 1), s));
    B200_CUDA(q.alloc(sizeof(kd::NodeInfo) * (size_t)n_cap * kdp::QHEAP, s));
    p.inds = (int *)inds.p; p.nb = (kd::Item *)nb.p; p.q = (kd::NodeInfo *)q.p;
    outliers_kernel<<<b200::ceil_div(n_cap, T), T, 0, s>>>(p);
    B200_LAUNCH_CHECK();
    return 0;
}
