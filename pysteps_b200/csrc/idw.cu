// idw.cu -- inverse-distance-weighted k-nearest-neighbour grid fill (sm_90a).
//
// Reference: pysteps/utils/interpolate.py:67-114 (idwinterp2d): cKDTree.query(grid, k) over
// every grid point, dist/mean_res + offset, w = 1/dist^power normalised, weighted sum of
// the k values.  This is 95 % of the reference's dense_lucaskanade wall time (16.7 s of
// 17.6 s at 2048^2, single-threaded tree queries).  With <= a few thousand source vectors
// an EXHAUSTIVE top-k per pixel is the GPU-natural form: the vectors are staged in shared
// memory once per CTA and every thread scans them for its own pixel, keeping the k best
// (squared distance, index) pairs sorted in registers.  It is FP64-ALU bound, not HBM
// bound (~5 FP64 ops per pixel-vector pair vs 16 B written per pixel); distances and
// weights are float64.
//
// Neighbour ORDER: an exhaustive scan has no tree, so equal distances are listed by lower index,
// scipy.spatial.cKDTree lists them in its tree's order.  Inside the list that only permutes equal
// weights (identical result up to the order of one addition); it matters where the k-th and the
// (k+1)-th neighbour are exactly equidistant, because then the two pick different vectors.  Every
// thread therefore tracks the smallest candidate it did NOT keep; a grid point whose k-th distance
// equals it is appended to a list and recomputed from scipy's own query (knn.cu: idw_fix_kernel,
// tree built on a side stream while this kernel runs).  The fill is then the reference's at every
// grid point (<= 1e-12; the weights use rsqrt where NumPy uses sqrt/power/divide).
//
// The search comes in four forms (32-bit keys, packed or unpacked 64-bit keys, an insertion list);
// idw_fill_kernel is the one rule that chooses among them, for b200_idw_fill and for the device plan
// of b200_idw_fill_planned alike, and idw_run the fill both entry points share.
#include <math_constants.h>

#include "common.cuh"
#include "knn_device.cuh"

namespace {

constexpr int IDW_TX = 16, IDW_TY = 16;           // pixel tile of one CTA (8 warps of 8x4 pixels)
constexpr int IDW_THREADS = IDW_TX * IDW_TY;
constexpr int IDW_CHUNK = 2048;                    // source vectors examined per round
constexpr int IDW_BINS = 256;                      // distance histogram of the tile centre

struct IDWParams {
    const double *xy;    // (npts,2)
    const double *vals;  // (npts,nvar)
    const int *npts_dev;
    int npts_cap, nvar, k;
    const double *gx, *gy;
    int nx, ny;
    double power, offset, mean_res;
    double *out;  // (nvar, ny, nx)
    double2 *twin;   // (ny, nx) pairs of the two variables, written beside `out` (or null; nvar == 2 only)
    const B200IdwPlan *plan;  // device plan of b200_idw_fill_planned (or null: the host chose the kernel)
    int *tie_list;   // grid points whose k-th and (k+1)-th neighbours are equidistant
    int *tie_count;
    uint8_t *tile_done;  // per pixel tile: filled by the 32-bit-key kernel (or null)
};

// dense_lucaskanade's weighting (two variables, power 1/2, unit resolution, positive offset): the
// weights come from rsqrt instead of NumPy's sqrt, power and divide
__host__ __device__ __forceinline__ bool fast_weights(const IDWParams &p) {
    return p.nvar == 2 && p.power == 0.5 && p.mean_res == 1.0 && p.offset > 0.0;
}

// Which kernel fills the field, for k neighbours among n vectors with key level `level`
// (coords_on_16th_grid: 2 half-pixel vectors on an integer grid, 1 every coordinate a multiple of 1/16
// below 2^14, 0 otherwise) and fast weights or not:
//   KEY32     k == 20 <= n <= IDW_CHUNK, level 2, fast weights: idw32_kernel<20>, then the PACKED
//             kernel over the tiles whose search radius the 32-bit keys do not hold
//   PACKED    k == 20 <= n <= IDW_CHUNK, level >= 1: idw_kernel<20, true, true, fastw>
//   UNPACKED  k == 20 <= n otherwise: idw_kernel<20, true, false, fastw>
//   INSERT    k != 20 or n < 20: idw_kernel<32, false, false, false>, the insertion list
//   NONE      n == 0: a device plan whose field is constant, zero or refused
// b200_idw_fill applies it to the counts it knows; a count on the device takes INSERT.  With a device
// plan every kernel the rule may pick is enqueued, and each applies it to the plan's n_fill with
// k = min(k, n_fill) to decide whether the field is its own.
enum IdwFill { IDW_NONE, IDW_KEY32, IDW_PACKED, IDW_UNPACKED, IDW_INSERT };

__host__ __device__ __forceinline__ IdwFill idw_fill_kernel(int k, int n, int level, bool fastw) {
    if (n < 1) return IDW_NONE;
    if (k != 20 || n < k) return IDW_INSERT;
    if (level == 0 || n > IDW_CHUNK) return IDW_UNPACKED;
    return (level == 2 && fastw) ? IDW_KEY32 : IDW_PACKED;
}

// with a device plan: the rule gives the field to another kernel than `mine`
__device__ __forceinline__ bool plan_declines(const IDWParams &p, IdwFill mine) {
    if (!p.plan) return false;
    const int n = p.plan->n_fill;
    const IdwFill f = idw_fill_kernel(min(p.k, n), n, p.plan->on_grid, fast_weights(p));
    return !(f == mine || (f == IDW_KEY32 && mine == IDW_PACKED));
}

// numpy's pairwise summation for n < 128 (8 accumulators, then the remainder)
template <int K>
__device__ __forceinline__ double np_sum(const double (&w)[K], int k) {
    if (k < 8) {
        double r = w[0];
#pragma unroll
        for (int i = 1; i < K; i++)
            if (i < k) r = __dadd_rn(r, w[i]);
        return r;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = w[j];
    const int lim = k - (k % 8);
#pragma unroll
    for (int i = 8; i < K; i++)
        if (i < lim) r[i & 7] = __dadd_rn(r[i & 7], w[i]);
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                           __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
#pragma unroll
    for (int i = 8; i < K; i++)
        if (i >= lim && i < k) res = __dadd_rn(res, w[i]);
    return res;
}

// One CTA fills a 32x8 pixel tile.  Exhaustive search is exact but wasteful (every pixel
// against every vector); the tile first bounds its search radius: with Rk >= distance from
// the tile centre c to its k-th nearest vector and r the tile's half diagonal, every pixel
// p of the tile has its k nearest within Rk + r of p, hence within Rk + 2r of c.  Vectors
// outside that disc cannot be among any pixel's k nearest and are dropped -- the result is
// identical to the exhaustive search, with ~k..3k candidates per tile instead of all.
// The candidates are bucketed by centre distance (counting sort on the histogram that gave
// Rk), so each pixel meets its near vectors first and later ones fail the `< worst` test
// without touching the sorted list.  Order of examination is irrelevant for the result:
// the list is ordered by (squared distance, index), i.e. equal distances resolve to the
// lower index exactly as cKDTree-free exhaustive scanning in index order would.
// Batcher odd-even merge sorting network of 20 (generated, verified exhaustively with the 0-1
// principle): a compile-time comparator list, so the sorted list never leaves registers.
__device__ constexpr int NET20[103][2] = {{0,1},{2,3},{4,5},{6,7},{8,9},{10,11},{12,13},{14,15},{16,17},{18,19},{0,2},{1,3},{4,6},{5,7},{8,10},{9,11},{12,14},{13,15},{16,18},{17,19},{1,2},{5,6},{9,10},{13,14},{17,18},{0,4},{1,5},{2,6},{3,7},{8,12},{9,13},{10,14},{11,15},{2,4},{3,5},{10,12},{11,13},{1,2},{3,4},{5,6},{9,10},{11,12},{13,14},{17,18},{0,8},{1,9},{2,10},{3,11},{4,12},{5,13},{6,14},{7,15},{4,8},{5,9},{6,10},{7,11},{2,4},{3,5},{6,8},{7,9},{10,12},{11,13},{1,2},{3,4},{5,6},{7,8},{9,10},{11,12},{13,14},{17,18},{0,16},{1,17},{2,18},{3,19},{8,16},{9,17},{10,18},{11,19},{4,8},{5,9},{6,10},{7,11},{12,16},{13,17},{14,18},{15,19},{2,4},{3,5},{6,8},{7,9},{10,12},{11,13},{14,16},{15,17},{1,2},{3,4},{5,6},{7,8},{9,10},{11,12},{13,14},{15,16},{17,18}};
template <int K> __device__ __forceinline__ constexpr int net_size() { return K == 20 ? 103 : 0; }
template <int K> __device__ __forceinline__ constexpr int net_a(int c) { return K == 20 ? NET20[c < 103 ? c : 0][0] : 0; }
template <int K> __device__ __forceinline__ constexpr int net_b(int c) { return K == 20 ? NET20[c < 103 ? c : 0][1] : 0; }

__device__ __forceinline__ bool key_less(unsigned long long da, int ia, unsigned long long db, int ib) {
    return da < db || (da == db && ia < ib);
}

// Sorted list of the k best (squared distance, index) pairs of one pixel.
// EXACT = true: k == K, the list lives in registers (every index is a compile-time constant).
// The first K candidates are loaded as they come and sorted once by a sorting network; every
// later candidate is tested against the current worst and, if better, inserted branch free:
// K independent "key < entry" predicates, then each slot takes its left neighbour, the key,
// or keeps its value.  Squared distances are >= 0, so their bit patterns order like the
// doubles; (bits, index) is compared as one integer key.
// EXACT = false (k < K: fewer vectors than neighbours, or an unusual k): insertion only, with
// a runtime length -- a rare, small-problem path.
// PACKED (fast path of dense_lucaskanade): all coordinates are multiples of 1/16 below 2^14
// and there are at most 2048 vectors, so a squared distance is a multiple of 1/256 below 2^29
// and the 11 low mantissa bits of its float64 pattern are zero: the vector index is stored
// there.  One 64-bit integer then carries (distance, index) in exactly the required order --
// a comparator is one compare and two selects, and the index array disappears.
template <int K, bool EXACT, bool PACKED>
__device__ __forceinline__ void topk_scan(const double2 *__restrict__ spt, const int *__restrict__ sidx,
                                          int ncand, double qx, double qy, int k, bool first,
                                          unsigned long long (&bd)[K], int (&bi)[K], unsigned long long &rej) {
    auto dist2 = [&](int t) -> unsigned long long {
        const double2 s = spt[t];
        const double dx = __dsub_rn(s.x, qx), dy = __dsub_rn(s.y, qy);
        const unsigned long long b =
            (unsigned long long)__double_as_longlong(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        return PACKED ? (b | (unsigned long long)sidx[t]) : b;
    };
    int t0 = 0;
    if (EXACT && first && ncand >= K) {
#pragma unroll
        for (int q = 0; q < K; q++) { bd[q] = dist2(q); if (!PACKED) bi[q] = sidx[q]; }
#pragma unroll
        for (int c = 0; c < net_size<K>(); c++) {
            const int a = net_a<K>(c), b = net_b<K>(c);
            if (PACKED) {
                const unsigned long long va = bd[a], vb = bd[b];
                const bool sw = vb < va;
                bd[a] = sw ? vb : va;
                bd[b] = sw ? va : vb;
            } else {
                const bool sw = key_less(bd[b], bi[b], bd[a], bi[a]);
                const unsigned long long va = bd[a], vb = bd[b];
                const int ia = bi[a], ib = bi[b];
                bd[a] = sw ? vb : va; bd[b] = sw ? va : vb;
                bi[a] = sw ? ib : ia; bi[b] = sw ? ia : ib;
            }
        }
        t0 = K;
    }
    for (int t = t0; t < ncand; t++) {
        const unsigned long long d2 = dist2(t);
        const int last = EXACT ? K - 1 : k - 1;
        unsigned long long wd = bd[K - 1];
        int wi = PACKED ? 0 : bi[K - 1];
        if (!EXACT) {
#pragma unroll
            for (int q = 0; q < K; q++)
                if (q == last) { wd = bd[q]; wi = bi[q]; }
        }
        const int id = PACKED ? 0 : sidx[t];
        const bool better = PACKED ? (d2 < wd) : key_less(d2, id, wd, wi);
        // smallest (squared distance) key that is not in the list: the evicted worst or the
        // rejected candidate
        const unsigned long long gone = better ? wd : d2;
        rej = gone < rej ? gone : rej;
        if (better) {
            bool lt[K];
#pragma unroll
            for (int q = 0; q < K; q++) lt[q] = PACKED ? (d2 < bd[q]) : key_less(d2, id, bd[q], bi[q]);
#pragma unroll
            for (int q = K - 1; q >= 1; q--) {
                if (EXACT || q <= last) {
                    const unsigned long long nd = lt[q - 1] ? bd[q - 1] : (lt[q] ? d2 : bd[q]);
                    bd[q] = nd;
                    if (!PACKED) {
                        const int ni = lt[q - 1] ? bi[q - 1] : (lt[q] ? id : bi[q]);
                        bi[q] = ni;
                    }
                }
            }
            if (lt[0]) { bd[0] = d2; if (!PACKED) bi[0] = id; }
        }
    }
}

// Search bound of one pixel tile (see the comment above idw_kernel): histogram of the vectors'
// distances to the tile centre, bin of the k-th, candidate bins [0, bmax]; leaves the exclusive
// bin offsets in `hist`, zeroes `fill`, caches the bins of the first IDW_CHUNK vectors in `sbin`.
struct TileBound {
    int bmax, total;
    double cx, cy, rt, binw;
    float inv_binw_f;
    __device__ __forceinline__ int bin_of(const double2 *__restrict__ pts, int t) const {
        const double2 s = pts[t];
        const float dx = (float)(s.x - cx), dy = (float)(s.y - cy);
        const float d = sqrtf(dx * dx + dy * dy) * inv_binw_f;
        return d < (float)(IDW_BINS - 1) ? (int)d : IDW_BINS - 1;
    }
};

__device__ __forceinline__ TileBound tile_bound(const IDWParams &p, const double2 *__restrict__ pts, int npts, int k,
                                                int *hist, int *fill, unsigned char *sbin, int *s_bmax,
                                                int *s_total, int bx, int by) {
    const int tid = threadIdx.x, lane = tid & 31;
    TileBound tb;
    // ---- tile centre, half diagonal, histogram of centre distances ---------------------
    const int j0 = bx * IDW_TX, j1 = min(j0 + IDW_TX, p.nx) - 1;
    const int i0 = by * IDW_TY, i1 = min(i0 + IDW_TY, p.ny) - 1;
    const double xa = p.gx[j0], xb = p.gx[j1], ya = p.gy[i0], yb = p.gy[i1];
    tb.cx = 0.5 * (xa + xb);
    tb.cy = 0.5 * (ya + yb);
    const double cx = tb.cx, cy = tb.cy;
    // grids are monotonic (np.arange in dense_lucaskanade); the tile extent bounds the radius
    const double rt = sqrt(0.25 * (xb - xa) * (xb - xa) + 0.25 * (yb - ya) * (yb - ya));
    const double binw = fmax(rt, 1e-300) * 0.5;
    const double inv_binw = 1.0 / binw;
    for (int b = tid; b < IDW_BINS; b += IDW_THREADS) { hist[b] = 0; fill[b] = 0; }
    __syncthreads();
    // The bin only has to be CONSERVATIVE (never below the true distance bin) and the same in
    // both passes, so it is computed in float32 with 1e-5 slack instead of an FP64 sqrt.
    const float inv_binw_f = (float)inv_binw * (1.0f + 1e-5f);
    tb.inv_binw_f = inv_binw_f;
    auto bin_of = [&](int t) -> int { return tb.bin_of(pts, t); };
    for (int t = tid; t < npts; t += IDW_THREADS) {
        const int b = bin_of(t);
        if (t < IDW_CHUNK) sbin[t] = (unsigned char)b;
        atomicAdd(&hist[b], 1);
    }
    __syncthreads();
    if (tid < 32) {
        // exclusive prefix over the bins (8 per lane), bin of the k-th vector, search bound
        int c[IDW_BINS / 32], sum = 0;
#pragma unroll
        for (int q = 0; q < IDW_BINS / 32; q++) { c[q] = hist[lane * (IDW_BINS / 32) + q]; sum += c[q]; }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        int run = incl - sum, bk = IDW_BINS;  // first bin whose inclusive count reaches k
#pragma unroll
        for (int q = 0; q < IDW_BINS / 32; q++) {
            hist[lane * (IDW_BINS / 32) + q] = run;
            run += c[q];
            if (run >= k && bk == IDW_BINS) bk = lane * (IDW_BINS / 32) + q;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) bk = min(bk, __shfl_xor_sync(0xffffffffu, bk, o));
        if (lane == 0) {
            int bmax = IDW_BINS - 1;  // overflow bin reached: every vector is a candidate
            if (bk < IDW_BINS - 1) {
                const double R = ((double)(bk + 1) * binw + 2.0 * rt) * (1.0 + 1e-9);
                const double bb = R * inv_binw * (1.0 + 1e-9);
                bmax = bb < (double)(IDW_BINS - 1) ? (int)bb : IDW_BINS - 1;
            }
            *s_bmax = bmax;
        }
    }
    __syncthreads();
    const int bmax = *s_bmax;
    if (tid == 0) *s_total = (bmax == IDW_BINS - 1) ? npts : hist[bmax + 1];
    __syncthreads();
    const int total = *s_total;

    tb.bmax = bmax;
    tb.total = total;
    tb.rt = rt;
    tb.binw = binw;
    tb.inv_binw_f = inv_binw_f;
    return tb;
}

// Lists grid point g of every lane whose `tie` is set: one atomicAdd per warp, stores compacted.
__device__ __forceinline__ void tie_append(const IDWParams &p, bool tie, int g) {
    const int lane = threadIdx.x & 31;
    const unsigned bal = __ballot_sync(0xffffffffu, tie);
    if (bal) {
        int base = 0;
        if (lane == __ffs(bal) - 1) base = atomicAdd(p.tie_count, __popc(bal));
        base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
        if (tie) p.tie_list[base + __popc(bal & ((1u << lane) - 1u))] = g;
    }
}

// The fast weighting (fast_weights) of grid point (i, j) over list entries q < k, entry(q, d2, id)
// giving the squared distance and vector index of each: w = (sqrt(d2) + offset)^-1/2 from two rsqrt
// (FMA pipe) instead of sqrt, pow and a divide per neighbour, normalised once -- relative error a few
// 1e-16.  Stores the planar field and its twin.
template <int K, typename Entry>
__device__ __forceinline__ void fast_weights_store(const IDWParams &p, int k, int i, int j, Entry entry) {
    double ws = 0.0, ax = 0.0, ay = 0.0;
    const double2 *__restrict__ v2 = reinterpret_cast<const double2 *>(p.vals);
#pragma unroll
    for (int q = 0; q < K; q++) {
        if (q < k) {
            double d2;
            int id;
            entry(q, d2, id);
            const double dist = d2 > 0.0 ? d2 * rsqrt(d2) : 0.0;
            const double w = rsqrt(dist + p.offset);
            const double2 v = v2[id];
            ws += w;
            ax = fma(w, v.x, ax);
            ay = fma(w, v.y, ay);
        }
    }
    const double inv = 1.0 / ws, fx = ax * inv, fy = ay * inv;
    p.out[((size_t)0 * p.ny + i) * p.nx + j] = fx;
    p.out[((size_t)1 * p.ny + i) * p.nx + j] = fy;
    if (p.twin) p.twin[(size_t)i * p.nx + j] = make_double2(fx, fy);
}

// FASTW: the fast weighting; otherwise the general NumPy-order epilogue.
// One pixel tile (bx, by) of idw_kernel.
template <int K, bool EXACT, bool PACKED, bool FASTW>
__device__ __forceinline__ void idw_tile(const IDWParams &p, int bx, int by, int tiles_x) {
    __shared__ double2 spt[IDW_CHUNK];
    __shared__ int sidx[IDW_CHUNK];
    __shared__ int hist[IDW_BINS];   // counts, then exclusive offsets
    __shared__ int fill[IDW_BINS];
    __shared__ unsigned char sbin[IDW_CHUNK];  // bin of the first IDW_CHUNK vectors
    __shared__ int s_bmax, s_total;
    if (p.tile_done && p.tile_done[by * tiles_x + bx]) return;
    const int npts = p.npts_dev ? min(*p.npts_dev, p.npts_cap) : p.npts_cap;
    const int k = min(min(p.k, npts), K);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // a warp covers a compact 8x4 pixel patch: its lanes agree on most insert decisions
    const int j = bx * IDW_TX + (wid & 1) * 8 + (lane & 7);   // column
    const int i = by * IDW_TY + (wid >> 1) * 4 + (lane >> 3);  // row
    const double2 *__restrict__ pts = reinterpret_cast<const double2 *>(p.xy);
    const bool active = j < p.nx && i < p.ny;
    const double qx = p.gx[min(j, p.nx - 1)], qy = p.gy[min(i, p.ny - 1)];

    const TileBound tb = tile_bound(p, pts, npts, k, hist, fill, sbin, &s_bmax, &s_total, bx, by);
    const int bmax = tb.bmax, total = tb.total;
    auto bin_of = [&](int t) -> int { return tb.bin_of(pts, t); };

    unsigned long long bd[K];  // squared distances as ordered bit patterns
    int bi[K];
#pragma unroll
    for (int q = 0; q < K; q++) { bd[q] = 0x7ff0000000000000ull; bi[q] = 0x7fffffff; }  // +inf
    unsigned long long rej = ~0ull;  // smallest key among the candidates that are not in the list

    // sorted: all candidates fit in shared memory (one round, counting sort by centre-distance
    // bin); otherwise plain exhaustive rounds over chunks of all vectors
    const bool sorted = total <= IDW_CHUNK;
    const int nrounds = sorted ? 1 : (npts + IDW_CHUNK - 1) / IDW_CHUNK;
    for (int r = 0; r < nrounds; r++) {
        int cnt;
        __syncthreads();
        if (sorted) {
            for (int t = tid; t < npts; t += IDW_THREADS) {
                const int b = t < IDW_CHUNK ? (int)sbin[t] : bin_of(t);
                if (b <= bmax) {
                    const int o = hist[b] + atomicAdd(&fill[b], 1);
                    spt[o] = pts[t];
                    sidx[o] = t;
                }
            }
            cnt = total;
        } else {
            const int base = r * IDW_CHUNK;
            cnt = min(IDW_CHUNK, npts - base);
            for (int t = tid; t < cnt; t += IDW_THREADS) {
                spt[t] = pts[base + t];
                sidx[t] = base + t;
            }
        }
        __syncthreads();
        if (active) topk_scan<K, EXACT, PACKED>(spt, sidx, cnt, qx, qy, k, r == 0, bd, bi, rej);
    }
    // ---- equidistant k-th / (k+1)-th neighbour: listed for the exact-order recomputation -----
    {
        unsigned long long kth = bd[K - 1];
        if (!EXACT) {
#pragma unroll
            for (int q = 0; q < K; q++)
                if (q == k - 1) kth = bd[q];
        }
        const unsigned long long dmask = PACKED ? ~2047ull : ~0ull;
        tie_append(p, active && k >= 1 && ((kth & dmask) == (rej & dmask)), i * p.nx + j);
    }
    if (!active || k < 1) return;
    if (FASTW) {
        fast_weights_store<K>(p, k, i, j, [&](int q, double &d2, int &id) {
            d2 = __longlong_as_double((long long)(PACKED ? (bd[q] & ~2047ull) : bd[q]));
            id = PACKED ? (int)(bd[q] & 2047ull) : bi[q];
        });
        return;
    }
    double w[K];
#pragma unroll
    for (int q = 0; q < K; q++) {
        if (PACKED) { bi[q] = (int)(bd[q] & 2047ull); bd[q] &= ~2047ull; }
        double d = sqrt(__longlong_as_double((long long)bd[q]));  // exact Euclidean distance
        if (p.mean_res != 1.0) d = __ddiv_rn(d, p.mean_res);  // interpolate.py:98 (x / 1.0 == x)
        d = __dadd_rn(d, p.offset);             // :101
        const double pw = (p.power == 0.5) ? sqrt(d) : pow(d, p.power);
        w[q] = (q < k) ? __ddiv_rn(1.0, pw) : 0.0;  // :102
    }
    const double ws = np_sum<K>(w, k);          // :103
    for (int v = 0; v < p.nvar; v++) {
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < K; q++)
            if (q < k) {
                const double term = __dmul_rn(p.vals[(size_t)bi[q] * p.nvar + v], __ddiv_rn(w[q], ws));
                acc = (q == 0) ? term : __dadd_rn(acc, term);  // :106-109
            }
        p.out[((size_t)v * p.ny + i) * p.nx + j] = acc;
    }
    if (p.twin) {  // this thread's own two stores, read back (keeps the K-wide loop's registers free)
        const size_t g = (size_t)i * p.nx + j, N = (size_t)p.ny * p.nx;
        p.twin[g] = make_double2(p.out[g], p.out[N + g]);
    }
}

// Every CTA walks the tiles in steps of the grid size.  A grid of one CTA per tile fills each tile at
// once; the kernels a device plan rarely chooses run on one wave of resident CTAs (resident_grid), so
// that declining costs one wave instead of one per tile.
template <int K, bool EXACT, bool PACKED, bool FASTW>
__global__ void __launch_bounds__(IDW_THREADS, FASTW ? 3 : 1) idw_kernel(const IDWParams p) {
    if (plan_declines(p, EXACT ? (PACKED ? IDW_PACKED : IDW_UNPACKED) : IDW_INSERT)) return;
    const int tiles_x = (p.nx + IDW_TX - 1) / IDW_TX, ntiles = tiles_x * ((p.ny + IDW_TY - 1) / IDW_TY);
    for (int t = blockIdx.y * gridDim.x + blockIdx.x; t < ntiles; t += gridDim.x * gridDim.y) {
        idw_tile<K, EXACT, PACKED, FASTW>(p, t % tiles_x, t / tiles_x, tiles_x);
        __syncthreads();  // the next tile reuses the shared memory
    }
}

// a grid of one wave of resident CTAs (at most one per tile)
template <typename F>
dim3 resident_grid(F kernel, dim3 full) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, IDW_THREADS, 0) != cudaSuccess || per_sm < 1)
        per_sm = 1;
    return dim3((unsigned)std::min<size_t>((size_t)full.x * full.y, (size_t)per_sm * b200::num_sms()));
}

// ---- 32-bit integer keys ---------------------------------------------------------------------
// dense_lucaskanade's vectors sit on the half-pixel grid (medians of integer corners) and the
// target grid on integers, so 4 * squared distance is a small INTEGER: with coordinates doubled,
// (dx2*dx2 + dy2*dy2) in int32 is exact, and while it stays below 2^21 (neighbours within 724 px)
// the pair (distance, vector index < 2048) is ONE 32-bit key.  The whole search then runs on the
// integer pipe with single-register compares and selects -- half the instructions of the 64-bit
// list, and no FP64 until the weights.  A tile whose search radius does not fit leaves its
// `tile_done` flag clear and is filled by the 64-bit kernel launched behind this one.
constexpr int IDW_KEY32_LIMIT = 1 << 21;

template <int K>
__global__ void __launch_bounds__(IDW_THREADS, 4) idw32_kernel(const IDWParams p) {
    __shared__ int2 spi[IDW_CHUNK];   // doubled coordinates of the candidates
    __shared__ int sidx[IDW_CHUNK];
    __shared__ int hist[IDW_BINS];
    __shared__ int fill[IDW_BINS];
    __shared__ unsigned char sbin[IDW_CHUNK];
    __shared__ int s_bmax, s_total;
    if (plan_declines(p, IDW_KEY32)) return;
    const int npts = p.npts_dev ? min(*p.npts_dev, p.npts_cap) : p.npts_cap;
    const int k = K;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int j = blockIdx.x * IDW_TX + (wid & 1) * 8 + (lane & 7);   // column
    const int i = blockIdx.y * IDW_TY + (wid >> 1) * 4 + (lane >> 3);  // row
    const double2 *__restrict__ pts = reinterpret_cast<const double2 *>(p.xy);
    const bool active = j < p.nx && i < p.ny;
    const double qx = p.gx[min(j, p.nx - 1)], qy = p.gy[min(i, p.ny - 1)];
    const TileBound tb = tile_bound(p, pts, npts, k, hist, fill, sbin, &s_bmax, &s_total, blockIdx.x, blockIdx.y);
    const int bmax = tb.bmax, total = tb.total;
    // every candidate lies within (bmax + 1) bins of the centre, every pixel within rt of it
    const double reach = 2.0 * ((double)(bmax + 1) * tb.binw + tb.rt) * (1.0 + 1e-6);
    if (total > IDW_CHUNK || bmax == IDW_BINS - 1 || !(reach * reach < (double)IDW_KEY32_LIMIT)) return;
    for (int t = tid; t < npts; t += IDW_THREADS) {
        const int b = t < IDW_CHUNK ? (int)sbin[t] : tb.bin_of(pts, t);
        if (b <= bmax) {
            const int o = hist[b] + atomicAdd(&fill[b], 1);
            const double2 s = pts[t];
            spi[o] = make_int2((int)(2.0 * s.x), (int)(2.0 * s.y));   // exact: multiples of 1/2
            sidx[o] = t;
        }
    }
    __syncthreads();
    unsigned bd[K];
    unsigned rej = ~0u;
    if (active) {
        const int qx2 = (int)(2.0 * qx), qy2 = (int)(2.0 * qy);
        auto key_of = [&](int t) -> unsigned {
            const int2 s = spi[t];
            const int dx = s.x - qx2, dy = s.y - qy2;
            return ((unsigned)(dx * dx + dy * dy) << 11) | (unsigned)sidx[t];
        };
#pragma unroll
        for (int q = 0; q < K; q++) bd[q] = key_of(q);   // total >= k == K
#pragma unroll
        for (int c = 0; c < net_size<K>(); c++) {
            const int a = net_a<K>(c), b = net_b<K>(c);
            const unsigned va = bd[a], vb = bd[b];
            bd[a] = min(va, vb);
            bd[b] = max(va, vb);
        }
        for (int t = K; t < total; t++) {
            const unsigned d2 = key_of(t);
            const unsigned wd = bd[K - 1];
            const bool better = d2 < wd;
            const unsigned gone = better ? wd : d2;
            rej = min(rej, gone);
            if (better) {
#pragma unroll
                for (int q = K - 1; q >= 1; q--) bd[q] = d2 < bd[q - 1] ? bd[q - 1] : (d2 < bd[q] ? d2 : bd[q]);
                if (d2 < bd[0]) bd[0] = d2;
            }
        }
    }
    tie_append(p, active && ((bd[K - 1] >> 11) == (rej >> 11)), i * p.nx + j);
    if (tid == 0) p.tile_done[blockIdx.y * gridDim.x + blockIdx.x] = 1;
    if (!active) return;
    fast_weights_store<K>(p, K, i, j, [&](int q, double &d2, int &id) {
        d2 = (double)(bd[q] >> 11) * 0.25;
        id = (int)(bd[q] & 2047u);
    });
}

// ---- device plan (b200_idw_plan) -----------------------------------------------------------------
// One CTA over the declustered vectors: the reference's early-outs and checks in their order
// (lucaskanade.py:245-269, decorators.py:190-208) and the key level the host path derives from the
// coordinates (xy * 16 integral with |xy| < 2^14; xy * 2 integral).
__global__ void __launch_bounds__(1024)
idw_plan_kernel(const int *__restrict__ counts, const double *__restrict__ xy, const double *__restrict__ uv,
                int cap, int grid_ok, B200IdwPlan *__restrict__ plan) {
    const int n_pool = counts[0], n_kept = counts[1];
    const int n = max(min(counts[2], cap), 0);
    const double u0 = n > 0 ? uv[0] : 0.0;
    bool bad_uv = false, bad_xy = false, differ = false, off16 = false, off2 = false;
    for (int t = threadIdx.x; t < 2 * n; t += blockDim.x) {
        const double u = uv[t], x = xy[t];
        bad_uv |= !isfinite(u);
        bad_xy |= !isfinite(x);
        differ |= !(u == u0);
        const double x16 = x * 16.0, x2 = x * 2.0;
        off16 |= !(x16 == rint(x16) && fabs(x) < 16384.0);
        off2 |= !(x2 == rint(x2));
    }
    bad_uv = __syncthreads_or(bad_uv);
    bad_xy = __syncthreads_or(bad_xy);
    differ = __syncthreads_or(differ);
    off16 = __syncthreads_or(off16);
    off2 = __syncthreads_or(off2);
    if (threadIdx.x != 0) return;
    B200IdwPlan r;
    r.n_pool = n_pool; r.n_kept = n_kept; r.n_dec = n;
    r.nonfinite = (bad_uv ? 1 : 0) | (bad_xy ? 2 : 0);
    r.on_grid = (grid_ok && !off16) ? (off2 ? 1 : 2) : 0;
    r.n_fill = 0;
    r.pad = 0;
    r.c0 = r.c1 = 0.0;
    if (n_pool == 0 || n == 0) {
        r.mode = B200_IDW_ZERO;
    } else if (bad_uv || bad_xy) {
        r.mode = B200_IDW_REFUSED;
    } else if (n == 1) {  // decorators.py:200-204
        r.mode = B200_IDW_CONSTANT;
        r.c0 = uv[0]; r.c1 = uv[1];
    } else if (!differ) {  // decorators.py:207-208, max == min: the first value everywhere
        r.mode = B200_IDW_CONSTANT;
        r.c0 = r.c1 = u0;
    } else {
        r.mode = B200_IDW_INTERPOLATE;
        r.n_fill = n;
    }
    *plan = r;
}

// the zero and constant fields of a plan, planar and (optionally) interleaved
__global__ void __launch_bounds__(256)
idw_plan_const_kernel(const B200IdwPlan *__restrict__ plan, double *__restrict__ out, double2 *__restrict__ twin,
                      size_t N) {
    const int mode = plan->mode;
    if (mode != B200_IDW_ZERO && mode != B200_IDW_CONSTANT) return;
    const double c0 = plan->c0, c1 = plan->c1;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < N; e += stride) {
        out[e] = c0;
        out[N + e] = c1;
        if (twin) twin[e] = make_double2(c0, c1);
    }
}

// ---- k = None: every vector weighs in (interpolate.py:82-88, scipy cdist) ------------------------
// One thread per grid point, the vectors staged through shared memory in chunks; weights and sums in
// float64 in index order (NumPy sums the same terms pairwise: relative differences ~1e-14).
constexpr int IDW_ALL_MAXVAR = 8;

__global__ void __launch_bounds__(256)
idw_all_kernel(const IDWParams p) {
    __shared__ double2 spt[1024];
    const int npts = p.npts_dev ? min(*p.npts_dev, p.npts_cap) : p.npts_cap;
    const int j = blockIdx.x * 32 + (threadIdx.x & 31), i = blockIdx.y * 8 + (threadIdx.x >> 5);
    const bool active = j < p.nx && i < p.ny;
    const double qx = p.gx[min(j, p.nx - 1)], qy = p.gy[min(i, p.ny - 1)];
    const double2 *__restrict__ pts = reinterpret_cast<const double2 *>(p.xy);
    double ws = 0.0, acc[IDW_ALL_MAXVAR];
#pragma unroll
    for (int v = 0; v < IDW_ALL_MAXVAR; v++) acc[v] = 0.0;
    for (int base = 0; base < npts; base += 1024) {
        const int cnt = min(1024, npts - base);
        __syncthreads();
        for (int t = threadIdx.x; t < cnt; t += 256) spt[t] = pts[base + t];
        __syncthreads();
        if (!active) continue;
        for (int t = 0; t < cnt; t++) {
            const double dx = __dsub_rn(spt[t].x, qx), dy = __dsub_rn(spt[t].y, qy);
            double d = sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
            if (p.mean_res != 1.0) d = __ddiv_rn(d, p.mean_res);
            d = __dadd_rn(d, p.offset);
            const double w = __ddiv_rn(1.0, (p.power == 0.5) ? sqrt(d) : pow(d, p.power));
            ws += w;
            for (int v = 0; v < p.nvar; v++) acc[v] += p.vals[(size_t)(base + t) * p.nvar + v] * w;
        }
    }
    if (!active) return;
    for (int v = 0; v < p.nvar; v++) p.out[((size_t)v * p.ny + i) * p.nx + j] = acc[v] / ws;
}

// library-internal side stream of the calling thread's device + fork/join events: the tree build
// (one CTA, latency bound) overlaps the exhaustive fill, the recomputation of the listed grid
// points waits for both
struct SideStream {
    cudaStream_t s = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
    int dev = -1;
};

int side_stream(SideStream **out) {
    static thread_local SideStream per_dev[16];
    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev));
    B200_REQUIRE(dev >= 0 && dev < 16, "device index out of range");
    SideStream &ss = per_dev[dev];
    if (ss.s == nullptr) {
        B200_CUDA(cudaStreamCreateWithFlags(&ss.s, cudaStreamNonBlocking));
        B200_CUDA(cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming));
        B200_CUDA(cudaEventCreateWithFlags(&ss.join, cudaEventDisableTiming));
        ss.dev = dev;
    }
    *out = &ss;
    return 0;
}

template <typename F>
void launch_tiles(F kernel, const IDWParams &p, dim3 grid, bool resident, cudaStream_t s) {
    kernel<<<resident ? resident_grid(kernel, grid) : grid, IDW_THREADS, 0, s>>>(p);
}

// Enqueues the kernel(s) of fill f (see idw_fill_kernel) on the full tile grid, or on one wave of
// resident CTAs.
int launch_fill(IdwFill f, IDWParams p, bool resident, b200::Scratch &done, cudaStream_t s) {
    const dim3 grid(b200::ceil_div(p.nx, IDW_TX), b200::ceil_div(p.ny, IDW_TY));
    const bool fastw = fast_weights(p);
    if (f == IDW_KEY32) {
        const size_t ntiles = (size_t)grid.x * grid.y;
        B200_CUDA(done.alloc(ntiles, s));
        B200_CUDA(cudaMemsetAsync(done.p, 0, ntiles, s));
        p.tile_done = (uint8_t *)done.p;
        idw32_kernel<20><<<grid, IDW_THREADS, 0, s>>>(p);
        B200_LAUNCH_CHECK();
        f = IDW_PACKED;  // over the tiles idw32_kernel leaves
    }
    if (f == IDW_PACKED && fastw) launch_tiles(idw_kernel<20, true, true, true>, p, grid, resident, s);
    else if (f == IDW_PACKED) launch_tiles(idw_kernel<20, true, true, false>, p, grid, resident, s);
    else if (f == IDW_UNPACKED && fastw) launch_tiles(idw_kernel<20, true, false, true>, p, grid, resident, s);
    else if (f == IDW_UNPACKED) launch_tiles(idw_kernel<20, true, false, false>, p, grid, resident, s);
    else launch_tiles(idw_kernel<32, false, false, false>, p, grid, resident, s);
    B200_LAUNCH_CHECK();
    return 0;
}

// The fill of both entry points for the p.npts_dev (or p.npts_cap) vectors: the cKDTree of the vectors on
// the side stream (see the header comment) while the fill kernels run on `s`, then the recomputation of
// the listed grid points.  Without a device plan the rule picks one fill from the key level `level`.  With
// one (p.plan) the plan's constant field is written first, and every fill the rule may pick is enqueued:
// the plan's usual choice on the full tile grid, the rare ones on one wave of resident CTAs.
int idw_run(IDWParams p, int level, cudaStream_t s) {
    const size_t N = (size_t)p.ny * p.nx;
    B200_REQUIRE(N < ((size_t)1 << 31), "grid too large");
    if (p.plan) {
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((N + 255) / 256, (size_t)b200::num_sms() * 8));
        idw_plan_const_kernel<<<blocks, 256, 0, s>>>(p.plan, p.out, p.twin, N);
        B200_LAUNCH_CHECK();
    }
    kdp::TreeScratch ts;
    b200::Scratch tie, done;
    SideStream *ss = nullptr;
    if (int rc = side_stream(&ss)) return rc;
    if (int rc = kdp::tree_alloc(ts, p.npts_cap, s)) return rc;
    B200_CUDA(tie.alloc(sizeof(int) * (N + 1), s));
    p.tie_count = (int *)tie.p;
    p.tie_list = p.tie_count + 1;
    B200_CUDA(cudaMemsetAsync(p.tie_count, 0, sizeof(int), s));
    B200_CUDA(cudaEventRecord(ss->fork, s));
    B200_CUDA(cudaStreamWaitEvent(ss->s, ss->fork, 0));
    if (int rc = kdp::tree_build(p.xy, p.npts_dev, p.npts_cap, ts.tb, ss->s)) return rc;
    B200_CUDA(cudaEventRecord(ss->join, ss->s));
    if (!p.plan) {
        const IdwFill f = p.npts_dev ? IDW_INSERT : idw_fill_kernel(p.k, p.npts_cap, level, fast_weights(p));
        if (int rc = launch_fill(f, p, false, done, s)) return rc;
    } else {
        if (p.k >= 20) {  // min(k, n_fill) can be 20
            if (int rc = launch_fill(fast_weights(p) ? IDW_KEY32 : IDW_PACKED, p, false, done, s)) return rc;
            if (int rc = launch_fill(IDW_UNPACKED, p, true, done, s)) return rc;
        }
        if (int rc = launch_fill(IDW_INSERT, p, true, done, s)) return rc;
    }
    B200_CUDA(cudaStreamWaitEvent(s, ss->join, 0));
    return kdp::idw_fix(p.xy, p.vals, p.nvar, p.k, p.power, p.offset, p.mean_res, p.gx, p.nx, p.gy, p.ny, ts.tb,
                        p.tie_list, p.tie_count, p.out, p.twin, s);
}

}  // namespace

extern "C" int b200_idw_fill(const double *xy, const double *vals, const int *npts_dev, int npts_cap,
                             int nvar, int k, double power, double dist_offset, double mean_res,
                             const double *xgrid, int nx, const double *ygrid, int ny,
                             int coords_on_16th_grid, double *out, void *stream) {
    B200_REQUIRE(xy && vals && xgrid && ygrid && out && npts_cap >= 1 && nvar >= 1 && nx >= 1 && ny >= 1 &&
                     k >= 1, "bad arguments");
    if (k > 32) {
        b200::set_error("idw: k must be <= 32 (k=None / larger k is not implemented)");
        return B200_ENOTSUP;
    }
    IDWParams p = {};
    p.xy = xy; p.vals = vals; p.npts_dev = npts_dev; p.npts_cap = npts_cap; p.nvar = nvar; p.k = k;
    p.gx = xgrid; p.gy = ygrid; p.nx = nx; p.ny = ny;
    p.power = power; p.offset = dist_offset; p.mean_res = mean_res; p.out = out;
    // the caller vouches for the key level: every coordinate (vectors and grid) a multiple of 1/16
    // below 2^14, and with 2 also the vectors on the half-pixel grid and the grid on integers
    return idw_run(p, coords_on_16th_grid, (cudaStream_t)stream);
}

extern "C" int b200_idw_plan(const int *counts, const double *xy, const double *uv, int cap, int grid_ok,
                             B200IdwPlan *plan, void *stream) {
    B200_REQUIRE(counts && xy && uv && plan && cap >= 1, "bad arguments");
    idw_plan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(counts, xy, uv, cap, grid_ok, plan);
    B200_LAUNCH_CHECK();
    return 0;
}

// b200_idw_fill with the vector count, the key level and the early-outs taken from a device plan: every
// kernel that may fill the field is enqueued (grids and scratch sized from the capacity) and each returns
// at once unless the rule of b200_idw_fill, applied to the plan, gives it the field; the zero and
// constant fields are written by idw_plan_const_kernel.  The field is therefore b200_idw_fill's for the
// same vectors, bit for bit.
extern "C" int b200_idw_fill_planned(const double *xy, const double *vals, const B200IdwPlan *plan, int npts_cap,
                                     int k, double power, double dist_offset, const double *xgrid, int nx,
                                     const double *ygrid, int ny, double *out, double *twin, void *stream) {
    B200_REQUIRE(xy && vals && plan && xgrid && ygrid && out && npts_cap >= 1 && nx >= 1 && ny >= 1 && k >= 1,
                 "bad arguments");
    if (k > 32) {
        b200::set_error("idw: k must be <= 32 (k=None / larger k is not implemented)");
        return B200_ENOTSUP;
    }
    IDWParams p = {};
    p.xy = xy; p.vals = vals; p.npts_dev = &plan->n_fill; p.npts_cap = npts_cap; p.nvar = 2; p.k = k;
    p.gx = xgrid; p.gy = ygrid; p.nx = nx; p.ny = ny;
    p.power = power; p.offset = dist_offset; p.mean_res = 1.0; p.out = out; p.twin = (double2 *)twin;
    p.plan = plan;
    return idw_run(p, 0, (cudaStream_t)stream);  // the plan holds the key level
}

extern "C" int b200_idw_fill_all(const double *xy, const double *vals, const int *npts_dev, int npts_cap, int nvar,
                                 double power, double dist_offset, double mean_res, const double *xgrid, int nx,
                                 const double *ygrid, int ny, double *out, void *stream) {
    B200_REQUIRE(xy && vals && xgrid && ygrid && out && npts_cap >= 1 && nx >= 1 && ny >= 1, "bad arguments");
    B200_REQUIRE(nvar >= 1 && nvar <= IDW_ALL_MAXVAR, "at most 8 variables");
    IDWParams p;
    memset(&p, 0, sizeof(p));
    p.xy = xy; p.vals = vals; p.npts_dev = npts_dev; p.npts_cap = npts_cap; p.nvar = nvar; p.k = npts_cap;
    p.gx = xgrid; p.gy = ygrid; p.nx = nx; p.ny = ny;
    p.power = power; p.offset = dist_offset; p.mean_res = mean_res; p.out = out;
    idw_all_kernel<<<dim3(b200::ceil_div(nx, 32), b200::ceil_div(ny, 8)), 256, 0, (cudaStream_t)stream>>>(p);
    B200_LAUNCH_CHECK();
    return 0;
}
