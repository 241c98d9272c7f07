// constant.cu -- the objective of the constant advection method (pysteps/motion/constant.py:41-49)
// on the device (sm_90a): one call is one evaluation of
//   f(v) = -corrcoef(next[mask], warped[mask])[0, 1]
// at the point v = (vx, vy) Nelder-Mead visits.  Six kernels, all on the caller's stream:
//   count    per 1024-pixel tile: how many pixels count (next finite, the order-0 tap of prev at
//            (y + vy, x + vx) inside the frame and finite -- the rule of spline_body.cuh)
//   scan     one CTA: exclusive tile offsets and N
//   compact  the counted pixels' values, in raster order, as two float64 rows
//   mean     NumPy's pairwise sum of each row (np.add.reduce: leaves of <= 128 values summed with
//            8 accumulators, split n/2 rounded down to a multiple of 8), bit for bit
//   centred  S00, S11, S01 in a fixed order (lane i % 65536, then a tree in each CTA)
//   tail     corrcoef's arithmetic after the dot product, in NumPy's order, and its warning bits
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"
#include "spline_body.cuh"

namespace {

using spl::add;
using spl::dvd;
using spl::mul;
using spl::sub;

constexpr int TILE_THREADS = 256, PER_THREAD = 4, TILE = TILE_THREADS * PER_THREAD;
constexpr int SCAN_THREADS = 1024;
constexpr int LEAF = 128;  // numpy's PW_BLOCKSIZE
constexpr int CHUNK = 64;  // below the root every leaf holds >= 64 values: one leaf start per chunk
constexpr int SUM_THREADS = 256, SUM_LANES = B200_CONST_SUM_BLOCKS * SUM_THREADS;
constexpr int MAX_DEPTH = 40;

// the pieces of one evaluation's scratch, carved from scratch (nullptr: only their size in bytes)
struct Layout {
    int64_t P, tiles, chunks, bytes;
    int *tile_count, *tile_off;
    long long *count;
    double *means, *part, *a, *b, *leafval, *nodeval;
    unsigned *arrive;
};

Layout layout(int m, int n, char *scratch) {
    Layout L;
    L.P = (int64_t)m * n;
    L.tiles = b200::ceil_div64(L.P, TILE);
    L.chunks = std::max<int64_t>(1, b200::ceil_div64(L.P, CHUNK));
    b200::Carver c{scratch};
    L.tile_count = (int *)c.take(sizeof(int) * L.tiles);
    L.tile_off = (int *)c.take(sizeof(int) * L.tiles);
    L.count = (long long *)c.take(sizeof(long long));
    L.means = (double *)c.take(2 * sizeof(double));
    L.part = (double *)c.take(3 * sizeof(double) * B200_CONST_SUM_BLOCKS);
    L.a = (double *)c.take(sizeof(double) * L.P);
    L.b = (double *)c.take(sizeof(double) * L.P);
    L.leafval = (double *)c.take(2 * sizeof(double) * L.chunks);
    L.nodeval = (double *)c.take(2 * sizeof(double) * L.chunks);
    L.arrive = (unsigned *)c.take(sizeof(unsigned) * L.chunks);
    L.bytes = c.off;
    return L;
}

struct Eval {
    const void *prev, *next;
    int m, n;
    double vx, vy;
};

// pixel p counts: its values go to the two rows of corrcoef (next[p], warped[p])
template <typename F>
__device__ __forceinline__ bool counted(const Eval &e, int64_t p, double &va, double &vb) {
    const double a = (double)static_cast<const F *>(e.next)[p];
    if (!isfinite(a)) return false;
    const int y = (int)(p / e.n), x = (int)(p % e.n);
    const double cy = add((double)y, e.vy), cx = add((double)x, e.vx);  // Y + v[1], X + v[0]
    if (spl::outside_grid(cy, cx, e.m, e.n)) return false;               // cval = nan
    const double b = add(0.0, (double)static_cast<const F *>(e.prev)[spl::order0_index(cy, cx, e.m, e.n,
                                                                                        B200_MODE_CONSTANT)]);
    if (!isfinite(b)) return false;
    va = a;
    vb = b;
    return true;
}

template <typename F>
__global__ void __launch_bounds__(TILE_THREADS) count_kernel(const Eval e, int64_t P, int *__restrict__ tile_count) {
    __shared__ int sh[TILE_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * TILE + (int64_t)threadIdx.x * PER_THREAD;
    int c = 0;
    for (int k = 0; k < PER_THREAD; k++) {
        double a, b;
        if (base + k < P && counted<F>(e, base + k, a, b)) c++;
    }
    int total;
    b200::block_exclusive_scan<TILE_THREADS>(c, sh, &total);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = total;
}

// one CTA: tile_off = exclusive prefix of tile_count, *count = N
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const int *__restrict__ tile_count, int64_t tiles,
                                                            int *__restrict__ tile_off, long long *__restrict__ count) {
    __shared__ int sh[SCAN_THREADS / 32];
    const int64_t seg = (tiles + SCAN_THREADS - 1) / SCAN_THREADS;
    const int64_t lo = min(tiles, (int64_t)threadIdx.x * seg), hi = min(tiles, lo + seg);
    int s = 0;
    for (int64_t t = lo; t < hi; t++) s += tile_count[t];
    int total;
    int run = b200::block_exclusive_scan<SCAN_THREADS>(s, sh, &total);
    for (int64_t t = lo; t < hi; t++) {
        tile_off[t] = run;
        run += tile_count[t];
    }
    if (threadIdx.x == 0) *count = total;
}

template <typename F>
__global__ void __launch_bounds__(TILE_THREADS) compact_kernel(const Eval e, int64_t P, const int *__restrict__ tile_off,
                                                               double *__restrict__ ra, double *__restrict__ rb) {
    __shared__ int sh[TILE_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * TILE + (int64_t)threadIdx.x * PER_THREAD;
    double va[PER_THREAD], vb[PER_THREAD];
    bool ok[PER_THREAD];
    int c = 0;
    for (int k = 0; k < PER_THREAD; k++) {
        ok[k] = base + k < P && counted<F>(e, base + k, va[k], vb[k]);
        c += ok[k];
    }
    int total;
    int64_t rank = (int64_t)tile_off[blockIdx.x] + b200::block_exclusive_scan<TILE_THREADS>(c, sh, &total);
    for (int k = 0; k < PER_THREAD; k++)
        if (ok[k]) {
            ra[rank] = va[k];
            rb[rank] = vb[k];
            rank++;
        }
}

// numpy's pairwise_sum (loops_utils.h.src) over a[lo, lo + n), n <= LEAF
__device__ double leaf_sum(const double *__restrict__ a, int64_t lo, int64_t n) {
    if (n < 8) {
        double res = 0.0;
        for (int64_t i = 0; i < n; i++) res = add(res, a[lo + i]);
        return res;
    }
    double r[8];
    for (int j = 0; j < 8; j++) r[j] = a[lo + j];
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; j++) r[j] = add(r[j], a[lo + i + j]);
    double res = add(add(add(r[0], r[1]), add(r[2], r[3])), add(add(r[4], r[5]), add(r[6], r[7])));
    for (; i < n; i++) res = add(res, a[lo + i]);
    return res;
}

// size of the left half of a node of n > LEAF values: n / 2 rounded down to a multiple of 8
__device__ __forceinline__ int64_t split_of(int64_t n) { return (n >> 1) & ~(int64_t)7; }

struct Node {
    int64_t off, n;
};

// the leaf holding rank r of the tree over [0, N); path[0, depth) = its ancestors, root first
__device__ int descend(int64_t N, int64_t r, Node *path, Node *leaf) {
    int64_t off = 0, n = N;
    int d = 0;
    while (n > LEAF) {
        path[d++] = Node{off, n};
        const int64_t h = split_of(n);
        if (r < off + h) {
            n = h;
        } else {
            off += h;
            n -= h;
        }
    }
    *leaf = Node{off, n};
    return d;
}

// a node's sum: a leaf's is stored at the chunk of its first rank, an inner node's at the chunk of
// its split (every rank where one leaf ends and the next begins is the split of exactly one node)
__device__ __forceinline__ double node_value(const double *leafval, const double *nodeval, int64_t chunks, int row,
                                             int64_t off, int64_t n) {
    if (n <= LEAF) return __ldcg(leafval + row * chunks + off / CHUNK);
    return __ldcg(nodeval + row * chunks + (off + split_of(n)) / CHUNK);
}

// One thread per chunk of 64 ranks sums the leaf that starts in it, then climbs: the second of two
// siblings to arrive at their parent adds them (left + right), so every inner node is the sum numpy
// forms, whatever the order of arrival.  The root's sum gives the means (0.0 + sum) / N.
__global__ void __launch_bounds__(256) mean_kernel(const double *__restrict__ ra, const double *__restrict__ rb,
                                                   const long long *__restrict__ count, int64_t chunks,
                                                   double *leafval, double *nodeval, unsigned *arrive,
                                                   double *__restrict__ means) {
    const int64_t N = *count;
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (N <= LEAF) {  // the root is a leaf (N == 0: 0 / 0 = nan, as np.mean of an empty row)
        if (c == 0) {
            means[0] = dvd(add(0.0, leaf_sum(ra, 0, N)), (double)N);
            means[1] = dvd(add(0.0, leaf_sum(rb, 0, N)), (double)N);
        }
        return;
    }
    const int64_t s0 = c * CHUNK;
    if (s0 >= N) return;
    Node path[MAX_DEPTH], leaf;
    int depth = descend(N, s0, path, &leaf);
    if (leaf.off != s0) {  // the leaf holding s0 started earlier: does the next one start in this chunk?
        const int64_t nxt = leaf.off + leaf.n;
        if (nxt >= s0 + CHUNK || nxt >= N) return;
        depth = descend(N, nxt, path, &leaf);
    }
    double v0 = leaf_sum(ra, leaf.off, leaf.n), v1 = leaf_sum(rb, leaf.off, leaf.n);
    leafval[leaf.off / CHUNK] = v0;
    leafval[chunks + leaf.off / CHUNK] = v1;
    for (int d = depth - 1; d >= 0; d--) {
        const Node p = path[d];
        const int64_t h = split_of(p.n), slot = (p.off + h) / CHUNK;
        __threadfence();
        if (atomicAdd(arrive + slot, 1u) == 0u) return;  // the sibling is not done yet: it climbs on
        arrive[slot] = 0u;                                // ready for the next evaluation
        __threadfence();
        v0 = add(node_value(leafval, nodeval, chunks, 0, p.off, h), node_value(leafval, nodeval, chunks, 0, p.off + h, p.n - h));
        v1 = add(node_value(leafval, nodeval, chunks, 1, p.off, h), node_value(leafval, nodeval, chunks, 1, p.off + h, p.n - h));
        if (d == 0) {
            means[0] = dvd(add(0.0, v0), (double)N);
            means[1] = dvd(add(0.0, v1), (double)N);
        } else {
            nodeval[slot] = v0;
            nodeval[chunks + slot] = v1;
        }
    }
}

// X -= avg[:, None]; the three distinct entries of dot(X, X.T): lane g sums ranks g, g + 65536, ...
// in sequence, then a halving tree inside the CTA
__global__ void __launch_bounds__(SUM_THREADS) centred_kernel(const double *__restrict__ ra, const double *__restrict__ rb,
                                                              const long long *__restrict__ count,
                                                              const double *__restrict__ means, double *__restrict__ part) {
    __shared__ double sh[3][SUM_THREADS];
    const int64_t N = *count;
    double s00 = 0.0, s11 = 0.0, s01 = 0.0;
    if (N > 0) {
        const double ma = means[0], mb = means[1];
        for (int64_t i = (int64_t)blockIdx.x * SUM_THREADS + threadIdx.x; i < N; i += SUM_LANES) {
            const double xa = sub(ra[i], ma), xb = sub(rb[i], mb);
            s00 = add(s00, mul(xa, xa));
            s11 = add(s11, mul(xb, xb));
            s01 = add(s01, mul(xa, xb));
        }
    }
    const int t = threadIdx.x;
    sh[0][t] = s00;
    sh[1][t] = s11;
    sh[2][t] = s01;
    __syncthreads();
    for (int s = SUM_THREADS / 2; s > 0; s >>= 1) {
        if (t < s)
            for (int k = 0; k < 3; k++) sh[k][t] = add(sh[k][t], sh[k][t + s]);
        __syncthreads();
    }
    if (t < 3) part[3 * blockIdx.x + t] = sh[t][0];
}

// the floating-point events of one quotient x / y under IEEE rules (NaN operands raise nothing)
__device__ int quotient_events(double x, double y, int invalid, int divzero, int overflow) {
    if (isnan(x) || isnan(y)) return 0;
    if ((x == 0.0 && y == 0.0) || (isinf(x) && isinf(y))) return invalid;
    if (y == 0.0) return isinf(x) ? 0 : divzero;
    if (isfinite(x) && isinf(dvd(x, y))) return overflow;
    return 0;
}

// corrcoef after the dot product (numpy/lib/_function_base_impl.py cov and corrcoef): c *= 1/fact,
// stddev = sqrt(diag(c)), c /= stddev[:, None], c /= stddev[None, :], clip to [-1, 1]
__global__ void tail_kernel(const long long *__restrict__ count, const double *__restrict__ part,
                            double *__restrict__ record) {
    const int64_t N = *count;
    double S[3] = {0.0, 0.0, 0.0};  // S00, S11, S01
    for (int g = 0; g < B200_CONST_SUM_BLOCKS; g++)
        for (int k = 0; k < 3; k++) S[k] = add(S[k], part[3 * g + k]);
    int flags = N == 0 ? B200_CONST_EMPTY : 0;
    double fact = (double)(N - 1);
    if (N - 1 <= 0) {
        flags |= B200_CONST_DOF;
        fact = 0.0;
    }
    const double inv = dvd(1.0, fact);
    double c[2][2] = {{S[0], S[2]}, {S[2], S[1]}};
    for (int i = 0; i < 2; i++)
        for (int j = 0; j < 2; j++) {
            if ((c[i][j] == 0.0 && isinf(inv)) || (isinf(c[i][j]) && inv == 0.0)) flags |= B200_CONST_SCALE_INVALID;
            c[i][j] = mul(c[i][j], inv);
        }
    const double sd[2] = {sqrt(c[0][0]), sqrt(c[1][1])};
    for (int i = 0; i < 2; i++)
        for (int j = 0; j < 2; j++) {
            flags |= quotient_events(c[i][j], sd[i], B200_CONST_ROW_INVALID, B200_CONST_ROW_DIVZERO,
                                     B200_CONST_ROW_OVERFLOW);
            c[i][j] = dvd(c[i][j], sd[i]);
        }
    for (int i = 0; i < 2; i++)
        for (int j = 0; j < 2; j++) {
            flags |= quotient_events(c[i][j], sd[j], B200_CONST_COL_INVALID, B200_CONST_COL_DIVZERO,
                                     B200_CONST_COL_OVERFLOW);
            c[i][j] = dvd(c[i][j], sd[j]);
        }
    const double r = c[0][1] < -1.0 ? -1.0 : (c[0][1] > 1.0 ? 1.0 : c[0][1]);  // NaN stays NaN
    record[0] = -r;
    record[1] = (double)N;
    record[2] = (double)flags;
}

template <typename F>
int eval(const Eval &e, const Layout &L, double *record, cudaStream_t s) {
    if (L.tiles > 0) {
        count_kernel<F><<<(unsigned)L.tiles, TILE_THREADS, 0, s>>>(e, L.P, L.tile_count);
        B200_LAUNCH_CHECK();
    }
    scan_kernel<<<1, SCAN_THREADS, 0, s>>>(L.tile_count, L.tiles, L.tile_off, L.count);
    B200_LAUNCH_CHECK();
    if (L.tiles > 0) {
        compact_kernel<F><<<(unsigned)L.tiles, TILE_THREADS, 0, s>>>(e, L.P, L.tile_off, L.a, L.b);
        B200_LAUNCH_CHECK();
    }
    mean_kernel<<<(unsigned)b200::ceil_div64(L.chunks, 256), 256, 0, s>>>(L.a, L.b, L.count, L.chunks, L.leafval,
                                                                           L.nodeval, L.arrive, L.means);
    B200_LAUNCH_CHECK();
    centred_kernel<<<B200_CONST_SUM_BLOCKS, SUM_THREADS, 0, s>>>(L.a, L.b, L.count, L.means, L.part);
    B200_LAUNCH_CHECK();
    tail_kernel<<<1, 1, 0, s>>>(L.count, L.part, record);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int b200_constant_scratch_bytes(int m, int n, int64_t *bytes) {
    B200_REQUIRE(m >= 0 && n >= 0 && bytes != nullptr, "bad arguments");
    B200_REQUIRE((int64_t)m * n <= (int64_t)1 << 30, "constant: frames of more than 2^30 pixels are not supported");
    *bytes = layout(m, n, nullptr).bytes;
    return 0;
}

extern "C" int b200_constant_eval(const void *prev, const void *next, int dtype, int m, int n, double vx, double vy,
                                  void *scratch, double *record, void *stream) {
    B200_REQUIRE(m >= 0 && n >= 0 && scratch != nullptr && record != nullptr, "bad arguments");
    B200_REQUIRE((int64_t)m * n <= (int64_t)1 << 30, "constant: frames of more than 2^30 pixels are not supported");
    B200_REQUIRE((int64_t)m * n == 0 || (prev != nullptr && next != nullptr), "bad arguments");
    const Layout L = layout(m, n, (char *)scratch);
    const Eval e{prev, next, m, n, vx, vy};
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("frame", dtype, [&](auto t) { return eval<typename decltype(t)::type>(e, L, record, s); });
}
