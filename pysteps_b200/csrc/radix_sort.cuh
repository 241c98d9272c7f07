// radix_sort.cuh -- the stable LSD radix sort of (64-bit key, 32-bit index) pairs and a three-kernel
// scan on the block scans of scan.cuh, shared by salient blending (blending.cu) and probability
// matching (probmatching.cu), sm_90a.
//   keys       order_key: an order-preserving 64-bit image of a double, -0.0 equal to +0.0
//   sort       8-bit digits, least significant first; one global histogram of all eight digits
//              plans the passes, and a digit that every key shares is skipped (plan_passes).  Each
//              pass counts its digit per tile, scans the counts and scatters every tile stably.
//   scan       scan_reduce / scan_blocks / scan_apply: an exclusive scan of unsigned values over an
//              Op that loads and stores them, in a fixed order (no atomics), so results repeat bit
//              for bit.
#pragma once
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace {

using b200::Carver;
using b200::quiet_nan;

constexpr int THREADS = 256;
constexpr int SORT_ITEMS = 16;
constexpr int TILE = THREADS * SORT_ITEMS;  // keys per radix tile and per scan block
constexpr int RADIX = 256;
constexpr int PASSES = 8;
constexpr unsigned FULL = 0xffffffffu;

// order-preserving 64-bit image of a double; -0.0 maps to +0.0 (rankdata treats them as equal)
__device__ __forceinline__ unsigned long long order_key(double d) {
    unsigned long long u = (unsigned long long)__double_as_longlong(d == 0.0 ? 0.0 : d);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_value(unsigned long long k) {
    if (k == ~0ull) return quiet_nan();
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// the double buffers of one sort of up to n keys, and the counts its passes scan
struct SortBuffers {
    unsigned long long *key[2];
    unsigned *idx[2];
    unsigned *tiles;  // RADIX x n_tiles digit counts, digit-major, then their exclusive scan
    unsigned *bsum;   // per scan block sums (also large enough for a scan over n values)
    unsigned *ghist;  // PASSES x RADIX global digit counts
    int *src;         // PASSES + 1: buffer each pass reads (-1: pass skipped); [PASSES]: the final buffer
};

static void carve_sort(SortBuffers *s, Carver &c, int64_t n) {
    const int64_t n_tiles = b200::ceil_div64(std::max<int64_t>(n, 1), TILE);
    const int64_t n_scan = std::max<int64_t>(RADIX * n_tiles, n);
    const int64_t n_bsum = b200::ceil_div64(n_scan, TILE);
    s->key[0] = (unsigned long long *)c.take(8 * n);
    s->key[1] = (unsigned long long *)c.take(8 * n);
    s->idx[0] = (unsigned *)c.take(4 * n);
    s->idx[1] = (unsigned *)c.take(4 * n);
    s->tiles = (unsigned *)c.take(4 * RADIX * n_tiles);
    s->bsum = (unsigned *)c.take(4 * n_bsum);
    s->ghist = (unsigned *)c.take(4 * PASSES * RADIX);
    s->src = (int *)c.take(4 * (PASSES + 1));
}

__global__ void __launch_bounds__(THREADS)
    global_hist(const unsigned long long *__restrict__ key, int64_t n, unsigned *__restrict__ ghist) {
    __shared__ unsigned h[PASSES][RADIX];
    for (int t = threadIdx.x; t < PASSES * RADIX; t += THREADS) (&h[0][0])[t] = 0;
    __syncthreads();
    for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n; j += (int64_t)gridDim.x * THREADS) {
        const unsigned long long k = key[j];
#pragma unroll
        for (int d = 0; d < PASSES; d++) atomicAdd(&h[d][(k >> (8 * d)) & 255], 1u);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < PASSES * RADIX; t += THREADS)
        if ((&h[0][0])[t]) atomicAdd(ghist + t, (&h[0][0])[t]);
}

// src[d]: the buffer pass d reads, or -1 when every key has the same digit d (the pass is skipped)
__global__ void plan_passes(const unsigned *__restrict__ ghist, int64_t n, int *__restrict__ src) {
    if (threadIdx.x != 0) return;
    int cur = 0;
    for (int d = 0; d < PASSES; d++) {
        bool trivial = false;
        for (int b = 0; b < RADIX; b++) trivial |= (int64_t)ghist[d * RADIX + b] == n;
        src[d] = trivial ? -1 : cur;
        if (!trivial) cur ^= 1;
    }
    src[PASSES] = cur;
}

__global__ void __launch_bounds__(THREADS)
    tile_hist(SortBuffers s, int64_t n, int64_t n_tiles, int pass) {
    const int b = s.src[pass];
    if (b < 0) return;
    __shared__ unsigned h[RADIX];
    h[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long *key = s.key[b];
    const int64_t t0 = (int64_t)blockIdx.x * TILE;
    for (int r = 0; r < SORT_ITEMS; r++) {
        const int64_t j = t0 + r * THREADS + threadIdx.x;
        if (j < n) atomicAdd(&h[(key[j] >> (8 * pass)) & 255], 1u);
    }
    __syncthreads();
    s.tiles[(int64_t)threadIdx.x * n_tiles + blockIdx.x] = h[threadIdx.x];
}

// the scan over the tile counts of a pass (exclusive, in place)
struct CountScan {
    SortBuffers s;
    int pass;
    __device__ bool skip() const { return s.src[pass] < 0; }
    __device__ unsigned load(int64_t i) const { return s.tiles[i]; }
    __device__ void store(int64_t i, unsigned excl, unsigned) const { s.tiles[i] = excl; }
};

// An Op has skip() (the whole scan is skipped), load(i) (the value at i) and store(i, excl, v) (the
// exclusive prefix sum before i and the value at i); store is called for every i < n.
template <typename Op>
__global__ void __launch_bounds__(THREADS) scan_reduce(Op op, int64_t n, unsigned *__restrict__ bsum) {
    if (op.skip()) return;
    __shared__ unsigned sh[THREADS / 32];
    const int64_t i0 = (int64_t)blockIdx.x * TILE + (int64_t)threadIdx.x * SORT_ITEMS;
    unsigned v = 0;
    for (int r = 0; r < SORT_ITEMS; r++)
        if (i0 + r < n) v += op.load(i0 + r);
    unsigned total;
    b200::block_exclusive_scan<THREADS>(v, sh, &total);
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

template <typename Op>
__global__ void __launch_bounds__(THREADS) scan_blocks(Op op, int64_t nb, unsigned *__restrict__ bsum) {
    if (op.skip()) return;
    b200::single_cta_scan<THREADS>(bsum, nb, bsum);
}

template <typename Op>
__global__ void __launch_bounds__(THREADS) scan_apply(Op op, int64_t n, const unsigned *__restrict__ bsum) {
    if (op.skip()) return;
    __shared__ unsigned sh[THREADS / 32];
    const int64_t i0 = (int64_t)blockIdx.x * TILE + (int64_t)threadIdx.x * SORT_ITEMS;
    unsigned v[SORT_ITEMS];
    unsigned sum = 0;
#pragma unroll
    for (int r = 0; r < SORT_ITEMS; r++) {
        v[r] = i0 + r < n ? op.load(i0 + r) : 0;
        sum += v[r];
    }
    unsigned total;
    unsigned run = bsum[blockIdx.x] + b200::block_exclusive_scan<THREADS>(sum, sh, &total);
#pragma unroll
    for (int r = 0; r < SORT_ITEMS; r++) {
        if (i0 + r < n) op.store(i0 + r, run, v[r]);
        run += v[r];
    }
}

// the three launches of one scan over n values; bsum holds ceil(n / TILE) values
template <typename Op> int scan(const Op &op, int64_t n, unsigned *bsum, cudaStream_t st) {
    if (n == 0) return 0;
    const int64_t nb = b200::ceil_div64(n, TILE);
    scan_reduce<<<(unsigned)nb, THREADS, 0, st>>>(op, n, bsum);
    B200_LAUNCH_CHECK();
    scan_blocks<<<1, THREADS, 0, st>>>(op, nb, bsum);
    B200_LAUNCH_CHECK();
    scan_apply<<<(unsigned)nb, THREADS, 0, st>>>(op, n, bsum);
    B200_LAUNCH_CHECK();
    return 0;
}

// stable scatter of one tile: keys are taken in index order, ranked within their warp by
// __match_any_sync and across the warps of a round by a per-digit scan in shared memory
__global__ void __launch_bounds__(THREADS) scatter_pass(SortBuffers s, int64_t n, int64_t n_tiles, int pass) {
    const int b = s.src[pass];
    if (b < 0) return;
    __shared__ unsigned base[RADIX];
    __shared__ unsigned wcnt[THREADS / 32][RADIX];
    __shared__ unsigned round_total[RADIX];
    const unsigned long long *ksrc = s.key[b];
    const unsigned *isrc = s.idx[b];
    unsigned long long *kdst = s.key[b ^ 1];
    unsigned *idst = s.idx[b ^ 1];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    base[threadIdx.x] = s.tiles[(int64_t)threadIdx.x * n_tiles + blockIdx.x];
    const int64_t t0 = (int64_t)blockIdx.x * TILE;
    for (int r = 0; r < SORT_ITEMS; r++) {
        for (int q = 0; q < THREADS / 32; q++) wcnt[q][threadIdx.x] = 0;
        __syncthreads();
        const int64_t j = t0 + (int64_t)r * THREADS + threadIdx.x;
        const bool valid = j < n;
        const unsigned long long k = valid ? ksrc[j] : 0ull;
        const unsigned digit = valid ? (unsigned)((k >> (8 * pass)) & 255) : RADIX + lane;
        const unsigned peers = __match_any_sync(FULL, digit);
        const unsigned below = __popc(peers & ((1u << lane) - 1u));
        if (valid && below == 0) wcnt[w][digit] = __popc(peers);
        __syncthreads();
        unsigned acc = 0;
        for (int q = 0; q < THREADS / 32; q++) {
            const unsigned c = wcnt[q][threadIdx.x];
            wcnt[q][threadIdx.x] = acc;
            acc += c;
        }
        round_total[threadIdx.x] = acc;
        __syncthreads();
        if (valid) {
            const unsigned pos = base[digit] + wcnt[w][digit] + below;
            kdst[pos] = k;
            idst[pos] = isrc[j];
        }
        __syncthreads();
        base[threadIdx.x] += round_total[threadIdx.x];
    }
}

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(b200::ceil_div64(n, THREADS), 132 * 16)); }

// sort the n keys in s.key[0] / s.idx[0] stably; the sorted pairs end in buffer s.src[PASSES]
// (a device value: kernels that read the result look it up there)
int radix_sort(const SortBuffers &s, int64_t n, cudaStream_t st) {
    if (n == 0) return 0;
    const int64_t n_tiles = b200::ceil_div64(n, TILE);
    B200_CUDA(cudaMemsetAsync(s.ghist, 0, 4 * PASSES * RADIX, st));
    global_hist<<<grid_for(n), THREADS, 0, st>>>(s.key[0], n, s.ghist);
    B200_LAUNCH_CHECK();
    plan_passes<<<1, 32, 0, st>>>(s.ghist, n, s.src);
    B200_LAUNCH_CHECK();
    const int64_t n_counts = RADIX * n_tiles;
    for (int d = 0; d < PASSES; d++) {
        tile_hist<<<(unsigned)n_tiles, THREADS, 0, st>>>(s, n, n_tiles, d);
        B200_LAUNCH_CHECK();
        if (int rc = scan(CountScan{s, d}, n_counts, s.bsum, st)) return rc;
        scatter_pass<<<(unsigned)n_tiles, THREADS, 0, st>>>(s, n, n_tiles, d);
        B200_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace
