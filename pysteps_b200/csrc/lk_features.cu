// lk_features.cu -- corner selection of cv::goodFeaturesToTrack on the device (sm_90a).
//
// Reference call site: pysteps/feature/shitomasi.py:153-162 (cv2.goodFeaturesToTrack with
// maxCorners, qualityLevel, minDistance, mask, blockSize=5).  Given the minimum-eigenvalue
// map (lk_dense.cu) OpenCV: (1) takes the maximum over the mask, (2) zeroes everything
// <= quality * max, (3) keeps pixels equal to their 3x3 dilation, non-zero, inside the mask
// and off the 1-pixel border, (4) sorts them by value descending (ties: larger raster
// address first), (5) accepts greedily if the squared distance to every accepted corner is
// >= minDistance^2, stopping at maxCorners.  Steps 1-3 are streaming passes; 4 is a bitonic
// sort of 64-bit keys (order-preserving value bits << 32 | address); 5 is inherently ordered
// and runs as one warp that tests 32 candidates at a time against a cell grid and resolves the
// order inside the batch with shuffles -- results are identical to the sequential loop.
#include <math_constants.h>

#include "common.cuh"

namespace {

constexpr int TX = 32, TY = 8;

// ---- (1) max over the mask -----------------------------------------------------------
__global__ void __launch_bounds__(256)
masked_max_partial(const float *__restrict__ eig, const uint8_t *__restrict__ valid, size_t N,
                   float *__restrict__ part) {
    __shared__ float sm[8];
    float v = -CUDART_INF_F;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride)
        if (!valid || valid[i]) v = fmaxf(v, eig[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        v = threadIdx.x < 8 ? sm[threadIdx.x] : -CUDART_INF_F;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
        if (threadIdx.x == 0) part[blockIdx.x] = v;
    }
}

// state[0] = threshold as float bits, state[1] = candidate count (reset here)
__global__ void __launch_bounds__(256)
masked_max_final(const float *__restrict__ part, int nparts, double quality, unsigned *__restrict__ state) {
    __shared__ float sm[8];
    float v = -CUDART_INF_F;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) v = fmaxf(v, part[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; i++) v = fmaxf(v, sm[i]);
        // minMaxLoc over an empty mask reports 0; threshold value is computed in double and
        // compared in float (cv::threshold, THRESH_TOZERO)
        const double mx = (v == -CUDART_INF_F) ? 0.0 : (double)v;
        const float thr = (float)(mx * quality);
        state[0] = __float_as_uint(thr);
        state[1] = 0u;
        state[2] = (v == -CUDART_INF_F) ? 1u : 0u;  // empty mask: no corner can be valid
    }
}

// ---- (2)+(3) threshold, 3x3 local maximum, mask, border; compact to keys ----------------
// Unsigned key in the order of the float value: every bit of a negative value flipped, only the
// sign bit of a positive one.  Candidates are negative when the masked maximum is (cornerMinEigenVal
// returns values like -1.5e-8 on straight edges) and quality > 1 puts the threshold below it.
// Never 0, the padding key, for a candidate (that would need the NaN 0xffffffff).
__device__ __forceinline__ unsigned order_key(float v) {
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(TX *TY)
candidates_kernel(const float *__restrict__ eig, const uint8_t *__restrict__ valid, int h, int w,
                  unsigned *__restrict__ state, unsigned long long *__restrict__ keys, unsigned cap) {
    const int x = blockIdx.x * TX + threadIdx.x, y = blockIdx.y * TY + threadIdx.y;
    if (x < 1 || y < 1 || x >= w - 1 || y >= h - 1) return;
    const float thr = __uint_as_float(state[0]);
    const size_t i = (size_t)y * w + x;
    const float v = eig[i];
    if (!(v > thr) || v == 0.f) return;
    if (valid && !valid[i]) return;
    bool ismax = true;
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
        for (int dx = -1; dx <= 1; dx++) {
            float u = eig[(size_t)(y + dy) * w + (x + dx)];
            u = (u > thr) ? u : 0.f;
            ismax &= !(u > v);
        }
    if (!ismax) return;
    const unsigned slot = atomicAdd(&state[1], 1u);
    if (slot < cap) keys[slot] = ((unsigned long long)order_key(v) << 32) | (unsigned)i;
}

// ---- (4) bitonic sort, descending, of n = 2^p keys (padding keys are 0) ----------------
constexpr int SORT_BLOCK = 1024;           // threads
constexpr int SORT_TILE = 2 * SORT_BLOCK;  // keys sorted per CTA in shared memory

__device__ __forceinline__ void cmpswap_desc(unsigned long long &a, unsigned long long &b, bool desc) {
    if ((a < b) == desc) {
        const unsigned long long t = a; a = b; b = t;
    }
}

// all stages k <= SORT_TILE in shared memory
__global__ void __launch_bounds__(SORT_BLOCK)
bitonic_local_kernel(unsigned long long *__restrict__ keys, unsigned n, unsigned k_start, unsigned k_end) {
    __shared__ unsigned long long sm[SORT_TILE];
    const unsigned base = blockIdx.x * SORT_TILE;
    for (unsigned t = threadIdx.x; t < SORT_TILE; t += SORT_BLOCK) sm[t] = (base + t < n) ? keys[base + t] : 0ull;
    __syncthreads();
    for (unsigned k = k_start; k <= k_end; k <<= 1) {
        const unsigned jmax = (k_start == k_end && k_start > SORT_TILE) ? SORT_TILE / 2 : k / 2;
        for (unsigned j = (jmax < k / 2 ? jmax : k / 2); j > 0; j >>= 1) {
            const unsigned t = threadIdx.x;
            const unsigned lo = 2 * t - (t & (j - 1));  // index with bit j cleared
            const unsigned hi = lo + j;
            const bool desc = (((base + lo) & k) == 0);  // first half of each k-block descending
            cmpswap_desc(sm[lo], sm[hi], desc);
            __syncthreads();
        }
    }
    for (unsigned t = threadIdx.x; t < SORT_TILE; t += SORT_BLOCK)
        if (base + t < n) keys[base + t] = sm[t];
}

// one compare-exchange pass with stride j >= SORT_TILE
__global__ void __launch_bounds__(256)
bitonic_global_kernel(unsigned long long *__restrict__ keys, unsigned n, unsigned k, unsigned j) {
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n / 2) return;
    const unsigned lo = 2 * t - (t & (j - 1));
    const unsigned hi = lo + j;
    const bool desc = ((lo & k) == 0);
    unsigned long long a = keys[lo], b = keys[hi];
    if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
}

// ---- (5) ordered greedy min-distance selection ---------------------------------------------
constexpr int CELL_CAP = 8;

// cv::goodFeaturesToTrack's distance test: squares and sum in float, compared in double with
// minDistance^2 squared in double.  A float threshold differs whenever minDistance^2 is not a float
// (minDistance = sqrt(50): 50 passes a float threshold, fails cv2's).  The intrinsics keep any
// build from fusing a multiply-add, which would round the sum differently above 2^24.
__device__ __forceinline__ bool too_close(float dx, float dy, double md2) {
    return (double)__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < md2;
}

struct SelectParams {
    const unsigned long long *keys;
    const unsigned *state;  // [1] = number of candidates
    unsigned cap;
    int h, w, max_corners;
    double md2;             // minDistance^2, in double
    bool use_dist;          // minDistance >= 1: otherwise every candidate is accepted
    int cell, gw, gh;
    int *cell_cnt;      // (gh*gw), zeroed
    short2 *cell_pts;   // (gh*gw*CELL_CAP)
    float *out_xy;      // (max_corners, 2)
    int *out_count;
};

__global__ void __launch_bounds__(32) select_kernel(const SelectParams p) {
    const int lane = threadIdx.x;
    const unsigned ncand = min(p.state[1], p.cap);
    int accepted = 0;
    const bool limited = p.max_corners > 0;
    for (unsigned basei = 0; basei < ncand; basei += 32) {
        const unsigned ci = basei + lane;
        bool ok = ci < ncand;
        int x = 0, y = 0;
        if (ok) {
            const unsigned addr = (unsigned)(p.keys[ci] & 0xffffffffull);
            y = addr / p.w;
            x = addr - y * p.w;
        }
        const int xc = x / p.cell, yc = y / p.cell;
        if (ok && p.use_dist) {
            const int x1 = max(0, xc - 1), y1 = max(0, yc - 1);
            const int x2 = min(p.gw - 1, xc + 1), y2 = min(p.gh - 1, yc + 1);
            for (int yy = y1; yy <= y2 && ok; yy++)
                for (int xx = x1; xx <= x2 && ok; xx++) {
                    const int c = yy * p.gw + xx;
                    const int cnt = min(p.cell_cnt[c], CELL_CAP);
                    for (int q = 0; q < cnt; q++) {
                        const short2 pt = p.cell_pts[c * CELL_CAP + q];
                        if (too_close((float)(x - pt.x), (float)(y - pt.y), p.md2)) { ok = false; break; }
                    }
                }
        }
        // resolve the order inside the batch: an earlier accepted candidate suppresses later ones
        for (int i = 0; i < 32; i++) {
            const bool oki = __shfl_sync(0xffffffffu, ok, i);
            const int xi = __shfl_sync(0xffffffffu, x, i), yi = __shfl_sync(0xffffffffu, y, i);
            if (oki && lane > i && ok && p.use_dist && too_close((float)(x - xi), (float)(y - yi), p.md2))
                ok = false;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        const int rank = __popc(bal & ((1u << lane) - 1u));
        const bool take = ok && (!limited || accepted + rank < p.max_corners);
        const int c = yc * p.gw + xc;
        // lanes of one batch landing in the same cell get distinct slots, in batch order
        int before = 0;
        for (int i = 0; i < 32; i++) {
            const int ci2 = __shfl_sync(0xffffffffu, c, i);
            const bool ti = __shfl_sync(0xffffffffu, take, i);
            if (ti && i < lane && ci2 == c) before++;
        }
        if (take) {
            const int o = accepted + rank;
            p.out_xy[2 * o] = (float)x;
            p.out_xy[2 * o + 1] = (float)y;
            if (p.use_dist) {
                const int slot = p.cell_cnt[c] + before;
                if (slot < CELL_CAP) p.cell_pts[c * CELL_CAP + slot] = make_short2((short)x, (short)y);
            }
        }
        __syncwarp();
        // publish the new per-cell counts after every lane has read the old ones
        if (take && p.use_dist) atomicAdd(&p.cell_cnt[c], 1);
        __threadfence_block();
        __syncwarp();
        accepted += __popc(bal);
        if (limited && accepted >= p.max_corners) { accepted = p.max_corners; break; }
    }
    if (lane == 0) *p.out_count = accepted;
}

// Same selection with the cell grid in SHARED memory: every cell is one 32-bit word,
// [1:0] = count (<= 3), then 3 x (5-bit x, 5-bit y) offsets inside the cell.  A cell of side
// round(minDistance) can hold at most two corners that are minDistance apart, so three slots
// are enough.  2048^2 at minDistance 10 is 205 x 205 cells = 168 KB: the whole grid stays on
// chip and a candidate test costs nine shared-memory loads instead of ~20 dependent global
// loads.
//
// The greedy selection is sequential in the candidate order, but most of a batch's instructions
// do not touch the grid: decoding the keys and the all-pairs proximity of the 32 candidates of a
// batch.  A lone warp issues one instruction every ~4.7 cycles (ncu, round 1: 52.6 k instructions
// in 249 k cycles), so SEL_WARPS warps take batches round-robin: each prepares its batch
// (keys, cells, all-pairs masks) on its own, then waits for the token -- a shared-memory word
// holding the index of the next batch allowed to read and update the grid -- runs the short serial
// part (nine grid words, the in-batch order, the insertions), and passes the token on.  Batches
// therefore meet the grid strictly in candidate order: the selection is the one a single warp makes.
constexpr int SEL_WARPS = 8;
constexpr unsigned SEL_DONE = 0xffffffffu;

__global__ void __launch_bounds__(32 * SEL_WARPS) select_smem_kernel(const SelectParams p) {
    extern __shared__ unsigned cells[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ncell = p.gw * p.gh;
    volatile unsigned *ctl = cells + ncell;  // [0] token: next batch to meet the grid, [1] accepted so far
    for (int i = threadIdx.x; i < ncell + 2; i += 32 * SEL_WARPS) cells[i] = 0u;
    __syncthreads();
    const unsigned ncand = min(p.state[1], p.cap);
    const unsigned nbatch = (ncand + 31u) / 32u;
    // integer form of d2 < md2 for the all-pairs test: d2 is an exact integer (images < 32768 px a side),
    // and below 2^24 (minDistance < 32.5 here) cv2's float sum of squares is that integer
    const unsigned md2i = (unsigned)ceil(p.md2);
    const bool limited = p.max_corners > 0;
    for (unsigned b = warp; b < nbatch; b += SEL_WARPS) {
        // ---- preparation: independent of every other batch
        const unsigned ci = b * 32u + lane;
        bool ok = ci < ncand;
        int x = 0, y = 0;
        if (ok) {
            const unsigned addr = (unsigned)(p.keys[ci] & 0xffffffffull);
            y = addr / p.w;
            x = addr - y * p.w;
        }
        const int xc = x / p.cell, yc = y / p.cell;
        unsigned close = 0u;  // earlier lanes of this batch within minDistance of this lane
#pragma unroll 8
        for (int i = 0; i < 32; i++) {
            const int xi = __shfl_sync(0xffffffffu, x, i), yi = __shfl_sync(0xffffffffu, y, i);
            const int dx = x - xi, dy = y - yi;
            if (i < lane && (unsigned)(dx * dx) + (unsigned)(dy * dy) < md2i) close |= 1u << i;
        }
        int nidx[9];  // the 3 x 3 neighbourhood's grid words (-1: outside the grid / no candidate)
#pragma unroll
        for (int k = 0; k < 9; k++) {
            const int xx = xc + k % 3 - 1, yy = yc + k / 3 - 1;
            nidx[k] = (ok && xx >= 0 && yy >= 0 && xx < p.gw && yy < p.gh) ? yy * p.gw + xx : -1;
        }
        // ---- wait for the token
        unsigned tok;
        while ((tok = ctl[0]) != b && tok != SEL_DONE) {}
        if (tok == SEL_DONE) break;  // uniform: every lane read the same word
        __syncwarp();
        int accepted = (int)ctl[1];
        // ---- serial part: the grid as all earlier batches left it.  Nine independent loads; the
        // neighbourhood is empty for most candidates (1000 corners in 42 k cells)
        unsigned wds[9], any = 0u;
#pragma unroll
        for (int k = 0; k < 9; k++) {
            wds[k] = nidx[k] >= 0 ? cells[nidx[k]] : 0u;
            any |= wds[k];
        }
        if (any) {
#pragma unroll
            for (int k = 0; k < 9; k++) {
                const unsigned wd = wds[k];
                const int cnt = wd & 3u;
                const int ox = (xc + k % 3 - 1) * p.cell, oy = (yc + k / 3 - 1) * p.cell;
                for (int q = 0; q < cnt; q++) {
                    const unsigned f = (wd >> (2 + 10 * q)) & 0x3ffu;
                    if (too_close((float)(x - (ox + (int)(f & 31u))), (float)(y - (oy + (int)(f >> 5))), p.md2))
                        ok = false;
                }
            }
        }
        // order inside the batch: an ACCEPTED earlier lane suppresses later lanes within
        // minDistance; only the few lanes that have a close earlier lane are resolved in order.
        const unsigned okmask = __ballot_sync(0xffffffffu, ok);
        close &= okmask;                                        // only valid lanes can suppress
        unsigned acc = __ballot_sync(0xffffffffu, ok && close == 0u);  // decided: accepted
        unsigned pend = okmask & ~acc;                          // need their earlier lanes decided
        while (pend) {
            const int i = __ffs(pend) - 1;                      // lowest undecided lane: all of its
            pend &= pend - 1;                                   // earlier lanes are decided now
            const bool oki = (__shfl_sync(0xffffffffu, close, i) & acc) == 0u;
            if (oki) acc |= 1u << i;
        }
        ok = (acc >> lane) & 1u;
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        const int rank = __popc(bal & ((1u << lane) - 1u));
        const bool take = ok && (!limited || accepted + rank < p.max_corners);
        if (take) {
            const int o = accepted + rank;
            p.out_xy[2 * o] = (float)x;
            p.out_xy[2 * o + 1] = (float)y;
        }
        // insert: lanes in different cells update their words concurrently; lanes sharing a
        // cell (rare) are serialised by the lowest lane of the group, in batch order
        const unsigned tmask = __ballot_sync(0xffffffffu, take);
        const int c = yc * p.gw + xc;
        if (take) {
            const unsigned grp = __match_any_sync(tmask, c);
            if (lane == __ffs(grp) - 1) {
                unsigned wd = cells[c];
                unsigned g = grp;
                while (g) {
                    const int j = __ffs(g) - 1;
                    g &= g - 1;
                    const int xj = __shfl_sync(grp, x, j), yj = __shfl_sync(grp, y, j);
                    const unsigned cnt = wd & 3u;
                    if (cnt < 3u) {
                        const unsigned f = (unsigned)(xj - xc * p.cell) | ((unsigned)(yj - yc * p.cell) << 5);
                        wd = (wd & ~3u) | (f << (2 + 10 * cnt)) | (cnt + 1u);
                    }
                }
                cells[c] = wd;
            } else {
                // non-leader members only serve the leader's shuffles
                unsigned g = grp;
                while (g) {
                    const int j = __ffs(g) - 1;
                    g &= g - 1;
                    __shfl_sync(grp, x, j);
                    __shfl_sync(grp, y, j);
                }
            }
        }
        __syncwarp();
        accepted += __popc(bal);
        const bool full = limited && accepted >= p.max_corners;
        if (full) accepted = p.max_corners;
        // ---- pass the token (after this warp's grid words and count are visible to the CTA)
        __threadfence_block();
        if (lane == 0) {
            ctl[1] = (unsigned)accepted;
            __threadfence_block();
            ctl[0] = full ? SEL_DONE : b + 1u;
        }
        if (full) break;
    }
    __syncthreads();
    if (threadIdx.x == 0) *p.out_count = (int)ctl[1];
}

}  // namespace

// eig (m,n) float32, valid (m,n) uint8 or NULL -> corners (x, y) float32, count.
// out_xy must hold max_corners pairs (max_corners > 0 required).
extern "C" int b200_good_features(const float *eig, const uint8_t *valid, int m, int n, int max_corners,
                                  double quality_level, double min_distance, float *out_xy,
                                  int *out_count, void *stream) {
    B200_REQUIRE(eig && out_xy && out_count && m >= 1 && n >= 1 && max_corners > 0, "bad arguments");
    B200_REQUIRE((int64_t)m * n < ((int64_t)1 << 31), "image too large");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t N = (size_t)m * n;
    const int nparts = b200::num_sms() * 4;
    b200::Scratch part, state, keys, cellc, cellp;
    B200_CUDA(part.alloc(sizeof(float) * nparts, s));
    B200_CUDA(state.alloc(sizeof(unsigned) * 4, s));
    masked_max_partial<<<nparts, 256, 0, s>>>(eig, valid, N, (float *)part.p);
    B200_LAUNCH_CHECK();
    masked_max_final<<<1, 256, 0, s>>>((const float *)part.p, nparts, quality_level, (unsigned *)state.p);
    B200_LAUNCH_CHECK();
    // every interior pixel can be a candidate on a plateau
    const unsigned cap = (unsigned)N;
    // the bitonic network sorts the next power of two above the candidate count (padding zeroed):
    // size the buffer for the largest count possible
    size_t cap_pow2 = SORT_TILE;
    while (cap_pow2 < (size_t)cap) cap_pow2 <<= 1;
    B200_CUDA(keys.alloc(sizeof(unsigned long long) * cap_pow2, s));
    candidates_kernel<<<dim3(b200::ceil_div(n, TX), b200::ceil_div(m, TY)), dim3(TX, TY), 0, s>>>(
        eig, valid, m, n, (unsigned *)state.p, (unsigned long long *)keys.p, cap);
    B200_LAUNCH_CHECK();
    unsigned hstate[4];
    B200_CUDA(cudaMemcpyAsync(hstate, state.p, sizeof(hstate), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));  // the sort network is sized by the candidate count
    unsigned ncand = hstate[1] < cap ? hstate[1] : cap;
    if (hstate[2]) ncand = 0;
    if (ncand == 0) {
        B200_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int), s));
        return 0;
    }
    unsigned npow = SORT_TILE;
    while (npow < ncand) npow <<= 1;
    if (npow > ncand)
        B200_CUDA(cudaMemsetAsync((unsigned long long *)keys.p + ncand, 0,
                                  sizeof(unsigned long long) * (npow - ncand), s));
    unsigned long long *K = (unsigned long long *)keys.p;
    bitonic_local_kernel<<<npow / SORT_TILE, SORT_BLOCK, 0, s>>>(K, npow, 2, SORT_TILE);
    B200_LAUNCH_CHECK();
    for (unsigned k = 2 * SORT_TILE; k <= npow; k <<= 1) {
        for (unsigned j = k / 2; j >= SORT_TILE; j >>= 1) {
            bitonic_global_kernel<<<b200::ceil_div((int)(npow / 2), 256), 256, 0, s>>>(K, npow, k, j);
            B200_LAUNCH_CHECK();
        }
        bitonic_local_kernel<<<npow / SORT_TILE, SORT_BLOCK, 0, s>>>(K, npow, k, k);
        B200_LAUNCH_CHECK();
    }
    SelectParams sp;
    sp.keys = K;
    sp.state = (const unsigned *)state.p;
    sp.cap = ncand;
    sp.h = m; sp.w = n;
    sp.max_corners = max_corners;
    sp.md2 = min_distance * min_distance;  // in double, like cv2
    sp.use_dist = min_distance >= 1.0;
    sp.cell = sp.use_dist ? (int)lrint(min_distance) : 1;
    sp.gw = (n + sp.cell - 1) / sp.cell;
    sp.gh = (m + sp.cell - 1) / sp.cell;
    const size_t ncell = (size_t)sp.gw * sp.gh;
    sp.out_xy = out_xy;
    sp.out_count = out_count;
    if (sp.use_dist && sp.cell <= 32 && ncell * sizeof(unsigned) <= 200 * 1024) {
        const size_t smem = (ncell + 2) * sizeof(unsigned);  // the grid + the token and the running count
        B200_CUDA(cudaFuncSetAttribute(select_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        select_smem_kernel<<<1, 32 * SEL_WARPS, smem, s>>>(sp);
        B200_LAUNCH_CHECK();
        return 0;
    }
    B200_CUDA(cellc.alloc(sizeof(int) * ncell, s));
    B200_CUDA(cellp.alloc(sizeof(short2) * ncell * CELL_CAP, s));
    B200_CUDA(cudaMemsetAsync(cellc.p, 0, sizeof(int) * ncell, s));
    sp.cell_cnt = (int *)cellc.p;
    sp.cell_pts = (short2 *)cellp.p;
    sp.out_xy = out_xy;
    sp.out_count = out_count;
    select_kernel<<<1, 32, 0, s>>>(sp);
    B200_LAUNCH_CHECK();
    return 0;
}
