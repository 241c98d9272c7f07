// lk_frontend.cu -- the per-frame front end of dense Lucas-Kanade as three passes over the frame
// instead of seven (sm_90a): what dense_lucaskanade does to a frame before any feature is
// looked for --
//   np.ma.masked_invalid + fill value          pysteps/motion/lucaskanade.py:207-219
//   utils.images.morph_opening (3x3 cross)     pysteps/utils/images.py:60-86
//   min / max of the opened image (4 row sets) pysteps/tracking/lucaskanade.py:144-160,
//   scaling to uint8 for the tracker ...       pysteps/feature/shitomasi.py:131-151
//   ... and for the detector, buffered mask
// Pass A  mask + min/max of the raw frame (the opening's threshold is the frame minimum);
// Pass B  opening recomputed from the raw frame in shared memory + min/max/count of the opened
//         image -- the opened float64 image is never written to HBM;
// Pass C  opening again + both uint8 scalings + the detector's validity map.
// (A global minimum separates A from B and B from C, hence three kernels; the 32 MB frame stays
// in the 126 MB L2 between them.)
//
// Passes B and C are stencils with a 2-pixel halo (opening = erode o dilate with the 3x3 cross:
// 5x5 footprint; 5x5 mask buffer).  Their float64 tiles are staged in shared memory by TMA:
// one elected thread issues cp.async.bulk.tensor.2d for a (64+4) x (16+4) box -- halo included,
// out-of-image parts filled by the copy engine -- into a two-deep ring, an mbarrier per slot
// counts the bytes in, and the CTA computes tile i while the copy of tile i+1 is in flight.
// Persistent CTAs (a multiple of the SM count) walk the tiles.  Results are those of the
// stand-alone stage kernels of lk_dense.cu bit for bit (tests/test_lk_gpu.py).
#include <cuda.h>

#include "common.cuh"
#include "lk_common.cuh"
#include "quantise_body.cuh"

namespace {

constexpr int FW = 64, FH = 16;          // pixel tile of one step
constexpr int HALO = 2;
constexpr int BW = FW + 2 * HALO, BH = FH + 2 * HALO;   // TMA box: 68 x 20 float64 (544-byte rows)
constexpr int FTHREADS = 256;
constexpr int MW = 80;                   // mask tile row pitch (bytes)

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// box (x0 .. x0+BW, y0 .. y0+BH) of the tensor map -> shared memory; coordinates may lie outside
// the image (halo of border tiles): those elements are filled by the copy engine
__device__ __forceinline__ void tma_load_box(void *dst, const CUtensorMap *map, int x0, int y0, unsigned long long *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(x0), "r"(y0), "r"(smem_u32(bar)) : "memory");
}

struct FrontParams {
    const uint8_t *mask;     // (m, n) from pass A
    const double *stats0;    // [min, max, count] of the raw frame
    double *stats;           // 12 doubles: written by pass B's last CTA, read by pass C
    int m, n, opening, dil, f32;
    MM *part;                // pass B: [4][nparts]
    unsigned *ticket;        // pass B: zeroed before the launch (mm_finish)
    int nparts;
    uint8_t *q_track, *q_det, *valid;   // pass C (q_det / valid may be null)
};

// The three stencils of a tile (threshold image -> erosion -> dilation = the 3x3-cross opening;
// the k x k buffered mask) are evaluated on BIT ROWS: a row of the 68-pixel box is one 128-bit word
// built by warp ballots, and erosion / dilation / buffering of a whole row are a handful of shifts and
// ANDs / ORs done by one thread per output row -- instead of 25 byte tests per pixel, or three
// byte-wise sweeps over shared memory with a divide per element (45 / 60 us per pass at 2048^2).
//   fg   pixel is foreground: inside the image, not masked, value > frame minimum (utils/images.py:66-70)
//   nz   fg or OUTSIDE the image (out-of-image neighbours do not erode)
//   mk   mask byte (0 outside the image)
typedef unsigned __int128 Row;
constexpr int SEG = (BW + 31) / 32;   // 32-bit words per bit row (3: columns 0-31, 32-63, 64-67)
constexpr int ROWS_PER_WARP = (BH + FTHREADS / 32 - 1) / (FTHREADS / 32);

__device__ __forceinline__ Row load_row(const unsigned (*a)[4], int r) {
    return (Row)a[r][0] | ((Row)a[r][1] << 32) | ((Row)a[r][2] << 64);
}

// uint8 scaling of float64 frames: qz::ScaleF64 (quantise_body.cuh, also compiled and tested on the host)
struct Scale : qz::ScaleF64 {
    __device__ __forceinline__ void init(const double *st, int set) { qz::ScaleF64::init(st[3 * set + 0], st[3 * set + 1]); }
};

// PASS = 1: statistics of the opened image.  PASS = 2: uint8 images.
// (4 CTAs per SM: the launch is 4 persistent CTAs per SM, all of which must be resident -- at 76
// registers only 3 were, and the 4th ran as a second wave)
template <int PASS>
__global__ void __launch_bounds__(FTHREADS, 4)
front_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ FrontParams p) {
    __shared__ __align__(128) double s_img[2][BH * BW];
    __shared__ unsigned s_fg[BH][4], s_nz[BH][4], s_mk[BH][4];
    __shared__ unsigned long long s_min[FH], s_dil[FH], s_mk0[FH];  // per output row, bit lx
    __shared__ __align__(8) unsigned long long s_bar[2];
    __shared__ MM s_mm[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int m = p.m, n = p.n;
    const int tiles_x = (n + FW - 1) / FW, tiles = tiles_x * ((m + FH - 1) / FH);
    if (tid == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    constexpr unsigned BOX_BYTES = BW * BH * sizeof(double);
    auto issue = [&](int t, int slot) {
        const int x0 = (t % tiles_x) * FW, y0 = (t / tiles_x) * FH;
        mbar_expect_tx(&s_bar[slot], BOX_BYTES);
        tma_load_box(s_img[slot], &tmap, x0 - HALO, y0 - HALO, &s_bar[slot]);
    };
    int t = blockIdx.x;
    if (t < tiles && tid == 0) issue(t, 0);
    // mask bytes of a tile (1 byte per pixel, 2-pixel halo, zero outside the image): fetched into
    // registers one tile ahead, so their L2 latency hides behind the current tile's arithmetic.
    // Warp w owns box rows w, w + 8, w + 16; a lane owns columns lane, lane + 32, lane + 64.
    // Bits 0-7 of a register: the mask byte; bit 8: the pixel lies inside the image.
    unsigned short mreg[ROWS_PER_WARP][SEG];
    auto fetch_mask = [&](int tt) {
        const int x0 = (tt % tiles_x) * FW - HALO, y0 = (tt / tiles_x) * FH - HALO;
#pragma unroll
        for (int k = 0; k < ROWS_PER_WARP; k++) {
            const int y = y0 + wid + k * (FTHREADS / 32);
#pragma unroll
            for (int sg = 0; sg < SEG; sg++) {
                const int lx = lane + 32 * sg, x = x0 + lx;
                const bool in = wid + k * (FTHREADS / 32) < BH && lx < BW && y >= 0 && y < m && x >= 0 && x < n;
                mreg[k][sg] = in ? (unsigned short)(0x100u | p.mask[(size_t)y * n + x]) : (unsigned short)0;
            }
        }
    };
    if (t < tiles) fetch_mask(t);

    const double minval = p.stats0[0];
    const bool opening = p.opening != 0;
    const bool any_masked = p.stats0[2] < (double)m * (double)n;
    const bool buffer = p.dil > 0 && any_masked;
    // set 1 leaves out row 0, or row 1 when anything is masked (masked_minmax_kernel of lk_dense.cu)
    const int set1_out = any_masked ? 1 : 0;
    const int dil_lo = -(p.dil / 2), dil_hi = p.dil - 1 - p.dil / 2;
    MM acc[4];
    if (PASS == 1) {
#pragma unroll
        for (int k = 0; k < 4; k++) { acc[k].mn = CUDART_INF; acc[k].mx = -CUDART_INF; acc[k].cnt = 0; }
    }
    Scale sc_track, sc_det;
    double fill = 0.0;
    bool any_clear = false;
    int det_set = 0, det_row0 = -1, det_row1 = -1;   // rows the detector masks: 0 and / or 1, or none
    if (PASS == 2) {
        const double *st = p.stats;
        fill = st[0];
        any_clear = st[11] > 0.0;
        // feature/shitomasi.py:131-151 (see quantise_kernel of lk_dense.cu, mode 1)
        if (p.dil > 0) {
            det_set = (any_clear ? 1 : 0) + (any_masked ? 1 : 0);
            det_row0 = any_clear ? 0 : -1;
            det_row1 = any_masked ? 1 : -1;
        }
        sc_track.init(st, 0);
        sc_det.init(st, det_set);
    }
    for (int it = 0; t < tiles; t += gridDim.x, it++) {
        const int slot = it & 1;
        const int tn = t + gridDim.x;
        // the other slot was last read in iteration it-1, which ended with a block barrier
        if (tn < tiles && tid == 0) issue(tn, slot ^ 1);
        const int tx0 = (t % tiles_x) * FW, ty0 = (t / tiles_x) * FH;
        const double *img = s_img[slot];
        mbar_wait(&s_bar[slot], (unsigned)((it >> 1) & 1));
        // ---- bit rows of the box (ballots) ------------------------------------------------------
#pragma unroll
        for (int k = 0; k < ROWS_PER_WARP; k++) {
            const int r = wid + k * (FTHREADS / 32);
            if (r < BH) {
#pragma unroll
                for (int sg = 0; sg < SEG; sg++) {
                    const int lx = lane + 32 * sg;
                    const unsigned mr = mreg[k][sg];
                    const bool in = (mr & 0x100u) != 0, mk = (mr & 0xffu) != 0;
                    const bool fg = in && !mk && img[r * BW + min(lx, BW - 1)] > minval;
                    const unsigned bfg = __ballot_sync(0xffffffffu, fg);
                    const unsigned bout = __ballot_sync(0xffffffffu, !in && lx < BW);
                    const unsigned bmk = __ballot_sync(0xffffffffu, mk);
                    if (lane == 0) { s_fg[r][sg] = bfg; s_nz[r][sg] = bfg | bout; s_mk[r][sg] = bmk; }
                }
            }
        }
        if (tn < tiles) fetch_mask(tn);
        __syncthreads();
        // ---- one thread per output row: opening and buffered mask as shifts of whole rows ----------
        if (tid < FH) {
            const int hy = tid + HALO;
            Row setmin = 0;
            if (opening) {
                // erosion with the 3x3 cross (a pixel outside the image does not erode), rows hy-1 .. hy+1
                Row ero[3];
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    const int r = hy - 1 + j;
                    const Row c = load_row(s_nz, r);
                    ero[j] = load_row(s_fg, r) & load_row(s_nz, r - 1) & load_row(s_nz, r + 1) & (c << 1) & (c >> 1);
                }
                // a foreground pixel survives the opening if the cross around it holds an eroded pixel;
                // otherwise it takes the frame minimum (utils/images.py:72-81)
                const Row keep = ero[1] | ero[0] | ero[2] | (ero[1] << 1) | (ero[1] >> 1);
                setmin = load_row(s_fg, hy) & ~keep;
            }
            const Row mk0 = load_row(s_mk, hy);
            Row dl = mk0;
            if (buffer) {
                // k x k buffered mask (feature/shitomasi.py:131-137), out-of-image taps ignored (mask bit 0)
                dl = 0;
                for (int dy = dil_lo; dy <= dil_hi; dy++) {
                    const Row rr = load_row(s_mk, hy + dy);
                    for (int dx = dil_lo; dx <= dil_hi; dx++) dl |= dx >= 0 ? (rr >> dx) : (rr << -dx);
                }
            }
            s_min[tid] = (unsigned long long)(setmin >> HALO);
            s_mk0[tid] = (unsigned long long)(mk0 >> HALO);
            s_dil[tid] = (unsigned long long)(dl >> HALO);
        }
        __syncthreads();
        // ---- output pixels ---------------------------------------------------------------------------
#pragma unroll
        for (int k = 0; k < FW * FH / FTHREADS; k++) {
            const int lx = tid % FW, ly = tid / FW + k * (FTHREADS / FW);
            const int x = tx0 + lx, y = ty0 + ly;
            if (x >= n || y >= m) continue;
            double v = img[(ly + HALO) * BW + lx + HALO];
            if ((s_min[ly] >> lx) & 1ull) v = minval;
            const bool mk0 = (s_mk0[ly] >> lx) & 1ull;
            const bool d = (s_dil[ly] >> lx) & 1ull;
            if (PASS == 1) {
                if (!mk0) {
                    acc[0].mn = fmin(acc[0].mn, v); acc[0].mx = fmax(acc[0].mx, v); acc[0].cnt++;
                    if (y != set1_out) { acc[1].mn = fmin(acc[1].mn, v); acc[1].mx = fmax(acc[1].mx, v); acc[1].cnt++; }
                    if (y >= 2) { acc[2].mn = fmin(acc[2].mn, v); acc[2].mx = fmax(acc[2].mx, v); acc[2].cnt++; }
                }
                if (!d) acc[3].cnt++;
            } else {
                const size_t i = (size_t)y * n + x;
                // tracking/lucaskanade.py:144-160
                const double vt = mk0 ? fill : v;
                p.q_track[i] = p.f32 ? cast_u8(qz::scale_f32(vt, sc_track.im_min, sc_track.im_max))
                                     : sc_track(vt);
                if (p.q_det) {
                    if (p.valid) p.valid[i] = d ? 0 : 1;
                    bool mk = mk0;
                    if (y == det_row0 || y == det_row1) mk = true;
                    const double vd = mk ? fill : v;
                    p.q_det[i] = p.f32 ? cast_u8(qz::scale_f32(vd, sc_det.im_min, sc_det.im_max))
                                       : sc_det(vd);
                }
            }
        }
        __syncthreads();  // everyone is done with this slot and the bit rows before they are refilled
    }
    if (PASS == 1) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const MM r = mm_block(acc[k], s_mm);
            if (tid == 0) p.part[(size_t)k * p.nparts + blockIdx.x] = r;
        }
        mm_finish(p.part, p.nparts, 4, p.stats, p.ticket, s_mm, tid, FTHREADS);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

}  // namespace

extern "C" int b200_lk_frontend(const double *img, const uint8_t *user_mask, int m, int n, int size_opening,
                                int buffer_mask, int flags, uint8_t *mask, double *stats0, double *stats,
                                uint8_t *q_track, uint8_t *q_det, uint8_t *valid, void *stream) {
    B200_REQUIRE(img && mask && stats0 && stats && q_track && m >= 1 && n >= 1, "bad arguments");
    B200_REQUIRE(size_opening == 0 || size_opening == 3, "only the 3x3 structuring element is implemented");
    B200_REQUIRE(buffer_mask >= 0 && buffer_mask <= 5, "buffer_mask must be 0..5 for the fused front end");
    // TMA needs 16-byte aligned rows: an even number of float64 columns
    B200_REQUIRE(n % 2 == 0 && ((uintptr_t)img & 15) == 0, "the fused front end needs an even width and a 16-byte aligned frame");
    cudaStream_t s = (cudaStream_t)stream;
    // ---- pass A: mask + min/max of the raw frame (kernels of lk_dense.cu) ---------------------
    if (int rc = b200_mask_invalid(img, user_mask, m, n, mask, stats0, stream)) return rc;
    // ---- tensor map of the frame: 2-D float64, box 68 x 20, zero fill outside ------------------
    EncodeTiledFn enc = encode_tiled();
    if (!enc) {
        b200::set_error("cuTensorMapEncodeTiled is not available from this driver");
        return B200_ENOTSUP;
    }
    CUtensorMap tmap;
    const cuuint64_t dims[2] = {(cuuint64_t)n, (cuuint64_t)m};
    const cuuint64_t strides[1] = {(cuuint64_t)n * sizeof(double)};
    const cuuint32_t box[2] = {BW, BH};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult cr = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, (void *)img, dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
        b200::set_error("cuTensorMapEncodeTiled failed (%d)", (int)cr);
        return B200_EINVAL;
    }
    const int tiles = b200::ceil_div(n, FW) * b200::ceil_div(m, FH);
    const int nparts = std::min(tiles, b200::num_sms() * 4);  // persistent CTAs: a multiple of the SM count
    b200::Scratch part;
    B200_CUDA(part.alloc(sizeof(MM) * nparts * 4 + 16, s));
    FrontParams p;
    memset(&p, 0, sizeof(p));
    p.mask = mask; p.stats0 = stats0; p.stats = stats; p.m = m; p.n = n; p.opening = size_opening != 0;
    p.dil = buffer_mask; p.f32 = (flags & B200_QUANTISE_F32) != 0; p.part = (MM *)part.p; p.nparts = nparts;
    p.ticket = (unsigned *)((MM *)part.p + (size_t)nparts * 4);
    p.q_track = q_track; p.q_det = q_det; p.valid = valid;
    B200_CUDA(cudaMemsetAsync(p.ticket, 0, sizeof(unsigned), s));
    front_kernel<1><<<nparts, FTHREADS, 0, s>>>(tmap, p);  // its last CTA writes `stats`
    B200_LAUNCH_CHECK();
    front_kernel<2><<<nparts, FTHREADS, 0, s>>>(tmap, p);
    B200_LAUNCH_CHECK();
    return 0;
}
