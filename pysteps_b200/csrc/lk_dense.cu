// lk_dense.cu -- the dense per-pixel stages of pysteps' Lucas-Kanade path (sm_90a):
// masking / min-max reductions, 3x3 cross opening, uint8 quantisation, Gaussian pyramid,
// Scharr derivative images and the Shi-Tomasi minimum-eigenvalue map.
//
// Reference call sites (pysteps is Python; the arithmetic is in opencv-python 4.13.0):
//   pysteps/motion/lucaskanade.py:207-224      masked_invalid, fill value, morph_opening
//   pysteps/utils/images.py:27-86              morph_opening (cv2.morphologyEx, 3x3 cross)
//   pysteps/feature/shitomasi.py:131-162       mask dilation, uint8 scaling, goodFeaturesToTrack
//   pysteps/tracking/lucaskanade.py:144-171    uint8 scaling, calcOpticalFlowPyrLK
// All of these are HBM/L2-streaming stencils over m x n pixels: one thread per pixel,
// 32-wide rows per warp for coalescing, halos served by L1 (reuse factor 9-25 in a tile).
// Integer stages are exact; the float32 stages reproduce OpenCV's operation order
// (explicit fmaf where the AVX-512 build fuses, plain mul/add elsewhere; --fmad=false).
#include <math_constants.h>

#include "common.cuh"
#include "lk_common.cuh"
#include "quantise_body.cuh"

namespace {

constexpr int TX = 32, TY = 8;

using b200::reflect101;

// mask = user_mask | !isfinite(img) (np.ma.masked_invalid); min/max over unmasked.
// A pure stream over the frame (8 B read + 1 B written per pixel): PAIR = two pixels per thread as one
// 16-byte load, four independent loads in flight per thread -- one 8-byte load per thread per
// iteration kept only ~1.2 MB in flight across the GPU (1.6 TB/s).  The last CTA to finish reduces
// the per-CTA partials (mm_finish), so the statistics cost no second launch.
template <bool PAIR>
__global__ void __launch_bounds__(256)
mask_invalid_kernel(const double *__restrict__ img, const uint8_t *__restrict__ user_mask, size_t N,
                    uint8_t *__restrict__ mask, MM *__restrict__ part, double *__restrict__ stats,
                    unsigned *ticket) {
    __shared__ MM sm[32];
    MM v;
    v.mn = CUDART_INF; v.mx = -CUDART_INF; v.cnt = 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    auto one = [&](double a, uint8_t um) -> uint8_t {
        const bool msk = um || !isfinite(a);
        if (!msk) { v.mn = fmin(v.mn, a); v.mx = fmax(v.mx, a); v.cnt++; }
        return msk ? 1 : 0;
    };
    if (PAIR) {
        const size_t NP = N / 2;  // N is even
        const double2 *img2 = reinterpret_cast<const double2 *>(img);
        const uchar2 *um2 = reinterpret_cast<const uchar2 *>(user_mask);
        uchar2 *mask2 = reinterpret_cast<uchar2 *>(mask);
#pragma unroll 4
        for (size_t i = i0; i < NP; i += stride) {
            const double2 a = img2[i];
            const uchar2 um = user_mask ? um2[i] : make_uchar2(0, 0);
            uchar2 o;
            o.x = one(a.x, um.x);
            o.y = one(a.y, um.y);
            mask2[i] = o;
        }
    } else {
#pragma unroll 4
        for (size_t i = i0; i < N; i += stride) mask[i] = one(img[i], user_mask ? user_mask[i] : (uint8_t)0);
    }
    v = mm_block(v, sm);
    if (threadIdx.x == 0) part[blockIdx.x] = v;
    mm_finish(part, gridDim.x, 1, stats, ticket, sm, threadIdx.x, blockDim.x);
}

// utils/images.py:66-81 : bin = filled > thr ; open with the 3x3 cross ; pixels removed by the
// opening are set to the minimum.  erode ignores out-of-image taps, so does dilate.
__global__ void __launch_bounds__(TX *TY)
morph_open_kernel(const double *__restrict__ img, const uint8_t *__restrict__ mask, int m, int n,
                  const double *__restrict__ thr_dev, const double *__restrict__ min_dev,
                  double *__restrict__ out) {
    const int x = blockIdx.x * TX + threadIdx.x, y = blockIdx.y * TY + threadIdx.y;
    if (x >= n || y >= m) return;
    const double thr = *thr_dev, minval = *min_dev;
    auto bin = [&](int yy, int xx) -> int {  // -1 outside the image
        if (yy < 0 || yy >= m || xx < 0 || xx >= n) return -1;
        const size_t i = (size_t)yy * n + xx;
        return (!mask[i] && img[i] > thr) ? 1 : 0;
    };
    auto eroded = [&](int yy, int xx) -> int {  // -1 outside
        const int c = bin(yy, xx);
        if (c < 0) return -1;
        // out-of-image neighbours do not erode (border = +max)
        return (c != 0) & (bin(yy - 1, xx) != 0) & (bin(yy + 1, xx) != 0) & (bin(yy, xx - 1) != 0) &
               (bin(yy, xx + 1) != 0);
    };
    const size_t i = (size_t)y * n + x;
    const double v = img[i];
    const int b = bin(y, x);
    double o = v;
    if (b == 1) {
        const bool opened = (eroded(y, x) == 1) | (eroded(y - 1, x) == 1) | (eroded(y + 1, x) == 1) |
                            (eroded(y, x - 1) == 1) | (eroded(y, x + 1) == 1);
        if (!opened) o = minval;
    }
    out[i] = o;
}

// min/max/count over unmasked pixels of all rows (set 0), of the rows left when the detector masks
// row 0 alone or row 1 alone (set 1) and of rows >= 2 (set 2), plus (set 3, count only) the number
// of pixels whose k x k dilated mask is clear.
// The row sets exist because feature/shitomasi.py:139 indexes the image with the uint8 mask
// (`input_image[mask] = masked`): NumPy treats it as INTEGER indexing, which masks row 0 when
// the buffered mask contains a 0 and row 1 when it contains a 1 -- not the buffered pixels.
// Nothing masked: the buffered mask is all 0, row 0 goes and set 1 is rows >= 1.  Something masked:
// set 1 serves only the case where the buffered mask is all 1 and row 1 alone goes -- rows != 1.
__global__ void __launch_bounds__(TX *TY)
masked_minmax_kernel(const double *__restrict__ img, const uint8_t *__restrict__ mask, int m, int n,
                     int dil, const double *__restrict__ stats0, MM *__restrict__ part, int nparts) {
    __shared__ MM sm[32];
    MM a[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { a[k].mn = CUDART_INF; a[k].mx = -CUDART_INF; a[k].cnt = 0; }
    // nothing masked (stats of b200_mask_invalid): the buffered mask is clear everywhere
    const bool any_masked = !stats0 || stats0[2] < (double)m * (double)n;
    const int tiles_x = (n + TX - 1) / TX, tiles = tiles_x * ((m + TY - 1) / TY);
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int x = (t % tiles_x) * TX + threadIdx.x, y = (t / tiles_x) * TY + threadIdx.y;
        if (x >= n || y >= m) continue;
        const size_t i = (size_t)y * n + x;
        const double v = img[i];
        bool d = mask[i] != 0;
        if (!d) {
            a[0].mn = fmin(a[0].mn, v); a[0].mx = fmax(a[0].mx, v); a[0].cnt++;
            if (any_masked ? y != 1 : y >= 1) { a[1].mn = fmin(a[1].mn, v); a[1].mx = fmax(a[1].mx, v); a[1].cnt++; }
            if (y >= 2) { a[2].mn = fmin(a[2].mn, v); a[2].mx = fmax(a[2].mx, v); a[2].cnt++; }
        }
        if (dil > 0 && any_masked) {
            const int r = dil / 2;
            for (int dy = -r; dy <= dil - 1 - r; dy++)
                for (int dx = -r; dx <= dil - 1 - r; dx++) {
                    const int yy = y + dy, xx = x + dx;
                    if (yy >= 0 && yy < m && xx >= 0 && xx < n) d |= mask[(size_t)yy * n + xx] != 0;
                }
        }
        if (!d) a[3].cnt++;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const MM r = mm_block(a[k], sm);
        if (threadIdx.x == 0 && threadIdx.y == 0) part[(size_t)k * nparts + blockIdx.x] = r;
    }
}

// mode 0 (tracking/lucaskanade.py:144-160): masked pixels take the fill value, min/max over
// the unmasked pixels.  mode 1 (feature/shitomasi.py:131-151): additionally row 0 / row 1 are
// masked as described above, min/max over what is left, and `valid` = buffered mask clear.
// F32: the frames were float32 at the API, so the reference scales them in float32
// (img.filled() - im_min) / (im_max - im_min) * 255 with float32 scalars; the values held here are
// those float32 numbers widened, so narrowing them back is exact.
template <bool F32>
__global__ void __launch_bounds__(TX *TY)
quantise_kernel(const double *__restrict__ img, const uint8_t *__restrict__ mask, int m, int n, int mode,
                int dil, const double *__restrict__ stats, const double *__restrict__ fill_dev,
                uint8_t *__restrict__ out, uint8_t *__restrict__ valid) {
    const int x = blockIdx.x * TX + threadIdx.x, y = blockIdx.y * TY + threadIdx.y;
    if (x >= n || y >= m) return;
    const size_t i = (size_t)y * n + x;
    bool msk = mask[i] != 0;
    int set = 0;
    if (mode == 1) {
        bool dmask = msk;
        const bool any_masked0 = stats[2] < (double)m * (double)n;
        if (dil > 0 && any_masked0) {  // nothing masked: the buffered mask is clear everywhere
            const int r = dil / 2;
            for (int dy = -r; dy <= dil - 1 - r; dy++)
                for (int dx = -r; dx <= dil - 1 - r; dx++) {
                    const int yy = y + dy, xx = x + dx;
                    if (yy >= 0 && yy < m && xx >= 0 && xx < n) dmask |= mask[(size_t)yy * n + xx] != 0;
                }
        }
        if (valid) valid[i] = dmask ? 0 : 1;
        const bool any_clear = stats[11] > 0.0;                       // buffered mask contains a 0
        const bool any_masked = stats[2] < (double)m * (double)n;     // ... contains a 1
        if (dil > 0) {
            // rows masked: row 0, row 1 or both; set 1 is the rows left by either single one
            set = (any_clear ? 1 : 0) + (any_masked ? 1 : 0);
            if ((y == 0 && any_clear) || (y == 1 && any_masked)) msk = true;
        }
    } else if (valid) {
        valid[i] = msk ? 0 : 1;
    }
    const double im_min = stats[3 * set + 0], im_max = stats[3 * set + 1];
    const double v = msk ? *fill_dev : img[i];
    double q;
    if (F32) {
        q = qz::scale_f32(v, im_min, im_max);
    } else if (__dsub_rn(im_max, im_min) > 1e-8)
        q = __dmul_rn(__ddiv_rn(__dsub_rn(v, im_min), __dsub_rn(im_max, im_min)), 255.0);
    else
        q = __dsub_rn(v, im_min);
    out[i] = cast_u8(q);
}

// cv::pyrDown on uint8: separable [1 4 6 4 1], BORDER_REFLECT_101, (sum + 128) >> 8
__global__ void __launch_bounds__(TX *TY)
pyrdown_kernel(const uint8_t *__restrict__ src, int h, int w, uint8_t *__restrict__ dst, int dh, int dw) {
    const int x = blockIdx.x * TX + threadIdx.x, y = blockIdx.y * TY + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const int wt[5] = {1, 4, 6, 4, 1};
    int xs[5];
#pragma unroll
    for (int k = 0; k < 5; k++) xs[k] = reflect101(2 * x + k - 2, w);
    int acc = 0;
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const uint8_t *r = src + (size_t)reflect101(2 * y + j - 2, h) * w;
        int row = 0;
#pragma unroll
        for (int k = 0; k < 5; k++) row += wt[k] * r[xs[k]];
        acc += wt[j] * row;
    }
    dst[(size_t)y * dw + x] = (uint8_t)((acc + 128) >> 8);
}

// calcScharrDeriv: smooth [3 10 3], diff [-1 0 1], BORDER_REFLECT_101, int16 (Ix, Iy)
__global__ void __launch_bounds__(TX *TY)
scharr_kernel(const uint8_t *__restrict__ src, int h, int w, short2 *__restrict__ dst) {
    const int x = blockIdx.x * TX + threadIdx.x, y = blockIdx.y * TY + threadIdx.y;
    if (x >= w || y >= h) return;
    const uint8_t *r0 = src + (size_t)reflect101(y - 1, h) * w;
    const uint8_t *r1 = src + (size_t)y * w;
    const uint8_t *r2 = src + (size_t)reflect101(y + 1, h) * w;
    const int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w);
    const int t0m = (r0[xm] + r2[xm]) * 3 + r1[xm] * 10;
    const int t0p = (r0[xp] + r2[xp]) * 3 + r1[xp] * 10;
    const int t1m = r2[xm] - r0[xm], t1c = r2[x] - r0[x], t1p = r2[xp] - r0[xp];
    dst[(size_t)y * w + x] = make_short2((short)(t0p - t0m), (short)((t1m + t1p) * 3 + t1c * 10));
}

// ---------------------------------------------------------------- Shi-Tomasi eigenvalue map
// cv::cornerMinEigenVal(u8, blockSize 5, ksize 3) as the 4.13.0 AVX-512 build evaluates it
// (pinned bit for bit, oracle/lk_oracle.c ora_min_eig_u8).
struct Cov { float xx, xy, yy; };

__device__ __forceinline__ Cov cov_at(const uint8_t *__restrict__ q, int h, int w, int y, int x, int tail0) {
    const float s = (float)(1.0 / 5100.0), s2 = (float)(2.0 / 5100.0);
    const int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w);
    float g[3], v[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint8_t *r = q + (size_t)reflect101(y + k - 1, h) * w;
        const float c0 = (float)r[xm], c1 = (float)r[x], c2 = (float)r[xp];
        g[k] = __fsub_rn(c2, c0);
        v[k] = (x < tail0) ? __fmaf_rn(c2, s, __fmaf_rn(c1, s2, __fmul_rn(c0, s)))
                           : __fadd_rn(__fadd_rn(__fmul_rn(c0, s), __fmul_rn(c1, s2)), __fmul_rn(c2, s));
    }
    const float dx = __fmaf_rn(s, __fadd_rn(g[0], g[2]), __fmul_rn(s2, g[1]));
    const float dy = __fsub_rn(v[2], v[0]);
    Cov c;
    c.xx = __fmul_rn(dx, dx);
    c.xy = __fmul_rn(dx, dy);
    c.yy = __fmul_rn(dy, dy);
    return c;
}

// per pixel: the three 5-tap row sums of the covariance products, in double, left to right.
// A CTA evaluates the products of its 64 x 8 tile plus two columns either side ONCE into shared
// memory (already widened to double), then every pixel adds its five neighbours: 9.6 u8 loads and
// conversions per pixel instead of 45 -- the conversion (XU) pipe bounded the per-pixel version.
constexpr int CR_W = 64, CR_H = 8, CR_P = CR_W + 4;

__global__ void __launch_bounds__(256)
cov_rowsum_kernel(const uint8_t *__restrict__ q, int h, int w, double *__restrict__ rs) {
    __shared__ double s_xx[CR_H][CR_P], s_xy[CR_H][CR_P], s_yy[CR_H][CR_P];
    const int x0 = blockIdx.x * CR_W, y0 = blockIdx.y * CR_H;
    const int tail0 = (w / 32) * 32;
    for (int i = threadIdx.x; i < CR_H * CR_P; i += 256) {
        const int r = i / CR_P, c = i - r * CR_P;
        const int y = y0 + r, xs = x0 - 2 + c;
        if (y < h && xs <= w + 1) {  // columns past w + 1 feed no pixel of the image
            const Cov cv = cov_at(q, h, w, y, reflect101(xs, w), tail0);
            s_xx[r][c] = (double)cv.xx;
            s_xy[r][c] = (double)cv.xy;
            s_yy[r][c] = (double)cv.yy;
        }
    }
    __syncthreads();
    const size_t N = (size_t)h * w;
    const int r = threadIdx.x >> 5, y = y0 + r;
    if (y >= h) return;
#pragma unroll
    for (int k = 0; k < CR_W / 32; k++) {
        const int c = (threadIdx.x & 31) + 32 * k, x = x0 + c;
        if (x >= w) break;
        double sxx = s_xx[r][c], sxy = s_xy[r][c], syy = s_yy[r][c];
#pragma unroll
        for (int d = 1; d < 5; d++) {
            sxx = __dadd_rn(sxx, s_xx[r][c + d]);
            sxy = __dadd_rn(sxy, s_xy[r][c + d]);
            syy = __dadd_rn(syy, s_yy[r][c + d]);
        }
        const size_t i = (size_t)y * w + x;
        rs[i] = sxx;
        rs[N + i] = sxy;
        rs[2 * N + i] = syy;
    }
}

// per column: OpenCV's running column sum (double) down the rows, then the eigenvalue.
// The recurrence is history dependent (add entering row, emit, subtract leaving row), so a
// column is one sequential chain; columns are independent and coalesced across the warp.
// The row leaving at step y is the row that entered at step y-4 (a 4-deep delay line in
// registers), so each step needs only the entering row.  Those loads do not depend on the
// chain: they are streamed BOX_R rows ahead into a shared-memory ring with cp.async
// (LDGSTS), one commit group per row, so a single resident warp per SM still covers the
// DRAM latency and the loop runs at the speed of its two dependent FP64 adds.
constexpr int BOX_R = 64;  // rows in flight per warp: 64 rows * 32 columns * 8 B = 16 KB

__device__ __forceinline__ void cp_async8(void *smem_dst, const void *gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
// the ring is read with plain shared loads right after the wait: the "memory" clobbers keep the
// compiler from moving those loads above it (or the refill's copies above the reads)
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// grid = (ceil(w/32), 3): one warp per (32 columns, covariance plane), so the three running
// sums of a column advance in parallel and a row step is ~10 instructions of one warp.
__global__ void __launch_bounds__(32)
box_chain_kernel(const double *__restrict__ rs, int h, int w, float *__restrict__ box) {
    __shared__ double ring_s[BOX_R][32];
    const int lane = threadIdx.x;
    const int x = blockIdx.x * 32 + lane;
    const int xc = min(x, w - 1);  // out-of-range lanes shadow the last column
    const size_t N = (size_t)h * w;
    const double *__restrict__ src = rs + (size_t)blockIdx.y * N;
    float *__restrict__ dst = box + (size_t)blockIdx.y * N;
    // rows -2, -1, 0, 1 (reflected): the initial sum and the first four leaving rows
    double delay[4];
    double S = 0.0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        delay[k] = src[(size_t)reflect101(k - 2, h) * w + xc];
        S = __dadd_rn(S, delay[k]);
    }
    auto issue = [&](int y) {  // entering row of step y
        if (y < h) cp_async8(&ring_s[y % BOX_R][lane], src + (size_t)reflect101(y + 2, h) * w + xc);
        cp_async_commit();  // one (possibly empty) group per row keeps the group count uniform
    };
    for (int y = 0; y < BOX_R; y++) issue(y);
    // BOX_U rows per round: ONE wait for the whole group, the BOX_U entering rows read from the ring
    // into registers (independent loads), then the dependent add / subtract chain alone on the
    // critical path -- the wait and the shared-memory latency are paid once per round, not per row.
    // A lone warp issues one instruction every ~4.6 cycles (ncu: issue active 22 %), so the row rate
    // is set by the INSTRUCTION COUNT of a row: interior rounds (all rows of the round and all rows
    // they prefetch inside the image) run without the reflection / bounds arithmetic -- ~11
    // instructions per row instead of 52.
    constexpr int BOX_U = 8;
    static_assert(BOX_R % BOX_U == 0 && BOX_U % 4 == 0, "ring slots and the delay line are addressed by u");
    // (lanes past the last column shadow column w - 1: they compute and store the very same values
    // to the very same addresses, so the stores need no predicate)
    const bool live = x < w;
    int y0 = 0;
    float *__restrict__ o = dst + xc;                                   // output row y0
    const double *__restrict__ nx = src + (size_t)(BOX_R + 2) * w + xc;  // entering row of step y0 + BOX_R
    for (; y0 + BOX_R + BOX_U + 2 <= h; y0 += BOX_U) {
        cp_async_wait<BOX_R - BOX_U>();  // rows y0 .. y0 + BOX_U - 1 have landed
        double(*slot)[32] = ring_s + (y0 % BOX_R);
        double in[BOX_U];
#pragma unroll
        for (int u = 0; u < BOX_U; u++) in[u] = slot[u][lane];
#pragma unroll
        for (int u = 0; u < BOX_U; u++) {
            const double a = __dadd_rn(S, in[u]);
            S = __dsub_rn(a, delay[u & 3]);
            delay[u & 3] = in[u];
            *o = __double2float_rn(a);
            o += w;
        }
#pragma unroll
        for (int u = 0; u < BOX_U; u++) {  // refill the slots just consumed
            cp_async8(&slot[u][lane], nx);
            cp_async_commit();
            nx += w;
        }
    }
    for (; y0 < h; y0 += BOX_U) {  // the last BOX_R + BOX_U + 2 rows: reflected prefetches, ragged end
        cp_async_wait<BOX_R - BOX_U>();
        double in[BOX_U];
#pragma unroll
        for (int u = 0; u < BOX_U; u++) in[u] = ring_s[(y0 + u) % BOX_R][lane];
#pragma unroll
        for (int u = 0; u < BOX_U; u++) {
            const int y = y0 + u;
            if (y < h) {
                const double a = __dadd_rn(S, in[u]);
                S = __dsub_rn(a, delay[u & 3]);  // y0 is a multiple of 4
                delay[u & 3] = in[u];
                if (live) dst[(size_t)y * w + x] = __double2float_rn(a);
            }
        }
#pragma unroll
        for (int u = 0; u < BOX_U; u++) issue(y0 + u + BOX_R);
    }
}

// eig = (a + c) - sqrt((a - c)^2 + b^2) with a = xx/2, b = xy, c = yy/2, float32 as OpenCV
__global__ void __launch_bounds__(256)
eig_from_box_kernel(const float *__restrict__ box, size_t N, float *__restrict__ eig) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride) {
        const float fa = __fmul_rn(box[i], 0.5f), fb = box[N + i], fc = __fmul_rn(box[2 * N + i], 0.5f);
        const float t = __fsub_rn(fa, fc);
        const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(t, t), __fmul_rn(fb, fb)));
        eig[i] = __fsub_rn(__fadd_rn(fa, fc), r);
    }
}

static dim3 grid2d(int m, int n) { return dim3(b200::ceil_div(n, TX), b200::ceil_div(m, TY)); }

}  // namespace

extern "C" int b200_mask_invalid(const double *img, const uint8_t *user_mask, int m, int n,
                                 uint8_t *mask_out, double *stats, void *stream) {
    B200_REQUIRE(img && mask_out && stats && m >= 1 && n >= 1, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t N = (size_t)m * n;
    const int nparts = b200::num_sms() * 4;  // persistent CTAs: a multiple of the SM count
    b200::Scratch part;
    B200_CUDA(part.alloc(sizeof(MM) * nparts + 16, s));
    unsigned *ticket = (unsigned *)((MM *)part.p + nparts);
    B200_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned), s));
    const bool pair = N % 2 == 0 && ((uintptr_t)img & 15) == 0 && ((uintptr_t)mask_out & 1) == 0 &&
                      ((uintptr_t)user_mask & 1) == 0;
    if (pair)
        mask_invalid_kernel<true><<<nparts, 256, 0, s>>>(img, user_mask, N, mask_out, (MM *)part.p, stats, ticket);
    else
        mask_invalid_kernel<false><<<nparts, 256, 0, s>>>(img, user_mask, N, mask_out, (MM *)part.p, stats, ticket);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_morph_opening(const double *img, const uint8_t *mask, int m, int n, int size,
                                  const double *thr_dev, const double *min_dev, double *out,
                                  void *stream) {
    B200_REQUIRE(img && mask && out && thr_dev && min_dev && m >= 1 && n >= 1, "bad arguments");
    if (size != 3) {
        b200::set_error("morph_opening: only the 3x3 structuring element is implemented");
        return B200_ENOTSUP;
    }
    morph_open_kernel<<<grid2d(m, n), dim3(TX, TY), 0, (cudaStream_t)stream>>>(img, mask, m, n, thr_dev, min_dev, out);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_masked_minmax(const double *img, const uint8_t *mask, int m, int n, int dilate,
                                  const double *stats0, double *stats, void *stream) {
    B200_REQUIRE(img && mask && stats && m >= 1 && n >= 1 && dilate >= 0 && dilate <= 31, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const int nparts = b200::num_sms() * 4;
    b200::Scratch part;
    B200_CUDA(part.alloc(sizeof(MM) * nparts * 4, s));
    masked_minmax_kernel<<<nparts, dim3(TX, TY), 0, s>>>(img, mask, m, n, dilate, stats0, (MM *)part.p, nparts);
    B200_LAUNCH_CHECK();
    mm_final_kernel<<<1, 256, 0, s>>>((const MM *)part.p, nparts, 4, stats);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_quantise_u8(const double *img, const uint8_t *mask, int m, int n, int mode,
                                int dilate, const double *stats, const double *fill_dev,
                                uint8_t *out, uint8_t *valid, void *stream) {
    B200_REQUIRE(img && mask && stats && fill_dev && out && m >= 1 && n >= 1 && dilate >= 0 &&
                     dilate <= 31 && (mode & ~3) == 0, "bad arguments");
    if (mode & B200_QUANTISE_F32)
        quantise_kernel<true><<<grid2d(m, n), dim3(TX, TY), 0, (cudaStream_t)stream>>>(img, mask, m, n, mode & 1, dilate,
                                                                                      stats, fill_dev, out, valid);
    else
        quantise_kernel<false><<<grid2d(m, n), dim3(TX, TY), 0, (cudaStream_t)stream>>>(img, mask, m, n, mode & 1, dilate,
                                                                                       stats, fill_dev, out, valid);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_pyr_down_u8(const uint8_t *src, int h, int w, uint8_t *dst, void *stream) {
    B200_REQUIRE(src && dst && h >= 1 && w >= 1, "bad arguments");
    const int dh = (h + 1) / 2, dw = (w + 1) / 2;
    pyrdown_kernel<<<grid2d(dh, dw), dim3(TX, TY), 0, (cudaStream_t)stream>>>(src, h, w, dst, dh, dw);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_scharr_i16(const uint8_t *src, int h, int w, int16_t *dst, void *stream) {
    B200_REQUIRE(src && dst && h >= 1 && w >= 1, "bad arguments");
    scharr_kernel<<<grid2d(h, w), dim3(TX, TY), 0, (cudaStream_t)stream>>>(src, h, w, (short2 *)dst);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_min_eig(const uint8_t *q, int m, int n, float *eig, void *stream) {
    B200_REQUIRE(q && eig && m >= 1 && n >= 1, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    b200::Scratch rs, box;
    const size_t N = (size_t)m * n;
    B200_CUDA(rs.alloc(sizeof(double) * 3 * N, s));
    B200_CUDA(box.alloc(sizeof(float) * 3 * N, s));
    cov_rowsum_kernel<<<dim3(b200::ceil_div(n, CR_W), b200::ceil_div(m, CR_H)), 256, 0, s>>>(q, m, n, (double *)rs.p);
    B200_LAUNCH_CHECK();
    box_chain_kernel<<<dim3(b200::ceil_div(n, 32), 3), 32, 0, s>>>((const double *)rs.p, m, n, (float *)box.p);
    B200_LAUNCH_CHECK();
    const int blocks = (int)std::min<size_t>((N + 255) / 256, (size_t)b200::num_sms() * 16);
    eig_from_box_kernel<<<blocks, 256, 0, s>>>((const float *)box.p, N, eig);
    B200_LAUNCH_CHECK();
    return 0;
}
