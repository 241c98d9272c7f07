// lk_track.cu -- sparse pyramidal Lucas-Kanade tracker (sm_90a).
//
// Reference call site: pysteps/tracking/lucaskanade.py:171 (cv2.calcOpticalFlowPyrLK with
// winSize (50,50), maxLevel 3, criteria (COUNT|EPS, 10, 0), minEigThreshold 1e-4).  The
// arithmetic restated here is OpenCV's LKTrackerInvoker (fixed-point bilinear patches with
// W_BITS = 14, int16 Scharr derivatives, float32 structure tensor / mismatch vector) and is
// BIT-IDENTICAL to the opencv-python 4.13.0 binary: the five window sums are accumulated in
// float32 in the lane order of its 128-bit SIMD loops (4 lanes over x mod 4 plus a scalar
// tail), which is what makes the 2500-pixel sums reproducible.
//
// Mapping: one CTA per feature, all pyramid levels inside the kernel (a feature's track is
// independent of every other feature's).  The window (<= 4096 pixels) lives in shared memory as
// int16; patch extraction and the per-iteration mismatch products are data parallel over
// the CTA; the ordered float32 accumulations are 15 (setup) / 10 (per iteration) independent
// sequential chains run by the lanes of warp 0 out of shared memory.
#include <climits>

#include "common.cuh"

namespace {

constexpr int LK_THREADS = 128;  // 9 CTAs/SM: 1000 features fit in one wave
constexpr int W_BITS = 14;

struct LKParams {
    const uint8_t *I, *J;   // pyramids (levels contiguous)
    const short2 *dI;       // Scharr derivative pyramid of I
    size_t off[B200_LK_MAX_LEVELS];
    int h[B200_LK_MAX_LEVELS], w[B200_LK_MAX_LEVELS];
    int max_level;          // coarsest level index actually built
    int win_w, win_h, max_count;
    double eps2, min_eig_thr;
    const float *prev_pts;  // (npts,2) level-0 coordinates
    const int *npts_dev;    // optional device count (NULL: use npts)
    int npts;
    float *next_pts;        // (npts,2)
    uint8_t *status;        // (npts)
};

using b200::reflect101;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// i / d for 0 <= i < 2^16 and any d >= 1 without an integer division (exact: (i + 0.5) / d sits
// at least 0.5/d from an integer, and the two float roundings move it by at most
// 2^-23 (i + 0.5) / d, which stays below that margin while i < 2^22)
__device__ __forceinline__ int div_small(int i, float inv_d) { return __float2int_rd(((float)i + 0.5f) * inv_d); }

// cvFloor as the x86 build of OpenCV computes it: NaN and values outside the int range give
// INT_MIN (cvtss2si's "integer indefinite"), where cvt.rmi would give 0 for NaN and clamp the
// rest.  Only the window bounds tests read it: a NaN coordinate must fail them as in cv2.
__device__ __forceinline__ int cv_floor(float v) {
    return (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rd(v) : INT_MIN;
}

// bilinear fixed-point weights of a sub-pixel offset (a, b)
__device__ __forceinline__ void make_weights(float a, float b, int &w00, int &w01, int &w10, int &w11) {
    w00 = __float2int_rn((1.f - a) * (1.f - b) * (float)(1 << W_BITS));
    w01 = __float2int_rn(a * (1.f - b) * (float)(1 << W_BITS));
    w10 = __float2int_rn((1.f - a) * b * (float)(1 << W_BITS));
    w11 = (1 << W_BITS) - w00 - w01 - w10;
}

__global__ void __launch_bounds__(LK_THREADS) lk_track_kernel(const LKParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int npts = p.npts_dev ? min(*p.npts_dev, p.npts) : p.npts;
    const int pt = blockIdx.x;
    if (pt >= npts) return;
    const int tid = threadIdx.x;
    const int ww = p.win_w, wh = p.win_h, npx = ww * wh;
    const int simd_w = (ww / 8) * 8;       // columns handled by OpenCV's 8-pixel SIMD loop
    const int nchunk = simd_w / 8, ntail = ww - simd_w;
    short *Iw = (short *)smem_raw;         // patch of I, 5 fractional bits
    short *Dx = Iw + npx;                  // interpolated Scharr derivatives
    short *Dy = Dx + npx;
    // per-iteration mismatch products, already widened to float32 in the order the chains
    // consume them: PX/PY[(y * nchunk + c) * 4 + q] = int32 pair sum of pixels (8c+q, 8c+q+4),
    // TX/TY[y * ntail + t] = single-pixel products of the scalar tail
    const int npair = wh * nchunk * 4, ntl = wh * ntail;
    float *PX = (float *)(Dy + npx + (npx & 1));
    float *PY = PX + npair;
    float *TXp = PY + npair;
    float *TYp = TXp + ntl;
    float *red = TYp + ntl;                // 16 floats: chain results
    __shared__ float s_b[2];

    const float inv_ww = 1.0f / (float)ww, inv_nchunk = nchunk > 0 ? 1.0f / (float)nchunk : 0.f,
                inv_ntail = ntail > 0 ? 1.0f / (float)ntail : 0.f;
    const float half_x = (ww - 1) * 0.5f, half_y = (wh - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (float)(1 << 20);
    // The ordered float32 sums are sequential chains run by ONE warp of the CTA while the others wait at
    // the barrier.  Warps go to the SM's four schedulers by warp index, so with warp 0 doing the chains in
    // every CTA the ~7 resident CTAs of an SM queued all their chain work on ONE scheduler (ncu: 43 % of
    // the stall samples at the barrier after the tensor chains, issue slots 38 % busy).  The chain warp is
    // therefore picked by CTA index: ct = this thread's lane in it, negative / >= 32 elsewhere.
    const int ct = tid - 32 * (blockIdx.x & (LK_THREADS / 32 - 1));
    float nx_out = 0.f, ny_out = 0.f;      // nextPts[ptidx] as carried between levels
    bool status = true;

    for (int level = p.max_level; level >= 0; level--) {
        const uint8_t *I = p.I + p.off[level];
        const uint8_t *J = p.J + p.off[level];
        const short2 *dI = p.dI + p.off[level];
        const int h = p.h[level], w = p.w[level];
        const float inv = (float)(1. / (double)(1 << level));
        float px = p.prev_pts[2 * pt] * inv, py = p.prev_pts[2 * pt + 1] * inv;
        float nx, ny;
        if (level == p.max_level) { nx = px; ny = py; }
        else { nx = nx_out * 2.f; ny = ny_out * 2.f; }
        nx_out = nx; ny_out = ny;
        px -= half_x; py -= half_y;
        const int ix = cv_floor(px), iy = cv_floor(py);
        if (ix < -ww || ix >= w || iy < -wh || iy >= h) {
            if (level == 0) status = false;
            continue;
        }
        int w00, w01, w10, w11;
        make_weights(px - (float)ix, py - (float)iy, w00, w01, w10, w11);

        // ---- patch of I and its derivatives (data parallel) --------------------------------
        __syncthreads();
        // window (incl. the +1 taps) fully inside the level: no border handling (the common case)
        const bool inI = ix >= 0 && iy >= 0 && ix + ww < w && iy + wh < h;
        for (int i = tid; i < npx; i += LK_THREADS) {
            const int y = div_small(i, inv_ww), x = i - y * ww;
            const int yy = iy + y, xx = ix + x;
            int v00, v01, v10, v11;
            short2 d00 = make_short2(0, 0), d01 = d00, d10 = d00, d11 = d00;
            if (inI) {
                const uint8_t *q0 = I + (size_t)yy * w + xx;
                v00 = q0[0]; v01 = q0[1]; v10 = q0[w]; v11 = q0[w + 1];
                const short2 *g0 = dI + (size_t)yy * w + xx;
                d00 = g0[0]; d01 = g0[1]; d10 = g0[w]; d11 = g0[w + 1];
            } else {
                const int r0 = reflect101(yy, h), r1 = reflect101(yy + 1, h);
                const int c0 = reflect101(xx, w), c1 = reflect101(xx + 1, w);
                v00 = I[(size_t)r0 * w + c0]; v01 = I[(size_t)r0 * w + c1];
                v10 = I[(size_t)r1 * w + c0]; v11 = I[(size_t)r1 * w + c1];
                // derivative border is zero (BORDER_CONSTANT), not reflected
                const bool y0in = yy >= 0 && yy < h, y1in = yy + 1 >= 0 && yy + 1 < h;
                const bool x0in = xx >= 0 && xx < w, x1in = xx + 1 >= 0 && xx + 1 < w;
                if (y0in && x0in) d00 = dI[(size_t)yy * w + xx];
                if (y0in && x1in) d01 = dI[(size_t)yy * w + xx + 1];
                if (y1in && x0in) d10 = dI[(size_t)(yy + 1) * w + xx];
                if (y1in && x1in) d11 = dI[(size_t)(yy + 1) * w + xx + 1];
            }
            Iw[i] = (short)descale(v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11, W_BITS - 5);
            Dx[i] = (short)descale(d00.x * w00 + d01.x * w01 + d10.x * w10 + d11.x * w11, W_BITS);
            Dy[i] = (short)descale(d00.y * w00 + d01.y * w01 + d10.y * w10 + d11.y * w11, W_BITS);
        }
        __syncthreads();

        // ---- structure tensor: 12 lane chains + 3 tail chains, OpenCV's float32 order ------
        // (ct: lane of this CTA's chain warp -- see below; each chain reads only the two derivative
        // arrays of ITS product through pointers picked once, with running indices)
        if (ct >= 0 && ct < 15) {
            const int acc = ct < 12 ? ct >> 2 : ct - 12;  // 0: A11 = sum Ix Ix, 1: A12 = sum Ix Iy, 2: A22 = sum Iy Iy
            const short *pa = acc == 2 ? Dy : Dx, *pb = acc == 0 ? Dx : Dy;
            float q = 0.f;
            if (ct < 12) {
                const int l = ct & 3;
                for (int y = 0; y < wh; y++) {
                    const short *ra = pa + y * ww, *rb = pb + y * ww;
#pragma unroll 4
                    for (int x = l; x < simd_w; x += 4) q = __fmul_rn((float)ra[x], (float)rb[x]) + q;
                }
            } else {
                for (int y = 0; y < wh; y++)
                    for (int x = simd_w; x < ww; x++) q += (float)((int)pa[y * ww + x] * (int)pb[y * ww + x]);
            }
            red[ct] = q;
        }
        __syncthreads();
        float A[3];
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float s = (red[4 * a + 0] + red[4 * a + 2]) + (red[4 * a + 1] + red[4 * a + 3]);
            A[a] = (red[12 + a] + s) * FLT_SCALE;
        }
        const float A11 = A[0], A12 = A[1], A22 = A[2];
        float D = A11 * A22 - A12 * A12;
        const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) /
                             (float)(2 * ww * wh);
        if ((double)minEig < p.min_eig_thr || D < 1.1920928955078125e-07f) {
            if (level == 0) status = false;
            continue;
        }
        D = 1.f / D;
        nx -= half_x; ny -= half_y;
        float pdx = 0.f, pdy = 0.f;
        for (int j = 0; j < p.max_count; j++) {
            const int jx = cv_floor(nx), jy = cv_floor(ny);
            if (jx < -ww || jx >= w || jy < -wh || jy >= h) {
                if (level == 0) status = false;
                break;
            }
            make_weights(nx - (float)jx, ny - (float)jy, w00, w01, w10, w11);
            // ---- mismatch J - I and its products with the derivatives (data parallel) --------
            __syncthreads();
            const bool inJ = jx >= 0 && jy >= 0 && jx + ww < w && jy + wh < h;
            auto mismatch = [&](int y, int x) -> int {
                int v00, v01, v10, v11;
                if (inJ) {
                    const uint8_t *q0 = J + (size_t)(jy + y) * w + (jx + x);
                    v00 = q0[0]; v01 = q0[1]; v10 = q0[w]; v11 = q0[w + 1];
                } else {
                    const int r0 = reflect101(jy + y, h), r1 = reflect101(jy + y + 1, h);
                    const int c0 = reflect101(jx + x, w), c1 = reflect101(jx + x + 1, w);
                    v00 = J[(size_t)r0 * w + c0]; v01 = J[(size_t)r0 * w + c1];
                    v10 = J[(size_t)r1 * w + c0]; v11 = J[(size_t)r1 * w + c1];
                }
                const int jv = descale(v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11, W_BITS - 5);
                return jv - (int)Iw[y * ww + x];
            };
            for (int i = tid; i < npair; i += LK_THREADS) {
                const int q = i & 3, y = div_small(i >> 2, inv_nchunk), c = (i >> 2) - y * nchunk;
                const int x0 = 8 * c + q, i0 = y * ww + x0;
                const int d0 = mismatch(y, x0), d1 = mismatch(y, x0 + 4);
                PX[i] = (float)(d0 * (int)Dx[i0] + d1 * (int)Dx[i0 + 4]);
                PY[i] = (float)(d0 * (int)Dy[i0] + d1 * (int)Dy[i0 + 4]);
            }
            for (int i = tid; i < ntl; i += LK_THREADS) {
                const int y = div_small(i, inv_ntail), x = simd_w + (i - y * ntail);
                const int d0 = mismatch(y, x);
                TXp[i] = (float)(d0 * (int)Dx[y * ww + x]);
                TYp[i] = (float)(d0 * (int)Dy[y * ww + x]);
            }
            __syncthreads();
            // ---- mismatch vector: 8 lane chains over pixel pairs (q, q+4) + 2 tail chains --
            if (ct >= 0 && ct < 10) {
                float q = 0.f;
                if (ct < 8) {
                    // qb0 = [x(0,4) y(0,4) x(1,5) y(1,5)], qb1 = [x(2,6) y(2,6) x(3,7) y(3,7)]
                    const int pair = (ct >> 2) * 2 + ((ct & 3) >> 1);
                    const float *P = (ct & 1) ? PY : PX;
                    const int nsteps = wh * nchunk;
#pragma unroll 8
                    for (int s = 0; s < nsteps; s++) q += P[4 * s + pair];
                } else {
                    const float *P = (ct == 9) ? TYp : TXp;
#pragma unroll 4
                    for (int s = 0; s < ntl; s++) q += P[s];
                }
                red[ct] = q;
            }
            __syncthreads();
            if (ct == 0) {
                // (qb0 + qb1) -> [X0 Y0 X1 Y1]; reduce_sum of [X0 X1 0 0] is (X0+0)+(X1+0)
                const float X0 = red[0] + red[4], Y0 = red[1] + red[5];
                const float X1 = red[2] + red[6], Y1 = red[3] + red[7];
                s_b[0] = (red[8] + ((X0 + 0.f) + (X1 + 0.f))) * FLT_SCALE;
                s_b[1] = (red[9] + ((Y0 + 0.f) + (Y1 + 0.f))) * FLT_SCALE;
            }
            __syncthreads();
            const float b1 = s_b[0], b2 = s_b[1];
            const float ddx = (A12 * b2 - A22 * b1) * D;
            const float ddy = (A12 * b1 - A11 * b2) * D;
            nx += ddx; ny += ddy;
            nx_out = nx + half_x; ny_out = ny + half_y;
            if ((double)ddx * (double)ddx + (double)ddy * (double)ddy <= p.eps2) break;
            if (j > 0 && fabs((double)(ddx + pdx)) < 0.01 && fabs((double)(ddy + pdy)) < 0.01) {
                nx_out -= ddx * 0.5f; ny_out -= ddy * 0.5f;
                break;
            }
            pdx = ddx; pdy = ddy;
        }
        if (status && level == 0) {
            // OpenCV's error pass re-checks that the final window origin is inside J
            const int fx = cv_floor(nx_out - half_x), fy = cv_floor(ny_out - half_y);
            if (fx < -ww || fx >= w || fy < -wh || fy >= h) status = false;
        }
    }
    if (tid == 0) {
        p.next_pts[2 * pt] = nx_out;
        p.next_pts[2 * pt + 1] = ny_out;
        p.status[pt] = status ? 1 : 0;
    }
}

// keep rows with status == 1 (tracking/lucaskanade.py:174-181), preserving order:
// xy = p0, uv = p1 - p0 as float32 pairs; appended to a float64 pool at *pool_count.
__global__ void __launch_bounds__(1024)
compact_tracks_kernel(const float *__restrict__ p0, const float *__restrict__ p1,
                      const uint8_t *__restrict__ st, const int *__restrict__ npts_dev, int npts_cap,
                      double *__restrict__ pool_xy, double *__restrict__ pool_uv, int *__restrict__ pool_count,
                      int pool_cap) {
    __shared__ int warp_tot[32];
    __shared__ int s_base;
    const int npts = npts_dev ? min(*npts_dev, npts_cap) : npts_cap;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_base = *pool_count;
    __syncthreads();
    for (int start = 0; start < npts; start += blockDim.x) {
        const int i = start + tid;
        const bool keep = i < npts && st[i] == 1;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[wid] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); k++) {
            if (k < wid) before += warp_tot[k];
            total += warp_tot[k];
        }
        if (keep) {
            const int o = s_base + before + __popc(bal & ((1u << lane) - 1u));
            if (o < pool_cap) {
                const float x0 = p0[2 * i], y0 = p0[2 * i + 1];
                pool_xy[2 * o] = (double)x0;
                pool_xy[2 * o + 1] = (double)y0;
                pool_uv[2 * o] = (double)(p1[2 * i] - x0);       // float32 difference, widened
                pool_uv[2 * o + 1] = (double)(p1[2 * i + 1] - y0);
            }
        }
        __syncthreads();
        if (tid == 0) s_base = min(s_base + total, pool_cap);
        __syncthreads();
    }
    if (tid == 0) *pool_count = s_base;
}

}  // namespace

// Pyramid geometry of cv::buildOpticalFlowPyramid: level sizes (h+1)/2, a level is kept only
// while both dimensions exceed the window, and max_level is not capped.  Returns the coarsest
// level index and the total number of pixels of all levels (levels are stored contiguously).
// B200_LK_MAX_LEVELS levels hold every geometry: a 16th halving needs both sides above 2^16.
extern "C" int b200_lk_pyramid_layout(int h, int w, int win_w, int win_h, int max_level,
                                      int *levels_out, int64_t *offsets, int *hs, int *ws,
                                      int64_t *total_pixels) {
    B200_REQUIRE(h >= 1 && w >= 1 && win_w >= 1 && win_h >= 1 && max_level >= 0, "bad arguments");
    int lv = 0;
    int64_t off = 0;
    int ch = h, cw = w;
    for (int level = 0;; level++) {
        if (offsets) offsets[level] = off;
        if (hs) hs[level] = ch;
        if (ws) ws[level] = cw;
        off += (int64_t)ch * cw;
        lv = level;
        if (level == max_level) break;
        const int nh = (ch + 1) / 2, nw = (cw + 1) / 2;
        if (nw <= win_w || nh <= win_h) break;
        B200_REQUIRE(level + 1 < B200_LK_MAX_LEVELS, "pyramid deeper than B200_LK_MAX_LEVELS levels");
        ch = nh; cw = nw;
    }
    if (levels_out) *levels_out = lv;
    if (total_pixels) *total_pixels = off;
    return 0;
}

// Build the Gaussian pyramid of a uint8 image into `pyr` and (optionally) the Scharr
// derivative pyramid into `deriv` (int16 pairs), layout as b200_lk_pyramid_layout.
extern "C" int b200_pyr_down_u8(const uint8_t *src, int h, int w, uint8_t *dst, void *stream);
extern "C" int b200_scharr_i16(const uint8_t *src, int h, int w, int16_t *dst, void *stream);

extern "C" int b200_lk_build_pyramid(const uint8_t *img, int h, int w, int win_w, int win_h,
                                     int max_level, uint8_t *pyr, int16_t *deriv, void *stream) {
    // img == NULL: the Gaussian levels in `pyr` already exist, only derivatives are computed
    B200_REQUIRE(pyr && (img || deriv), "bad arguments");
    int lv, hs[B200_LK_MAX_LEVELS], ws[B200_LK_MAX_LEVELS];
    int64_t off[B200_LK_MAX_LEVELS], total;
    int rc = b200_lk_pyramid_layout(h, w, win_w, win_h, max_level, &lv, off, hs, ws, &total);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (img) {
        B200_CUDA(cudaMemcpyAsync(pyr, img, (size_t)h * w, cudaMemcpyDeviceToDevice, s));
        for (int l = 1; l <= lv; l++) {
            rc = b200_pyr_down_u8(pyr + off[l - 1], hs[l - 1], ws[l - 1], pyr + off[l], stream);
            if (rc) return rc;
        }
    }
    if (deriv)
        for (int l = 0; l <= lv; l++) {
            rc = b200_scharr_i16(pyr + off[l], hs[l], ws[l], deriv + 2 * off[l], stream);
            if (rc) return rc;
        }
    return 0;
}

extern "C" int b200_lk_track(const uint8_t *pyrI, const uint8_t *pyrJ, const int16_t *derivI, int h,
                             int w, int win_w, int win_h, int max_level, int max_count, double epsilon,
                             double min_eig_thr, const float *prev_pts, int npts, const int *npts_dev,
                             float *next_pts, uint8_t *status, void *stream) {
    B200_REQUIRE(pyrI && pyrJ && derivI && prev_pts && next_pts && status, "bad arguments");
    B200_REQUIRE(win_w >= 1 && win_h >= 1 && win_w * win_h <= 64 * 64, "window must be 1..64x64 pixels");
    if (npts <= 0) return 0;
    LKParams p;
    memset(&p, 0, sizeof(p));
    int lv;
    int64_t off[B200_LK_MAX_LEVELS], total;
    int rc = b200_lk_pyramid_layout(h, w, win_w, win_h, max_level, &lv, off, p.h, p.w, &total);
    if (rc) return rc;
    for (int l = 0; l <= lv; l++) p.off[l] = (size_t)off[l];
    p.I = pyrI; p.J = pyrJ; p.dI = (const short2 *)derivI;
    p.max_level = lv;
    p.win_w = win_w; p.win_h = win_h;
    p.max_count = max_count;
    p.eps2 = epsilon * epsilon;
    p.min_eig_thr = min_eig_thr;
    p.prev_pts = prev_pts;
    p.npts = npts; p.npts_dev = npts_dev;
    p.next_pts = next_pts; p.status = status;
    const int npx = win_w * win_h;
    const int nchunk = win_w / 8, ntail = win_w - nchunk * 8;
    const size_t smem = sizeof(short) * (3 * (size_t)npx + (npx & 1)) +
                        sizeof(float) * (2 * (size_t)win_h * nchunk * 4 + 2 * (size_t)win_h * ntail + 16);
    B200_CUDA(cudaFuncSetAttribute(lk_track_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    lk_track_kernel<<<npts, LK_THREADS, smem, (cudaStream_t)stream>>>(p);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_lk_compact_tracks(const float *p0, const float *p1, const uint8_t *status,
                                      const int *npts_dev, int npts_cap, double *pool_xy,
                                      double *pool_uv, int *pool_count, int pool_cap, void *stream) {
    B200_REQUIRE(p0 && p1 && status && pool_xy && pool_uv && pool_count && npts_cap >= 0 && pool_cap >= 0,
                 "bad arguments");
    if (npts_cap == 0) return 0;
    compact_tracks_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(p0, p1, status, npts_dev, npts_cap, pool_xy,
                                                               pool_uv, pool_count, pool_cap);
    B200_LAUNCH_CHECK();
    return 0;
}
