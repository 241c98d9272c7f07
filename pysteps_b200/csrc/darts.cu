// darts.cu -- the device passes of the DARTS motion method (pysteps/motion/darts.py:22-220), sm_90a.
//
//   b200_darts_spectrum    the (K_t, K_y, K_x) block of the 3-D DFT of the (T, m, n) frames that the
//                          reference reads, as three passes: x (real rows against a twiddle table,
//                          the dominant pass), then t, then y
//   b200_darts_normal      MM = M^H M and M^H y straight from that block, M never materialised:
//                          per-CTA partials over fixed blocks of 512 rows, then one ordered pass
//   b200_darts_synthesize  the (2, m, n) field Re(ifft2(fill(coefficients))) from separable factors
//
// Every sum runs in a fixed order without float atomics, so repeated calls are bit-identical.
#include <algorithm>

#include "common.cuh"

namespace {

// ---- x pass: P[row, f] = sum_x frames[row, x] * tw_x[f, x], row = t * m + y -------------------
constexpr int XR = 64, XF = 64, XK = 16, XTHREADS = 256;

template <typename F>
__global__ void __launch_bounds__(XTHREADS) darts_rows_kernel(const F *__restrict__ frames, int64_t rows, int n,
                                                              const double2 *__restrict__ tw, int fx,
                                                              double2 *__restrict__ P) {
    __shared__ double As[XK][XR];
    __shared__ double2 Bs[XK][XF];
    const int tr = threadIdx.x / 16, tf = threadIdx.x % 16;
    const int64_t r0 = (int64_t)blockIdx.x * XR;
    const int f0 = blockIdx.y * XF;
    const double c0 = (double)frames[0];  // see b200_darts_spectrum: the DC term is that of frames - c0
    double ar[4][4], ai[4][4];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int j = 0; j < 4; j++) ar[r][j] = ai[r][j] = 0.0;
    for (int x0 = 0; x0 < n; x0 += XK) {
        for (int e = threadIdx.x; e < XR * XK; e += XTHREADS) {
            const int r = e / XK, xx = e % XK, x = x0 + xx;
            const int64_t row = r0 + r;
            As[xx][r] = (row < rows && x < n) ? (double)frames[row * n + x] - c0 : 0.0;
        }
        for (int e = threadIdx.x; e < XF * XK; e += XTHREADS) {
            const int f = e / XK, xx = e % XK, x = x0 + xx;
            Bs[xx][f] = (f0 + f < fx && x < n) ? tw[(int64_t)(f0 + f) * n + x] : make_double2(0.0, 0.0);
        }
        __syncthreads();
#pragma unroll
        for (int xx = 0; xx < XK; xx++) {
            double a[4];
            double2 w[4];
#pragma unroll
            for (int r = 0; r < 4; r++) a[r] = As[xx][tr * 4 + r];
#pragma unroll
            for (int j = 0; j < 4; j++) w[j] = Bs[xx][tf + 16 * j];
#pragma unroll
            for (int r = 0; r < 4; r++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    ar[r][j] = fma(a[r], w[j].x, ar[r][j]);
                    ai[r][j] = fma(a[r], w[j].y, ai[r][j]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int64_t row = r0 + tr * 4 + r;
            const int f = f0 + tf + 16 * j;
            if (row < rows && f < fx) P[row * fx + f] = make_double2(ar[r][j], ai[r][j]);
        }
}

// ---- t pass: Q[kt, y, kx] = sum_t tw_t[kt, t] * X_x[t, y, kx] ---------------------------------
// X_x[., ., kx] of the numpy index kx (wrapped to w = kx mod n) is P[., ., w] when 2w <= n, else
// conj(P[., ., n - w]): real rows, so aliased indices read the same coefficient.
__global__ void __launch_bounds__(256) darts_time_kernel(const double2 *__restrict__ P, int T, int m, int n, int fx,
                                                         int K, const double2 *__restrict__ tw, int Kt,
                                                         double2 *__restrict__ Q) {
    const int Kx = 2 * K + 1;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)Kt * m * Kx) return;
    const int kxi = (int)(idx % Kx), y = (int)((idx / Kx) % m), kti = (int)(idx / ((int64_t)Kx * m));
    int w = (kxi - K) % n;
    if (w < 0) w += n;
    const bool cj = 2 * w > n;
    const int f = cj ? n - w : w;
    double re = 0.0, im = 0.0;
    for (int t = 0; t < T; t++) {
        double2 p = P[((int64_t)t * m + y) * fx + f];
        if (cj) p.y = -p.y;
        const double2 c = tw[(int64_t)kti * T + t];
        re = fma(c.x, p.x, re);
        re = fma(-c.y, p.y, re);
        im = fma(c.x, p.y, im);
        im = fma(c.y, p.x, im);
    }
    Q[idx] = make_double2(re, im);
}

// ---- y pass: X[kt, ky, kx] = sum_y tw_y[ky, y] * Q[kt, y, kx] ---------------------------------
constexpr int YKY = 16, YKX = 32, YY = 32;

__global__ void __launch_bounds__(256) darts_cols_kernel(const double2 *__restrict__ Q, int m, int Kx,
                                                         const double2 *__restrict__ tw, int Ky,
                                                         double2 *__restrict__ X) {
    __shared__ double2 Ws[YKY][YY + 1];
    __shared__ double2 Qs[YY][YKX];
    const int kt = blockIdx.z, ky0 = blockIdx.y * YKY, kx0 = blockIdx.x * YKX;
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    double re0 = 0.0, im0 = 0.0, re1 = 0.0, im1 = 0.0;
    const double2 zero = make_double2(0.0, 0.0);
    for (int y0 = 0; y0 < m; y0 += YY) {
        for (int e = threadIdx.x; e < YKY * YY; e += 256) {
            const int a = e / YY, yy = e % YY;
            Ws[a][yy] = (ky0 + a < Ky && y0 + yy < m) ? tw[(int64_t)(ky0 + a) * m + y0 + yy] : zero;
        }
        for (int e = threadIdx.x; e < YY * YKX; e += 256) {
            const int yy = e / YKX, b = e % YKX;
            Qs[yy][b] = (y0 + yy < m && kx0 + b < Kx) ? Q[((int64_t)kt * m + y0 + yy) * Kx + kx0 + b] : zero;
        }
        __syncthreads();
#pragma unroll 8
        for (int yy = 0; yy < YY; yy++) {
            const double2 w = Ws[ty][yy], q0 = Qs[yy][tx], q1 = Qs[yy][tx + 16];
            re0 = fma(w.x, q0.x, re0);
            re0 = fma(-w.y, q0.y, re0);
            im0 = fma(w.x, q0.y, im0);
            im0 = fma(w.y, q0.x, im0);
            re1 = fma(w.x, q1.x, re1);
            re1 = fma(-w.y, q1.y, re1);
            im1 = fma(w.x, q1.y, im1);
            im1 = fma(w.y, q1.x, im1);
        }
        __syncthreads();
    }
    const int ky = ky0 + ty;
    if (ky >= Ky) return;
    double2 *out = X + ((int64_t)kt * Ky + ky) * Kx;
    if (kx0 + tx < Kx) out[kx0 + tx] = make_double2(re0, im0);
    if (kx0 + tx + 16 < Kx) out[kx0 + tx + 16] = make_double2(re1, im1);
}

// ---- normal equations ------------------------------------------------------------------------
constexpr int NR_ROWS = B200_DARTS_NORMAL_ROWS, NR_SUB = 32, NR_THREADS = 256, NR_PER = 4;
constexpr int NR_SLAB = NR_THREADS * NR_PER;

struct Normal {
    const double2 *X;
    int Nx, Ny, Nt, Mx, My;
    int Kx, Ky;
    int64_t rows;
    int hw, nc, npairs;
    double sx, sy;
};

// pair p -> (c, d): the upper triangle c <= d < nc column by column, then the column d = nc (M^H y)
__device__ __forceinline__ void pair_of(int p, int nc, int &c, int &d) {
    const int tri = nc * (nc + 1) / 2;
    if (p >= tri) {
        d = nc;
        c = p - tri;
        return;
    }
    int q = 0;
    while ((q + 1) * (q + 2) / 2 <= p) q++;
    d = q;
    c = p - q * (q + 1) / 2;
}

// Rows i of M run over (k_t, k_y, k_x) in the reference's order; column c < hw is A (scale
// (c1 / T_y) * i_), hw <= c < nc is B ((c1 / T_x) * j_), and column nc holds y = k_t * X[k_y, k_x, k_t].
__global__ void __launch_bounds__(NR_THREADS) darts_normal_kernel(const Normal a, double2 *__restrict__ part) {
    extern __shared__ double2 Ms[];
    const int ld = a.nc + 1;
    const int wx = 2 * a.Nx + 1, wy = 2 * a.Ny + 1, mw = 2 * a.Mx + 1;
    int cc[NR_PER], dd[NR_PER];
    double re[NR_PER], im[NR_PER];
#pragma unroll
    for (int j = 0; j < NR_PER; j++) {
        const int p = blockIdx.y * NR_SLAB + threadIdx.x + j * NR_THREADS;
        cc[j] = dd[j] = -1;
        if (p < a.npairs) pair_of(p, a.nc, cc[j], dd[j]);
        re[j] = im[j] = 0.0;
    }
    const int64_t rbeg = (int64_t)blockIdx.x * NR_ROWS, rend = min(a.rows, rbeg + NR_ROWS);
    for (int64_t s0 = rbeg; s0 < rend; s0 += NR_SUB) {
        const int cnt = (int)min((int64_t)NR_SUB, rend - s0);
        for (int e = threadIdx.x; e < cnt * ld; e += NR_THREADS) {
            const int r = e / ld, c = e % ld;
            const int i = (int)(s0 + r);
            const int kx = i % wx - a.Nx, ky = (i / wx) % wy - a.Ny, kt = i / (wx * wy) - a.Nt;
            const double2 *plane = a.X + (int64_t)(kt + a.Nt) * a.Ky * a.Kx;
            double2 v;
            if (c == a.nc) {
                const double2 z = plane[(int64_t)(ky + a.Ny + a.My) * a.Kx + kx + a.Nx + a.Mx];
                v = make_double2(__dmul_rn((double)kt, z.x), __dmul_rn((double)kt, z.y));
            } else {
                const int q = c % a.hw;
                const int iy = ky - (q / mw - a.My), jx = kx - (q % mw - a.Mx);
                const double2 z = plane[(int64_t)(iy + a.Ny + a.My) * a.Kx + jx + a.Nx + a.Mx];
                const double s = c < a.hw ? __dmul_rn(a.sy, (double)iy) : __dmul_rn(a.sx, (double)jx);
                v = make_double2(__dmul_rn(s, z.x), __dmul_rn(s, z.y));
            }
            Ms[r * ld + c] = v;
        }
        __syncthreads();
        for (int r = 0; r < cnt; r++) {
#pragma unroll
            for (int j = 0; j < NR_PER; j++) {
                if (cc[j] < 0) continue;
                const double2 u = Ms[r * ld + cc[j]], v = Ms[r * ld + dd[j]];  // conj(u) * v
                re[j] = __dadd_rn(re[j], __dadd_rn(__dmul_rn(u.x, v.x), __dmul_rn(u.y, v.y)));
                im[j] = __dadd_rn(im[j], __dsub_rn(__dmul_rn(u.x, v.y), __dmul_rn(u.y, v.x)));
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < NR_PER; j++)
        if (cc[j] >= 0)
            part[(int64_t)blockIdx.x * a.npairs + blockIdx.y * NR_SLAB + threadIdx.x + j * NR_THREADS] =
                make_double2(re[j], im[j]);
}

// the partials of the row blocks summed in block order; MM is written whole (lower = conj(upper))
__global__ void __launch_bounds__(256) darts_normal_final_kernel(const double2 *__restrict__ part, int G, int npairs,
                                                                 int nc, double2 *__restrict__ mm,
                                                                 double2 *__restrict__ mhy) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    double re = 0.0, im = 0.0;
    for (int g = 0; g < G; g++) {
        const double2 v = part[(int64_t)g * npairs + p];
        re = __dadd_rn(re, v.x);
        im = __dadd_rn(im, v.y);
    }
    int c, d;
    pair_of(p, nc, c, d);
    if (d == nc) {
        mhy[c] = make_double2(re, im);
        return;
    }
    mm[(int64_t)c * nc + d] = make_double2(re, im);
    if (c != d) mm[(int64_t)d * nc + c] = make_double2(re, -im);
}

// ---- synthesis: out[comp, y, x] = Re(sum_b G[b] * ex[b, x]) * scale, G[b] = sum_a coef[comp, a, b] * ey[a, y]
__global__ void __launch_bounds__(256) darts_synth_kernel(const double2 *__restrict__ coef, int h, int w,
                                                          const double2 *__restrict__ ey,
                                                          const double2 *__restrict__ ex, int m, int n,
                                                          double scale, double *__restrict__ out) {
    __shared__ double2 G[B200_DARTS_MAX_SIDE];
    const int y = blockIdx.x, comp = blockIdx.y;
    for (int b = threadIdx.x; b < w; b += blockDim.x) {
        double re = 0.0, im = 0.0;
#pragma unroll 1
        for (int a = 0; a < h; a++) {
            const double2 c = coef[((int64_t)comp * h + a) * w + b], e = ey[(int64_t)a * m + y];
            re = fma(c.x, e.x, re);
            re = fma(-c.y, e.y, re);
            im = fma(c.x, e.y, im);
            im = fma(c.y, e.x, im);
        }
        G[b] = make_double2(re, im);
    }
    __syncthreads();
    double *row = out + ((int64_t)comp * m + y) * n;
    for (int x = threadIdx.x; x < n; x += blockDim.x) {
        double v = 0.0;
#pragma unroll 1
        for (int b = 0; b < w; b++) {
            const double2 g = G[b], e = ex[(int64_t)b * n + x];
            v = fma(g.x, e.x, v);
            v = fma(-g.y, e.y, v);
        }
        row[x] = __dmul_rn(v, scale);
    }
}

template <typename F>
int spectrum(const F *frames, int T, int m, int n, const double2 *tw_x, int fx, const double2 *tw_y, int Ky,
             const double2 *tw_t, int Kt, int K, double2 *work, double2 *X, cudaStream_t s) {
    const int Kx = 2 * K + 1;
    const int64_t rows = (int64_t)T * m;
    double2 *P = work, *Q = work + rows * fx;
    darts_rows_kernel<F><<<dim3((unsigned)b200::ceil_div64(rows, XR), (unsigned)b200::ceil_div(fx, XF)), XTHREADS, 0, s>>>(
        frames, rows, n, tw_x, fx, P);
    B200_LAUNCH_CHECK();
    const int64_t nq = (int64_t)Kt * m * Kx;
    darts_time_kernel<<<(unsigned)b200::ceil_div64(nq, 256), 256, 0, s>>>(P, T, m, n, fx, K, tw_t, Kt, Q);
    B200_LAUNCH_CHECK();
    darts_cols_kernel<<<dim3((unsigned)b200::ceil_div(Kx, YKX), (unsigned)b200::ceil_div(Ky, YKY), (unsigned)Kt), 256, 0,
                        s>>>(Q, m, Kx, tw_y, Ky, X);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int b200_darts_spectrum(const void *frames, int dtype, int T, int m, int n, const double *tw_x, int fx,
                                   const double *tw_y, int Ky, const double *tw_t, int Kt, int K, double *work,
                                   double *spectrum_out, void *stream) {
    B200_REQUIRE(T > 0 && m > 0 && n > 0 && K >= 0 && Kt > 0 && Ky > 0 && fx > 0, "darts: bad sizes");
    B200_REQUIRE(2 * K + 1 <= 2 * n + 1 && fx <= n / 2 + 1 && (int64_t)T * m * n < ((int64_t)1 << 40),
                 "darts: bad sizes");
    B200_REQUIRE(frames && tw_x && tw_y && tw_t && work && spectrum_out, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const double2 *tx = (const double2 *)tw_x, *ty = (const double2 *)tw_y, *tt = (const double2 *)tw_t;
    double2 *w = (double2 *)work, *X = (double2 *)spectrum_out;
    return b200::with_dtype("frame", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        return spectrum<F>((const F *)frames, T, m, n, tx, fx, ty, Ky, tt, Kt, K, w, X, s);
    });
}

extern "C" int b200_darts_normal(const double *spectrum_in, int N_x, int N_y, int N_t, int M_x, int M_y, double sx,
                                 double sy, double *work, double *mm, double *mhy, void *stream) {
    B200_REQUIRE(N_x >= 0 && N_y >= 0 && N_t >= 0 && M_x >= 0 && M_y >= 0, "darts: bad sizes");
    B200_REQUIRE(spectrum_in && work && mm && mhy, "bad arguments");
    Normal a;
    a.X = (const double2 *)spectrum_in;
    a.Nx = N_x, a.Ny = N_y, a.Nt = N_t, a.Mx = M_x, a.My = M_y;
    a.Kx = 2 * (N_x + M_x) + 1, a.Ky = 2 * (N_y + M_y) + 1;
    a.rows = (int64_t)(2 * N_t + 1) * (2 * N_y + 1) * (2 * N_x + 1);
    a.hw = (2 * M_x + 1) * (2 * M_y + 1);
    a.nc = 2 * a.hw;
    B200_REQUIRE(a.nc <= B200_DARTS_MAX_COLS, "darts: more than B200_DARTS_MAX_COLS columns");
    B200_REQUIRE(a.rows < ((int64_t)1 << 31) && (int64_t)a.Kx * a.Ky * (2 * N_t + 1) < ((int64_t)1 << 40),
                 "darts: more than 2^31 rows");
    a.npairs = a.nc * (a.nc + 1) / 2 + a.nc;
    a.sx = sx, a.sy = sy;
    const int G = (int)b200::ceil_div64(a.rows, NR_ROWS);
    const size_t smem = sizeof(double2) * NR_SUB * (a.nc + 1);
    B200_CUDA(cudaFuncSetAttribute(darts_normal_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaStream_t s = (cudaStream_t)stream;
    double2 *part = (double2 *)work;
    darts_normal_kernel<<<dim3((unsigned)G, (unsigned)b200::ceil_div(a.npairs, NR_SLAB)), NR_THREADS, smem, s>>>(a, part);
    B200_LAUNCH_CHECK();
    darts_normal_final_kernel<<<(unsigned)b200::ceil_div(a.npairs, 256), 256, 0, s>>>(part, G, a.npairs, a.nc,
                                                                                      (double2 *)mm, (double2 *)mhy);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_darts_synthesize(const double *coef, int h, int w, const double *ey, const double *ex, int m,
                                     int n, double *out, void *stream) {
    B200_REQUIRE(h > 0 && w > 0 && m > 0 && n > 0 && h <= m && w <= n, "darts: bad sizes");
    B200_REQUIRE(w <= B200_DARTS_MAX_SIDE, "darts: more than B200_DARTS_MAX_SIDE output columns");
    B200_REQUIRE(m <= 2147483647 / 2 && coef && ey && ex && out, "bad arguments");
    const double scale = 1.0 / ((double)m * (double)n);
    darts_synth_kernel<<<dim3((unsigned)m, 2), 256, 0, (cudaStream_t)stream>>>(
        (const double2 *)coef, h, w, (const double2 *)ey, (const double2 *)ex, m, n, scale, out);
    B200_LAUNCH_CHECK();
    return 0;
}
