// spline_body.cuh -- per-thread bodies of the spline kernels (spline.cu), written so that the
// SAME source also compiles as plain host C++: tests/host_kernels/ builds it with g++
// (-ffp-contract=off) and tests/test_kernel_bodies.py runs every body on the CPU against the
// oracle, bit for bit, without a GPU.  On the device every float64 operation is an explicit
// round-to-nearest intrinsic; on the host it is the plain operator.
#pragma once
#include <limits.h>
#include <math.h>
#include <stddef.h>

#include "../../include/pysteps_b200.h"

#if defined(__CUDACC__)
#define SPL_FN __host__ __device__ __forceinline__
#else
#define SPL_FN inline
#endif

namespace spl {

#if defined(__CUDA_ARCH__)
SPL_FN double add(double a, double b) { return __dadd_rn(a, b); }
SPL_FN double sub(double a, double b) { return __dsub_rn(a, b); }
SPL_FN double mul(double a, double b) { return __dmul_rn(a, b); }
SPL_FN double dvd(double a, double b) { return __ddiv_rn(a, b); }
SPL_FN double ld(const double *p) { return __ldg(p); }
#else
SPL_FN double add(double a, double b) { return a + b; }
SPL_FN double sub(double a, double b) { return a - b; }
SPL_FN double mul(double a, double b) { return a * b; }
SPL_FN double dvd(double a, double b) { return a / b; }
SPL_FN double ld(const double *p) { return *p; }
#endif

constexpr int NPAD = 12;  // scipy.ndimage._prepad_for_spline_filter

// ---- preparation: element e of the padded float64 copy (+ the two masks) -------------------------
template <typename F>
SPL_FN void prepare_element(size_t e, const F *precip, int m, int n, int pad, const double *stats,
                            int zero_fill, int want_masks, double *f, double *mask_min, double *mask_fin) {
    const int N = n + 2 * pad;
    const int i = (int)(e / (size_t)N), j = (int)(e % (size_t)N);
    int si = i - pad, sj = j - pad;
    si = si < 0 ? 0 : (si > m - 1 ? m - 1 : si);
    sj = sj < 0 ? 0 : (sj > n - 1 ? n - 1 : sj);
    const double v = (double)precip[(size_t)si * n + sj];
    const bool fin = isfinite(v);
    f[e] = (zero_fill && !fin) ? 0.0 : v;  // semilagrangian.py:150-152
    if (want_masks && i - pad == si && j - pad == sj) {
        const double minval = stats[1];  // np.nanmin(precip), :147
        const size_t q = (size_t)si * n + sj;
        mask_min[q] = (v > minval) ? 1.0 : 0.0;         // :148 (NaN > x is False)
        mask_fin[q] = (zero_fill && !fin) ? 0.0 : 1.0;  // :149-155
    }
}

// ---- one line of the prefilter: L samples with stride S, in place -------------------------------
// scipy's apply_filter: the gain of all poles first, then for every pole z the causal
// initialisation, the causal recursion, the anti-causal initialisation and recursion.
// reflect == 0: "mirror" initialisation, zpow = z^(L-1); reflect != 0: "reflect", zpow = z^L
SPL_FN void filter_pole(double *c, int L, size_t S, double z, double zpow, int reflect) {
#define SPL_C(i) c[(size_t)(i) * S]
    double s;
    if (!reflect) {
        double z_i = z;
        s = add(SPL_C(0), mul(zpow, SPL_C(L - 1)));
        for (int i = 1; i < L - 1; i++) {
            s = add(s, mul(z_i, add(SPL_C(i), mul(zpow, SPL_C(L - 1 - i)))));
            z_i = mul(z_i, z);
        }
        s = dvd(s, sub(1.0, mul(zpow, zpow)));
    } else {
        double z_i = z;
        const double c0 = SPL_C(0);
        s = add(c0, mul(zpow, SPL_C(L - 1)));
        for (int i = 1; i < L; i++) {
            // scipy accumulates into c[0] in place, so the last term (i == L-1) pairs c[L-1]
            // with the PARTIAL SUM standing in c[0], not with the original first sample
            const double partner = (i == L - 1) ? s : SPL_C(L - 1 - i);
            s = add(s, mul(z_i, add(SPL_C(i), mul(zpow, partner))));
            z_i = mul(z_i, z);
        }
        s = mul(s, dvd(z, sub(1.0, mul(zpow, zpow))));
        s = add(s, c0);
    }
    // causal recursion c[i] += z * c[i-1]
    double prev = s;
    double before = s;  // c[L-2] after the causal pass
    SPL_C(0) = s;
    for (int i = 1; i < L; i++) {
        const double cur = add(SPL_C(i), mul(z, prev));
        SPL_C(i) = cur;
        before = prev;
        prev = cur;
    }
    // anti-causal initialisation
    double last;
    if (!reflect)
        last = dvd(mul(add(mul(z, before), prev), z), sub(mul(z, z), 1.0));
    else
        last = mul(prev, dvd(z, sub(z, 1.0)));
    SPL_C(L - 1) = last;
    // anti-causal recursion c[i] = z * (c[i+1] - c[i])
    double next = last;
    for (int i = L - 2; i >= 0; i--) {
        const double cur = mul(z, sub(next, SPL_C(i)));
        SPL_C(i) = cur;
        next = cur;
    }
#undef SPL_C
}

struct FilterParams {
    int npoles, reflect;
    double gain;        // prod over poles of (1 - z)(1 - 1/z), evaluated on the host
    double z[2], zpow[2];
};

SPL_FN void filter_line(double *c, int L, size_t S, const FilterParams &fp) {
    if (L <= 1) return;
    for (int i = 0; i < L; i++) c[(size_t)i * S] = mul(c[(size_t)i * S], fp.gain);
    for (int k = 0; k < fp.npoles; k++) filter_pole(c, L, S, fp.z[k], fp.zpow[k], fp.reflect);
}

// ---- (R, C) -> (C, R) through a 32x32 tile: the two phases of one thread (tx < 32, ty < 8) of a
// block whose tile starts at column bx, row by; a barrier separates them ------------------------------
SPL_FN void transpose_load(double (*tile)[33], const double *in, int R, int C, int bx, int by, int tx, int ty) {
    for (int r = ty; r < 32; r += 8) {
        const int y = by + r, x = bx + tx;
        if (y < R && x < C) tile[r][tx] = in[(size_t)y * C + x];
    }
}

SPL_FN void transpose_store(double (*tile)[33], double *out, int R, int C, int bx, int by, int tx, int ty) {
    for (int r = ty; r < 32; r += 8) {
        const int y = bx + r, x = by + tx;  // coordinates in the transposed array
        if (y < C && x < R) out[(size_t)y * R + x] = tile[tx][r];
    }
}

// ---- sampling ------------------------------------------------------------------------------------
// (npy_intp)floor(c) on x86-64: out of range or non-finite -> INT64_MIN
SPL_FN long long cast_floor(double f) {
    if (!(f >= -9223372036854775808.0 && f < 9223372036854775808.0)) return LLONG_MIN;
    return (long long)f;
}

SPL_FN long long mirror_index(long long idx, long long len) {
    if (len <= 1) return 0;
    const long long s2 = 2 * len - 2;
    if (idx < 0) {
        idx = s2 * (-idx / s2) + idx;
        idx = idx <= 1 - len ? idx + s2 : -idx;
    } else if (idx >= len) {
        idx -= s2 * (idx / s2);
        if (idx >= len) idx = s2 - idx;
    }
    return idx;
}

SPL_FN long long tap_index(long long base, long long off, long long len, int mode) {
    if (mode == B200_MODE_CONSTANT) return mirror_index(base + off, len);
    const long long i = (long long)((unsigned long long)base + (unsigned long long)off);  // wraps like scipy
    return i < 0 ? 0 : (i >= len ? len - 1 : i);
}

// mode="constant": a coordinate outside [0, M-1] x [0, N-1] samples cval
SPL_FN bool outside_grid(double cy, double cx, long long M, long long N) {
    return !(cy >= 0.0 && cy <= (double)(M - 1) && cx >= 0.0 && cx <= (double)(N - 1));
}

// order 0: flat index of the nearest tap, floor(c + 0.5) on both axes (used by sample_pixel and by
// the shifted-frame correlation of constant.cu)
SPL_FN long long order0_index(double cy, double cx, long long M, long long N, int mode) {
    const long long iy = tap_index(cast_floor(floor(add(cy, 0.5))), 0, M, mode);
    const long long ix = tap_index(cast_floor(floor(add(cx, 0.5))), 0, N, mode);
    return iy * N + ix;
}

// get_spline_interpolation_weights of scipy's ni_splines.c (orders 2..5): x becomes the offset from
// the middle knot, the last weight is one minus the others
SPL_FN void spline_weights(double x, int order, double *w) {
    x = (order & 1) ? sub(x, floor(x)) : sub(x, floor(add(x, 0.5)));
    double y = x, z = sub(1.0, x), t;
    switch (order) {
    case 2:
        w[1] = sub(0.75, mul(x, x));
        y = sub(0.5, x);
        w[0] = mul(mul(0.5, y), y);
        break;
    case 3:
        w[1] = dvd(add(mul(mul(mul(y, y), sub(y, 2.0)), 3.0), 4.0), 6.0);
        w[2] = dvd(add(mul(mul(mul(z, z), sub(z, 2.0)), 3.0), 4.0), 6.0);
        w[0] = dvd(mul(mul(z, z), z), 6.0);
        break;
    case 4:
        t = mul(x, x);
        w[2] = add(mul(t, sub(mul(t, 0.25), 0.625)), 115.0 / 192.0);
        y = add(1.0, x);
        w[1] = add(mul(y, add(mul(y, sub(dvd(mul(y, sub(5.0, y)), 6.0), 1.25)), 5.0 / 24.0)), 55.0 / 96.0);
        w[3] = add(mul(z, add(mul(z, sub(dvd(mul(z, sub(5.0, z)), 6.0), 1.25)), 5.0 / 24.0)), 55.0 / 96.0);
        t = sub(0.5, x);
        t = mul(t, t);
        w[0] = dvd(mul(t, t), 24.0);
        break;
    case 5:
        t = mul(y, y);
        w[2] = add(mul(t, sub(mul(t, sub(0.25, dvd(y, 12.0))), 0.5)), 0.55);
        t = mul(z, z);
        w[3] = add(mul(t, sub(mul(t, sub(0.25, dvd(z, 12.0))), 0.5)), 0.55);
        y = add(y, 1.0);
        w[1] = add(mul(y, add(mul(y, sub(mul(y, add(mul(y, sub(dvd(y, 24.0), 0.375)), 1.25)), 1.75)), 0.625)), 0.425);
        z = add(z, 1.0);
        w[4] = add(mul(z, add(mul(z, sub(mul(z, add(mul(z, sub(dvd(z, 24.0), 0.375)), 1.25)), 1.75)), 0.625)), 0.425);
        z = sub(1.0, x);
        t = mul(z, z);
        w[0] = dvd(mul(mul(z, t), t), 120.0);
        break;
    default:
        break;
    }
    double last = 1.0;
    for (int i = 0; i < order; i++) last = sub(last, w[i]);
    w[order] = last;
}

// scipy map_coordinates(order=1, prefilter=False) of a float64 (m, n) array, generic path
// (see sl.cu / oracle/sl_oracle.c for the pinned semantics)
SPL_FN double sample_order1(const double *a, int m, int n, double cy, double cx, int mode, double cval) {
    if (mode == B200_MODE_CONSTANT) {
        if (!(cy >= 0.0 && cy <= (double)(m - 1) && cx >= 0.0 && cx <= (double)(n - 1))) return cval;
    }
    const double fy = floor(cy), fx = floor(cx);
    const double ty = sub(cy, fy), tx = sub(cx, fx);
    const long long iy = cast_floor(fy), ix = cast_floor(fx);
    long long ys[2], xs[2];
    if (mode == B200_MODE_NEAREST) {
        for (int l = 0; l < 2; l++) {
            const long long ty_ = iy == LLONG_MIN ? iy : iy + l, tx_ = ix == LLONG_MIN ? ix : ix + l;
            ys[l] = ty_ < 0 ? 0 : (ty_ >= m ? m - 1 : ty_);
            xs[l] = tx_ < 0 ? 0 : (tx_ >= n ? n - 1 : tx_);
        }
    } else {  // only the tap one past the end (c == L-1) can be out of range: mirrored
        ys[0] = iy; xs[0] = ix;
        ys[1] = (iy + 1 < m) ? iy + 1 : (m > 1 ? m - 2 : 0);
        xs[1] = (ix + 1 < n) ? ix + 1 : (n > 1 ? n - 2 : 0);
    }
    double wy[2], wx[2];
    wy[0] = sub(1.0, ty); wy[1] = sub(1.0, wy[0]);
    wx[0] = sub(1.0, tx); wx[1] = sub(1.0, wx[0]);
    double t = 0.0;
    for (int j = 0; j < 2; j++)
        for (int k = 0; k < 2; k++) t = add(t, mul(mul(ld(a + ys[j] * n + xs[k]), wy[j]), wx[k]));
    return t;
}

struct SampleParams {
    const double *coeffs;   // (m + 2 pad, n + 2 pad) prepared field
    const double *xy;       // (2, m, n) or null -> pixel grid
    const double *disp;     // (T, 2, rows, n) displacement after every leadtime
    const double *mask_min, *mask_fin, *stats;  // order > 1 only
    void *out;              // (T, rows, n)
    int m, n, pad, order, mode, T, row0, rows;
    double cval;
};

// value of output pixel (row0 + yl, x) at leadtime t (semilagrangian.py:221-253)
SPL_FN double sample_pixel(const SampleParams &p, int x, int yl, int t) {
    const int y = p.row0 + yl;
    const size_t NB = (size_t)p.rows * p.n, NF = (size_t)p.m * p.n;
    const size_t idx = (size_t)yl * p.n + x, gidx = (size_t)y * p.n + x;
    const double gx = p.xy ? p.xy[gidx] : (double)x;
    const double gy = p.xy ? p.xy[NF + gidx] : (double)y;
    const double *d = p.disp + (size_t)t * 2 * NB;
    const double cx0 = add(gx, d[idx]);  // coords_warped = xy_coords + displacement (:221-222)
    const double cy0 = add(gy, d[NB + idx]);
    const long long M = p.m + 2 * p.pad, N = p.n + 2 * p.pad;
    const double cy = add(cy0, (double)p.pad), cx = add(cx0, (double)p.pad);
    double v;
    bool outside = false;
    if (p.mode == B200_MODE_CONSTANT) outside = outside_grid(cy, cx, M, N);
    if (outside) {
        v = p.cval;
    } else if (p.order == 0) {
        v = add(0.0, ld(p.coeffs + order0_index(cy, cx, M, N, p.mode)));
    } else {
        const int order = p.order, half = p.order / 2;
        const long long by = cast_floor((order & 1) ? floor(cy) : floor(add(cy, 0.5)));
        const long long bx = cast_floor((order & 1) ? floor(cx) : floor(add(cx, 0.5)));
        long long ys[6], xs[6];
        for (int l = 0; l <= order; l++) {
            ys[l] = tap_index(by, l - half, M, p.mode);
            xs[l] = tap_index(bx, l - half, N, p.mode);
        }
        double wy[6], wx[6];
        spline_weights(cy, order, wy);
        spline_weights(cx, order, wx);
        v = 0.0;
        for (int j = 0; j <= order; j++)
            for (int k = 0; k <= order; k++) v = add(v, mul(mul(ld(p.coeffs + ys[j] * N + xs[k]), wy[j]), wx[k]));
    }
    if (p.order > 1) {  // :234-253
        if (sample_order1(p.mask_min, p.m, p.n, cy0, cx0, p.mode, 0.0) < 0.5) v = p.stats[1];
        if (sample_order1(p.mask_fin, p.m, p.n, cy0, cx0, p.mode, 0.0) < 0.5) v = (double)NAN;
    }
    return v;
}

}  // namespace spl
