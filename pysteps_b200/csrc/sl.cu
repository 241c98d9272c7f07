// sl.cu -- semi-Lagrangian backward-trajectory extrapolation (sm_90a).
//
// Replaces the leadtime loop of pysteps/extrapolation/semilagrangian.py:181-232:
// per leadtime, two bilinear gathers of the advection field along the
// trajectory (interpolate_motion, :181-198) and one bilinear warp of the
// precipitation field (:221-232).  In the reference each of these is a
// full-array scipy.ndimage.map_coordinates call plus NumPy temporaries.  Here a
// pixel's whole trajectory is independent of every other pixel's, so ONE kernel
// carries (displacement, velocity increment) of a pixel in float64 registers
// through all T leadtimes: the only HBM traffic is the compulsory read of the
// fields (L2 resident afterwards) and the T output planes.
//
// Arithmetic contract (pinned against scipy 1.18.1, see oracle/sl_oracle.c):
// every float64 operation of the reference is issued in the same order with
// round-to-nearest and NO fused multiply-add, so trajectories -- and therefore
// the integer tap indices -- are bit-identical to the CPU path.
#include "common.cuh"

namespace {

constexpr int SL_MAX_T = 32;  // leadtimes per launch; longer sequences are chunked
constexpr int SL_BX = 32, SL_BY = 4;  // 32x4 pixel CTAs measured best (0.45 vs 0.48 ms at 32x8, 0.50 at 32x16)

enum { SL_INIT_FRESH = 0, SL_INIT_PREV = 1, SL_INIT_RESUME = 2 };

struct SLParams {
    const void *Vi;         // (m,n) double2 (vx,vy)
    const void *precip;     // (m,n) float64 or null
    const double *xy;       // (2,m,n) or null -> pixel grid
    const double *disp_in;  // (2,m,n) or null
    const double *vinc_in;  // (2,m,n), RESUME only
    double *disp_out;       // (2,m,n) or null
    double *vinc_out;       // (2,m,n) or null
    void *out;              // (T,m,n) planes of this chunk
    int m, n, T, n_iter, ti_offset, init_mode, mode, has_prev;
    int row0, rows;         // output band [row0, row0 + rows): band-shaped out / disp arrays
    // batched members (blockIdx.z): element strides between consecutive members, 0 when unused
    size_t zs_vi, zs_precip, zs_disp, zs_out;
    double vts, td0, cval;
    double scale[SL_MAX_T];  // td / vel_timestep per leadtime
};

// ---- exact float64 building blocks ---------------------------------------------------
// The XU pipe (conversions, FRND, MUFU) is the scarce unit for this kernel, so the hot
// path avoids it: fields are pre-widened to float64 once per call, floor() comes from a
// magic-constant add on the FP64 pipe, and no division is issued per leadtime.

constexpr double SL_MAGIC = 6755399441055744.0;  // 2^52 + 2^51

// floor(c) and (int)floor(c) for -2^31 < c < 2^31 without FRND/F2I
__device__ __forceinline__ void floor_magic(double c, double &f, int &i) {
    const double t = __dadd_rn(c, SL_MAGIC);  // nearest integer (ties to even) in the low bits
    i = __double2loint(t);
    f = __dsub_rn(t, SL_MAGIC);
    if (f > c) {
        f = __dsub_rn(f, 1.0);
        i -= 1;
    }
}

struct Axis {
    int i0, i1;      // tap indices, mode "nearest" (clamped to [0, L-1])
    int f0;          // (int)floor(c), unclamped, valid when `inside`
    double w0, w1;   // 1 - t, 1 - w0
    bool inside;     // 0 <= c <= L-1  (mode "constant" validity)
};

// one axis of scipy's order-1 footprint: taps floor(c), floor(c)+1; weights w0 = 1 - t,
// w1 = 1 - w0 with t = c - floor(c).
__device__ __forceinline__ Axis make_axis(double c, int L) {
    Axis a;
    double f;
    int i;
    if (c > -2.0 && c < (double)L + 1.0) {
        floor_magic(c, f, i);
    } else {
        // rare (trajectory far outside the domain, or NaN): generic path.
        // (npy_intp)floor(c) on x86-64: out-of-range / non-finite -> INT64_MIN (both taps 0)
        f = floor(c);
        double fc = (fabs(f) < 9223372036854775808.0) ? f : -1.0;
        fc = fmin(fmax(fc, -1.0), (double)L);
        i = (int)fc;
    }
    const double t = __dsub_rn(c, f);
    a.w0 = __dsub_rn(1.0, t);
    a.w1 = __dsub_rn(1.0, a.w0);
    a.f0 = i;
    a.i0 = min(max(i, 0), L - 1);
    a.i1 = min(max(i + 1, 0), L - 1);
    a.inside = (c >= 0.0) && (c <= (double)(L - 1));
    return a;
}

// sum_{taps} ((a * wy) * wx), left to right from 0.0 (scipy accumulation order)
// (the leading 0.0 + is scipy's accumulator start: it turns a first product of -0.0 into +0.0.
// Doing that with integer compares instead, and velocity_inc / 2 by an exponent decrement, adds
// integer instructions to a kernel that is as much issue-bound as FP64-bound)
__device__ __forceinline__ double bilin(double a00, double a01, double a10, double a11,
                                        double wy0, double wy1, double wx0, double wx1) {
    double t = __dadd_rn(0.0, __dmul_rn(__dmul_rn(a00, wy0), wx0));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(a01, wy0), wx1));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(a10, wy1), wx0));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(a11, wy1), wx1));
    return t;
}

// ---- slow (generic) path: any coordinate, per-tap index clamping --------------------
// (results by value: reference parameters of a non-inlined function would pin the caller's
// velocity registers to the local-memory stack -- one STL pair per sample on the FAST path too)
__device__ __noinline__ double2 slow_velocity(const double2 *__restrict__ Vi, int m, int n, double cy,
                                              double cx) {
    const Axis ay = make_axis(cy, m), ax = make_axis(cx, n);
    const double2 *r0 = Vi + (size_t)ay.i0 * n;
    const double2 *r1 = Vi + (size_t)ay.i1 * n;
    const double2 a00 = __ldg(r0 + ax.i0), a01 = __ldg(r0 + ax.i1);
    const double2 a10 = __ldg(r1 + ax.i0), a11 = __ldg(r1 + ax.i1);
    return make_double2(bilin(a00.x, a01.x, a10.x, a11.x, ay.w0, ay.w1, ax.w0, ax.w1),
                        bilin(a00.y, a01.y, a10.y, a11.y, ay.w0, ay.w1, ax.w0, ax.w1));
}

// map_coordinates(precip, order=1, mode, cval) for one pixel (:221-232), generic path
// (PT: storage type of the field; the trajectory kernel reads float64, widened once per call)
template <typename PT>
__device__ __noinline__ double slow_precip(const PT *__restrict__ P, int m, int n, double cy,
                                           double cx, int mode, double cval) {
    const Axis ay = make_axis(cy, m), ax = make_axis(cx, n);
    int y0 = ay.i0, y1 = ay.i1, x0 = ax.i0, x1 = ax.i1;
    if (mode == B200_MODE_CONSTANT) {
        if (!(ay.inside && ax.inside)) return cval;
        // the tap one past the end (only when c == L-1) is mirrored and still read
        y0 = ay.f0; x0 = ax.f0;
        y1 = (y0 + 1 < m) ? y0 + 1 : (m > 1 ? m - 2 : 0);
        x1 = (x0 + 1 < n) ? x0 + 1 : (n > 1 ? n - 2 : 0);
    }
    const PT *r0 = P + (size_t)y0 * n;
    const PT *r1 = P + (size_t)y1 * n;
    return bilin((double)__ldg(r0 + x0), (double)__ldg(r0 + x1), (double)__ldg(r1 + x0), (double)__ldg(r1 + x1),
                 ay.w0, ay.w1, ax.w0, ax.w1);
}

// ---- fast path: footprint strictly inside the array ------------------------------------
// floor via a round-DOWN add of 2^52+2^51: the sum's low word IS (int)floor(c) and its high
// word is 0x43380000 exactly when 0 <= floor(c) < 2^32, so validity, floor and the integer
// index cost two FP64-pipe adds and integer compares -- no FRND/F2I/I2F (XU pipe).
struct Foot {
    int base;  // y0 * n + x0
    double wy0, wy1, wx0, wx1;
    bool interior;  // taps (y0, y0+1) x (x0, x0+1) all in range: modes coincide, no clamping
};

__device__ __forceinline__ Foot footprint(double cy, double cx, int n, int ymax, int xmax) {
    Foot f;
    const double sy = __dadd_rd(cy, SL_MAGIC), sx = __dadd_rd(cx, SL_MAGIC);
    const int iy = __double2loint(sy), ix = __double2loint(sx);
    // (unsigned compares against ymax + 1 = m - 1 >= 0: the high-word test admits 0 <= floor < 2^32, an index
    // of 2^31 or more reads as a negative int and must fail like every other index beyond the last row)
    f.interior = (__double2hiint(sy) == 0x43380000) & (__double2hiint(sx) == 0x43380000) &
                 ((unsigned)iy < (unsigned)(ymax + 1)) & ((unsigned)ix < (unsigned)(xmax + 1));
    const double ty = __dsub_rn(cy, __dsub_rn(sy, SL_MAGIC));
    const double tx = __dsub_rn(cx, __dsub_rn(sx, SL_MAGIC));
    f.wy0 = __dsub_rn(1.0, ty); f.wy1 = __dsub_rn(1.0, f.wy0);
    f.wx0 = __dsub_rn(1.0, tx); f.wx1 = __dsub_rn(1.0, f.wx0);
    f.base = iy * n + ix;
    return f;
}

// interpolate_motion (semilagrangian.py:181-198) for one pixel; returns the footprint so
// the precip warp at the same coordinates can reuse it
template <bool VF32>
__device__ __forceinline__ Foot sample_velocity(const double2 *__restrict__ Vi, int m, int n,
                                                int ymax, int xmax, double cy, double cx,
                                                double scale, int n_iter,
                                                double &vx, double &vy) {
    const Foot f = footprint(cy, cx, n, ymax, xmax);
    if (f.interior) {
        const double2 *q = Vi + f.base;
        const double2 a00 = __ldg(q), a01 = __ldg(q + 1);
        const double2 a10 = __ldg(q + n), a11 = __ldg(q + n + 1);
        vx = bilin(a00.x, a01.x, a10.x, a11.x, f.wy0, f.wy1, f.wx0, f.wx1);
        vy = bilin(a00.y, a01.y, a10.y, a11.y, f.wy0, f.wy1, f.wx0, f.wx1);
    } else {
        const double2 v = slow_velocity(Vi, m, n, cy, cx);
        vx = v.x;
        vy = v.y;
    }
    if (VF32) {
        // float32 velocity: map_coordinates returns the input dtype, so the reference
        // stores the sampled increment rounded to float32 (:192-193)
        vx = (double)__double2float_rn(vx);
        vy = (double)__double2float_rn(vy);
    }
    if (n_iter > 1) {  // :195-196
        vx = __ddiv_rn(vx, (double)n_iter);
        vy = __ddiv_rn(vy, (double)n_iter);
    }
    vx = __dmul_rn(vx, scale);  // :198
    vy = __dmul_rn(vy, scale);
    return f;
}

template <typename F> __device__ __forceinline__ F from_double(double v);
template <> __device__ __forceinline__ float from_double<float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double from_double<double>(double v) { return v; }

// NITER1: n_iter == 1 (the default and what every nowcast method uses) compiled without
// the inner loop / division branches.
// VF32: the velocity was float32 at the API (a compile-time fact of the launch: the rounding of
// the sampled increments costs conversion-pipe slots even when predicated off).
// One pixel's whole trajectory (all T leadtimes of the launch).  PT: storage type of the
// precipitation field (float64 in the trajectory kernel; the input type when this runs as the exact
// fallback of the float32-tap kernel below).
template <typename F, bool NITER1, bool VF32, bool BATCH, typename PT>
__device__ __forceinline__ void sl_pixel(const SLParams &p, const int x, const int yl, const size_t z) {
    const int y = p.row0 + yl;
    const int m = p.m, n = p.n;
    const int ymax = m - 2, xmax = n - 2;  // largest interior floor index (negative: none)
    const size_t N = (size_t)p.rows * n;   // plane stride of the band-shaped arrays
    const size_t NF = (size_t)m * n;       // plane stride of the full-frame arrays
    const int idx = yl * n + x;            // pixel index inside the band
    const int gidx = y * n + x;            // pixel index inside the full frame
    const double2 *__restrict__ Vi = (const double2 *)p.Vi + (BATCH ? z * p.zs_vi : 0);
    const PT *__restrict__ P = (const PT *)p.precip + (BATCH ? z * p.zs_precip : 0);
    F *__restrict__ out = (F *)p.out + (BATCH ? z * p.zs_out : 0) + idx;
    const double *__restrict__ disp_in = p.disp_in + (BATCH ? z * p.zs_disp : 0);
    double *__restrict__ disp_out = p.disp_out ? p.disp_out + (BATCH ? z * p.zs_disp : 0) : nullptr;
    const int n_iter = NITER1 ? 1 : p.n_iter;
    const int mode = p.mode;
    const double cval = p.cval;
    const int T = p.T;

    double gx, gy;  // xy_coords of this pixel (:174-179)
    if (p.xy) {
        gx = p.xy[gidx];
        gy = p.xy[NF + gidx];
    } else {
        gx = (double)x;
        gy = (double)y;
    }

    double dx, dy, ux, uy;  // displacement, velocity increment
    if (p.init_mode == SL_INIT_FRESH) {
        // :201-203  displacement = 0 ; velocity_inc = V * tdiff[0] / vel_timestep
        dx = 0.0; dy = 0.0;
        const double2 v = Vi[gidx];
        ux = __ddiv_rn(__dmul_rn(v.x, p.td0), p.vts);
        uy = __ddiv_rn(__dmul_rn(v.y, p.td0), p.vts);
    } else if (p.init_mode == SL_INIT_PREV) {
        // :205-207
        dx = disp_in[idx]; dy = disp_in[N + idx];
        sample_velocity<VF32>(Vi, m, n, ymax, xmax, __dadd_rn(gy, dy), __dadd_rn(gx, dx), p.scale[0],
                        n_iter, ux, uy);
    } else {
        dx = disp_in[idx]; dy = disp_in[N + idx];
        ux = p.vinc_in[idx]; uy = p.vinc_in[N + idx];
    }

    for (int ti = 0; ti < T; ti++) {
        const double scale = p.scale[ti];  // td / vel_timestep (:198), divided on the host
        Foot f;
        f.interior = false;
        bool have_foot = false;  // f describes xy + displacement
        if (n_iter > 0) {
            for (int k = 0; k < n_iter; k++) {  // :211-214
                // velocity_inc / 2.0 == velocity_inc * 0.5 exactly
                const double hx = __dsub_rn(dx, __dmul_rn(ux, 0.5));
                const double hy = __dsub_rn(dy, __dmul_rn(uy, 0.5));
                sample_velocity<VF32>(Vi, m, n, ymax, xmax, __dadd_rn(gy, hy), __dadd_rn(gx, hx), scale,
                                n_iter, ux, uy);
                dx = __dsub_rn(dx, ux);
                dy = __dsub_rn(dy, uy);
                f = sample_velocity<VF32>(Vi, m, n, ymax, xmax, __dadd_rn(gy, dy), __dadd_rn(gx, dx),
                                    scale, n_iter, ux, uy);
            }
            // the precip warp samples at xy + displacement: the coordinates (hence footprint
            // and weights) of the last velocity gather
            have_foot = true;
        } else {  // :215-219
            if (ti + p.ti_offset > 0 || p.has_prev)
                sample_velocity<VF32>(Vi, m, n, ymax, xmax, __dadd_rn(gy, dy), __dadd_rn(gx, dx), scale,
                                n_iter, ux, uy);
            dx = __dsub_rn(dx, ux);
            dy = __dsub_rn(dy, uy);
        }
        if (P) {
            const double cy = __dadd_rn(gy, dy), cx = __dadd_rn(gx, dx);
            if (!have_foot) f = footprint(cy, cx, n, ymax, xmax);
            double v;
            if (f.interior) {
                const PT *q = P + f.base;
                v = bilin((double)__ldg(q), (double)__ldg(q + 1), (double)__ldg(q + n), (double)__ldg(q + n + 1),
                          f.wy0, f.wy1, f.wx0, f.wx1);
            } else {
                v = slow_precip(P, m, n, cy, cx, mode, cval);
            }
            out[(size_t)ti * N] = from_double<F>(v);
        }
    }
    if (disp_out) {
        disp_out[idx] = dx;
        disp_out[N + idx] = dy;
    }
    if (p.vinc_out) {
        p.vinc_out[idx] = ux;
        p.vinc_out[N + idx] = uy;
    }
}

template <typename F, bool NITER1, bool VF32, bool BATCH = false>
__global__ void __launch_bounds__(SL_BX *SL_BY)
sl_multistep_kernel(const __grid_constant__ SLParams p) {
    const int x = blockIdx.x * SL_BX + threadIdx.x;
    const int yl = blockIdx.y * SL_BY + threadIdx.y;  // row inside the band
    if (x >= p.n || yl >= p.rows) return;
    sl_pixel<F, NITER1, VF32, BATCH, double>(p, x, yl, BATCH ? blockIdx.z : 0);  // z: member of a batched launch
}

// ---- float32-tap variant (opt-in: tolerance on the VALUES, certified INDICES) ----------------------
// The trajectory stays in float64 (displacement, coordinates, floor, fractional weights), but the
// fields are sampled from float32 copies with float32 arithmetic: 8 instead of 16 bytes per velocity
// tap and ~20 instead of ~94 FP64-pipe instructions per pixel and leadtime.  What keeps the integer tap
// indices identical to the exact kernel's is a running error bound per pixel:
//   E   >= |displacement here - displacement of the exact kernel|  (max norm, pixels)
//   Eu  >= |velocity increment here - exact increment|
// A sample at coordinates c is CERTIFIED when its four taps are inside the array and the fractional
// parts lie in (e, 1 - e) for the bound e on |c - c_exact|: then both kernels floor to the same cell,
// and inside a cell the bilinear interpolant is Lipschitz with the slopes G read off the four taps, so
//   Eu' <= |scale| * (G * e + eps32 * (4.5 |v| + 4 G)),   eps32 = 2^-23, v the sampled velocity
// (with u = 2^-24 and every tap within G of v: tap rounding u(|v|+G); the two weights G u/2; the three
// lerps 3u(|v|+G) + 4u G inherited through the differences; the final rounding u|v|; the scale factor and
// its product 2u|v|; a float32 velocity's increment rounded by the reference, u|v|: u(8|v| + 7.5 G) in all).
// A pixel with ANY uncertified sample -- near a cell boundary (~1e-4 of the pixels at 12 leadtimes),
// near the array border, outside it, non-finite -- is recomputed from the start by sl_pixel, the exact
// kernel's own code, so every mode / outval / NaN rule holds unchanged.  Net contract: floor indices of
// every sample equal to the exact kernel's; values within float32 rounding of it (tests/test_sl_gpu.py
// states the tolerance).
struct SLFastParams {
    const float2 *Vf;   // (m,n) float32 (vx,vy)
    const void *Pf;     // (m,n) precipitation in its input type F
    float scale[SL_MAX_T];
    float s0;           // tdiff[0] / vel_timestep
    unsigned *nlist;    // number of listed pixels (zeroed before the launch)
    int *list;          // band-local pixel indices to recompute exactly (capacity: the band)
};

constexpr float SLF_EPS = 1.1920929e-07f;  // 2^-23
constexpr float SLF_INFLATE = 1.001f;      // slack for the float32 evaluation of the bound itself

struct FootF {
    int base;
    float tx, ty;
    bool ok;  // interior and certified
};

// one velocity sample of the float32 path at (cy, cx) with position error bound e;
// returns the sampled velocity (vx, vy) and the bound g >= (Gx + Gy) slope + the rounding term's factor
__device__ __forceinline__ FootF sample_f32(const float2 *__restrict__ Vf, int n, int ymax, int xmax, double cy,
                                            double cx, float e, float &vx, float &vy, float &err_coef) {
    FootF f;
    const double sy = __dadd_rd(cy, SL_MAGIC), sx = __dadd_rd(cx, SL_MAGIC);
    const int iy = __double2loint(sy), ix = __double2loint(sx);
    // (unsigned compares against ymax + 1 = m - 1 >= 0, see footprint())
    const bool interior = (__double2hiint(sy) == 0x43380000) & (__double2hiint(sx) == 0x43380000) &
                          ((unsigned)iy < (unsigned)(ymax + 1)) & ((unsigned)ix < (unsigned)(xmax + 1));
    f.ty = (float)__dsub_rn(cy, __dsub_rn(sy, SL_MAGIC));
    f.tx = (float)__dsub_rn(cx, __dsub_rn(sx, SL_MAGIC));
    // both fractions in (lo, 1 - lo) with lo = e + 2 eps  <=>  max |t - 1/2| < 1/2 - lo
    f.ok = interior & (fmaxf(fabsf(f.ty - 0.5f), fabsf(f.tx - 0.5f)) < 0.5f - (e + 2.f * SLF_EPS));
    f.base = iy * n + ix;
    if (f.ok) {
        const float2 *q = Vf + f.base;
        const float2 a00 = __ldg(q), a01 = __ldg(q + 1), a10 = __ldg(q + n), a11 = __ldg(q + n + 1);
        const float d0x = a01.x - a00.x, d1x = a11.x - a10.x, d0y = a01.y - a00.y, d1y = a11.y - a10.y;
        const float x0 = __fmaf_rn(f.tx, d0x, a00.x), x1 = __fmaf_rn(f.tx, d1x, a10.x);
        const float y0 = __fmaf_rn(f.tx, d0y, a00.y), y1 = __fmaf_rn(f.tx, d1y, a10.y);
        const float wx = x1 - x0, wy = y1 - y0;
        vx = __fmaf_rn(f.ty, wx, x0);
        vy = __fmaf_rn(f.ty, wy, y0);
        // slopes inside the cell: |d/dx| <= max(|d0|,|d1|) <= |d0|+|d1| =: D ; |d/dy| <= |w| + D
        const float gx = __fmaf_rn(2.f, fabsf(d0x) + fabsf(d1x), fabsf(wx));
        const float gy = __fmaf_rn(2.f, fabsf(d0y) + fabsf(d1y), fabsf(wy));
        const float g = fmaxf(gx, gy);
        const float av = fmaxf(fabsf(vx), fabsf(vy));
        err_coef = __fmaf_rn(g, e, SLF_EPS * __fmaf_rn(4.f, g, 4.5f * av));
    }
    return f;
}

// n_iter == 1, pixel-grid coordinates, a precipitation field, T <= SL_MAX_T (one launch).
// Pixels with an uncertified sample stop at once and are LISTED (one atomic per warp); the exact code
// runs on the compacted list in a second launch -- done inline, every warp holding a single such pixel
// (most warps, at a few percent of the pixels) would pay for the exact trajectory on top of the fast one.
template <typename F, bool VF32>
__global__ void __launch_bounds__(SL_BX *SL_BY)
sl_f32_kernel(const __grid_constant__ SLParams p, const __grid_constant__ SLFastParams q) {
    const int x = blockIdx.x * SL_BX + threadIdx.x;
    const int yl = blockIdx.y * SL_BY + threadIdx.y;
    const bool inb = x < p.n && yl < p.rows;
    const int n = p.n;
    const int idx = yl * n + x;
    bool good = true;
    if (inb) {
        const int y = p.row0 + yl;
        const int ymax = p.m - 2, xmax = n - 2;
        const size_t N = (size_t)p.rows * n;
        const int gidx = y * n + x;
        const float2 *__restrict__ Vf = q.Vf;
        const F *__restrict__ Pf = (const F *)q.Pf;
        F *__restrict__ out = (F *)p.out + idx;
        const double gx = (double)x, gy = (double)y;
        const int T = p.T;
        double dx, dy;
        float ux, uy, E = 0.f, Eu;
        if (p.init_mode == SL_INIT_FRESH) {
            dx = 0.0; dy = 0.0;
            const float2 v = Vf[gidx];
            ux = v.x * q.s0; uy = v.y * q.s0;
            Eu = 2.f * SLF_EPS * fmaxf(fabsf(ux), fabsf(uy));  // V -> float32, the scale factor, the product: 3 * 2^-24
        } else {  // SL_INIT_PREV
            dx = p.disp_in[idx]; dy = p.disp_in[N + idx];
            float vx = 0.f, vy = 0.f, ec = 0.f;
            const FootF f = sample_f32(Vf, n, ymax, xmax, __dadd_rn(gy, dy), __dadd_rn(gx, dx), 0.f, vx, vy, ec);
            good = f.ok;
            const float sf = q.scale[0];
            ux = vx * sf; uy = vy * sf;
            Eu = fabsf(sf) * ec * SLF_INFLATE;
        }
        for (int ti = 0; ti < T && good; ti++) {
            const float sf = q.scale[ti], sa = fabsf(sf) * SLF_INFLATE;
            float vx = 0.f, vy = 0.f, ec = 0.f;
            // midpoint sample at displacement - increment / 2
            const double hx = __fma_rn(-0.5, (double)ux, dx), hy = __fma_rn(-0.5, (double)uy, dy);
            FootF f = sample_f32(Vf, n, ymax, xmax, __dadd_rn(gy, hy), __dadd_rn(gx, hx), __fmaf_rn(0.5f, Eu, E), vx, vy, ec);
            good = f.ok;
            ux = vx * sf; uy = vy * sf;
            dx = __dsub_rn(dx, (double)ux);
            dy = __dsub_rn(dy, (double)uy);
            E = (E + sa * ec) * SLF_INFLATE + 1e-12f;
            // end-point sample: the next increment, and the footprint of the precipitation warp
            f = sample_f32(Vf, n, ymax, xmax, __dadd_rn(gy, dy), __dadd_rn(gx, dx), E, vx, vy, ec);
            good &= f.ok;
            ux = vx * sf; uy = vy * sf;
            Eu = sa * ec;
            if (good) {
                const F *r = Pf + f.base;
                const float a00 = (float)__ldg(r), a01 = (float)__ldg(r + 1), a10 = (float)__ldg(r + n),
                            a11 = (float)__ldg(r + n + 1);
                const float v0 = __fmaf_rn(f.tx, a01 - a00, a00), v1 = __fmaf_rn(f.tx, a11 - a10, a10);
                out[(size_t)ti * N] = (F)__fmaf_rn(f.ty, v1 - v0, v0);
            }
        }
        if (good && p.disp_out) {
            p.disp_out[idx] = dx;
            p.disp_out[N + idx] = dy;
        }
    }
    // list the pixels to recompute: one atomic per warp
    const unsigned bad = __ballot_sync(0xffffffffu, !good);
    if (bad) {
        const int lane = (threadIdx.y * SL_BX + threadIdx.x) & 31;
        unsigned base = 0;
        if (lane == __ffs(bad) - 1) base = atomicAdd(q.nlist, __popc(bad));
        base = __shfl_sync(0xffffffffu, base, __ffs(bad) - 1);
        if (!good) q.list[base + __popc(bad & ((1u << lane) - 1u))] = idx;
    }
}

// the listed pixels, by the exact kernel's own code (rewrites every leadtime and the displacement)
template <typename F, bool VF32>
__global__ void __launch_bounds__(128)
sl_f32_fixup_kernel(const __grid_constant__ SLParams p, const unsigned *__restrict__ nlist,
                    const int *__restrict__ list, unsigned long long *nfallback) {
    const unsigned cnt = *nlist;
    const unsigned stride = gridDim.x * blockDim.x;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += stride) {
        const int idx = list[i];
        const int yl = idx / p.n;
        sl_pixel<F, true, VF32, false, F>(p, idx - yl * p.n, yl, 0);
    }
    if (nfallback && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(nfallback, (unsigned long long)cnt);
}

// (2,m,n) planar or (m,n,2) interleaved pairs of type F -> (m,n) pairs of type P2 (rounded to nearest)
template <typename F, typename P2, bool INTERLEAVED>
__global__ void __launch_bounds__(256)
relayout_kernel(const F *__restrict__ V, P2 *__restrict__ out, size_t N) {
    using E = decltype(P2::x);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride) {
        P2 v;
        if (INTERLEAVED) {
            v.x = (E)__ldg(V + 2 * i);
            v.y = (E)__ldg(V + 2 * i + 1);
        } else {
            v.x = (E)__ldg(V + i);
            v.y = (E)__ldg(V + N + i);
        }
        out[i] = v;
    }
}

__global__ void __launch_bounds__(256)
widen_field_kernel(const float *__restrict__ a, double *__restrict__ o, size_t N) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride)
        o[i] = (double)__ldg(a + i);
}

// blocks of 256 threads for a grid-stride loop over N elements, at most per_sm of them per SM
int stream_blocks(size_t N, int per_sm) {
    return (int)std::min<size_t>((N + 255) / 256, (size_t)b200::num_sms() * per_sm);
}

// The velocity as (m,n) pairs of type P2: the caller's buffer when it already is one, otherwise a copy
// in `buf`, re-laid out and widened (float64 pairs: exact) or rounded (float32 pairs) from type F.
template <typename P2, typename F>
int velocity_pairs(const void *velocity, int layout, size_t N, b200::Scratch &buf, const P2 *&pairs,
                   cudaStream_t stream) {
    constexpr bool SAME = sizeof(P2) == 2 * sizeof(F);
    if (SAME && layout == B200_LAYOUT_INTERLEAVED) {
        pairs = (const P2 *)velocity;
        return 0;
    }
    B200_CUDA(buf.alloc(N * sizeof(P2), stream));
    pairs = (const P2 *)buf.p;
    const int blocks = stream_blocks(N, 16);
    if (layout == B200_LAYOUT_PLANAR)
        relayout_kernel<F, P2, false><<<blocks, 256, 0, stream>>>((const F *)velocity, (P2 *)buf.p, N);
    else if constexpr (!SAME)
        relayout_kernel<F, P2, true><<<blocks, 256, 0, stream>>>((const F *)velocity, (P2 *)buf.p, N);
    B200_LAUNCH_CHECK();
    return 0;
}

// The argument rules the row-band entry points share, in the order they are checked.  `args_ok` and
// `args_msg` are the entry point's own rule for its pointer arguments.
int check_band(int m, int n, int row0, int rows, int layout, bool args_ok, const char *args_msg,
               const double *tdiff, int T, int n_iter, int mode) {
    B200_REQUIRE(row0 >= 0 && rows >= 1 && row0 + rows <= m, "row band out of range");
    B200_REQUIRE(layout == B200_LAYOUT_PLANAR || layout == B200_LAYOUT_INTERLEAVED, "unknown velocity layout");
    B200_REQUIRE(args_ok, args_msg);
    B200_REQUIRE(tdiff != nullptr && T >= 1, "need at least one timestep");
    B200_REQUIRE(m >= 1 && n >= 1 && (int64_t)m * n < ((int64_t)1 << 30), "grid must have 1 .. 2^30 pixels");
    B200_REQUIRE(n_iter >= 0, "n_iter must be >= 0");
    B200_REQUIRE(mode == B200_MODE_CONSTANT || mode == B200_MODE_NEAREST, "unsupported mode");
    return 0;
}

// The fields of a trajectory launch that every driver sets alike, starting from `disp_prev` (or from rest).
// T, the scales, the outputs, and the resume and batch fields are the driver's.
SLParams sl_params(const double2 *Vi, const void *precip, const double *xy, const double *disp_prev, int m, int n,
                   int row0, int rows, int n_iter, int mode, double outval, double vts, double td0) {
    SLParams p;
    memset(&p, 0, sizeof(p));
    p.Vi = Vi;
    p.precip = precip;
    p.xy = xy;
    p.m = m; p.n = n;
    p.row0 = row0; p.rows = rows;
    p.n_iter = n_iter;
    p.mode = mode;
    p.vts = vts;
    p.td0 = td0;
    p.cval = outval;
    p.has_prev = disp_prev != nullptr;
    p.init_mode = disp_prev ? SL_INIT_PREV : SL_INIT_FRESH;
    p.disp_in = disp_prev;
    return p;
}

// The trajectory kernel over T lead times, `per_launch` of them per launch; each launch after the first
// resumes from the displacement and velocity increment the one before it left.  `out` (optional) holds
// the T output planes.  `disp_steps` (optional) receives every launch's displacement, one (2,rows,n)
// block per launch; without it the last launch's displacement goes to `disp_out` (optional).
template <typename F, bool VF32>
int sl_launches(const SLParams &start, const double *tdiff, int T, int per_launch, void *out, double *disp_out,
                double *disp_steps, cudaStream_t stream) {
    const size_t NB = (size_t)start.rows * start.n;
    const int launches = (T + per_launch - 1) / per_launch;
    b200::Scratch st_disp, st_vinc;
    if (launches > 1) {
        if (!disp_steps) B200_CUDA(st_disp.alloc(2 * NB * sizeof(double), stream));
        B200_CUDA(st_vinc.alloc(2 * NB * sizeof(double), stream));
    }
    dim3 block(SL_BX, SL_BY);
    dim3 grid(b200::ceil_div(start.n, SL_BX), b200::ceil_div(start.rows, SL_BY));
    const double *carried = nullptr;  // the displacement the previous launch wrote
    for (int c = 0; c < launches; c++) {
        SLParams p = start;
        p.ti_offset = c * per_launch;
        p.T = std::min(per_launch, T - p.ti_offset);
        for (int i = 0; i < p.T; i++) p.scale[i] = tdiff[p.ti_offset + i] / p.vts;
        if (c > 0) {
            p.init_mode = SL_INIT_RESUME;
            p.disp_in = carried;
            p.vinc_in = (const double *)st_vinc.p;
        }
        const bool last = (c == launches - 1);
        p.disp_out = disp_steps ? disp_steps + (size_t)c * 2 * NB : last ? disp_out : (double *)st_disp.p;
        p.vinc_out = last ? nullptr : (double *)st_vinc.p;
        p.out = out ? (void *)((F *)out + (size_t)p.ti_offset * NB) : nullptr;
        if (p.n_iter == 1)
            sl_multistep_kernel<F, true, VF32><<<grid, block, 0, stream>>>(p);
        else
            sl_multistep_kernel<F, false, VF32><<<grid, block, 0, stream>>>(p);
        B200_LAUNCH_CHECK();
        carried = p.disp_out;
    }
    return 0;
}

}  // namespace

// Displacement field after EVERY leadtime (for samplers other than the built-in order-1 warp):
// the trajectory kernel run one leadtime per launch through the same resume mechanism that
// chunks long sequences, so the arithmetic is that of the fused loop.
extern "C" int b200_sl_trajectories(const void *velocity, const double *xy_coords, const double *disp_prev,
                                    const double *tdiff, int T, double vel_timestep, int n_iter,
                                    int velocity_dtype, int velocity_layout, int m, int n, int row_begin,
                                    int row_count, double *disp_steps, void *stream) {
    if (int rc = check_band(m, n, row_begin, row_count, velocity_layout, velocity != nullptr && disp_steps != nullptr,
                            "velocity / disp_steps is NULL", tdiff, T, n_iter, B200_MODE_CONSTANT))
        return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("velocity", velocity_dtype, [&](auto fv) {
        using FV = typename decltype(fv)::type;
        b200::Scratch vi;
        const double2 *Vi;
        if (int rc = velocity_pairs<double2, FV>(velocity, velocity_layout, (size_t)m * n, vi, Vi, s)) return rc;
        const SLParams p = sl_params(Vi, nullptr, xy_coords, disp_prev, m, n, row_begin, row_count, n_iter,
                                     B200_MODE_CONSTANT, 0.0, vel_timestep, tdiff[0]);
        return sl_launches<double, sizeof(FV) == 4>(p, tdiff, T, 1, nullptr, nullptr, disp_steps, s);
    });
}

extern "C" int b200_sl_extrapolate_rows(const void *precip, const void *velocity,
                                        const double *xy_coords, const double *disp_prev,
                                        const double *tdiff, int T, double vel_timestep, int n_iter,
                                        double outval, int mode, int velocity_dtype, int velocity_layout,
                                        int precip_dtype, int m, int n, int row_begin, int row_count,
                                        void *out, double *disp_out, void *stream) {
    if (int rc = check_band(m, n, row_begin, row_count, velocity_layout, velocity != nullptr, "velocity is NULL",
                            tdiff, T, n_iter, mode))
        return rc;
    B200_REQUIRE((precip == nullptr) == (out == nullptr), "precip and out must both be given or both NULL");
    B200_REQUIRE(precip != nullptr || disp_out != nullptr, "nothing to compute");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(velocity_dtype, precip_dtype, [&](auto fv, auto fp) {
        using FV = typename decltype(fv)::type;
        using F = typename decltype(fp)::type;
        const size_t N = (size_t)m * n;  // full frame (inputs)
        b200::Scratch vi, pw;
        // widen the fields to float64 once (exact), so the trajectory loop issues no conversions
        const double2 *Vi;
        if (int rc = velocity_pairs<double2, FV>(velocity, velocity_layout, N, vi, Vi, s)) return rc;
        const void *p_ptr = precip;
        if (precip && sizeof(F) == 4) {
            B200_CUDA(pw.alloc(N * sizeof(double), s));
            p_ptr = pw.p;
            widen_field_kernel<<<stream_blocks(N, 16), 256, 0, s>>>((const float *)precip, (double *)pw.p, N);
            B200_LAUNCH_CHECK();
        }
        const SLParams p = sl_params(Vi, p_ptr, xy_coords, disp_prev, m, n, row_begin, row_count, n_iter, mode,
                                     outval, vel_timestep, tdiff[0]);
        return sl_launches<F, sizeof(FV) == 4>(p, tdiff, T, SL_MAX_T, out, disp_out, nullptr, s);
    });
}

// Opt-in float32-tap variant of b200_sl_extrapolate_rows (see sl_f32_kernel): n_iter = 1, pixel-grid
// coordinates, a precipitation field, at most 32 timesteps.  Tap indices are certified equal to the
// exact kernel's (uncertified pixels are recomputed by the exact code); values carry float32 rounding.
// `fallback_count` (device, optional, NOT reset here) receives the number of recomputed pixels.
extern "C" int b200_sl_extrapolate_rows_f32(const void *precip, const void *velocity, const double *disp_prev,
                                            const double *tdiff, int T, double vel_timestep, double outval,
                                            int mode, int velocity_dtype, int velocity_layout, int precip_dtype,
                                            int m, int n, int row_begin, int row_count, void *out,
                                            double *disp_out, unsigned long long *fallback_count, void *stream) {
    if (int rc = check_band(m, n, row_begin, row_count, velocity_layout,
                            velocity != nullptr && precip != nullptr && out != nullptr,
                            "precip, velocity and out are required", tdiff, T, 1, mode))
        return rc;
    if (T > SL_MAX_T) {
        b200::set_error("the float32-tap kernel takes at most %d timesteps per call", SL_MAX_T);
        return B200_ENOTSUP;
    }
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(velocity_dtype, precip_dtype, [&](auto fv, auto fp) {
        using FV = typename decltype(fv)::type;
        using F = typename decltype(fp)::type;
        constexpr bool VF32 = sizeof(FV) == 4;
        const size_t N = (size_t)m * n, NB = (size_t)row_count * n;
        b200::Scratch vi, vf, lst;
        const double2 *Vi;  // exact float64 pairs, for the pixels that fall back
        if (int rc = velocity_pairs<double2, FV>(velocity, velocity_layout, N, vi, Vi, s)) return rc;
        const float2 *Vf;
        if (int rc = velocity_pairs<float2, FV>(velocity, velocity_layout, N, vf, Vf, s)) return rc;
        // the precipitation in its input type: sl_pixel<..., PT = F>
        SLParams p = sl_params(Vi, precip, nullptr, disp_prev, m, n, row_begin, row_count, 1, mode, outval,
                               vel_timestep, tdiff[0]);
        p.T = T;
        p.disp_out = disp_out;
        p.out = out;
        SLFastParams q;
        memset(&q, 0, sizeof(q));
        for (int i = 0; i < T; i++) {
            p.scale[i] = tdiff[i] / vel_timestep;
            q.scale[i] = (float)p.scale[i];
        }
        q.s0 = (float)(tdiff[0] / vel_timestep);
        q.Vf = Vf;
        q.Pf = precip;
        B200_CUDA(lst.alloc(sizeof(int) * (NB + 4), s));
        q.nlist = (unsigned *)lst.p;
        q.list = (int *)lst.p + 4;
        B200_CUDA(cudaMemsetAsync(q.nlist, 0, sizeof(unsigned), s));
        dim3 block(SL_BX, SL_BY);
        dim3 grid(b200::ceil_div(n, SL_BX), b200::ceil_div(row_count, SL_BY));
        sl_f32_kernel<F, VF32><<<grid, block, 0, s>>>(p, q);
        B200_LAUNCH_CHECK();
        sl_f32_fixup_kernel<F, VF32><<<b200::num_sms() * 8, 128, 0, s>>>(p, q.nlist, q.list, fallback_count);
        B200_LAUNCH_CHECK();
        return 0;
    });
}

extern "C" int b200_sl_extrapolate(const void *precip, const void *velocity,
                                   const double *xy_coords, const double *disp_prev,
                                   const double *tdiff, int T, double vel_timestep, int n_iter,
                                   double outval, int mode, int velocity_dtype, int velocity_layout,
                                   int precip_dtype, int m, int n, void *out, double *disp_out,
                                   void *stream) {
    return b200_sl_extrapolate_rows(precip, velocity, xy_coords, disp_prev, tdiff, T, vel_timestep, n_iter,
                                    outval, mode, velocity_dtype, velocity_layout, precip_dtype, m, n, 0, m,
                                    out, disp_out, stream);
}

extern "C" int b200_sl_extrapolate_host(const void *precip, const void *velocity,
                                        const double *xy_coords, const double *disp_prev,
                                        const double *tdiff, int T, double vel_timestep,
                                        int n_iter, double outval, int mode, int velocity_dtype,
                                        int precip_dtype, int m, int n, void *out,
                                        double *disp_out) {
    size_t fs = 0, vs = 0;
    if (int rc = b200::with_dtypes(velocity_dtype, precip_dtype, [&](auto fv, auto fp) {
            vs = sizeof(typename decltype(fv)::type);
            fs = sizeof(typename decltype(fp)::type);
            return 0;
        }))
        return rc;
    B200_REQUIRE(velocity != nullptr && m >= 1 && n >= 1 && T >= 1, "bad arguments");
    const size_t N = (size_t)m * n;
    cudaStream_t s = nullptr;
    b200::Scratch dP, dV, dXY, dDP, dOut, dDO;
    B200_CUDA(dV.alloc(2 * N * vs, s));
    B200_CUDA(cudaMemcpyAsync(dV.p, velocity, 2 * N * vs, cudaMemcpyHostToDevice, s));
    if (precip) {
        B200_CUDA(dP.alloc(N * fs, s));
        B200_CUDA(cudaMemcpyAsync(dP.p, precip, N * fs, cudaMemcpyHostToDevice, s));
        B200_CUDA(dOut.alloc((size_t)T * N * fs, s));
    }
    if (xy_coords) {
        B200_CUDA(dXY.alloc(2 * N * 8, s));
        B200_CUDA(cudaMemcpyAsync(dXY.p, xy_coords, 2 * N * 8, cudaMemcpyHostToDevice, s));
    }
    if (disp_prev) {
        B200_CUDA(dDP.alloc(2 * N * 8, s));
        B200_CUDA(cudaMemcpyAsync(dDP.p, disp_prev, 2 * N * 8, cudaMemcpyHostToDevice, s));
    }
    if (disp_out) B200_CUDA(dDO.alloc(2 * N * 8, s));
    int rc = b200_sl_extrapolate(precip ? dP.p : nullptr, dV.p, xy_coords ? (const double *)dXY.p : nullptr,
                                 disp_prev ? (const double *)dDP.p : nullptr, tdiff, T, vel_timestep,
                                 n_iter, outval, mode, velocity_dtype, B200_LAYOUT_PLANAR, precip_dtype,
                                 m, n, precip ? dOut.p : nullptr,
                                 disp_out ? (double *)dDO.p : nullptr, s);
    if (rc) return rc;
    if (precip && out)
        B200_CUDA(cudaMemcpyAsync(out, dOut.p, (size_t)T * N * fs, cudaMemcpyDeviceToHost, s));
    if (disp_out)
        B200_CUDA(cudaMemcpyAsync(disp_out, dDO.p, 2 * N * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    return 0;
}

extern "C" int b200_sl_interleave_velocity(const void *velocity, int velocity_dtype, int m, int n,
                                           void *out, void *stream) {
    B200_REQUIRE(velocity != nullptr && out != nullptr && m >= 1 && n >= 1, "bad arguments");
    const size_t N = (size_t)m * n;
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("velocity", velocity_dtype, [&](auto fv) {
        using F = typename decltype(fv)::type;
        using F2 = std::conditional_t<sizeof(F) == 4, float2, double2>;
        relayout_kernel<F, F2, false><<<stream_blocks(N, 16), 256, 0, s>>>((const F *)velocity, (F2 *)out, N);
        B200_LAUNCH_CHECK();
        return 0;
    });
}

// BPS motion perturbation (pysteps/noise/motion.py:129-180) at one grid node: out = V + (a*V_par + b*V_perp)/vsf
// with V_par = V/|V| (zero where |V| <= 1e-12), V_perp = (-V_par.y, V_par.x), a = g_par(t)*eps_par,
// b = g_perp(t)*eps_perp; WHAT selects V_par alone (B200_BPS_UNIT) or the perturbation alone
// (B200_BPS_PERTURBATION).  The norm and the division run in the field's own dtype, as NumPy does
// (linalg.norm and V/N keep float32; the result is stored into a float64 array, :138-139).
template <typename F, int WHAT>
static __device__ __forceinline__ double2 bps_point(const F vx, const F vy, double a, double b, double vsf) {
    double nx, ny;
    if (sizeof(F) == 4) {
        const float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn((float)vx, (float)vx), __fmul_rn((float)vy, (float)vy)));
        const bool ok = nrm > (float)1e-12;  // NaN compares false
        nx = ok ? (double)__fdiv_rn((float)vx, nrm) : 0.0;
        ny = ok ? (double)__fdiv_rn((float)vy, nrm) : 0.0;
    } else {
        const double nrm = __dsqrt_rn(__dadd_rn(__dmul_rn((double)vx, (double)vx), __dmul_rn((double)vy, (double)vy)));
        const bool ok = nrm > 1e-12;
        nx = ok ? __ddiv_rn((double)vx, nrm) : 0.0;
        ny = ok ? __ddiv_rn((double)vy, nrm) : 0.0;
    }
    if (WHAT == B200_BPS_UNIT) return make_double2(nx, ny);
    double ox = __ddiv_rn(__dadd_rn(__dmul_rn(a, nx), __dmul_rn(b, -ny)), vsf);
    double oy = __ddiv_rn(__dadd_rn(__dmul_rn(a, ny), __dmul_rn(b, nx)), vsf);
    if (WHAT != B200_BPS_PERTURBATION) {
        ox = __dadd_rn((double)vx, ox);
        oy = __dadd_rn((double)vy, oy);
    }
    return make_double2(ox, oy);
}

// the perturbation applied while the field is re-laid out for the trajectory kernel
template <typename F, int WHAT>
__global__ void __launch_bounds__(256)
bps_perturb_kernel(const F *__restrict__ V, double *__restrict__ out, size_t N, double a, double b,
                   double vsf, double *__restrict__ n_nonfinite) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    int bad = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride) {
        const F vx = __ldg(V + i), vy = __ldg(V + N + i);
        const double2 o = bps_point<F, WHAT>(vx, vy, a, b, vsf);
        bad += !isfinite(o.x);
        bad += !isfinite(o.y);
        if (WHAT == B200_BPS_FIELD_INTERLEAVED) {
            reinterpret_cast<double2 *>(out)[i] = o;
        } else {
            out[i] = o.x;
            out[N + i] = o.y;
        }
    }
    // number of non-finite output elements (the check of semilagrangian.py:116-123 on the
    // perturbed field) -- exact in a double up to 2^53; atomics only in the rare bad case
    if (n_nonfinite != nullptr && __any_sync(0xffffffffu, bad != 0)) {
        if (bad) atomicAdd(n_nonfinite, (double)bad);
    }
}

template <typename F>
static int bps_launch(const void *velocity, size_t N, double a, double b, double vsf, int what, double *out,
                      double *nnf, cudaStream_t s) {
    if (nnf) B200_CUDA(cudaMemsetAsync(nnf, 0, sizeof(double), s));
    const int blocks = stream_blocks(N, 16);
    const F *V = (const F *)velocity;
    switch (what) {
    case B200_BPS_FIELD_INTERLEAVED:
        bps_perturb_kernel<F, B200_BPS_FIELD_INTERLEAVED><<<blocks, 256, 0, s>>>(V, out, N, a, b, vsf, nnf); break;
    case B200_BPS_FIELD_PLANAR:
        bps_perturb_kernel<F, B200_BPS_FIELD_PLANAR><<<blocks, 256, 0, s>>>(V, out, N, a, b, vsf, nnf); break;
    case B200_BPS_PERTURBATION:
        bps_perturb_kernel<F, B200_BPS_PERTURBATION><<<blocks, 256, 0, s>>>(V, out, N, a, b, vsf, nnf); break;
    case B200_BPS_UNIT:
        bps_perturb_kernel<F, B200_BPS_UNIT><<<blocks, 256, 0, s>>>(V, out, N, a, b, vsf, nnf); break;
    default:
        b200::set_error("unknown BPS output selector %d", what);
        return B200_EINVAL;
    }
    B200_LAUNCH_CHECK();
    return 0;
}

// ---- all members of a GPU in one launch per lead time ---------------------------------------
// nowcasts/utils.py:440-458 advances every ensemble member by one single-step extrapolator call
// per lead time: its own perturbed motion field, its own precipitation field, its own carried
// displacement.  The per-member calls cost ~80 us of host time each on top of ~170 us of kernels;
// here the members of a rank go through ONE perturbation launch and ONE trajectory launch
// (grid.y / grid.z = member), SL_BATCH members at a time (that bounds the scratch for the
// perturbed fields to SL_BATCH x 64 MB at 2048^2).
constexpr int SL_BATCH = 8;
struct BpsBatch { double a[SL_BATCH], b[SL_BATCH]; };

template <typename F>
__global__ void __launch_bounds__(256)
bps_perturb_batched_kernel(const F *__restrict__ V, double2 *__restrict__ out, size_t N, const BpsBatch ab,
                           double vsf, double *__restrict__ n_nonfinite) {
    const int mem = blockIdx.y;
    const double a = ab.a[mem], b = ab.b[mem];
    double2 *__restrict__ o = out + (size_t)mem * N;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    int bad = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += stride) {
        const F vx = __ldg(V + i), vy = __ldg(V + N + i);
        const double2 v = bps_point<F, B200_BPS_FIELD_INTERLEAVED>(vx, vy, a, b, vsf);
        bad += !isfinite(v.x);
        bad += !isfinite(v.y);
        o[i] = v;
    }
    if (n_nonfinite != nullptr && __any_sync(0xffffffffu, bad != 0)) {
        if (bad) atomicAdd(n_nonfinite + mem, (double)bad);
    }
}

extern "C" int b200_sl_step_batched(const void *velocity, int velocity_dtype, int m, int n, int members,
                                    const double *pert_coefs, double vsf, const void *precip, int precip_dtype,
                                    const double *disp_prev, double tdiff, double vel_timestep, double outval,
                                    int mode, void *out, double *disp_out, double *n_nonfinite, void *stream) {
    B200_REQUIRE(velocity && pert_coefs && precip && out && disp_out, "bad arguments");
    B200_REQUIRE(m >= 1 && n >= 1 && (int64_t)m * n < ((int64_t)1 << 30) && members >= 1, "bad sizes");
    B200_REQUIRE(mode == B200_MODE_CONSTANT || mode == B200_MODE_NEAREST, "unsupported mode");
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtypes(velocity_dtype, precip_dtype, [&](auto fv, auto fp) {
        using FV = typename decltype(fv)::type;
        using F = typename decltype(fp)::type;
        const size_t N = (size_t)m * n;
        const int ch_max = std::min(members, SL_BATCH);
        b200::Scratch vp, pw;
        B200_CUDA(vp.alloc((size_t)ch_max * N * sizeof(double2), s));
        if (sizeof(F) == 4) B200_CUDA(pw.alloc((size_t)ch_max * N * sizeof(double), s));
        if (n_nonfinite) B200_CUDA(cudaMemsetAsync(n_nonfinite, 0, sizeof(double) * members, s));
        const int sblocks = stream_blocks(N, 8);
        for (int m0 = 0; m0 < members; m0 += SL_BATCH) {
            const int ch = std::min(SL_BATCH, members - m0);
            BpsBatch ab;
            for (int j = 0; j < SL_BATCH; j++) {
                ab.a[j] = j < ch ? pert_coefs[2 * (m0 + j)] : 0.0;
                ab.b[j] = j < ch ? pert_coefs[2 * (m0 + j) + 1] : 0.0;
            }
            bps_perturb_batched_kernel<FV><<<dim3(sblocks, ch), 256, 0, s>>>(
                (const FV *)velocity, (double2 *)vp.p, N, ab, vsf, n_nonfinite ? n_nonfinite + m0 : nullptr);
            B200_LAUNCH_CHECK();
            const void *p_ptr = (const F *)precip + (size_t)m0 * N;
            if (sizeof(F) == 4) {
                widen_field_kernel<<<stream_blocks((size_t)ch * N, 16), 256, 0, s>>>((const float *)p_ptr,
                                                                                     (double *)pw.p, (size_t)ch * N);
                B200_LAUNCH_CHECK();
                p_ptr = pw.p;
            }
            const double *d_prev = disp_prev ? disp_prev + (size_t)m0 * 2 * N : nullptr;
            SLParams p = sl_params((const double2 *)vp.p, p_ptr, nullptr, d_prev, m, n, 0, m, 1, mode, outval,
                                   vel_timestep, tdiff);
            p.T = 1;
            p.scale[0] = tdiff / vel_timestep;
            p.disp_out = disp_out + (size_t)m0 * 2 * N;
            p.out = (F *)out + (size_t)m0 * N;
            p.zs_vi = N; p.zs_precip = N; p.zs_disp = 2 * N; p.zs_out = N;
            dim3 block(SL_BX, SL_BY);
            dim3 grid(b200::ceil_div(n, SL_BX), b200::ceil_div(m, SL_BY), ch);
            // VF32 = false: the perturbed field is float64 (noise/motion.py:138-139)
            sl_multistep_kernel<F, true, false, true><<<grid, block, 0, s>>>(p);
            B200_LAUNCH_CHECK();
        }
        return 0;
    });
}

extern "C" int b200_bps_perturb_velocity(const void *velocity, int velocity_dtype, int m, int n,
                                         double a_par, double a_perp, double vsf, int what,
                                         double *out, double *n_nonfinite, void *stream) {
    B200_REQUIRE(velocity != nullptr && out != nullptr && m >= 1 && n >= 1, "bad arguments");
    const size_t N = (size_t)m * n;
    cudaStream_t s = (cudaStream_t)stream;
    return b200::with_dtype("velocity", velocity_dtype, [&](auto fv) {
        return bps_launch<typename decltype(fv)::type>(velocity, N, a_par, a_perp, vsf, what, out, n_nonfinite, s);
    });
}
