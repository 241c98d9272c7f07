// spline.cu -- interp_order 0 and 2..5 of the semi-Lagrangian extrapolator (sm_90a).
//
// pysteps/extrapolation/semilagrangian.py:144-157,224-253: for interp_order > 1 the field is
// warped with scipy.ndimage.map_coordinates(order, prefilter=True) and two auxiliary order-1
// warps of a "wet" mask and a "finite" mask restore the no-precipitation value and the NaNs.
// scipy's algorithm (restated and pinned bit for bit in oracle/spline_oracle.c):
//   prefilter : per axis (axis 0 first, then axis 1) the gain prod (1-z)(1-1/z), then per pole z
//               causal and anti-causal first-order recursions (order/2 poles, e.g. the double
//               nearest to sqrt(3)-2 for order 3);
//               boundary "mirror" for mode constant; for mode nearest the field is edge-padded
//               by 12 samples and the boundary is "reflect";
//   sampling  : (order+1)^2 taps from floor(c)-order/2 (odd) or floor(c+0.5)-order/2 (even),
//               B-spline weights with the last one as one minus the others, value = sum over taps
//               (rows outer) of ((a*wy)*wx) from 0.0; taps mirrored (constant) or clamped
//               (nearest); order 0 reads the tap floor(c+0.5).
// Every float64 operation is issued in scipy's order, round-to-nearest, no FMA (--fmad=false).
// The recursions are sequential along a line by construction (each line is one chain; lines run
// in parallel, one thread per line with coalesced access across the warp); the row pass runs as
// a column pass on the transposed array.
#include "common.cuh"
#include "spline_body.cuh"

namespace {

using spl::NPAD;
using spl::SampleParams;

template <typename F>
__global__ void __launch_bounds__(256)
spline_prepare_kernel(const F *__restrict__ precip, int m, int n, int pad, const double *__restrict__ stats,
                      int zero_fill, int want_masks, double *__restrict__ f, double *__restrict__ mask_min,
                      double *__restrict__ mask_fin) {
    const size_t total = (size_t)(m + 2 * pad) * (size_t)(n + 2 * pad);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride)
        spl::prepare_element<F>(e, precip, m, n, pad, stats, zero_fill, want_masks, f, mask_min, mask_fin);
}

// one thread per column: the line of L samples has stride ncols, accesses coalesce across the warp
__global__ void __launch_bounds__(128)
spline_filter_columns_kernel(double *__restrict__ a, int L, int ncols, const __grid_constant__ spl::FilterParams fp) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ncols) return;
    spl::filter_line(a + j, L, (size_t)ncols, fp);
}

// (R, C) -> (C, R), 32x32 tiles through shared memory
__global__ void __launch_bounds__(256)
transpose_kernel(const double *__restrict__ in, double *__restrict__ out, int R, int C) {
    __shared__ double tile[32][33];
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
    spl::transpose_load(tile, in, R, C, bx, by, threadIdx.x, threadIdx.y);
    __syncthreads();
    spl::transpose_store(tile, out, R, C, bx, by, threadIdx.x, threadIdx.y);
}

template <typename F> __device__ __forceinline__ F narrow(double v);
template <> __device__ __forceinline__ float narrow<float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double narrow<double>(double v) { return v; }

template <typename F>
__global__ void __launch_bounds__(128)
spline_sample_kernel(const __grid_constant__ SampleParams p) {
    const int x = blockIdx.x * 32 + threadIdx.x;
    const int yl = blockIdx.y * 4 + threadIdx.y;
    const int t = blockIdx.z;
    if (x >= p.n || yl >= p.rows) return;
    const double v = spl::sample_pixel(p, x, yl, t);
    ((F *)p.out)[(size_t)t * p.rows * p.n + (size_t)yl * p.n + x] = narrow<F>(v);
}

}  // namespace

extern "C" int b200_spline_prepare(const void *precip, int precip_dtype, int m, int n, int order, int mode,
                                   const double *stats, int zero_fill, const double *poles,
                                   const double *zpow_axis0, const double *zpow_axis1, double *coeffs,
                                   double *mask_min, double *mask_finite, void *stream) {
    B200_REQUIRE(precip != nullptr && coeffs != nullptr && m >= 1 && n >= 1, "bad arguments");
    B200_REQUIRE(order == 0 || (order >= 2 && order <= 5), "spline order must be 0 or 2..5");
    B200_REQUIRE(order == 0 || (poles && zpow_axis0 && zpow_axis1), "order >= 2 needs the filter poles");
    B200_REQUIRE(mode == B200_MODE_CONSTANT || mode == B200_MODE_NEAREST, "unsupported mode");
    B200_REQUIRE(order == 0 || (stats != nullptr && mask_min != nullptr && mask_finite != nullptr),
                 "order >= 2 needs the field statistics and both mask buffers");
    cudaStream_t s = (cudaStream_t)stream;
    const int pad = (order > 1 && mode == B200_MODE_NEAREST) ? NPAD : 0;
    const int M = m + 2 * pad, N = n + 2 * pad;
    const size_t total = (size_t)M * N;
    const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)b200::num_sms() * 16);
    const int want_masks = order > 1;
    if (int rc = b200::with_dtype("precip", precip_dtype, [&](auto t) {
            using F = typename decltype(t)::type;
            spline_prepare_kernel<F><<<blocks, 256, 0, s>>>((const F *)precip, m, n, pad, stats, zero_fill, want_masks,
                                                             coeffs, mask_min, mask_finite);
            B200_LAUNCH_CHECK();
            return 0;
        }))
        return rc;
    if (order <= 1) return 0;
    spl::FilterParams f0;
    memset(&f0, 0, sizeof(f0));
    f0.npoles = order / 2;
    f0.reflect = mode == B200_MODE_NEAREST;
    f0.gain = 1.0;
    for (int k = 0; k < f0.npoles; k++) {
        f0.z[k] = poles[k];
        f0.gain *= (1.0 - poles[k]) * (1.0 - 1.0 / poles[k]);
    }
    spl::FilterParams f1 = f0;
    for (int k = 0; k < f0.npoles; k++) {
        f0.zpow[k] = zpow_axis0[k];
        f1.zpow[k] = zpow_axis1[k];
    }
    // axis 0: every column is a line of M samples
    spline_filter_columns_kernel<<<b200::ceil_div(N, 128), 128, 0, s>>>(coeffs, M, N, f0);
    B200_LAUNCH_CHECK();
    // axis 1: every row is a line of N samples -> columns of the transposed array
    b200::Scratch tr;
    B200_CUDA(tr.alloc(total * sizeof(double), s));
    dim3 tb(32, 8);
    transpose_kernel<<<dim3(b200::ceil_div(N, 32), b200::ceil_div(M, 32)), tb, 0, s>>>(coeffs, (double *)tr.p, M, N);
    B200_LAUNCH_CHECK();
    spline_filter_columns_kernel<<<b200::ceil_div(M, 128), 128, 0, s>>>((double *)tr.p, N, M, f1);
    B200_LAUNCH_CHECK();
    transpose_kernel<<<dim3(b200::ceil_div(M, 32), b200::ceil_div(N, 32)), tb, 0, s>>>((const double *)tr.p, coeffs, N, M);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_spline_sample(const double *coeffs, int m, int n, int order, int mode, const double *xy_coords,
                                  const double *disp_steps, int T, int row_begin, int row_count, double outval,
                                  const double *mask_min, const double *mask_finite, const double *stats,
                                  int out_dtype, void *out, void *stream) {
    B200_REQUIRE(coeffs != nullptr && disp_steps != nullptr && out != nullptr && m >= 1 && n >= 1 && T >= 1,
                 "bad arguments");
    B200_REQUIRE(T <= 65535, "too many leadtimes for one launch");
    B200_REQUIRE(order == 0 || (order >= 2 && order <= 5), "spline order must be 0 or 2..5");
    B200_REQUIRE(mode == B200_MODE_CONSTANT || mode == B200_MODE_NEAREST, "unsupported mode");
    B200_REQUIRE(row_begin >= 0 && row_count >= 1 && row_begin + row_count <= m, "row band out of range");
    B200_REQUIRE(order == 0 || (mask_min && mask_finite && stats), "order >= 2 needs masks and statistics");
    SampleParams p;
    memset(&p, 0, sizeof(p));
    p.coeffs = coeffs; p.xy = xy_coords; p.disp = disp_steps;
    p.mask_min = mask_min; p.mask_fin = mask_finite; p.stats = stats;
    p.out = out;
    p.m = m; p.n = n; p.order = order; p.mode = mode; p.T = T;
    p.pad = (order > 1 && mode == B200_MODE_NEAREST) ? NPAD : 0;
    p.row0 = row_begin; p.rows = row_count;
    p.cval = outval;
    dim3 block(32, 4), grid(b200::ceil_div(n, 32), b200::ceil_div(row_count, 4), T);
    return b200::with_dtype("output", out_dtype, [&](auto t) {
        spline_sample_kernel<typename decltype(t)::type><<<grid, block, 0, (cudaStream_t)stream>>>(p);
        B200_LAUNCH_CHECK();
        return 0;
    });
}
