// proesmans.cu -- the Proesmans et al. (1994) anisotropic-diffusion optical flow (sm_90a).
//
// Replaces the native extension of the reference, pysteps/motion/_proesmans.pyx
// (_compute_advection_field, :19-44): an image pyramid, and per level num_iter iterations of
//   (a) forward-backward consistency maps of the two flow fields (a map + a mean, :190-254),
//   (b) one relaxation sweep per flow field (:81-164).
// (b) is a raster-order GAUSS-SEIDEL sweep -- every pixel reads the west and north neighbours
// already updated in the same sweep -- so it cannot be a plain data-parallel kernel.  Pixels with
// equal t = x + 2y are independent and depend only on smaller t (proesmans_body.cuh), hence a
// sweep is (w-2) + 2(h-2) wavefronts.  One CTA of 1024 threads runs all wavefronts of one flow
// field with a block barrier between them (the two fields' sweeps are independent: two CTAs); the
// work per wavefront is at most min(h, w/2) pixels, so the sweep is barrier/latency bound, not
// throughput bound: ~6 k barriers per sweep at 2048^2 instead of 4 M sequential pixel updates.
// The per-pixel arithmetic is the reference's, operation by operation (the reference itself is
// built with -ffast-math, so parity is to a tolerance; the update ORDER is exact).
#include "common.cuh"
#include "proesmans_body.cuh"

namespace {

constexpr int SWEEP_THREADS = 1024;

template <typename F>
__global__ void __launch_bounds__(256)
scale_kernel(const F *__restrict__ in, double *__restrict__ out, size_t count, double lo, double hi, int do_scale) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < count; e += stride)
        out[e] = pro::scale_value((double)in[e], lo, hi, do_scale);
}

// one axis of the Gaussian pre-filter: axis 0 filters columns, axis 1 rows
__global__ void __launch_bounds__(256)
gauss_axis_kernel(const double *__restrict__ in, double *__restrict__ out, int h, int w, int axis,
                  const __grid_constant__ pro::GaussKernel k) {
    const size_t total = (size_t)h * w, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int y = (int)(e / w), x = (int)(e % w);
        out[e] = axis == 0 ? pro::gauss_line_value(in + x, h, (size_t)w, y, k)
                           : pro::gauss_line_value(in + (size_t)y * w, w, 1, x, k);
    }
}

__global__ void __launch_bounds__(256)
pyr_kernel(const double *__restrict__ src, int sw, double *__restrict__ dst, int dh, int dw) {
    const size_t total = (size_t)dh * dw, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride)
        dst[e] = pro::pyr_pixel(src, sw, (int)(e / dw), (int)(e % dw));
}

// G (2,2,h,w): gradients of both images
__global__ void __launch_bounds__(256)
grad_kernel(const double *__restrict__ R, int h, int w, double *__restrict__ G) {
    const size_t N = (size_t)h * w, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < 2 * N; e += stride) {
        const int img = (int)(e / N);
        const size_t q = e % N;
        double gx, gy;
        pro::grad_pixel(R + (size_t)img * N, h, w, (int)(q / w), (int)(q % w), gx, gy);
        G[(size_t)(2 * img) * N + q] = gx;
        G[(size_t)(2 * img + 1) * N + q] = gy;
    }
}

// inconsistency maps of both directions (2,h,w)
__global__ void __launch_bounds__(256)
cons_map_kernel(const double *__restrict__ V, int h, int w, double *__restrict__ gamma) {
    const size_t N = (size_t)h * w, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < 2 * N; e += stride) {
        const size_t q = e % N;
        gamma[e] = pro::cons_pixel(V, h, w, (int)(e / N), (int)(q / w), (int)(q % w));
    }
}

// one thread per (direction, row): sum and count of the row's valid pixels, a fixed sequential chain
__global__ void __launch_bounds__(128)
cons_rows_kernel(const double *__restrict__ gamma, int h, int w, double *__restrict__ row_sum,
                 long long *__restrict__ row_cnt) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= 2 * h) return;
    double s;
    long long c;
    pro::cons_row_sum(gamma + (size_t)r * w, w, s, c);
    row_sum[r] = s;
    row_cnt[r] = c;
}

// K[i] = 0.9 * c_sum / c_count (:229-233), row results added in row order
__global__ void cons_final_kernel(const double *__restrict__ row_sum, const long long *__restrict__ row_cnt, int h,
                                  double *__restrict__ K) {
    const int i = threadIdx.x;
    if (i < 2) K[i] = pro::cons_K(row_sum + (size_t)i * h, row_cnt + (size_t)i * h, h);
}

__global__ void __launch_bounds__(256)
cons_weight_kernel(double *__restrict__ gamma, size_t N, const double *__restrict__ K) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < 2 * N; e += stride)
        gamma[e] = pro::cons_weight(gamma[e], K[e / N]);
}

// Gauss-Seidel sweep of flow field j = blockIdx.x, all wavefronts, then the border fill.
// V is read and written by the same CTA between barriers: plain pointers, no read-only path.
__global__ void __launch_bounds__(SWEEP_THREADS)
sweep_kernel(const double *__restrict__ R, const double *__restrict__ G, const double *__restrict__ gamma,
             double *V, int h, int w, double lam) {
    const int j = blockIdx.x;
    const size_t N = (size_t)h * w;
    const double *R1 = R + (size_t)j * N, *R2 = R + (size_t)(1 - j) * N;
    const double *G1 = G + (size_t)(2 * j) * N, *G2 = G + (size_t)(2 * j + 1) * N;
    const double *gam = gamma + (size_t)j * N;
    double *Vj = V + (size_t)(2 * j) * N;
    if (h < 3 || w < 3) return;  // no interior pixel: the field of such a level is identically zero
    const int t_last = pro::sweep_last_t(h, w);
    for (int t = pro::sweep_first_t(); t <= t_last; t++) {
        int ylo, yhi;
        pro::sweep_rows_of(t, h, w, ylo, yhi);
        for (int y = ylo + (int)threadIdx.x; y <= yhi; y += SWEEP_THREADS)
            pro::sweep_pixel(R1, R2, G1, G2, gam, Vj, h, w, t - 2 * y, y, lam);
        __syncthreads();
    }
    const int ne = pro::fill_edge_count(h, w);
    for (int c = 0; c < 2; c++)
        for (int e = threadIdx.x; e < ne; e += SWEEP_THREADS) pro::fill_edge_element(Vj + (size_t)c * N, h, w, e);
}

// Vn (4, hn, wn) from Vp (4, hp, wp)
__global__ void __launch_bounds__(256)
next_level_kernel(const double *__restrict__ Vp, int hp, int wp, double *__restrict__ Vn, int hn, int wn) {
    const size_t Nn = (size_t)hn * wn, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < 4 * Nn; e += stride) {
        const int c = (int)(e / Nn);
        const size_t q = e % Nn;
        Vn[e] = pro::next_level_pixel(Vp + (size_t)c * hp * wp, hp, wp, (int)(q / wn), (int)(q % wn));
    }
}

int grid_for(size_t count) {
    return (int)std::max<size_t>(1, std::min<size_t>((count + 255) / 256, (size_t)b200::num_sms() * 8));
}

// :190-254 on the device: gamma (2,h,w) from V (2,2,h,w)
int consistency(const double *V, int h, int w, double *gamma, double *row_sum, long long *row_cnt, double *K,
                cudaStream_t s) {
    const size_t N = (size_t)h * w;
    cons_map_kernel<<<grid_for(2 * N), 256, 0, s>>>(V, h, w, gamma);
    B200_LAUNCH_CHECK();
    cons_rows_kernel<<<b200::ceil_div(2 * h, 128), 128, 0, s>>>(gamma, h, w, row_sum, row_cnt);
    B200_LAUNCH_CHECK();
    cons_final_kernel<<<1, 32, 0, s>>>(row_sum, row_cnt, h, K);
    B200_LAUNCH_CHECK();
    cons_weight_kernel<<<grid_for(2 * N), 256, 0, s>>>(gamma, N, K);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int b200_proesmans_scale(const void *frames, int dtype, int64_t count, double im_min, double im_max,
                                    int do_scale, double *out, void *stream) {
    B200_REQUIRE(frames != nullptr && out != nullptr && count >= 1, "bad arguments");
    return b200::with_dtype("frame", dtype, [&](auto t) {
        using F = typename decltype(t)::type;
        scale_kernel<F><<<grid_for((size_t)count), 256, 0, (cudaStream_t)stream>>>((const F *)frames, out, (size_t)count,
                                                                                    im_min, im_max, do_scale);
        B200_LAUNCH_CHECK();
        return 0;
    });
}

extern "C" int b200_gaussian_filter(const double *in, int h, int w, const double *weights, int radius, double *out,
                                    void *stream) {
    B200_REQUIRE(in != nullptr && out != nullptr && weights != nullptr && h >= 1 && w >= 1, "bad arguments");
    B200_REQUIRE(radius >= 0 && radius <= pro::GAUSS_MAX_RADIUS, "kernel radius must be 0..64 (sigma <= 16)");
    cudaStream_t s = (cudaStream_t)stream;
    pro::GaussKernel k;
    memset(&k, 0, sizeof(k));
    k.lw = radius;
    for (int i = 0; i < 2 * radius + 1; i++) k.w[i] = weights[i];
    b200::Scratch tmp;
    const size_t N = (size_t)h * w;
    B200_CUDA(tmp.alloc(N * sizeof(double), s));
    gauss_axis_kernel<<<grid_for(N), 256, 0, s>>>(in, (double *)tmp.p, h, w, 0, k);
    B200_LAUNCH_CHECK();
    gauss_axis_kernel<<<grid_for(N), 256, 0, s>>>((const double *)tmp.p, out, h, w, 1, k);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200_proesmans_field(const double *frames, int m, int n, double lam, int num_iter, int num_levels,
                                    double *advfield, double *quality, void *stream) {
    B200_REQUIRE(frames != nullptr && advfield != nullptr && quality != nullptr, "NULL argument");
    B200_REQUIRE(m >= 1 && n >= 1 && (int64_t)m * n < ((int64_t)1 << 30), "grid must have 1 .. 2^30 pixels");
    B200_REQUIRE(num_levels >= 1 && num_levels <= 16 && num_iter >= 0, "bad num_levels / num_iter");
    cudaStream_t s = (cudaStream_t)stream;
    // level geometry (:60-76): sizes halve with int(m / 2)
    int hs[16], ws[16];
    size_t off[17];
    hs[0] = m; ws[0] = n; off[0] = 0;
    for (int l = 1; l < num_levels; l++) {
        hs[l] = hs[l - 1] / 2;
        ws[l] = ws[l - 1] / 2;
    }
    B200_REQUIRE(hs[num_levels - 1] >= 1 && ws[num_levels - 1] >= 1, "the coarsest pyramid level is empty");
    for (int l = 0; l < num_levels; l++) off[l + 1] = off[l] + (size_t)hs[l] * ws[l];
    const size_t N0 = (size_t)m * n, P = off[num_levels];
    b200::Scratch pyr, grad, gam, va, vb, psum, pcnt, kbuf;
    B200_CUDA(pyr.alloc(2 * P * sizeof(double), s));       // image 0 levels, then image 1 levels
    B200_CUDA(grad.alloc(4 * N0 * sizeof(double), s));
    B200_CUDA(gam.alloc(2 * N0 * sizeof(double), s));
    B200_CUDA(va.alloc(4 * N0 * sizeof(double), s));
    B200_CUDA(vb.alloc(4 * N0 * sizeof(double), s));
    B200_CUDA(psum.alloc(2 * (size_t)m * sizeof(double), s));       // per-row sums / counts
    B200_CUDA(pcnt.alloc(2 * (size_t)m * sizeof(long long), s));
    B200_CUDA(kbuf.alloc(2 * sizeof(double), s));
    double *pyr0 = (double *)pyr.p, *pyr1 = pyr0 + P;
    B200_CUDA(cudaMemcpyAsync(pyr0, frames, N0 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    B200_CUDA(cudaMemcpyAsync(pyr1, frames + N0, N0 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    for (int l = 1; l < num_levels; l++)
        for (int img = 0; img < 2; img++) {
            double *base = img ? pyr1 : pyr0;
            pyr_kernel<<<grid_for((size_t)hs[l] * ws[l]), 256, 0, s>>>(base + off[l - 1], ws[l - 1], base + off[l],
                                                                       hs[l], ws[l]);
            B200_LAUNCH_CHECK();
        }
    double *Vc = (double *)va.p, *Vn = (double *)vb.p;
    b200::Scratch rl;  // the two images of a level, contiguous (2,h,w)
    B200_CUDA(rl.alloc(2 * N0 * sizeof(double), s));
    const int hc = hs[num_levels - 1], wc = ws[num_levels - 1];
    B200_CUDA(cudaMemsetAsync(Vc, 0, 4 * (size_t)hc * wc * sizeof(double), s));
    for (int l = num_levels - 1; l >= 0; l--) {
        const int h = hs[l], w = ws[l];
        const size_t N = (size_t)h * w;
        double *R = (double *)rl.p;
        B200_CUDA(cudaMemcpyAsync(R, pyr0 + off[l], N * sizeof(double), cudaMemcpyDeviceToDevice, s));
        B200_CUDA(cudaMemcpyAsync(R + N, pyr1 + off[l], N * sizeof(double), cudaMemcpyDeviceToDevice, s));
        grad_kernel<<<grid_for(2 * N), 256, 0, s>>>(R, h, w, (double *)grad.p);
        B200_LAUNCH_CHECK();
        for (int it = 0; it < num_iter; it++) {
            int rc = consistency(Vc, h, w, (double *)gam.p, (double *)psum.p, (long long *)pcnt.p, (double *)kbuf.p, s);
            if (rc) return rc;
            sweep_kernel<<<2, SWEEP_THREADS, 0, s>>>(R, (const double *)grad.p, (const double *)gam.p, Vc, h, w, lam);
            B200_LAUNCH_CHECK();
        }
        if (l > 0) {
            next_level_kernel<<<grid_for(4 * (size_t)hs[l - 1] * ws[l - 1]), 256, 0, s>>>(Vc, h, w, Vn, hs[l - 1],
                                                                                         ws[l - 1]);
            B200_LAUNCH_CHECK();
            std::swap(Vc, Vn);
        }
    }
    // :43 the consistency maps of the final fields, and the fields themselves
    int rc = consistency(Vc, m, n, quality, (double *)psum.p, (long long *)pcnt.p, (double *)kbuf.p, s);
    if (rc) return rc;
    B200_CUDA(cudaMemcpyAsync(advfield, Vc, 4 * N0 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    return 0;
}
