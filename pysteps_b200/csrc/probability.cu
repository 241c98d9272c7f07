// probability.cu -- the neighbourhood step of the local Lagrangian probability nowcast
// (pysteps/nowcasts/lagrangian_probability.py) on the device (sm_90a).  Per lead time, two kernels
// over one (m, n + 1) scratch plane that every lead reuses:
//   prefix  one CTA per row: the exclusive row prefix sums of (exceeds, valid) of the extrapolated
//           field, packed in one 64-bit word (exceedances in the low half, valid pixels in the high
//           half: both halves stay below 2^31, so packed sums and differences never carry)
//   ratio   one thread per pixel: the exact disk counts from two prefix lookups per kernel row that
//           overlaps the frame, then count / valid in float64, clipped to [0, 1]; NaN at NaN pixels
// The sums are integers in a fixed order, so the result is the exact one, the same on every call.
#include "common.cuh"
#include "scan.cuh"

namespace {

constexpr int PREFIX_THREADS = 256, PREFIX_PER_THREAD = 4, PREFIX_TILE = PREFIX_THREADS * PREFIX_PER_THREAD;
constexpr int RATIO_X = 32, RATIO_Y = 8;
constexpr unsigned long long VALID_ONE = 1ull << 32;

// NaN pixels hold `threshold - 1` in the reference and exceed when that value does (nan_word); every
// other pixel is valid and exceeds when (double)v >= threshold, the comparison NumPy makes in the
// field's dtype (a float32 threshold widens exactly)
template <typename F>
__device__ __forceinline__ unsigned long long pixel_word(F v, double threshold, unsigned long long nan_word) {
    const double d = (double)v;
    if (isnan(d)) return nan_word;
    return VALID_ONE | (d >= threshold ? 1ull : 0ull);
}

template <typename F>
__global__ void __launch_bounds__(PREFIX_THREADS)
    prefix_kernel(const F *__restrict__ plane, int n, double threshold, unsigned long long nan_word,
                  unsigned long long *__restrict__ prefix) {
    __shared__ unsigned long long sh[PREFIX_THREADS / 32];
    const F *row = plane + (int64_t)blockIdx.x * n;
    unsigned long long *out = prefix + (int64_t)blockIdx.x * (n + 1);
    unsigned long long carry = 0ull;
    for (int base = 0; base < n; base += PREFIX_TILE) {
        const int x0 = base + threadIdx.x * PREFIX_PER_THREAD;
        unsigned long long w[PREFIX_PER_THREAD], sum = 0ull;
#pragma unroll
        for (int k = 0; k < PREFIX_PER_THREAD; k++) {
            w[k] = x0 + k < n ? pixel_word(row[x0 + k], threshold, nan_word) : 0ull;
            sum += w[k];
        }
        unsigned long long total;
        unsigned long long run = carry + b200::block_exclusive_scan<PREFIX_THREADS>(sum, sh, &total);
#pragma unroll
        for (int k = 0; k < PREFIX_PER_THREAD; k++) {
            if (x0 + k < n) out[x0 + k] = run;
            run += w[k];
        }
        carry += total;
    }
    if (threadIdx.x == 0) out[n] = carry;
}

struct Lead {
    int s;            // kernel diameter int(t * slope); 0: the plane stays binary
    int c;            // (s - 1) // 2, the centre scipy's mode="same" keeps
    const int *runs;  // s pairs (b0, b1): kernel row a covers columns b0..b1
};

// count(y, x) = sum over kernel rows a of the pixels (y + c - a, x + c - b), b0(a) <= b <= b1(a),
// inside the frame: per row one difference of two prefix words
__global__ void __launch_bounds__(RATIO_X *RATIO_Y)
    ratio_kernel(const unsigned long long *__restrict__ prefix, int m, int n, int tiles_x, const Lead lead,
                 double *__restrict__ out) {
    const int x = (int)(blockIdx.x % tiles_x) * RATIO_X + threadIdx.x;
    const int y = (int)(blockIdx.x / tiles_x) * RATIO_Y + threadIdx.y;
    if (x >= n || y >= m) return;
    const int64_t stride = (int64_t)n + 1;
    const unsigned long long *own = prefix + y * stride;
    const unsigned long long self = own[x + 1] - own[x];
    double r;
    if (!(self >> 32)) {
        r = __longlong_as_double(0x7ff8000000000000ll);  // NaN pixel
    } else if (lead.s == 0) {
        r = (double)(self & 1ull);
    } else {
        // rows a with 0 <= y + c - a < m
        const int a0 = max(0, y + lead.c - (m - 1)), a1 = min(lead.s - 1, y + lead.c);
        const int xc = x + lead.c;
        unsigned long long acc = 0ull;
        const unsigned long long *row = prefix + (int64_t)(y + lead.c - a0) * stride;
#pragma unroll 4
        for (int a = a0; a <= a1; a++, row -= stride) {
            const int2 run = __ldg(reinterpret_cast<const int2 *>(lead.runs) + a);
            const int lo = max(0, xc - run.y), hi = min(n - 1, xc - run.x);
            if (lo <= hi) acc += __ldg(row + hi + 1) - __ldg(row + lo);
        }
        const double e = (double)(unsigned)(acc & 0xffffffffull), v = (double)(unsigned)(acc >> 32);
        r = fmin(e / v, 1.0);  // v >= 1: the pixel is in its own neighbourhood
    }
    out[(int64_t)y * n + x] = r;
}

template <typename F>
int run(const F *field, int64_t plane_stride, int T, int m, int n, double threshold, int nan_exceeds,
        const int *scales, const int *runs, unsigned long long *scratch, double *out, cudaStream_t st) {
    const unsigned long long nan_word = nan_exceeds ? 1ull : 0ull;
    const int tiles_x = b200::ceil_div(n, RATIO_X);
    const unsigned tiles = (unsigned)(tiles_x * b200::ceil_div64(m, RATIO_Y));
    int64_t run_off = 0;
    for (int t = 0; t < T; t++) {
        prefix_kernel<F><<<m, PREFIX_THREADS, 0, st>>>(field + t * plane_stride, n, threshold, nan_word, scratch);
        B200_LAUNCH_CHECK();
        const Lead lead{scales[t], (scales[t] - 1) / 2, runs + 2 * run_off};
        ratio_kernel<<<tiles, dim3(RATIO_X, RATIO_Y), 0, st>>>(scratch, m, n, tiles_x, lead, out + (int64_t)t * m * n);
        B200_LAUNCH_CHECK();
        run_off += scales[t];
    }
    return 0;
}

}  // namespace

extern "C" int b200_probability(const void *field, int dtype, int64_t plane_stride, int T, int m, int n,
                                double threshold, int nan_exceeds, const int *scales, const int *runs,
                                unsigned long long *scratch, double *out, void *stream) {
    B200_REQUIRE(T >= 0 && m >= 0 && n >= 0 && plane_stride >= 0 && scales != nullptr, "bad arguments");
    B200_REQUIRE((int64_t)m * n < ((int64_t)1 << 31), "probability: frames of 2^31 pixels or more are not supported");
    return b200::with_dtype("field", dtype, [&](auto tf) {
        using F = typename decltype(tf)::type;
        if (T == 0 || (int64_t)m * n == 0) return 0;
        B200_REQUIRE(field != nullptr && scratch != nullptr && out != nullptr, "bad arguments");
        for (int t = 0; t < T; t++) {
            B200_REQUIRE(scales[t] >= 0 && scales[t] <= B200_PROBABILITY_MAX_SCALE,
                         "probability: kernel diameters must lie in 0 .. B200_PROBABILITY_MAX_SCALE");
            B200_REQUIRE((int64_t)(m > n ? m : n) + scales[t] < ((int64_t)1 << 31), "probability: index range");
            B200_REQUIRE(scales[t] == 0 || runs != nullptr, "bad arguments");
        }
        return run<F>((const F *)field, plane_stride, T, m, n, threshold, nan_exceeds, scales, runs, scratch, out,
                      (cudaStream_t)stream);
    });
}
