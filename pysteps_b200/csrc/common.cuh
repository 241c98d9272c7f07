// common.cuh -- shared helpers for libpysteps_b200.so (sm_90a only): error reporting, scratch
// allocation and carving, and small device helpers that restate NumPy and OpenCV conventions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/pysteps_b200.h"

namespace b200 {

void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);
int num_sms();
void count_launch();

#define B200_CUDA(call)                                                    \
    do {                                                                   \
        cudaError_t _e = (call);                                           \
        if (_e != cudaSuccess)                                             \
            return ::b200::cuda_fail(_e, #call, __FILE__, __LINE__);       \
    } while (0)

#define B200_LAUNCH_CHECK()                                                \
    do {                                                                   \
        cudaError_t _e = cudaGetLastError();                               \
        ::b200::count_launch();                                            \
        if (_e != cudaSuccess)                                             \
            return ::b200::cuda_fail(_e, "kernel launch", __FILE__, __LINE__); \
    } while (0)

#define B200_REQUIRE(cond, msg)                                            \
    do {                                                                   \
        if (!(cond)) {                                                     \
            ::b200::set_error("%s (%s:%d)", msg, __FILE__, __LINE__);      \
            return B200_EINVAL;                                            \
        }                                                                  \
    } while (0)

template <typename T> struct Type { using type = T; };

// f(Type<float>{}) or f(Type<double>{}) for a dtype code; any other code is refused, named as the dtype of `what`
template <typename Fn>
int with_dtype(const char *what, int dtype, Fn &&f) {
    if (dtype == B200_F32) return f(Type<float>{});
    if (dtype == B200_F64) return f(Type<double>{});
    set_error("unknown %s dtype %d", what, dtype);
    return B200_EINVAL;
}

// f(Type<A>{}, Type<B>{}) for the dtype codes of two fields, refused before f runs when either code is unknown
template <typename Fn>
int with_dtypes(int a, int b, Fn &&f) {
    if ((a != B200_F32 && a != B200_F64) || (b != B200_F32 && b != B200_F64)) {
        set_error("unknown field dtypes %d / %d", a, b);
        return B200_EINVAL;
    }
    return with_dtype("field", a, [&](auto ta) { return with_dtype("field", b, [&](auto tb) { return f(ta, tb); }); });
}

// stream-ordered scratch allocation that is released on scope exit
struct Scratch {
    void *p = nullptr;
    cudaStream_t s = nullptr;
    cudaError_t alloc(size_t bytes, cudaStream_t stream) {
        s = stream;
        return cudaMallocAsync(&p, bytes ? bytes : 1, stream);
    }
    ~Scratch() {
        if (p) cudaFreeAsync(p, s);
    }
};

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

// consecutive 256-byte aligned pieces of one scratch allocation; base == nullptr only sizes them
struct Carver {
    char *base;
    int64_t off = 0;
    void *take(int64_t bytes) {
        char *p = base ? base + off : nullptr;
        off += align256(bytes);
        return p;
    }
};

__device__ __forceinline__ double quiet_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

// the dtype NumPy computes a difference of an F and an O in
template <typename F, typename O> struct Promote { using T = double; };
template <> struct Promote<float, float> { using T = float; };

// OpenCV's BORDER_REFLECT_101: the index of i reflected into [0, L) without repeating the edge
__device__ __forceinline__ int reflect101(int i, int L) {
    if (L == 1) return 0;
    while (i < 0 || i >= L) {
        if (i < 0) i = -i;
        if (i >= L) i = 2 * L - 2 - i;
    }
    return i;
}

}  // namespace b200
