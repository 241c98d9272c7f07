// pairwise_body.cuh -- NumPy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src,
// pairwise_sum) as host/device source, shared between csrc/verification.cu and the host build of
// tests/test_pairwise_body.py, so that the CPU suite pins it against np.sum bit for bit.
//
// np.sum of a contiguous 1-D array, and np.sum(A, axis=1) of every row of a C-contiguous 2-D
// array, is 0 + pw(a, n) in the array's dtype, where
//   pw(a, n) = a[0] + ... + a[n-1] left to right               for n < 8
//            = eight strided accumulators r[j] = a[j] + a[j+8] + ..., combined as
//              ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n % 8 tail   for 8 <= n <= 128
//            = pw(a, h) + pw(a + h, n - h), h = n/2 rounded down to a multiple of 8   for n > 128
// Every leaf of that tree starts at a multiple of 8 and holds at most 128 elements; the right child is
// never shorter than the left.  The device sums a long array one leaf per thread and combines the
// leaves level by level along the same tree (csrc/verification.cu); a short one runs pairwise_sum.
// The translation units compile without FMA contraction (--fmad=false, -ffp-contract=off).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PW_FN __host__ __device__ __forceinline__
#else
#define PW_FN inline
#endif

namespace pw {

constexpr int64_t LEAF = 128;

// the split of a node of n > LEAF elements: its left child's length
PW_FN int64_t left_len(int64_t n) {
    const int64_t h = n / 2;
    return h - h % 8;
}

// a level count D such that every node at depth D of the tree of n elements is a leaf (or lies below
// one): the right child of m elements has at most ceil(m / 2) + 7
PW_FN int depth_bound(int64_t n) {
    int d = 0;
    while (n > LEAF) {
        n = (n + 1) / 2 + 7;
        d++;
    }
    return d;
}

// pw over a leaf of n <= LEAF elements, get(i) for i in [lo, lo + n)
template <typename F, typename Get>
PW_FN F leaf(const Get &get, int64_t lo, int64_t n) {
    if (n < 8) {
        F r = F(0);
        for (int64_t i = 0; i < n; i++) r = r + get(lo + i);
        return r;
    }
    F r[8];
    for (int j = 0; j < 8; j++) r[j] = get(lo + j);
    int64_t i = 8;
    for (; i < n - n % 8; i += 8)
        for (int j = 0; j < 8; j++) r[j] = r[j] + get(lo + i + j);
    F res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res = res + get(lo + i);
    return res;
}

// the node at depth `level` reached by the path whose bits (most significant first) are the low
// `level` bits of u; false when a leaf lies above it (the node does not exist)
PW_FN bool node(int64_t n, int level, int64_t u, int64_t *lo, int64_t *len) {
    int64_t a = 0, m = n;
    for (int l = 0; l < level; l++) {
        if (m <= LEAF) return false;
        const int64_t h = left_len(m);
        if ((u >> (level - 1 - l)) & 1) {
            a += h;
            m -= h;
        } else {
            m = h;
        }
    }
    *lo = a;
    *len = m;
    return true;
}

// 0 + pw(get, n) evaluated serially with an explicit stack; MAXD must exceed depth_bound(n)
template <typename F, int MAXD, typename Get>
PW_FN F pairwise_sum(const Get &get, int64_t n) {
    int64_t lo[MAXD + 1], len[MAXD + 1];
    F left[MAXD + 1];
    int state[MAXD + 1];  // 0: the left child is next, 1: the right child is next
    int sp = 0;
    lo[0] = 0;
    len[0] = n;
    state[0] = 0;
    F ret = F(0);
    for (;;) {
        if (len[sp] <= LEAF) {
            ret = leaf<F>(get, lo[sp], len[sp]);
        } else {
            const int64_t h = left_len(len[sp]);
            lo[sp + 1] = state[sp] == 0 ? lo[sp] : lo[sp] + h;
            len[sp + 1] = state[sp] == 0 ? h : len[sp] - h;
            state[sp + 1] = 0;
            sp++;
            continue;
        }
        // hand ret up to the parents whose right child it completes
        for (;;) {
            if (sp == 0) return F(0) + ret;
            sp--;
            if (state[sp] == 0) {
                left[sp] = ret;
                state[sp] = 1;
                break;
            }
            ret = left[sp] + ret;
        }
    }
}

}  // namespace pw
