// knn_device.cuh -- device-side cKDTree (knn.cu) as used by the outlier test and the grid fill.
#pragma once
#include <algorithm>

#include "common.cuh"
#include "knn_body.cuh"

namespace kdp {

constexpr int NMAX = 4096;      // points of the shared-memory build (more: sequential fallback)
constexpr int WARPS = 8;        // warps of the build CTA, one tree node each
constexpr int QCAP = 512;       // nodes per tree level that still split (each holds > 16 points)
constexpr int QHEAP = 64;       // pending-node heap of one query (typical depth: 10..40)
constexpr int QTHREADS = 32;    // queries per CTA (one thread each)
constexpr int NBSMEM = 32;      // neighbour-heap entries per thread kept in shared memory
constexpr int ARENA = 1 << 17;  // spill space (NodeInfo entries) for queries that outgrow QHEAP

struct TreeBuf {
    int *idx;            // tree order of the points (scipy: tree.indices)
    kd::Node *nodes;     // node 0 is the root
    int *meta;           // [0] node count, [1] point count, [2] next free arena entry
    double *bounds;      // maxes[2], mins[2]
    kd::NodeInfo *arena;
};

struct TreeScratch {
    b200::Scratch idx, nodes, meta, bounds, arena;
    TreeBuf tb;
};

#if defined(__CUDACC__)
__device__ __forceinline__ kd::Tree tree_of(const TreeBuf &tb, const double *xy) {
    kd::Tree t;
    t.data = xy;
    t.n = tb.meta[1];
    t.idx = tb.idx;
    t.nodes = tb.nodes;
    t.nnodes = tb.meta[0];
    for (int c = 0; c < 2; c++) {
        t.maxes[c] = tb.bounds[c];
        t.mins[c] = tb.bounds[2 + c];
    }
    return t;
}

// A query queues at most one far child per internal node it visits, so a heap of `node count`
// entries cannot overflow.  The per-thread heap is QHEAP entries; the rare query that fills it
// moves once to a node-count-sized piece of the arena.  An exhausted arena is a hard error
// (__trap: the next CUDA call fails), never a silently wrong neighbour list.
struct ArenaGrow {
    const TreeBuf &tb;
    __device__ explicit ArenaGrow(const TreeBuf &t) : tb(t) {}
    __device__ bool operator()(kd::Strided<kd::NodeInfo> &q, int &qcap, int qn) const {
        const int need = tb.meta[0];
        if (qcap >= need) return false;
        const int off = atomicAdd(&tb.meta[2], need);
        if (off + need > ARENA) __trap();
        kd::NodeInfo *big = tb.arena + off;
        for (int i = 0; i < qn; i++) big[i] = q[i];
        q.p = big;
        q.stride = 1;
        qcap = need;
        return true;
    }
};

#endif

int tree_alloc(TreeScratch &ts, int n_cap, cudaStream_t s);
int tree_build(const double *xy, const int *n_dev, int n_cap, const TreeBuf &tb, cudaStream_t s);
// recompute the listed grid points (list_count == nullptr: all of them) from scipy's query; twin (or
// null, nvar == 2 only): the (ny, nx) pairs kept beside out, rewritten at the same points
int idw_fix(const double *xy, const double *vals, int nvar, int k, double power, double dist_offset,
            double mean_res, const double *xgrid, int nx, const double *ygrid, int ny, const TreeBuf &tb,
            const int *list, const int *list_count, double *out, double2 *twin, cudaStream_t s);

}  // namespace kdp
