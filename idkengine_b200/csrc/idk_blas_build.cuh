// BLAS.Build + PreSplitting.PreSplit on the device (idkpt_blas_build): the engine's SweepSAH builder with pre-splitting,
// node for node equal to the host mirror (host_mirror/bvh_build.cpp) under libidkpt's flags (-fmad=false, IEEE div and
// sqrt; fmaf only in HalfArea, where the mirror uses it). DESIGN §8f.5 gives the stages and why each one is exact.
//
// Stages (the mirror's function in brackets):
//   1. pre-split [preSplit]: priorities per triangle; their float sum in triangle order by one thread; split counts and
//      their exclusive scan; each triangle splits into its own output range, using the range's tail as its stack.
//   2. sorts [radixSortFragments]: three stable sorts of fragment ids by floatToKey(min + max) (CUB radix sort).
//   3. tree [processSubtree, trySplit]: level by level, one block per node above SMALL_NODE fragments (full prefix and
//      suffix box scans, first strict minimum of L[i] + R[i+1]), then one thread per remaining subtree (the mirror's serial
//      trySplit). Node ids do not depend on the order nodes are split in.
//   4. post passes [computeRequiredStackSize, optimizeStackSize, removeEmptySubtrees, unindex*, computeGlobalSAH]: parallel
//      except for the double sums, which one thread adds in the mirror's DFS order.
//
// The scalar arithmetic comes from idk_bvh_math.h, which the mirror compiles too: boxes, Triangle.Split, the priority, the
// split count, one pre-split step, the serial trySplit (stage 3's one-thread subtrees), the leaf-cost test and side swap that
// end k_split_large, and the SAH and collapse terms. This file keeps the kernels, the block scans and partitions, the
// post-pass kernels and the driver.
#pragma once
#include <cfloat>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include <cub/cub.cuh>

#include "../../include/idk_gpu_types.h"
#include "idk_bvh_math.h"

namespace idkbb {

constexpr int SMALL_NODE = 64;          // subtrees of at most this many fragments are finished by one thread
constexpr int BIG_THREADS = 512;
constexpr int BIG_ITEMS = 4;
constexpr int BIG_TILE = BIG_THREADS * BIG_ITEMS;
constexpr int MAX_FRAGMENTS = 1 << 24;  // float counters are exact up to here
constexpr int DEPTH_NONE = 0x7F7F7F7F;  // memset byte 0x7F: larger than any depth

using namespace idkbvh;

// exact identity of the ordered combine (for padding partial tiles); boxEmpty() is a real first element
__device__ __forceinline__ Box boxIdentity() { return {{INFINITY, INFINITY, INFINITY}, {-INFINITY, -INFINITY, -INFINITY}}; }
__device__ __forceinline__ void storeBox(Box* b, size_t i, const Box& v) {
    float2* p = reinterpret_cast<float2*>(b + i);
    p[0] = make_float2(v.mn[0], v.mn[1]); p[1] = make_float2(v.mn[2], v.mx[0]); p[2] = make_float2(v.mx[1], v.mx[2]);
}

// ---------------------------------------------------------------------------------------------------------------- pre-split
__device__ __forceinline__ Tri loadTri(const PackedVec3* pos, const GpuBlasTriangle* tris, int i) {
    const GpuBlasTriangle t = tris[i];
    const int id[3] = {t.X, t.Y, t.Z};
    Tri r;
    for (int k = 0; k < 3; k++) { const PackedVec3 q = pos[(uint32_t)id[k]]; r.p[k] = {{q.x, q.y, q.z}}; }
    return r;
}

__global__ void k_priorities(const PackedVec3* pos, const GpuBlasTriangle* tris, int n, float* prio) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) prio[i] = priority(loadTri(pos, tris, i));
}

// Ordered sums: one thread adds the values in index order, as the mirror does (float addition is not associative).
// The block stages tiles through shared memory so that the one adding thread reads nothing from HBM itself.
constexpr int SUM_THREADS = 1024;
template <class T, int TILE>
__global__ void __launch_bounds__(SUM_THREADS) k_ordered_sum(const T* v, int n, const int* nDev, T* acc) {
    __shared__ T tile[TILE];
    if (nDev) n = *nDev;
    T s = threadIdx.x == 0 ? *acc : T(0);
    for (int base = 0; base < n; base += TILE) {
        const int m = min(TILE, n - base);
        for (int k = threadIdx.x; k < m; k += SUM_THREADS) tile[k] = v[base + k];
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll 8
            for (int k = 0; k < m; k++) s += tile[k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *acc = s;
}

__global__ void k_split_counts(const float* prio, const float* total, int n, float splitFactor, unsigned long long* counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { counts[n] = 0; return; }
    counts[i] = splitCount(prio[i], *total, n, splitFactor);
}

// Box of every vertex in triangle order (p0, p1, p2 of each): per-thread chunks folded in order, chunks combined in order.
__global__ void __launch_bounds__(1024) k_global_box(const PackedVec3* pos, const GpuBlasTriangle* tris, int n, Box* out) {
    __shared__ Box part[1024];
    __shared__ int has[1024];
    const int per = (n + 1023) / 1024;
    const int b0 = min(n, threadIdx.x * per), e0 = min(n, b0 + per);
    Box acc = boxIdentity();
    for (int i = b0; i < e0; i++) {
        const Tri t = loadTri(pos, tris, i);
        for (int k = 0; k < 3; k++) { Box p = {{t.p[k].v[0], t.p[k].v[1], t.p[k].v[2]}, {t.p[k].v[0], t.p[k].v[1], t.p[k].v[2]}}; acc = combine(acc, p); }
    }
    part[threadIdx.x] = acc;
    has[threadIdx.x] = e0 > b0;
    __syncthreads();
    if (threadIdx.x == 0) {
        Box g = boxEmpty();
        for (int t = 0; t < 1024; t++) if (has[t]) g = combine(g, part[t]);
        *out = g;
    }
}

// One thread per triangle, writing its fragments to [off[i], off[i+1]). The split stack lives in the same range, growing
// down from its end: the stack's items hold at least one fragment each and together exactly the ones not yet written, so
// they never reach the slot the next fragment goes to. Item j: box in bounds[end-1-j], split count in ids[end-1-j].
__global__ void k_presplit(const PackedVec3* pos, const GpuBlasTriangle* tris, int n, const unsigned long long* off,
                           const Box* globalBox, Box* bounds, int* origIds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Box g = *globalBox;
    const Tri tri = loadTri(pos, tris, i);
    const size_t begin = (size_t)off[i], end = (size_t)off[i + 1];
    size_t counter = begin;
    int sp = 0;
    storeBox(bounds, end - 1, boxFromTri(tri));
    origIds[end - 1] = (int)(end - begin);
    sp = 1;
    while (sp > 0) {
        sp--;
        const Box box = loadBox(bounds, (int)(end - 1 - sp));
        const int splits = origIds[end - 1 - sp];
        if (splits == 1) {
            storeBox(bounds, counter, box);
            origIds[counter] = i;
            counter++;
            continue;
        }
        Box l, r;
        const int leftCount = presplitStep(tri, box, splits, g, l, r);
        storeBox(bounds, end - 1 - sp, r);
        origIds[end - 1 - sp] = splits - leftCount;
        sp++;
        storeBox(bounds, end - 1 - sp, l);
        origIds[end - 1 - sp] = leftCount;
        sp++;
    }
}

__global__ void k_tri_bounds(const PackedVec3* pos, const GpuBlasTriangle* tris, int n, Box* bounds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) storeBox(bounds, i, boxFromTri(loadTri(pos, tris, i)));
}

__global__ void k_sort_keys(const Box* bounds, int n, int axis, uint32_t* keys, int* vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Box b = loadBox(bounds, i);
    keys[i] = floatToKey(b.mn[axis] + b.mx[axis]);
    vals[i] = i;
}

// ---------------------------------------------------------------------------------------------------------------- tree
struct TreeArgs {
    const Box* bounds;
    int* ids[3];
    int* aux;
    uint8_t* table;
    float* rcost;               // right costs by fragment position (the mirror's rightCostsAccum)
    GpuBlasNode* nodes;
    int* parent;                // per node id: its parent, the root's is 0
    int* depth;                 // per node id: depth below the root (-1: id not used)
    int* ostart;                // per node id: first fragment of its range (also for nodes later split)
    int* ocount;                // per node id: fragments in its range
    const int2* tasks;          // (parentNodeId, newNodesId) of this level's large nodes
    int2* nextTasks;
    int* nextCount;
    int2* small;                // subtrees left to one thread each
    int* smallCount;
    Params p;
};

__device__ __forceinline__ void pushTask(const TreeArgs& a, int2 t, int count) {
    if (count > SMALL_NODE) a.nextTasks[atomicAdd(a.nextCount, 1)] = t;
    else a.small[atomicAdd(a.smallCount, 1)] = t;
}

__device__ __forceinline__ void writeChildren(const TreeArgs& a, int pid, int2 task, int start, int count, int split) {
    GpuBlasNode& parent = a.nodes[pid];
    const int leftId = task.y, rightId = leftId + 1;
    const int lc = split - start, rc = count - lc;
    GpuBlasNode l = {}, r = {};
    l.TriStartOrChild = start; l.TriCount = lc;
    r.TriStartOrChild = split; r.TriCount = rc;
    a.nodes[leftId] = l;
    a.nodes[rightId] = r;
    const int d = a.depth[pid] + 1;
    a.parent[leftId] = pid; a.parent[rightId] = pid;
    a.depth[leftId] = d; a.depth[rightId] = d;
    a.ostart[leftId] = start; a.ocount[leftId] = lc;
    a.ostart[rightId] = split; a.ocount[rightId] = rc;
    parent.TriStartOrChild = leftId;
    parent.TriCount = 0;
}

// ---- block-wide ordered scans
__device__ __forceinline__ Box shflUpBox(const Box& v, int o) {
    Box r;
    for (int i = 0; i < 3; i++) { r.mn[i] = __shfl_up_sync(0xffffffffu, v.mn[i], o); r.mx[i] = __shfl_up_sync(0xffffffffu, v.mx[i], o); }
    return r;
}

// Exclusive ordered scan of one box per thread over the block; `total` is the fold of all of them.
__device__ Box blockScanBox(Box v, Box& total) {
    __shared__ Box warpTot[BIG_THREADS / 32];
    __shared__ Box warpPre[BIG_THREADS / 32];
    __shared__ Box all;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Box inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const Box other = shflUpBox(inc, o);
        if (lane >= o) inc = combine(other, inc);
    }
    Box exc = shflUpBox(inc, 1);
    if (lane == 0) exc = boxIdentity();
    if (lane == 31) warpTot[warp] = inc;
    __syncthreads();
    if (threadIdx.x == 0) {
        Box acc = boxIdentity();
        for (int w = 0; w < BIG_THREADS / 32; w++) { warpPre[w] = acc; acc = combine(acc, warpTot[w]); }
        all = acc;
    }
    __syncthreads();
    total = all;
    const Box r = combine(warpPre[warp], exc);
    __syncthreads();   // the shared words are reused by the next call
    return r;
}

__device__ int blockScanInt(int v, int& total) {
    __shared__ int warpTot[BIG_THREADS / 32];
    __shared__ int warpPre[BIG_THREADS / 32 + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int other = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += other;
    }
    if (lane == 31) warpTot[warp] = inc;
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int w = 0; w < BIG_THREADS / 32; w++) { warpPre[w] = acc; acc += warpTot[w]; }
        warpPre[BIG_THREADS / 32] = acc;
    }
    __syncthreads();
    total = warpPre[BIG_THREADS / 32];
    const int r = warpPre[warp] + inc - v;
    __syncthreads();
    return r;
}

__device__ unsigned long long blockMinU64(unsigned long long v) {
    __shared__ unsigned long long s;
    if (threadIdx.x == 0) s = ~0ull;
    __syncthreads();
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_down_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) atomicMin(&s, v);
    __syncthreads();
    const unsigned long long r = s;
    __syncthreads();
    return r;
}

// computeBoundingBox: Box::empty() grown by the fragments [lo, hi) of `ids` in order.
__device__ Box blockRangeBox(const Box* bounds, const int* ids, int lo, int hi) {
    Box carry = boxEmpty();
    for (int base = lo; base < hi; base += BIG_TILE) {
        Box loc = boxIdentity();
        for (int k = 0; k < BIG_ITEMS; k++) {
            const int i = base + threadIdx.x * BIG_ITEMS + k;
            if (i < hi) loc = combine(loc, loadBox(bounds, ids[i]));
        }
        Box total;
        blockScanBox(loc, total);
        carry = combine(carry, total);
    }
    return carry;
}

// Stable partition of ids[start, end) by table[id] (ones first), through aux; `ones` is the number of ones.
__device__ void blockPartition(int* ids, int* aux, const uint8_t* table, int start, int end, int ones) {
    int carryOnes = 0;
    for (int base = start; base < end; base += BIG_TILE) {
        int id[BIG_ITEMS];
        int f = 0;
        for (int k = 0; k < BIG_ITEMS; k++) {
            const int i = base + threadIdx.x * BIG_ITEMS + k;
            id[k] = i < end ? ids[i] : -1;
            f += (id[k] >= 0 && table[id[k]]) ? 1 : 0;
        }
        int total;
        int before = carryOnes + blockScanInt(f, total);
        for (int k = 0; k < BIG_ITEMS; k++) {
            const int i = base + threadIdx.x * BIG_ITEMS + k;
            if (i >= end) break;
            if (table[id[k]]) aux[start + before++] = id[k];
            else aux[start + ones + (i - start) - before] = id[k];
        }
        carryOnes += total;
    }
    __syncthreads();
    for (int i = start + threadIdx.x; i < end; i += BIG_THREADS) ids[i] = aux[i];
    __syncthreads();
}

// One block per node: BLAS.TrySplit over full scans (DESIGN §8f.5), then the split.
__global__ void __launch_bounds__(BIG_THREADS) k_split_large(TreeArgs a) {
    const int2 task = a.tasks[blockIdx.x];
    const int pid = task.x;
    const int start = a.nodes[pid].TriStartOrChild, count = a.nodes[pid].TriCount, end = start + count;
    const Box pbox = blockRangeBox(a.bounds, a.ids[0], start, end);
    if (threadIdx.x == 0) setBounds(a.nodes[pid], pbox);
    if (count <= a.p.stopSplittingThreshold) return;

    float bestCost = FLT_MAX;
    int bestAxis = 0, bestSplit = 0;
    for (int axis = 0; axis < 3; axis++) {
        const int* ids = a.ids[axis];
        // suffix: R[i] = HalfArea(box of [i, end)) * (end - i), i in [start + 1, end)
        Box carry = boxEmpty();
        for (int jb = 0; jb < count - 1; jb += BIG_TILE) {
            Box b[BIG_ITEMS];
            Box loc = boxIdentity();
            for (int k = 0; k < BIG_ITEMS; k++) {
                const int j = jb + threadIdx.x * BIG_ITEMS + k;
                b[k] = j < count - 1 ? loadBox(a.bounds, ids[end - 1 - j]) : boxIdentity();
                loc = combine(loc, b[k]);
            }
            Box total;
            Box acc = combine(carry, blockScanBox(loc, total));
            for (int k = 0; k < BIG_ITEMS; k++) {
                const int j = jb + threadIdx.x * BIG_ITEMS + k;
                acc = combine(acc, b[k]);
                if (j < count - 1) a.rcost[end - 1 - j] = halfArea(acc) * (float)(j + 1);
            }
            carry = combine(carry, total);
        }
        __syncthreads();
        // prefix: L[i] = HalfArea(box of [start, i]) * (i - start + 1); candidate split i + 1 costs L[i] + R[i + 1]
        unsigned long long best = ~0ull;
        carry = boxEmpty();
        for (int base = start; base < end - 1; base += BIG_TILE) {
            Box b[BIG_ITEMS];
            Box loc = boxIdentity();
            for (int k = 0; k < BIG_ITEMS; k++) {
                const int i = base + threadIdx.x * BIG_ITEMS + k;
                b[k] = i < end - 1 ? loadBox(a.bounds, ids[i]) : boxIdentity();
                loc = combine(loc, b[k]);
            }
            Box total;
            Box acc = combine(carry, blockScanBox(loc, total));
            for (int k = 0; k < BIG_ITEMS; k++) {
                const int i = base + threadIdx.x * BIG_ITEMS + k;
                acc = combine(acc, b[k]);
                if (i < end - 1) {
                    const float cost = halfArea(acc) * (float)(i - start + 1) + a.rcost[i + 1];
                    if (cost < FLT_MAX) best = min(best, ((unsigned long long)__float_as_uint(cost) << 32) | (uint32_t)(i + 1));
                }
            }
            carry = combine(carry, total);
        }
        best = blockMinU64(best);
        if (best != ~0ull) {
            const float c = __uint_as_float((uint32_t)(best >> 32));
            if (c < bestCost) { bestCost = c; bestAxis = axis; bestSplit = (int)(uint32_t)best; }
        }
    }
    if (!keepSplit(a.p, pbox, start, count, bestCost, bestAxis, bestSplit)) return;
    int* ids = a.ids[bestAxis];
    const Box lbox = blockRangeBox(a.bounds, ids, start, bestSplit);
    const Box rbox = blockRangeBox(a.bounds, ids, bestSplit, end);
    const bool swap = swapSides(lbox, rbox);
    for (int i = start + threadIdx.x; i < end; i += BIG_THREADS) a.table[ids[i]] = i < bestSplit ? !swap : swap;
    __syncthreads();
    const int ones = swap ? end - bestSplit : bestSplit - start;
    if (swap) blockPartition(ids, a.aux, a.table, start, end, ones);
    blockPartition(a.ids[(bestAxis + 1) % 3], a.aux, a.table, start, end, ones);
    blockPartition(a.ids[(bestAxis + 2) % 3], a.aux, a.table, start, end, ones);
    if (threadIdx.x == 0) {
        const int split = start + ones;
        writeChildren(a, pid, task, start, count, split);
        const int lc = split - start;
        pushTask(a, make_int2(task.y, task.y + 2), lc);
        pushTask(a, make_int2(task.y + 1, task.y + 1 + (2 * lc - 1)), count - lc);
    }
}

// ---- one thread per subtree: the mirror's processSubtree around the shared serial trySplit
__global__ void k_split_small(TreeArgs a, int n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    int2 stack[SMALL_NODE + 1];   // a subtree of c fragments is at most c - 1 deep
    int sp = 0;
    stack[sp++] = a.small[t];
    while (sp > 0) {
        const int2 task = stack[--sp];
        GpuBlasNode& parent = a.nodes[task.x];
        const int start = parent.TriStartOrChild, count = parent.TriCount;
        const Box box = rangeBox(a.bounds, a.ids[0], start, start + count);
        setBounds(parent, box);
        const int split = trySplitSerial(a.bounds, a.ids, a.rcost, a.table, a.aux, a.p, box, start, count);
        if (split < 0) continue;
        writeChildren(a, task.x, task, start, count, split);
        const int lc = split - start;
        stack[sp++] = make_int2(task.y + 1, task.y + 1 + (2 * lc - 1));
        stack[sp++] = make_int2(task.y, task.y + 2);
    }
}

// ---------------------------------------------------------------------------------------------------------------- post passes
__global__ void k_root_duplicate(GpuBlasNode* nodes, int* parent, int* depth, int* ostart, int* ocount, int n) {
    GpuBlasNode root = nodes[1];
    nodes[2] = root;
    nodes[3] = root;
    root.TriStartOrChild = 2;
    root.TriCount = 0;
    nodes[1] = root;
    for (int k = 2; k < 4; k++) { parent[k] = 1; depth[k] = 1; ostart[k] = 0; ocount[k] = n; }
}

// computeRequiredStackSize, bottom up: g(v) = 0 if both children of v are leaves, g(inner child) if one is, and
// max(g(l), g(r)) + 1 if both are. Each climb starts at a node with two leaf children; at a node with two inner children
// the second arrival continues.
__global__ void k_stack_size(const GpuBlasNode* nodes, const int* parent, const int* depth, int cap, int* g, int* arrive) {
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < 1 || v >= cap || depth[v] < 0 || nodes[v].TriCount > 0) return;
    const int c0 = nodes[v].TriStartOrChild;
    if (!(nodes[c0].TriCount > 0 && nodes[c0 + 1].TriCount > 0)) return;
    int gv = 0;
    g[v] = 0;
    for (;;) {
        const int p = parent[v];
        if (p <= 0) return;
        const int c = nodes[p].TriStartOrChild;
        const bool li = !(nodes[c].TriCount > 0), ri = !(nodes[c + 1].TriCount > 0);
        if (li && ri) {
            __threadfence();
            if (atomicAdd(&arrive[p], 1) == 0) return;
            __threadfence();
            const int gl = ((volatile int*)g)[c], gr = ((volatile int*)g)[c + 1];
            gv = max(gl, gr) + 1;
        }
        ((volatile int*)g)[p] = gv;
        v = p;
    }
}

// Pre-order ranks: the nodes whose range starts at fragment s are a chain of left children, one per depth from the
// highest one (dmin) down to a leaf (dleaf); pre-order lists the chains by s. rank = base[s] + depth - dmin[s].
__global__ void k_chain_ends(const GpuBlasNode* nodes, const int* depth, const int* ostart, int cap, int* dmin, int* dleaf) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < 1 || v >= cap || depth[v] < 0) return;
    atomicMin(&dmin[ostart[v]], depth[v]);
    if (nodes[v].TriCount > 0) dleaf[ostart[v]] = depth[v];
}
__global__ void k_chain_len(const int* dmin, const int* dleaf, int n, int* len) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) len[s] = dmin[s] == DEPTH_NONE ? 0 : dleaf[s] - dmin[s] + 1;
}
__global__ void k_preorder(const int* depth, const int* ostart, int cap, const int* dmin, const int* base, int* order) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < 1 || v >= cap || depth[v] < 0) return;
    const int s = ostart[v];
    order[base[s] + depth[v] - dmin[s]] = v;
}
__global__ void k_preorder_root_duplicate(int* order) { order[0] = 1; order[1] = 2; order[2] = 3; }

// computeGlobalSAH terms in pre-order; leaf counts from `counts` (by node id) or, for the compacted tree, `final`.
__global__ void k_sah_terms(const int* order, int m, const GpuBlasNode* nodes, const GpuBlasNode* final, const int* fidx,
                            float triangleCost, double* terms) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int v = order[j];
    const GpuBlasNode n = final ? final[fidx[v]] : nodes[v];
    const GpuBlasNode root = final ? final[1] : nodes[1];
    terms[j] = sahTerm(n, 1.0 / (double)nodeHalfArea(root), triangleCost);
}

// collapseDeepestLevel's cost terms, in pre-order (the nodes that add one never contain each other, so this is also the
// mirror's post-order among them). First pass: inner nodes deeper than `level` whose children are both leaves. Later passes:
// inner nodes at depth `level`, whose children are leaves after the pass's collapse and hold their whole subtrees.
__global__ void k_collapse_terms(const int* order, int m, const GpuBlasNode* nodes, const int* depth, const int* ocount,
                                 int level, int firstPass, float triangleCost, double* terms, uint8_t* flags) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int v = order[j];
    const GpuBlasNode n = nodes[v];
    bool q = false;
    if (!(n.TriCount > 0)) {
        const int c = n.TriStartOrChild;
        q = firstPass ? (depth[v] > level && nodes[c].TriCount > 0 && nodes[c + 1].TriCount > 0) : depth[v] == level;
        if (q) {
            terms[j] = collapseTerm(n, nodes[c], nodes[c + 1], ocount[c], ocount[c + 1], nodes[1], triangleCost);
        }
    }
    flags[j] = q;
}

__global__ void k_reachable(const int* order, int m, const int* depth, int maxDepth, uint8_t* flags) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) flags[j] = depth[order[j]] <= maxDepth;
}

// After the collapse passes a node is inner if it was split and is shallower than the collapsed level.
__device__ __forceinline__ bool finalInner(const GpuBlasNode* nodes, const int* depth, int v, int maxDepth) {
    return !(nodes[v].TriCount > 0) && depth[v] < maxDepth;
}
__global__ void k_inner_flags(const int* order, int m, const GpuBlasNode* nodes, const int* depth, int maxDepth, int* flags) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) flags[j] = finalInner(nodes, depth, order[j], maxDepth);
}
__global__ void k_inner_ranks(const int* order, int m, const int* scan, int* rankOf) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) rankOf[order[j]] = scan[j];
}

// removeEmptySubtrees: the children of the inner node of pre-order rank k land at 2 + 2k.
__global__ void k_final_nodes(const int* order, int m, const GpuBlasNode* nodes, const int* parent, const int* depth,
                              const int* ostart, const int* ocount, const int* rankOf, int maxDepth, GpuBlasNode* final, int* fidx) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int v = order[j];
    int fi = 1;
    if (v != 1) {
        const int p = parent[v];
        fi = 2 + 2 * rankOf[p] + (v == nodes[p].TriStartOrChild + 1 ? 1 : 0);
    }
    fidx[v] = fi;
    GpuBlasNode out = nodes[v];
    if (finalInner(nodes, depth, v, maxDepth)) { out.TriStartOrChild = 2 + 2 * rankOf[v]; out.TriCount = 0; }
    else { out.TriStartOrChild = ostart[v]; out.TriCount = ocount[v]; }
    final[fi] = out;
}

// BLAS.GetUnindexedTriangles: leaves in node order, fragment = triangle. The array holds n triangles; when the root is a
// leaf, its two copies list all n each, and the second one's triangles would land past the end: the mirror writes them
// beyond its n-element array (heap overflow), so what it returns is the first copy's n triangles and the second leaf's
// offset n. The writes past n are dropped here.
__global__ void k_leaf_counts(const GpuBlasNode* final, int f, int* counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < f) counts[i] = (i >= 2 && final[i].TriCount > 0) ? final[i].TriCount : 0;
}
__global__ void k_unindex_plain(GpuBlasNode* final, int f, const int* offsets, const int* ids0, const GpuBlasTriangle* in,
                                GpuBlasTriangle* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 2 || i >= f || !(final[i].TriCount > 0)) return;
    const int s = final[i].TriStartOrChild, c = final[i].TriCount, o = offsets[i];
    for (int k = 0; k < c && o + k < n; k++) out[o + k] = in[ids0[s + k]];
    final[i].TriStartOrChild = o;
}

// PreSplitting.GetUnindexedTriangles: per leaf the sorted unique triangle ids, from one sort of (leaf start, triangle id)
__global__ void k_leaf_marks(const GpuBlasNode* final, int f, int* marks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 && i < f && final[i].TriCount > 0) marks[final[i].TriStartOrChild] = final[i].TriStartOrChild;
}
__global__ void k_leaf_keys(const int* segStart, const int* ids0, const int* origIds, int n, unsigned long long* keys) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < n) keys[q] = ((unsigned long long)(uint32_t)segStart[q] << 32) | (uint32_t)origIds[ids0[q]];
}

struct MaxOp { __device__ int operator()(int x, int y) const { return x > y ? x : y; } };

struct Uniq {   // walks the sorted ids of one leaf, skipping repeats
    const unsigned long long* k;
    int i, end;
    __device__ Uniq(const unsigned long long* keys, const GpuBlasNode& leaf) : k(keys), i(leaf.TriStartOrChild), end(leaf.TriStartOrChild + leaf.TriCount) {}
    __device__ bool done() const { return i >= end; }
    __device__ int cur() const { return (int)(uint32_t)k[i]; }
    __device__ void next() { const int c = cur(); while (i < end && cur() == c) i++; }
};
__device__ int uniqueCount(const unsigned long long* keys, const GpuBlasNode& leaf) {
    int c = 0;
    for (Uniq u(keys, leaf); !u.done(); u.next()) c++;
    return c;
}
__device__ int sharedCount(const unsigned long long* keys, const GpuBlasNode& l, const GpuBlasNode& r) {
    int c = 0;
    Uniq a(keys, l), b(keys, r);
    while (!a.done() && !b.done()) {
        if (a.cur() < b.cur()) a.next();
        else if (b.cur() < a.cur()) b.next();
        else { c++; a.next(); b.next(); }
    }
    return c;
}

__global__ void k_pair_sizes(const GpuBlasNode* final, int pairs, const unsigned long long* keys, int* sizes) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > pairs) return;
    if (p == pairs) { sizes[p] = 0; return; }
    const GpuBlasNode l = final[2 + 2 * p], r = final[3 + 2 * p];
    const bool ll = l.TriCount > 0, rl = r.TriCount > 0;
    int s = 0;
    if (ll && rl) s = uniqueCount(keys, l) + uniqueCount(keys, r) - sharedCount(keys, l, r);
    else if (ll) s = uniqueCount(keys, l);
    else if (rl) s = uniqueCount(keys, r);
    sizes[p] = s;
}

__global__ void k_pair_write(GpuBlasNode* final, int pairs, const unsigned long long* keys, const int* offsets,
                             const GpuBlasTriangle* in, GpuBlasTriangle* out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= pairs) return;
    GpuBlasNode& l = final[2 + 2 * p];
    GpuBlasNode& r = final[3 + 2 * p];
    const bool ll = l.TriCount > 0, rl = r.TriCount > 0;
    const int counter = offsets[p];
    if (ll && rl) {
        const GpuBlasNode L = l, R = r;
        const int lu = uniqueCount(keys, L), ru = uniqueCount(keys, R);
        int onlyLeft = 0, backwards = 0;
        {   // left ids ascending: the ones also in the right leaf fill the end of the left range backwards
            Uniq a(keys, L), b(keys, R);
            for (; !a.done(); a.next()) {
                const int id = a.cur();
                while (!b.done() && b.cur() < id) b.next();
                if (!b.done() && b.cur() == id) out[counter + lu - backwards++ - 1] = in[id];
                else out[counter + onlyLeft++] = in[id];
            }
        }
        int onlyRight = 0;
        {
            Uniq a(keys, R), b(keys, L);
            for (; !a.done(); a.next()) {
                const int id = a.cur();
                while (!b.done() && b.cur() < id) b.next();
                if (!(!b.done() && b.cur() == id)) out[counter + lu + onlyRight++] = in[id];
            }
        }
        l.TriStartOrChild = counter; l.TriCount = lu;
        r.TriStartOrChild = counter + onlyLeft; r.TriCount = ru;
    } else if (ll || rl) {
        GpuBlasNode& leaf = ll ? l : r;
        const GpuBlasNode Lf = leaf;
        int c = 0;
        for (Uniq u(keys, Lf); !u.done(); u.next()) out[counter + c++] = in[u.cur()];
        leaf.TriStartOrChild = counter;
        leaf.TriCount = c;
    }
}

// BLAS.ComputeGlobalSAH (BLAS.cs:629-656) of one BLAS as the device holds it (built, refitted or rebuilt): one thread walks
// the tree in the engine's pre-order, left child first, and adds the terms in that order. `stack` holds the pending right
// children: at most one per level, so the node count bounds it.
__global__ void k_global_sah(const GpuBlasNode* nodes, int* stack, float triangleCost, double* out) {
    const double rootArea = 1.0 / (double)nodeHalfArea(nodes[1]);
    double cost = 0.0;
    int sp = 0, v = 1;
    for (;;) {
        const GpuBlasNode n = nodes[v];
        cost += sahTerm(n, rootArea, triangleCost);
        if (!(n.TriCount > 0)) {
            stack[sp++] = n.TriStartOrChild + 1;
            v = n.TriStartOrChild;
        } else if (sp > 0) {
            v = stack[--sp];
        } else {
            break;
        }
    }
    *out = cost;
}

}  // namespace idkbb

// ---------------------------------------------------------------------------------------------------------------- host driver
struct IdkPtBlasBuild {
    std::vector<GpuBlasNode> nodes;
    std::vector<GpuBlasTriangle> tris;
    int32_t requiredStackSize = 0;
    int32_t fragmentCount = 0;
    double sah = 0.0;
};

namespace idkbb {

// Device allocations of one build, freed together.
struct Arena {
    std::vector<void*> ptrs;
    ~Arena() { for (void* p : ptrs) cudaFree(p); }
    template <class T> cudaError_t get(T*& out, size_t count) {
        void* p = nullptr;
        cudaError_t e = cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(p);
        out = (T*)p;
        return e;
    }
};

// Per-stage device times (IDKPT_BLAS_TIMING=1 prints them to stderr, like the host mirror's IDKHOST_TIMING).
struct StageTimer {
    cudaStream_t s;
    std::vector<std::pair<const char*, cudaEvent_t>> marks;
    explicit StageTimer(cudaStream_t st) : s(st) {}
    ~StageTimer() { for (auto& m : marks) cudaEventDestroy(m.second); }
    void mark(const char* what) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return;
        cudaEventRecord(e, s);
        marks.push_back({what, e});
    }
    float total() {
        float ms = 0.0f;
        if (marks.size() >= 2) cudaEventElapsedTime(&ms, marks.front().second, marks.back().second);
        return ms;
    }
    void print(int fragments) {
        if (!getenv("IDKPT_BLAS_TIMING")) return;
        for (size_t i = 1; i < marks.size(); i++) {
            float ms = 0.0f;
            cudaEventElapsedTime(&ms, marks[i - 1].second, marks[i].second);
            fprintf(stderr, "[idkpt_blas_build] %-14s %8.2f ms\n", marks[i].first, ms);
        }
        fprintf(stderr, "[idkpt_blas_build] %-14s %8.2f ms (%d fragments)\n", "total", total(), fragments);
    }
};

template <class F> static inline int blocksFor(F n, int t) { return (int)((n + t - 1) / t); }

enum { BB_OK = 0, BB_CUDA = 1, BB_TOO_MANY_FRAGMENTS = 2 };

#define BB_CK(call)                                                                                     \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess) { err = std::string(#call) + ": " + cudaGetErrorString(e_); return BB_CUDA; } \
    } while (0)

// One build's result on the device: the nodes, the triangles and the SAH live in allocations of the caller's arena.
struct DeviceResult {
    GpuBlasNode* nodes = nullptr;
    int nodeCount = 0;
    GpuBlasTriangle* tris = nullptr;
    int triCount = 0;
    int requiredStackSize = 0;
    int fragmentCount = 0;
    double* sah = nullptr;
};

// Runs the whole build on `stream` from device arrays (global vertex ids into `pos`); the arguments have been validated.
// The result goes to `out`, in allocations of `keep`; the scratch is freed on return, after the stream has been waited for.
static int build_device(cudaStream_t stream, const PackedVec3* pos, const GpuBlasTriangle* tris, int triCount, const Params& p,
                        Arena& keep, DeviceResult& out, StageTimer& tm, std::string& err) {
    Arena ar;

    // ---- 1. fragments
    int n = triCount;
    Box* bounds = nullptr;
    int* origIds = nullptr;
    void* cubTemp = nullptr;
    size_t cubBytes = 0;
    auto cubScratch = [&](size_t need) -> cudaError_t {
        if (need <= cubBytes) return cudaSuccess;
        uint8_t* q;
        cudaError_t e = ar.get(q, need);
        if (e == cudaSuccess) { cubTemp = q; cubBytes = need; }
        return e;
    };
    if (p.doPreSplit) {
        float* prio;
        float* total;
        unsigned long long *counts, *offsets;
        Box* gbox;
        BB_CK(ar.get(prio, triCount));
        BB_CK(ar.get(total, 1));
        BB_CK(ar.get(counts, (size_t)triCount + 1));
        BB_CK(ar.get(offsets, (size_t)triCount + 1));
        BB_CK(ar.get(gbox, 1));
        k_priorities<<<blocksFor(triCount, 256), 256, 0, stream>>>(pos, tris, triCount, prio);
        tm.mark("priorities");
        BB_CK(cudaMemsetAsync(total, 0, sizeof(float), stream));
        k_ordered_sum<float, 8192><<<1, SUM_THREADS, 0, stream>>>(prio, triCount, nullptr, total);
        tm.mark("priority sum");
        k_split_counts<<<blocksFor(triCount + 1, 256), 256, 0, stream>>>(prio, total, triCount, p.splitFactor, counts);
        size_t need = 0;
        BB_CK(cub::DeviceScan::ExclusiveSum(nullptr, need, counts, offsets, triCount + 1, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceScan::ExclusiveSum(cubTemp, need, counts, offsets, triCount + 1, stream));
        unsigned long long fragments = 0;
        BB_CK(cudaMemcpyAsync(&fragments, offsets + triCount, sizeof(fragments), cudaMemcpyDeviceToHost, stream));
        BB_CK(cudaStreamSynchronize(stream));
        if (fragments > (unsigned long long)MAX_FRAGMENTS) {
            err = "pre-splitting makes " + std::to_string(fragments) + " fragments, more than 2^24";
            return BB_TOO_MANY_FRAGMENTS;
        }
        n = (int)fragments;
        BB_CK(ar.get(bounds, n));
        BB_CK(ar.get(origIds, n));
        k_global_box<<<1, 1024, 0, stream>>>(pos, tris, triCount, gbox);
        k_presplit<<<blocksFor(triCount, 128), 128, 0, stream>>>(pos, tris, triCount, offsets, gbox, bounds, origIds);
        tm.mark("split");
    } else {
        BB_CK(ar.get(bounds, n));
        k_tri_bounds<<<blocksFor(n, 256), 256, 0, stream>>>(pos, tris, n, bounds);
        tm.mark("bounds");
    }

    // ---- 2. three stable sorts by centroid key
    TreeArgs a = {};
    {
        uint32_t *keys, *keysOut;
        int* vals;
        BB_CK(ar.get(keys, n));
        BB_CK(ar.get(keysOut, n));
        BB_CK(ar.get(vals, n));
        for (int axis = 0; axis < 3; axis++) {
            BB_CK(ar.get(a.ids[axis], n));
            k_sort_keys<<<blocksFor(n, 256), 256, 0, stream>>>(bounds, n, axis, keys, vals);
            size_t need = 0;
            BB_CK(cub::DeviceRadixSort::SortPairs(nullptr, need, keys, keysOut, vals, a.ids[axis], n, 0, 32, stream));
            BB_CK(cubScratch(need));
            BB_CK(cub::DeviceRadixSort::SortPairs(cubTemp, need, keys, keysOut, vals, a.ids[axis], n, 0, 32, stream));
        }
    }
    tm.mark("sort");

    // ---- 3. tree
    const int cap = std::max(2 * n, 4);
    a.bounds = bounds;
    a.p = p;
    BB_CK(ar.get(a.aux, n));
    BB_CK(ar.get(a.table, n));
    BB_CK(ar.get(a.rcost, n));
    BB_CK(ar.get(a.nodes, cap));
    BB_CK(ar.get(a.parent, cap));
    BB_CK(ar.get(a.depth, cap));
    BB_CK(ar.get(a.ostart, cap));
    BB_CK(ar.get(a.ocount, cap));
    const int bigCap = n / (SMALL_NODE + 1) + 2;
    int2 *big[2], *small;
    int* counters;   // [0]: next level's large nodes, [1]: small subtrees
    BB_CK(ar.get(big[0], bigCap));
    BB_CK(ar.get(big[1], bigCap));
    BB_CK(ar.get(small, n + 1));
    BB_CK(ar.get(counters, 2));
    BB_CK(cudaMemsetAsync(a.nodes, 0, (size_t)cap * sizeof(GpuBlasNode), stream));
    BB_CK(cudaMemsetAsync(a.depth, 0xFF, (size_t)cap * sizeof(int), stream));
    BB_CK(cudaMemsetAsync(counters, 0, 2 * sizeof(int), stream));
    {
        GpuBlasNode root = {};
        root.TriStartOrChild = 0;
        root.TriCount = n;
        const int zero = 0;
        const int2 task = make_int2(1, 2);
        BB_CK(cudaMemcpyAsync(a.nodes + 1, &root, sizeof(root), cudaMemcpyHostToDevice, stream));
        BB_CK(cudaMemcpyAsync(a.parent + 1, &zero, 4, cudaMemcpyHostToDevice, stream));
        BB_CK(cudaMemcpyAsync(a.depth + 1, &zero, 4, cudaMemcpyHostToDevice, stream));
        BB_CK(cudaMemcpyAsync(a.ostart + 1, &zero, 4, cudaMemcpyHostToDevice, stream));
        BB_CK(cudaMemcpyAsync(a.ocount + 1, &n, 4, cudaMemcpyHostToDevice, stream));
        if (n > SMALL_NODE) BB_CK(cudaMemcpyAsync(big[0], &task, sizeof(task), cudaMemcpyHostToDevice, stream));
        else {
            const int one = 1;
            BB_CK(cudaMemcpyAsync(small, &task, sizeof(task), cudaMemcpyHostToDevice, stream));
            BB_CK(cudaMemcpyAsync(counters + 1, &one, 4, cudaMemcpyHostToDevice, stream));
        }
        BB_CK(cudaStreamSynchronize(stream));   // the host values above go out of scope
    }
    a.nextCount = counters;
    a.small = small;
    a.smallCount = counters + 1;
    int levelCount = n > SMALL_NODE ? 1 : 0, cur = 0;
    int hostCounters[2] = {0, 0};
    while (levelCount > 0) {
        a.tasks = big[cur];
        a.nextTasks = big[cur ^ 1];
        BB_CK(cudaMemsetAsync(counters, 0, sizeof(int), stream));
        k_split_large<<<levelCount, BIG_THREADS, 0, stream>>>(a);
        BB_CK(cudaMemcpyAsync(hostCounters, counters, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        BB_CK(cudaStreamSynchronize(stream));
        levelCount = hostCounters[0];
        cur ^= 1;
    }
    tm.mark("tree (large)");
    BB_CK(cudaMemcpyAsync(hostCounters, counters, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    if (hostCounters[1] > 0) k_split_small<<<blocksFor(hostCounters[1], 64), 64, 0, stream>>>(a, hostCounters[1]);
    BB_CK(cudaGetLastError());
    tm.mark("tree (small)");

    // ---- 4. post passes
    GpuBlasNode hRoot;
    BB_CK(cudaMemcpyAsync(&hRoot, a.nodes + 1, sizeof(hRoot), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    const bool rootLeaf = hRoot.TriCount > 0;
    if (rootLeaf) k_root_duplicate<<<1, 1, 0, stream>>>(a.nodes, a.parent, a.depth, a.ostart, a.ocount, n);

    int *g, *arrive;
    BB_CK(ar.get(g, cap));
    BB_CK(ar.get(arrive, cap));
    BB_CK(cudaMemsetAsync(arrive, 0, (size_t)cap * sizeof(int), stream));
    k_stack_size<<<blocksFor(cap, 256), 256, 0, stream>>>(a.nodes, a.parent, a.depth, cap, g, arrive);
    int requiredStackSize = 0;
    BB_CK(cudaMemcpyAsync(&requiredStackSize, g + 1, 4, cudaMemcpyDeviceToHost, stream));

    // pre-order of every node of the built tree
    int* order;
    int m = 0;
    BB_CK(ar.get(order, cap));
    if (rootLeaf) {
        k_preorder_root_duplicate<<<1, 1, 0, stream>>>(order);
        m = 3;
    } else {
        int *dmin, *dleaf, *len, *base;
        BB_CK(ar.get(dmin, n));
        BB_CK(ar.get(dleaf, n));
        BB_CK(ar.get(len, n + 1));
        BB_CK(ar.get(base, n + 1));
        BB_CK(cudaMemsetAsync(dmin, 0x7F, (size_t)n * sizeof(int), stream));   // DEPTH_NONE
        k_chain_ends<<<blocksFor(cap, 256), 256, 0, stream>>>(a.nodes, a.depth, a.ostart, cap, dmin, dleaf);
        k_chain_len<<<blocksFor(n, 256), 256, 0, stream>>>(dmin, dleaf, n, len);
        BB_CK(cudaMemsetAsync(len + n, 0, sizeof(int), stream));
        size_t need = 0;
        BB_CK(cub::DeviceScan::ExclusiveSum(nullptr, need, len, base, n + 1, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceScan::ExclusiveSum(cubTemp, need, len, base, n + 1, stream));
        k_preorder<<<blocksFor(cap, 256), 256, 0, stream>>>(a.depth, a.ostart, cap, dmin, base, order);
        BB_CK(cudaMemcpyAsync(&m, base + n, 4, cudaMemcpyDeviceToHost, stream));
    }
    BB_CK(cudaStreamSynchronize(stream));
    tm.mark("stack size");

    double* terms;
    double* acc;   // [0]: SAH of the built tree, [1]: added collapse cost, [2]: final SAH
    double* packed;
    uint8_t* flags;
    int* selCount;
    BB_CK(ar.get(terms, cap));
    BB_CK(ar.get(packed, cap));
    BB_CK(keep.get(acc, 3));
    BB_CK(ar.get(flags, cap));
    BB_CK(ar.get(selCount, 1));
    BB_CK(cudaMemsetAsync(acc, 0, 3 * sizeof(double), stream));
    auto flaggedSum = [&](double* dst) -> int {   // dst += the flagged terms, in order
        size_t need = 0;
        BB_CK(cub::DeviceSelect::Flagged(nullptr, need, terms, flags, packed, selCount, m, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceSelect::Flagged(cubTemp, need, terms, flags, packed, selCount, m, stream));
        k_ordered_sum<double, 4096><<<1, SUM_THREADS, 0, stream>>>(packed, 0, selCount, dst);
        return BB_OK;
    };

    // OptimizeStackSize
    int maxDepth = INT_MAX;   // nodes deeper than this are gone after the collapse passes
    if (requiredStackSize >= p.stackOptThreshold) {
        k_sah_terms<<<blocksFor(m, 256), 256, 0, stream>>>(order, m, a.nodes, nullptr, nullptr, p.triangleCost, terms);
        k_ordered_sum<double, 4096><<<1, SUM_THREADS, 0, stream>>>(terms, m, nullptr, acc + 0);
        k_collapse_terms<<<blocksFor(m, 256), 256, 0, stream>>>(order, m, a.nodes, a.depth, a.ocount, requiredStackSize - 1, 1,
                                                                 p.triangleCost, terms, flags);
        if (int rc = flaggedSum(acc + 1)) return rc;
        double h[2];
        BB_CK(cudaMemcpyAsync(h, acc, sizeof(h), cudaMemcpyDeviceToHost, stream));
        BB_CK(cudaStreamSynchronize(stream));
        // (no collapse of at most 2^24 fragments exceeds STACK_OPT_MAX_LEAF_TRIANGLE_COUNT, so that test is not made here)
        double increasePercent = h[1] / h[0];
        while (increasePercent <= (double)p.stackOptSahIncreaseAcceptance && requiredStackSize > 0) {
            const int level = --requiredStackSize;
            maxDepth = level + 1;
            k_collapse_terms<<<blocksFor(m, 256), 256, 0, stream>>>(order, m, a.nodes, a.depth, a.ocount, level, 0,
                                                                     p.triangleCost, terms, flags);
            if (int rc = flaggedSum(acc + 1)) return rc;
            BB_CK(cudaMemcpyAsync(h, acc, sizeof(h), cudaMemcpyDeviceToHost, stream));
            BB_CK(cudaStreamSynchronize(stream));
            increasePercent = h[1] / h[0];
        }
    }
    tm.mark("stack opt");

    // removeEmptySubtrees: the nodes left after the collapse, in pre-order
    int* order2 = order;
    int m2 = m;
    if (maxDepth != INT_MAX) {
        BB_CK(ar.get(order2, m));
        k_reachable<<<blocksFor(m, 256), 256, 0, stream>>>(order, m, a.depth, maxDepth, flags);
        size_t need = 0;
        BB_CK(cub::DeviceSelect::Flagged(nullptr, need, order, flags, order2, selCount, m, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceSelect::Flagged(cubTemp, need, order, flags, order2, selCount, m, stream));
        BB_CK(cudaMemcpyAsync(&m2, selCount, 4, cudaMemcpyDeviceToHost, stream));
        BB_CK(cudaStreamSynchronize(stream));
    }
    int *innerFlag, *innerScan, *rankOf, *fidx;
    BB_CK(ar.get(innerFlag, m2 + 1));
    BB_CK(ar.get(innerScan, m2 + 1));
    BB_CK(ar.get(rankOf, cap));
    BB_CK(ar.get(fidx, cap));
    k_inner_flags<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, a.nodes, a.depth, maxDepth, innerFlag);
    BB_CK(cudaMemsetAsync(innerFlag + m2, 0, sizeof(int), stream));
    {
        size_t need = 0;
        BB_CK(cub::DeviceScan::ExclusiveSum(nullptr, need, innerFlag, innerScan, m2 + 1, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceScan::ExclusiveSum(cubTemp, need, innerFlag, innerScan, m2 + 1, stream));
    }
    int inner = 0;
    BB_CK(cudaMemcpyAsync(&inner, innerScan + m2, 4, cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    k_inner_ranks<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, innerScan, rankOf);
    const int f = 2 + 2 * inner;
    GpuBlasNode* final;
    BB_CK(keep.get(final, f));
    BB_CK(cudaMemsetAsync(final, 0, sizeof(GpuBlasNode) * 2, stream));
    k_final_nodes<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, a.nodes, a.parent, a.depth, a.ostart, a.ocount, rankOf,
                                                          maxDepth, final, fidx);
    tm.mark("compact");

    // unindexing
    GpuBlasTriangle* outTris;
    BB_CK(keep.get(outTris, n));
    int triOut = n;
    if (!p.doPreSplit) {
        int *cnt, *off;
        BB_CK(ar.get(cnt, f));
        BB_CK(ar.get(off, f));
        k_leaf_counts<<<blocksFor(f, 256), 256, 0, stream>>>(final, f, cnt);
        size_t need = 0;
        BB_CK(cub::DeviceScan::ExclusiveSum(nullptr, need, cnt, off, f, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceScan::ExclusiveSum(cubTemp, need, cnt, off, f, stream));
        k_unindex_plain<<<blocksFor(f, 256), 256, 0, stream>>>(final, f, off, a.ids[0], tris, outTris, n);
    } else {
        int *marks, *segStart, *sizes, *off;
        unsigned long long *keys, *keysSorted;
        BB_CK(ar.get(marks, n));
        BB_CK(ar.get(segStart, n));
        BB_CK(ar.get(keys, n));
        BB_CK(ar.get(keysSorted, n));
        BB_CK(ar.get(sizes, inner + 1));
        BB_CK(ar.get(off, inner + 1));
        BB_CK(cudaMemsetAsync(marks, 0, (size_t)n * sizeof(int), stream));
        k_leaf_marks<<<blocksFor(f, 256), 256, 0, stream>>>(final, f, marks);
        size_t need = 0;
        BB_CK(cub::DeviceScan::InclusiveScan(nullptr, need, marks, segStart, MaxOp(), n, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceScan::InclusiveScan(cubTemp, need, marks, segStart, MaxOp(), n, stream));
        k_leaf_keys<<<blocksFor(n, 256), 256, 0, stream>>>(segStart, a.ids[0], origIds, n, keys);
        int endBit = 32;
        while ((1 << (endBit - 32)) < n && endBit < 64) endBit++;
        need = 0;
        BB_CK(cub::DeviceRadixSort::SortKeys(nullptr, need, keys, keysSorted, n, 0, endBit, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceRadixSort::SortKeys(cubTemp, need, keys, keysSorted, n, 0, endBit, stream));
        k_pair_sizes<<<blocksFor(inner + 1, 256), 256, 0, stream>>>(final, inner, keysSorted, sizes);
        need = 0;
        BB_CK(cub::DeviceScan::ExclusiveSum(nullptr, need, sizes, off, inner + 1, stream));
        BB_CK(cubScratch(need));
        BB_CK(cub::DeviceScan::ExclusiveSum(cubTemp, need, sizes, off, inner + 1, stream));
        k_pair_write<<<blocksFor(inner, 256), 256, 0, stream>>>(final, inner, keysSorted, off, tris, outTris);
        BB_CK(cudaMemcpyAsync(&triOut, off + inner, 4, cudaMemcpyDeviceToHost, stream));
    }
    tm.mark("unindex");

    k_sah_terms<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, nullptr, final, fidx, p.triangleCost, terms);
    k_ordered_sum<double, 4096><<<1, SUM_THREADS, 0, stream>>>(terms, m2, nullptr, acc + 2);
    tm.mark("sah");
    BB_CK(cudaGetLastError());
    BB_CK(cudaStreamSynchronize(stream));
    out.nodes = final;
    out.nodeCount = f;
    out.tris = outTris;
    out.triCount = triOut;
    out.requiredStackSize = requiredStackSize;
    out.fragmentCount = n;
    out.sah = acc + 2;
    return BB_OK;
}

// idkpt_blas_build: build_device between an upload of the host arrays and a download of its result. Fills `out` and the
// total device time.
static int build(cudaStream_t stream, const PackedVec3* hPos, uint64_t vertexCount, const GpuBlasTriangle* hTris, int triCount,
                 const Params& p, IdkPtBlasBuild& out, float& totalMs, std::string& err) {
    Arena ar;
    StageTimer tm(stream);
    tm.mark("start");
    PackedVec3* pos;
    GpuBlasTriangle* tris;
    BB_CK(ar.get(pos, vertexCount));
    BB_CK(ar.get(tris, triCount));
    BB_CK(cudaMemcpyAsync(pos, hPos, vertexCount * sizeof(PackedVec3), cudaMemcpyHostToDevice, stream));
    BB_CK(cudaMemcpyAsync(tris, hTris, (size_t)triCount * sizeof(GpuBlasTriangle), cudaMemcpyHostToDevice, stream));
    tm.mark("upload");
    DeviceResult r;
    if (int rc = build_device(stream, pos, tris, triCount, p, ar, r, tm, err)) return rc;

    out.nodes.resize(r.nodeCount);
    out.tris.resize(r.triCount);
    BB_CK(cudaMemcpyAsync(out.nodes.data(), r.nodes, (size_t)r.nodeCount * sizeof(GpuBlasNode), cudaMemcpyDeviceToHost, stream));
    if (r.triCount) BB_CK(cudaMemcpyAsync(out.tris.data(), r.tris, (size_t)r.triCount * sizeof(GpuBlasTriangle), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaMemcpyAsync(&out.sah, r.sah, sizeof(double), cudaMemcpyDeviceToHost, stream));
    tm.mark("download");
    BB_CK(cudaStreamSynchronize(stream));
    out.requiredStackSize = r.requiredStackSize;
    out.fragmentCount = r.fragmentCount;
    totalMs = tm.total();
    tm.print(r.fragmentCount);
    return BB_OK;
}

#undef BB_CK

}  // namespace idkbb
