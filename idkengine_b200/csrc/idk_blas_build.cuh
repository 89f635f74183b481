// BLAS.Build + PreSplitting.PreSplit on the device (idkpt_blas_build): the engine's SweepSAH builder with pre-splitting,
// node for node equal to the host mirror (host_mirror/bvh_build.cpp) under libidkpt's flags (-fmad=false, IEEE div and
// sqrt; fmaf only in HalfArea, where the mirror uses it). DESIGN §8f.5 gives the stages and why each one is exact.
//
// The driver builds a batch of BLASes at once (idkpt_blas_build is a batch of one): each BLAS owns its own ranges of
// fragment positions and node ids, and every stage runs over the whole batch; each BLAS comes out as it would alone.
//
// Stages (the mirror's function in brackets):
//   1. pre-split [preSplit]: priorities per triangle; their float sum in triangle order by one thread; split counts and
//      their exclusive scan; each triangle splits into its own output range, using the range's tail as its stack.
//   2. sorts [radixSortFragments]: three stable sorts of fragment ids by (BLAS, floatToKey(min + max)) (CUB radix sort).
//   3. tree [processSubtree, trySplit]: level by level, one block per node above SMALL_NODE fragments (full prefix and
//      suffix box scans, first strict minimum of L[i] + R[i+1]), then one thread per remaining subtree (the mirror's serial
//      trySplit). Node ids do not depend on the order nodes are split in.
//   4. post passes [computeRequiredStackSize, optimizeStackSize, removeEmptySubtrees, unindex*, computeGlobalSAH]: parallel
//      except for the double sums, which one thread per BLAS adds in the mirror's DFS order.
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

// ---------------------------------------------------------------------------------------------------------------- batch
// A batch of B BLASes shares one set of arrays. BLAS s owns the concatenated input triangles [tri[s], tri[s + 1]) (its range
// of the caller's array starts at in[s]), the fragment positions [frag[s], frag[s + 1]), the node ids [node[s], node[s + 1])
// with its root at node[s] + 1, the pre-order positions [order[s], order[s + 1]) and the output nodes [final[s],
// final[s + 1]). Every range is non-empty, so each table is strictly ascending.
struct Segs {
    int B;
    const int* tri;
    const long long* in;
    const int* pre;        // DoPreSplit
    const int* frag;
    const int* node;
    const int* order;
    const int* final;
    const int* maxDepth;   // nodes deeper than this are gone after the collapse passes (INT_MAX: no pass collapsed)
    const int* level;      // the collapse round's level
    const int* pass;       // the collapse round: 0 retired, 1 first pass, 2 a later pass
};

// The segment holding x: the last s with starts[s] <= x.
__device__ __forceinline__ int segOf(const int* starts, int B, int x) {
    int lo = 0, hi = B;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (starts[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

template <class T>
__global__ void k_gather(const T* v, const int* idx, int n, T* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v[idx[i]];
}

// out[scan[j]] = v[j] for the flagged j (scan: the exclusive sum of the flags)
template <class T>
__global__ void k_pack(const T* v, const int* flags, const int* scan, int m, T* out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m && flags[j]) out[scan[j]] = v[j];
}

// ---------------------------------------------------------------------------------------------------------------- pre-split
__device__ __forceinline__ Tri loadTri(const PackedVec3* pos, const GpuBlasTriangle* tris, int i) {
    const GpuBlasTriangle t = tris[i];
    const int id[3] = {t.X, t.Y, t.Z};
    Tri r;
    for (int k = 0; k < 3; k++) { const PackedVec3 q = pos[(uint32_t)id[k]]; r.p[k] = {{q.x, q.y, q.z}}; }
    return r;
}

__global__ void k_priorities(const PackedVec3* pos, const GpuBlasTriangle* tris, Segs sg, int n, float* prio) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = segOf(sg.tri, sg.B, i);
    if (sg.pre[s]) prio[i] = priority(loadTri(pos, tris + sg.in[s], i - sg.tri[s]));
}

// Ordered sums, one block per segment [begin[b], begin[b + 1]) (through `remap` when given): one thread adds the values
// in index order onto acc[b], as the mirror does (float addition is not associative). Blocks whose `active` entry is 0 do
// nothing. The block stages tiles through shared memory so that the one adding thread reads nothing from HBM itself.
constexpr int SUM_THREADS = 1024;
template <class T, int TILE>
__global__ void __launch_bounds__(SUM_THREADS) k_ordered_sum(const T* v, const int* begin, const int* remap, const int* active, T* acc) {
    __shared__ T tile[TILE];
    const int b = blockIdx.x;
    if (active && !active[b]) return;
    int lo = begin[b], hi = begin[b + 1];
    if (remap) { lo = remap[lo]; hi = remap[hi]; }
    T s = threadIdx.x == 0 ? acc[b] : T(0);
    for (int base = lo; base < hi; base += TILE) {
        const int m = min(TILE, hi - base);
        for (int k = threadIdx.x; k < m; k += SUM_THREADS) tile[k] = v[base + k];
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll 8
            for (int k = 0; k < m; k++) s += tile[k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) acc[b] = s;
}

// Fragments per triangle: its split count in a pre-split BLAS, 1 in the others. counts[n] = 0 ends the scan.
__global__ void k_split_counts(const float* prio, const float* total, Segs sg, int n, float splitFactor, unsigned long long* counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { counts[n] = 0; return; }
    const int s = segOf(sg.tri, sg.B, i);
    counts[i] = sg.pre[s] ? splitCount(prio[i], total[s], sg.tri[s + 1] - sg.tri[s], splitFactor) : 1ull;
}

// Box of every vertex of a pre-split BLAS in triangle order (p0, p1, p2 of each), one block per BLAS: per-thread chunks
// folded in order, chunks combined in order.
__global__ void __launch_bounds__(1024) k_global_box(const PackedVec3* pos, const GpuBlasTriangle* tris, Segs sg, Box* out) {
    __shared__ Box part[1024];
    __shared__ int has[1024];
    const int s = blockIdx.x;
    if (!sg.pre[s]) return;
    const GpuBlasTriangle* t0 = tris + sg.in[s];
    const int n = sg.tri[s + 1] - sg.tri[s];
    const int per = (n + 1023) / 1024;
    const int b0 = min(n, threadIdx.x * per), e0 = min(n, b0 + per);
    Box acc = boxIdentity();
    for (int i = b0; i < e0; i++) {
        const Tri t = loadTri(pos, t0, i);
        for (int k = 0; k < 3; k++) { Box p = {{t.p[k].v[0], t.p[k].v[1], t.p[k].v[2]}, {t.p[k].v[0], t.p[k].v[1], t.p[k].v[2]}}; acc = combine(acc, p); }
    }
    part[threadIdx.x] = acc;
    has[threadIdx.x] = e0 > b0;
    __syncthreads();
    if (threadIdx.x == 0) {
        Box g = boxEmpty();
        for (int t = 0; t < 1024; t++) if (has[t]) g = combine(g, part[t]);
        out[s] = g;
    }
}

// One thread per triangle, writing its fragments to [off[i], off[i+1]). The split stack lives in the same range, growing
// down from its end: the stack's items hold at least one fragment each and together exactly the ones not yet written, so
// they never reach the slot the next fragment goes to. Item j: box in bounds[end-1-j], split count in ids[end-1-j].
// A triangle of one fragment (every triangle of a BLAS that is not pre-split) writes its own box. origIds are BLAS-local.
__global__ void k_presplit(const PackedVec3* pos, const GpuBlasTriangle* tris, Segs sg, int n, const unsigned long long* off,
                           const Box* globalBox, Box* bounds, int* origIds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = segOf(sg.tri, sg.B, i);
    const int local = i - sg.tri[s];
    const Tri tri = loadTri(pos, tris + sg.in[s], local);
    const size_t begin = (size_t)off[i], end = (size_t)off[i + 1];
    if (end - begin == 1) {
        storeBox(bounds, begin, boxFromTri(tri));
        origIds[begin] = local;
        return;
    }
    const Box g = globalBox[s];
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
            origIds[counter] = local;
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

__global__ void k_sort_keys(const Box* bounds, int n, int axis, uint32_t* keys, int* vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Box b = loadBox(bounds, i);
    keys[i] = floatToKey(b.mn[axis] + b.mx[axis]);
    vals[i] = i;
}
// the BLAS of each fragment id, for the second (stable) sort pass
__global__ void k_seg_keys(const int* ids, int n, Segs sg, uint32_t* keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keys[i] = (uint32_t)segOf(sg.frag, sg.B, ids[i]);
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
// One thread per BLAS: seeds its root (node[s] + 1 over its fragments) as a task of the first level or as a small subtree.
// A root's parent is -1.
__global__ void k_seed_roots(TreeArgs a, Segs sg) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sg.B) return;
    const int r = sg.node[s] + 1, start = sg.frag[s], count = sg.frag[s + 1] - start;
    GpuBlasNode root = {};
    root.TriStartOrChild = start;
    root.TriCount = count;
    a.nodes[r] = root;
    a.parent[r] = -1;
    a.depth[r] = 0;
    a.ostart[r] = start;
    a.ocount[r] = count;
    pushTask(a, make_int2(r, r + 1), count);
}

// A root that stayed a leaf becomes an inner node over two copies of itself (BLAS.Build's leaf-root case).
__global__ void k_root_duplicate(GpuBlasNode* nodes, int* parent, int* depth, int* ostart, int* ocount, Segs sg) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sg.B) return;
    const int r = sg.node[s] + 1;
    GpuBlasNode root = nodes[r];
    if (!(root.TriCount > 0)) return;
    nodes[r + 1] = root;
    nodes[r + 2] = root;
    root.TriStartOrChild = r + 1;
    root.TriCount = 0;
    nodes[r] = root;
    for (int k = r + 1; k < r + 3; k++) { parent[k] = r; depth[k] = 1; ostart[k] = sg.frag[s]; ocount[k] = sg.frag[s + 1] - sg.frag[s]; }
}
// The second copy of a duplicated leaf root: the only right child that starts where its parent starts.
__device__ __forceinline__ bool rootCopy(const GpuBlasNode* nodes, const int* parent, const int* ostart, int v) {
    const int p = parent[v];
    return p >= 0 && v == nodes[p].TriStartOrChild + 1 && ostart[v] == ostart[p];
}

// computeRequiredStackSize, bottom up: g(v) = 0 if both children of v are leaves, g(inner child) if one is, and
// max(g(l), g(r)) + 1 if both are. Each climb starts at a node with two leaf children; at a node with two inner children
// the second arrival continues.
__global__ void k_stack_size(const GpuBlasNode* nodes, const int* parent, const int* depth, int cap, int* g, int* arrive) {
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= cap || depth[v] < 0 || nodes[v].TriCount > 0) return;
    const int c0 = nodes[v].TriStartOrChild;
    if (!(nodes[c0].TriCount > 0 && nodes[c0 + 1].TriCount > 0)) return;
    int gv = 0;
    g[v] = 0;
    for (;;) {
        const int p = parent[v];
        if (p < 0) return;
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
// highest one (dmin) down to a leaf (dleaf); pre-order lists the chains by s, and so the BLASes of a batch one after
// another. rank = base[s] + depth - dmin[s]. A duplicated leaf root's second copy comes after the first: one more rank.
__global__ void k_chain_ends(const GpuBlasNode* nodes, const int* parent, const int* depth, const int* ostart, int cap, int* dmin, int* dleaf) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= cap || depth[v] < 0) return;
    atomicMin(&dmin[ostart[v]], depth[v]);
    if (nodes[v].TriCount > 0) atomicMax(&dleaf[ostart[v]], depth[v] + (rootCopy(nodes, parent, ostart, v) ? 1 : 0));
}
__global__ void k_chain_len(const int* dmin, const int* dleaf, int n, int* len) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) len[s] = dmin[s] == DEPTH_NONE ? 0 : dleaf[s] - dmin[s] + 1;
}
__global__ void k_preorder(const GpuBlasNode* nodes, const int* parent, const int* depth, const int* ostart, int cap, const int* dmin,
                           const int* base, int* order) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= cap || depth[v] < 0) return;
    const int s = ostart[v];
    order[base[s] + depth[v] - dmin[s] + (rootCopy(nodes, parent, ostart, v) ? 1 : 0)] = v;
}

// Per BLAS: its first pre-order position (s <= B) and its RequiredStackSize (s < B).
__global__ void k_order_info(const int* base, const int* g, Segs sg, int* orderStart, int* stackSize) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s > sg.B) return;
    orderStart[s] = base[sg.frag[s]];
    if (s < sg.B) stackSize[s] = g[sg.node[s] + 1];
}

// computeGlobalSAH terms in pre-order: of the built tree (final == nullptr) or of the compacted one.
__global__ void k_sah_terms(const int* order, int m, Segs sg, const GpuBlasNode* nodes, const GpuBlasNode* final, const int* fidx,
                            float triangleCost, double* terms) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int s = segOf(sg.order, sg.B, j);
    const int v = order[j];
    const GpuBlasNode n = final ? final[fidx[v]] : nodes[v];
    const GpuBlasNode root = final ? final[sg.final[s] + 1] : nodes[sg.node[s] + 1];
    terms[j] = sahTerm(n, 1.0 / (double)nodeHalfArea(root), triangleCost);
}

// collapseDeepestLevel's cost terms, in pre-order (the nodes that add one never contain each other, so this is also the
// mirror's post-order among them), for the BLASes still in the collapse rounds. First pass: inner nodes deeper than
// `level` whose children are both leaves. Later passes: inner nodes at depth `level`, whose children are leaves after the
// pass's collapse and hold their whole subtrees.
__global__ void k_collapse_terms(const int* order, int m, Segs sg, const GpuBlasNode* nodes, const int* depth, const int* ocount,
                                 float triangleCost, double* terms, int* flags) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > m) return;
    if (j == m) { flags[m] = 0; return; }
    const int s = segOf(sg.order, sg.B, j);
    const int pass = sg.pass[s], level = sg.level[s];
    const int v = order[j];
    const GpuBlasNode n = nodes[v];
    bool q = false;
    if (pass && !(n.TriCount > 0)) {
        const int c = n.TriStartOrChild;
        q = pass == 1 ? (depth[v] > level && nodes[c].TriCount > 0 && nodes[c + 1].TriCount > 0) : depth[v] == level;
        if (q) terms[j] = collapseTerm(n, nodes[c], nodes[c + 1], ocount[c], ocount[c + 1], nodes[sg.node[s] + 1], triangleCost);
    }
    flags[j] = q;
}

__global__ void k_reachable(const int* order, int m, Segs sg, const int* depth, int* flags) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) flags[j] = depth[order[j]] <= sg.maxDepth[segOf(sg.order, sg.B, j)];
    if (j == m) flags[m] = 0;
}

// After the collapse passes a node is inner if it was split and is shallower than the collapsed level.
__global__ void k_inner_flags(const int* order, int m, Segs sg, const GpuBlasNode* nodes, const int* depth, int* flags) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == m) flags[m] = 0;
    if (j >= m) return;
    const int v = order[j];
    flags[j] = !(nodes[v].TriCount > 0) && depth[v] < sg.maxDepth[segOf(sg.order, sg.B, j)];
}
// BLAS-local pre-order ranks of the inner nodes
__global__ void k_inner_ranks(const int* order, int m, Segs sg, const int* scan, int* rankOf) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) rankOf[order[j]] = scan[j] - scan[sg.order[segOf(sg.order, sg.B, j)]];
}

// removeEmptySubtrees: the children of the inner node of pre-order rank k land at 2 + 2k of the BLAS's output range, whose
// node 0 is zero. Leaves keep their absolute fragment range until the unindexing.
__global__ void k_final_nodes(const int* order, int m, Segs sg, const GpuBlasNode* nodes, const int* parent, const int* depth,
                              const int* ostart, const int* ocount, const int* rankOf, GpuBlasNode* final, int* fidx) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int s = segOf(sg.order, sg.B, j);
    const int v = order[j], o = sg.final[s];
    int fi = 1;
    const int p = parent[v];
    if (p >= 0) fi = 2 + 2 * rankOf[p] + (v == nodes[p].TriStartOrChild + 1 ? 1 : 0);
    else final[o] = GpuBlasNode{};
    fidx[v] = o + fi;
    GpuBlasNode out = nodes[v];
    if (!(nodes[v].TriCount > 0) && depth[v] < sg.maxDepth[s]) { out.TriStartOrChild = 2 + 2 * rankOf[v]; out.TriCount = 0; }
    else { out.TriStartOrChild = ostart[v]; out.TriCount = ocount[v]; }
    final[o + fi] = out;
}

// PreSplitting.GetUnindexedTriangles: per leaf the sorted unique triangle ids, from one sort of (leaf start, triangle id)
__global__ void k_leaf_marks(const GpuBlasNode* final, int f, Segs sg, int* marks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < f && i - sg.final[segOf(sg.final, sg.B, i)] >= 2 && final[i].TriCount > 0) marks[final[i].TriStartOrChild] = final[i].TriStartOrChild;
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

// Output triangles per output node (counts[f] = 0 ends the scan). BLAS.GetUnindexedTriangles (not pre-split): each leaf's
// fragments, which are its triangles. When the root is a leaf, its two copies list all n each, and the second one's
// triangles would land past the end: the mirror writes them beyond its n-element array (heap overflow), so what it returns
// is the first copy's n triangles and the second leaf's offset n; the second copy counts none here. Pre-split: the left
// node of each sibling pair counts the pair's unique triangles.
__global__ void k_tri_counts(const GpuBlasNode* final, int f, Segs sg, const unsigned long long* keys, int* counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > f) return;
    if (i == f) { counts[f] = 0; return; }
    const int s = segOf(sg.final, sg.B, i), li = i - sg.final[s];
    int c = 0;
    if (li >= 2 && !sg.pre[s]) {
        const GpuBlasNode n = final[i];
        if (n.TriCount > 0 && !(li == 3 && final[i - 1].TriCount > 0 && final[i - 1].TriStartOrChild == n.TriStartOrChild)) c = n.TriCount;
    } else if (li >= 2 && !(li & 1)) {
        const GpuBlasNode l = final[i], r = final[i + 1];
        const bool ll = l.TriCount > 0, rl = r.TriCount > 0;
        if (ll && rl) c = uniqueCount(keys, l) + uniqueCount(keys, r) - sharedCount(keys, l, r);
        else if (ll) c = uniqueCount(keys, l);
        else if (rl) c = uniqueCount(keys, r);
    }
    counts[i] = c;
}

// Writes each output node's triangles at offsets[i] and makes leaf ranges BLAS-local (offsets[final[s]] is the BLAS's first
// output triangle). `in` is the input array; a BLAS's fragments and origIds index its own range of it.
__global__ void k_unindex(GpuBlasNode* final, int f, Segs sg, const int* offsets, const int* ids0, const int* origIds,
                          const unsigned long long* keys, const GpuBlasTriangle* tris, GpuBlasTriangle* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f) return;
    const int s = segOf(sg.final, sg.B, i), li = i - sg.final[s];
    if (li < 2) return;
    const GpuBlasTriangle* in = tris + sg.in[s];
    const int first = offsets[sg.final[s]];
    const int counter = offsets[i];
    if (!sg.pre[s]) {
        if (!(final[i].TriCount > 0)) return;
        const int st = final[i].TriStartOrChild, c = final[i].TriCount, o = counter - first, n = sg.frag[s + 1] - sg.frag[s];
        for (int k = 0; k < c && o + k < n; k++) out[counter + k] = in[origIds[ids0[st + k]]];
        final[i].TriStartOrChild = o;
        return;
    }
    if (li & 1) return;
    GpuBlasNode& l = final[i];
    GpuBlasNode& r = final[i + 1];
    const bool ll = l.TriCount > 0, rl = r.TriCount > 0;
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
        l.TriStartOrChild = counter - first; l.TriCount = lu;
        r.TriStartOrChild = counter - first + onlyLeft; r.TriCount = ru;
    } else if (ll || rl) {
        GpuBlasNode& leaf = ll ? l : r;
        const GpuBlasNode Lf = leaf;
        int c = 0;
        for (Uniq u(keys, Lf); !u.done(); u.next()) out[counter + c++] = in[u.cur()];
        leaf.TriStartOrChild = counter - first;
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
// A finished build on the host: the BLASes' nodes and triangles one after another, and per BLAS its desc (NodeOffset,
// NodeCount, TriangleOffset, TriangleCount, RequiredStackSize; the rest as the caller's), fragment count and SAH.
struct IdkPtBlasBuild {
    std::vector<GpuBlasNode> nodes;
    std::vector<GpuBlasTriangle> tris;
    std::vector<GpuBlasDesc> descs;
    std::vector<int32_t> fragmentCounts;
    std::vector<double> sahs;
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
    void print(int blases, long long fragments) {
        if (!getenv("IDKPT_BLAS_TIMING")) return;
        for (size_t i = 1; i < marks.size(); i++) {
            float ms = 0.0f;
            cudaEventElapsedTime(&ms, marks[i - 1].second, marks[i].second);
            fprintf(stderr, "[idkpt_blas_build] %-14s %8.2f ms\n", marks[i].first, ms);
        }
        fprintf(stderr, "[idkpt_blas_build] %-14s %8.2f ms (%d BLASes, %lld fragments)\n", "total", total(), blases, fragments);
    }
};

template <class F> static inline int blocksFor(F n, int t) { return (int)((n + t - 1) / t); }

enum { BB_OK = 0, BB_CUDA = 1, BB_TOO_MANY_FRAGMENTS = 2, BB_TOO_MANY_NODES = 3 };

#define BB_CK(call)                                                                                     \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess) { err = std::string(#call) + ": " + cudaGetErrorString(e_); return BB_CUDA; } \
    } while (0)

// One BLAS of a batch: its triangles tris[offset, offset + count) of the caller's array, and whether it is pre-split.
struct Input {
    long long offset;
    int count;
    int preSplit;
};

// A batch's result on the device: the nodes and triangles of all BLASes one after another, in allocations of the caller's
// arena, and per BLAS its ranges and values.
struct DeviceResult {
    GpuBlasNode* nodes = nullptr;
    GpuBlasTriangle* tris = nullptr;
    std::vector<int> nodeStart, triStart;   // B + 1 each
    std::vector<int> requiredStackSize, fragmentCount;
    std::vector<double> sah;
};

// The node ids a batch of BLASes of these fragment counts needs, or -1 when they do not fit in int32.
template <class C> static long long nodeIdCount(const C& fragments, size_t B) {
    long long total = 0;
    for (size_t s = 0; s < B; s++) {
        total += std::max<long long>(2 * (long long)fragments[s], 4);
        if (total >= (1ll << 31)) return -1;
    }
    return total;
}

// Builds the BLASes `in` together on `stream` from device arrays (global vertex ids into `pos`); the arguments have been
// validated, except for the fragment limits that pre-splitting decides. Every BLAS comes out as it would alone: the stages
// run over the whole batch, with the per-BLAS tables of Segs. The result goes to `out`, in allocations of `keep`; the
// scratch is freed on return, after the stream has been waited for.
static int build_device(cudaStream_t stream, const PackedVec3* pos, const GpuBlasTriangle* tris, const std::vector<Input>& in,
                        const Params& p, Arena& keep, DeviceResult& out, StageTimer& tm, std::string& err) {
    Arena ar;
    const int B = (int)in.size();
    void* cubTemp = nullptr;
    size_t cubBytes = 0;
    auto cubScratch = [&](size_t need) -> cudaError_t {
        if (need <= cubBytes) return cudaSuccess;
        uint8_t* q;
        cudaError_t e = ar.get(q, need);
        if (e == cudaSuccess) { cubTemp = q; cubBytes = need; }
        return e;
    };
    auto exclusiveSum = [&](auto* src, auto* dst, int count) -> cudaError_t {
        size_t need = 0;
        cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, need, src, dst, count, stream);
        if (e == cudaSuccess) e = cubScratch(need);
        if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(cubTemp, need, src, dst, count, stream);
        return e;
    };

    // ---- the per-BLAS tables (host copies, uploaded as they become known)
    std::vector<int> hTri(B + 1), hPre(B), hFrag(B + 1), hNode(B + 1), hOrder(B + 1), hFinal(B + 1), hMaxDepth(B, INT_MAX),
        hLevel(B, 0), hPass(B, 0), hStack(B);
    std::vector<long long> hIn(B);
    bool anyPre = false;
    for (int s = 0; s < B; s++) {
        hTri[s + 1] = hTri[s] + in[s].count;
        hIn[s] = in[s].offset;
        hPre[s] = in[s].preSplit;
        anyPre |= in[s].preSplit != 0;
    }
    const int M = hTri[B];
    int *dTri, *dPre, *dFrag, *dNode, *dOrder, *dFinal, *dMaxDepth, *dLevel, *dPass;
    long long* dIn;
    BB_CK(ar.get(dTri, B + 1));
    BB_CK(ar.get(dPre, B));
    BB_CK(ar.get(dFrag, B + 1));
    BB_CK(ar.get(dNode, B + 1));
    BB_CK(ar.get(dOrder, B + 1));
    BB_CK(ar.get(dFinal, B + 1));
    BB_CK(ar.get(dMaxDepth, B));
    BB_CK(ar.get(dLevel, B));
    BB_CK(ar.get(dPass, B));
    BB_CK(ar.get(dIn, B));
    const Segs sg = {B, dTri, dIn, dPre, dFrag, dNode, dOrder, dFinal, dMaxDepth, dLevel, dPass};
    auto up = [&](int* d, const std::vector<int>& h) { return cudaMemcpyAsync(d, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, stream); };
    BB_CK(up(dTri, hTri));
    BB_CK(up(dPre, hPre));
    BB_CK(cudaMemcpyAsync(dIn, hIn.data(), B * sizeof(long long), cudaMemcpyHostToDevice, stream));

    // ---- 1. fragments: split counts (1 for a BLAS that is not pre-split), their scan, then the fragments themselves
    float *prio, *total;
    unsigned long long *counts, *offsets, *fragStart;
    Box* gbox;
    BB_CK(ar.get(counts, (size_t)M + 1));
    BB_CK(ar.get(offsets, (size_t)M + 1));
    BB_CK(ar.get(fragStart, B + 1));
    BB_CK(ar.get(total, B));
    BB_CK(ar.get(gbox, B));
    if (anyPre) {
        BB_CK(ar.get(prio, M));
        k_priorities<<<blocksFor(M, 256), 256, 0, stream>>>(pos, tris, sg, M, prio);
        tm.mark("priorities");
        BB_CK(cudaMemsetAsync(total, 0, B * sizeof(float), stream));
        k_ordered_sum<float, 8192><<<B, SUM_THREADS, 0, stream>>>(prio, dTri, nullptr, dPre, total);
        tm.mark("priority sum");
    } else {
        prio = nullptr;
    }
    k_split_counts<<<blocksFor(M + 1, 256), 256, 0, stream>>>(prio, total, sg, M, p.splitFactor, counts);
    BB_CK(exclusiveSum(counts, offsets, M + 1));
    k_gather<<<blocksFor(B + 1, 256), 256, 0, stream>>>(offsets, dTri, B + 1, fragStart);
    std::vector<unsigned long long> hFrag64(B + 1);
    BB_CK(cudaMemcpyAsync(hFrag64.data(), fragStart, (B + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    std::vector<unsigned long long> fragCount(B);
    for (int s = 0; s < B; s++) {
        fragCount[s] = hFrag64[s + 1] - hFrag64[s];
        if (fragCount[s] > (unsigned long long)MAX_FRAGMENTS) {
            err = "pre-splitting makes " + std::to_string(fragCount[s]) + " fragments of BLAS " + std::to_string(s) + ", more than 2^24";
            return BB_TOO_MANY_FRAGMENTS;
        }
    }
    const long long capTotal = nodeIdCount(fragCount, B);
    if (capTotal < 0) {
        err = "the batch's " + std::to_string(hFrag64[B]) + " fragments need 2^31 or more node ids";
        return BB_TOO_MANY_NODES;
    }
    const int n = (int)hFrag64[B];   // fragments of the whole batch
    const int cap = (int)capTotal;
    for (int s = 0; s < B; s++) {
        hFrag[s + 1] = (int)hFrag64[s + 1];
        hNode[s + 1] = hNode[s] + std::max(2 * (int)fragCount[s], 4);
    }
    BB_CK(up(dFrag, hFrag));
    BB_CK(up(dNode, hNode));
    Box* bounds;
    int* origIds;
    BB_CK(ar.get(bounds, n));
    BB_CK(ar.get(origIds, n));
    if (anyPre) k_global_box<<<B, 1024, 0, stream>>>(pos, tris, sg, gbox);
    k_presplit<<<blocksFor(M, 128), 128, 0, stream>>>(pos, tris, sg, M, offsets, gbox, bounds, origIds);
    tm.mark("split");

    // ---- 2. three stable sorts by (BLAS, centroid key): by the key, then (in a batch) stably by the BLAS
    TreeArgs a = {};
    {
        uint32_t *keys, *keysOut;
        int *vals, *byKey = nullptr;
        BB_CK(ar.get(keys, n));
        BB_CK(ar.get(keysOut, n));
        BB_CK(ar.get(vals, n));
        if (B > 1) BB_CK(ar.get(byKey, n));
        int segBits = 0;
        while ((1 << segBits) < B) segBits++;
        for (int axis = 0; axis < 3; axis++) {
            BB_CK(ar.get(a.ids[axis], n));
            int* first = B > 1 ? byKey : a.ids[axis];
            k_sort_keys<<<blocksFor(n, 256), 256, 0, stream>>>(bounds, n, axis, keys, vals);
            size_t need = 0;
            BB_CK(cub::DeviceRadixSort::SortPairs(nullptr, need, keys, keysOut, vals, first, n, 0, 32, stream));
            BB_CK(cubScratch(need));
            BB_CK(cub::DeviceRadixSort::SortPairs(cubTemp, need, keys, keysOut, vals, first, n, 0, 32, stream));
            if (B > 1) {
                k_seg_keys<<<blocksFor(n, 256), 256, 0, stream>>>(byKey, n, sg, keys);
                need = 0;
                BB_CK(cub::DeviceRadixSort::SortPairs(nullptr, need, keys, keysOut, byKey, a.ids[axis], n, 0, segBits, stream));
                BB_CK(cubScratch(need));
                BB_CK(cub::DeviceRadixSort::SortPairs(cubTemp, need, keys, keysOut, byKey, a.ids[axis], n, 0, segBits, stream));
            }
        }
    }
    tm.mark("sort");

    // ---- 3. tree: every BLAS's root is a task of the first level; the levels of all BLASes advance together
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
    a.nextCount = counters;
    a.small = small;
    a.smallCount = counters + 1;
    a.nextTasks = big[0];
    k_seed_roots<<<blocksFor(B, 128), 128, 0, stream>>>(a, sg);
    int levelCount = 0, cur = 0;
    for (int s = 0; s < B; s++) levelCount += fragCount[s] > (unsigned long long)SMALL_NODE;
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
    k_root_duplicate<<<blocksFor(B, 128), 128, 0, stream>>>(a.nodes, a.parent, a.depth, a.ostart, a.ocount, sg);
    int *g, *arrive;
    BB_CK(ar.get(g, cap));
    BB_CK(ar.get(arrive, cap));
    BB_CK(cudaMemsetAsync(arrive, 0, (size_t)cap * sizeof(int), stream));
    k_stack_size<<<blocksFor(cap, 256), 256, 0, stream>>>(a.nodes, a.parent, a.depth, cap, g, arrive);

    // pre-order of every node of the built trees, BLAS after BLAS
    int *order, *dmin, *dleaf, *len, *base, *dStack;
    BB_CK(ar.get(order, cap));
    BB_CK(ar.get(dmin, n));
    BB_CK(ar.get(dleaf, n));
    BB_CK(ar.get(len, n + 1));
    BB_CK(ar.get(base, n + 1));
    BB_CK(ar.get(dStack, B));
    BB_CK(cudaMemsetAsync(dmin, 0x7F, (size_t)n * sizeof(int), stream));   // DEPTH_NONE
    BB_CK(cudaMemsetAsync(dleaf, 0, (size_t)n * sizeof(int), stream));
    k_chain_ends<<<blocksFor(cap, 256), 256, 0, stream>>>(a.nodes, a.parent, a.depth, a.ostart, cap, dmin, dleaf);
    k_chain_len<<<blocksFor(n, 256), 256, 0, stream>>>(dmin, dleaf, n, len);
    BB_CK(cudaMemsetAsync(len + n, 0, sizeof(int), stream));
    BB_CK(exclusiveSum(len, base, n + 1));
    k_preorder<<<blocksFor(cap, 256), 256, 0, stream>>>(a.nodes, a.parent, a.depth, a.ostart, cap, dmin, base, order);
    k_order_info<<<blocksFor(B + 1, 256), 256, 0, stream>>>(base, g, sg, dOrder, dStack);
    BB_CK(cudaMemcpyAsync(hOrder.data(), dOrder, (B + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaMemcpyAsync(hStack.data(), dStack, B * sizeof(int), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    const int m = hOrder[B];
    tm.mark("stack size");

    double* terms;
    double* acc;   // per BLAS: [0, B) SAH of the built tree, [B, 2B) added collapse cost, [2B, 3B) final SAH
    double* packed;
    int *flags, *scan;
    BB_CK(ar.get(terms, cap));
    BB_CK(ar.get(packed, cap));
    BB_CK(ar.get(acc, 3 * (size_t)B));
    BB_CK(ar.get(flags, cap + 1));
    BB_CK(ar.get(scan, cap + 1));
    BB_CK(cudaMemsetAsync(acc, 0, 3 * (size_t)B * sizeof(double), stream));

    // OptimizeStackSize, in rounds: a BLAS whose RequiredStackSize reaches the threshold takes part from the first round,
    // which adds the first pass's collapse cost, and leaves the rounds when its next pass is not accepted. One host read
    // per round for the whole batch. (No collapse of at most 2^24 fragments exceeds STACK_OPT_MAX_LEAF_TRIANGLE_COUNT, so
    // that test is not made here.)
    bool collapsing = false, collapsed = false;
    for (int s = 0; s < B; s++) {
        if (hStack[s] >= p.stackOptThreshold) { hPass[s] = 1; hLevel[s] = hStack[s] - 1; collapsing = true; }
    }
    if (collapsing) {
        BB_CK(up(dPass, hPass));
        k_sah_terms<<<blocksFor(m, 256), 256, 0, stream>>>(order, m, sg, a.nodes, nullptr, nullptr, p.triangleCost, terms);
        k_ordered_sum<double, 4096><<<B, SUM_THREADS, 0, stream>>>(terms, dOrder, nullptr, dPass, acc);
    }
    std::vector<double> hAcc(2 * (size_t)B);
    while (collapsing) {
        BB_CK(up(dPass, hPass));
        BB_CK(up(dLevel, hLevel));
        k_collapse_terms<<<blocksFor(m + 1, 256), 256, 0, stream>>>(order, m, sg, a.nodes, a.depth, a.ocount, p.triangleCost, terms, flags);
        BB_CK(exclusiveSum(flags, scan, m + 1));
        k_pack<<<blocksFor(m, 256), 256, 0, stream>>>(terms, flags, scan, m, packed);
        k_ordered_sum<double, 4096><<<B, SUM_THREADS, 0, stream>>>(packed, dOrder, scan, dPass, acc + B);
        BB_CK(cudaMemcpyAsync(hAcc.data(), acc, hAcc.size() * sizeof(double), cudaMemcpyDeviceToHost, stream));
        BB_CK(cudaStreamSynchronize(stream));
        collapsing = false;
        for (int s = 0; s < B; s++) {
            if (!hPass[s]) continue;
            const double increasePercent = hAcc[B + s] / hAcc[s];
            if (increasePercent <= (double)p.stackOptSahIncreaseAcceptance && hStack[s] > 0) {
                hLevel[s] = --hStack[s];
                hMaxDepth[s] = hLevel[s] + 1;
                hPass[s] = 2;
                collapsing = collapsed = true;
            } else {
                hPass[s] = 0;
            }
        }
    }
    BB_CK(up(dMaxDepth, hMaxDepth));
    tm.mark("stack opt");

    // removeEmptySubtrees: the nodes left after the collapse, in pre-order
    int* order2 = order;
    int* dOrder2 = dOrder;
    std::vector<int> hOrder2 = hOrder;
    if (collapsed) {
        BB_CK(ar.get(order2, m));
        BB_CK(ar.get(dOrder2, B + 1));
        k_reachable<<<blocksFor(m + 1, 256), 256, 0, stream>>>(order, m, sg, a.depth, flags);
        BB_CK(exclusiveSum(flags, scan, m + 1));
        k_pack<<<blocksFor(m, 256), 256, 0, stream>>>(order, flags, scan, m, order2);
        k_gather<<<blocksFor(B + 1, 256), 256, 0, stream>>>(scan, dOrder, B + 1, dOrder2);
        BB_CK(cudaMemcpyAsync(hOrder2.data(), dOrder2, (B + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream));
        BB_CK(cudaStreamSynchronize(stream));
    }
    const int m2 = hOrder2[B];
    Segs sg2 = sg;
    sg2.order = dOrder2;
    int *rankOf, *fidx, *innerStart;
    BB_CK(ar.get(rankOf, cap));
    BB_CK(ar.get(fidx, cap));
    BB_CK(ar.get(innerStart, B + 1));
    k_inner_flags<<<blocksFor(m2 + 1, 256), 256, 0, stream>>>(order2, m2, sg2, a.nodes, a.depth, flags);
    BB_CK(exclusiveSum(flags, scan, m2 + 1));
    k_gather<<<blocksFor(B + 1, 256), 256, 0, stream>>>(scan, dOrder2, B + 1, innerStart);
    std::vector<int> hInner(B + 1);
    BB_CK(cudaMemcpyAsync(hInner.data(), innerStart, (B + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    k_inner_ranks<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, sg2, scan, rankOf);
    for (int s = 0; s < B; s++) hFinal[s + 1] = hFinal[s] + 2 + 2 * (hInner[s + 1] - hInner[s]);
    BB_CK(up(dFinal, hFinal));
    const int f = hFinal[B];
    GpuBlasNode* final;
    BB_CK(keep.get(final, f));
    k_final_nodes<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, sg2, a.nodes, a.parent, a.depth, a.ostart, a.ocount, rankOf, final, fidx);
    tm.mark("compact");

    // unindexing: per output node its triangle count, one scan, then the triangles
    unsigned long long* keysSorted = nullptr;
    if (anyPre) {
        int *marks, *segStart;
        unsigned long long* keys;
        BB_CK(ar.get(marks, n));
        BB_CK(ar.get(segStart, n));
        BB_CK(ar.get(keys, n));
        BB_CK(ar.get(keysSorted, n));
        BB_CK(cudaMemsetAsync(marks, 0, (size_t)n * sizeof(int), stream));
        k_leaf_marks<<<blocksFor(f, 256), 256, 0, stream>>>(final, f, sg2, marks);
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
    }
    int *cnt, *off, *triStart;
    BB_CK(ar.get(cnt, (size_t)f + 1));
    BB_CK(ar.get(off, (size_t)f + 1));
    BB_CK(ar.get(triStart, B + 1));
    k_tri_counts<<<blocksFor(f + 1, 256), 256, 0, stream>>>(final, f, sg2, keysSorted, cnt);
    BB_CK(exclusiveSum(cnt, off, f + 1));
    k_gather<<<blocksFor(B + 1, 256), 256, 0, stream>>>(off, dFinal, B + 1, triStart);
    out.triStart.assign(B + 1, 0);
    BB_CK(cudaMemcpyAsync(out.triStart.data(), triStart, (B + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream));
    BB_CK(cudaStreamSynchronize(stream));
    GpuBlasTriangle* outTris;
    BB_CK(keep.get(outTris, out.triStart[B]));
    k_unindex<<<blocksFor(f, 256), 256, 0, stream>>>(final, f, sg2, off, a.ids[0], origIds, keysSorted, tris, outTris);
    tm.mark("unindex");

    k_sah_terms<<<blocksFor(m2, 256), 256, 0, stream>>>(order2, m2, sg2, nullptr, final, fidx, p.triangleCost, terms);
    k_ordered_sum<double, 4096><<<B, SUM_THREADS, 0, stream>>>(terms, dOrder2, nullptr, nullptr, acc + 2 * B);
    out.sah.assign(B, 0.0);
    BB_CK(cudaMemcpyAsync(out.sah.data(), acc + 2 * B, B * sizeof(double), cudaMemcpyDeviceToHost, stream));
    tm.mark("sah");
    BB_CK(cudaGetLastError());
    BB_CK(cudaStreamSynchronize(stream));
    out.nodes = final;
    out.tris = outTris;
    out.nodeStart = hFinal;
    out.requiredStackSize = hStack;
    out.fragmentCount.resize(B);
    for (int s = 0; s < B; s++) out.fragmentCount[s] = (int)fragCount[s];
    return BB_OK;
}

// idkpt_blas_build and idkpt_blas_build_batch: build_device between an upload of the host arrays and a download of its
// result. Fills `out` (descs from `descs`, whose other fields are kept) and the total device time.
static int build(cudaStream_t stream, const PackedVec3* hPos, uint64_t vertexCount, const GpuBlasTriangle* hTris, uint64_t triCount,
                 const std::vector<Input>& in, const std::vector<GpuBlasDesc>& descs, const Params& p, IdkPtBlasBuild& out,
                 float& totalMs, std::string& err) {
    Arena ar;
    StageTimer tm(stream);
    tm.mark("start");
    PackedVec3* pos;
    GpuBlasTriangle* tris;
    BB_CK(ar.get(pos, vertexCount));
    BB_CK(ar.get(tris, triCount));
    BB_CK(cudaMemcpyAsync(pos, hPos, vertexCount * sizeof(PackedVec3), cudaMemcpyHostToDevice, stream));
    BB_CK(cudaMemcpyAsync(tris, hTris, triCount * sizeof(GpuBlasTriangle), cudaMemcpyHostToDevice, stream));
    tm.mark("upload");
    DeviceResult r;
    if (int rc = build_device(stream, pos, tris, in, p, ar, r, tm, err)) return rc;

    const size_t B = in.size();
    out.nodes.resize(r.nodeStart[B]);
    out.tris.resize(r.triStart[B]);
    BB_CK(cudaMemcpyAsync(out.nodes.data(), r.nodes, out.nodes.size() * sizeof(GpuBlasNode), cudaMemcpyDeviceToHost, stream));
    if (!out.tris.empty()) BB_CK(cudaMemcpyAsync(out.tris.data(), r.tris, out.tris.size() * sizeof(GpuBlasTriangle), cudaMemcpyDeviceToHost, stream));
    tm.mark("download");
    BB_CK(cudaStreamSynchronize(stream));
    out.descs = descs;
    for (size_t s = 0; s < B; s++) {
        GpuBlasDesc& d = out.descs[s];
        d.NodeOffset = r.nodeStart[s];
        d.NodeCount = r.nodeStart[s + 1] - r.nodeStart[s];
        d.TriangleOffset = r.triStart[s];
        d.TriangleCount = r.triStart[s + 1] - r.triStart[s];
        d.RequiredStackSize = r.requiredStackSize[s];
    }
    out.fragmentCounts = r.fragmentCount;
    out.sahs = r.sah;
    totalMs = tm.total();
    long long fragments = 0;
    for (int c : r.fragmentCount) fragments += c;
    tm.print((int)B, fragments);
    return BB_OK;
}

#undef BB_CK

}  // namespace idkbb
