// Scalar arithmetic of the BVH builders, shared by the host build (host_mirror/bvh_build.cpp) and the device build
// (idk_blas_build.cuh, k_tlas_build in idk_dynamic.cuh): boxes, triangle splits, one pre-split step, the serial SweepSAH
// split, the SAH and collapse cost terms, the TLAS Morton keys, and the build settings' defaults. The device build equals
// the host build node for node and SAH bit for bit because both run this code.
//
// Float semantics: C# does not contract a*b+c; only MyMath.HalfArea uses an explicit fused multiply-add. The host compiles
// this with g++ -ffp-contract=off, the device with nvcc -fmad=false; fmaf is used exactly where the reference fuses.
// Bit casts go through memcpy so that both compilers take the same source.
#ifndef IDK_BVH_MATH_H
#define IDK_BVH_MATH_H

#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/idk_gpu_types.h"
#include "idk_cbrt.h"

#if defined(__CUDACC__)
#define IDK_BVH_HD __host__ __device__ __forceinline__
#define IDK_BVH_UNROLL _Pragma("unroll")
#else
#define IDK_BVH_HD static inline
#define IDK_BVH_UNROLL _Pragma("GCC unroll 3")
#endif

namespace idkbvh {

// BLAS.BuildSettings (BLAS.cs:31-48) + PreSplitting.Settings (PreSplitting.cs:17-24), with the engine's defaults.
struct Params {
    int stopSplittingThreshold = 1;
    int maxLeafTriangleCount = 2;
    float triangleCost = 1.1f;
    int stackOptThreshold = 16;
    float stackOptSahIncreaseAcceptance = 0.0009745f;
    float splitFactor = 0.3f;
    int doPreSplit = 1;   // !IsRefittable (BVH.cs:324-333)
};
// BLAS.BuildSettings.StackOptMaxLeafTriangleCount: no collapse of at most 2^24 fragments exceeds it.
constexpr float STACK_OPT_MAX_LEAF_TRIANGLE_COUNT = (float)INT_MAX;

struct V3 { float v[3]; };
struct Tri { V3 p[3]; };
struct Box { float mn[3], mx[3]; };

IDK_BVH_HD uint32_t floatBits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
IDK_BVH_HD float bitsFloat(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// Vector128.MinNative / MaxNative on x86 (minps / maxps): (a < b) ? a : b. Folding a sequence with them keeps, among equal
// values, the last one (which matters for +-0), and the operation is associative, so a scan that combines (earlier, later)
// in order is exact.
IDK_BVH_HD float minN(float a, float b) { return a < b ? a : b; }
IDK_BVH_HD float maxN(float a, float b) { return a > b ? a : b; }

IDK_BVH_HD Box boxEmpty() { return {{FLT_MAX, FLT_MAX, FLT_MAX}, {-FLT_MAX, -FLT_MAX, -FLT_MAX}}; }
IDK_BVH_HD void grow(Box& b, const V3& p) {
    for (int i = 0; i < 3; i++) { b.mn[i] = minN(b.mn[i], p.v[i]); b.mx[i] = maxN(b.mx[i], p.v[i]); }
}
IDK_BVH_HD Box combine(const Box& a, const Box& b) {
    Box r;
    IDK_BVH_UNROLL   // without it g++ -O2 keeps r in memory, and the host's scans take twice as long
    for (int i = 0; i < 3; i++) { r.mn[i] = minN(a.mn[i], b.mn[i]); r.mx[i] = maxN(a.mx[i], b.mx[i]); }
    return r;
}
IDK_BVH_HD void clip(Box& b, const Box& to) {
    for (int i = 0; i < 3; i++) { b.mn[i] = maxN(b.mn[i], to.mn[i]); b.mx[i] = minN(b.mx[i], to.mx[i]); }
}
IDK_BVH_HD float boxSize(const Box& b, int i) { return b.mx[i] - b.mn[i]; }
IDK_BVH_HD int largestAxis(const Box& b) {
    int axis = 0;
    if (boxSize(b, 0) < boxSize(b, 1)) axis = 1;
    if (boxSize(b, axis) < boxSize(b, 2)) axis = 2;
    return axis;
}
IDK_BVH_HD float largestExtent(const Box& b) { return maxN(boxSize(b, 0), maxN(boxSize(b, 1), boxSize(b, 2))); }
IDK_BVH_HD float halfArea(const Box& b) {   // MyMath.HalfArea: fma(x + y, z, x * y)
    const float sx = b.mx[0] - b.mn[0], sy = b.mx[1] - b.mn[1], sz = b.mx[2] - b.mn[2];
    return fmaf(sx + sy, sz, sx * sy);
}
IDK_BVH_HD float nodeHalfArea(const GpuBlasNode& n) {
    const float sx = n.Max[0] - n.Min[0], sy = n.Max[1] - n.Min[1], sz = n.Max[2] - n.Min[2];
    return fmaf(sx + sy, sz, sx * sy);
}
IDK_BVH_HD void setBounds(GpuBlasNode& n, const Box& b) {
    for (int i = 0; i < 3; i++) { n.Min[i] = b.mn[i]; n.Max[i] = b.mx[i]; }
}
// Box i of an array of boxes: on the device as three 8-byte loads.
IDK_BVH_HD Box loadBox(const Box* b, int i) {
#if defined(__CUDA_ARCH__)
    const float2* p = reinterpret_cast<const float2*>(b + i);
    const float2 a = p[0], c = p[1], d = p[2];
    return {{a.x, a.y, c.x}, {c.y, d.x, d.y}};
#else
    return b[i];
#endif
}

IDK_BVH_HD Box boxFromTri(const Tri& t) {
    Box b = {{t.p[0].v[0], t.p[0].v[1], t.p[0].v[2]}, {t.p[0].v[0], t.p[0].v[1], t.p[0].v[2]}};
    grow(b, t.p[1]);
    grow(b, t.p[2]);
    return b;
}

// Algorithms.FloatToKey: an unsigned key in the float's order.
IDK_BVH_HD uint32_t floatToKey(float v) {
    const uint32_t f = floatBits(v);
    return f ^ (uint32_t)(((int32_t)f >> 31) | (int32_t)0x80000000);
}

// (int)float in C# on x86-64 (cvttss2si): NaN and out of range give INT_MIN.
IDK_BVH_HD int csFloatToInt(float f) {
    if (!(f > -2147483904.0f && f < 2147483648.0f)) return INT_MIN;
    return (int)f;
}

// ---------------------------------------------------------------------------------------------------------------- pre-split
// Triangle.Split (Shapes/Triangle.cs:47-92): the boxes of the triangle's parts on either side of `position` on `axis`.
IDK_BVH_HD void triSplit(const Tri& t, int axis, float position, Box& l, Box& r) {
    l = boxEmpty();
    r = boxEmpty();
    const bool q[3] = {t.p[0].v[axis] <= position, t.p[1].v[axis] <= position, t.p[2].v[axis] <= position};
    for (int k = 0; k < 3; k++) { if (q[k]) grow(l, t.p[k]); else grow(r, t.p[k]); }
    for (int k = 0; k < 3; k++) {
        const int k1 = (k + 1) % 3;
        if (q[k] ^ q[k1]) {
            const V3 a = t.p[k], b = t.p[k1];
            const float tt = (position - a.v[axis]) / (b.v[axis] - a.v[axis]);
            V3 m;
            for (int i = 0; i < 3; i++) m.v[i] = a.v[i] + tt * (b.v[i] - a.v[i]);
            grow(l, m);
            grow(r, m);
        }
    }
}

// PreSplitting.GetPriority. MathF.Cbrt is libm's cbrtf, which idk_cbrtf reproduces bit for bit.
IDK_BVH_HD float priority(const Tri& t) {
    const Box b = boxFromTri(t);
    const float le = largestExtent(b);
    const float extentPrio = le * le;
    float e1[3], e2[3];
    for (int i = 0; i < 3; i++) { e1[i] = t.p[1].v[i] - t.p[0].v[i]; e2[i] = t.p[2].v[i] - t.p[0].v[i]; }
    const float cx = e1[1] * e2[2] - e1[2] * e2[1], cy = e1[2] * e2[0] - e1[0] * e2[2], cz = e1[0] * e2[1] - e1[1] * e2[0];
    const float triArea = sqrtf(cx * cx + cy * cy + cz * cz) * 0.5f;
    const float emptyAreaPrio = halfArea(b) * 2.0f - triArea;
    return idk_cbrtf(extentPrio * emptyAreaPrio);
}

// PreSplitting.GetSplitCount: how many fragments a triangle becomes.
IDK_BVH_HD unsigned long long splitCount(float prio, float totalPrio, int triCount, float splitFactor) {
    const float shareOfTris = prio / totalPrio * (float)triCount;
    int c = csFloatToInt(shareOfTris * splitFactor);
    if (c == INT_MIN || c < 0) c = 0;   // guard for degenerate input; the reference would overflow
    return 1ull + (unsigned long long)c;
}

// PreSplitting.GetNodeSize: the power of two below extent / globalSize, times globalSize.
IDK_BVH_HD float nodeSize(float extent, float globalSize) {
    const float alpha = extent / globalSize;
    return bitsFloat(floatBits(alpha) & (255u << 23)) * globalSize;
}

// One step of PreSplit's loop (PreSplitting.cs:60-100): splits the item (`box`, `splits` > 1) of triangle `tri` at a grid
// position of the global box `g`. Returns the left part's split count; `l` and `r` are the clipped boxes of the two parts.
IDK_BVH_HD int presplitStep(const Tri& tri, const Box& box, int splits, const Box& g, Box& l, Box& r) {
    const int axis = largestAxis(box);
    const float le = largestExtent(box);
    float size = nodeSize(le, g.mx[axis] - g.mn[axis]);
    if (size >= le - 0.0001f) size *= 0.5f;
    const float midPos = (box.mn[axis] + box.mx[axis]) * 0.5f;
    const float index = rintf((midPos - g.mn[axis]) / size);   // MathF.Round: half to even
    const float splitPos = g.mn[axis] + index * size;
    triSplit(tri, axis, splitPos, l, r);
    clip(l, box);
    clip(r, box);
    const float leftExtent = largestExtent(l), rightExtent = largestExtent(r);
    int leftCount = csFloatToInt((float)splits * (leftExtent / (leftExtent + rightExtent)));
    leftCount = leftCount > 1 ? leftCount : 1;
    return leftCount < splits - 1 ? leftCount : splits - 1;
}

// ---------------------------------------------------------------------------------------------------------------- tree
// computeBoundingBox: boxEmpty() grown by the boxes of ids[lo, hi) in order.
IDK_BVH_HD Box rangeBox(const Box* bounds, const int* ids, int lo, int hi) {
    Box b = boxEmpty();
    for (int i = lo; i < hi; i++) b = combine(b, loadBox(bounds, ids[i]));
    return b;
}

// Algorithms.StablePartition: the ids whose table entry is set first, through `aux`; returns their count.
IDK_BVH_HD int stablePartition(int* source, int count, int* aux, const uint8_t* table) {
    int l = 0, r = 0;
    for (int i = 0; i < count; i++) {
        const int id = source[i];
        if (table[id]) source[l++] = id; else aux[r++] = id;
    }
    for (int i = 0; i < r; i++) source[l + i] = aux[i];
    return l;
}

// The end of BLAS.TrySplit after the sweep: a node whose costs were all non-finite takes the median split on axis 0 (the
// reference would index out of range); a node of at most maxLeafTriangleCount fragments stays a leaf when splitting
// costs more. Returns false for a leaf.
IDK_BVH_HD bool keepSplit(const Params& p, const Box& parentBox, int start, int count, float bestCost, int& bestAxis, int& bestSplit) {
    if (bestCost == FLT_MAX) { bestAxis = 0; bestSplit = start + count / 2; }
    if (count <= p.maxLeafTriangleCount) {
        const float notSplitCost = p.triangleCost * (float)count;
        const float newCost = 1.0f /*TRAVERSAL_COST*/ + (p.triangleCost * bestCost / halfArea(parentBox));
        if (newCost >= notSplitCost) return false;
    }
    return true;
}

// The larger child goes left: the two sides swap when the left one is smaller.
IDK_BVH_HD bool swapSides(const Box& left, const Box& right) { return halfArea(left) < halfArea(right); }

// BLAS.TrySplit (Bvh/BLAS.cs:730-873), serial, over the node's fragments [start, start + count) of the three sorted id
// arrays. `rcost` holds the right costs by fragment position, `table` one flag per fragment id, `aux` the partition's
// scratch by position. Returns the split index, or -1 for a leaf.
IDK_BVH_HD int trySplitSerial(const Box* bounds, int* const ids[3], float* rcost, uint8_t* table, int* aux, const Params& p,
                              const Box& parentBox, int start, int count) {
    if (count <= p.stopSplittingThreshold) return -1;
    const int end = start + count;
    float bestCost = FLT_MAX;
    int bestAxis = 0, bestSplit = 0;
    for (int axis = 0; axis < 3; axis++) {
        const int* axisIds = ids[axis];
        int firstRight = start + 1;
        Box rightAcc = boxEmpty();
        float rightCounter = 0.0f;
        for (int i = end - 1; i >= firstRight; i--) {
            rightCounter++;
            rightAcc = combine(rightAcc, loadBox(bounds, axisIds[i]));
            const float rightCost = halfArea(rightAcc) * rightCounter;
            rcost[i] = rightCost;
            if (rightCost >= bestCost) { firstRight = i + 1; break; }
        }
        Box leftAcc = boxEmpty();
        float leftCounter = (float)(firstRight - start) - 1.0f;
        for (int i = start; i < firstRight - 1; i++) leftAcc = combine(leftAcc, loadBox(bounds, axisIds[i]));
        for (int i = firstRight - 1; i < end - 1; i++) {
            leftCounter++;
            leftAcc = combine(leftAcc, loadBox(bounds, axisIds[i]));
            const float leftCost = halfArea(leftAcc) * leftCounter;
            const float cost = leftCost + rcost[i + 1];
            if (cost < bestCost) { bestSplit = i + 1; bestAxis = axis; bestCost = cost; }
            else if (leftCost >= bestCost) break;
        }
    }
    if (!keepSplit(p, parentBox, start, count, bestCost, bestAxis, bestSplit)) return -1;
    int* splitIds = ids[bestAxis];
    const bool swap = swapSides(rangeBox(bounds, splitIds, start, bestSplit), rangeBox(bounds, splitIds, bestSplit, end));
    for (int i = start; i < bestSplit; i++) table[splitIds[i]] = !swap;
    for (int i = bestSplit; i < end; i++) table[splitIds[i]] = swap;
    aux += start;
    if (swap) bestSplit = start + stablePartition(splitIds + start, count, aux, table);
    stablePartition(ids[(bestAxis + 1) % 3] + start, count, aux, table);
    stablePartition(ids[(bestAxis + 2) % 3] + start, count, aux, table);
    return bestSplit;
}

// ---------------------------------------------------------------------------------------------------------------- post passes
// computeGlobalSAH's term of one node; rootArea is 1 / the root's half area. triangleCost * count is a float product in
// C#, then widened.
IDK_BVH_HD double sahTerm(const GpuBlasNode& n, double rootArea, float triangleCost) {
    const double prob = (double)nodeHalfArea(n) * rootArea;
    return n.TriCount > 0 ? (double)(triangleCost * (float)n.TriCount) * prob : 1.0 * prob;
}

// collapseDeepestLevel's added cost of turning `parent`, whose children l and r hold lc and rc fragments, into one leaf.
IDK_BVH_HD double collapseTerm(const GpuBlasNode& parent, const GpuBlasNode& l, const GpuBlasNode& r, int lc, int rc,
                               const GpuBlasNode& root, float triangleCost) {
    const double leavesCost = (double)triangleCost * ((double)lc * (double)nodeHalfArea(l) + (double)rc * (double)nodeHalfArea(r));
    const double newParentLeafCost = (double)triangleCost * (double)(lc + rc);
    return ((double)nodeHalfArea(parent) * (newParentLeafCost - 1.0) - leavesCost) / (double)nodeHalfArea(root);
}

// ---------------------------------------------------------------------------------------------------------------- TLAS
// MyMath.InsertTwoZerosAfterEachBit
IDK_BVH_HD uint32_t insertTwoZeros(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
// (uint)(f * 1024) as C# converts it on x86-64, clamped to 10 bits
IDK_BVH_HD uint32_t mortonQuantise(float f) {
    const float s = f * 1024.0f;
    const uint32_t u = s <= 0.0f ? 0u : (s >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)s);
    return u < 1023u ? u : 1023u;
}
// MyMath.GetMortonCode30 of a point in [0, 1]^3
IDK_BVH_HD uint32_t mortonKey(float x, float y, float z) {
    return (insertTwoZeros(mortonQuantise(x)) << 2) | (insertTwoZeros(mortonQuantise(y)) << 1) | insertTwoZeros(mortonQuantise(z));
}
// MyMath.MapToZeroOne (Remap onto [0, 1]); an empty range maps to 0
IDK_BVH_HD float mapToZeroOne(float v, float lo, float hi) {
    const float t = hi - lo;
    float m = (v - lo) / t * (1.0f - 0.0f) + 0.0f;
    if (t == 0.0f) m = 0.0f;
    return m;
}
// TLAS.Build's leaf key: the Morton code of the box centre, mapped into the global box
IDK_BVH_HD uint32_t centreKey(const Box& b, const Box& global) {
    float m[3];
    for (int a = 0; a < 3; a++) m[a] = mapToZeroOne((b.mx[a] + b.mn[a]) * 0.5f, global.mn[a], global.mx[a]);
    return mortonKey(m[0], m[1], m[2]);
}
// Box.Transformed (Shapes/Box.cs:166-175): the 8 corners through the rows of a 3x4 model matrix. OpenTK's Vector4 * Matrix4
// is x*Row0 + y*Row1 + z*Row2 + w*Row3, added left to right.
IDK_BVH_HD Box transformedBox(const Box& local, const float m[12]) {
    Box b = boxEmpty();
    for (int c = 0; c < 8; c++) {
        const float x = (c & 1) ? local.mx[0] : local.mn[0], y = (c & 2) ? local.mx[1] : local.mn[1], z = (c & 4) ? local.mx[2] : local.mn[2];
        V3 p;
        for (int k = 0; k < 3; k++) p.v[k] = ((x * m[4 * k] + y * m[4 * k + 1]) + z * m[4 * k + 2]) + 1.0f * m[4 * k + 3];
        grow(b, p);
    }
    return b;
}

}  // namespace idkbvh

#endif
