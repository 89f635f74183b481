// Dynamic geometry (SURVEY.md 8f.2): vertex skinning and BLAS refit on the device, so that an animated scene never leaves HBM.
//   k_skin_vertices                  Skinning/compute.glsl:14-49 (ModelManager.ComputeSkinnedPositions, ModelManager.cs:263-280)
//   k_refit_prepare / k_refit_climb  BLASRefit/compute.glsl:14-49 (BVH.GpuBlasesRefit, BVH.cs:472-489); same boxes as BLAS.Refit (BLAS.cs:276-293)
// The reference keeps GetParentIndices / GetLeafIndices tables (BLAS.cs:481-515) in two SSBOs. Here the parent table is
// derived on the device from the node array itself (children always follow their parent) and the leaf list is replaced by
// "one thread per node, leaves start the climb": no host pre-pass, no extra upload.
#pragma once
#include "idk_kernels.cuh"
#include "idk_bvh_math.h"

__device__ __forceinline__ uint32_t compress_sr11g11b10(f3 v) {
    // CompressSR11G11B10 (Compression.glsl:1-28). GLSL leaves round()'s half-way case to the implementation; this and the
    // oracle both use floor(x + 0.5).
    const float x = v.x * 0.5f + 0.5f, y = v.y * 0.5f + 0.5f, z = v.z * 0.5f + 0.5f;
    const uint32_t r = (uint32_t)floorf(x * 2047.0f + 0.5f);
    const uint32_t g = (uint32_t)floorf(y * 2047.0f + 0.5f);
    const uint32_t b = (uint32_t)floorf(z * 1023.0f + 0.5f);
    return (b << 22) | (g << 11) | r;
}

struct SkinArgs {
    const uint32_t* unskinned;    // GpuUnskinnedVertex[], 13 words each
    const float4* joints;         // row_major mat4x3: 3 x float4 per joint
    float* positions;             // PackedVec3[]
    uint4* vertices;              // GpuVertex[]
    float4* vtxFrame;             // derived normal/tangent records (k_prepare_vertices)
    uint32_t inOffset, outOffset, jointOffset, count;
};

__global__ void __launch_bounds__(256) k_skin_vertices(SkinArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.count) return;
    const uint32_t* u = a.unskinned + 13 * (size_t)(a.inOffset + i);   // 52-byte records: scalar loads
    const uint32_t j[4] = {u[0], u[1], u[2], u[3]};
    const float w[4] = {__uint_as_float(u[4]), __uint_as_float(u[5]), __uint_as_float(u[6]), __uint_as_float(u[7])};
    const f3 position = mk3(__uint_as_float(u[8]), __uint_as_float(u[9]), __uint_as_float(u[10]));
    const uint32_t packedTangent = u[11], packedNormal = u[12];
    // skinMatrix = w.x * M[j.x] + w.y * M[j.y] + w.z * M[j.z] + w.w * M[j.w]: component-wise, left to right
    float4 rows[3];
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const float4 m0 = a.joints[3 * (size_t)(a.jointOffset + j[0]) + r];
        const float4 m1 = a.joints[3 * (size_t)(a.jointOffset + j[1]) + r];
        const float4 m2 = a.joints[3 * (size_t)(a.jointOffset + j[2]) + r];
        const float4 m3 = a.joints[3 * (size_t)(a.jointOffset + j[3]) + r];
        rows[r].x = ((w[0] * m0.x + w[1] * m1.x) + w[2] * m2.x) + w[3] * m3.x;
        rows[r].y = ((w[0] * m0.y + w[1] * m1.y) + w[2] * m2.y) + w[3] * m3.y;
        rows[r].z = ((w[0] * m0.z + w[1] * m1.z) + w[2] * m2.z) + w[3] * m3.z;
        rows[r].w = ((w[0] * m0.w + w[1] * m1.w) + w[2] * m2.w) + w[3] * m3.w;
    }
    const f3 tangent = decompress_sr11g11b10(packedTangent);
    const f3 normal = decompress_sr11g11b10(packedNormal);
    f3 p, n, t;
    p.x = ((rows[0].x * position.x + rows[0].y * position.y) + rows[0].z * position.z) + rows[0].w * 1.0f;
    p.y = ((rows[1].x * position.x + rows[1].y * position.y) + rows[1].z * position.z) + rows[1].w * 1.0f;
    p.z = ((rows[2].x * position.x + rows[2].y * position.y) + rows[2].z * position.z) + rows[2].w * 1.0f;
    n.x = (rows[0].x * normal.x + rows[0].y * normal.y) + rows[0].z * normal.z;
    n.y = (rows[1].x * normal.x + rows[1].y * normal.y) + rows[1].z * normal.z;
    n.z = (rows[2].x * normal.x + rows[2].y * normal.y) + rows[2].z * normal.z;
    t.x = (rows[0].x * tangent.x + rows[0].y * tangent.y) + rows[0].z * tangent.z;
    t.y = (rows[1].x * tangent.x + rows[1].y * tangent.y) + rows[1].z * tangent.z;
    t.z = (rows[2].x * tangent.x + rows[2].y * tangent.y) + rows[2].z * tangent.z;
    n = normalize3(n);
    t = normalize3(t);
    const size_t o = (size_t)a.outOffset + i;
    a.positions[3 * o] = p.x; a.positions[3 * o + 1] = p.y; a.positions[3 * o + 2] = p.z;
    uint4 v = a.vertices[o];
    v.z = compress_sr11g11b10(t);
    v.w = compress_sr11g11b10(n);
    a.vertices[o] = v;
    // the path tracer reads the decoded copy (same bits as decoding at every hit)
    const f3 dn = decompress_sr11g11b10(v.w), dt = decompress_sr11g11b10(v.z);
    a.vtxFrame[2 * o] = make_float4(dn.x, dn.y, dn.z, dt.x);
    a.vtxFrame[2 * o + 1] = make_float4(dt.y, dt.z, 0.0f, 0.0f);
}

struct RefitArgs {
    float4* nodes;               // this BLAS's nodes (2 x float4 each), BLAS-local indexing
    const int4* blasTris;        // global triangle array
    const float* positions;
    float4* triRec;              // global derived triangle records
    int32_t* parents;            // scratch, nodeCount entries
    uint32_t* locks;             // scratch, nodeCount entries
    uint32_t nodeCount, triOffset, triCount;
};

// GetParentIndices (BLAS.cs:481-498) on the device + blasRefitLockBuffer.Fill(0) (BVH.cs:478)
__global__ void __launch_bounds__(256) k_refit_prepare(RefitArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.nodeCount) return;
    a.locks[i] = 0u;
    if (i < 2) a.parents[i] = -1;
    if (i >= 1) {
        const int child = __float_as_int(a.nodes[2 * (size_t)i].w), count = __float_as_int(a.nodes[2 * (size_t)i + 1].w);
        if (count == 0) { a.parents[child] = (int)i; a.parents[child + 1] = (int)i; }
    }
}

// Leaves recompute their box from the (moved) vertices and climb; the second arrival at a parent merges its children.
// Also refreshes the leaf's derived triangle records (p0, e1, e2, n), which the reference recomputes at every ray/triangle test.
__global__ void __launch_bounds__(256) k_refit_climb(RefitArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    if (i >= a.nodeCount) return;
    const float4 nA = a.nodes[2 * (size_t)i], nB = a.nodes[2 * (size_t)i + 1];
    const int start = __float_as_int(nA.w), count = __float_as_int(nB.w);
    if (count <= 0) return;
    f3 lo = mk3(3.4028235e38f, 3.4028235e38f, 3.4028235e38f), hi = mk3(-3.4028235e38f, -3.4028235e38f, -3.4028235e38f);
    for (uint32_t k = a.triOffset + (uint32_t)start; k < a.triOffset + (uint32_t)start + (uint32_t)count; k++) {
        const int4 t = a.blasTris[k];
        const f3 p0 = mk3(a.positions[3 * (size_t)t.x], a.positions[3 * (size_t)t.x + 1], a.positions[3 * (size_t)t.x + 2]);
        const f3 p1 = mk3(a.positions[3 * (size_t)t.y], a.positions[3 * (size_t)t.y + 1], a.positions[3 * (size_t)t.y + 2]);
        const f3 p2 = mk3(a.positions[3 * (size_t)t.z], a.positions[3 * (size_t)t.z + 1], a.positions[3 * (size_t)t.z + 2]);
        lo = mk3(fminf(fminf(fminf(lo.x, p0.x), p1.x), p2.x), fminf(fminf(fminf(lo.y, p0.y), p1.y), p2.y), fminf(fminf(fminf(lo.z, p0.z), p1.z), p2.z));
        hi = mk3(fmaxf(fmaxf(fmaxf(hi.x, p0.x), p1.x), p2.x), fmaxf(fmaxf(fmaxf(hi.y, p0.y), p1.y), p2.y), fmaxf(fmaxf(fmaxf(hi.z, p0.z), p1.z), p2.z));
        const f3 e1 = p1 - p0, e2 = p2 - p0, n = cross3(e1, e2);
        a.triRec[4 * (size_t)k + 0] = make_float4(p0.x, p0.y, p0.z, e1.x);
        a.triRec[4 * (size_t)k + 1] = make_float4(e1.y, e1.z, e2.x, e2.y);
        a.triRec[4 * (size_t)k + 2] = make_float4(e2.z, n.x, n.y, n.z);
    }
    a.nodes[2 * (size_t)i] = make_float4(lo.x, lo.y, lo.z, nA.w);
    a.nodes[2 * (size_t)i + 1] = make_float4(hi.x, hi.y, hi.z, nB.w);
    int parent = a.parents[i];
    while (parent != -1) {
        __threadfence();                                   // publish this subtree's boxes before taking the ticket
        if (atomicExch(&a.locks[parent], 1u) == 0u) return; // first arrival: the sibling subtree is not refitted yet
        __threadfence();
        volatile float4* vn = (volatile float4*)a.nodes;
        const int child = __float_as_int(vn[2 * (size_t)parent].w);
        const float lAx = vn[2 * (size_t)child].x, lAy = vn[2 * (size_t)child].y, lAz = vn[2 * (size_t)child].z;
        const float lBx = vn[2 * (size_t)child + 1].x, lBy = vn[2 * (size_t)child + 1].y, lBz = vn[2 * (size_t)child + 1].z;
        const float rAx = vn[2 * (size_t)child + 2].x, rAy = vn[2 * (size_t)child + 2].y, rAz = vn[2 * (size_t)child + 2].z;
        const float rBx = vn[2 * (size_t)child + 3].x, rBy = vn[2 * (size_t)child + 3].y, rBz = vn[2 * (size_t)child + 3].z;
        vn[2 * (size_t)parent].x = fminf(lAx, rAx); vn[2 * (size_t)parent].y = fminf(lAy, rAy); vn[2 * (size_t)parent].z = fminf(lAz, rAz);
        vn[2 * (size_t)parent + 1].x = fmaxf(lBx, rBx); vn[2 * (size_t)parent + 1].y = fmaxf(lBy, rBy); vn[2 * (size_t)parent + 1].z = fmaxf(lBz, rBz);
        parent = a.parents[parent];
    }
}

// ------------------------------------------------------------------------------------------------ TLAS build on the device
// BVH.TlasBuild (BVH.cs:278-298) + TLAS.Build (TLAS.cs:28-141, the serial PLOC variant: Morton-ordered leaves, every node
// picks the neighbour within `searchRadius` that gives the smallest merged half area, mutual picks merge) for animated scenes:
// the world-space bounds come from the (refitted) BLAS roots and the current mesh transforms, both already in HBM, so a moving
// scene never reads its roots back to the host. One CTA (instance counts are tens to thousands): the parallel parts are the
// box transform, the Morton keys, the stable rank sort and the O(n * radius) neighbour search; the ordered placement of merged /
// unmerged nodes runs on one thread, exactly as the reference's loop does, so the node array equals the host build bit for bit
// (idkhost_tlas_build, tests/test_dynamic.py): both take the box, key and half-area arithmetic from idk_bvh_math.h.
struct TlasBuildArgs {
    const float4* blasNodes;         // global GpuBlasNode array (2 x float4 each)
    const GpuBlasDesc* descs;
    const GpuBlasInstance* instances;
    const float4* xforms;            // 9 x float4 per GpuMeshTransform, rows 0..2 = ModelMatrix
    float4* nodes;                   // out: 2n-1 GpuTlasNode (2 x float4 each), root at 0
    float4* temp;                    // scratch: 2n-1 nodes
    float4* leaves;                  // scratch: n nodes
    uint32_t* keys;                  // scratch: n
    int* pref;                       // scratch: n
    int* need;                       // scratch: 2n-1; need[0] on exit = traversal stack entries the TLAS walk needs (tree height)
    int n, searchRadius;
};

__global__ void __launch_bounds__(1024) k_tlas_build(TlasBuildArgs a) {
    __shared__ float s_min[3][32], s_max[3][32];
    __shared__ float s_gmin[3], s_gmax[3];
    __shared__ int s_range[2];
    using namespace idkbvh;
    const int n = a.n, nodeCount = 2 * n - 1, tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < nodeCount; i += nt) { a.nodes[2 * i] = make_float4(0, 0, 0, 0); a.nodes[2 * i + 1] = make_float4(0, 0, 0, 0); }
    // ---- world-space box of every instance: Box.Transformed(BLAS root, ModelMatrix) = the 8 corners through the 3x4 matrix
    float lmn[3] = {3.4028235e38f, 3.4028235e38f, 3.4028235e38f}, lmx[3] = {-3.4028235e38f, -3.4028235e38f, -3.4028235e38f};
    for (int i = tid; i < n; i += nt) {
        const GpuBlasInstance bi = a.instances[i];
        const float4* root = a.blasNodes + 2 * ((size_t)a.descs[bi.BlasId].NodeOffset + 1);
        const float4 rA = root[0], rB = root[1];
        const float4* m = a.xforms + 9 * (size_t)bi.MeshTransformId;
        const float4 m0 = m[0], m1 = m[1], m2 = m[2];
        const float m12[12] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w, m2.x, m2.y, m2.z, m2.w};
        const Box b = transformedBox({{rA.x, rA.y, rA.z}, {rB.x, rB.y, rB.z}}, m12);
        a.leaves[2 * i] = make_float4(b.mn[0], b.mn[1], b.mn[2], __uint_as_float(0x80000000u | (uint32_t)i));
        a.leaves[2 * i + 1] = make_float4(b.mx[0], b.mx[1], b.mx[2], 0.0f);
        for (int k = 0; k < 3; k++) { lmn[k] = minN(lmn[k], b.mn[k]); lmx[k] = maxN(lmx[k], b.mx[k]); }
    }
    // global box: min / max are exact, so the reduction order does not matter
    for (int k = 0; k < 3; k++) {
        float mn = lmn[k], mx = lmx[k];
        for (int off = 16; off > 0; off >>= 1) { mn = fminf(mn, __shfl_down_sync(0xffffffffu, mn, off)); mx = fmaxf(mx, __shfl_down_sync(0xffffffffu, mx, off)); }
        if ((tid & 31) == 0) { s_min[k][tid >> 5] = mn; s_max[k][tid >> 5] = mx; }
    }
    __syncthreads();
    if (tid < 3) {
        float mn = 3.4028235e38f, mx = -3.4028235e38f;
        for (int w = 0; w < (nt + 31) / 32; w++) { mn = fminf(mn, s_min[tid][w]); mx = fmaxf(mx, s_max[tid][w]); }
        s_gmin[tid] = mn; s_gmax[tid] = mx;
    }
    __syncthreads();
    // ---- Morton code of the box centre mapped to [0, 1] by the global box (MyMath.GetMortonCode30 / MapToZeroOne)
    for (int i = tid; i < n; i += nt) {
        const float4 A = a.leaves[2 * i], B = a.leaves[2 * i + 1];
        a.keys[i] = centreKey({{A.x, A.y, A.z}, {B.x, B.y, B.z}}, {{s_gmin[0], s_gmin[1], s_gmin[2]}, {s_gmax[0], s_gmax[1], s_gmax[2]}});
    }
    __syncthreads();
    // ---- stable sort by key (rank sort): the leaf with rank r goes to nodes[nodeCount - n + r]
    for (int i = tid; i < n; i += nt) {
        const uint32_t k = a.keys[i];
        int rank = 0;
        for (int j = 0; j < n; j++) { const uint32_t kj = a.keys[j]; rank += (kj < k || (kj == k && j < i)) ? 1 : 0; }
        a.nodes[2 * (nodeCount - n + rank)] = a.leaves[2 * i];
        a.nodes[2 * (nodeCount - n + rank) + 1] = a.leaves[2 * i + 1];
    }
    if (tid == 0) { s_range[0] = n; s_range[1] = nodeCount; }
    __syncthreads();
    // ---- PLOC iterations
    while (s_range[0] > 1) {
        const int count = s_range[0], end = s_range[1], start = end - count;
        for (int i = tid; i < count; i += nt) {
            const int node = start + i;
            const int s = max(node - a.searchRadius, start), e = min(node + a.searchRadius + 1, end);
            const float4 nA = a.nodes[2 * node], nB = a.nodes[2 * node + 1];
            float smallest = 3.4028235e38f;
            int best = -1;
            for (int j = s; j < e; j++) {
                if (j == node) continue;
                const float4 oA = a.nodes[2 * j], oB = a.nodes[2 * j + 1];
                const float area = halfArea(combine({{nA.x, nA.y, nA.z}, {nB.x, nB.y, nB.z}}, {{oA.x, oA.y, oA.z}, {oB.x, oB.y, oB.z}}));
                if (area < smallest) { smallest = area; best = j; }
            }
            a.pref[i] = best - start;
        }
        __syncthreads();
        if (tid == 0) {
            int merged = 0;
            for (int i = 0; i < count; i++) { const int b = a.pref[i], c = a.pref[b]; if (i == c && i < b) merged += 2; }
            const int unmerged = count - merged, newNodes = merged / 2;
            int mergedHead = end - merged;
            const int newBegin = mergedHead - unmerged - newNodes;
            int unmergedHead = newBegin;
            for (int i = 0; i < count; i++) {
                const int b = a.pref[i], c = a.pref[b];
                const int aId = i + start;
                if (i == c) {
                    if (i < b) {
                        const int bId = b + start;
                        const float4 cA0 = a.nodes[2 * aId], cB0 = a.nodes[2 * aId + 1], cA1 = a.nodes[2 * bId], cB1 = a.nodes[2 * bId + 1];
                        a.temp[2 * mergedHead] = cA0; a.temp[2 * mergedHead + 1] = cB0;
                        a.temp[2 * (mergedHead + 1)] = cA1; a.temp[2 * (mergedHead + 1) + 1] = cB1;
                        a.temp[2 * unmergedHead] = make_float4(minN(cA0.x, cA1.x), minN(cA0.y, cA1.y), minN(cA0.z, cA1.z), __uint_as_float((uint32_t)mergedHead));
                        a.temp[2 * unmergedHead + 1] = make_float4(maxN(cB0.x, cB1.x), maxN(cB0.y, cB1.y), maxN(cB0.z, cB1.z), 0.0f);
                        unmergedHead++;
                        mergedHead += 2;
                    }
                } else {
                    a.temp[2 * unmergedHead] = a.nodes[2 * aId]; a.temp[2 * unmergedHead + 1] = a.nodes[2 * aId + 1];
                    unmergedHead++;
                }
            }
            s_range[0] = count - merged / 2;
            s_range[1] = end - merged;
            a.pref[0] = newBegin;        // hand the copy range to the other threads
        }
        __syncthreads();
        {
            const int newBegin = a.pref[0];
            for (int i = newBegin + tid; i < end; i += nt) { a.nodes[2 * i] = a.temp[2 * i]; a.nodes[2 * i + 1] = a.temp[2 * i + 1]; }
        }
        __syncthreads();
    }
    // stack entries the TLAS walk (BVHIntersect.glsl:205-272, fixed 24-entry stack) needs = the height of the tree; children
    // always follow their parent in the array, so one backward sweep suffices. The host rejects a TLAS that is too deep.
    if (tid == 0) {
        for (int i = nodeCount - 1; i >= 0; i--) {
            const uint32_t w = __float_as_uint(a.nodes[2 * i].w);
            const int c = (int)(w & 0x7FFFFFFFu);
            a.need[i] = (w >> 31) ? 0 : 1 + max(a.need[c], a.need[c + 1]);
        }
    }
}
