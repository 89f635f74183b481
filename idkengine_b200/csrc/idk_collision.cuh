// Scene versus moving spheres for sm_90a: Intersections.SceneVsMovingSphereCollisionRoutine (Intersections.cs:492-593) with the
// callbacks of Camera.CollisionDetection (Camera.cs:152-169, Plane.Project) and LightManager.CollisionDetection
// (LightManager.cs:237-258, Plane.Reflect), over the device scene.
//
//   k_collide_spheres  one thread per sphere. Each test step walks the scene in the order BVH.Intersect(in Box) visits it with
//                      CpuUseTlas == false (BVH.cs:195-223): every instance in index order, the sphere's box taken into
//                      instance space by Box.Transformed (the AABB of its 8 corners times InvModelMatrix), then BLAS.Intersect
//                      (BLAS.cs:388-439): the root test and the sibling-pair loop, the contiguous leaf range of a pair, the
//                      right child pushed when both children are entered. The traversal stack lives in shared memory
//                      (IDK_BLOCK columns of the scene's BlasStackSize entries, as in k_trace_rays); the pushes of this walk
//                      follow the same rule as the ray walk's, so RequiredStackSize bounds them.
//   k_collide_spheres_tlas  the same per-sphere routine over the visit order of BVH.Intersect(in Box) with CpuUseTlas == true:
//                      TLAS.Intersect(Box) (TLAS.cs:209-264). From node 0 (whose own box is not tested), a leaf hands its
//                      instance to the same per-instance walk as above; an interior node tests both children (id, id + 1)
//                      with BoxVsBox against the world-space query box, goes left when both overlap and pushes right, goes to
//                      the one that overlaps, or pops. Only double overlaps push, so a TLAS of height h keeps at most h - 1
//                      entries live; the per-thread stack of IDK_TLAS_STACK_SIZE entries is the bound idkpt_set_scene, the
//                      full-array idkpt_update_range and the device build enforce, as for the ray walk (k_trace_rays).
//                      Candidates therefore come in depth-first TLAS order, and instances whose TLAS leaf box misses the query
//                      box are never walked.
//
// Float semantics: OpenTK's Vector3 formulas in fp32, left to right, no contraction (the library is built with -fmad=false):
// Dot = x*x' + y*y' + z*z', Distance = sqrt of the sum of the squared differences, Vector3 / float divides each component,
// Vector4(p, 1) * Matrix4 = ((x*m0 + y*m1) + z*m2) + m3 per row of the stored 3x4. The CPU oracle
// (tests/cpp/collision_oracle.cpp) restates the same rules; the two agree bit for bit.
#pragma once
#include "idk_kernels.cuh"

struct CollideArgs {
    const float4* nodes;           // 2 x float4 per GpuBlasNode
    const int4* blasTris;          // GpuBlasTriangle
    const float* positions;        // PackedVec3
    const GpuBlasDesc* descs;
    const GpuBlasInstance* instances;
    const float4* xforms;          // 9 x float4 per GpuMeshTransform: ModelMatrix, InvModelMatrix, PrevModelMatrix rows
    uint32_t instanceCount;
    const IdkPtMovingSphere* spheres;
    IdkPtSphereCollision* out;
    uint32_t count;
    IdkPtCollisionSettings st;
    const float4* tlasNodes;       // 2 x float4 per GpuTlasNode, root at 0; read by k_collide_spheres_tlas only
};

namespace idkcol {

struct v3 { float x, y, z; };
__device__ __forceinline__ v3 operator+(v3 a, v3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ v3 operator-(v3 a, v3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ v3 operator*(v3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ v3 operator/(v3 a, float s) { return {a.x / s, a.y / s, a.z / s}; }
__device__ __forceinline__ float dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// Vector4(p, 1) * Matrix4 of the stored rows r[0..2]
__device__ __forceinline__ v3 xform(const float4* r, v3 p) {
    return {((p.x * r[0].x + p.y * r[0].y) + p.z * r[0].z) + r[0].w,
            ((p.x * r[1].x + p.y * r[1].y) + p.z * r[1].z) + r[1].w,
            ((p.x * r[2].x + p.y * r[2].y) + p.z * r[2].z) + r[2].w};
}

// Intersections.TriangleClosestPoint (Intersections.cs:38-94)
__device__ __forceinline__ v3 closest_point(v3 a, v3 b, v3 c, v3 p) {
    const v3 ab = b - a, ac = c - a, ap = p - a;
    const float d1 = dot(ab, ap), d2 = dot(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return a;
    const v3 bp = p - b;
    const float d3 = dot(ab, bp), d4 = dot(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return b;
    const float vc = d1 * d4 - d3 * d2;
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) return a + ab * (d1 / (d1 - d3));
    const v3 cp = p - c;
    const float d5 = dot(ab, cp), d6 = dot(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return c;
    const float vb = d5 * d2 - d1 * d6;
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) return a + ac * (d2 / (d2 - d6));
    const float va = d3 * d6 - d5 * d4;
    if (va <= 0.0f && (d4 - d3) >= 0.0f && (d5 - d6) >= 0.0f) return b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)));
    const float denom = 1.0f / (va + vb + vc);
    return (a + ab * (vb * denom)) + ac * (vc * denom);
}

// Intersections.BoxVsBox (Intersections.cs:150-153) of the query box against a node's box
__device__ __forceinline__ bool box_vs_node(v3 mn, v3 mx, float4 nmin, float4 nmax) {
    return mn.x <= nmax.x && mn.y <= nmax.y && mn.z <= nmax.z && mx.x >= nmin.x && mx.y >= nmin.y && mx.z >= nmin.z;
}

// Plane.Project (SLIDE) or Plane.Reflect (REFLECT) of v on the plane with normal n (Plane.cs)
__device__ __forceinline__ v3 respond(v3 v, v3 n, bool reflect) {
    return reflect ? v - n * (2.0f * dot(n, v)) : v - n * dot(n, v);
}

struct Best { float d, pen; v3 n; };

// One instance of BVH.Intersect(in Box): the query box [bmin, bmax] taken into instance space, then BLAS.Intersect(Box) with
// SphereVsTriangle and the callback's "first at the smallest distance" rule on every candidate triangle, in visit order.
__device__ __forceinline__ void sphere_vs_instance(const CollideArgs& a, uint32_t i, v3 c, float radius, v3 bmin, v3 bmax,
                                                   uint32_t* stack, Best& best) {
    const GpuBlasInstance inst = a.instances[i];
    const GpuBlasDesc desc = a.descs[inst.BlasId];
    const float4* mt = a.xforms + 9 * (size_t)inst.MeshTransformId;
    // Box.Transformed (Box.cs): Box.Empty() grown by the 8 corners with MinNative / MaxNative
    v3 lmin = {FLT_MAX, FLT_MAX, FLT_MAX}, lmax = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const v3 p = xform(mt + 3, {(k & 1) ? bmax.x : bmin.x, (k & 2) ? bmax.y : bmin.y, (k & 4) ? bmax.z : bmin.z});
        lmin = {lmin.x < p.x ? lmin.x : p.x, lmin.y < p.y ? lmin.y : p.y, lmin.z < p.z ? lmin.z : p.z};
        lmax = {lmax.x > p.x ? lmax.x : p.x, lmax.y > p.y ? lmax.y : p.y, lmax.z > p.z ? lmax.z : p.z};
    }
    const float4* nodes = a.nodes + 2 * (size_t)desc.NodeOffset;
    if (!box_vs_node(lmin, lmax, nodes[2], nodes[3])) return;   // the root, Nodes[1]
    const float4 m0 = mt[0], m1 = mt[1], m2 = mt[2];
    const float4 model[3] = {m0, m1, m2};
    uint32_t sp = 0;
    int top = 2;
    for (;;) {
        const float4 lmn = nodes[2 * top], lmx = nodes[2 * top + 1], rmn = nodes[2 * top + 2], rmx = nodes[2 * top + 3];
        const int lChild = __float_as_int(lmn.w), lCount = __float_as_int(lmx.w);
        const int rChild = __float_as_int(rmn.w), rCount = __float_as_int(rmx.w);
        const bool hitL = box_vs_node(lmin, lmax, lmn, lmx), hitR = box_vs_node(lmin, lmax, rmn, rmx);
        const bool il = hitL && lCount > 0, ir = hitR && rCount > 0;
        if (il || ir) {
            const int first = il ? lChild : rChild;
            const int end = !ir ? first + lCount : rChild + rCount;
            for (int t = first; t < end; t++) {
                const int4 tri = a.blasTris[desc.TriangleOffset + t];
                const float* p0 = a.positions + 3 * (size_t)tri.x;
                const float* p1 = a.positions + 3 * (size_t)tri.y;
                const float* p2 = a.positions + 3 * (size_t)tri.z;
                const v3 w0 = xform(model, {p0[0], p0[1], p0[2]});
                const v3 w1 = xform(model, {p1[0], p1[1], p1[2]});
                const v3 w2 = xform(model, {p2[0], p2[1], p2[2]});
                const v3 q = closest_point(w0, w1, w2, c);
                const v3 dq = c - q;
                const float d = sqrtf(dq.x * dq.x + dq.y * dq.y + dq.z * dq.z);
                const float pen = radius - d;
                if (!(pen > 0.0f) || d >= best.d || d == 0.0f) continue;
                best.d = d;
                best.pen = pen;
                best.n = dq / d;
            }
        }
        const bool tl = hitL && !(lCount > 0), tr = hitR && !(rCount > 0);
        if (tl || tr) {
            top = tl ? lChild : rChild;
            if (tl && tr) stack[IDK_BLOCK * sp++] = (uint32_t)rChild;
        } else {
            if (sp == 0) break;
            top = (int)stack[IDK_BLOCK * --sp];
        }
    }
}

// One SceneVsMovingSphere test: every candidate triangle of BVH.Intersect(box) in visit order. TLAS = false: every instance in
// index order (CpuUseTlas == false); TLAS = true: the instances TLAS.Intersect(Box) reaches, in its depth-first order.
template <bool TLAS>
__device__ __forceinline__ void scene_vs_sphere(const CollideArgs& a, v3 c, float radius, uint32_t* stack, Best& best) {
    const v3 r3 = {radius, radius, radius};
    const v3 bmin = c - r3, bmax = c + r3;
    if (!TLAS) {
        for (uint32_t i = 0; i < a.instanceCount; i++) sphere_vs_instance(a, i, c, radius, bmin, bmax, stack, best);
        return;
    }
    uint32_t tstack[IDK_TLAS_STACK_SIZE];
    uint32_t sp = 0, top = 0;
    for (;;) {
        const uint32_t word = __float_as_uint(ldg4(a.tlasNodes + 2 * (size_t)top).w);
        const uint32_t id = word & 0x7FFFFFFFu;
        if (word >> 31) {
            sphere_vs_instance(a, id, c, radius, bmin, bmax, stack, best);
            if (sp == 0) break;
            top = tstack[--sp];
            continue;
        }
        const float4* child = a.tlasNodes + 2 * (size_t)id;
        const bool tl = box_vs_node(bmin, bmax, ldg4(child), ldg4(child + 1));
        const bool tr = box_vs_node(bmin, bmax, ldg4(child + 2), ldg4(child + 3));
        if (tl || tr) {
            top = tl ? id : id + 1;
            if (tl && tr) tstack[sp++] = id + 1;
        } else {
            if (sp == 0) break;
            top = tstack[--sp];
        }
    }
}

// SceneVsMovingSphereCollisionRoutine for the sphere of this thread, with the BVH walk TLAS picks. `a` is taken by value and
// the shared stack is declared here, not passed in: either way round changes the register allocation of k_collide_spheres.
template <bool TLAS>
__device__ __forceinline__ void collide_sphere(CollideArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    const uint32_t gid = blockIdx.x * IDK_BLOCK + threadIdx.x;
    if (gid >= a.count) return;
    const IdkPtMovingSphere s = a.spheres[gid];
    const float radius = s.Radius;
    const bool reflect = a.st.Response == IDKPT_COLLISION_REFLECT;
    v3 center = {s.PrevPosition[0], s.PrevPosition[1], s.PrevPosition[2]};
    v3 prev = center;
    v3 dest = {s.Position[0], s.Position[1], s.Position[2]};
    v3 vel = {s.Velocity[0], s.Velocity[1], s.Velocity[2]};
    int hits = 0;
    for (int r = 0; r < a.st.RecursiveSteps; r++) {
        // SceneVsMovingSphere (Intersections.cs:521-593)
        const v3 step = (dest - center) / (float)a.st.TestSteps;
        Best best = {FLT_MAX, 0.0f, {0.0f, 0.0f, 0.0f}};
        for (int i = 0; i < a.st.TestSteps; i++) {
            center = center + step;
            scene_vs_sphere<TLAS>(a, center, radius, stack, best);
            if (best.d != FLT_MAX) break;
        }
        if (best.d == FLT_MAX) break;
        center = center + best.n * best.pen;
        // SceneVsMovingSphereCollisionRoutine, then the caller's callback: the destination it rewrites is the next step's target
        center = center + best.n * a.st.EpsilonNormalOffset;
        hits++;
        dest = center + respond(dest - prev, best.n, reflect);
        vel = respond(vel, best.n, reflect);
        prev = center;
    }
    IdkPtSphereCollision o;
    o.Position[0] = dest.x; o.Position[1] = dest.y; o.Position[2] = dest.z;
    o.Hits = hits;
    o.Velocity[0] = vel.x; o.Velocity[1] = vel.y; o.Velocity[2] = vel.z;
    o._pad0 = 0.0f;
    a.out[gid] = o;
}

}  // namespace idkcol

__global__ void __launch_bounds__(IDK_BLOCK) k_collide_spheres(CollideArgs a) {
    idkcol::collide_sphere<false>(a);
}

__global__ void __launch_bounds__(IDK_BLOCK) k_collide_spheres_tlas(CollideArgs a) {
    idkcol::collide_sphere<true>(a);
}
