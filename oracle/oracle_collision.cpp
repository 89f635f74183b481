// ORACLE (TEST INFRASTRUCTURE ONLY) -- scene versus moving spheres, the checker of idkpt_collide_spheres and
// idkpt_collide_spheres_tlas.
//
// Part of liboracle.so (wrapped by tests/collision_oracle.py). It includes oracle.cpp and reuses its scene access, vec3 and
// C#-semantics helpers (csDot, minN / maxN) unchanged; the float rules are the same: fp32, left to right, no contraction
// (-ffp-contract=off), IEEE divide and sqrt. OpenTK Vector3 formulas: csDot, Distance = sqrt of the summed squared
// differences, Vector3 / float per component. Vector4(p, 1) * Matrix4 (Triangle.Transformed, Box.Transformed) of a stored
// 3x4: ((x*m0 + y*m1) + z*m2) + m3 per row.
//
// One routine serves both of the engine's modes; only the instance-level walk of BVH.Intersect(in Box) differs. With
// CpuUseTlas == false it visits every instance in index order; with CpuUseTlas == true it walks TLAS.Intersect(Box), whose
// leaves run Box.Transformed and BLAS.Intersect(Box) as the linear walk does.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Source/Shapes/Intersections.cs:492-593   SceneVsMovingSphereCollisionRoutine with the Camera / LightManager callbacks
//   Source/Shapes/Intersections.cs:38-153    TriangleClosestPoint, SphereVsTriangle, BoxVsBox
//   Source/Bvh/BVH.cs:195-223                BVH.Intersect(in Box), both CpuUseTlas modes
//   Source/Bvh/TLAS.cs:209-264               TLAS.Intersect(Box)
//   Source/Bvh/BLAS.cs:388-439               BLAS.Intersect(Box)
//   Source/Shapes/Box.cs, Plane.cs           Box.Transformed, Plane.Project / Plane.Reflect
//
// DESIGN.md 8f.6 pins the rules.
#pragma once
#include "oracle.cpp"

namespace {

// Vector4(p, 1) * Matrix4 of a stored 3x4
static ORACLE_INLINE vec3 CsTransformPoint(const float m[3][4], vec3 p) {
    return {((p.x * m[0][0] + p.y * m[0][1]) + p.z * m[0][2]) + m[0][3],
            ((p.x * m[1][0] + p.y * m[1][1]) + p.z * m[1][2]) + m[1][3],
            ((p.x * m[2][0] + p.y * m[2][1]) + p.z * m[2][2]) + m[2][3]};
}
// Intersections.TriangleClosestPoint (Intersections.cs:38-94)
static ORACLE_INLINE vec3 CsTriangleClosestPoint(vec3 a, vec3 b, vec3 c, vec3 p) {
    vec3 ab = b - a, ac = c - a, ap = p - a;
    float d1 = csDot(ab, ap), d2 = csDot(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) return a;
    vec3 bp = p - b;
    float d3 = csDot(ab, bp), d4 = csDot(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) return b;
    float vc = d1 * d4 - d3 * d2;
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) { float v = d1 / (d1 - d3); return a + v * ab; }
    vec3 cp = p - c;
    float d5 = csDot(ab, cp), d6 = csDot(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) return c;
    float vb = d5 * d2 - d1 * d6;
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) { float w = d2 / (d2 - d6); return a + w * ac; }
    float va = d3 * d6 - d5 * d4;
    if (va <= 0.0f && (d4 - d3) >= 0.0f && (d5 - d6) >= 0.0f) { float w = (d4 - d3) / ((d4 - d3) + (d5 - d6)); return b + w * (c - b); }
    float denom = 1.0f / (va + vb + vc);
    float v = vb * denom, w = vc * denom;
    return a + ab * v + ac * w;
}
// Intersections.SphereVsTriangle (Intersections.cs:134-141)
static ORACLE_INLINE bool CsSphereVsTriangle(vec3 center, float radius, vec3 p0, vec3 p1, vec3 p2, vec3& q, float& distance, float& penetration) {
    q = CsTriangleClosestPoint(p0, p1, p2, center);
    distance = sqrtf((center.x - q.x) * (center.x - q.x) + (center.y - q.y) * (center.y - q.y) + (center.z - q.z) * (center.z - q.z));
    penetration = radius - distance;
    return penetration > 0.0f;
}
// Intersections.BoxVsBox (Intersections.cs:150-153)
static ORACLE_INLINE bool CsBoxVsBox(const float* amin, const float* amax, const float* bmin, const float* bmax) {
    return amin[0] <= bmax[0] && amin[1] <= bmax[1] && amin[2] <= bmax[2] && amax[0] >= bmin[0] && amax[1] >= bmin[1] && amax[2] >= bmin[2];
}
// Box.Transformed (Box.cs): Box.Empty() grown by the 8 transformed corners, MinNative / MaxNative
static ORACLE_INLINE void CsBoxTransformed(const float mn[3], const float mx[3], const float m[3][4], float outMin[3], float outMax[3]) {
    for (int k = 0; k < 3; k++) { outMin[k] = FLT_MAX; outMax[k] = -FLT_MAX; }
    for (int i = 0; i < 8; i++) {
        vec3 p = CsTransformPoint(m, {(i & 1) ? mx[0] : mn[0], (i & 2) ? mx[1] : mn[1], (i & 4) ? mx[2] : mn[2]});
        const float c[3] = {p.x, p.y, p.z};
        for (int k = 0; k < 3; k++) {
            outMin[k] = minN(outMin[k], c[k]);
            outMax[k] = maxN(outMax[k], c[k]);
        }
    }
}
// BLAS.Intersect(Box) (BLAS.cs:388-439): calls f(triangle index within the BLAS) for every candidate, in visit order.
template <class F>
static void CsBlasIntersectBox(const Scene& s, const GpuBlasDesc& desc, const float bmin[3], const float bmax[3], F&& f) {
    const GpuBlasNode* nodes = s.d.BlasNodes + desc.NodeOffset;
    int stack[128];
    int stackPtr = 0, stackTop = 2;
    if (!CsBoxVsBox(bmin, bmax, nodes[1].Min, nodes[1].Max)) return;
    while (true) {
        const GpuBlasNode& l = nodes[stackTop];
        const GpuBlasNode& r = nodes[stackTop + 1];
        bool hitLeft = CsBoxVsBox(bmin, bmax, l.Min, l.Max);
        bool hitRight = CsBoxVsBox(bmin, bmax, r.Min, r.Max);
        bool il = hitLeft && l.TriCount > 0, ir = hitRight && r.TriCount > 0;
        if (il || ir) {
            int first = il ? l.TriStartOrChild : r.TriStartOrChild;
            int end = !ir ? (first + l.TriCount) : (r.TriStartOrChild + r.TriCount);
            for (int i = first; i < end; i++) f(i);
        }
        bool tl = hitLeft && !(l.TriCount > 0), tr = hitRight && !(r.TriCount > 0);
        if (tl || tr) {
            stackTop = tl ? l.TriStartOrChild : r.TriStartOrChild;
            if (tl && tr) stack[stackPtr++] = r.TriStartOrChild;
        } else {
            if (stackPtr == 0) break;
            stackTop = stack[--stackPtr];
        }
    }
}
// TLAS.Intersect(Box) (TLAS.cs:209-264): calls f(instance index) for every TLAS leaf the walk reaches, in visit order.
template <class F>
static void CsTlasIntersectBox(const Scene& s, const float bmin[3], const float bmax[3], F&& f) {
    const GpuTlasNode* tlasNodes = s.d.TlasNodes;
    if (s.d.TlasNodeCount == 0) return;
    int stackPtr = 0;
    int stackTop = 0;
    int stack[128];
    while (true) {
        const GpuTlasNode& parent = tlasNodes[stackTop];
        if ((parent.IsLeafAndChildOrInstanceId >> 31) == 1) {
            int blasInstanceId = (int)(parent.IsLeafAndChildOrInstanceId & ((1u << 31) - 1));
            f(blasInstanceId);
            if (stackPtr == 0) break;
            stackTop = stack[--stackPtr];
            continue;
        }
        int leftNodeId = (int)(parent.IsLeafAndChildOrInstanceId & ((1u << 31) - 1));
        int rightNodeId = leftNodeId + 1;
        const GpuTlasNode& leftNode = tlasNodes[leftNodeId];
        const GpuTlasNode& rightNode = tlasNodes[rightNodeId];
        bool traverseLeft = CsBoxVsBox(leftNode.Min, leftNode.Max, bmin, bmax);
        bool traverseRight = CsBoxVsBox(rightNode.Min, rightNode.Max, bmin, bmax);
        if (traverseLeft || traverseRight) {
            stackTop = traverseLeft ? leftNodeId : rightNodeId;
            if (traverseLeft && traverseRight) stack[stackPtr++] = rightNodeId;
        } else {
            if (stackPtr == 0) break;
            stackTop = stack[--stackPtr];
        }
    }
}
// The instance-level walk of BVH.Intersect(in Box) (BVH.cs:196-223): TLAS.Intersect(Box) with CpuUseTlas == true, every
// instance in index order with CpuUseTlas == false.
template <class F>
static void CsBvhIntersectBox(const Scene& s, bool cpuUseTlas, const float bmin[3], const float bmax[3], F&& f) {
    if (cpuUseTlas) {
        CsTlasIntersectBox(s, bmin, bmax, f);
    } else {
        for (uint64_t i = 0; i < s.d.BlasInstanceCount; i++) f((int)i);
    }
}
// The winner of one SceneVsMovingSphere test step; tri / inst: global BLAS triangle and instance index, -1 when none.
struct CsSphereHit { vec3 normal; float distance, penetration; int32_t tri, inst; };
// One test step of SceneVsMovingSphere (Intersections.cs:521-593) with the walk cpuUseTlas picks: BVH.Intersect(hitBox) and
// the callback's "first candidate at the smallest distance" rule (d >= best rejects ties).
static bool CsSceneVsSphere(const Scene& s, bool cpuUseTlas, vec3 center, float radius, CsSphereHit& best) {
    const float bmin[3] = {center.x - radius, center.y - radius, center.z - radius};
    const float bmax[3] = {center.x + radius, center.y + radius, center.z + radius};
    best = {{0.0f, 0.0f, 0.0f}, FLT_MAX, 0.0f, -1, -1};
    CsBvhIntersectBox(s, cpuUseTlas, bmin, bmax, [&](int i) {
        const GpuBlasInstance& inst = s.d.BlasInstances[i];
        const GpuBlasDesc& desc = s.d.BlasDescs[inst.BlasId];
        const GpuMeshTransform& mt = s.d.MeshTransforms[inst.MeshTransformId];
        float lmin[3], lmax[3];
        CsBoxTransformed(bmin, bmax, mt.InvModelMatrix, lmin, lmax);
        CsBlasIntersectBox(s, desc, lmin, lmax, [&](int t) {
            const int32_t g = desc.TriangleOffset + t;
            const GpuBlasTriangle& tri = s.d.BlasTriangles[g];
            vec3 w0 = CsTransformPoint(mt.ModelMatrix, pos(s, tri.X));
            vec3 w1 = CsTransformPoint(mt.ModelMatrix, pos(s, tri.Y));
            vec3 w2 = CsTransformPoint(mt.ModelMatrix, pos(s, tri.Z));
            vec3 q;
            float d, pen;
            if (!CsSphereVsTriangle(center, radius, w0, w1, w2, q, d, pen) || d >= best.distance) return;
            if (d == 0.0f) return;
            best.normal = (center - q) / d;   // SlidingPlane.Normal
            best.distance = d;
            best.penetration = pen;
            best.tri = g;
            best.inst = (int32_t)i;
        });
    });
    return best.tri >= 0;
}
// Plane.Project / Plane.Reflect (Plane.cs)
static ORACLE_INLINE vec3 CsPlaneProject(vec3 v, vec3 n) { return v - csDot(n, v) * n; }
static ORACLE_INLINE vec3 CsPlaneReflect(vec3 v, vec3 n) { return v - 2.0f * csDot(n, v) * n; }
// SceneVsMovingSphereCollisionRoutine for one sphere with the walk cpuUseTlas picks; `first` (may be null) receives the first
// recursive step's winner.
static IdkPtSphereCollision CsCollideSphere(const Scene& s, bool cpuUseTlas, const IdkPtMovingSphere& sp, const IdkPtCollisionSettings& st,
                                            CsSphereHit* first) {
    vec3 center = V(sp.PrevPosition);
    vec3 prev = center;
    vec3 dest = V(sp.Position);
    vec3 vel = V(sp.Velocity);
    int32_t hits = 0;
    if (first) *first = {{0.0f, 0.0f, 0.0f}, FLT_MAX, 0.0f, -1, -1};
    for (int r = 0; r < st.RecursiveSteps; r++) {
        vec3 step = (dest - center) / (float)st.TestSteps;
        CsSphereHit hit;
        bool found = false;
        for (int i = 0; i < st.TestSteps && !found; i++) {
            center = center + step;
            if (CsSceneVsSphere(s, cpuUseTlas, center, sp.Radius, hit)) {
                center = center + hit.normal * hit.penetration;
                found = true;
            }
        }
        if (!found) break;
        if (first && hits == 0) *first = hit;
        center = center + hit.normal * st.EpsilonNormalOffset;
        hits++;
        vec3 delta = dest - prev;
        bool reflect = st.Response == IDKPT_COLLISION_REFLECT;
        dest = center + (reflect ? CsPlaneReflect(delta, hit.normal) : CsPlaneProject(delta, hit.normal));
        vel = reflect ? CsPlaneReflect(vel, hit.normal) : CsPlaneProject(vel, hit.normal);
        prev = center;
    }
    IdkPtSphereCollision o = {};
    o.Position[0] = dest.x; o.Position[1] = dest.y; o.Position[2] = dest.z;
    o.Hits = hits;
    o.Velocity[0] = vel.x; o.Velocity[1] = vel.y; o.Velocity[2] = vel.z;
    return o;
}

} // namespace

extern "C" {

// C#-semantics scene versus moving spheres with the instance-level walk BVH.CpuUseTlas picks: cpuUseTlas == 0, every instance
// in index order (idkpt_collide_spheres); otherwise the TLAS walk over the scene's TlasNodes (idkpt_collide_spheres_tlas).
// firstTri (may be null): per sphere, the global BLAS triangle and the instance index that won the first recursive step (-1, -1
// without a hit); firstDistance (may be null): its distance to the sphere's centre (FLT_MAX without a hit).
ORACLE_API int oracle_collide_spheres(const IdkPtSceneDesc* scene, const IdkPtMovingSphere* spheres, uint64_t count,
                                      const IdkPtCollisionSettings* settings, IdkPtSphereCollision* out, int32_t* firstTri,
                                      float* firstDistance, int threads, int cpuUseTlas) {
    Scene s; s.d = *scene;
    parallel_for(count, threads, [&](size_t b, size_t e, int) {
        for (size_t i = b; i < e; i++) {
            CsSphereHit h;
            out[i] = CsCollideSphere(s, cpuUseTlas != 0, spheres[i], *settings, &h);
            if (firstTri) { firstTri[2 * i] = h.tri; firstTri[2 * i + 1] = h.inst; }
            if (firstDistance) firstDistance[i] = h.distance;
        }
    });
    return 0;
}

} // extern "C"
