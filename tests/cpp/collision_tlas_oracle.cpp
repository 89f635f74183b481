// ORACLE -- TEST INFRASTRUCTURE ONLY: the C#-semantics checker of idkpt_collide_spheres_tlas, loaded by
// tests/collision_tlas_oracle.py.
//
// Intersections.SceneVsMovingSphereCollisionRoutine (Intersections.cs:492-593) over BVH.Intersect(in Box) with
// CpuUseTlas == true (BVH.cs:196-201): TLAS.Intersect(Box) (TLAS.cs:209-264), whose leaves run Box.Transformed and
// BLAS.Intersect(Box) as the linear walk does. It includes the linear oracle (collision_oracle.cpp) unchanged and builds on its
// restatements of BLAS.Intersect(Box), Box.Transformed, SphereVsTriangle, BoxVsBox and Plane.Project / Plane.Reflect; the float
// rules are the same. The routine below takes the instance-level walk as a parameter, so it also runs the linear walk
// (oracle_collide_spheres_walk with cpuUseTlas = 0), which the tests hold byte-equal to oracle_collide_spheres.
#include "collision_oracle.cpp"

namespace {

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
// One test step of SceneVsMovingSphere (Intersections.cs:521-593) with the walk cpuUseTlas picks: BVH.Intersect(hitBox) and
// the callback's "first candidate at the smallest distance" rule (d >= best rejects ties).
static bool CsSceneVsSphereWalk(const Scene& s, bool cpuUseTlas, vec3 center, float radius, CsSphereHit& best) {
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
// SceneVsMovingSphereCollisionRoutine for one sphere with the walk cpuUseTlas picks; `first` (may be null) receives the first
// recursive step's winner.
static IdkPtSphereCollision CsCollideSphereWalk(const Scene& s, bool cpuUseTlas, const IdkPtMovingSphere& sp,
                                                const IdkPtCollisionSettings& st, CsSphereHit* first) {
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
            if (CsSceneVsSphereWalk(s, cpuUseTlas, center, sp.Radius, hit)) {
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

}  // namespace

extern "C" {

// C#-semantics scene versus moving spheres with the instance-level walk BVH.CpuUseTlas picks (cpuUseTlas != 0: the TLAS walk
// over the scene's TlasNodes, as idkpt_collide_spheres_tlas; 0: every instance in index order, as idkpt_collide_spheres).
// firstTri / firstDistance as in oracle_collide_spheres; firstTri's instance index is the TLAS leaf's.
ORACLE_API int oracle_collide_spheres_walk(const IdkPtSceneDesc* scene, const IdkPtMovingSphere* spheres, uint64_t count,
                                           const IdkPtCollisionSettings* settings, IdkPtSphereCollision* out, int32_t* firstTri,
                                           float* firstDistance, int threads, int cpuUseTlas) {
    Scene s; s.d = *scene;
    parallel_for(count, threads, [&](size_t b, size_t e, int) {
        for (size_t i = b; i < e; i++) {
            CsSphereHit h;
            out[i] = CsCollideSphereWalk(s, cpuUseTlas != 0, spheres[i], *settings, &h);
            if (firstTri) { firstTri[2 * i] = h.tri; firstTri[2 * i + 1] = h.inst; }
            if (firstDistance) firstDistance[i] = h.distance;
        }
    });
    return 0;
}

// The checker of idkpt_collide_spheres_tlas: oracle_collide_spheres_walk with the TLAS walk, the same signature as
// oracle_collide_spheres.
ORACLE_API int oracle_collide_spheres_tlas(const IdkPtSceneDesc* scene, const IdkPtMovingSphere* spheres, uint64_t count,
                                           const IdkPtCollisionSettings* settings, IdkPtSphereCollision* out, int32_t* firstTri,
                                           float* firstDistance, int threads) {
    return oracle_collide_spheres_walk(scene, spheres, count, settings, out, firstTri, firstDistance, threads, 1);
}

}  // extern "C"
