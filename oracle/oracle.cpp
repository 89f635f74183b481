// ORACLE -- TEST INFRASTRUCTURE ONLY.
//
// CPU restatement of the reference's path-tracing hot path, used as the checker
// for the CUDA kernels. Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library; the product
// (idkengine_b200/, libidkpt.so) never does.
//
// PARITY UNPINNED: the reference ships no tests, golden images or known-answer
// vectors for this path and neither C# nor GLSL can run in this image, so this
// oracle is pinned only by (a) following the sources below line by line,
// (b) a brute-force all-triangles intersector, (c) the builder's structural
// invariants (tests/test_bvh_build.py).
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/include/BVHIntersect.glsl:27-105,183-291  IntersectBlas, TraceRay (closest, no-TLAS + TLAS)
//   Resource/Shaders/include/IntersectionRoutines.glsl:6-69   ray/triangle, ray/box, ray/sphere
//   Resource/Shaders/include/Ray.glsl:7-12                    RayTransform
//   Resource/Shaders/include/Random.glsl:16-33                PCG hash RNG
//   Resource/Shaders/include/Sampling.glsl:4-19,59-68,86-114  R2, Cranley-Patterson, SampleSphere, SampleDisk
//   Resource/Shaders/include/Compression.glsl:11-37,41-73     R11G11B10, unorm8, octahedral encode/decode
//   Resource/Shaders/include/Surface.glsl:25-111              Surface, GetSurface (constant textures), modifications
//   Resource/Shaders/include/Pbr.glsl:19-27,64-67             BaseReflectivity, FresnelSchlick
//   Resource/Shaders/include/Math.glsl:6-15,41-57,104-137     camera dir, CubemapFaceNormal, Interpolate, TBN
//   Resource/Shaders/PathTracing/FirstHit/compute.glsl        ray-gen + first hit (all)
//   Resource/Shaders/PathTracing/NHit/compute.glsl            bounce (all)
//   Resource/Shaders/PathTracing/FinalDraw/compute.glsl:24-62 accumulate
//   Resource/Shaders/PathTracing/include/{Shading,RussianRoulette}.glsl
//   Resource/Shaders/PathTracing/CountingSort/**              semantics only: stable sort by 21-bit key
//   Source/Render/PathTracer.cs:214-297                        host sequencing
//   Source/Bvh/BLAS.cs:313-386, Source/Bvh/BVH.cs:162-193,
//   Source/Shapes/Intersections.cs:363-396                     CPU (collision/picking) traversal = cpu baseline
//
// Canonical choices for the reference's unordered atomics (SURVEY.md 8c): alive
// lists are appended in ascending slot / ray-index order, sorting is stable.
//
// Float semantics (DESIGN.md): every GLSL operation is evaluated in fp32, left
// to right, WITHOUT fused multiply-add (-ffp-contract=off), IEEE divide/sqrt;
// normalize(v) = v * (1/sqrt(dot(v,v))); pow(x,5) = ((x*x)*(x*x))*x; sin/cos/exp
// are the polynomial routines below (glibc's and CUDA's libm differ in the last
// ulp, so both sides implement the same documented algorithm instead).
//
// The pass oracles (oracle_*.cpp) include this file and each other; oracle/liboracle.cpp includes them all, so the whole
// checker is one translation unit and one library, oracle/liboracle.so (oracle/build.py).
#pragma once

#include <cstdint>
#include <cstring>
#include <cmath>
#include <cfloat>
#include <vector>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <atomic>
#include <functional>
#include <algorithm>
#include <chrono>

#include "../include/idkpt.h"

// The small helpers below are inlined whatever the size of the translation unit, so the traversal and shading loops that
// bench.py times do not change speed as pass oracles are added to the library.
#define ORACLE_INLINE inline __attribute__((always_inline))

namespace {

// ------------------------------------------------------------------ vec3
struct vec3 { float x, y, z; };
static ORACLE_INLINE vec3 V(float x, float y, float z) { return {x, y, z}; }
static ORACLE_INLINE vec3 V(const float* p) { return {p[0], p[1], p[2]}; }
static ORACLE_INLINE vec3 operator+(vec3 a, vec3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
static ORACLE_INLINE vec3 operator-(vec3 a, vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
static ORACLE_INLINE vec3 operator-(vec3 a) { return {-a.x, -a.y, -a.z}; }
static ORACLE_INLINE vec3 operator*(vec3 a, vec3 b) { return {a.x * b.x, a.y * b.y, a.z * b.z}; }
static ORACLE_INLINE vec3 operator*(vec3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
static ORACLE_INLINE vec3 operator*(float s, vec3 a) { return {s * a.x, s * a.y, s * a.z}; }
static ORACLE_INLINE vec3 operator/(vec3 a, float s) { return {a.x / s, a.y / s, a.z / s}; }
static ORACLE_INLINE vec3 operator/(vec3 a, vec3 b) { return {a.x / b.x, a.y / b.y, a.z / b.z}; }
static ORACLE_INLINE float dot(vec3 a, vec3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
static ORACLE_INLINE vec3 cross(vec3 a, vec3 b) { return {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; }
static ORACLE_INLINE vec3 normalize(vec3 v) { float inv = 1.0f / sqrtf(dot(v, v)); return v * inv; }
static ORACLE_INLINE float mixf(float x, float y, float a) { return x * (1.0f - a) + y * a; }
static ORACLE_INLINE vec3 mix(vec3 x, vec3 y, float a) { return {mixf(x.x, y.x, a), mixf(x.y, y.y, a), mixf(x.z, y.z, a)}; }
static ORACLE_INLINE float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
static ORACLE_INLINE float fractf(float x) { return x - floorf(x); }
static ORACLE_INLINE vec3 reflect(vec3 I, vec3 N) { return I - (2.0f * dot(N, I)) * N; }
static ORACLE_INLINE vec3 refract(vec3 I, vec3 N, float eta) {
    float d = dot(N, I);
    float k = 1.0f - eta * eta * (1.0f - d * d);
    if (k < 0.0f) return V(0.0f, 0.0f, 0.0f);
    return eta * I - (eta * d + sqrtf(k)) * N;
}

#define PI_F 3.14159265f
#define FLOAT_MAX 3.4028235e+38f

// ------------------------------------------------------------------ deterministic sin/cos/exp
// sincos for x in [0, 2*pi]: quadrant reduction with a two-term pi/2 (Cody-Waite), then the
// classic single-precision minimax polynomials on [-pi/4, pi/4] (Cephes sinf/cosf coefficients).
static ORACLE_INLINE void det_sincos(float x, float* s, float* c) {
    float q = floorf(x * 0.63661977236758134f + 0.5f); // nearest multiple of pi/2
    int n = (int)q;
    float r = (x - q * 1.5703125f) - q * 4.83826794897e-4f; // pi/2 = 1.5703125 + 4.83826794897e-4
    float z = r * r;
    float sp = ((-1.9515295891e-4f * z + 8.3321608736e-3f) * z - 1.6666654611e-1f) * z * r + r;
    float cp = ((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z + 4.166664568298827e-2f) * z * z - 0.5f * z + 1.0f;
    switch (n & 3) {
        case 0: *s = sp; *c = cp; break;
        case 1: *s = cp; *c = -sp; break;
        case 2: *s = -sp; *c = -cp; break;
        default: *s = -cp; *c = sp; break;
    }
}

// exp(x): n = round(x*log2e), r = x - n*ln2 (two-term), degree-5 polynomial (Cephes expf), scale by 2^n.
static ORACLE_INLINE float det_exp(float x) {
    if (x < -87.0f) return 0.0f;
    if (x > 88.0f) return INFINITY;
    float fn = floorf(x * 1.44269504088896341f + 0.5f);
    float r = (x - fn * 0.693359375f) - fn * -2.12194440e-4f;
    float z = r * r;
    float p = ((((1.9875691500e-4f * r + 1.3981999507e-3f) * r + 8.3334519073e-3f) * r + 4.1665795894e-2f) * r + 1.6666665459e-1f) * r + 5.0000001201e-1f;
    float e = p * z + r + 1.0f;
    int n = (int)fn;
    uint32_t bits = (uint32_t)(n + 127) << 23;
    float scale;
    memcpy(&scale, &bits, 4);
    return e * scale;
}

// ------------------------------------------------------------------ scene access
struct Scene {
    IdkPtSceneDesc d;
    float skyColor[3];
    int skyFaceSize = 0;           // 0 = constant colour
    const float* skyFaces[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // rgba32f, +X,-X,+Y,-Y,+Z,-Z
};

struct Ray { vec3 o, d; };

struct HitInfo {
    float bx, by;
    float T;
    uint32_t TriangleId;
    uint32_t MeshTransformId;
};

struct Counters { uint32_t steps, tris, instances; float debugCost; };

// IntersectionRoutines.glsl:6-23
static ORACLE_INLINE bool RayTriangleIntersect(const Ray& ray, vec3 p0, vec3 p1, vec3 p2, vec3& bary, float& t) {
    vec3 p1p0 = p1 - p0;
    vec3 p2p0 = p2 - p0;
    vec3 rop0 = ray.o - p0;
    vec3 normal = cross(p1p0, p2p0);
    vec3 q = cross(rop0, ray.d);
    float invDet = 1.0f / dot(ray.d, normal);
    t = dot(-normal, rop0) * invDet;
    bary.y = dot(-q, p2p0) * invDet;
    bary.z = dot(q, p1p0) * invDet;
    bary.x = 1.0f - bary.y - bary.z;
    return bary.x >= 0.0f && bary.y >= 0.0f && bary.z >= 0.0f && t >= 0.0f;
}

// IntersectionRoutines.glsl:25-46 (invDir hoisted by the caller: 1.0 / ray.Direction)
static ORACLE_INLINE bool RayBoxIntersect(const Ray& ray, vec3 invDir, const float* bmin, const float* bmax, float& t1) {
    vec3 t0s = (V(bmin) - ray.o) * invDir;
    vec3 t1s = (V(bmax) - ray.o) * invDir;
    vec3 ts = {fminf(t0s.x, t1s.x), fminf(t0s.y, t1s.y), fminf(t0s.z, t1s.z)};
    vec3 tb = {fmaxf(t0s.x, t1s.x), fmaxf(t0s.y, t1s.y), fmaxf(t0s.z, t1s.z)};
    t1 = fmaxf(ts.x, fmaxf(ts.y, fmaxf(ts.z, 0.0f)));
    float t2 = fminf(tb.x, fminf(tb.y, tb.z));
    return t1 <= t2;
}

// IntersectionRoutines.glsl:48-69
static ORACLE_INLINE bool RaySphereIntersect(const Ray& ray, vec3 position, float radius, float& t1, float& t2) {
    t1 = FLOAT_MAX;
    t2 = FLOAT_MAX;
    vec3 sphereToRay = ray.o - position;
    float b = dot(ray.d, sphereToRay);
    float c = dot(sphereToRay, sphereToRay) - radius * radius;
    float discriminant = b * b - c;
    if (discriminant < 0.0f) return false;
    float squareRoot = sqrtf(discriminant);
    t1 = -b - squareRoot;
    t2 = -b + squareRoot;
    return t1 <= t2 && t2 > 0.0f;
}

static ORACLE_INLINE vec3 pos(const Scene& s, int32_t i) { const PackedVec3& p = s.d.VertexPositions[i]; return {p.x, p.y, p.z}; }

// BVHIntersect.glsl:27-105
static bool IntersectBlas(const Scene& s, const Ray& ray, const GpuBlasDesc& blasDesc, HitInfo& hitInfo, Counters& cnt, bool useTlas) {
    bool hit = false;
    float tMinLeft, tMinRight;
    const GpuBlasNode* nodes = s.d.BlasNodes + blasDesc.NodeOffset;
    vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};

    if (!useTlas) {
        const GpuBlasNode& rootNode = nodes[1];
        if (!(RayBoxIntersect(ray, invDir, rootNode.Min, rootNode.Max, tMinLeft) && tMinLeft < hitInfo.T)) return false;
    }

    uint32_t stack[256];
    uint32_t stackPtr = 0;
    uint32_t stackTop = 2;
    while (true) {
        cnt.debugCost += 1.0f;
        cnt.steps++;
        const GpuBlasNode& leftNode = nodes[stackTop];
        const GpuBlasNode& rightNode = nodes[stackTop + 1];

        bool hitLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft <= hitInfo.T;
        bool hitRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight <= hitInfo.T;

        bool intersectLeft = hitLeft && leftNode.TriCount > 0;
        bool intersectRight = hitRight && rightNode.TriCount > 0;
        if (intersectLeft || intersectRight) {
            uint32_t first = intersectLeft ? (uint32_t)leftNode.TriStartOrChild : (uint32_t)rightNode.TriStartOrChild;
            uint32_t end = !intersectRight ? (uint32_t)(leftNode.TriStartOrChild + leftNode.TriCount) : (uint32_t)(rightNode.TriStartOrChild + rightNode.TriCount);
            first += (uint32_t)blasDesc.TriangleOffset;
            end += (uint32_t)blasDesc.TriangleOffset;
            cnt.debugCost += (float)(end - first) * 1.1f;
            cnt.tris += end - first;
            for (uint32_t i = first; i < end; i++) {
                const GpuBlasTriangle& tri = s.d.BlasTriangles[i];
                vec3 bary;
                float hitT;
                if (RayTriangleIntersect(ray, pos(s, tri.X), pos(s, tri.Y), pos(s, tri.Z), bary, hitT) && hitT < hitInfo.T) {
                    hit = true;
                    hitInfo.TriangleId = i;
                    hitInfo.bx = bary.x;
                    hitInfo.by = bary.y;
                    hitInfo.T = hitT;
                }
            }
        }

        bool traverseLeft = hitLeft && leftNode.TriCount == 0;
        bool traverseRight = hitRight && rightNode.TriCount == 0;
        if (traverseLeft || traverseRight) {
            if (traverseLeft && traverseRight) {
                bool leftCloser = tMinLeft < tMinRight;
                stackTop = leftCloser ? leftNode.TriStartOrChild : rightNode.TriStartOrChild;
                stack[stackPtr++] = leftCloser ? rightNode.TriStartOrChild : leftNode.TriStartOrChild;
            } else {
                stackTop = traverseLeft ? leftNode.TriStartOrChild : rightNode.TriStartOrChild;
            }
        } else {
            if (stackPtr == 0) break;
            stackTop = stack[--stackPtr];
        }
    }
    return hit;
}

// Ray.glsl:7-12 with mat4(mat4x3): rows of the stored 3x4.
static ORACLE_INLINE Ray RayTransform(const Ray& ray, const float m[3][4]) {
    Ray r;
    r.o.x = ((m[0][0] * ray.o.x + m[0][1] * ray.o.y) + m[0][2] * ray.o.z) + m[0][3];
    r.o.y = ((m[1][0] * ray.o.x + m[1][1] * ray.o.y) + m[1][2] * ray.o.z) + m[1][3];
    r.o.z = ((m[2][0] * ray.o.x + m[2][1] * ray.o.y) + m[2][2] * ray.o.z) + m[2][3];
    r.d.x = (m[0][0] * ray.d.x + m[0][1] * ray.d.y) + m[0][2] * ray.d.z;
    r.d.y = (m[1][0] * ray.d.x + m[1][1] * ray.d.y) + m[1][2] * ray.d.z;
    r.d.z = (m[2][0] * ray.d.x + m[2][1] * ray.d.y) + m[2][2] * ray.d.z;
    return r;
}

// BVHIntersect.glsl:183-291
static bool TraceRay(const Scene& s, const Ray& ray, HitInfo& hitInfo, Counters& cnt, bool traceLights, float maxDist) {
    hitInfo.T = maxDist;
    hitInfo.TriangleId = ~0u;
    hitInfo.MeshTransformId = 0;
    hitInfo.bx = hitInfo.by = 0.0f;
    cnt.debugCost = 0.0f;

    if (traceLights) {
        float tMin, tMax;
        for (uint64_t i = 0; i < s.d.LightCount; i++) {
            const GpuLight& light = s.d.Lights[i];
            if (RaySphereIntersect(ray, V(light.Position), light.Radius, tMin, tMax) && tMin < hitInfo.T) {
                hitInfo.T = tMin < 0.0f ? tMax : tMin;
                hitInfo.MeshTransformId = (uint32_t)i;
                hitInfo.TriangleId = ~0u;
            }
        }
    }

    if (s.d.UseTlas) {
        float tMinLeft, tMinRight;
        uint32_t stackPtr = 0, stackTop = 0;
        uint32_t stack[24];
        vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};
        while (true) {
            const GpuTlasNode& parent = s.d.TlasNodes[stackTop];
            bool isLeaf = (parent.IsLeafAndChildOrInstanceId >> 31) == 1;
            uint32_t childOrInstanceId = parent.IsLeafAndChildOrInstanceId & ((1u << 31) - 1);
            if (isLeaf) {
                const GpuBlasInstance& inst = s.d.BlasInstances[childOrInstanceId];
                const GpuBlasDesc& desc = s.d.BlasDescs[inst.BlasId];
                const GpuMeshTransform& mt = s.d.MeshTransforms[inst.MeshTransformId];
                Ray localRay = RayTransform(ray, mt.InvModelMatrix);
                cnt.instances++;
                if (IntersectBlas(s, localRay, desc, hitInfo, cnt, true)) hitInfo.MeshTransformId = inst.MeshTransformId;
                if (stackPtr == 0) break;
                stackTop = stack[--stackPtr];
                continue;
            }
            uint32_t leftChildId = childOrInstanceId, rightChildId = leftChildId + 1;
            const GpuTlasNode& leftNode = s.d.TlasNodes[leftChildId];
            const GpuTlasNode& rightNode = s.d.TlasNodes[rightChildId];
            bool traverseLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft < hitInfo.T;
            bool traverseRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight < hitInfo.T;
            if (traverseLeft || traverseRight) {
                if (traverseLeft && traverseRight) {
                    bool leftCloser = tMinLeft < tMinRight;
                    stackTop = leftCloser ? leftChildId : rightChildId;
                    stack[stackPtr++] = leftCloser ? rightChildId : leftChildId;
                } else {
                    stackTop = traverseLeft ? leftChildId : rightChildId;
                }
            } else {
                if (stackPtr == 0) break;
                stackTop = stack[--stackPtr];
            }
        }
    } else {
        for (uint64_t i = 0; i < s.d.BlasInstanceCount; i++) {
            const GpuBlasInstance& inst = s.d.BlasInstances[i];
            const GpuBlasDesc& desc = s.d.BlasDescs[inst.BlasId];
            const GpuMeshTransform& mt = s.d.MeshTransforms[inst.MeshTransformId];
            Ray localRay = RayTransform(ray, mt.InvModelMatrix);
            cnt.instances++;
            if (IntersectBlas(s, localRay, desc, hitInfo, cnt, false)) hitInfo.MeshTransformId = inst.MeshTransformId;
        }
    }
    return hitInfo.T != maxDist;
}

// Brute force: same instance loop and triangle rule, no BVH. Closest hit with "first encountered wins" replaced by
// (smallest t, then smallest triangle id) -- used only to validate the BVH's (t) and, where t is unique, the id.
static bool BruteForce(const Scene& s, const Ray& ray, HitInfo& hitInfo, float maxDist) {
    hitInfo.T = maxDist;
    hitInfo.TriangleId = ~0u;
    hitInfo.MeshTransformId = 0;
    hitInfo.bx = hitInfo.by = 0.0f;
    for (uint64_t i = 0; i < s.d.BlasInstanceCount; i++) {
        const GpuBlasInstance& inst = s.d.BlasInstances[i];
        const GpuBlasDesc& desc = s.d.BlasDescs[inst.BlasId];
        Ray localRay = RayTransform(ray, s.d.MeshTransforms[inst.MeshTransformId].InvModelMatrix);
        for (int32_t k = desc.TriangleOffset; k < desc.TriangleOffset + desc.TriangleCount; k++) {
            const GpuBlasTriangle& tri = s.d.BlasTriangles[k];
            vec3 bary;
            float t;
            if (RayTriangleIntersect(localRay, pos(s, tri.X), pos(s, tri.Y), pos(s, tri.Z), bary, t) && t < hitInfo.T) {
                hitInfo.T = t;
                hitInfo.TriangleId = (uint32_t)k;
                hitInfo.bx = bary.x;
                hitInfo.by = bary.y;
                hitInfo.MeshTransformId = inst.MeshTransformId;
            }
        }
    }
    return hitInfo.T != maxDist;
}

// ------------------------------------------------------------------ CPU (C#) traversal = baseline
// Intersections.RayVsBox (Intersections.cs:363-377): division based, MaxNative/MinNative.
static ORACLE_INLINE float minN(float a, float b) { return a < b ? a : b; }
static ORACLE_INLINE float maxN(float a, float b) { return a > b ? a : b; }
static ORACLE_INLINE bool CsRayVsBox(const Ray& ray, const float* bmin, const float* bmax, float& t1) {
    vec3 t0s = (V(bmin) - ray.o) / ray.d;
    vec3 t1s = (V(bmax) - ray.o) / ray.d;
    vec3 ts = {minN(t0s.x, t1s.x), minN(t0s.y, t1s.y), minN(t0s.z, t1s.z)};
    vec3 tb = {maxN(t0s.x, t1s.x), maxN(t0s.y, t1s.y), maxN(t0s.z, t1s.z)};
    t1 = maxN(ts.x, maxN(ts.y, maxN(ts.z, 0.0f)));
    float t2 = minN(tb.x, minN(tb.y, tb.z));
    return t1 <= t2;
}
// Intersections.RayVsTriangle (Intersections.cs:379-396): divisions by x, t > 0. OpenTK Vector3.Cross/Dot.
static ORACLE_INLINE vec3 csCross(vec3 l, vec3 r) { return {l.y * r.z - l.z * r.y, l.z * r.x - l.x * r.z, l.x * r.y - l.y * r.x}; }
static ORACLE_INLINE float csDot(vec3 a, vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static ORACLE_INLINE bool CsRayVsTriangle(const Ray& ray, vec3 p0, vec3 p1, vec3 p2, vec3& bary, float& t) {
    vec3 v1v0 = p1 - p0, v2v0 = p2 - p0, rov0 = ray.o - p0;
    vec3 normal = csCross(v1v0, v2v0);
    vec3 q = csCross(rov0, ray.d);
    float x = csDot(ray.d, normal);
    bary.y = csDot(-q, v2v0) / x;
    bary.z = csDot(q, v1v0) / x;
    bary.x = 1.0f - bary.y - bary.z;
    t = csDot(-normal, rov0) / x;
    return bary.x >= 0.0f && bary.y >= 0.0f && bary.z >= 0.0f && t > 0.0f;
}
// BLAS.Intersect (BLAS.cs:313-386)
static bool CsBlasIntersect(const Scene& s, const GpuBlasDesc& desc, const Ray& ray, HitInfo& hit, float tMaxDist, Counters& cnt) {
    const GpuBlasNode* nodes = s.d.BlasNodes + desc.NodeOffset;
    hit.T = tMaxDist;
    int stack[128];
    int stackPtr = 0, stackTop = 2;
    float tmp;
    if (!CsRayVsBox(ray, nodes[1].Min, nodes[1].Max, tmp)) return false;
    while (true) {
        const GpuBlasNode& l = nodes[stackTop];
        const GpuBlasNode& r = nodes[stackTop + 1];
        float tMinLeft, tMinRight;
        bool hitLeft = CsRayVsBox(ray, l.Min, l.Max, tMinLeft) && tMinLeft <= hit.T;
        bool hitRight = CsRayVsBox(ray, r.Min, r.Max, tMinRight) && tMinRight <= hit.T;
        cnt.steps++;
        bool il = hitLeft && l.TriCount > 0, ir = hitRight && r.TriCount > 0;
        if (il || ir) {
            int first = il ? l.TriStartOrChild : r.TriStartOrChild;
            int end = !ir ? (first + l.TriCount) : (r.TriStartOrChild + r.TriCount);
            for (int i = first; i < end; i++) {
                const GpuBlasTriangle& tri = s.d.BlasTriangles[desc.TriangleOffset + i];
                vec3 bary;
                float t;
                if (CsRayVsTriangle(ray, pos(s, tri.X), pos(s, tri.Y), pos(s, tri.Z), bary, t) && t < hit.T) {
                    hit.bx = bary.x; hit.by = bary.y; hit.T = t; hit.TriangleId = (uint32_t)i;
                }
            }
            cnt.tris += (uint32_t)(end - first);
        }
        bool tl = hitLeft && !(l.TriCount > 0), tr = hitRight && !(r.TriCount > 0);
        if (tl || tr) {
            if (tl && tr) {
                bool leftCloser = tMinLeft < tMinRight;
                stackTop = leftCloser ? l.TriStartOrChild : r.TriStartOrChild;
                stack[stackPtr++] = leftCloser ? r.TriStartOrChild : l.TriStartOrChild;
            } else {
                stackTop = tl ? l.TriStartOrChild : r.TriStartOrChild;
            }
        } else {
            if (stackPtr == 0) break;
            stackTop = stack[--stackPtr];
        }
    }
    return hit.T != tMaxDist;
}
// BVH.Intersect (BVH.cs:162-193), no TLAS. Inlined into oracle_cpu_intersect's worker, the cpu_baseline loop bench.py times.
static ORACLE_INLINE bool CsBvhIntersect(const Scene& s, const Ray& ray, HitInfo& hitInfo, float tMax, Counters& cnt) {
    hitInfo.T = tMax;
    hitInfo.TriangleId = ~0u;
    hitInfo.MeshTransformId = 0;
    hitInfo.bx = hitInfo.by = 0.0f;
    for (uint64_t i = 0; i < s.d.BlasInstanceCount; i++) {
        const GpuBlasInstance& inst = s.d.BlasInstances[i];
        const GpuBlasDesc& desc = s.d.BlasDescs[inst.BlasId];
        Ray localRay = RayTransform(ray, s.d.MeshTransforms[inst.MeshTransformId].InvModelMatrix);
        HitInfo bh = {};
        cnt.instances++;
        if (CsBlasIntersect(s, desc, localRay, bh, hitInfo.T, cnt)) {
            hitInfo.bx = bh.bx; hitInfo.by = bh.by; hitInfo.T = bh.T;
            hitInfo.TriangleId = (uint32_t)desc.TriangleOffset + bh.TriangleId;
            hitInfo.MeshTransformId = (uint32_t)i; // BlasInstanceId
        }
    }
    return hitInfo.T != tMax;
}

// ------------------------------------------------------------------ RNG / sampling / compression
struct Rng { uint32_t seed; };
static ORACLE_INLINE uint32_t GetPCGHash(uint32_t& seed) {
    seed = seed * 747796405u + 2891336453u;
    uint32_t word = ((seed >> ((seed >> 28u) + 4u)) ^ seed) * 277803737u;
    return (word >> 22u) ^ word;
}
static ORACLE_INLINE float GetRandomFloat01(Rng& r) { return (float)GetPCGHash(r.seed) / 4294967296.0f; }

static ORACLE_INLINE void R2Sequence(uint32_t id, float& u, float& v) {
    const float g = 1.32471795724474602596f;
    const float a1 = 1.0f / g;
    const float a2 = 1.0f / (g * g);
    u = fractf((float)id * a1);
    v = fractf((float)id * a2);
}

static ORACLE_INLINE vec3 SampleSphere(float rnd0, float rnd1) {
    float cosTheta = rnd0 * 2.0f - 1.0f;
    float phi = rnd1 * 2.0f * PI_F;
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    float sinPhi, cosPhi;
    det_sincos(phi, &sinPhi, &cosPhi);
    return {sinTheta * cosPhi, sinTheta * sinPhi, cosTheta};
}
static ORACLE_INLINE vec3 CosineSampleHemisphere(vec3 normal, float u, float v) { return normalize(normal + SampleSphere(u, v)); }

static ORACLE_INLINE void SampleDisk(Rng& rng, float& px, float& py) {
    float dist;
    float lastRnd = GetRandomFloat01(rng);
    do {
        float thisRnd = GetRandomFloat01(rng);
        px = lastRnd;
        py = thisRnd;
        dist = px * px + py * py;
        lastRnd = thisRnd;
    } while (dist > 1.0f);
    px = px * 2.0f - 1.0f;
    py = py * 2.0f - 1.0f;
}

static ORACLE_INLINE vec3 DecompressSR11G11B10(uint32_t data) {
    float r = (float)((data >> 0) & ((1u << 11) - 1));
    float g = (float)((data >> 11) & ((1u << 11) - 1));
    float b = (float)((data >> 22) & ((1u << 10) - 1));
    r /= 2047.0f;
    g /= 2047.0f;
    b /= 1023.0f;
    return {r * 2.0f - 1.0f, g * 2.0f - 1.0f, b * 2.0f - 1.0f};
}

static ORACLE_INLINE void EncodeUnitVec(vec3 n, float& ex, float& ey) {
    float l1 = (fabsf(n.x) + fabsf(n.y)) + fabsf(n.z);
    n = n / l1;
    float nx = n.x, ny = n.y;
    if (!(n.z > 0.0f)) {
        // OctWrap(n.xy)
        float wx = 1.0f - fabsf(n.y);
        float wy = 1.0f - fabsf(n.x);
        if (n.x < 0.0f) wx = -wx;
        if (n.y < 0.0f) wy = -wy;
        nx = wx;
        ny = wy;
    }
    ex = nx * 0.5f + 0.5f;
    ey = ny * 0.5f + 0.5f;
}
static ORACLE_INLINE vec3 DecodeUnitVec(float fx, float fy) {
    fx = fx * 2.0f - 1.0f;
    fy = fy * 2.0f - 1.0f;
    vec3 n = {fx, fy, 1.0f - fabsf(fx) - fabsf(fy)};
    float t = fmaxf(-n.z, 0.0f);
    n.x += n.x >= 0.0f ? -t : t;
    n.y += n.y >= 0.0f ? -t : t;
    return normalize(n);
}

static ORACLE_INLINE vec3 CubemapFaceNormal(vec3 dir) {
    vec3 a = {fabsf(dir.x), fabsf(dir.y), fabsf(dir.z)};
    float mx = a.x >= fmaxf(a.y, a.z) ? 1.0f : 0.0f;
    float my = a.y >= fmaxf(a.z, a.x) ? 1.0f : 0.0f;
    float mz = a.z >= fmaxf(a.x, a.y) ? 1.0f : 0.0f;
    auto sgn = [](float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); };
    return {mx * -sgn(dir.x), my * -sgn(dir.y), mz * -sgn(dir.z)};
}

// texture(skyBoxUBO.Albedo, dir).rgb (FirstHit:227, NHit:208). Face selection and (s,t) per the OpenGL 4.6 spec table
// 8.19 (major axis; ties x >= y >= z), then bilinear filtering inside the face with clamp-to-edge texel indices. Not forced
// inline: it runs once per ray that leaves the scene, and out of line it keeps its texel lambdas inlined.
struct Scene;
static inline vec3 SampleSky(const float* const faces[6], int size, const float* constant, vec3 d) {
    if (size == 0) return V(constant);
    const float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
    int face;
    float sc, tc, ma;
    if (ax >= ay && ax >= az) { face = d.x >= 0.0f ? 0 : 1; sc = d.x >= 0.0f ? -d.z : d.z; tc = -d.y; ma = ax; }
    else if (ay >= az) { face = d.y >= 0.0f ? 2 : 3; sc = d.x; tc = d.y >= 0.0f ? d.z : -d.z; ma = ay; }
    else { face = d.z >= 0.0f ? 4 : 5; sc = d.z >= 0.0f ? d.x : -d.x; tc = -d.y; ma = az; }
    const float s = 0.5f * (sc / ma + 1.0f), t = 0.5f * (tc / ma + 1.0f);
    const float px = s * (float)size - 0.5f, py = t * (float)size - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    // GL_TEXTURE_CUBE_MAP_SEAMLESS (SkyBoxManager.cs:74; OpenGL 4.6 spec 8.17): texels beyond an edge come from the face across
    // it; the missing fourth texel at a cube corner is the mean of the other three. Texel centres as odd integers
    // c = 2*texel + 1 - size on the cube [-size, size]^3: crossing an edge is an exact integer fold.
    const int x0 = (int)fx0, x1 = x0 + 1, y0 = (int)fy0, y1 = y0 + 1;
    auto inside = [&](int f, int x, int y) { const float* p = faces[f] + 4 * ((size_t)y * size + x); return V(p[0], p[1], p[2]); };
    auto tx = [&](int x, int y) -> vec3 {
        if (x >= 0 && x < size && y >= 0 && y < size) return inside(face, x, y);
        const int s2 = 2 * x + 1 - size, t2 = 2 * y + 1 - size;
        int P[3];
        switch (face) {
            case 0: P[0] = size; P[1] = -t2; P[2] = -s2; break;
            case 1: P[0] = -size; P[1] = -t2; P[2] = s2; break;
            case 2: P[0] = s2; P[1] = size; P[2] = t2; break;
            case 3: P[0] = s2; P[1] = -size; P[2] = -t2; break;
            case 4: P[0] = s2; P[1] = -t2; P[2] = size; break;
            default: P[0] = -s2; P[1] = -t2; P[2] = -size; break;
        }
        const int major = face >> 1;                       // axis of the face we came from
        int over = -1;
        for (int k = 0; k < 3; k++) if (P[k] > size || P[k] < -size) over = k;
        P[over] = P[over] > 0 ? size : -size;              // the overhanging coordinate lands on the neighbouring face ...
        P[major] += P[major] > 0 ? -1 : 1;                 // ... one half-texel step in from the shared edge
        int nf, ns, nt;
        if (over == 0) { nf = P[0] > 0 ? 0 : 1; ns = P[0] > 0 ? -P[2] : P[2]; nt = -P[1]; }
        else if (over == 1) { nf = P[1] > 0 ? 2 : 3; ns = P[0]; nt = P[1] > 0 ? P[2] : -P[2]; }
        else { nf = P[2] > 0 ? 4 : 5; ns = P[2] > 0 ? P[0] : -P[0]; nt = -P[1]; }
        return inside(nf, (ns + size - 1) / 2, (nt + size - 1) / 2);
    };
    const bool ox0 = x0 < 0, ox1 = x1 >= size, oy0 = y0 < 0, oy1 = y1 >= size;
    vec3 t00, t10, t01, t11;
    if ((ox0 || ox1) && (oy0 || oy1)) {
        const bool c00 = ox0 && oy0, c10 = ox1 && oy0, c01 = ox0 && oy1;
        const vec3 zero = V(0, 0, 0);
        t00 = c00 ? zero : tx(x0, y0); t10 = c10 ? zero : tx(x1, y0); t01 = c01 ? zero : tx(x0, y1);
        t11 = (c00 || c10 || c01) ? tx(x1, y1) : zero;
        const vec3 mean = ((t00 + t10) + (t01 + t11)) / 3.0f;
        if (c00) t00 = mean; else if (c10) t10 = mean; else if (c01) t01 = mean; else t11 = mean;
    } else {
        t00 = tx(x0, y0); t10 = tx(x1, y0); t01 = tx(x0, y1); t11 = tx(x1, y1);
    }
    const vec3 a = mix(t00, t10, fx), b = mix(t01, t11, fx);
    return mix(a, b, fy);
}

// ------------------------------------------------------------------ Surface / shading
struct Surface {
    vec3 Albedo; float Alpha;
    vec3 Normal, Emissive, Absorbance;
    float Metallic, Roughness, Transmission, IOR, AlphaCutoff;
    bool IsVolumetric, TintOnTransmissive;
};
static Surface GetDefaultSurface() {
    Surface s;
    s.Albedo = V(1, 1, 1); s.Alpha = 1.0f;
    s.Normal = V(0, 0, 0); s.Emissive = V(0, 0, 0); s.Absorbance = V(0, 0, 0);
    s.Metallic = 0.0f; s.Roughness = 0.0f; s.Transmission = 0.0f; s.IOR = 1.5f;
    s.AlphaCutoff = 0.5f; s.IsVolumetric = false; s.TintOnTransmissive = true;
    return s;
}
// Surface.glsl:49-77 with every sampler = 1x1 white (texture(...) == vec4(1)).
// texture(sampler2D, uv) at lod 0 (compute shaders have no derivatives, Surface.glsl:57-60): explicit fp32 bilinear on the base
// level, glTF wrap modes, sRGB decode before filtering. Handle 0 = 1x1 white, k = Textures[k-1] (include/idkpt.h).
struct Vec4 { float x, y, z, w; };
static ORACLE_INLINE int TexWrap(int i, int n, int mode) {
    if (mode == 33071) return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
    if (mode == 33648) { int m = i % (2 * n); if (m < 0) m += 2 * n; return m < n ? m : 2 * n - 1 - m; }
    int m = i % n;
    return m < 0 ? m + n : m;
}
static const float* SrgbLut() {
    static float lut[256];
    static bool init = false;
    if (!init) {
        for (int i = 0; i < 256; i++) {
            const double cs = i / 255.0;
            lut[i] = (float)(cs <= 0.04045 ? cs / 12.92 : pow((cs + 0.055) / 1.055, 2.4));
        }
        init = true;
    }
    return lut;
}
// The oracle samples UNCOMPRESSED texels only (RGBA8 unorm / sRGB, R / RG / RGBA 32F; GL channel defaults (R,G,0,1) for missing
// channels). Block-compressed textures reach it already decoded by tests/bcn_ref.py, an implementation that shares no code
// with the CUDA decoders (csrc/idk_bcn.cuh) -- the two are then compared through the rendered images.
static ORACLE_INLINE Vec4 TexFetch(const IdkPtTextureDesc& t, int x, int y) {
    const size_t i = (size_t)y * t.Width + x;
    Vec4 r;
    if (t.Format == IDKPT_TEX_RG32F) { const float* c = (const float*)t.Pixels + 2 * i; r = {c[0], c[1], 0.0f, 1.0f}; }
    else if (t.Format == IDKPT_TEX_R32F) { r = {((const float*)t.Pixels)[i], 0.0f, 0.0f, 1.0f}; }
    else if (t.Format == IDKPT_TEX_RGBA32F) { const float* c = (const float*)t.Pixels + 4 * i; r = {c[0], c[1], c[2], c[3]}; }
    else {
        const uint8_t* c = (const uint8_t*)t.Pixels + 4 * i;
        if (t.Format == IDKPT_TEX_RGBA8_SRGB) { const float* lut = SrgbLut(); r = {lut[c[0]], lut[c[1]], lut[c[2]], (float)c[3] / 255.0f}; }
        else r = {(float)c[0] / 255.0f, (float)c[1] / 255.0f, (float)c[2] / 255.0f, (float)c[3] / 255.0f};
    }
    if (t.Flags & IDKPT_TEX_FLAG_R_FROM_B) r.x = r.z;      // texture.SetSwizzleR(Swizzle.B), ModelLoader.cs:989-994
    return r;
}
static ORACLE_INLINE Vec4 TexLerp(Vec4 a, Vec4 b, float t) {
    const float s = 1.0f - t;
    return {a.x * s + b.x * t, a.y * s + b.y * t, a.z * s + b.z * t, a.w * s + b.w * t};
}
static Vec4 TexSample(const IdkPtSceneDesc& d, uint64_t handle, float u, float v) {
    if (handle == 0) return {1.0f, 1.0f, 1.0f, 1.0f};
    const IdkPtTextureDesc& t = d.Textures[handle - 1];
    if (t.WrapS == 10497) u = u - floorf(u);
    if (t.WrapT == 10497) v = v - floorf(v);
    if (t.Flags & IDKPT_TEX_FLAG_MAG_NEAREST)      // lod 0 = magnification: the sampler's MagFilter applies (ModelLoader.cs:1166-1196); NEAREST = the containing texel
        return TexFetch(t, TexWrap((int)floorf(u * (float)t.Width), t.Width, t.WrapS), TexWrap((int)floorf(v * (float)t.Height), t.Height, t.WrapT));
    const float px = u * (float)t.Width - 0.5f, py = v * (float)t.Height - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    const int x0 = TexWrap((int)fx0, t.Width, t.WrapS), x1 = TexWrap((int)fx0 + 1, t.Width, t.WrapS);
    const int y0 = TexWrap((int)fy0, t.Height, t.WrapT), y1 = TexWrap((int)fy0 + 1, t.Height, t.WrapT);
    const Vec4 a = TexLerp(TexFetch(t, x0, y0), TexFetch(t, x1, y0), fx);
    const Vec4 b = TexLerp(TexFetch(t, x0, y1), TexFetch(t, x1, y1), fx);
    return TexLerp(a, b, fy);
}
static ORACLE_INLINE bool MaterialHasTextures(const GpuMaterial& m) {
    return (m.BaseColorTexture | m.MetallicRoughnessTexture | m.NormalTexture | m.EmissiveTexture | m.TransmissionTexture) != 0;
}

static Surface GetSurface(const GpuMaterial& m);
// GetSurface(gpuMaterial, uv), Surface.glsl:49-77
static Surface GetSurface(const IdkPtSceneDesc& d, const GpuMaterial& m, float u, float v) {
    if (!MaterialHasTextures(m)) return GetSurface(m);
    Surface s;
    const uint32_t c = m.BaseColorFactor;
    const Vec4 base = TexSample(d, m.BaseColorTexture, u, v);
    s.Albedo = {base.x * ((float)(c & 255u) / 255.0f), base.y * ((float)((c >> 8) & 255u) / 255.0f), base.z * ((float)((c >> 16) & 255u) / 255.0f)};
    s.Alpha = base.w * ((float)((c >> 24) & 255u) / 255.0f);
    const Vec4 nt = TexSample(d, m.NormalTexture, u, v);
    s.Normal = {nt.x * 2.0f - 1.0f, nt.y * 2.0f - 1.0f, sqrtf(fmaxf(1.0f - (nt.x * nt.x + nt.y * nt.y), 0.0f))};   // ReconstructPackedNormal, Compression.glsl:78-84
    const Vec4 et = TexSample(d, m.EmissiveTexture, u, v);
    s.Emissive = {et.x * m.EmissiveFactor[0], et.y * m.EmissiveFactor[1], et.z * m.EmissiveFactor[2]};
    s.Absorbance = V(m.Absorbance);
    const Vec4 mr = TexSample(d, m.MetallicRoughnessTexture, u, v);
    s.Metallic = mr.x * m.MetallicFactor;
    s.Roughness = mr.y * m.RoughnessFactor;
    s.Transmission = TexSample(d, m.TransmissionTexture, u, v).x * m.TransmissionFactor;
    s.IOR = m.IOR;
    s.AlphaCutoff = m.AlphaCutoff;
    s.IsVolumetric = m.IsVolumetric != 0;
    s.TintOnTransmissive = true;
    return s;
}
static ORACLE_INLINE void InterpTexCoord(const IdkPtSceneDesc& d, const GpuBlasTriangle& tri, float b0, float b1, float b2, float& u, float& v) {
    const GpuVertex& v0 = d.Vertices[tri.X]; const GpuVertex& v1 = d.Vertices[tri.Y]; const GpuVertex& v2 = d.Vertices[tri.Z];
    u = (v0.TexCoord[0] * b0 + v1.TexCoord[0] * b1) + v2.TexCoord[0] * b2;   // Interpolate(), Math.glsl:54-57
    v = (v0.TexCoord[1] * b0 + v1.TexCoord[1] * b1) + v2.TexCoord[1] * b2;
}

static Surface GetSurface(const GpuMaterial& m) {
    Surface s;
    uint32_t c = m.BaseColorFactor;
    s.Albedo = {(float)(c & 255u) / 255.0f, (float)((c >> 8) & 255u) / 255.0f, (float)((c >> 16) & 255u) / 255.0f};
    s.Alpha = (float)((c >> 24) & 255u) / 255.0f;
    s.Normal = {1.0f, 1.0f, 0.0f}; // ReconstructPackedNormal(vec2(1,1))
    s.Emissive = V(m.EmissiveFactor);
    s.Absorbance = V(m.Absorbance);
    s.Metallic = m.MetallicFactor;
    s.Roughness = m.RoughnessFactor;
    s.Transmission = m.TransmissionFactor;
    s.IOR = m.IOR;
    s.AlphaCutoff = m.AlphaCutoff;
    s.IsVolumetric = m.IsVolumetric != 0;
    s.TintOnTransmissive = true;
    return s;
}
static void SurfaceApplyModificatons(Surface& s, const GpuMesh& mesh) {
    s.Emissive = s.Emissive * 1.0f + mesh.EmissiveBias * s.Albedo;
    vec3 a = s.Absorbance + V(mesh.AbsorbanceBias);
    s.Absorbance = {fmaxf(a.x, 0.0f), fmaxf(a.y, 0.0f), fmaxf(a.z, 0.0f)};
    s.Metallic = clampf(s.Metallic + mesh.SpecularBias, 0.0f, 1.0f);
    s.Roughness = clampf(s.Roughness + mesh.RoughnessBias, 0.0f, 1.0f);
    s.Transmission = clampf(s.Transmission + mesh.TransmissionBias, 0.0f, 1.0f);
    s.IOR = fmaxf(s.IOR + mesh.IORBias, 1.0f);
    s.TintOnTransmissive = mesh.TintOnTransmissive != 0;
}
static ORACLE_INLINE float GetSurfaceVariance(float specularChance, float transmissionChance, float roughness) {
    float diffuseChance = 1.0f - specularChance - transmissionChance;
    return diffuseChance + specularChance * roughness + transmissionChance * roughness;
}
static ORACLE_INLINE float pow5(float x) { float x2 = x * x; return (x2 * x2) * x; }

enum { BSDF_DIFFUSE = 0, BSDF_SPECULAR = 1, BSDF_TRANSMISSIVE = 2 };
struct SampleMaterialResult { vec3 RayDirection; uint32_t BsdfType; vec3 Bsdf; float Pdf; float NewIor; };

// Shading.glsl:52-150. gidX/gidY = gl_GlobalInvocationID of the invoking shader.
static SampleMaterialResult SampleMaterial(Rng& rng, vec3 incomming, Surface surface, float prevIor, bool fromInside,
                                           uint32_t gidX, uint32_t gidY, uint32_t accumulatedSamples) {
    surface.Roughness *= surface.Roughness;
    float cosTheta = dot(-incomming, surface.Normal);
    {
        float diffuseChance = 1.0f - surface.Metallic - surface.Transmission;
        float r0 = (prevIor - surface.IOR) / (prevIor + surface.IOR);
        float f0 = r0 * r0;
        float fres = f0 + (1.0f - f0) * pow5(1.0f - cosTheta);
        surface.Metallic = mixf(surface.Metallic, 1.0f, fres);
        surface.Transmission = fmaxf(1.0f - diffuseChance - surface.Metallic, 0.0f);
    }
    SampleMaterialResult result;
    {
        float specularChance = surface.Metallic;
        float transmissionChance = surface.Transmission;
        float rnd = GetRandomFloat01(rng);
        if (specularChance > rnd) result.BsdfType = BSDF_SPECULAR;
        else if (specularChance + transmissionChance > rnd) result.BsdfType = BSDF_TRANSMISSIVE;
        else result.BsdfType = BSDF_DIFFUSE;
    }
    uint32_t saved = rng.seed;
    rng.seed = gidY * 4096u + gidX;
    float r2u, r2v;
    R2Sequence(accumulatedSamples, r2u, r2v);
    float po0 = GetRandomFloat01(rng);
    float po1 = GetRandomFloat01(rng);
    float u = fractf(r2u + po0), v = fractf(r2v + po1);
    vec3 diffuseRayDir = CosineSampleHemisphere(surface.Normal, u, v);
    rng.seed = saved;

    if (result.BsdfType == BSDF_DIFFUSE) {
        result.RayDirection = diffuseRayDir;
        result.NewIor = prevIor;
        result.Bsdf = surface.Albedo;
        result.Pdf = 1.0f;
    } else if (result.BsdfType == BSDF_SPECULAR) {
        vec3 reflectionRayDir = reflect(incomming, surface.Normal);
        reflectionRayDir = normalize(mix(reflectionRayDir, diffuseRayDir, surface.Roughness));
        result.RayDirection = reflectionRayDir;
        result.Bsdf = surface.Albedo;
        result.Pdf = 1.0f;
        result.NewIor = prevIor;
    } else {
        result.NewIor = fromInside ? 1.0f : surface.IOR;
        vec3 refractionRayDir;
        bool totalInternalReflection;
        if (!surface.IsVolumetric) {
            refractionRayDir = incomming;
            totalInternalReflection = false;
            result.NewIor = 1.0f;
        } else {
            refractionRayDir = refract(incomming, surface.Normal, prevIor / result.NewIor);
            totalInternalReflection = refractionRayDir.x == 0.0f && refractionRayDir.y == 0.0f && refractionRayDir.z == 0.0f;
            if (totalInternalReflection) {
                refractionRayDir = reflect(incomming, surface.Normal);
                result.NewIor = prevIor;
            }
        }
        refractionRayDir = normalize(mix(refractionRayDir, !totalInternalReflection ? -diffuseRayDir : diffuseRayDir, surface.Roughness));
        result.RayDirection = refractionRayDir;
        bool gltfWantsTint = surface.IsVolumetric || !fromInside;
        result.Bsdf = (gltfWantsTint && surface.TintOnTransmissive) ? surface.Albedo : V(1, 1, 1);
        result.Pdf = 1.0f;
    }
    result.Pdf = fmaxf(result.Pdf, 0.0001f);
    return result;
}

struct WRay {  // GpuWavefrontRay in registers
    vec3 Origin; float PrevIOROrCost; vec3 Throughput; float PdX; vec3 Radiance; float PdY;
};
struct AovRay { vec3 Albedo; float NewWeight; vec3 Normal; };

struct Settings {
    IdkPtGpuSettings g;
    uint32_t accumulatedSamples;
};

struct RayStats { uint32_t steps, tris, instances; bool hitGeometry; };

// FirstHit/compute.glsl:100-234 and NHit/compute.glsl:91-215 (they differ only where marked).
static bool ShadeTraceRay(const Scene& s, const Settings& st, Rng& rng, WRay& ray, AovRay& aov, bool firstHit,
                          uint32_t gidX, uint32_t gidY, uint32_t& sortingKey, RayStats& rs) {
    vec3 rayDir = DecodeUnitVec(ray.PdX, ray.PdY);
    HitInfo hitInfo;
    Counters cnt = {0, 0, 0, 0.0f};
    bool hitScene = TraceRay(s, Ray{ray.Origin, rayDir}, hitInfo, cnt, st.g.DoTraceLights != 0, FLOAT_MAX);
    rs.steps = cnt.steps; rs.tris = cnt.tris; rs.instances = cnt.instances;
    rs.hitGeometry = hitScene && hitInfo.TriangleId != ~0u;
    sortingKey = 0;

    if (firstHit && st.g.DoDebugBVHTraversal) {
        ray.PrevIOROrCost = cnt.debugCost;
        return false;
    }

    if (hitScene) {
        ray.Origin = ray.Origin + rayDir * hitInfo.T;

        Surface surface = GetDefaultSurface();
        vec3 geometricNormal = V(0, 0, 0);
        bool hitLight = hitInfo.TriangleId == ~0u;
        if (!hitLight) {
            sortingKey = hitInfo.TriangleId;
            const GpuBlasTriangle& tri = s.d.BlasTriangles[hitInfo.TriangleId];
            const GpuVertex& v0 = s.d.Vertices[tri.X];
            const GpuVertex& v1 = s.d.Vertices[tri.Y];
            const GpuVertex& v2 = s.d.Vertices[tri.Z];
            vec3 bary = {hitInfo.bx, hitInfo.by, 1.0f - hitInfo.bx - hitInfo.by};
            float texU, texV;
            InterpTexCoord(s.d, tri, bary.x, bary.y, bary.z, texU, texV);
            vec3 n0 = DecompressSR11G11B10(v0.Normal), n1 = DecompressSR11G11B10(v1.Normal), n2 = DecompressSR11G11B10(v2.Normal);
            vec3 interpNormal = normalize((n0 * bary.x + n1 * bary.y) + n2 * bary.z);
            vec3 t0 = DecompressSR11G11B10(v0.Tangent), t1 = DecompressSR11G11B10(v1.Tangent), t2 = DecompressSR11G11B10(v2.Tangent);
            vec3 interpTangent = normalize((t0 * bary.x + t1 * bary.y) + t2 * bary.z);

            const GpuMeshTransform& mt = s.d.MeshTransforms[hitInfo.MeshTransformId];
            const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
            const GpuMaterial& material = s.d.Materials[mesh.MaterialId];

            surface = GetSurface(s.d, material, texU, texV);
            SurfaceApplyModificatons(surface, mesh);

            float alphaCutoff = (surface.AlphaCutoff == 2.0f) ? GetRandomFloat01(rng) : surface.AlphaCutoff;
            if (surface.Alpha < alphaCutoff) {
                ray.Origin = ray.Origin + rayDir * 0.001f;
                return true;
            }

            // unitVecToWorld = mat3(transpose(InvModelMatrix)):  (U*v)[i] = sum_j Inv[j][i] * v[j]
            const float (*im)[4] = mt.InvModelMatrix;
            auto toWorld = [&](vec3 v) {
                return vec3{(im[0][0] * v.x + im[1][0] * v.y) + im[2][0] * v.z,
                            (im[0][1] * v.x + im[1][1] * v.y) + im[2][1] * v.z,
                            (im[0][2] * v.x + im[1][2] * v.y) + im[2][2] * v.z};
            };
            vec3 worldNormal = normalize(toWorld(interpNormal));
            vec3 worldTangent = normalize(toWorld(interpTangent));
            // GetTBN (Math.glsl:129-137)
            vec3 N = normalize(worldNormal);
            vec3 T = normalize(worldTangent);
            vec3 B = normalize(cross(N, T));
            vec3 sn = surface.Normal; // tbn * surface.Normal = T*x + B*y + N*z
            vec3 tbnN = (T * sn.x + B * sn.y) + N * sn.z;
            surface.Normal = normalize(mix(worldNormal, tbnN, mesh.NormalMapStrength));

            vec3 p0 = pos(s, tri.X), p1 = pos(s, tri.Y), p2 = pos(s, tri.Z);
            geometricNormal = normalize(cross(p1 - p0, p2 - p0));
            geometricNormal = normalize(toWorld(geometricNormal));
        } else if (st.g.DoTraceLights) {
            sortingKey = hitInfo.MeshTransformId;
            const GpuLight& light = s.d.Lights[hitInfo.MeshTransformId];
            surface.Emissive = V(light.Color);
            surface.Albedo = V(light.Color);
            surface.Normal = (ray.Origin - V(light.Position)) / light.Radius;
            geometricNormal = surface.Normal;
        }

        float prevIor = firstHit ? 1.0f : ray.PrevIOROrCost;
        bool fromInside = dot(-rayDir, geometricNormal) < 0.0f;
        if (fromInside) {
            if (firstHit) prevIor = surface.IOR; // FirstHit:174
            geometricNormal = geometricNormal * -1.0f;
            if (surface.IsVolumetric) {
                vec3 e = -surface.Absorbance * hitInfo.T;
                ray.Throughput = ray.Throughput * V(det_exp(e.x), det_exp(e.y), det_exp(e.z));
            }
        }

        float cosTheta = dot(-rayDir, surface.Normal);
        if (cosTheta < 0.0f) {
            surface.Normal = surface.Normal * -1.0f;
            cosTheta *= -1.0f;
        }
        cosTheta = fminf(cosTheta, 1.0f);
        (void)cosTheta;

        ray.Radiance = ray.Radiance + surface.Emissive * ray.Throughput;

        SampleMaterialResult result = SampleMaterial(rng, rayDir, surface, prevIor, fromInside, gidX, gidY, st.accumulatedSamples);
        ray.Throughput = ray.Throughput * (result.Bsdf / result.Pdf);

        {
            float weight = GetSurfaceVariance(surface.Metallic, surface.Transmission, surface.Roughness);
            if (firstHit) {
                aov.Albedo = surface.Albedo * weight;
                aov.Normal = surface.Normal * weight;
                aov.NewWeight = (1.0f - weight);
            } else {
                aov.Albedo = aov.Albedo + aov.NewWeight * surface.Albedo * weight;
                aov.Normal = aov.Normal + aov.NewWeight * surface.Normal * weight;
                aov.NewWeight *= (1.0f - weight);
            }
        }

        if (!firstHit && st.g.DoRussianRoulette) {
            // RussianRoulette.glsl:3-12
            float p = fmaxf(ray.Throughput.x, fmaxf(ray.Throughput.y, ray.Throughput.z));
            if (GetRandomFloat01(rng) > p) return false;
            ray.Throughput = ray.Throughput / p;
        }

        if (result.BsdfType == BSDF_TRANSMISSIVE) geometricNormal = geometricNormal * -1.0f;
        ray.Origin = ray.Origin + geometricNormal * 0.001f;
        ray.PrevIOROrCost = result.NewIor;
        EncodeUnitVec(result.RayDirection, ray.PdX, ray.PdY);
        return true;
    } else {
        vec3 albedo = SampleSky(s.skyFaces, s.skyFaceSize, s.skyColor, rayDir);
        if (firstHit) {
            aov.Albedo = albedo;
            aov.Normal = CubemapFaceNormal(rayDir);
        } else {
            aov.Albedo = aov.Albedo + aov.NewWeight * albedo;
            aov.Normal = aov.Normal + aov.NewWeight * CubemapFaceNormal(rayDir);
        }
        aov.NewWeight = 0.0f;
        ray.Radiance = ray.Radiance + albedo * ray.Throughput;
        return false;
    }
}

// FirstHit/compute.glsl:236-262 for every work group: swizzled group -> un-swizzled gl_WorkGroupID
static void BuildSwizzleInverse(uint32_t ngx, uint32_t ngy, uint32_t n, std::vector<uint32_t>& inv) {
    inv.assign((size_t)ngx * ngy, 0);
    for (uint32_t wy = 0; wy < ngy; wy++) {
        for (uint32_t wx = 0; wx < ngx; wx++) {
            uint32_t idx = wy * ngx + wx;
            uint32_t columnSize = ngy * n;
            uint32_t fullColumnCount = ngx / n;
            uint32_t lastColumnWidth = ngx % n;
            uint32_t columnIdx = idx / columnSize;
            uint32_t idxInColumn = idx % columnSize;
            uint32_t columnWidth = n;
            if (columnIdx == fullColumnCount) columnWidth = lastColumnWidth;
            uint32_t sy = idxInColumn / columnWidth;
            uint32_t sx = idxInColumn % columnWidth + columnIdx * n;
            inv[(size_t)sy * ngx + sx] = idx;
        }
    }
}

static vec3 mat4MulXYZ(const float* m, float x, float y, float z, float w) {
    // GLSL column-major: (M*v)[i] = sum_c M[c*4+i]*v[c]
    return {((m[0] * x + m[4] * y) + m[8] * z) + m[12] * w,
            ((m[1] * x + m[5] * y) + m[9] * z) + m[13] * w,
            ((m[2] * x + m[6] * y) + m[10] * z) + m[14] * w};
}

static vec3 TurboColormap(float x) {
    x = clampf(x, 0.0f, 1.0f);
    float v4[4] = {1.0f, x, x * x, x * x * x};
    float v2[2] = {v4[2] * v4[2], v4[3] * v4[2]};
    auto d4 = [&](float a, float b, float c, float d) { return ((v4[0] * a + v4[1] * b) + v4[2] * c) + v4[3] * d; };
    auto d2 = [&](float a, float b) { return v2[0] * a + v2[1] * b; };
    return {d4(0.13572138f, 4.61539260f, -42.66032258f, 132.13108234f) + d2(-152.94239396f, 59.28637943f),
            d4(0.09140261f, 2.19418839f, 4.84296658f, -14.18503333f) + d2(4.27729857f, 2.82956604f),
            d4(0.10667330f, 12.64194608f, -60.58204836f, 110.36276771f) + d2(-89.90310912f, 27.34824973f)};
}

// Persistent worker pool with dynamic chunking (round-1 verdict: spawning `threads` fresh std::threads per phase per bounce
// made the CPU arm noisy by 2x between boxes). Workers are created once and parked on a condition variable; a job is a
// range cut into chunks that the workers (and the calling thread, as worker 0) claim with an atomic counter, so uneven
// rows / rays balance themselves. f(begin, end, workerId) may be called several times per worker. Every entry point of
// liboracle.so shares the one pool, and it runs one job at a time.
class WorkerPool {
public:
    static WorkerPool& get() { static WorkerPool p; return p; }
    template <typename F>
    void run(size_t n, int threads, F& f) {
        std::unique_lock<std::mutex> runLock(runMutex_);          // one job at a time (callers are single-threaded anyway)
        const int want = std::max(1, threads);
        grow(want - 1);
        const size_t chunk = std::max<size_t>(64, n / ((size_t)want * 8));
        Job job;
        job.n = n; job.chunk = chunk; job.next.store(0); job.active = want - 1;
        job.fn = [&f](size_t b, size_t e, int tid) { f(b, e, tid); };
        {
            std::lock_guard<std::mutex> lk(m_);
            job_ = &job; generation_++; pending_ = want - 1;
        }
        cv_.notify_all();
        work(job, 0);
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [&] { return pending_ == 0; });
        job_ = nullptr;
    }
private:
    struct Job { size_t n, chunk; std::atomic<size_t> next; int active; std::function<void(size_t, size_t, int)> fn; };
    static void work(Job& j, int tid) {
        for (;;) {
            const size_t b = j.next.fetch_add(j.chunk);
            if (b >= j.n) break;
            j.fn(b, std::min(j.n, b + j.chunk), tid);
        }
    }
    void grow(int workers) {
        while ((int)threads_.size() < workers) {
            const int tid = (int)threads_.size() + 1;
            threads_.emplace_back([this, tid]() {
                uint64_t seen = 0;
                for (;;) {
                    Job* j = nullptr;
                    {
                        std::unique_lock<std::mutex> lk(m_);
                        cv_.wait(lk, [&] { return stop_ || (generation_ != seen && job_ && tid <= job_->active); });
                        if (stop_) return;
                        seen = generation_;
                        j = job_;
                    }
                    work(*j, tid);
                    std::lock_guard<std::mutex> lk(m_);
                    if (--pending_ == 0) done_.notify_all();
                }
            });
        }
    }
    ~WorkerPool() {
        { std::lock_guard<std::mutex> lk(m_); stop_ = true; }
        cv_.notify_all();
        for (auto& t : threads_) t.join();
    }
    std::mutex m_, runMutex_;
    std::condition_variable cv_, done_;
    std::vector<std::thread> threads_;
    Job* job_ = nullptr;
    uint64_t generation_ = 0;
    int pending_ = 0;
    bool stop_ = false;
};

template <typename F>
static void parallel_for(size_t n, int threads, F f) {
    if (threads <= 1 || n < 256) { f(0, n, 0); return; }
    WorkerPool::get().run(n, threads, f);
}

} // namespace

extern "C" {

#define ORACLE_API __attribute__((visibility("default")))

// GLSL-semantics closest hit for a batch of rays (BVHIntersect.glsl TraceRay).
ORACLE_API int oracle_trace_rays(const IdkPtSceneDesc* scene, const IdkPtRay* rays, uint64_t count, int traceLights, IdkPtHit* out, int threads) {
    Scene s; s.d = *scene; s.skyColor[0] = s.skyColor[1] = s.skyColor[2] = 0.0f;
    parallel_for(count, threads, [&](size_t b, size_t e, int) {
        for (size_t i = b; i < e; i++) {
            HitInfo h; Counters c = {0, 0, 0, 0.0f};
            TraceRay(s, Ray{V(rays[i].Origin), V(rays[i].Direction)}, h, c, traceLights != 0, rays[i].TMax);
            out[i] = IdkPtHit{h.bx, h.by, h.T, h.TriangleId, h.MeshTransformId, c.steps, c.tris, 0};
        }
    });
    return 0;
}

ORACLE_API int oracle_brute_force(const IdkPtSceneDesc* scene, const IdkPtRay* rays, uint64_t count, IdkPtHit* out, int threads) {
    Scene s; s.d = *scene;
    parallel_for(count, threads, [&](size_t b, size_t e, int) {
        for (size_t i = b; i < e; i++) {
            HitInfo h;
            BruteForce(s, Ray{V(rays[i].Origin), V(rays[i].Direction)}, h, rays[i].TMax);
            out[i] = IdkPtHit{h.bx, h.by, h.T, h.TriangleId, h.MeshTransformId, 0, 0, 0};
        }
    });
    return 0;
}

// C#-semantics BVH.Intersect for a batch of rays: the reference's CPU (collision / picking) traversal.
// Returns elapsed seconds of the traversal loop (threads = worker count).
ORACLE_API double oracle_cpu_intersect(const IdkPtSceneDesc* scene, const IdkPtRay* rays, uint64_t count, IdkPtHit* out, int threads) {
    Scene s; s.d = *scene;
    auto t0 = std::chrono::steady_clock::now();
    parallel_for(count, threads, [&](size_t b, size_t e, int) {
        for (size_t i = b; i < e; i++) {
            HitInfo h; Counters c = {0, 0, 0, 0.0f};
            CsBvhIntersect(s, Ray{V(rays[i].Origin), V(rays[i].Direction)}, h, rays[i].TMax, c);
            if (out) out[i] = IdkPtHit{h.bx, h.by, h.T, h.TriangleId, h.MeshTransformId, c.steps * 2 /*BoxIntersections*/, c.tris, 0};
        }
    });
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// Primary camera rays exactly as Gui.Test builds them (Gui.cs:1484-1503, Ray.cs:30-39): ndc = (x,y)/res*2-1.
ORACLE_API void oracle_gui_test_rays(const GpuPerFrameData* f, int width, int height, int y0, int y1, IdkPtRay* out) {
    size_t k = 0;
    for (int y = y0; y < y1; y++) {
        for (int x = 0; x < width; x++) {
            float nx = (float)x / (float)width * 2.0f - 1.0f;
            float ny = (float)y / (float)height * 2.0f - 1.0f;
            const float* ip = f->InvProjection;
            // ndc * Matrix2(Row0.Xy, Row1.Xy) (row vector)
            float vx = nx * ip[0] + ny * ip[4];
            float vy = nx * ip[1] + ny * ip[5];
            const float* iv = f->InvView;
            // (rayView * inverseView).Xyz, row vector times row-major OpenTK matrix
            vec3 w = {vx * iv[0] + vy * iv[4] + -1.0f * iv[8] + 0.0f * iv[12],
                      vx * iv[1] + vy * iv[5] + -1.0f * iv[9] + 0.0f * iv[13],
                      vx * iv[2] + vy * iv[6] + -1.0f * iv[10] + 0.0f * iv[14]};
            float len = sqrtf(w.x * w.x + w.y * w.y + w.z * w.z);
            w = {w.x / len, w.y / len, w.z / len};
            IdkPtRay r = {{f->ViewPos[0], f->ViewPos[1], f->ViewPos[2]}, FLOAT_MAX, {w.x, w.y, w.z}, 0.0f};
            out[k++] = r;
        }
    }
}

// PathTracer.Compute() (PathTracer.cs:214-271) on the CPU with canonical compaction order.
// result/albedo/normal: full-image rgba32f (W*H*4 floats), updated in place on the tile's rows.
// raysOut (optional): GpuWavefrontRay[W*H] = SSBO 30 after the last sample (tile rows only).
ORACLE_API int oracle_path_trace(const IdkPtSceneDesc* scene, const IdkPtSkyDesc* sky, const GpuPerFrameData* frame,
                                 const IdkPtSettings* settings, int width, int height,
                                 int tileStripeHeight, int tileIndex, int tileCount,
                                 uint32_t* accumulatedSamples, float* result, float* albedoImg, float* normalImg,
                                 GpuWavefrontRay* raysOut, IdkPtStats* stats, int threads) {
    Scene s; s.d = *scene;
    for (int i = 0; i < 3; i++) s.skyColor[i] = sky ? sky->Color[i] : 0.0f;
    if (sky && sky->FaceSize > 0) { s.skyFaceSize = sky->FaceSize; for (int i = 0; i < 6; i++) s.skyFaces[i] = sky->Faces[i]; }
    if (tileCount < 1) tileCount = 1;
    if (tileStripeHeight <= 0) tileStripeHeight = 8;

    std::vector<int> rows;
    for (int y = 0; y < height; y++) if (((y / tileStripeHeight) % tileCount) == tileIndex) rows.push_back(y);
    const size_t nLocal = rows.size() * (size_t)width;

    const uint32_t ngx = (uint32_t)((width + 7) / 8), ngy = (uint32_t)((height + 7) / 8);
    std::vector<uint32_t> swzInv;
    BuildSwizzleInverse(ngx, ngy, 20, swzInv);

    std::vector<WRay> rays(nLocal);
    std::vector<AovRay> aovs(nLocal);
    std::vector<uint32_t> alive, aliveNext, keys, keysNext;
    std::vector<uint8_t> cont(nLocal);
    std::vector<uint32_t> keyOf(nLocal);
    if (stats) memset(stats, 0, sizeof(*stats));
    const int T = std::max(1, threads);
    std::vector<uint64_t> accS(T), accT(T), accI(T), accH(T);

    auto t0 = std::chrono::steady_clock::now();
    for (int sample = 0; sample < settings->SamplesPerPixel; sample++) {
        Settings st; st.g = settings->Gpu; st.accumulatedSamples = *accumulatedSamples;
        std::fill(accS.begin(), accS.end(), 0); std::fill(accT.begin(), accT.end(), 0);
        std::fill(accI.begin(), accI.end(), 0); std::fill(accH.begin(), accH.end(), 0);

        // ---- FirstHit (FirstHit/compute.glsl:44-98)
        parallel_for(nLocal, T, [&](size_t b, size_t e, int tid) {
            uint64_t lS = 0, lT = 0, lI = 0, lH = 0;      // per-chunk sums: the per-worker slots share cache lines
            for (size_t li = b; li < e; li++) {
                int x = (int)(li % (size_t)width), y = rows[li / (size_t)width];
                uint32_t unsw = swzInv[(size_t)(y / 8) * ngx + (size_t)(x / 8)];
                uint32_t gidX = (unsw % ngx) * 8u + (uint32_t)(x % 8), gidY = (unsw / ngx) * 8u + (uint32_t)(y % 8);
                Rng rng; rng.seed = (uint32_t)(y * 4096 + x) * (st.accumulatedSamples + 1u);
                float sx = GetRandomFloat01(rng), sy = GetRandomFloat01(rng);
                float ndcx = ((float)x + sx) / (float)width * 2.0f - 1.0f;
                float ndcy = ((float)y + sy) / (float)height * 2.0f - 1.0f;
                const float* ip = frame->InvProjection;
                float rvx = ip[0] * ndcx + ip[4] * ndcy; // mat2(inverseProj) * ndc
                float rvy = ip[1] * ndcx + ip[5] * ndcy;
                vec3 camDir = normalize(mat4MulXYZ(frame->InvView, rvx, rvy, -1.0f, 0.0f));
                vec3 focalPoint = V(frame->ViewPos) + camDir * st.g.FocalLength;
                float dx, dy;
                SampleDisk(rng, dx, dy);
                vec3 pointOnLense = mat4MulXYZ(frame->InvView, st.g.LenseRadius * dx, st.g.LenseRadius * dy, 0.0f, 1.0f);
                camDir = normalize(focalPoint - pointOnLense);

                WRay r;
                r.Origin = pointOnLense;
                EncodeUnitVec(camDir, r.PdX, r.PdY);
                r.Throughput = V(1, 1, 1);
                r.Radiance = V(0, 0, 0);
                r.PrevIOROrCost = 1.0f;
                AovRay a = {V(0, 0, 0), 1.0f, V(0, 0, 0)};
                uint32_t key; RayStats rs;
                bool c = ShadeTraceRay(s, st, rng, r, a, true, gidX, gidY, key, rs);
                rays[li] = r; aovs[li] = a; cont[li] = c ? 1 : 0;
                lS += rs.steps; lT += rs.tris; lI += rs.instances; lH += rs.hitGeometry ? 1 : 0;
            }
            accS[tid] += lS; accT[tid] += lT; accI[tid] += lI; accH[tid] += lH;
        });
        alive.clear();
        for (size_t li = 0; li < nLocal; li++) if (cont[li]) alive.push_back((uint32_t)li);
        if (stats) { stats->Rays += nLocal; stats->BounceRays[0] += nLocal; }

        // ---- bounces (PathTracer.cs:228-255)
        for (int j = 1; j < settings->RayDepth; j++) {
            if (settings->DoRaySorting && j > 1) {
                // CountingSort/**: stable sort of the alive list by the cached 21-bit key
                std::vector<uint32_t> order(alive.size());
                for (size_t i = 0; i < order.size(); i++) order[i] = (uint32_t)i;
                std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
                std::vector<uint32_t> sorted(alive.size());
                for (size_t i = 0; i < order.size(); i++) sorted[i] = alive[order[i]];
                alive.swap(sorted);
            }
            const size_t n = alive.size();
            if (stats) { stats->Rays += n; if (j < IDKPT_MAX_RAY_DEPTH) stats->BounceRays[j] += n; }
            std::vector<uint8_t> c2(n);
            std::vector<uint32_t> k2(n);
            parallel_for(n, T, [&](size_t b, size_t e, int tid) {
                uint64_t lS = 0, lT = 0, lI = 0, lH = 0;
                for (size_t gid = b; gid < e; gid++) {
                    Rng rng; rng.seed = (uint32_t)gid * 4096u + st.accumulatedSamples;
                    uint32_t rayIndex = alive[gid];
                    WRay r = rays[rayIndex];
                    AovRay a = aovs[rayIndex];
                    uint32_t key; RayStats rs;
                    bool c = ShadeTraceRay(s, st, rng, r, a, false, (uint32_t)gid, 0u, key, rs);
                    rays[rayIndex] = r; aovs[rayIndex] = a;
                    c2[gid] = c ? 1 : 0; k2[gid] = key & (~0u >> (32 - 21));
                    lS += rs.steps; lT += rs.tris; lI += rs.instances; lH += rs.hitGeometry ? 1 : 0;
                }
                accS[tid] += lS; accT[tid] += lT; accI[tid] += lI; accH[tid] += lH;
            });
            aliveNext.clear(); keysNext.clear();
            for (size_t gid = 0; gid < n; gid++) if (c2[gid]) { aliveNext.push_back(alive[gid]); keysNext.push_back(k2[gid]); }
            alive.swap(aliveNext); keys.swap(keysNext);
        }

        // ---- FinalDraw (FinalDraw/compute.glsl:24-62)
        const float w = 1.0f / ((float)st.accumulatedSamples + 1.0f);
        for (size_t li = 0; li < nLocal; li++) {
            int x = (int)(li % (size_t)width), y = rows[li / (size_t)width];
            size_t p = ((size_t)y * width + x) * 4;
            vec3 nr = rays[li].Radiance;
            if (st.g.DoDebugBVHTraversal) nr = TurboColormap(rays[li].PrevIOROrCost / 150.0f);
            vec3 last = {result[p], result[p + 1], result[p + 2]};
            vec3 o = mix(last, nr, w);
            result[p] = o.x; result[p + 1] = o.y; result[p + 2] = o.z; result[p + 3] = 1.0f;
            if (settings->OutputAOVs && albedoImg && normalImg) {
                vec3 la = {albedoImg[p], albedoImg[p + 1], albedoImg[p + 2]};
                vec3 oa = mix(la, aovs[li].Albedo, w);
                albedoImg[p] = oa.x; albedoImg[p + 1] = oa.y; albedoImg[p + 2] = oa.z; albedoImg[p + 3] = 1.0f;
                vec3 ln = {normalImg[p], normalImg[p + 1], normalImg[p + 2]};
                vec3 on = mix(ln, aovs[li].Normal, w);
                normalImg[p] = on.x; normalImg[p + 1] = on.y; normalImg[p + 2] = on.z; normalImg[p + 3] = 1.0f;
            }
        }
        (*accumulatedSamples)++;
        if (stats) for (int t = 0; t < T; t++) { stats->NodePairFetches += accS[t]; stats->TriangleTests += accT[t]; stats->InstanceVisits += accI[t]; stats->Hits += accH[t]; }
    }
    if (stats) stats->TotalMs = (float)(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() * 1000.0);

    if (raysOut) {
        for (size_t li = 0; li < nLocal; li++) {
            int x = (int)(li % (size_t)width), y = rows[li / (size_t)width];
            GpuWavefrontRay& o = raysOut[(size_t)y * width + x];
            const WRay& r = rays[li];
            o.Origin[0] = r.Origin.x; o.Origin[1] = r.Origin.y; o.Origin[2] = r.Origin.z;
            o.PreviousIOROrTraverseCost = r.PrevIOROrCost;
            o.Throughput[0] = r.Throughput.x; o.Throughput[1] = r.Throughput.y; o.Throughput[2] = r.Throughput.z;
            o.PackedDirectionX = r.PdX;
            o.Radiance[0] = r.Radiance.x; o.Radiance[1] = r.Radiance.y; o.Radiance[2] = r.Radiance.z;
            o.PackedDirectionY = r.PdY;
        }
    }
    return 0;
}

// texture(samplerCube, dir) on its own (unit tests of the seamless filtering)
ORACLE_API void oracle_sample_sky(const IdkPtSkyDesc* sky, const float* dirs, uint64_t n, float* out3) {
    const float* faces[6];
    for (int i = 0; i < 6; i++) faces[i] = sky->Faces[i];
    for (uint64_t i = 0; i < n; i++) {
        const vec3 c = SampleSky(faces, sky->FaceSize, sky->Color, V(dirs + 3 * i));
        out3[3 * i] = c.x; out3[3 * i + 1] = c.y; out3[3 * i + 2] = c.z;
    }
}

// exposed for unit tests of the deterministic math against libm
ORACLE_API void oracle_det_sincos(const float* x, uint64_t n, float* s, float* c) { for (uint64_t i = 0; i < n; i++) det_sincos(x[i], &s[i], &c[i]); }
ORACLE_API void oracle_det_exp(const float* x, uint64_t n, float* y) { for (uint64_t i = 0; i < n; i++) y[i] = det_exp(x[i]); }
ORACLE_API void oracle_encode_decode(const float* dirs, uint64_t n, float* enc2, float* dec3) {
    for (uint64_t i = 0; i < n; i++) {
        EncodeUnitVec(V(dirs + 3 * i), enc2[2 * i], enc2[2 * i + 1]);
        vec3 d = DecodeUnitVec(enc2[2 * i], enc2[2 * i + 1]);
        dec3[3 * i] = d.x; dec3[3 * i + 1] = d.y; dec3[3 * i + 2] = d.z;
    }
}
ORACLE_API uint32_t oracle_pcg(uint32_t seed, uint32_t* nextSeed) { uint32_t s = seed; uint32_t r = GetPCGHash(s); *nextSeed = s; return r; }

} // extern "C"

#include "oracle_vxgi.inc"

// ------------------------------------------------------------------------------------------------ "next" rows (SURVEY 8f.1)
// Any-hit traversal (BVHIntersect.glsl:107-181, 299-411) and the ray-traced point-light shadow pass
// (ShadowsRayTraced/compute.glsl, dispatched by PointShadowManager.ComputeRayTracedShadowMaps, PointShadowManager.cs:53-75).
namespace {

// IntersectBlasAny, BVHIntersect.glsl:107-181: left-first descent, returns at the first accepted triangle.
static bool IntersectBlasAny(const Scene& s, const Ray& ray, const GpuBlasDesc& blasDesc, HitInfo& hitInfo, bool useTlas) {
    float tMinLeft, tMinRight;
    const GpuBlasNode* nodes = s.d.BlasNodes + blasDesc.NodeOffset;
    vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};
    if (!useTlas) {
        const GpuBlasNode& rootNode = nodes[1];
        if (!(RayBoxIntersect(ray, invDir, rootNode.Min, rootNode.Max, tMinLeft) && tMinLeft < hitInfo.T)) return false;
    }
    uint32_t stack[256];
    uint32_t stackPtr = 0, stackTop = 2;
    while (true) {
        const GpuBlasNode& leftNode = nodes[stackTop];
        const GpuBlasNode& rightNode = nodes[stackTop + 1];
        bool hitLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft <= hitInfo.T;
        bool hitRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight <= hitInfo.T;
        bool intersectLeft = hitLeft && leftNode.TriCount > 0;
        bool intersectRight = hitRight && rightNode.TriCount > 0;
        if (intersectLeft || intersectRight) {
            uint32_t first = intersectLeft ? (uint32_t)leftNode.TriStartOrChild : (uint32_t)rightNode.TriStartOrChild;
            uint32_t end = !intersectRight ? (uint32_t)(leftNode.TriStartOrChild + leftNode.TriCount) : (uint32_t)(rightNode.TriStartOrChild + rightNode.TriCount);
            first += (uint32_t)blasDesc.TriangleOffset;
            end += (uint32_t)blasDesc.TriangleOffset;
            for (uint32_t i = first; i < end; i++) {
                const GpuBlasTriangle& tri = s.d.BlasTriangles[i];
                vec3 bary;
                float hitT;
                if (RayTriangleIntersect(ray, pos(s, tri.X), pos(s, tri.Y), pos(s, tri.Z), bary, hitT) && hitT < hitInfo.T) {
                    hitInfo.TriangleId = i;
                    hitInfo.bx = bary.x;
                    hitInfo.by = bary.y;
                    hitInfo.T = hitT;
                    return true;
                }
            }
        }
        bool traverseLeft = hitLeft && leftNode.TriCount == 0;
        bool traverseRight = hitRight && rightNode.TriCount == 0;
        if (traverseLeft || traverseRight) {
            if (traverseLeft && traverseRight) {
                stackTop = leftNode.TriStartOrChild;
                stack[stackPtr++] = rightNode.TriStartOrChild;
            } else {
                stackTop = traverseLeft ? leftNode.TriStartOrChild : rightNode.TriStartOrChild;
            }
        } else {
            if (stackPtr == 0) break;
            stackTop = stack[--stackPtr];
        }
    }
    return false;
}

// TraceRayAny, BVHIntersect.glsl:299-411 (no-TLAS instance loop and TLAS walk)
static bool TraceRayAny(const Scene& s, const Ray& ray, HitInfo& hitInfo, bool traceLights, float maxDist) {
    hitInfo.T = maxDist;
    hitInfo.TriangleId = ~0u;
    hitInfo.MeshTransformId = 0;
    hitInfo.bx = hitInfo.by = 0.0f;
    if (traceLights) {
        float tMin, tMax;
        for (uint64_t i = 0; i < s.d.LightCount; i++) {
            const GpuLight& light = s.d.Lights[i];
            if (RaySphereIntersect(ray, V(light.Position), light.Radius, tMin, tMax) && tMin < hitInfo.T) {
                hitInfo.T = tMin < 0.0f ? tMax : tMin;
                hitInfo.MeshTransformId = (uint32_t)i;
                return true;
            }
        }
    }
    if (s.d.UseTlas) {
        float tMinLeft, tMinRight;
        uint32_t stackPtr = 0, stackTop = 0;
        uint32_t stack[24];
        vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};
        while (true) {
            const GpuTlasNode& parent = s.d.TlasNodes[stackTop];
            bool isLeaf = (parent.IsLeafAndChildOrInstanceId >> 31) == 1;
            uint32_t id = parent.IsLeafAndChildOrInstanceId & ((1u << 31) - 1);
            if (isLeaf) {
                const GpuBlasInstance& inst = s.d.BlasInstances[id];
                Ray localRay = RayTransform(ray, s.d.MeshTransforms[inst.MeshTransformId].InvModelMatrix);
                if (IntersectBlasAny(s, localRay, s.d.BlasDescs[inst.BlasId], hitInfo, true)) { hitInfo.MeshTransformId = inst.MeshTransformId; return true; }
                if (stackPtr == 0) break;
                stackTop = stack[--stackPtr];
                continue;
            }
            const GpuTlasNode& leftNode = s.d.TlasNodes[id];
            const GpuTlasNode& rightNode = s.d.TlasNodes[id + 1];
            bool traverseLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft < hitInfo.T;
            bool traverseRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight < hitInfo.T;
            if (traverseLeft || traverseRight) {
                if (traverseLeft && traverseRight) {
                    bool leftCloser = tMinLeft < tMinRight;
                    stackTop = leftCloser ? id : id + 1;
                    stack[stackPtr++] = leftCloser ? id + 1 : id;
                } else {
                    stackTop = traverseLeft ? id : id + 1;
                }
            } else {
                if (stackPtr == 0) break;
                stackTop = stack[--stackPtr];
            }
        }
    } else {
        for (uint64_t i = 0; i < s.d.BlasInstanceCount; i++) {
            const GpuBlasInstance& inst = s.d.BlasInstances[i];
            Ray localRay = RayTransform(ray, s.d.MeshTransforms[inst.MeshTransformId].InvModelMatrix);
            if (IntersectBlasAny(s, localRay, s.d.BlasDescs[inst.BlasId], hitInfo, false)) { hitInfo.MeshTransformId = inst.MeshTransformId; return true; }
        }
    }
    return false;
}

// Math.glsl:104-117 ConstructBasis, Sampling.glsl:21-33 SampleCone, :35-57 SampleSphere(toSphere, radius, ...)
static vec3 SampleSphereLight(vec3 toSphere, float sphereRadius, float rnd0, float rnd1, float& distanceToSphere) {
    float radiusSq = sphereRadius * sphereRadius;
    float distanceSq = dot(toSphere, toSphere);
    float sinThetaMaxSq = radiusSq / distanceSq;
    float cosThetaMax = sqrtf(fmaxf(1.0f - sinThetaMaxSq, 0.0f));
    float phiMax = 2.0f * PI_F;
    float phi = phiMax * rnd0;
    float cosTheta = mixf(cosThetaMax, 1.0f, fmaxf(rnd1, 0.001f));
    float sinTheta = sqrtf(fmaxf(1.0f - cosTheta * cosTheta, 0.0f));
    distanceToSphere = sqrtf(dot(toSphere, toSphere)) * cosTheta - sqrtf(fmaxf(radiusSq - distanceSq * sinTheta * sinTheta, 0.0f));
    vec3 normal = normalize(toSphere);
    float sinPhi, cosPhi;
    det_sincos(phi, &sinPhi, &cosPhi);
    vec3 local = {cosPhi * sinTheta, cosTheta, sinPhi * sinTheta};
    vec3 up = fabsf(normal.z) < 0.999f ? V(0.0f, 0.0f, 1.0f) : V(1.0f, 0.0f, 0.0f);
    vec3 tangent = normalize(cross(up, normal));
    vec3 bitangent = cross(normal, tangent);
    // mat3(tangent, normal, bitangent) * local
    return (tangent * local.x + normal * local.y) + bitangent * local.z;
}

} // namespace

extern "C" {

ORACLE_API int oracle_trace_rays_any(const IdkPtSceneDesc* scene, const IdkPtRay* rays, uint64_t count, int traceLights, IdkPtHit* out, int threads) {
    Scene s; s.d = *scene;
    parallel_for(count, threads, [&](size_t b, size_t e, int) {
        for (size_t i = b; i < e; i++) {
            HitInfo h;
            bool hit = TraceRayAny(s, Ray{V(rays[i].Origin), V(rays[i].Direction)}, h, traceLights != 0, rays[i].TMax);
            out[i] = IdkPtHit{h.bx, h.by, h.T, h.TriangleId, h.MeshTransformId, hit ? 1u : 0u, 0, 0};
        }
    });
    return 0;
}

// ShadowsRayTraced/compute.glsl for one light: visibility image [height][width] (untouched where depth == 1).
ORACLE_API int oracle_shadows_ray_traced(const IdkPtSceneDesc* scene, const GpuPerFrameData* frame, const float* depth, const float* normalRG,
                                         int width, int height, int lightIndex, int samples, uint32_t noiseIndex0, const float* taaJitter,
                                         float* visibilityOut, int threads) {
    Scene s; s.d = *scene;
    if (lightIndex < 0 || (uint64_t)lightIndex >= s.d.LightCount || samples < 1) return -1;
    const GpuLight& light = s.d.Lights[lightIndex];
    parallel_for((size_t)height, threads, [&](size_t yb, size_t ye, int) {
        for (size_t y = yb; y < ye; y++)
            for (int x = 0; x < width; x++) {
                const size_t p = y * width + x;
                const float d = depth[p];
                if (d == 1.0f) continue;
                const float u = ((float)x + 0.5f) / (float)width, v = ((float)y + 0.5f) / (float)height;
                const float nx = (u * 2.0f - 1.0f) - taaJitter[0], ny = (v * 2.0f - 1.0f) - taaJitter[1];
                const float* m = frame->InvProjView;
                const float wx = ((m[0] * nx + m[4] * ny) + m[8] * d) + m[12] * 1.0f;
                const float wy = ((m[1] * nx + m[5] * ny) + m[9] * d) + m[13] * 1.0f;
                const float wz = ((m[2] * nx + m[6] * ny) + m[10] * d) + m[14] * 1.0f;
                const float ww = ((m[3] * nx + m[7] * ny) + m[11] * d) + m[15] * 1.0f;
                vec3 fragPos = {wx / ww, wy / ww, wz / ww};
                vec3 normal = DecodeUnitVec(normalRG[2 * p], normalRG[2 * p + 1]);
                float cosTheta = dot(normal, normalize(V(light.Position) - fragPos));
                if (cosTheta <= 0.0f) { visibilityOut[p] = 0.0f; continue; }
                float visibility = 0.0f;
                uint32_t noiseIndex = noiseIndex0;
                for (int i = 0; i < samples; i++) {
                    vec3 biasedPosition = fragPos + normal * 0.01f;
                    float rnd0 = InterleavedGradientNoise((float)x, (float)y, noiseIndex + 0);
                    float rnd1 = InterleavedGradientNoise((float)x, (float)y, noiseIndex + 1);
                    noiseIndex++;
                    vec3 fragToLight = V(light.Position) - biasedPosition;
                    float distanceToLight;
                    vec3 direction = SampleSphereLight(fragToLight, light.Radius, rnd0, rnd1, distanceToLight);
                    Ray ray = {biasedPosition, direction};
                    HitInfo hitInfo;
                    Counters cnt = {0, 0, 0, 0.0f};
                    float thisVisibility = 1.0f;
                    while (TraceRay(s, ray, hitInfo, cnt, true, distanceToLight - 0.001f)) {
                        if (hitInfo.TriangleId == ~0u) {
                            if (hitInfo.MeshTransformId != (uint32_t)lightIndex) thisVisibility = 0.0f;
                            break;
                        }
                        const GpuBlasTriangle& tri = s.d.BlasTriangles[hitInfo.TriangleId];
                        const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
                        float texU, texV;
                        InterpTexCoord(s.d, tri, hitInfo.bx, hitInfo.by, 1.0f - hitInfo.bx - hitInfo.by, texU, texV);
                        Surface surface = GetSurface(s.d, s.d.Materials[mesh.MaterialId], texU, texV);
                        SurfaceApplyModificatons(surface, mesh);
                        if (surface.AlphaCutoff == 2.0f) thisVisibility *= 1.0f - surface.Alpha;
                        else if (surface.Alpha > surface.AlphaCutoff) thisVisibility = 0.0f;
                        if (thisVisibility < 0.01f) break;
                        float dist = hitInfo.T + 0.001f;
                        ray.o = ray.o + ray.d * dist;
                        distanceToLight -= dist;
                    }
                    visibility += thisVisibility;
                }
                visibilityOut[p] = visibility / (float)samples;
            }
    });
    return 0;
}

} // extern "C"

// ---- dynamic geometry (SURVEY.md 8f.2) --------------------------------------------------------------------------------------
// Test infrastructure like the rest of this file: CPU restatement of Skinning/compute.glsl and of BLAS.Refit.

static ORACLE_INLINE uint32_t CompressSR11G11B10(vec3 v) {
    // Compression.glsl:1-28; round() half-way case: floor(x + 0.5) (GLSL leaves it to the implementation)
    const float x = v.x * 0.5f + 0.5f, y = v.y * 0.5f + 0.5f, z = v.z * 0.5f + 0.5f;
    const uint32_t r = (uint32_t)floorf(x * 2047.0f + 0.5f);
    const uint32_t g = (uint32_t)floorf(y * 2047.0f + 0.5f);
    const uint32_t b = (uint32_t)floorf(z * 1023.0f + 0.5f);
    return (b << 22) | (g << 11) | r;
}

extern "C" {

// Skinning/compute.glsl:14-49 for one command. joints: row-major mat4x3 (3 x vec4 per joint).
ORACLE_API void oracle_skin_vertices(const GpuUnskinnedVertex* unskinned, const float* joints, PackedVec3* positions, GpuVertex* vertices,
                                     uint32_t inOffset, uint32_t outOffset, uint32_t jointOffset, uint32_t count) {
    for (uint32_t i = 0; i < count; i++) {
        const GpuUnskinnedVertex& u = unskinned[inOffset + i];
        float rows[3][4];
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 4; c++) {
                const float m0 = joints[12 * (size_t)(jointOffset + u.JointIndices[0]) + 4 * r + c];
                const float m1 = joints[12 * (size_t)(jointOffset + u.JointIndices[1]) + 4 * r + c];
                const float m2 = joints[12 * (size_t)(jointOffset + u.JointIndices[2]) + 4 * r + c];
                const float m3 = joints[12 * (size_t)(jointOffset + u.JointIndices[3]) + 4 * r + c];
                rows[r][c] = ((u.JointWeights[0] * m0 + u.JointWeights[1] * m1) + u.JointWeights[2] * m2) + u.JointWeights[3] * m3;
            }
        const vec3 position = {u.Position[0], u.Position[1], u.Position[2]};
        const vec3 normal = DecompressSR11G11B10(u.Normal), tangent = DecompressSR11G11B10(u.Tangent);
        float p[3], n[3], t[3];
        for (int r = 0; r < 3; r++) {
            p[r] = ((rows[r][0] * position.x + rows[r][1] * position.y) + rows[r][2] * position.z) + rows[r][3] * 1.0f;
            n[r] = (rows[r][0] * normal.x + rows[r][1] * normal.y) + rows[r][2] * normal.z;
            t[r] = (rows[r][0] * tangent.x + rows[r][1] * tangent.y) + rows[r][2] * tangent.z;
        }
        const vec3 nn = normalize(vec3{n[0], n[1], n[2]}), tt = normalize(vec3{t[0], t[1], t[2]});
        positions[outOffset + i] = {p[0], p[1], p[2]};
        vertices[outOffset + i].Normal = CompressSR11G11B10(nn);
        vertices[outOffset + i].Tangent = CompressSR11G11B10(tt);
    }
}

// BLAS.Refit (BLAS.cs:276-293): reverse sweep; the boxes BLASRefit/compute.glsl's leaf-up climb must also produce.
ORACLE_API void oracle_blas_refit(GpuBlasNode* allNodes, const GpuBlasDesc* desc, const GpuBlasTriangle* blasTriangles, const PackedVec3* positions) {
    GpuBlasNode* nodes = allNodes + desc->NodeOffset;
    for (int i = desc->NodeCount - 1; i >= 1; i--) {
        GpuBlasNode& nd = nodes[i];
        if (nd.TriCount > 0) {
            float lo[3] = {3.4028235e38f, 3.4028235e38f, 3.4028235e38f}, hi[3] = {-3.4028235e38f, -3.4028235e38f, -3.4028235e38f};
            for (int k = 0; k < nd.TriCount; k++) {
                const GpuBlasTriangle& t = blasTriangles[desc->TriangleOffset + nd.TriStartOrChild + k];
                const int idx[3] = {t.X, t.Y, t.Z};
                for (int v = 0; v < 3; v++) {
                    const PackedVec3& p = positions[idx[v]];
                    lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
                    hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
                }
            }
            for (int c = 0; c < 3; c++) { nd.Min[c] = lo[c]; nd.Max[c] = hi[c]; }
            continue;
        }
        const GpuBlasNode& l = nodes[nd.TriStartOrChild];
        const GpuBlasNode& r = nodes[nd.TriStartOrChild + 1];
        for (int c = 0; c < 3; c++) { nd.Min[c] = fminf(l.Min[c], r.Min[c]); nd.Max[c] = fmaxf(l.Max[c], r.Max[c]); }
    }
}

} // extern "C"
#include "oracle_post.inc"

extern "C" {
// Test hook: TexSample of one texture at n (u, v) points -> rgba floats.
ORACLE_API void oracle_tex_sample(const IdkPtTextureDesc* tex, const float* uv, uint64_t n, float* out) {
    IdkPtSceneDesc d = {};
    d.Textures = tex; d.TextureCount = 1;
    for (uint64_t i = 0; i < n; i++) {
        const Vec4 c = TexSample(d, 1, uv[2 * i], uv[2 * i + 1]);
        out[4 * i] = c.x; out[4 * i + 1] = c.y; out[4 * i + 2] = c.z; out[4 * i + 3] = c.w;
    }
}
}
