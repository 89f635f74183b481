// ORACLE (TEST INFRASTRUCTURE ONLY) -- the G-buffer pass, ray-cast at pixel centres.
//
// Part of liboracle.so (wrapped by tests/gbuffer_oracle.py). It includes oracle.cpp and reuses its scene access,
// RayTriangleIntersect, RayBoxIntersect, RayTransform, GetSurface,
// SurfaceApplyModificatons, TexSample, InterpTexCoord, DecompressSR11G11B10, EncodeUnitVec and the half conversion unchanged;
// the serial walk with the depth test's acceptance rules and the fragment stage are restated here.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/GBuffer/VertexPath/vertex.glsl:17-47      per-vertex world normal / tangent, PrevClipPos, jittered clip
//   Resource/Shaders/GBuffer/fragment.glsl:24-58               GetSurface, alpha discard, GetTBN, gl_FrontFacing, velocity
//   Resource/Shaders/include/BVHIntersect.glsl:27-291          the walk (instance loop or TLAS), here with the acceptance rules
//   Source/Render/RasterPipeline.cs:364-414, 648-681           the two draws (CullFace for single-sided), the attachment formats
//   Resource/Shaders/MeshCulling/Camera/Cull/compute.glsl:44-49  transparents culled from the pass
//   OpenGL 4.6 core spec 2.3.4.3 (unsigned 11- / 10-bit floats), 14.6.1 (face culling), 15 (depth test LESS)
//
// DESIGN.md 8f.1g pins the rules: the ray through the pixel centre; a triangle takes the hit only if it beats t and is not
// clipped (screen-linear depth outside [0, 1]), blended, back-facing on a single-sided material (det(Model) * dot(n, d) sign)
// or alpha-discarded; depth = (sum b_i clip_i.z) / (sum b_i clip_i.w); the vertex shader's order (transform, then interpolate);
// R11G11B10F nearest-even, RG8 through the R8 rule, RG16F nearest-even.
#pragma once
#include "oracle.cpp"

#include <cmath>
#include <cstring>

namespace {

struct Vec4f { float x, y, z, w; };

// GLSL column-major mat4 times vec4(p, 1)
static inline Vec4f GbClip(const float* m, vec3 p) {
    return {((m[0] * p.x + m[4] * p.y) + m[8] * p.z) + m[12], ((m[1] * p.x + m[5] * p.y) + m[9] * p.z) + m[13],
            ((m[2] * p.x + m[6] * p.y) + m[10] * p.z) + m[14], ((m[3] * p.x + m[7] * p.y) + m[11] * p.z) + m[15]};
}
// mat4(mat4x3) * vec4(p, 1): rows of the stored 3x4
static inline vec3 GbXformPoint(const float m[3][4], vec3 p) {
    return {((m[0][0] * p.x + m[0][1] * p.y) + m[0][2] * p.z) + m[0][3], ((m[1][0] * p.x + m[1][1] * p.y) + m[1][2] * p.z) + m[1][3],
            ((m[2][0] * p.x + m[2][1] * p.y) + m[2][2] * p.z) + m[2][3]};
}
// mat3(transpose(InvModelMatrix)) * v
static inline vec3 GbUnitVecToWorld(const float im[3][4], vec3 v) {
    return {(im[0][0] * v.x + im[1][0] * v.y) + im[2][0] * v.z, (im[0][1] * v.x + im[1][1] * v.y) + im[2][1] * v.z,
            (im[0][2] * v.x + im[1][2] * v.y) + im[2][2] * v.z};
}
static inline float GbDet(const float m[3][4]) {
    return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])) +
           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}
// gl_FrontFacing of the triangle as seen along local direction ld in an instance with det(Model) = det: CCW is front in window
// space (lower-left origin); a mirroring model matrix flips the winding.
static inline bool GbFrontFacing(float det, vec3 nLocal, vec3 ld) {
    const float dn = dot(nLocal, ld);
    return (det > 0.0f && dn < 0.0f) || (det < 0.0f && dn > 0.0f);
}
static inline vec3 GbPosition(const PackedVec3* positions, int32_t i) { return {positions[i].x, positions[i].y, positions[i].z}; }

// Screen-linear depth at barycentrics (b0, b1, b2): the unjittered clip positions' z and w interpolated, then divided.
static float GbDepth(const float* projView, const PackedVec3* positions, const float model[3][4], const GpuBlasTriangle& tri,
                     float b0, float b1, float b2) {
    const Vec4f c0 = GbClip(projView, GbXformPoint(model, GbPosition(positions, tri.X)));
    const Vec4f c1 = GbClip(projView, GbXformPoint(model, GbPosition(positions, tri.Y)));
    const Vec4f c2 = GbClip(projView, GbXformPoint(model, GbPosition(positions, tri.Z)));
    return ((c0.z * b0 + c1.z * b1) + c2.z * b2) / ((c0.w * b0 + c1.w * b1) + c2.w * b2);
}

// The depth test's acceptance of a candidate fragment of triangle k of an instance.
static bool GbAccept(const Scene& s, const GpuPerFrameData& f, const GpuMeshTransform& mt, float det, const Ray& localRay, uint32_t k,
                     float b0, float b1) {
    const GpuBlasTriangle& tri = s.d.BlasTriangles[k];
    const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
    const GpuMaterial& material = s.d.Materials[mesh.MaterialId];
    if (material.AlphaCutoff == 2.0f) return false;   // blended: culled from the pass
    if (!material.IsDoubleSided) {
        const vec3 p0 = pos(s, tri.X), p1 = pos(s, tri.Y), p2 = pos(s, tri.Z);
        if (!GbFrontFacing(det, cross(p1 - p0, p2 - p0), localRay.d)) return false;
    }
    const float b2 = 1.0f - b0 - b1;
    const float depth = GbDepth(f.ProjView, s.d.VertexPositions, mt.ModelMatrix, tri, b0, b1, b2);
    if (!(depth >= 0.0f && depth <= 1.0f)) return false;   // clipped by the near or far plane
    float u, v;
    InterpTexCoord(s.d, tri, b0, b1, b2, u, v);
    Surface surface = GetSurface(s.d, material, u, v);
    SurfaceApplyModificatons(surface, mesh);
    return !(surface.Alpha < surface.AlphaCutoff);
}

// IntersectBlas (BVHIntersect.glsl:27-105) where a closer triangle takes the hit only if GbAccept holds.
static bool GbIntersectBlas(const Scene& s, const GpuPerFrameData& f, const GpuMeshTransform& mt, const Ray& ray, const GpuBlasDesc& blasDesc,
                            HitInfo& hitInfo, bool useTlas) {
    bool hit = false;
    float tMinLeft, tMinRight;
    const GpuBlasNode* nodes = s.d.BlasNodes + blasDesc.NodeOffset;
    const vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};
    const float det = GbDet(mt.ModelMatrix);
    if (!useTlas) {
        const GpuBlasNode& rootNode = nodes[1];
        if (!(RayBoxIntersect(ray, invDir, rootNode.Min, rootNode.Max, tMinLeft) && tMinLeft < hitInfo.T)) return false;
    }
    uint32_t stack[256];
    uint32_t stackPtr = 0, stackTop = 2;
    while (true) {
        const GpuBlasNode& leftNode = nodes[stackTop];
        const GpuBlasNode& rightNode = nodes[stackTop + 1];
        const bool hitLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft <= hitInfo.T;
        const bool hitRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight <= hitInfo.T;
        const bool intersectLeft = hitLeft && leftNode.TriCount > 0;
        const bool intersectRight = hitRight && rightNode.TriCount > 0;
        if (intersectLeft || intersectRight) {
            uint32_t first = intersectLeft ? (uint32_t)leftNode.TriStartOrChild : (uint32_t)rightNode.TriStartOrChild;
            uint32_t end = !intersectRight ? (uint32_t)(leftNode.TriStartOrChild + leftNode.TriCount) : (uint32_t)(rightNode.TriStartOrChild + rightNode.TriCount);
            first += (uint32_t)blasDesc.TriangleOffset;
            end += (uint32_t)blasDesc.TriangleOffset;
            for (uint32_t i = first; i < end; i++) {
                const GpuBlasTriangle& tri = s.d.BlasTriangles[i];
                vec3 bary;
                float hitT;
                if (RayTriangleIntersect(ray, pos(s, tri.X), pos(s, tri.Y), pos(s, tri.Z), bary, hitT) && hitT < hitInfo.T &&
                    GbAccept(s, f, mt, det, ray, i, bary.x, bary.y)) {
                    hit = true;
                    hitInfo.TriangleId = i;
                    hitInfo.bx = bary.x;
                    hitInfo.by = bary.y;
                    hitInfo.T = hitT;
                }
            }
        }
        const bool traverseLeft = hitLeft && leftNode.TriCount == 0;
        const bool traverseRight = hitRight && rightNode.TriCount == 0;
        if (traverseLeft || traverseRight) {
            if (traverseLeft && traverseRight) {
                const bool leftCloser = tMinLeft < tMinRight;
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

// TraceRay (BVHIntersect.glsl:183-291) without lights, with the acceptance rules.
static bool GbTraceRay(const Scene& s, const GpuPerFrameData& f, const Ray& ray, HitInfo& hitInfo) {
    hitInfo.T = FLOAT_MAX;
    hitInfo.TriangleId = ~0u;
    hitInfo.MeshTransformId = 0;
    hitInfo.bx = hitInfo.by = 0.0f;
    auto instance = [&](uint32_t id, bool useTlas) {
        const GpuBlasInstance& inst = s.d.BlasInstances[id];
        const GpuMeshTransform& mt = s.d.MeshTransforms[inst.MeshTransformId];
        const Ray localRay = RayTransform(ray, mt.InvModelMatrix);
        if (GbIntersectBlas(s, f, mt, localRay, s.d.BlasDescs[inst.BlasId], hitInfo, useTlas)) hitInfo.MeshTransformId = inst.MeshTransformId;
    };
    if (s.d.UseTlas) {
        float tMinLeft, tMinRight;
        uint32_t stackPtr = 0, stackTop = 0;
        uint32_t stack[24];
        const vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};
        while (true) {
            const GpuTlasNode& parent = s.d.TlasNodes[stackTop];
            const uint32_t childOrInstanceId = parent.IsLeafAndChildOrInstanceId & ((1u << 31) - 1);
            if ((parent.IsLeafAndChildOrInstanceId >> 31) == 1) {
                instance(childOrInstanceId, true);
                if (stackPtr == 0) break;
                stackTop = stack[--stackPtr];
                continue;
            }
            const uint32_t leftChildId = childOrInstanceId, rightChildId = leftChildId + 1;
            const GpuTlasNode& leftNode = s.d.TlasNodes[leftChildId];
            const GpuTlasNode& rightNode = s.d.TlasNodes[rightChildId];
            const bool traverseLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft < hitInfo.T;
            const bool traverseRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight < hitInfo.T;
            if (traverseLeft || traverseRight) {
                if (traverseLeft && traverseRight) {
                    const bool leftCloser = tMinLeft < tMinRight;
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
        for (uint64_t i = 0; i < s.d.BlasInstanceCount; i++) instance((uint32_t)i, false);
    }
    return hitInfo.TriangleId != ~0u;
}

// GL core spec 2.3.4.3: unsigned float with `mbits` mantissa bits and a 5-bit exponent (bias 15), nearest with ties to even.
static float GbUnsignedFloat(float v, int mbits, float maxFinite) {
    if (std::isnan(v)) return v;
    if (!(v > 0.0f)) return 0.0f;                       // negative, -0, -inf
    if (std::isinf(v)) return v;                        // +inf
    uint32_t bits;
    std::memcpy(&bits, &v, 4);
    const int e = std::max((int)((bits >> 23) & 255u) - 127, -14);   // denormals of the small format below 2^-14
    const float quantum = std::ldexp(1.0f, e - mbits);
    return std::fmin(std::nearbyint(v / quantum) * quantum, maxFinite);
}
static float GbUnorm8(float v) { return std::floor(clampf(v, 0.0f, 1.0f) * 255.0f + 0.5f) / 255.0f; }

// The six attachments of one pixel.
struct GbPixel { float depth, normal[2], albedo[3], mr[2], emissive[3], velocity[2]; };

static GbPixel GbShadePixel(const Scene& s, const GpuPerFrameData& f, const PackedVec3* prevPositions, int x, int y, int w, int h,
                            const float jitter[2]) {
    GbPixel px = {1.0f, {0.0f, 0.0f}, {0.0f, 0.0f, 0.0f}, {0.0f, 0.0f}, {0.0f, 0.0f, 0.0f}, {0.0f, 0.0f}};
    const float ndcX = ((float)x + 0.5f) / (float)w * 2.0f - 1.0f - jitter[0];
    const float ndcY = ((float)y + 0.5f) / (float)h * 2.0f - 1.0f - jitter[1];
    const float* m = f.InvProjView;   // PerspectiveTransform(vec3(ndc, 1), InvProjView)
    const float hx = ((m[0] * ndcX + m[4] * ndcY) + m[8] * 1.0f) + m[12] * 1.0f;
    const float hy = ((m[1] * ndcX + m[5] * ndcY) + m[9] * 1.0f) + m[13] * 1.0f;
    const float hz = ((m[2] * ndcX + m[6] * ndcY) + m[10] * 1.0f) + m[14] * 1.0f;
    const float hw = ((m[3] * ndcX + m[7] * ndcY) + m[11] * 1.0f) + m[15] * 1.0f;
    const vec3 viewPos = V(f.ViewPos);
    const vec3 dir = normalize(V(hx / hw, hy / hw, hz / hw) - viewPos);
    HitInfo hit;
    if (!GbTraceRay(s, f, Ray{viewPos, dir}, hit)) return px;

    const GpuBlasTriangle& tri = s.d.BlasTriangles[hit.TriangleId];
    const GpuMeshTransform& mt = s.d.MeshTransforms[hit.MeshTransformId];
    const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
    const GpuMaterial& material = s.d.Materials[mesh.MaterialId];
    const float b0 = hit.bx, b1 = hit.by, b2 = 1.0f - hit.bx - hit.by;
    px.depth = GbDepth(f.ProjView, s.d.VertexPositions, mt.ModelMatrix, tri, b0, b1, b2);

    // vertex shader: world normal / tangent per vertex; rasteriser: interpolation; fragment shader: GetTBN and the normal map
    const GpuVertex* vs[3] = {&s.d.Vertices[tri.X], &s.d.Vertices[tri.Y], &s.d.Vertices[tri.Z]};
    vec3 wn[3], wt[3];
    for (int i = 0; i < 3; i++) {
        wn[i] = normalize(GbUnitVecToWorld(mt.InvModelMatrix, DecompressSR11G11B10(vs[i]->Normal)));
        wt[i] = normalize(GbUnitVecToWorld(mt.InvModelMatrix, DecompressSR11G11B10(vs[i]->Tangent)));
    }
    const vec3 interpNormal = normalize((wn[0] * b0 + wn[1] * b1) + wn[2] * b2);
    const vec3 interpTangent = normalize((wt[0] * b0 + wt[1] * b1) + wt[2] * b2);
    float u, v;
    InterpTexCoord(s.d, tri, b0, b1, b2, u, v);
    Surface surface = GetSurface(s.d, material, u, v);
    SurfaceApplyModificatons(surface, mesh);
    const vec3 N = normalize(interpNormal), T = normalize(interpTangent), B = normalize(cross(N, T));
    const vec3 sn = surface.Normal;
    vec3 normal = normalize(mix(interpNormal, (T * sn.x + B * sn.y) + N * sn.z, mesh.NormalMapStrength));
    const vec3 p0 = pos(s, tri.X), p1 = pos(s, tri.Y), p2 = pos(s, tri.Z);
    if (!GbFrontFacing(GbDet(mt.ModelMatrix), cross(p1 - p0, p2 - p0), RayTransform(Ray{viewPos, dir}, mt.InvModelMatrix).d)) normal = normal * -1.0f;

    // PrevClipPos, interpolated
    Vec4f q[3];
    const int32_t ids[3] = {tri.X, tri.Y, tri.Z};
    for (int i = 0; i < 3; i++) q[i] = GbClip(f.PrevProjView, GbXformPoint(mt.PrevModelMatrix, GbPosition(prevPositions, ids[i])));
    const float pcx = (q[0].x * b0 + q[1].x * b1) + q[2].x * b2;
    const float pcy = (q[0].y * b0 + q[1].y * b1) + q[2].y * b2;
    const float pcw = (q[0].w * b0 + q[1].w * b1) + q[2].w * b2;

    float ex, ey;
    EncodeUnitVec(normal, ex, ey);
    px.normal[0] = GbUnorm8(ex); px.normal[1] = GbUnorm8(ey);
    const float albedo[3] = {surface.Albedo.x, surface.Albedo.y, surface.Albedo.z};
    const float emissive[3] = {surface.Emissive.x, surface.Emissive.y, surface.Emissive.z};
    for (int c = 0; c < 3; c++) {
        px.albedo[c] = c < 2 ? GbUnsignedFloat(albedo[c], 6, 65024.0f) : GbUnsignedFloat(albedo[c], 5, 64512.0f);
        px.emissive[c] = c < 2 ? GbUnsignedFloat(emissive[c], 6, 65024.0f) : GbUnsignedFloat(emissive[c], 5, 64512.0f);
    }
    px.mr[0] = GbUnorm8(surface.Metallic); px.mr[1] = GbUnorm8(surface.Roughness);
    px.velocity[0] = to_half_and_back((ndcX - pcx / pcw) * 0.5f);
    px.velocity[1] = to_half_and_back((ndcY - pcy / pcw) * 0.5f);
    return px;
}

} // namespace

extern "C" {

// idkpt_gbuffer: six planar arrays [h][w][c] (Depth 1, NormalRG 2, AlbedoRGB 3, MetallicRoughness 2, EmissiveRGB 3, VelocityRG 2).
// jitter and prevPositions may be null (0, and this frame's positions).
ORACLE_API int oracle_gbuffer(const IdkPtSceneDesc* scene, const GpuPerFrameData* frame, int w, int h, const float* jitter,
                              const PackedVec3* prevPositions, float* depth, float* normal, float* albedo, float* mr, float* emissive,
                              float* velocity, int threads) {
    if (!scene || !frame || w < 1 || h < 1) return 1;
    Scene s; s.d = *scene;
    const float jit[2] = {jitter ? jitter[0] : 0.0f, jitter ? jitter[1] : 0.0f};
    const PackedVec3* prev = prevPositions ? prevPositions : scene->VertexPositions;
    parallel_for((size_t)w * h, threads, [&](size_t begin, size_t end, int) {
        for (size_t p = begin; p < end; p++) {
            const GbPixel px = GbShadePixel(s, *frame, prev, (int)(p % w), (int)(p / w), w, h, jit);
            depth[p] = px.depth;
            for (int c = 0; c < 2; c++) { normal[2 * p + c] = px.normal[c]; mr[2 * p + c] = px.mr[c]; velocity[2 * p + c] = px.velocity[c]; }
            for (int c = 0; c < 3; c++) { albedo[3 * p + c] = px.albedo[c]; emissive[3 * p + c] = px.emissive[c]; }
        }
    });
    return 0;
}

// The attachment conversions on their own: kind 0 R11G11B10F red/green channel, 1 its blue channel, 2 RG8 unorm, 3 RG16F.
ORACLE_API void oracle_gbuffer_store(int kind, const float* in, uint64_t n, float* out) {
    for (uint64_t i = 0; i < n; i++)
        out[i] = kind == 0 ? GbUnsignedFloat(in[i], 6, 65024.0f) : kind == 1 ? GbUnsignedFloat(in[i], 5, 64512.0f)
               : kind == 2 ? GbUnorm8(in[i]) : to_half_and_back(in[i]);
}

} // extern "C"
