// ORACLE (TEST INFRASTRUCTURE ONLY) -- transparency: the record pass's blended fragments, ray-cast at pixel centres, lit, and
// resolved front to back over the lit image.
//
// Built as its own library (tests/transparency_oracle.py -> oracle/liboracle_transparency.so). It compiles
// oracle_deferred.cpp (and with it oracle_point_shadows.cpp and oracle.cpp) into the same translation unit and reuses its
// EvaluateLighting / GGXBrdf (DfSurface carries the IOR), the 21-tap PCF filter (DfVisibility), DfPerspective, and oracle.cpp's
// RayTriangleIntersect, RayBoxIntersect, RayTransform, GetSurface, SurfaceApplyModificatons, InterpTexCoord,
// DecompressSR11G11B10, SampleSky, InterleavedGradientNoise, vx_trace_cone and the half conversion unchanged. oracle.cpp has no
// include guard, so oracle_gbuffer.cpp (which includes it too) cannot join the same translation unit: the G-buffer pass's
// geometric rules it needs (clip position, depth, front face, the per-vertex world normal) are the few lines restated below.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/RecordTransparent/fragment.glsl            the record fragment shader (lighting, premultiplied rgba16f)
//   Resource/Shaders/ResolveTransparent/compute.glsl            the stable insertion sort and the front-to-back blend
//   Resource/Shaders/VXGI/ConeTraceGI/include/Impl.glsl:27-80   IndirectLight (gl_FragCoord noise, the skybox texture)
//   Resource/Shaders/include/BVHIntersect.glsl:27-291           the walk, here with the record pass's fragment tests
//   Source/Render/RasterPipeline.cs:518-588                     the draw (depth LESS, no depth writes, CullFace single-sided)
//
// DESIGN.md 8f.1h pins the rules: the G-buffer pass's ray; a candidate is kept if blended, front-facing or double-sided, depth
// in [0, 1] and below the opaque depth, alpha != 0; the 10 smallest (depth, BLAS triangle, MeshTransformId) are kept, in that
// order; the walk's bound is the reconstructed opaque distance times 1.125 (unbounded where the depth is not below 1).
#include "oracle_deferred.cpp"

namespace {

constexpr int kLayers = 10;
constexpr float kTMargin = 1.125f;

struct TrLayer { float depth; uint32_t tri, xf; float bx, by; };

static inline bool TrBefore(const TrLayer& a, const TrLayer& b) {
    return a.depth < b.depth || (a.depth == b.depth && (a.tri < b.tri || (a.tri == b.tri && a.xf < b.xf)));
}

// The G-buffer pass's geometric rules (DESIGN.md 8f.1g rules 2-4), as oracle_gbuffer.cpp states them.
static inline vec3 TrXformPoint(const float m[3][4], vec3 p) {
    return {((m[0][0] * p.x + m[0][1] * p.y) + m[0][2] * p.z) + m[0][3], ((m[1][0] * p.x + m[1][1] * p.y) + m[1][2] * p.z) + m[1][3],
            ((m[2][0] * p.x + m[2][1] * p.y) + m[2][2] * p.z) + m[2][3]};
}
static inline vec3 TrUnitVecToWorld(const float im[3][4], vec3 v) {
    return {(im[0][0] * v.x + im[1][0] * v.y) + im[2][0] * v.z, (im[0][1] * v.x + im[1][1] * v.y) + im[2][1] * v.z,
            (im[0][2] * v.x + im[1][2] * v.y) + im[2][2] * v.z};
}
static inline float TrDet(const float m[3][4]) {
    return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])) +
           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}
static inline bool TrFrontFacing(float det, vec3 nLocal, vec3 ld) {
    const float dn = dot(nLocal, ld);
    return (det > 0.0f && dn < 0.0f) || (det < 0.0f && dn > 0.0f);
}
static float TrDepth(const float* pv, const Scene& s, const float model[3][4], const GpuBlasTriangle& tri, float b0, float b1, float b2) {
    float cz[3], cw[3];
    const int32_t ids[3] = {tri.X, tri.Y, tri.Z};
    for (int i = 0; i < 3; i++) {
        const vec3 p = TrXformPoint(model, pos(s, ids[i]));
        cz[i] = ((pv[2] * p.x + pv[6] * p.y) + pv[10] * p.z) + pv[14];
        cw[i] = ((pv[3] * p.x + pv[7] * p.y) + pv[11] * p.z) + pv[15];
    }
    return ((cz[0] * b0 + cz[1] * b1) + cz[2] * b2) / ((cw[0] * b0 + cw[1] * b1) + cw[2] * b2);
}

struct TrWalk {
    const Scene& s;
    const GpuPerFrameData& f;
    float opaqueDepth;
    std::vector<TrLayer> kept;   // sorted, at most kLayers
    uint64_t candidates = 0;     // fragments that passed the tests (before the cap)

    void Record(const TrLayer& l) {
        candidates++;
        auto it = std::upper_bound(kept.begin(), kept.end(), l, TrBefore);
        kept.insert(it, l);
        if ((int)kept.size() > kLayers) kept.pop_back();
    }
    // the record pass's fragment tests for triangle k of an instance
    void Test(const GpuMeshTransform& mt, uint32_t xf, float det, const Ray& localRay, uint32_t k, float b0, float b1) {
        const GpuBlasTriangle& tri = s.d.BlasTriangles[k];
        const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
        const GpuMaterial& material = s.d.Materials[mesh.MaterialId];
        if (material.AlphaCutoff != 2.0f) return;
        if (!material.IsDoubleSided) {
            const vec3 p0 = pos(s, tri.X), p1 = pos(s, tri.Y), p2 = pos(s, tri.Z);
            if (!TrFrontFacing(det, cross(p1 - p0, p2 - p0), localRay.d)) return;
        }
        const float b2 = 1.0f - b0 - b1;
        const float depth = TrDepth(f.ProjView, s, mt.ModelMatrix, tri, b0, b1, b2);
        if (!(depth >= 0.0f && depth <= 1.0f && depth < opaqueDepth)) return;
        float u, v;
        InterpTexCoord(s.d, tri, b0, b1, b2, u, v);
        Surface surface = GetSurface(s.d, material, u, v);
        SurfaceApplyModificatons(surface, mesh);
        if (surface.Alpha == 0.0f) return;
        Record(TrLayer{depth, k, xf, b0, b1});
    }
    // IntersectBlas (BVHIntersect.glsl:27-105) with t fixed at tMax: every triangle hit closer than tMax is tested.
    void Blas(const GpuMeshTransform& mt, uint32_t xf, const Ray& ray, const GpuBlasDesc& blasDesc, float tMax, bool useTlas) {
        float tMinLeft, tMinRight;
        const GpuBlasNode* nodes = s.d.BlasNodes + blasDesc.NodeOffset;
        const vec3 invDir = {1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z};
        const float det = TrDet(mt.ModelMatrix);
        if (!useTlas) {
            const GpuBlasNode& rootNode = nodes[1];
            if (!(RayBoxIntersect(ray, invDir, rootNode.Min, rootNode.Max, tMinLeft) && tMinLeft < tMax)) return;
        }
        uint32_t stack[256];
        uint32_t stackPtr = 0, stackTop = 2;
        while (true) {
            const GpuBlasNode& leftNode = nodes[stackTop];
            const GpuBlasNode& rightNode = nodes[stackTop + 1];
            const bool hitLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft <= tMax;
            const bool hitRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight <= tMax;
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
                    if (RayTriangleIntersect(ray, pos(s, tri.X), pos(s, tri.Y), pos(s, tri.Z), bary, hitT) && hitT < tMax)
                        Test(mt, xf, det, ray, i, bary.x, bary.y);
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
    }
    // TraceRay (BVHIntersect.glsl:183-291) without lights: the instance loop or the TLAS walk.
    void Trace(const Ray& ray, float tMax) {
        auto instance = [&](uint32_t id, bool useTlas) {
            const GpuBlasInstance& inst = s.d.BlasInstances[id];
            const GpuMeshTransform& mt = s.d.MeshTransforms[inst.MeshTransformId];
            Blas(mt, inst.MeshTransformId, RayTransform(ray, mt.InvModelMatrix), s.d.BlasDescs[inst.BlasId], tMax, useTlas);
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
                const bool traverseLeft = RayBoxIntersect(ray, invDir, leftNode.Min, leftNode.Max, tMinLeft) && tMinLeft < tMax;
                const bool traverseRight = RayBoxIntersect(ray, invDir, rightNode.Min, rightNode.Max, tMinRight) && tMinRight < tMax;
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
    }
};

struct TrInputs {
    const GpuPointShadow* shadows; const int32_t* sizes; const uint16_t* texels; int shadowCount;
    std::vector<size_t> offsets;
    int shadowMode, isVxgi;
    const VxGrid* grid; IdkVxConeSettings cone;
    const float* skyFaces[6]; int skyFaceSize; const float* skyColor;
    int bound;                     // 1: the walk starts from the opaque distance bound, 0: unbounded
};

// One pixel: the walk, then the kept layers lit in order, rounded to rgba16f and blended; false if no layer was kept.
static bool TrPixel(const Scene& s, const GpuPerFrameData& f, const TrInputs& in, int x, int y, int w, int h, const float jitter[2],
                    float opaqueDepth, const float opaque[4], float out[4], TrLayer* layersOut, int* countOut, float* layerColorsOut) {
    const float ndcX = ((float)x + 0.5f) / (float)w * 2.0f - 1.0f - jitter[0];
    const float ndcY = ((float)y + 0.5f) / (float)h * 2.0f - 1.0f - jitter[1];
    const vec3 viewPos = V(f.ViewPos);
    const vec3 dir = normalize(DfPerspective(f.InvProjView, ndcX, ndcY, 1.0f) - viewPos);
    float tMax = FLOAT_MAX;
    if (in.bound && opaqueDepth < 1.0f) {
        const vec3 e = DfPerspective(f.InvProjView, ndcX, ndcY, opaqueDepth) - viewPos;
        const float t = sqrtf(dot(e, e)) * kTMargin;
        tMax = t <= FLOAT_MAX ? t : FLOAT_MAX;
    }
    TrWalk walk{s, f, opaqueDepth, {}};
    walk.Trace(Ray{viewPos, dir}, tMax);
    if (countOut) *countOut = (int)walk.kept.size();
    if (layersOut) for (size_t i = 0; i < walk.kept.size(); i++) layersOut[i] = walk.kept[i];
    if (walk.kept.empty()) return false;

    const float u = ((float)x + 0.5f) / (float)w, v = ((float)y + 0.5f) / (float)h;
    const float nx = u * 2.0f - 1.0f, ny = v * 2.0f - 1.0f;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    int li = 0;
    for (const TrLayer& l : walk.kept) {
        const GpuBlasTriangle& tri = s.d.BlasTriangles[l.tri];
        const GpuMeshTransform& mt = s.d.MeshTransforms[l.xf];
        const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
        const GpuMaterial& material = s.d.Materials[mesh.MaterialId];
        const float b0 = l.bx, b1 = l.by, b2 = 1.0f - l.bx - l.by;
        // the vertex shader's world normal / tangent per vertex, interpolated; GetTBN, the normal map, gl_FrontFacing
        const GpuVertex* vs[3] = {&s.d.Vertices[tri.X], &s.d.Vertices[tri.Y], &s.d.Vertices[tri.Z]};
        vec3 wn[3], wt[3];
        for (int i = 0; i < 3; i++) {
            wn[i] = normalize(TrUnitVecToWorld(mt.InvModelMatrix, DecompressSR11G11B10(vs[i]->Normal)));
            wt[i] = normalize(TrUnitVecToWorld(mt.InvModelMatrix, DecompressSR11G11B10(vs[i]->Tangent)));
        }
        const vec3 interpNormal = normalize((wn[0] * b0 + wn[1] * b1) + wn[2] * b2);
        const vec3 interpTangent = normalize((wt[0] * b0 + wt[1] * b1) + wt[2] * b2);
        float tu, tv;
        InterpTexCoord(s.d, tri, b0, b1, b2, tu, tv);
        Surface surface = GetSurface(s.d, material, tu, tv);
        SurfaceApplyModificatons(surface, mesh);
        const vec3 N = normalize(interpNormal), T = normalize(interpTangent), B = normalize(cross(N, T));
        const vec3 sn = surface.Normal;
        vec3 normal = normalize(mix(interpNormal, (T * sn.x + B * sn.y) + N * sn.z, mesh.NormalMapStrength));
        const vec3 p0 = pos(s, tri.X), p1 = pos(s, tri.Y), p2 = pos(s, tri.Z);
        if (!TrFrontFacing(TrDet(mt.ModelMatrix), cross(p1 - p0, p2 - p0), RayTransform(Ray{viewPos, dir}, mt.InvModelMatrix).d)) normal = normal * -1.0f;

        const vec3 fragPos = DfPerspective(f.InvProjView, nx, ny, l.depth);
        const vec3 unjitteredFragPos = DfPerspective(f.InvProjView, nx - jitter[0], ny - jitter[1], l.depth);
        DfSurface ds;
        ds.Albedo = surface.Albedo; ds.Normal = normal; ds.Emissive = surface.Emissive;
        ds.Metallic = surface.Metallic; ds.Roughness = surface.Roughness; ds.IOR = surface.IOR;
        vec3 direct = V(0, 0, 0);
        for (uint64_t i = 0; i < s.d.LightCount; i++) {
            const GpuLight& light = s.d.Lights[i];
            vec3 contribution = EvaluateLighting(light, ds, fragPos, viewPos, 0.0f);
            if (contribution.x != 0.0f || contribution.y != 0.0f || contribution.z != 0.0f) {
                float shadow = 0.0f;
                const int k = light.PointShadowIndex;
                if (k == -1) {
                    shadow = 0.0f;
                } else if (in.shadowMode == 1) {
                    shadow = 1.0f - DfVisibility(in.shadows[k], in.sizes[k], in.texels + in.offsets[k], unjitteredFragPos - V(light.Position));
                } else if (in.shadowMode == 2) {
                    // the engine leaves ray-traced shadows on transparents unimplemented: unshadowed
                }
                contribution = contribution * (1.0f - shadow);
            }
            direct = direct + contribution;
        }
        vec3 indirect;
        if (in.isVxgi) {
            // IndirectLight with GetPixelCoord() = gl_FragCoord.xy and the skybox texture
            const IdkVxConeSettings& st = in.cone;
            const vec3 incomming = fragPos - viewPos;
            float roughness = surface.Roughness * surface.Roughness;
            const float metallic = surface.Metallic;
            const float materialVariance = GetSurfaceVariance(metallic, 0.0f, roughness);
            const uint32_t samples = (uint32_t)mixf(1.0f, (float)st.MaxSamples, materialVariance);
            uint32_t noiseIndex = st.NoiseIndex;
            const float px = (float)x + 0.5f, py = (float)y + 0.5f;
            vec3 irradiance = V(0, 0, 0);
            uint64_t steps = 0;
            for (uint32_t i = 0; i < samples; i++) {
                const float rnd0 = InterleavedGradientNoise(px, py, noiseIndex + 0);
                const float rnd1 = InterleavedGradientNoise(px, py, noiseIndex + 1);
                const float rnd2 = InterleavedGradientNoise(px, py, noiseIndex + 2);
                noiseIndex++;
                const vec3 diffuseDir = CosineSampleHemisphere(normal, rnd0, rnd1);
                vec3 cdir;
                float coneAngle;
                if (metallic > rnd2) {
                    cdir = normalize(mix(reflect(incomming, normal), diffuseDir, roughness));
                    coneAngle = mixf(0.0f, 0.32f, roughness);
                } else {
                    cdir = diffuseDir;
                    coneAngle = 0.32f;
                }
                f4 c = vx_trace_cone(*in.grid, fragPos, cdir, normal, coneAngle, st.StepMultiplier, st.NormalRayOffset, 0.99f, steps);
                const vec3 sky = SampleSky(in.skyFaces, in.skyFaceSize, in.skyColor, cdir);
                const float k = 1.0f - c.w;
                c.x += k * (sky.x * st.GISkyBoxBoost);
                c.y += k * (sky.y * st.GISkyBoxBoost);
                c.z += k * (sky.z * st.GISkyBoxBoost);
                irradiance = irradiance + V(c.x, c.y, c.z);
            }
            irradiance = irradiance / (float)samples;
            indirect = (irradiance * st.GIBoost) * surface.Albedo;
        } else {
            indirect = V(0.015f, 0.015f, 0.015f) * surface.Albedo;
        }
        const vec3 c = (direct + indirect) + surface.Emissive;
        const float layer[4] = {to_half_and_back(c.x * surface.Alpha), to_half_and_back(c.y * surface.Alpha), to_half_and_back(c.z * surface.Alpha),
                                to_half_and_back(surface.Alpha)};
        if (layerColorsOut) for (int k = 0; k < 4; k++) layerColorsOut[4 * li + k] = layer[k];
        li++;
        const float weight = 1.0f - acc[3];
        for (int k = 0; k < 4; k++) acc[k] = acc[k] + weight * layer[k];
    }
    const float k = 1.0f - acc[3];
    for (int c = 0; c < 3; c++) out[c] = acc[c] + k * opaque[c];
    out[3] = 1.0f;
    return true;
}

} // namespace

extern "C" {

// idkpt_transparency on the CPU: color (rgba32f [h][w]) is composited in place; pixels without a layer are not written.
// layers (optional): per pixel kLayers records of (depth, tri, xf) as 3 floats/uints each, and counts (optional) the kept
// count; layerColors (optional): per pixel kLayers rgba records of the kept layers' premultiplied, half-rounded colours (the
// engine's ImgRecordedColors, in the kept order; unused records are left as they are). levels: the voxel grid's rgba16f levels
// back to back (IsVXGI). bound: 1 the walk's bound, 0 unbounded.
ORACLE_API int oracle_transparency(const IdkPtSceneDesc* scene, const IdkPtSkyDesc* sky, const GpuPerFrameData* frame, int shadowMode,
                                   int isVxgi, const GpuPointShadow* shadows, const int32_t* sizes, const uint16_t* texels, int shadowCount,
                                   const IdkVxCreateInfo* ci, const uint16_t* levels, const IdkVxConeSettings* cone, const float* depth,
                                   int w, int h, const float* jitter, int bound, float* color, uint32_t* layers, int32_t* counts, float* layerColors,
                                   int threads) {
    if (!scene || !frame || !depth || !color || w < 1 || h < 1 || shadowMode < 0 || shadowMode > 2 || (isVxgi && (!ci || !levels || !cone)))
        return -1;
    Scene s; s.d = *scene;
    TrInputs in;
    in.shadows = shadows; in.sizes = sizes; in.texels = texels; in.shadowCount = shadowCount;
    in.offsets.assign(std::max(shadowCount, 1), 0);
    for (int i = 1; i < shadowCount; i++) in.offsets[i] = in.offsets[i - 1] + 6 * (size_t)sizes[i - 1] * (size_t)sizes[i - 1];
    in.shadowMode = shadowMode; in.isVxgi = isVxgi; in.bound = bound;
    const float noSky[3] = {0.0f, 0.0f, 0.0f};
    for (int i = 0; i < 6; i++) in.skyFaces[i] = sky ? sky->Faces[i] : nullptr;
    in.skyFaceSize = sky ? sky->FaceSize : 0;
    in.skyColor = sky ? sky->Color : noSky;
    VxGrid g;
    if (isVxgi) {
        g.size[0] = ci->Width; g.size[1] = ci->Height; g.size[2] = ci->Depth;
        for (int i = 0; i < 3; i++) { g.gmin[i] = ci->GridMin[i]; g.gmax[i] = std::max(ci->GridMax[i], ci->GridMin[i] + 0.1f); }
        const int mx = std::max(g.size[0], std::max(g.size[1], g.size[2]));
        g.levels = 1;
        while ((mx >> g.levels) > 0) g.levels++;
        g.mip.resize(g.levels);
        uint64_t off = 0;
        for (int l = 0; l < g.levels; l++) {
            const size_t n = (size_t)g.lsize(l, 0) * g.lsize(l, 1) * g.lsize(l, 2);
            g.mip[l].assign(levels + off * 4, levels + (off + n) * 4);
            off += n;
        }
        in.cone = *cone;
    }
    in.grid = &g;
    const float jit[2] = {jitter ? jitter[0] : 0.0f, jitter ? jitter[1] : 0.0f};
    parallel_for((size_t)w * h, threads, [&](size_t begin, size_t end, int) {
        for (size_t p = begin; p < end; p++) {
            TrLayer kept[kLayers];
            int count = 0;
            float out[4];
            if (TrPixel(s, *frame, in, (int)(p % w), (int)(p / w), w, h, jit, depth[p], color + 4 * p, out, kept, &count,
                        layerColors ? layerColors + 4 * (size_t)p * kLayers : nullptr))
                for (int c = 0; c < 4; c++) color[4 * p + c] = out[c];
            if (counts) counts[p] = count;
            if (layers)
                for (int i = 0; i < kLayers; i++) {
                    uint32_t* r = layers + 3 * ((size_t)p * kLayers + i);
                    const float d = i < count ? kept[i].depth : INFINITY;
                    memcpy(r, &d, 4);
                    r[1] = i < count ? kept[i].tri : ~0u;
                    r[2] = i < count ? kept[i].xf : ~0u;
                }
        }
    });
    return 0;
}

} // extern "C"
