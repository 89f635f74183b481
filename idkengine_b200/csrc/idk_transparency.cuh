// The raster mode's transparency for sm_90a: RasterPipeline.Render's "Record transparent fragments" draw and "Resolve transparent
// fragments" dispatch (RasterPipeline.cs:518-588, RecordTransparent/fragment.glsl, ResolveTransparent/compute.glsl), fused and
// ray-cast at pixel centres like the G-buffer pass. The engine's record images (TRANSPARENT_LAYERS rgba16f colours and r32f
// depths per pixel, about 250 MB at 1080p) are never materialised: each thread keeps its pixel's layer list in registers.
//
//   k_transparency<VXGI>   one thread per pixel, 8x8 pixel tiles (four per CTA), the shared-memory traversal stack of
//                          k_trace_rays: one walk through trace_ray<false, false, AcceptTransparent> whose predicate records every
//                          blended fragment the depth test keeps into the list of the IDK_TRANSPARENT_LAYERS closest (and never
//                          takes a hit); then each listed layer is lit as the record shader lights it (direct light with the
//                          surface's IOR, PCF shadows, VXGI or ambient indirect light), premultiplied, rounded to rgba16f and
//                          blended front to back over the lit image, in place
//
// The rules are spelled out in DESIGN.md 8f.1h and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_gbuffer.cuh"
#include "idk_vxgi.cuh"

#define IDK_TRANSPARENT_LAYERS 10   // RasterPipeline.TRANSPARENT_LAYERS
#define IDK_TRANSPARENT_T_MARGIN 1.125f

// The kept layers, closest first: ordered by (depth, BLAS triangle, MeshTransformId); empty entries are (+inf, ~0, ~0). The
// barycentrics are not kept: the shading pass intersects the layer's triangle again, with the walk's own local ray and test.
struct TransparentList {
    float depth[IDK_TRANSPARENT_LAYERS];
    uint32_t tri[IDK_TRANSPARENT_LAYERS], xf[IDK_TRANSPARENT_LAYERS];
};

// One compare-and-swap pass down the list: the new fragment settles before the first entry it orders before and pushes the
// rest back; what falls off the end is dropped. Fully unrolled, so the list stays in registers.
__device__ __forceinline__ void transparent_insert(TransparentList& L, float depth, uint32_t tri, uint32_t xf) {
#pragma unroll
    for (int k = 0; k < IDK_TRANSPARENT_LAYERS; k++) {
        const bool before = depth < L.depth[k] || (depth == L.depth[k] && (tri < L.tri[k] || (tri == L.tri[k] && xf < L.xf[k])));
        if (before) {
            const float d = L.depth[k];
            const uint32_t t = L.tri[k], x = L.xf[k];
            L.depth[k] = depth; L.tri[k] = tri; L.xf[k] = xf;
            depth = d; tri = t; xf = x;
        }
    }
}

// The record pass's fragment tests for one instance: blended (AlphaCutoff == 2), front-facing or double-sided, depth in [0, 1]
// and LESS than the opaque depth, alpha not 0. A fragment that passes is recorded; the predicate never lets a triangle take the
// hit, so the walk's t bound stays where it started.
struct AcceptTransparentInstance {
    const float* projView;
    const float* positions;
    const float4* model;
    float det;
    f3 ld;
    uint32_t xf;
    float opaqueDepth;
    TransparentList* list;
    __device__ __forceinline__ bool operator()(const DeviceScene& sc, uint32_t i, float bx, float by, float) const {
        const int4 tri = __ldg(sc.blasTris + i);
        const GpuMaterial& mat = sc.materials[sc.meshes[tri.w].MaterialId];
        if (mat.AlphaCutoff != 2.0f) return false;
        if (!mat.IsDoubleSided) {
            const float4 nr = ldg4(sc.triRec + 4 * (size_t)i + 2);
            if (!gbuffer_front(det, mk3(nr.y, nr.z, nr.w), ld)) return false;
        }
        const float b2 = 1.0f - bx - by;
        const float depth = gbuffer_depth(projView, positions, model, tri, bx, by, b2);
        if (!(depth >= 0.0f && depth <= 1.0f && depth < opaqueDepth)) return false;
        if (gbuffer_alpha(sc, mat, tri, bx, by, b2) == 0.0f) return false;
        transparent_insert(*list, depth, i, xf);
        return false;
    }
};
struct AcceptTransparent {
    const float* projView;
    const float* positions;
    float opaqueDepth;
    TransparentList* list;
    __device__ __forceinline__ AcceptTransparentInstance at(const DeviceScene& sc, uint32_t xf, f3 ld) const {
        const float4* model = sc.xforms + 9 * (size_t)xf;
        return AcceptTransparentInstance{projView, positions, model, gbuffer_det(model), ld, xf, opaqueDepth, list};
    }
};

// The walk's bound: the distance from the eye to the opaque point the pixel's depth reconstructs on the ray (PerspectiveTransform
// of (ndc, depth)), times IDK_TRANSPARENT_T_MARGIN; unbounded (IDK_FLOAT_MAX) where the depth is not below 1 or the distance is
// not finite. The margin absorbs the rounding of depth against distance, so the bound never drops a fragment the depth test keeps.
__device__ __forceinline__ float transparent_t_max(const float* invProjView, f3 o, float ndcX, float ndcY, float opaqueDepth) {
    if (!(opaqueDepth < 1.0f)) return IDK_FLOAT_MAX;
    const f3 e = deferred_perspective(invProjView, ndcX, ndcY, opaqueDepth) - o;
    const float t = sqrtf(dot3(e, e)) * IDK_TRANSPARENT_T_MARGIN;
    return t <= IDK_FLOAT_MAX ? t : IDK_FLOAT_MAX;
}

struct TransparencyArgs {
    DeviceScene sc;
    const float* positions;        // PackedVec3 per vertex
    float projView[16], invProjView[16];
    float viewPos[3];
    float jitter[2];
    int w, h;
    const float* depth;            // the opaque depth [h][w] (D32F)
    float4* color;                 // the lit image [h][w], composited in place
    int shadowMode;                // 0 None, 1 Pcf, 2 RayTraced (no shadow on transparents)
    PointShadowMapsDev shadows;
    VxGridDev g;                   // VXGI only: the grid and the cone settings
    VxConeParams cone;
};

template <bool VXGI>
__global__ void __launch_bounds__(IDK_BLOCK) k_transparency(TransparencyArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    int x, y;
    if (!deferred_pixel(a.w, a.h, x, y)) return;
    const DeviceScene& sc = a.sc;
    const size_t p = (size_t)y * a.w + x;
    const float opaqueDepth = a.depth[p];
    // the ray of k_gbuffer (rule 1)
    const float ndcX = ((float)x + 0.5f) / (float)a.w * 2.0f - 1.0f - a.jitter[0];
    const float ndcY = ((float)y + 0.5f) / (float)a.h * 2.0f - 1.0f - a.jitter[1];
    const f3 o = mk3(a.viewPos[0], a.viewPos[1], a.viewPos[2]);
    const f3 d = normalize3(deferred_perspective(a.invProjView, ndcX, ndcY, 1.0f) - o);
    TransparentList L;
#pragma unroll
    for (int k = 0; k < IDK_TRANSPARENT_LAYERS; k++) {
        L.depth[k] = __int_as_float(0x7f800000); L.tri[k] = ~0u; L.xf[k] = ~0u;
    }
    HitRec hit;
    uint32_t hitXf, S = 0, T = 0, I = 0;
    float cost = 0.0f;
    trace_ray<false, false>(sc, o, d, transparent_t_max(a.invProjView, o, ndcX, ndcY, opaqueDepth), false, stack, hit, hitXf, S, T, I,
                            cost, AcceptTransparent{a.projView, a.positions, opaqueDepth, &L});
    if (L.tri[0] == ~0u) return;   // no layer: the pixel keeps its bytes

    // the record shader's fragment position at gl_FragCoord = (x + 0.5, y + 0.5, depth)
    const float nx = ((float)x + 0.5f) / (float)a.w * 2.0f - 1.0f, ny = ((float)y + 0.5f) / (float)a.h * 2.0f - 1.0f;
    const f3 viewPos = o;
    float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll 1
    for (int layer = 0; layer < IDK_TRANSPARENT_LAYERS && L.tri[0] != ~0u; layer++) {
        const uint32_t triIndex = L.tri[0];
        const int4 tri = __ldg(sc.blasTris + triIndex);
        const float4* mt = sc.xforms + 9 * (size_t)L.xf[0];
        const float depth = L.depth[0];
#pragma unroll
        for (int k = 0; k + 1 < IDK_TRANSPARENT_LAYERS; k++) {   // pop the front
            L.depth[k] = L.depth[k + 1]; L.tri[k] = L.tri[k + 1]; L.xf[k] = L.xf[k + 1];
        }
        L.tri[IDK_TRANSPARENT_LAYERS - 1] = ~0u;
        // the walk's barycentrics: trace_instance's local ray against the triangle record, the same test on the same inputs
        float b0, b1, b2;
        {
            const float4 r0 = ldg4(mt + 3), r1 = ldg4(mt + 4), r2 = ldg4(mt + 5);
            const f3 lo = xform_point(r0, r1, r2, o), ld = xform_vector(r0, r1, r2, d);
            float4 ta, tb, tc;
            ldg_tri(sc.triRec, triIndex, ta, tb, tc);
            float t;
            ray_triangle(lo, ld, mk3(ta.x, ta.y, ta.z), mk3(ta.w, tb.x, tb.y), mk3(tb.z, tb.w, tc.x), mk3(tc.y, tc.z, tc.w), b0, b1, t);
            b2 = 1.0f - b0 - b1;
        }

        Surface s;
        const f3 normal = gbuffer_surface(sc, triIndex, tri, mt, b0, b1, b2, d, s);
        const f3 fragPos = deferred_perspective(a.invProjView, nx, ny, depth);
        const f3 unjitteredFragPos = deferred_perspective(a.invProjView, nx - a.jitter[0], ny - a.jitter[1], depth);

        // EvaluateLighting with the surface's IOR (prevIor 1.0) and no ambient occlusion
        const float r = s.Roughness * s.Roughness;
        float r0 = (1.0f - s.IOR) / (1.0f + s.IOR);
        r0 *= r0;
        const f3 f0 = mk3(mix1(r0, s.Albedo.x, s.Metallic), mix1(r0, s.Albedo.y, s.Metallic), mix1(r0, s.Albedo.z, s.Metallic));
        const f3 diffuseBrdf = s.Albedo * (1.0f - 0.0f);
        const f3 V = normalize3(viewPos - fragPos);
        f3 direct = mk3(0.0f, 0.0f, 0.0f);
        for (uint32_t i = 0; i < sc.lightCount; i++) {
            const GpuLight& light = sc.lights[i];
            f3 contribution = deferred_evaluate_light(light, fragPos, normal, V, f0, diffuseBrdf, 1.0f - s.Metallic, fmaxf(r, 0.005f), fmaxf(r, 0.0001f));
            if (contribution.x != 0.0f || contribution.y != 0.0f || contribution.z != 0.0f) {
                // shadow = 1 - Visibility for Pcf, 0 otherwise (no shadow for RayTraced, as in the engine); contribution *= 1 - shadow
                float shadow = 0.0f;
                if (light.PointShadowIndex != -1 && a.shadowMode == 1) {
                    const f3 lightPos = mk3(light.Position[0], light.Position[1], light.Position[2]);
                    shadow = 1.0f - deferred_pcf(a.shadows, light.PointShadowIndex, unjitteredFragPos - lightPos);
                }
                contribution = contribution * (1.0f - shadow);
            }
            direct = direct + contribution;
        }
        f3 indirect;
        if (VXGI) {
            uint32_t steps = 0;
            const f3 incomming = fragPos - viewPos;
#define TR_NOISE(i) vx_ign((float)x + 0.5f, (float)y + 0.5f, i)
#define TR_SKY(dir) (sample_sky(sc, dir) * a.cone.giSkyBoxBoost)
            VX_INDIRECT_LIGHT(irradiance, a.g, a.cone.maxSamples, a.cone.noiseIndex, a.cone.stepMultiplier, a.cone.normalRayOffset, fragPos,
                              normal, s.Metallic, s.Roughness, incomming, TR_NOISE, TR_SKY, steps)
#undef TR_NOISE
#undef TR_SKY
            indirect = (irradiance * a.cone.giBoost) * s.Albedo;
        } else {
            indirect = mk3(0.015f, 0.015f, 0.015f) * s.Albedo;
        }
        const f3 c = (direct + indirect) + s.Emissive;
        // the rgba16f record of the premultiplied colour, blended front to back in fp32
        const float4 layerColor = make_float4(gbuffer_half(c.x * s.Alpha), gbuffer_half(c.y * s.Alpha), gbuffer_half(c.z * s.Alpha), gbuffer_half(s.Alpha));
        const float weight = 1.0f - acc.w;
        acc = make_float4(acc.x + weight * layerColor.x, acc.y + weight * layerColor.y, acc.z + weight * layerColor.z, acc.w + weight * layerColor.w);
    }
    const float4 opaque = a.color[p];
    const float k = 1.0f - acc.w;
    a.color[p] = make_float4(acc.x + k * opaque.x, acc.y + k * opaque.y, acc.z + k * opaque.z, 1.0f);
}
