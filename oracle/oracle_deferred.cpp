// ORACLE (TEST INFRASTRUCTURE ONLY) -- the raster mode's G-buffer lighting: SSAO and the deferred lighting pass with its
// PCF / ray-traced point shadows and VXGI indirect light.
//
// Part of liboracle.so (wrapped by tests/deferred_oracle.py). It includes oracle_point_shadows.cpp (and with it oracle.cpp)
// and reuses its cube-map footprint (CubeFootprint),
// GetLogarithmicDepth, DecodeUnitVec, SampleSphere, InterleavedGradientNoise and the det_exp / det_log2 polynomials
// unchanged; what it adds is restated here from the shaders.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/SSAO/compute.glsl                          the SSAO pass; Source/Render/SSAO.cs (settings, R8Unorm)
//   Resource/Shaders/DeferredLighting/fragment.glsl             the deferred lighting pass
//   Resource/Shaders/DeferredLighting/include/Impl.glsl         EvaluateLighting, GetLightSpaceDepth, Visibility (21-tap PCF)
//   Resource/Shaders/include/Pbr.glsl                           GetAttenuationFactor, BaseReflectivity, DistributionGGX,
//                                                                SmithGGXCorrelated, FresnelSchlick, GGXBrdf
//   Resource/Shaders/include/Math.glsl:75-87                    PerspectiveTransform, PerspectiveTransformUvDepth
//   Source/Render/CpuPointShadow.cs:211-218, 242                 the shadow sampler (LINEAR, compare LESS); R8Unorm RT images
#pragma once
#include "oracle_point_shadows.cpp"

namespace {

// PerspectiveTransform(ndc, m): m * vec4(ndc, 1.0), xyz / w
static inline vec3 DfPerspective(const float* m, float x, float y, float z) {
    const float wx = ((m[0] * x + m[4] * y) + m[8] * z) + m[12] * 1.0f;
    const float wy = ((m[1] * x + m[5] * y) + m[9] * z) + m[13] * 1.0f;
    const float wz = ((m[2] * x + m[6] * y) + m[10] * z) + m[14] * 1.0f;
    const float ww = ((m[3] * x + m[7] * y) + m[11] * z) + m[15] * 1.0f;
    return V(wx / ww, wy / ww, wz / ww);
}

// Texel of texture(sampler, uv) along an axis of n texels, NEAREST with clamp to edge, clamped in float (NaN -> texel 0).
static inline int DfNearest(float u, int n) { return (int)fminf(fmaxf(floorf(u * (float)n), 0.0f), (float)(n - 1)); }

// An R8Unorm store: round(clamp(v, 0, 1) * 255), halves up; NaN stores 0.
static inline uint8_t DfStoreR8(float v) {
    if (v != v) return 0;
    return (uint8_t)floorf(clampf(v, 0.0f, 1.0f) * 255.0f + 0.5f);
}

// SSAO/compute.glsl at w x h.
static void Ssao(const GpuPerFrameData& f, const IdkPtSsaoSettings& st, const float* depth, const float* nrg, int w, int h, uint8_t* out) {
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const size_t p = (size_t)y * w + x;
            if (depth[p] == 1.0f) { out[p] = 0; continue; }
            const float u = ((float)x + 0.5f) / (float)w, v = ((float)y + 0.5f) / (float)h;
            const vec3 normal = DecodeUnitVec(nrg[2 * p], nrg[2 * p + 1]);
            vec3 fragPos = DfPerspective(f.InvProjView, u * 2.0f - 1.0f, v * 2.0f - 1.0f, depth[p]);
            fragPos = fragPos + normal * 0.04f;
            float occlusion = 0.0f;
            uint32_t noiseIndex = st.NoiseIndex;
            for (int i = 0; i < st.SampleCount; i++) {
                const float rnd0 = InterleavedGradientNoise((float)x, (float)y, noiseIndex++);
                const float rnd1 = InterleavedGradientNoise((float)x, (float)y, noiseIndex++);
                const float rnd2 = InterleavedGradientNoise((float)x, (float)y, noiseIndex++);
                const vec3 samplePos = fragPos + CosineSampleHemisphere(normal, rnd0, rnd1) * st.Radius * rnd2;
                vec3 projected = DfPerspective(f.ProjView, samplePos.x, samplePos.y, samplePos.z);
                projected.x = projected.x * 0.5f + 0.5f;
                projected.y = projected.y * 0.5f + 0.5f;
                const float sampleDepth = depth[(size_t)DfNearest(projected.y, h) * w + DfNearest(projected.x, w)];
                if (projected.z > sampleDepth) {
                    const vec3 sampleToFrag = fragPos - samplePos;
                    occlusion += dot(sampleToFrag, sampleToFrag) / (st.Radius * st.Radius);
                }
            }
            occlusion /= (float)st.SampleCount;
            occlusion *= st.Strength;
            out[p] = DfStoreR8(occlusion);
        }
}

// pow(x, y) as the library evaluates it: exp(log2(x) * ln2 * y)
static inline float DfPow(float x, float y) { return det_exp((det_log2(x) * 0.69314718f) * y); }

struct DfSurface { vec3 Albedo, Normal, Emissive; float Metallic, Roughness, IOR; };

// GGXBrdf (Pbr.glsl:69-93) with DistributionGGX, SmithGGXCorrelated, FresnelSchlick and BaseReflectivity as written.
static vec3 GGXBrdf(DfSurface surface, vec3 Vd, vec3 Ld, float prevIor, vec3& F) {
    surface.Roughness *= surface.Roughness;
    float r0 = (prevIor - surface.IOR) / (prevIor + surface.IOR);
    r0 *= r0;
    const vec3 f0 = mix(V(r0, r0, r0), surface.Albedo, surface.Metallic);
    const vec3 f90 = V(1.0f, 1.0f, 1.0f);
    const vec3 H = normalize(Vd + Ld);
    const float NoV = fabsf(dot(surface.Normal, Vd));
    const float NoL = clampf(dot(surface.Normal, Ld), 0.0f, 1.0f);
    const float NoH = clampf(dot(surface.Normal, H), 0.0f, 1.0f);
    const float LoH = clampf(dot(Ld, H), 0.0f, 1.0f);
    float roughness = fmaxf(surface.Roughness, 0.005f);       // DistributionGGX
    const float a = NoH * roughness;
    const float k = roughness / (1.0f - NoH * NoH + a * a);
    const float D = k * k / PI_F;
    roughness = fmaxf(surface.Roughness, 0.0001f);             // SmithGGXCorrelated
    const float ggxl = NoV * sqrtf((-NoL * roughness + NoL) * NoL + roughness);
    const float ggxv = NoL * sqrtf((-NoV * roughness + NoV) * NoV + roughness);
    const float G = 0.5f / (ggxv + ggxl);
    const float p = DfPow(1.0f - LoH, 5.0f);                   // FresnelSchlick
    F = f0 + (f90 - f0) * p;
    return D * G * F;
}

// EvaluateLighting (Impl.glsl:5-23)
static vec3 EvaluateLighting(const GpuLight& light, const DfSurface& surface, vec3 fragPos, vec3 viewPos, float ambientOcclusion) {
    const vec3 surfaceToLight = V(light.Position) - fragPos;
    const vec3 dirSurfaceToCam = normalize(viewPos - fragPos);
    const vec3 dirSurfaceToLight = normalize(surfaceToLight);
    const float distSq = dot(surfaceToLight, surfaceToLight);
    const float lightRadius = fmaxf(light.Radius, 0.0001f);    // GetAttenuationFactor
    const float attenuation = (lightRadius * lightRadius) / fmaxf(distSq, 0.0001f);
    vec3 fresnelTerm;
    const vec3 specularBrdf = GGXBrdf(surface, dirSurfaceToCam, dirSurfaceToLight, 1.0f, fresnelTerm);
    const vec3 diffuseBrdf = surface.Albedo * (1.0f - ambientOcclusion);
    const vec3 combinedBrdf = specularBrdf + diffuseBrdf * (V(1.0f, 1.0f, 1.0f) - fresnelTerm) * (1.0f - surface.Metallic);
    const float cosTheta = clampf(dot(surface.Normal, dirSurfaceToLight), 0.0f, 1.0f);
    return combinedBrdf * attenuation * cosTheta * V(light.Color);
}

// texture(samplerCubeShadow, vec4(dir, ref)): LINEAR, compare LESS, seamless (CubeFootprint of the point-shadow oracle; a
// missing corner texel is the mean of the other three). A zero or non-finite direction is lit.
static float DfShadowTexture(const uint16_t* map, int size, vec3 dir, float ref) {
    const float m = fmaxf(fabsf(dir.x), fmaxf(fabsf(dir.y), fabsf(dir.z)));
    if (!(m > 0.0f) || std::isinf(m)) return 1.0f;
    const CubeTaps f = CubeFootprint(size, dir);
    float d[4];
    for (int k = 0; k < 4; k++) d[k] = k == f.corner ? 0.0f : (float)map[((size_t)f.face[k] * size + f.y[k]) * size + f.x[k]] / 65535.0f;
    if (f.corner >= 0) d[f.corner] = ((d[0] + d[1]) + (d[2] + d[3])) / 3.0f;
    float c[4];
    for (int k = 0; k < 4; k++) c[k] = ref < d[k] ? 1.0f : 0.0f;
    return mixf(mixf(c[0], c[1], f.fx), mixf(c[2], c[3], f.fx), f.fy);
}

// Visibility (Impl.glsl:38-64): 21 taps at lightToSample + offset * 0.04, ref = GetLightSpaceDepth(samplePos * (1 - 0.01))
// clamped to [0, 1] (fixed-point depth format).
static float DfVisibility(const GpuPointShadow& ps, int size, const uint16_t* map, vec3 lightToSample) {
    static const float ShadowSampleOffsets[21][3] = {
        {0.0f, 0.0f, 0.0f},
        {1.0f, 1.0f, 1.0f}, {1.0f, -1.0f, 1.0f}, {-1.0f, -1.0f, 1.0f}, {-1.0f, 1.0f, 1.0f},
        {1.0f, 1.0f, -1.0f}, {1.0f, -1.0f, -1.0f}, {-1.0f, -1.0f, -1.0f}, {-1.0f, 1.0f, -1.0f},
        {1.0f, 1.0f, 0.0f}, {1.0f, -1.0f, 0.0f}, {-1.0f, -1.0f, 0.0f}, {-1.0f, 1.0f, 0.0f},
        {1.0f, 0.0f, 1.0f}, {-1.0f, 0.0f, 1.0f}, {1.0f, 0.0f, -1.0f}, {-1.0f, 0.0f, -1.0f},
        {0.0f, 1.0f, 1.0f}, {0.0f, -1.0f, 1.0f}, {0.0f, -1.0f, -1.0f}, {0.0f, 1.0f, -1.0f}};
    const float bias = 0.01f, sampleDiskRadius = 0.04f;
    float visibilityFactor = 0.0f;
    for (int i = 0; i < 21; i++) {
        const vec3 samplePos = lightToSample + V(ShadowSampleOffsets[i]) * sampleDiskRadius;
        const vec3 b = samplePos * (1.0f - bias);
        const float dist = fmaxf(fabsf(b.x), fmaxf(fabsf(b.y), fabsf(b.z)));
        const float depth = clampf(GetLogarithmicDepth(ps.NearPlane, ps.FarPlane, dist), 0.0f, 1.0f);
        visibilityFactor += DfShadowTexture(map, size, samplePos, depth);
    }
    visibilityFactor /= 21.0f;
    return visibilityFactor;
}

struct DfInputs {
    const GpuLight* lights; uint64_t lightCount;
    const GpuPointShadow* shadows; const int32_t* sizes; const uint16_t* texels; int shadowCount;
    const float *depth, *nrg, *albedo, *mr, *emissive;
    const uint8_t* ssao;           // IsSSAO, else null
    const float* indirect;         // IsVXGI (rgba32f), else null
    const float* const* rt;        // ShadowMode 2
};

// DeferredLighting/fragment.glsl at w x h into rgba32f (alpha 1).
static void DeferredLighting(const GpuPerFrameData& f, int shadowMode, const DfInputs& in, int w, int h, const float* jitter, float* out) {
    std::vector<size_t> offsets(std::max(in.shadowCount, 0), 0);
    for (int i = 1; i < in.shadowCount; i++) offsets[i] = offsets[i - 1] + 6 * (size_t)in.sizes[i - 1] * (size_t)in.sizes[i - 1];
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const size_t p = (size_t)y * w + x;
            float* o = out + 4 * p;
            const float depth = in.depth[p];
            if (depth == 1.0f) { o[0] = o[1] = o[2] = 0.0f; o[3] = 1.0f; continue; }
            const float uvx = ((float)x + 0.5f) / (float)w, uvy = ((float)y + 0.5f) / (float)h;
            const vec3 ndc = V(uvx * 2.0f - 1.0f, uvy * 2.0f - 1.0f, depth);
            const vec3 fragPos = DfPerspective(f.InvProjView, ndc.x, ndc.y, ndc.z);
            const vec3 unjitteredFragPos = DfPerspective(f.InvProjView, ndc.x - jitter[0], ndc.y - jitter[1], ndc.z);
            const float ambientOcclusion = in.ssao ? (float)in.ssao[p] / 255.0f : 0.0f;
            DfSurface surface;
            surface.Albedo = V(in.albedo + 3 * p);
            surface.Normal = DecodeUnitVec(in.nrg[2 * p], in.nrg[2 * p + 1]);
            surface.Metallic = in.mr[2 * p];
            surface.Roughness = in.mr[2 * p + 1];
            surface.Emissive = V(in.emissive + 3 * p);
            surface.IOR = 1.0f;
            vec3 directLighting = V(0, 0, 0);
            for (uint64_t i = 0; i < in.lightCount; i++) {
                const GpuLight& light = in.lights[i];
                vec3 contribution = EvaluateLighting(light, surface, fragPos, V(f.ViewPos), ambientOcclusion);
                if (contribution.x != 0.0f || contribution.y != 0.0f || contribution.z != 0.0f) {
                    const int k = light.PointShadowIndex;
                    if (k == -1) {
                    } else if (shadowMode == 1) {
                        const vec3 lightToSample = unjitteredFragPos - V(light.Position);
                        contribution = contribution * DfVisibility(in.shadows[k], in.sizes[k], in.texels + offsets[k], lightToSample);
                    } else if (shadowMode == 2) {
                        contribution = contribution * ((float)DfStoreR8(in.rt[k][p]) / 255.0f);
                    }
                }
                directLighting = directLighting + contribution;
            }
            vec3 indirectLight;
            if (in.indirect) indirectLight = V(in.indirect + 4 * p) * surface.Albedo;
            else indirectLight = V(0.015f, 0.015f, 0.015f) * surface.Albedo;
            const vec3 c = (directLighting + indirectLight) + surface.Emissive;
            o[0] = c.x; o[1] = c.y; o[2] = c.z; o[3] = 1.0f;
        }
}

} // namespace

extern "C" {

// SSAO.Compute (idkpt_ssao): depth [h][w], octahedral normal [h][w][2] -> R8Unorm [h][w]. Returns 0, or -1 for an argument the
// library rejects.
ORACLE_API int oracle_ssao(const GpuPerFrameData* frame, const IdkPtSsaoSettings* st, const float* depth, const float* nrg, int w, int h, uint8_t* out) {
    if (st->SampleCount < 1 || st->SampleCount > 1024 || w < 1 || h < 1) return -1;
    Ssao(*frame, *st, depth, nrg, w, h, out);
    return 0;
}

// The deferred lighting draw (idkpt_deferred_lighting): `shadowCount` shadows with their face sizes and maps back to back; ssao
// (R8, IsSSAO) / indirect (rgba32f, IsVXGI) null when off; rt: one float image per shadow (ShadowMode 2). out: w*h*4 floats.
// Returns 0, or -1 for an argument the library rejects.
ORACLE_API int oracle_deferred_lighting(const GpuLight* lights, uint64_t lightCount, const GpuPerFrameData* frame, int shadowMode,
                                        const GpuPointShadow* shadows, const int32_t* sizes, const uint16_t* texels, int shadowCount,
                                        const float* depth, const float* nrg, const float* albedo, const float* mr, const float* emissive,
                                        int w, int h, const float* jitter, const uint8_t* ssao, const float* indirect,
                                        const float* const* rt, int rtCount, float* out) {
    if (shadowMode < 0 || shadowMode > 2 || w < 1 || h < 1) return -1;
    if (shadowMode != 0)
        for (uint64_t i = 0; i < lightCount; i++)
            if (lights[i].PointShadowIndex != -1 && (lights[i].PointShadowIndex < 0 || lights[i].PointShadowIndex >= shadowCount)) return -1;
    if (shadowMode == 2 && rtCount < shadowCount) return -1;
    const float noJitter[2] = {0.0f, 0.0f};
    const DfInputs in = {lights, lightCount, shadows, sizes, texels, shadowCount, depth, nrg, albedo, mr, emissive, ssao, indirect, rt};
    DeferredLighting(*frame, shadowMode, in, w, h, jitter ? jitter : noJitter, out);
    return 0;
}

// The PCF filter on its own, for n light-to-sample vectors into one map.
ORACLE_API void oracle_deferred_visibility(const GpuPointShadow* shadow, int size, const uint16_t* map, const float* lightToSample,
                                           uint64_t n, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = DfVisibility(*shadow, size, map, V(lightToSample + 3 * i));
}

// GGXBrdf on its own (n surfaces: albedo[3], metallic, roughness, normal[3], V[3], L[3] per row of 14 floats) -> specular rgb
// and F rgb (6 floats per row).
ORACLE_API void oracle_ggx_brdf(const float* rows, uint64_t n, float* out) {
    for (uint64_t i = 0; i < n; i++) {
        const float* r = rows + 14 * i;
        DfSurface s;
        s.Albedo = V(r); s.Metallic = r[3]; s.Roughness = r[4]; s.Normal = V(r + 5); s.Emissive = V(0, 0, 0); s.IOR = 1.0f;
        vec3 F;
        const vec3 spec = GGXBrdf(s, V(r + 8), V(r + 11), 1.0f, F);
        float* o = out + 6 * i;
        o[0] = spec.x; o[1] = spec.y; o[2] = spec.z; o[3] = F.x; o[4] = F.y; o[5] = F.z;
    }
}

// The R8Unorm store rule on its own.
ORACLE_API void oracle_store_r8(const float* v, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = DfStoreR8(v[i]);
}

} // extern "C"
