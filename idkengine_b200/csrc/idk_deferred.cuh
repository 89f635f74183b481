// The raster mode's lighting of the G-buffer for sm_90a: the SSAO pass (SSAO.Compute, Source/Render/SSAO.cs:35-44) and the
// deferred lighting pass (RasterPipeline.Render's "Deferred Lighting" draw, RasterPipeline.cs:426-458), restated on the
// device. They read the G-buffer in place (or its upload), the point-shadow cube maps where k_point_shadow_faces rendered them,
// the ray-traced visibility images and the cone trace's indirect light, and chain on the device: SSAO -> deferred lighting.
//
//   k_ssao               SSAO/compute.glsl: one thread per G-buffer pixel, 8x8 pixel tiles (four per CTA); SampleCount
//                        cosine-weighted hemisphere samples tested against the G-buffer depth; R8Unorm result
//   k_deferred_lighting  DeferredLighting/fragment.glsl + DeferredLighting/include/Impl.glsl: one thread per G-buffer pixel,
//                        same tiles; every scene light (staged in shared memory per CTA) through the GGX BRDF of Pbr.glsl,
//                        shadowed by the 21-tap PCF filter, the ray-traced visibility images or not at all; rgba32f result
//                        (alpha 1). The engine's target is R11G11B10F; packing to it is the consumer's business.
//
// The rules are spelled out in DESIGN.md 8f.1d and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_volumetric.cuh"
#include "idk_shadows.cuh"

// The G-buffer attachments, float arrays in the engine's channel layout, [h][w] pixels each.
struct DeferredGBuffer {
    const float* depth;            // D32F
    const float2* normalRG;        // octahedral normal (RG8 in the engine)
    const float* albedo;           // rgb (R11G11B10F)
    const float2* metallicRoughness;
    const float* emissive;         // rgb (R11G11B10F)
    int w, h;
};

struct SsaoArgs {
    DeferredGBuffer g;
    uint8_t* out;                  // R8Unorm [h][w]
    float invProjView[16], projView[16];
    int sampleCount;
    float radius, strength;
    uint32_t noiseIndex;
};

// PerspectiveTransform(ndc, m) (Math.glsl:75-79): m * vec4(ndc, 1), then xyz / w.
__device__ __forceinline__ f3 deferred_perspective(const float* m, float x, float y, float z) {
    const float wx = ((m[0] * x + m[4] * y) + m[8] * z) + m[12] * 1.0f;
    const float wy = ((m[1] * x + m[5] * y) + m[9] * z) + m[13] * 1.0f;
    const float wz = ((m[2] * x + m[6] * y) + m[10] * z) + m[14] * 1.0f;
    const float ww = ((m[3] * x + m[7] * y) + m[11] * z) + m[15] * 1.0f;
    return mk3(wx / ww, wy / ww, wz / ww);
}

// imageStore into R8Unorm / the read of an R8Unorm texel: floor(clamp(v, 0, 1) * 255 + 0.5), the rule of the D16 store; NaN
// stores 0 (fmaxf returns the non-NaN operand).
__device__ __forceinline__ uint8_t deferred_r8(float v) { return (uint8_t)floorf(clamp1(v, 0.0f, 1.0f) * 255.0f + 0.5f); }

// The pixel of thread t of CTA b over w x h pixels in 8x8 tiles, four per CTA (k_volumetric_march's shape); false past the image.
__device__ __forceinline__ bool deferred_pixel(int w, int h, int& x, int& y) {
    const int tilesX = (w + 7) / 8;
    const int tile = (int)blockIdx.x * 4 + (int)threadIdx.x / 64, local = (int)threadIdx.x % 64;
    x = (tile % tilesX) * 8 + local % 8; y = (tile / tilesX) * 8 + local / 8;
    return x < w && y < h;
}

__global__ void __launch_bounds__(256) k_ssao(SsaoArgs a) {
    int x, y;
    if (!deferred_pixel(a.g.w, a.g.h, x, y)) return;
    const size_t p = (size_t)y * a.g.w + x;
    const float depth = a.g.depth[p];
    if (depth == 1.0f) { a.out[p] = 0; return; }
    const float u = ((float)x + 0.5f) / (float)a.g.w, v = ((float)y + 0.5f) / (float)a.g.h;
    const float2 nrg = a.g.normalRG[p];
    const f3 normal = decode_unit_vec(nrg.x, nrg.y);
    // PerspectiveTransformUvDepth(vec3(uv, depth), InvProjView): no jitter term
    f3 fragPos = deferred_perspective(a.invProjView, u * 2.0f - 1.0f, v * 2.0f - 1.0f, depth);
    fragPos = fragPos + normal * 0.04f;
    float occlusion = 0.0f;
    uint32_t noiseIndex = a.noiseIndex;
    const float radiusSq = a.radius * a.radius;
    for (int i = 0; i < a.sampleCount; i++) {
        const float rnd0 = ign_noise((float)x, (float)y, noiseIndex++);
        const float rnd1 = ign_noise((float)x, (float)y, noiseIndex++);
        const float rnd2 = ign_noise((float)x, (float)y, noiseIndex++);
        const f3 dir = normalize3(normal + sample_sphere(rnd0, rnd1));   // CosineSampleHemisphere
        const f3 samplePos = fragPos + (dir * a.radius) * rnd2;
        const f3 proj = deferred_perspective(a.projView, samplePos.x, samplePos.y, samplePos.z);
        const float su = proj.x * 0.5f + 0.5f, sv = proj.y * 0.5f + 0.5f;
        // texture(Depth, uv): NEAREST, clamp to edge
        const float sampleDepth = __ldg(a.g.depth + (size_t)nearest_texel(sv, a.g.h) * a.g.w + nearest_texel(su, a.g.w));
        if (proj.z > sampleDepth) {
            const f3 sampleToFrag = fragPos - samplePos;
            occlusion += dot3(sampleToFrag, sampleToFrag) / radiusSq;
        }
    }
    occlusion /= (float)a.sampleCount;
    occlusion *= a.strength;
    a.out[p] = deferred_r8(occlusion);
}

struct DeferredArgs {
    DeferredGBuffer g;
    const uint8_t* ssao;           // R8Unorm [h][w] (IsSSAO), else null
    const float4* indirect;        // rgba32f [h][w] (IsVXGI), else null
    const float* const* rtVisibility;   // one float [h][w] image per point shadow (ShadowMode RayTraced), else null
    const GpuLight* lights;
    int lightCount;                // <= IDK_GPU_MAX_UBO_LIGHT_COUNT
    PointShadowMapsDev shadows;    // ShadowMode Pcf
    float4* out;                   // rgba32f [h][w]
    float invProjView[16];
    float viewPos[3];
    float jitter[2];
    int shadowMode;                // 0 None, 1 Pcf, 2 RayTraced (RasterPipeline.ShadowMode)
};

// One PCF tap: texture(samplerCubeShadow, vec4(dir, ref)) with LINEAR filtering, compare LESS and seamless filtering, the
// same footprint-and-compare rule as point_shadow_visibility (idk_point_shadows.cuh). It is a second copy rather than a
// core factored out of that lookup because the factored version compiles the voxelisers to different (equivalent) SASS.
__device__ __forceinline__ float deferred_pcf_tap(const uint16_t* map, int size, float ref, f3 dir) {
    const CubeFootprint fp = cube_footprint(dir, size);
    const size_t n = (size_t)size;
    auto depth = [&](CubeTexel c) { return (float)__ldg(map + ((size_t)c.face * n + c.y) * n + c.x) / 65535.0f; };
    float d00 = fp.corner == 0 ? 0.0f : depth(fp.t00);
    float d10 = fp.corner == 1 ? 0.0f : depth(fp.t10);
    float d01 = fp.corner == 2 ? 0.0f : depth(fp.t01);
    float d11 = fp.corner == 3 ? 0.0f : depth(fp.t11);
    if (fp.corner >= 0) {
        const float mean = ((d00 + d10) + (d01 + d11)) / 3.0f;
        if (fp.corner == 0) d00 = mean; else if (fp.corner == 1) d10 = mean; else if (fp.corner == 2) d01 = mean; else d11 = mean;
    }
    const float c00 = ref < d00 ? 1.0f : 0.0f, c10 = ref < d10 ? 1.0f : 0.0f, c01 = ref < d01 ? 1.0f : 0.0f, c11 = ref < d11 ? 1.0f : 0.0f;
    return mix1(mix1(c00, c10, fp.fx), mix1(c01, c11, fp.fx), fp.fy);
}

// Visibility(pointShadow, normal, lightToSample) (Impl.glsl:38-64): 21 taps in table order, each at lightToSample + offset *
// 0.04 with ref = GetLightSpaceDepth(samplePos * (1 - 0.01)) clamped to [0, 1] and the footprint of samplePos, summed in
// order and divided by 21. A tap at the light itself or in a non-finite direction is lit.
__device__ __forceinline__ float deferred_pcf(const PointShadowMapsDev& m, int shadow, f3 lightToSample) {
    const PointShadowDev ps = m.shadows[shadow];
    const uint16_t* map = m.texels + ps.offset;
    // ShadowSampleOffsets as written (centre, the 8 corners, the 12 edge midpoints), one bit per tap and axis: component
    // nonzero (NZ), and if so negative (NEG). In registers, so the loop needs neither local nor constant memory.
    const uint32_t NZ[3] = {0x1FFFEu, 0x1E1FFEu, 0x1FE1FEu}, NEG[3] = {0x15998u, 0xC0CCCu, 0x1981E0u};
    float visibility = 0.0f;
#pragma unroll 1
    for (int i = 0; i < 21; i++) {
        auto off = [&](int axis) {   // offset * 0.04 (exact)
            return ((NZ[axis] >> i) & 1u) ? (((NEG[axis] >> i) & 1u) ? -1.0f : 1.0f) * 0.04f : 0.0f * 0.04f;
        };
        const f3 samplePos = lightToSample + mk3(off(0), off(1), off(2));
        const f3 b = samplePos * (1.0f - 0.01f);
        const float dist = fmaxf(fabsf(b.x), fmaxf(fabsf(b.y), fabsf(b.z)));
        float tap = 1.0f;
        if (dist > 0.0f && dist <= IDK_FLOAT_MAX) {
            const float ref = clamp1(point_shadow_depth(ps.nearPlane, ps.farPlane, dist), 0.0f, 1.0f);
            tap = deferred_pcf_tap(map, ps.size, ref, samplePos);
        }
        visibility += tap;
    }
    return visibility / 21.0f;
}

// EvaluateLighting (Impl.glsl:5-23) of one light, unshadowed: GGXBrdf with the per-surface terms precomputed by the caller
// (f0 = mix(vec3(r0), albedo, metallic) with r0 of the caller's IOR, diffuseBrdf = albedo * (1 - ao), 1 - metallic, and the
// squared roughness clamped for DistributionGGX (rD) and SmithGGXCorrelated (rG)); V = normalize(viewPos - fragPos).
__device__ __forceinline__ f3 deferred_evaluate_light(const GpuLight& light, f3 fragPos, f3 normal, f3 V, f3 f0, f3 diffuseBrdf,
                                                      float oneMinusMetallic, float rD, float rG) {
    const f3 lightPos = mk3(light.Position[0], light.Position[1], light.Position[2]);
    const f3 surfaceToLight = lightPos - fragPos;
    const f3 L = normalize3(surfaceToLight);
    const float distSq = dot3(surfaceToLight, surfaceToLight);
    const float lr = fmaxf(light.Radius, 0.0001f);
    const float attenuation = (lr * lr) / fmaxf(distSq, 0.0001f);   // GetAttenuationFactor
    const f3 H = normalize3(V + L);
    const float NoV = fabsf(dot3(normal, V));
    const float NoL = clamp1(dot3(normal, L), 0.0f, 1.0f);
    const float NoH = clamp1(dot3(normal, H), 0.0f, 1.0f);
    const float LoH = clamp1(dot3(L, H), 0.0f, 1.0f);
    const float aD = NoH * rD;                                        // DistributionGGX
    const float k = rD / ((1.0f - NoH * NoH) + aD * aD);
    const float D = (k * k) / IDK_PI;
    const float ggxl = NoV * sqrtf((-NoL * rG + NoL) * NoL + rG);     // SmithGGXCorrelated
    const float ggxv = NoL * sqrtf((-NoV * rG + NoV) * NoV + rG);
    const float G = 0.5f / (ggxv + ggxl);
    const float fw = det_exp((det_log2(1.0f - LoH) * 0.69314718f) * 5.0f);   // FresnelSchlick: pow(1 - LoH, 5)
    const f3 F = mk3(f0.x + (1.0f - f0.x) * fw, f0.y + (1.0f - f0.y) * fw, f0.z + (1.0f - f0.z) * fw);
    const f3 specular = F * (D * G);
    const f3 combined = specular + (diffuseBrdf * (mk3(1.0f, 1.0f, 1.0f) - F)) * oneMinusMetallic;
    const float cosTheta = clamp1(dot3(normal, L), 0.0f, 1.0f);
    return ((combined * attenuation) * cosTheta) * mk3(light.Color[0], light.Color[1], light.Color[2]);
}

// The fragment shader at one sample: every G-buffer read at texel p (imgCoord), the NDC from uv() (a float2, evaluated after
// the sky test). Hands the lit value (alpha 1; the sky, depth 1, is black) to store(float4). k_deferred_lighting runs it once
// per pixel, k_deferred_lighting_vrs (idk_vrs.cuh) once per coarse fragment. The callbacks keep k_deferred_lighting's SASS
// what it was before the body was shared.
template <class Uv, class Store>
__device__ __forceinline__ void deferred_shade(const DeferredArgs& a, const GpuLight* s_lights, size_t p, Uv&& uv, Store&& store) {
    const float depth = a.g.depth[p];
    if (depth == 1.0f) { store(make_float4(0.0f, 0.0f, 0.0f, 1.0f)); return; }

    const float2 uvs = uv();
    const float u = uvs.x, v = uvs.y;
    const float nx = u * 2.0f - 1.0f, ny = v * 2.0f - 1.0f;
    const f3 fragPos = deferred_perspective(a.invProjView, nx, ny, depth);
    const f3 unjitteredFragPos = deferred_perspective(a.invProjView, nx - a.jitter[0], ny - a.jitter[1], depth);
    const float ao = a.ssao ? (float)a.ssao[p] / 255.0f : 0.0f;   // an unbound texture unit reads 0

    const f3 albedo = mk3(a.g.albedo[3 * p], a.g.albedo[3 * p + 1], a.g.albedo[3 * p + 2]);
    const float2 nrg = a.g.normalRG[p];
    const f3 normal = decode_unit_vec(nrg.x, nrg.y);
    const float2 mr = a.g.metallicRoughness[p];
    const float metallic = mr.x, roughness = mr.y;
    const f3 emissive = mk3(a.g.emissive[3 * p], a.g.emissive[3 * p + 1], a.g.emissive[3 * p + 2]);

    // GGXBrdf's per-surface terms: squared roughness, f0 = mix(vec3(r0), albedo, metallic) with r0 of IOR 1.0 -> 1.0 as written
    const float r = roughness * roughness;
    float r0 = (1.0f - 1.0f) / (1.0f + 1.0f);
    r0 *= r0;
    const f3 f0 = mk3(mix1(r0, albedo.x, metallic), mix1(r0, albedo.y, metallic), mix1(r0, albedo.z, metallic));
    const float rD = fmaxf(r, 0.005f), rG = fmaxf(r, 0.0001f);
    const f3 diffuseBrdf = albedo * (1.0f - ao);
    const float oneMinusMetallic = 1.0f - metallic;
    const f3 viewPos = mk3(a.viewPos[0], a.viewPos[1], a.viewPos[2]);
    const f3 V = normalize3(viewPos - fragPos);

    f3 direct = mk3(0.0f, 0.0f, 0.0f);
    for (int i = 0; i < a.lightCount; i++) {
        const GpuLight& light = s_lights[i];
        const f3 lightPos = mk3(light.Position[0], light.Position[1], light.Position[2]);
        f3 contribution = deferred_evaluate_light(light, fragPos, normal, V, f0, diffuseBrdf, oneMinusMetallic, rD, rG);
        if ((contribution.x != 0.0f || contribution.y != 0.0f || contribution.z != 0.0f) && light.PointShadowIndex != -1) {
            if (a.shadowMode == 1) {
                contribution = contribution * deferred_pcf(a.shadows, light.PointShadowIndex, unjitteredFragPos - lightPos);
            } else if (a.shadowMode == 2) {   // the engine's R8Unorm image: the float input goes through the R8 store rule
                contribution = contribution * ((float)deferred_r8(a.rtVisibility[light.PointShadowIndex][p]) / 255.0f);
            }
        }
        direct = direct + contribution;
    }
    f3 indirect;
    if (a.indirect) {
        const float4 gi = a.indirect[p];
        indirect = mk3(gi.x, gi.y, gi.z) * albedo;
    } else {
        indirect = mk3(0.015f, 0.015f, 0.015f) * albedo;
    }
    const f3 c = (direct + indirect) + emissive;
    store(make_float4(c.x, c.y, c.z, 1.0f));
}

__global__ void __launch_bounds__(256) k_deferred_lighting(DeferredArgs a) {
    __shared__ GpuLight s_lights[IDK_GPU_MAX_UBO_LIGHT_COUNT];
    for (int i = threadIdx.x; i < a.lightCount; i += blockDim.x) s_lights[i] = a.lights[i];
    __syncthreads();
    int x, y;
    if (!deferred_pixel(a.g.w, a.g.h, x, y)) return;
    const size_t p = (size_t)y * a.g.w + x;
    deferred_shade(a, s_lights, p, [&]() { return make_float2(((float)x + 0.5f) / (float)a.g.w, ((float)y + 0.5f) / (float)a.g.h); },
                   [&](float4 c) { a.out[p] = c; });
}
