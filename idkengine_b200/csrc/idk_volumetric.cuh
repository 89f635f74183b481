// Volumetric point-light scattering for sm_90a: VolumetricLighting.Compute (Source/Render/VolumetricLighting.cs:57-81), its
// two dispatches restated on the device, reading the point-shadow cube maps where k_point_shadow_faces rendered them.
//
//   k_volumetric_march    VolumetricLight/compute.glsl: one thread per render pixel, 8x8 pixel tiles (four per CTA); per
//                         shadow (outer loop) SampleCount samples along the view ray (inner loop), each tested against the
//                         shadow's cube map with a NEAREST lookup and lit by Henyey-Greenstein in-scattering
//   k_volumetric_upscale  VolumetricLight/Upscale/compute.glsl: one thread per presentation pixel, four depth-weighted
//                         bilinear taps of the render-size image
//
// The rules are spelled out in DESIGN.md 8f.1c and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_point_shadows.cuh"
#include "idk_post.cuh"

// What the march reads of one shadow and of its light (Lights[shadow.LightIndex]), gathered into shared memory per CTA.
struct VolumetricShadowRec {
    float lightPos[3], radius, color[3];
    float nearPlane, farPlane;
    int size;
    unsigned long long offset;     // first texel of the shadow's cube map in VolumetricMarchArgs::maps
};

struct VolumetricMarchArgs {
    const PointShadowDev* shadows; // the context's point shadows (idkpt_set_point_shadows)
    const int32_t* lightIndex;     // their LightIndex, each below the scene's light count
    const GpuLight* lights;
    const uint16_t* maps;          // D16 cube maps, PointShadowMapsDev layout
    int count;
    const float* gdepth;           // G-buffer depth [gh][gw]
    int gw, gh;
    uint2* color;                  // render-size rgba16f result [h][w]
    float* depth;                  // render-size r32f depth [h][w]
    int w, h;
    float invProjView[16];
    float viewPos[3];
    float jitter[2];
    float absorbance[3];
    int sampleCount;
    float scattering, strength, maxDist;
};

// texture(sampler, uv) with NEAREST filtering and clamp to edge along one axis of n texels. The clamp is done in float so
// that a NaN coordinate selects texel 0 (fmaxf returns the non-NaN operand).
__device__ __forceinline__ int nearest_texel(float u, int n) {
    return (int)fminf(fmaxf(floorf(u * (float)n), 0.0f), (float)(n - 1));
}

// texture(samplerCube, dir).r with NEAREST filtering (seamless filtering does not apply): GL face selection, then texel
// clamp(floor(s * N), 0, N - 1), the same for t. D16 -> fp32 as D / 65535.
__device__ __forceinline__ float cube_nearest_d16(const uint16_t* map, int size, f3 d) {
    float s, t;
    const int face = cube_face_st(d, s, t);
    const int x = nearest_texel(s, size), y = nearest_texel(t, size);
    return (float)__ldg(map + ((size_t)face * size + y) * size + x) / 65535.0f;
}

// Dither pattern of VolumetricLight/compute.glsl:29-35 as written (0.22 where a Bayer table has 0.25); first index x % 4.
__constant__ float c_volumetric_dither[4][4] = {
    {0.0f, 0.5f, 0.125f, 0.625f}, {0.75f, 0.22f, 0.875f, 0.375f}, {0.1875f, 0.6875f, 0.0625f, 0.5625f}, {0.9375f, 0.4375f, 0.8125f, 0.3125f}};

__global__ void __launch_bounds__(256) k_volumetric_march(VolumetricMarchArgs a) {
    __shared__ VolumetricShadowRec s_rec[IDKPT_MAX_POINT_SHADOWS];
    for (int i = threadIdx.x; i < a.count; i += blockDim.x) {
        const PointShadowDev ps = a.shadows[i];
        const GpuLight& L = a.lights[a.lightIndex[i]];
        VolumetricShadowRec r;
        for (int k = 0; k < 3; k++) { r.lightPos[k] = L.Position[k]; r.color[k] = L.Color[k]; }
        r.radius = L.Radius;
        r.nearPlane = ps.nearPlane; r.farPlane = ps.farPlane;
        r.size = ps.size; r.offset = ps.offset;
        s_rec[i] = r;
    }
    __syncthreads();
    const int tilesX = (a.w + 7) / 8;
    const int tile = (int)blockIdx.x * 4 + (int)threadIdx.x / 64, local = (int)threadIdx.x % 64;
    const int x = (tile % tilesX) * 8 + local % 8, y = (tile / tilesX) * 8 + local / 8;
    if (x >= a.w || y >= a.h) return;   // partial tiles, and the CTA's tiles past the last one

    const float u = ((float)x + 0.5f) / (float)a.w, v = ((float)y + 0.5f) / (float)a.h;
    const float d = a.gdepth[(size_t)nearest_texel(v, a.gh) * a.gw + nearest_texel(u, a.gw)];
    // PerspectiveTransform(vec3(uv * 2 - 1 - Jitter, depth), InvProjView)
    const float nx = (u * 2.0f - 1.0f) - a.jitter[0], ny = (v * 2.0f - 1.0f) - a.jitter[1];
    const float* m = a.invProjView;
    const float wx = ((m[0] * nx + m[4] * ny) + m[8] * d) + m[12] * 1.0f;
    const float wy = ((m[1] * nx + m[5] * ny) + m[9] * d) + m[13] * 1.0f;
    const float wz = ((m[2] * nx + m[6] * ny) + m[10] * d) + m[14] * 1.0f;
    const float ww = ((m[3] * nx + m[7] * ny) + m[11] * d) + m[15] * 1.0f;
    const f3 viewPos = mk3(a.viewPos[0], a.viewPos[1], a.viewPos[2]);
    f3 viewToFrag = mk3(wx / ww, wy / ww, wz / ww) - viewPos;
    const float viewToFragLen = sqrtf(dot3(viewToFrag, viewToFrag));
    const f3 viewDir = viewToFrag / viewToFragLen;
    if (viewToFragLen > a.maxDist) viewToFrag = viewDir * a.maxDist;
    const float n = (float)a.sampleCount;
    const f3 deltaStep = viewToFrag / n;
    const f3 origin = viewPos + deltaStep * c_volumetric_dither[x % 4][y % 4];
    const f3 negViewDir = -viewDir;
    const float g = a.scattering;
    const float hgNum = 1.0f - g * g, hgBase = 1.0f + g * g, hg2g = 2.0f * g, fourPi = 4.0f * IDK_PI;

    f3 scattered = mk3(0.0f, 0.0f, 0.0f);
    for (int i = 0; i < a.count; i++) {   // UniformScatter(light, pointShadow, origin, viewDir, deltaStep, SampleCount)
        const VolumetricShadowRec& r = s_rec[i];
        const f3 lightPos = mk3(r.lightPos[0], r.lightPos[1], r.lightPos[2]);
        const uint16_t* map = a.maps + r.offset;
        f3 sum = mk3(0.0f, 0.0f, 0.0f);
        f3 samplePoint = origin;
        for (int k = 0; k < a.sampleCount; k++) {
            const f3 lightToSample = samplePoint - lightPos;
            // Shadow(): GetLogarithmicDepth of the max-norm distance against the nearest texel, no bias, no clamp
            const float dist = fmaxf(fabsf(lightToSample.x), fmaxf(fabsf(lightToSample.y), fabsf(lightToSample.z)));
            const float depth = point_shadow_depth(r.nearPlane, r.farPlane, dist);
            if (!(depth > cube_nearest_d16(map, r.size, lightToSample))) {
                const float len = sqrtf(dot3(lightToSample, lightToSample));
                const float lr = fmaxf(r.radius, 0.0001f), dsq = fmaxf(len * len, 0.0001f);
                const float attenuation = (lr * lr) / dsq;   // GetAttenuationFactor (Pbr.glsl:9-17)
                const f3 absorbed = mk3(det_exp(-a.absorbance[0] * len), det_exp(-a.absorbance[1] * len), det_exp(-a.absorbance[2] * len));
                const float cosTheta = dot3(lightToSample / len, negViewDir);
                // ComputeScattering: Henyey-Greenstein, pow(x, 1.5) = exp(log2(x) ln2 1.5)
                const float base = hgBase - hg2g * cosTheta;
                const float phase = hgNum / (fourPi * det_exp((det_log2(base) * 0.69314718f) * 1.5f));
                sum = sum + ((mk3(r.color[0], r.color[1], r.color[2]) * phase) * attenuation) * absorbed;
            }
            samplePoint = samplePoint + deltaStep;
        }
        sum = sum / n;
        const f3 e = origin - samplePoint;
        const float el = sqrtf(dot3(e, e));
        sum = sum * mk3(det_exp(-a.absorbance[0] * el), det_exp(-a.absorbance[1] * el), det_exp(-a.absorbance[2] * el));
        scattered = scattered + sum;
    }
    const size_t p = (size_t)y * a.w + x;
    a.color[p] = post_pack_half(scattered * a.strength);
    a.depth[p] = d;
}

struct VolumetricUpscaleArgs {
    const float* gdepth;           // G-buffer depth [gh][gw]
    int gw, gh;
    PostImage march;               // render-size rgba16f result
    const float* depth;            // render-size r32f depth, same size
    uint2* out;                    // presentation-size rgba16f [H][W]
    int W, H;
    float nearPlane, farPlane;
};

// LogarithmicDepthToLinearViewDepth (Math.glsl:68-73), with its [-1, 1] formula, over FarPlane
__device__ __forceinline__ float volumetric_linear_depth(float nearPlane, float farPlane, float z) {
    return ((2.0f * nearPlane) * farPlane) / ((farPlane + nearPlane) - z * (farPlane - nearPlane)) / farPlane;
}

__global__ void __launch_bounds__(256) k_volumetric_upscale(VolumetricUpscaleArgs a) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.W || y >= a.H) return;
    const float fw = (float)a.W, fh = (float)a.H;
    const float u = ((float)x + 0.5f) / fw, v = ((float)y + 0.5f) / fh;
    const float high = volumetric_linear_depth(a.nearPlane, a.farPlane, a.gdepth[(size_t)nearest_texel(v, a.gh) * a.gw + nearest_texel(u, a.gw)]);
    const int ox = x % 2 == 0 ? -1 : 1, oy = y % 2 == 0 ? -1 : 1;
    const int dx[4] = {0, 0, ox, ox}, dy[4] = {0, oy, 0, oy};
    f3 color = mk3(0.0f, 0.0f, 0.0f);
    float total = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float su = ((float)(x + dx[i]) + 0.5f) / fw, sv = ((float)(y + dy[i]) + 0.5f) / fh;
        const f3 c = post_bilinear(a.march, su, sv, 0, 0);
        const float low = volumetric_linear_depth(a.nearPlane, a.farPlane,
                                                  __ldg(a.depth + (size_t)nearest_texel(sv, a.march.h_) * a.march.w + nearest_texel(su, a.march.w)));
        const float wt = fmaxf(1.0f - 0.05f * fabsf(low - high), 0.0f);
        color = color + c * wt;
        total = total + wt;
    }
    a.out[(size_t)y * a.W + x] = post_pack_half(color / (total + 0.0001f));
}
