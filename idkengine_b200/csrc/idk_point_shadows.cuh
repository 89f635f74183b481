// Point-shadow cube maps for sm_90a: the depth cube map the engine's raster pass draws for a light with PointShadowIndex >= 0
// (PointShadowManager.RenderShadowMaps, CpuPointShadow.RenderShadowMap), traced instead of rasterised, and the PCF lookup of
// the voxeliser's fragment stage into it (Voxelize/fragment.glsl:100-117).
//
//   k_point_shadow_faces     one thread per texel, 8x8 texel tiles (four per CTA), grid = CTAs x faces in the mask:
//                            one closest-hit ray per texel centre, trace_ray<false, false>, lights off
//   point_shadow_visibility  texture(samplerCubeShadow, vec4(lightToSample, ref)): LINEAR, compare LESS, seamless
//
// The rules are spelled out in DESIGN.md 8f.1b and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_kernels.cuh"

// What the device reads of a GpuPointShadow, plus where its map lives in the context's allocation.
struct PointShadowDev {
    float pos[3];
    float nearPlane, farPlane;
    int size;                      // face size N
    unsigned long long offset;     // first texel of face 0 in PointShadowMapsDev::texels (6 * N^2 texels per shadow)
};

struct PointShadowMapsDev {
    const PointShadowDev* shadows;
    const uint16_t* texels;        // D16, face-major (+X,-X,+Y,-Y,+Z,-Z), row y = t, x fastest
    uint32_t count;
};

// GetLogarithmicDepth (Math.glsl:59-66), IEEE divides, no FMA.
__device__ __forceinline__ float point_shadow_depth(float nearPlane, float farPlane, float viewZ) {
    return (1.0f / viewZ - 1.0f / nearPlane) / (1.0f / farPlane - 1.0f / nearPlane);
}

// Direction through the centre of texel (x, y) of `face`: the inverse of GL table 8.19 with major component 1, so that the
// ray parameter is the face's view depth.
__device__ __forceinline__ f3 point_shadow_texel_dir(int face, int x, int y, int size) {
    const float sc = (float)(2 * x + 1) / (float)size - 1.0f, tc = (float)(2 * y + 1) / (float)size - 1.0f;
    switch (face) {
        case 0: return mk3(1.0f, -tc, -sc);
        case 1: return mk3(-1.0f, -tc, sc);
        case 2: return mk3(sc, 1.0f, tc);
        case 3: return mk3(sc, -1.0f, -tc);
        case 4: return mk3(sc, -tc, 1.0f);
        default: return mk3(-sc, -tc, -1.0f);
    }
}

struct PointShadowRenderArgs {
    DeviceScene sc;
    float pos[3];
    float nearPlane, farPlane;
    int size;
    uint16_t* map;                 // this shadow's 6 * size^2 texels
    int faces[6];                  // blockIdx.y -> face
};

// The depth a rasteriser stores at a texel centre: the closest surface along the ray through it after near/far clipping
// (the ray starts on the near plane and ends on the far plane), no face culling. D16 = floor(clamp(d, 0, 1) * 65535 + 0.5);
// nothing in range = 65535, the value ShadowMap.Fill(1.0) clears to.
__global__ void __launch_bounds__(IDK_BLOCK) k_point_shadow_faces(PointShadowRenderArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    const int n = a.size, tilesX = (n + 7) / 8;
    const int tile = (int)blockIdx.x * (IDK_BLOCK / 64) + (int)threadIdx.x / 64, local = (int)threadIdx.x % 64;
    const int x = (tile % tilesX) * 8 + local % 8, y = (tile / tilesX) * 8 + local / 8;
    if (x >= n || y >= n) return;   // partial tiles, and the CTA's tiles past the last one
    const int face = a.faces[blockIdx.y];
    const f3 d = point_shadow_texel_dir(face, x, y, n);
    const f3 o = mk3(a.pos[0] + d.x * a.nearPlane, a.pos[1] + d.y * a.nearPlane, a.pos[2] + d.z * a.nearPlane);
    HitRec hit;
    uint32_t xf, S = 0, T = 0, I = 0;
    float cost = 0.0f;
    uint16_t v = 65535u;
    if (trace_ray<false, false>(a.sc, o, d, a.farPlane - a.nearPlane, false, stack, hit, xf, S, T, I, cost)) {
        const float depth = point_shadow_depth(a.nearPlane, a.farPlane, a.nearPlane + hit.t);
        v = (uint16_t)floorf(clamp1(depth, 0.0f, 1.0f) * 65535.0f + 0.5f);
    }
    a.map[((size_t)face * n + y) * n + x] = v;
}

// Visibility(pointShadow, lightToSample) (fragment.glsl:100-117): texture(samplerCubeShadow, vec4(lightToSample, ref)) with
// LINEAR filtering, compare LESS and seamless cube filtering. ref = GetLightSpaceDepth of the 2 %-biased point, clamped to
// [0, 1] (fixed-point depth texture); the footprint is that of the unbiased direction (cube_footprint). Each tap compares
// ref < depth in fp32 (depth = D16 / 65535); at a cube corner the missing tap's depth is the mean of the other three and is
// compared like them (GL: texel selection, then compare). The four results are filtered with the fp32 bilinear weights in
// mix order. A sample at the light itself (no direction) is visible.
__device__ __forceinline__ float point_shadow_visibility(const PointShadowMapsDev& m, int shadow, f3 lightToSample) {
    const PointShadowDev ps = m.shadows[shadow];
    const f3 b = lightToSample * (1.0f - 0.02f);
    const float dist = fmaxf(fabsf(b.x), fmaxf(fabsf(b.y), fabsf(b.z)));
    if (!(dist > 0.0f)) return 1.0f;
    const float ref = clamp1(point_shadow_depth(ps.nearPlane, ps.farPlane, dist), 0.0f, 1.0f);
    const CubeFootprint fp = cube_footprint(lightToSample, ps.size);
    const uint16_t* map = m.texels + ps.offset;
    const size_t n = (size_t)ps.size;
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
