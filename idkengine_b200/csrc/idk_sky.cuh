// The engine's sky cube map generated on the device for sm_90a: SkyBoxManager's two GPU passes, written into the context's sky
// (6 faces x n^2 rgba32f texels, +X,-X,+Y,-Y,+Z,-Z, row y = t of GL table 8.19) in the layout idkpt_set_sky fills.
//
//   k_sky_atmosphere   AtmosphericScattering/compute.glsl (AtmosphericScatterer.Compute): one thread per texel, 8x8 CTAs x 6
//                      faces as the engine dispatches it; the single-scattering march with ISteps primary and JSteps light
//                      samples, stored in fp32 with alpha 1
//   k_sky_equirect     UnprojectEquirectangular/compute.glsl (SkyBoxManager.LoadSkyBoxEquirectangular): one thread per texel,
//                      the same grid; the texel direction's (atan, asin) coordinate, a bilinear REPEAT lookup of the RGB16F
//                      source, SrgbToLinear, rounded to the RGBA16F face format
//
// The rules are spelled out in DESIGN.md 8f.1j and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include <cuda_fp16.h>
#include "idk_device.cuh"

// GetWorldSpaceDirection(ndc, face) (Math.glsl:17-39), normalised.
__device__ __forceinline__ f3 sky_face_direction(int face, float x, float y) {
    f3 d;
    switch (face) {
        case 0: d = mk3(1.0f, -y, -x); break;
        case 1: d = mk3(-1.0f, -y, x); break;
        case 2: d = mk3(x, 1.0f, y); break;
        case 3: d = mk3(x, -1.0f, -y); break;
        case 4: d = mk3(x, -y, 1.0f); break;
        default: d = mk3(-x, -y, -1.0f); break;
    }
    return normalize3(d);
}

// The texel this thread writes, and its direction: uv = (xy + 0.5) / n, ndc = uv * 2 - 1.
__device__ __forceinline__ bool sky_texel(int n, int& x, int& y, int& face, f3& dir) {
    x = blockIdx.x * blockDim.x + threadIdx.x;
    y = blockIdx.y * blockDim.y + threadIdx.y;
    face = blockIdx.z;
    if (x >= n || y >= n) return false;
    const float u = ((float)x + 0.5f) / (float)n, v = ((float)y + 0.5f) / (float)n;
    dir = sky_face_direction(face, u * 2.0f - 1.0f, v * 2.0f - 1.0f);
    return true;
}

// Rsi: the ray r0 + t rd against the sphere of radius sr around the origin; (1e5, -1e5) when it misses.
__device__ __forceinline__ void sky_rsi(f3 r0, f3 rd, float sr, float& t0, float& t1) {
    const float a = dot3(rd, rd);
    const float b = 2.0f * dot3(rd, r0);
    const float c = dot3(r0, r0) - sr * sr;
    const float d = b * b - 4.0f * a * c;
    if (d < 0.0f) { t0 = 1e5f; t1 = -1e5f; return; }
    t0 = (-b - sqrtf(d)) / (2.0f * a);
    t1 = (-b + sqrtf(d)) / (2.0f * a);
}

struct SkyAtmosphereArgs {
    float4* faces;
    int n;
    int iSteps, jSteps;
    float lightIntensity;          // already max(LightIntensity, 0)
    float azimuth, elevation;
};

// Atmosphere() with main()'s arguments: the ray from (0, 6376e3, 0), a 6371 km planet under a 6471 km atmosphere, Rayleigh
// (5.5, 13.0, 22.4)e-6 at 8 km, Mie 21e-6 at 1.2 km with g = 0.758.
__device__ __forceinline__ f3 sky_atmosphere(f3 r, f3 pSun, float iSun, int iSteps, int jSteps) {
    const f3 r0 = mk3(0.0f, 6376e3f, 0.0f);
    const float rPlanet = 6371e3f, rAtmos = 6471e3f;
    const f3 kRlh = mk3(5.5e-6f, 13.0e-6f, 22.4e-6f);
    const float kMie = 21e-6f, shRlh = 8e3f, shMie = 1.2e3f, g = 0.758f;
    pSun = normalize3(pSun);
    r = normalize3(r);
    float px, py;
    sky_rsi(r0, r, rAtmos, px, py);
    if (px > py) return mk3(0.0f, 0.0f, 0.0f);
    float planetNear, planetFar;
    sky_rsi(r0, r, rPlanet, planetNear, planetFar);
    py = fminf(py, planetNear);    // also when planetNear is the 1e5 sentinel or behind the origin, as written
    const float iStepSize = (py - px) / (float)iSteps;
    float iTime = 0.0f;            // the march starts at the origin, not at px, as written
    f3 totalRlh = mk3(0.0f, 0.0f, 0.0f), totalMie = mk3(0.0f, 0.0f, 0.0f);
    float iOdRlh = 0.0f, iOdMie = 0.0f;
    const float mu = dot3(r, pSun);
    const float mumu = mu * mu;
    const float gg = g * g;
    const float pRlh = 3.0f / (16.0f * IDK_PI) * (1.0f + mumu);
    const float powBase = 1.0f + gg - 2.0f * mu * g;
    const float pMie = 3.0f / (8.0f * IDK_PI) * ((1.0f - gg) * (mumu + 1.0f)) /
                       (det_exp((det_log2(powBase) * 0.69314718f) * 1.5f) * (2.0f + gg));
#pragma unroll 1
    for (int i = 0; i < iSteps; i++) {
        const f3 iPos = r0 + r * (iTime + iStepSize * 0.5f);
        const float iHeight = sqrtf(dot3(iPos, iPos)) - rPlanet;
        const float odStepRlh = det_exp(-iHeight / shRlh) * iStepSize;
        const float odStepMie = det_exp(-iHeight / shMie) * iStepSize;
        iOdRlh += odStepRlh;
        iOdMie += odStepMie;
        float s0, s1;
        sky_rsi(iPos, pSun, rAtmos, s0, s1);
        const float jStepSize = s1 / (float)jSteps;
        float jTime = 0.0f, jOdRlh = 0.0f, jOdMie = 0.0f;
#pragma unroll 1
        for (int j = 0; j < jSteps; j++) {
            const f3 jPos = iPos + pSun * (jTime + jStepSize * 0.5f);
            const float jHeight = sqrtf(dot3(jPos, jPos)) - rPlanet;
            jOdRlh += det_exp(-jHeight / shRlh) * jStepSize;
            jOdMie += det_exp(-jHeight / shMie) * jStepSize;
            jTime += jStepSize;
        }
        const float odMie = kMie * (iOdMie + jOdMie), odRlh = iOdRlh + jOdRlh;
        const f3 attn = mk3(det_exp(-(odMie + kRlh.x * odRlh)), det_exp(-(odMie + kRlh.y * odRlh)), det_exp(-(odMie + kRlh.z * odRlh)));
        totalRlh = totalRlh + odStepRlh * attn;
        totalMie = totalMie + odStepMie * attn;
        iTime += iStepSize;
    }
    return iSun * ((pRlh * kRlh) * totalRlh + (pMie * kMie) * totalMie);
}

__global__ void __launch_bounds__(64) k_sky_atmosphere(SkyAtmosphereArgs a) {
    int x, y, face;
    f3 dir;
    if (!sky_texel(a.n, x, y, face, dir)) return;
    float sinTheta, cosTheta, sinPhi, cosPhi;   // PolarToCartesian(Azimuth, Elevation) (Math.glsl:139-153)
    det_sincos(a.elevation, &sinTheta, &cosTheta);
    det_sincos(a.azimuth, &sinPhi, &cosPhi);
    const f3 sun = mk3(sinTheta * cosPhi, cosTheta, sinTheta * sinPhi) * 1.0f;
    const f3 c = sky_atmosphere(dir, sun, a.lightIntensity, a.iSteps, a.jSteps);
    a.faces[((size_t)face * a.n + y) * a.n + x] = make_float4(c.x, c.y, c.z, 1.0f);
}

struct SkyEquirectArgs {
    const float* rgb;              // [h][w][3] fp32, row 0 first (t = 0)
    int w, h;
    float4* faces;
    int n;
};

__device__ __forceinline__ float sky_half(float v) { return __half2float(__float2half_rn(v)); }

// One texel of the RGB16F source.
__device__ __forceinline__ f3 sky_source(const SkyEquirectArgs& a, int x, int y) {
    const float* p = a.rgb + ((size_t)y * a.w + x) * 3;
    return mk3(sky_half(__ldg(p)), sky_half(__ldg(p + 1)), sky_half(__ldg(p + 2)));
}

// SrgbToLinear for one channel; a NaN passes through (the pow rule's det_log2 would turn it into a number).
__device__ __forceinline__ float sky_srgb_to_linear(float s) {
    if (s != s) return s;
    if (s < 0.04045f) return s / 12.92f;
    return det_exp((det_log2((s + 0.055f) / 1.055f) * 0.69314718f) * 2.4f);
}

__global__ void __launch_bounds__(64) k_sky_equirect(SkyEquirectArgs a) {
    int x, y, face;
    f3 dir;
    if (!sky_texel(a.n, x, y, face, dir)) return;
    // SampleSphericalMap, then texture() at level 0: bilinear with REPEAT on both texel indices (GL 4.6 8.14.2)
    const float u = det_atan2(dir.z, dir.x) * 0.1591f + 0.5f;
    const float v = det_asin(dir.y) * 0.3183f + 0.5f;
    const float px = u * (float)a.w - 0.5f, py = v * (float)a.h - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    const int x0 = tex_wrap((int)fx0, a.w, 10497), x1 = tex_wrap((int)fx0 + 1, a.w, 10497);
    const int y0 = tex_wrap((int)fy0, a.h, 10497), y1 = tex_wrap((int)fy0 + 1, a.h, 10497);
    const float gx = 1.0f - fx, gy = 1.0f - fy;
    const f3 c00 = sky_source(a, x0, y0), c10 = sky_source(a, x1, y0), c01 = sky_source(a, x0, y1), c11 = sky_source(a, x1, y1);
    const f3 top = mk3(c00.x * gx + c10.x * fx, c00.y * gx + c10.y * fx, c00.z * gx + c10.z * fx);
    const f3 bottom = mk3(c01.x * gx + c11.x * fx, c01.y * gx + c11.y * fx, c01.z * gx + c11.z * fx);
    const f3 c = mk3(top.x * gy + bottom.x * fy, top.y * gy + bottom.y * fy, top.z * gy + bottom.z * fy);
    // alpha: the source's 1 filters to within an ulp of 1, which the RGBA16F face rounds to 1
    a.faces[((size_t)face * a.n + y) * a.n + x] =
        make_float4(sky_half(sky_srgb_to_linear(c.x)), sky_half(sky_srgb_to_linear(c.y)), sky_half(sky_srgb_to_linear(c.z)), 1.0f);
}
