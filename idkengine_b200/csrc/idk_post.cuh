// Present chain of the path-traced frame (SURVEY.md 8f.3): Bloom.Compute(PathTracerPipeline.Result) followed by
// TonemapAndGamma.Compute(Result, Bloom.Result) (Application.cs:217-223), producing the RGBA8 frame the swapchain shows,
// without leaving the device.
//   k_bloom_down / k_bloom_up   Bloom/compute.glsl (13-tap downsample + prefilter, 3x3 tent upsample), Bloom.cs:56-130
//   k_agx_matrices, k_tonemap   TonemapAndGammaCorrect/compute.glsl (AgX dual-section curve, sRGB transfer, Bayer dither)
// Texture sampling follows the rule DESIGN.md states for VXGI: bilinear filtering evaluated explicitly in fp32
// (lerp in x, then y; clamp-to-edge; texel offsets applied before the clamp); the bloom mip chain is rgba16f with
// round-to-nearest-even stores.
#pragma once
#include "idk_device.cuh"
#include <cuda_fp16.h>

struct PostImage {          // one 2-D level: rgba32f (f != null) or rgba16f (h != null)
    const float4* f;
    const uint2* h;
    int w, h_;
};

__device__ __forceinline__ f3 post_fetch(const PostImage& t, int x, int y) {
    if (t.f) { const float4 v = __ldg(t.f + (size_t)y * t.w + x); return mk3(v.x, v.y, v.z); }
    const uint2 v = __ldg(t.h + (size_t)y * t.w + x);
    return mk3(__half2float(__ushort_as_half((unsigned short)(v.x & 0xFFFFu))), __half2float(__ushort_as_half((unsigned short)(v.x >> 16))),
               __half2float(__ushort_as_half((unsigned short)(v.y & 0xFFFFu))));
}
__device__ __forceinline__ int post_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
__device__ __forceinline__ f3 post_lerp(f3 a, f3 b, float t) {
    const float s = 1.0f - t;
    return mk3(a.x * s + b.x * t, a.y * s + b.y * t, a.z * s + b.z * t);
}
// textureLodOffset(sampler2D, uv, lod, ivec2(ox, oy)).rgb on one level
__device__ __forceinline__ f3 post_bilinear(const PostImage& t, float u, float v, int ox, int oy) {
    const float px = u * (float)t.w - 0.5f, py = v * (float)t.h_ - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    const int x0 = post_clampi((int)fx0 + ox, 0, t.w - 1), x1 = post_clampi((int)fx0 + 1 + ox, 0, t.w - 1);
    const int y0 = post_clampi((int)fy0 + oy, 0, t.h_ - 1), y1 = post_clampi((int)fy0 + 1 + oy, 0, t.h_ - 1);
    const f3 a = post_lerp(post_fetch(t, x0, y0), post_fetch(t, x1, y0), fx);
    const f3 b = post_lerp(post_fetch(t, x0, y1), post_fetch(t, x1, y1), fx);
    return post_lerp(a, b, fy);
}
__device__ __forceinline__ uint2 post_pack_half(f3 c) {   // imageStore(vec4(c, 1.0)) into rgba16f
    const uint32_t r = __half_as_ushort(__float2half_rn(c.x)), g = __half_as_ushort(__float2half_rn(c.y));
    const uint32_t b = __half_as_ushort(__float2half_rn(c.z)), a = __half_as_ushort(__float2half_rn(1.0f));
    return make_uint2(r | (g << 16), b | (a << 16));
}

struct BloomDownArgs {
    PostImage src;
    uint2* dst;
    int dw, dh;
    int prefilter;          // the shader's Lod uniform is 0: down levels 0 and 1
    float maxColor, threshold;
};

__global__ void __launch_bounds__(256) k_bloom_down(BloomDownArgs a) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.dw || y >= a.dh) return;
    const float u = ((float)x + 0.5f) / (float)a.dw, v = ((float)y + 0.5f) / (float)a.dh;
    const PostImage& s = a.src;
    const f3 center = post_bilinear(s, u, v, 0, 0);
    const f3 yellowUpRight = post_bilinear(s, u, v, 0, 2);
    const f3 yellowDownLeft = post_bilinear(s, u, v, -2, 0);
    const f3 greenDownRight = post_bilinear(s, u, v, 2, 0);
    const f3 blueDownLeft = post_bilinear(s, u, v, 0, -2);
    f3 yellow = post_bilinear(s, u, v, -2, 2);
    yellow = yellow + yellowUpRight; yellow = yellow + center; yellow = yellow + yellowDownLeft;
    f3 green = yellowUpRight;
    green = green + post_bilinear(s, u, v, 2, 2); green = green + greenDownRight; green = green + center;
    f3 blue = center;
    blue = blue + greenDownRight; blue = blue + post_bilinear(s, u, v, 2, -2); blue = blue + blueDownLeft;
    f3 lila = yellowDownLeft;
    lila = lila + center; lila = lila + blueDownLeft; lila = lila + post_bilinear(s, u, v, -2, -2);
    f3 red = post_bilinear(s, u, v, -1, 1);
    red = red + post_bilinear(s, u, v, 1, 1); red = red + post_bilinear(s, u, v, 1, -1); red = red + post_bilinear(s, u, v, -1, -1);
    f3 result = (red * 0.5f + (((yellow + green) + blue) + lila) * 0.125f) * 0.25f;
    if (a.prefilter) {   // Prefilter(), Bloom/compute.glsl:124-137
        const float knee = 0.2f;
        f3 color = mk3(fminf(a.maxColor, result.x), fminf(a.maxColor, result.y), fminf(a.maxColor, result.z));
        const float brightness = fmaxf(fmaxf(color.x, color.y), color.z);
        const float cx = a.threshold - knee, cy = knee * 2.0f, cz = 0.25f / knee;
        float rq = clamp1(brightness - cx, 0.0f, cy);
        rq = (rq * rq) * cz;
        const float k = fmaxf(rq, brightness - a.threshold) / fmaxf(brightness, 0.0001f);
        result = color * k;
    }
    a.dst[(size_t)y * a.dw + x] = post_pack_half(result);
}

struct BloomUpArgs {
    PostImage up;           // SamplerUpsample at Lod
    PostImage down;         // SamplerDownsample at Lod
    uint2* dst;
    int dw, dh;
};

__global__ void __launch_bounds__(256) k_bloom_up(BloomUpArgs a) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.dw || y >= a.dh) return;
    const float u = ((float)x + 0.5f) / (float)a.dw, v = ((float)y + 0.5f) / (float)a.dh;
    const PostImage& s = a.up;
    f3 r = post_bilinear(s, u, v, -1, 1) * 1.0f;
    r = r + post_bilinear(s, u, v, 0, 1) * 2.0f;
    r = r + post_bilinear(s, u, v, 1, 1) * 1.0f;
    r = r + post_bilinear(s, u, v, -1, 0) * 2.0f;
    r = r + post_bilinear(s, u, v, 0, 0) * 4.0f;
    r = r + post_bilinear(s, u, v, 1, 0) * 2.0f;
    r = r + post_bilinear(s, u, v, -1, -1) * 1.0f;
    r = r + post_bilinear(s, u, v, 0, -1) * 2.0f;
    r = r + post_bilinear(s, u, v, 1, -1) * 1.0f;
    r = r / 16.0f;
    a.dst[(size_t)y * a.dw + x] = post_pack_half(r + post_bilinear(a.down, u, v, 0, 0));
}

// ---- AgX (TonemapAndGammaCorrect/compute.glsl:71-167). mat3 are column-major: m[c][r].
struct PostMat3 { float m[3][3]; };

__device__ __forceinline__ f3 post_mul(const PostMat3& M, f3 v) {
    return mk3((M.m[0][0] * v.x + M.m[1][0] * v.y) + M.m[2][0] * v.z,
               (M.m[0][1] * v.x + M.m[1][1] * v.y) + M.m[2][1] * v.z,
               (M.m[0][2] * v.x + M.m[1][2] * v.y) + M.m[2][2] * v.z);
}
__device__ __forceinline__ PostMat3 post_matmul(const PostMat3& A, const PostMat3& B) {   // A * B
    PostMat3 R;
    for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++) R.m[c][r] = (A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1]) + A.m[2][r] * B.m[c][2];
    return R;
}
__device__ __forceinline__ PostMat3 post_inverse(const PostMat3& A) {   // adjugate / determinant
    const float a00 = A.m[0][0], a01 = A.m[0][1], a02 = A.m[0][2];
    const float a10 = A.m[1][0], a11 = A.m[1][1], a12 = A.m[1][2];
    const float a20 = A.m[2][0], a21 = A.m[2][1], a22 = A.m[2][2];
    const float b01 = a22 * a11 - a12 * a21;
    const float b11 = a12 * a20 - a22 * a10;
    const float b21 = a21 * a10 - a11 * a20;
    const float det = (a00 * b01 + a01 * b11) + a02 * b21;
    PostMat3 R;
    R.m[0][0] = b01 / det;
    R.m[0][1] = (a02 * a21 - a22 * a01) / det;
    R.m[0][2] = (a12 * a01 - a02 * a11) / det;
    R.m[1][0] = b11 / det;
    R.m[1][1] = (a22 * a00 - a02 * a20) / det;
    R.m[1][2] = (a02 * a10 - a12 * a00) / det;
    R.m[2][0] = b21 / det;
    R.m[2][1] = (a01 * a20 - a21 * a00) / det;
    R.m[2][2] = (a11 * a00 - a01 * a10) / det;
    return R;
}
__device__ __forceinline__ f3 post_unproject(float x, float y) {   // xyYToXYZ(vec3(x, y, 1))
    const float Y = 1.0f;
    return mk3((x * Y) / y, Y, (((1.0f - x) - y) * Y) / y);
}
__device__ __forceinline__ PostMat3 post_primaries(float rx, float ry, float gx, float gy, float bx, float by, float wx, float wy) {
    const f3 R = post_unproject(rx, ry), G = post_unproject(gx, gy), B = post_unproject(bx, by), W = post_unproject(wx, wy);
    PostMat3 t;
    t.m[0][0] = R.x; t.m[0][1] = 1.0f; t.m[0][2] = R.z;
    t.m[1][0] = G.x; t.m[1][1] = 1.0f; t.m[1][2] = G.z;
    t.m[2][0] = B.x; t.m[2][1] = 1.0f; t.m[2][2] = B.z;
    const f3 scale = post_mul(post_inverse(t), W);
    PostMat3 o;
    o.m[0][0] = R.x * scale.x; o.m[0][1] = R.y * scale.x; o.m[0][2] = R.z * scale.x;
    o.m[1][0] = G.x * scale.y; o.m[1][1] = G.y * scale.y; o.m[1][2] = G.z * scale.y;
    o.m[2][0] = B.x * scale.z; o.m[2][1] = B.y * scale.z; o.m[2][2] = B.z * scale.z;
    return o;
}
__device__ __forceinline__ float post_mix(float a, float b, float t) { return a * (1.0f - t) + b * t; }

struct PostTonemapConsts {
    PostMat3 srgbToAdjusted, adjustedToSrgb;
    float exposureScale;        // pow(2.0, Exposure)
};

// One thread: the per-frame constants every pixel of the shader recomputes.
__global__ void k_agx_matrices(float exposure, float compression, PostTonemapConsts* out) {
    const PostMat3 sRGB_to_XYZ = post_primaries(0.64f, 0.33f, 0.3f, 0.6f, 0.15f, 0.06f, 0.3127f, 0.3290f);
    const float scale_factor = 1.0f / (1.0f - compression);
    const float wx = 0.3127f, wy = 0.3290f;
    const PostMat3 adjusted_to_XYZ = post_primaries(post_mix(wx, 0.64f, scale_factor), post_mix(wy, 0.33f, scale_factor),
                                                    post_mix(wx, 0.3f, scale_factor), post_mix(wy, 0.6f, scale_factor),
                                                    post_mix(wx, 0.15f, scale_factor), post_mix(wy, 0.06f, scale_factor), wx, wy);
    const PostMat3 XYZ_to_adjusted = post_inverse(adjusted_to_XYZ);
    out->srgbToAdjusted = post_matmul(sRGB_to_XYZ, XYZ_to_adjusted);
    out->adjustedToSrgb = post_inverse(out->srgbToAdjusted);
    out->exposureScale = det_exp(exposure * 0.69314718f);   // pow(2, e) = exp(e ln 2)
}

__device__ __forceinline__ float post_dual_section(float x, float linear, float peak) {
    const float S = peak * linear;
    if (x < S) return x;
    const float C = peak / (peak - S);
    return peak - (peak - S) * det_exp(((0.0f - C) * (x - S)) / peak);
}
__device__ __forceinline__ float post_linear_to_srgb(float x) {
    if (x < 0.0031308f) return x * 12.92f;
    return 1.055f * det_exp((det_log2(x) * 0.69314718f) * (1.0f / 2.4f)) - 0.055f;   // pow(x, 1/2.4)
}

struct TonemapArgs {
    PostImage src0, src1;       // src1.f == src1.h == null: not bound
    uchar4* dst;
    int w, h;
    float saturation, linear, peak;
    int doTonemap;
    const PostTonemapConsts* consts;
};

__constant__ unsigned char c_bayer8[8][8] = {
    {1, 49, 13, 61, 4, 52, 16, 64}, {33, 17, 45, 29, 36, 20, 48, 32}, {9, 57, 5, 53, 12, 60, 8, 56}, {41, 25, 37, 21, 44, 28, 40, 24},
    {3, 51, 15, 63, 2, 50, 14, 62}, {35, 19, 47, 31, 34, 18, 46, 30}, {11, 59, 7, 55, 10, 58, 6, 54}, {43, 27, 39, 23, 42, 26, 38, 22}};

__global__ void __launch_bounds__(256) k_tonemap(TonemapArgs a) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.w || y >= a.h) return;
    const float u = ((float)x + 0.5f) / (float)a.w, v = ((float)y + 0.5f) / (float)a.h;
    f3 hdr = mk3(0.0f, 0.0f, 0.0f);
    hdr = hdr + post_bilinear(a.src0, u, v, 0, 0);
    if (a.src1.f || a.src1.h) hdr = hdr + post_bilinear(a.src1, u, v, 0, 0);
    f3 c;
    if (a.doTonemap) {
        const PostTonemapConsts& k = *a.consts;
        f3 wc = mk3(fmaxf(hdr.x, 0.0f), fmaxf(hdr.y, 0.0f), fmaxf(hdr.z, 0.0f)) * k.exposureScale;
        wc = post_mul(k.srgbToAdjusted, wc);
        wc = mk3(clamp1(post_dual_section(wc.x, a.linear, a.peak), 0.0f, 1.0f), clamp1(post_dual_section(wc.y, a.linear, a.peak), 0.0f, 1.0f),
                 clamp1(post_dual_section(wc.z, a.linear, a.peak), 0.0f, 1.0f));
        const float desat = (wc.x * 0.2126729f + wc.y * 0.7151522f) + wc.z * 0.0721750f;
        wc = mk3(post_mix(desat, wc.x, a.saturation), post_mix(desat, wc.y, a.saturation), post_mix(desat, wc.z, a.saturation));
        wc = mk3(clamp1(wc.x, 0.0f, 1.0f), clamp1(wc.y, 0.0f, 1.0f), clamp1(wc.z, 0.0f, 1.0f));
        wc = post_mul(k.adjustedToSrgb, wc);
        c = mk3(post_linear_to_srgb(wc.x), post_linear_to_srgb(wc.y), post_linear_to_srgb(wc.z));
    } else {
        c = mk3(clamp1(hdr.x, 0.0f, 1.0f), clamp1(hdr.y, 0.0f, 1.0f), clamp1(hdr.z, 0.0f, 1.0f));
    }
    // Dither(): BayerMatrix8[x % 8][y % 8], entries n / 65
    const float bayer = (float)((double)c_bayer8[x & 7][y & 7] / 65.0);
    const float ditherVal = (bayer - 0.5f) / 64.0f;
    c = mk3(c.x + ditherVal, c.y + ditherVal, c.z + ditherVal);
    // imageStore into R8G8B8A8Unorm: clamp, scale, round to nearest
    const unsigned char r = (unsigned char)floorf(clamp1(c.x, 0.0f, 1.0f) * 255.0f + 0.5f);
    const unsigned char g = (unsigned char)floorf(clamp1(c.y, 0.0f, 1.0f) * 255.0f + 0.5f);
    const unsigned char b = (unsigned char)floorf(clamp1(c.z, 0.0f, 1.0f) * 255.0f + 0.5f);
    a.dst[(size_t)y * a.w + x] = make_uchar4(r, g, b, 255);
}

// ------------------------------------------------------------------------------------------------ denoise hand-off (SURVEY 8f.3)
// PathTracerPipeline.Denoise (PathTracerPipeline.cs:165-194) downloads Result / Albedo / Normal as packed RGB floats into
// OIDN buffers, runs the filter on the host side and uploads the output. Here the three images are packed into the same
// OIDN layout (Format.Float3, width*height*3 floats) ON THE DEVICE -- an OIDN CUDA device can wrap those pointers with
// oidnNewSharedBuffer, nothing crosses PCIe -- and, so that the chain also works without the OIDN library, a guided
// edge-avoiding a-trous wavelet filter (Dammertz et al. 2010: 5x5 B3-spline taps, step 1, 2, 4, ..; colour / normal / albedo
// edge-stopping weights, colour sigma halved per iteration; albedo demodulated before filtering and re-applied after) produces
// the "Denoised" output texture. Deterministic fp32 (fixed tap order, no FMA, det_exp), restated by oracle/oracle_post.inc.
struct DenoisePrepareArgs {
    const float4* result; const float4* albedo; const float4* normal;
    float* oidnBeauty; float* oidnAlbedo; float* oidnNormal;     // packed RGB floats (OIDN Format.Float3)
    float4* work;                                                // filter input: (demodulated) colour
    int count, demodulate;
};

__global__ void __launch_bounds__(256) k_denoise_prepare(DenoisePrepareArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.count) return;
    const float4 c = a.result[i], al = a.albedo[i], n = a.normal[i];
    a.oidnBeauty[3 * (size_t)i] = c.x; a.oidnBeauty[3 * (size_t)i + 1] = c.y; a.oidnBeauty[3 * (size_t)i + 2] = c.z;
    a.oidnAlbedo[3 * (size_t)i] = al.x; a.oidnAlbedo[3 * (size_t)i + 1] = al.y; a.oidnAlbedo[3 * (size_t)i + 2] = al.z;
    a.oidnNormal[3 * (size_t)i] = n.x; a.oidnNormal[3 * (size_t)i + 1] = n.y; a.oidnNormal[3 * (size_t)i + 2] = n.z;
    f3 v = mk3(c.x, c.y, c.z);
    if (a.demodulate) v = mk3(v.x / fmaxf(al.x, 0.001f), v.y / fmaxf(al.y, 0.001f), v.z / fmaxf(al.z, 0.001f));
    a.work[i] = make_float4(v.x, v.y, v.z, 1.0f);
}

struct DenoiseAtrousArgs {
    const float4* in; float4* out;
    const float4* albedo; const float4* normal;
    int w, h, step;
    float invSigmaColor2, invSigmaNormal2, invSigmaAlbedo2, invStep2;
};

__global__ void __launch_bounds__(256) k_denoise_atrous(DenoiseAtrousArgs a) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.w || y >= a.h) return;
    const size_t p = (size_t)y * a.w + x;
    const float4 cp4 = a.in[p], ap4 = a.albedo[p], np4 = a.normal[p];
    const f3 cp = mk3(cp4.x, cp4.y, cp4.z), ap = mk3(ap4.x, ap4.y, ap4.z), np_ = mk3(np4.x, np4.y, np4.z);
    const float kw[3] = {0.375f, 0.25f, 0.0625f};
    f3 sum = mk3(0.0f, 0.0f, 0.0f);
    float wsum = 0.0f;
    for (int dy = -2; dy <= 2; dy++) {
        for (int dx = -2; dx <= 2; dx++) {
            const int qx = x + dx * a.step, qy = y + dy * a.step;
            if (qx < 0 || qy < 0 || qx >= a.w || qy >= a.h) continue;
            const size_t q = (size_t)qy * a.w + qx;
            const float4 cq4 = __ldg(a.in + q), aq4 = __ldg(a.albedo + q), nq4 = __ldg(a.normal + q);
            const f3 cq = mk3(cq4.x, cq4.y, cq4.z);
            const f3 dc = cq - cp, dn = mk3(nq4.x, nq4.y, nq4.z) - np_, da = mk3(aq4.x, aq4.y, aq4.z) - ap;
            const float wc = fminf(det_exp(-(dot3(dc, dc) * a.invSigmaColor2)), 1.0f);
            const float wn = fminf(det_exp(-(fmaxf(dot3(dn, dn) * a.invStep2, 0.0f) * a.invSigmaNormal2)), 1.0f);
            const float wa = fminf(det_exp(-(dot3(da, da) * a.invSigmaAlbedo2)), 1.0f);
            const float w = ((wc * wn) * wa) * (kw[dx < 0 ? -dx : dx] * kw[dy < 0 ? -dy : dy]);
            sum = sum + cq * w;
            wsum = wsum + w;
        }
    }
    a.out[p] = make_float4(sum.x / wsum, sum.y / wsum, sum.z / wsum, 1.0f);
}

struct DenoiseFinishArgs {
    const float4* filtered; const float4* albedo;
    float4* denoised; float* oidnOutput;
    int count, demodulate;
};

__global__ void __launch_bounds__(256) k_denoise_finish(DenoiseFinishArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.count) return;
    const float4 c = a.filtered[i], al = a.albedo[i];
    f3 v = mk3(c.x, c.y, c.z);
    if (a.demodulate) v = mk3(v.x * fmaxf(al.x, 0.001f), v.y * fmaxf(al.y, 0.001f), v.z * fmaxf(al.z, 0.001f));
    a.denoised[i] = make_float4(v.x, v.y, v.z, 1.0f);
    a.oidnOutput[3 * (size_t)i] = v.x; a.oidnOutput[3 * (size_t)i + 1] = v.y; a.oidnOutput[3 * (size_t)i + 2] = v.z;
}
