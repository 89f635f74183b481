// The end of the raster frame for sm_90a: SSR.Compute, the "Merge Textures" dispatch and TaaResolve.Compute
// (RasterPipeline.Render, RasterPipeline.cs:595-614), restated on the device. They read the G-buffer, the lit image (a caller
// array, the deferred lighting image or the merged image), the context's sky and the TAA history, and chain on the device:
// deferred lighting -> SSR + merge -> TAA resolve.
//
//   k_ssr            SSR/compute.glsl fused with MergeTextures/compute.glsl: one thread per G-buffer pixel, 8x8 pixel tiles
//                    (four per CTA); a view-space ray march against the G-buffer depth with the shader's binary search, the
//                    source colour at the hit or the sky on a miss; rgba16f SSR image and rgba32f merged image (source + SSR)
//   k_taa_resolve    TAAResolve/compute.glsl: one thread per presentation pixel, same tiles; naive or neighbourhood-clamped
//                    resolve of the render-size colour against the rgba16f history (Catmull-Rom in nine bilinear taps)
//
// The rules are spelled out in DESIGN.md 8f.1e and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_deferred.cuh"

// imageStore(vec4(c, alpha)) into rgba16f, round to nearest even (post_pack_half with the alpha as an argument: SSR's early out
// stores alpha 0)
__device__ __forceinline__ uint2 ssr_pack_half(f3 c, float alpha) {
    const uint32_t r = __half_as_ushort(__float2half_rn(c.x)), g = __half_as_ushort(__float2half_rn(c.y));
    const uint32_t b = __half_as_ushort(__float2half_rn(c.z)), a = __half_as_ushort(__float2half_rn(alpha));
    return make_uint2(r | (g << 16), b | (a << 16));
}

// rgb of an rgba16f texel as fp32
__device__ __forceinline__ f3 ssr_unpack_half(uint2 v) {
    return mk3(__half2float(__ushort_as_half((unsigned short)(v.x & 0xFFFFu))), __half2float(__ushort_as_half((unsigned short)(v.x >> 16))),
               __half2float(__ushort_as_half((unsigned short)(v.y & 0xFFFFu))));
}

struct SsrArgs {
    DeferredGBuffer g;             // depth, normalRG, albedo, metallicRoughness (emissive unused)
    const float4* src;             // the lit image, rgba32f [h][w]
    uint2* ssr;                    // rgba16f [h][w]
    float4* merged;                // rgba32f [h][w]: src.rgb + SSR, alpha 1
    DeviceScene sc;                // the sky (sample_sky)
    float projection[16], invProjection[16], invView[16];
    int sampleCount, binarySearchCount;
    float maxDist;
};

// texture(gBufferDataUBO.Depth, uv).r: NEAREST, clamp to edge
__device__ __forceinline__ float ssr_depth(const DeferredGBuffer& g, float u, float v) {
    return __ldg(g.depth + (size_t)nearest_texel(v, g.h) * g.w + nearest_texel(u, g.w));
}

// PerspectiveTransform(samplePoint, Projection) with xy mapped to [0, 1]
__device__ __forceinline__ f3 ssr_project(const float* m, f3 p) {
    const f3 q = deferred_perspective(m, p.x, p.y, p.z);
    return mk3(q.x * 0.5f + 0.5f, q.y * 0.5f + 0.5f, q.z);
}

// SSR(normal, fragPos) (SSR/compute.glsl:49-105) as written, view space
__device__ __forceinline__ f3 ssr_trace(const SsrArgs& a, const PostImage& src, f3 normal, f3 fragPos) {
    const f3 reflectDir = reflect3(normalize3(fragPos), normal);     // fragPos - VIEW_POS with VIEW_POS = 0
    const f3 maxReflectPoint = fragPos + reflectDir * a.maxDist;
    f3 deltaStep = (maxReflectPoint - fragPos) / (float)a.sampleCount;
    f3 samplePoint = fragPos;
    for (int i = 0; i < a.sampleCount; i++) {
        samplePoint = samplePoint + deltaStep;
        f3 projected = ssr_project(a.projection, samplePoint);
        if (projected.x >= 1.0f || projected.y >= 1.0f || projected.x < 0.0f || projected.y < 0.0f || projected.z > 1.0f)
            return mk3(0.0f, 0.0f, 0.0f);
        if (projected.z > ssr_depth(a.g, projected.x, projected.y)) {
            // BinarySearch: halve the step, back off by half of it, BinarySearchCount - 1 refinements; the colour is read at
            // the last projection made (the hit step's when there is none)
            deltaStep = deltaStep * 0.5f;
            samplePoint = samplePoint - deltaStep * 0.5f;
            for (int k = 1; k < a.binarySearchCount; k++) {
                projected = ssr_project(a.projection, samplePoint);
                const float depth = ssr_depth(a.g, projected.x, projected.y);
                deltaStep = deltaStep * 0.5f;
                if (projected.z > depth) samplePoint = samplePoint - deltaStep;
                else samplePoint = samplePoint + deltaStep;
            }
            return post_bilinear(src, projected.x, projected.y, 0, 0);
        }
    }
    const float* m = a.invView;                                      // (InvView * vec4(reflectDir, 0)).xyz
    const f3 r = reflectDir;
    const f3 world = mk3(((m[0] * r.x + m[4] * r.y) + m[8] * r.z) + m[12] * 0.0f, ((m[1] * r.x + m[5] * r.y) + m[9] * r.z) + m[13] * 0.0f,
                         ((m[2] * r.x + m[6] * r.y) + m[10] * r.z) + m[14] * 0.0f);
    return sample_sky(a.sc, world);
}

__global__ void __launch_bounds__(256) k_ssr(SsrArgs a) {
    int x, y;
    if (!deferred_pixel(a.g.w, a.g.h, x, y)) return;
    const size_t p = (size_t)y * a.g.w + x;
    const PostImage src = {a.src, nullptr, a.g.w, a.g.h};
    const float2 mr = a.g.metallicRoughness[p];
    const float specular = mr.x;
    const float depth = a.g.depth[p];
    uint2 packed;
    if (specular < 0.001f || depth == 1.0f) {
        packed = ssr_pack_half(mk3(0.0f, 0.0f, 0.0f), 0.0f);
    } else {
        const float u = ((float)x + 0.5f) / (float)a.g.w, v = ((float)y + 0.5f) / (float)a.g.h;
        const f3 fragPos = deferred_perspective(a.invProjection, u * 2.0f - 1.0f, v * 2.0f - 1.0f, depth);
        const float2 nrg = a.g.normalRG[p];
        const f3 n = decode_unit_vec(nrg.x, nrg.y);
        const float* m = a.invView;                                  // mat3(transpose(InvView)) * n, not renormalised
        const f3 normal = mk3((m[0] * n.x + m[1] * n.y) + m[2] * n.z, (m[4] * n.x + m[5] * n.y) + m[6] * n.z,
                              (m[8] * n.x + m[9] * n.y) + m[10] * n.z);
        f3 color = ssr_trace(a, src, normal, fragPos) * specular;
        color = color * mk3(a.g.albedo[3 * p], a.g.albedo[3 * p + 1], a.g.albedo[3 * p + 2]);
        packed = ssr_pack_half(color, 1.0f);
    }
    a.ssr[p] = packed;
    // Merge Textures: texelFetch(lit) + texelFetch(SSR) with the SSR value as its rgba16f texel holds it
    const float4 s = a.src[p];
    const f3 r = ssr_unpack_half(packed);
    a.merged[p] = make_float4(s.x + r.x, s.y + r.y, s.z + r.z, 1.0f);
}

struct TaaArgs {
    PostImage color;               // render-size lit image (rgba32f)
    const float* depth;            // render-size depth [rh][rw]
    const float2* velocity;        // render-size velocity [rh][rw]
    PostImage history;             // presentation-size rgba16f PrevResult
    uint2* out;                    // presentation-size rgba16f Result [H][W]
    int W, H;
    int isNaive, sampleCount;
    float preferAliasingOverBlur;
};

// min, max and clamp in one stated form (DESIGN.md 8f.1e): min(x, y) = y < x ? y : x, max(x, y) = y > x ? y : x,
// clamp(x, lo, hi) = min(max(x, lo), hi)
__device__ __forceinline__ float taa_min(float x, float y) { return y < x ? y : x; }
__device__ __forceinline__ float taa_max(float x, float y) { return y > x ? y : x; }
__device__ __forceinline__ f3 taa_min3(f3 x, f3 y) { return mk3(taa_min(x.x, y.x), taa_min(x.y, y.y), taa_min(x.z, y.z)); }
__device__ __forceinline__ f3 taa_max3(f3 x, f3 y) { return mk3(taa_max(x.x, y.x), taa_max(x.y, y.y), taa_max(x.z, y.z)); }

// texture(sampler, uv) with NEAREST filtering of a render-size image: the texel index
__device__ __forceinline__ size_t taa_nearest(const PostImage& t, float u, float v) {
    return (size_t)nearest_texel(v, t.h_) * t.w + nearest_texel(u, t.w);
}

// SampleTextureCatmullRom (TAAResolve/compute.glsl:105-154) as written: nine bilinear taps of the history
__device__ __forceinline__ f3 taa_catmull_rom(const PostImage& t, float u, float v) {
    const float tsx = 1.0f / (float)t.w, tsy = 1.0f / (float)t.h_;
    const float spx = u / tsx, spy = v / tsy;
    const float t1x = floorf(spx - 0.5f) + 0.5f, t1y = floorf(spy - 0.5f) + 0.5f;
    const float fx = spx - t1x, fy = spy - t1y;
    const float w0x = fx * (-0.5f + fx * (1.0f - 0.5f * fx)), w0y = fy * (-0.5f + fy * (1.0f - 0.5f * fy));
    const float w1x = 1.0f + (fx * fx) * (-2.5f + 1.5f * fx), w1y = 1.0f + (fy * fy) * (-2.5f + 1.5f * fy);
    const float w2x = fx * (0.5f + fx * (2.0f - 1.5f * fx)), w2y = fy * (0.5f + fy * (2.0f - 1.5f * fy));
    const float w3x = (fx * fx) * (-0.5f + 0.5f * fx), w3y = (fy * fy) * (-0.5f + 0.5f * fy);
    const float w12x = w1x + w2x, w12y = w1y + w2y;
    const float o12x = w2x / (w1x + w2x), o12y = w2y / (w1y + w2y);
    const float t0x = (t1x - 1.0f) * tsx, t0y = (t1y - 1.0f) * tsy;
    const float t3x = (t1x + 2.0f) * tsx, t3y = (t1y + 2.0f) * tsy;
    const float t12x = (t1x + o12x) * tsx, t12y = (t1y + o12y) * tsy;
    f3 r = (post_bilinear(t, t0x, t0y, 0, 0) * w0x) * w0y;
    r = r + (post_bilinear(t, t12x, t0y, 0, 0) * w12x) * w0y;
    r = r + (post_bilinear(t, t3x, t0y, 0, 0) * w3x) * w0y;
    r = r + (post_bilinear(t, t0x, t12y, 0, 0) * w0x) * w12y;
    r = r + (post_bilinear(t, t12x, t12y, 0, 0) * w12x) * w12y;
    r = r + (post_bilinear(t, t3x, t12y, 0, 0) * w3x) * w12y;
    r = r + (post_bilinear(t, t0x, t3y, 0, 0) * w0x) * w3y;
    r = r + (post_bilinear(t, t12x, t3y, 0, 0) * w12x) * w3y;
    r = r + (post_bilinear(t, t3x, t3y, 0, 0) * w3x) * w3y;
    return r;
}

// Alpha is 1 on every path, so only rgb is carried: the colour is read as rgb with alpha 1 (the engine's R11G11B10F), so the
// neighbourhood min and max alpha are 1 and the clamp pins the history's alpha to 1 (DESIGN.md 8f.1e).
__global__ void __launch_bounds__(256) k_taa_resolve(TaaArgs a) {
    int x, y;
    if (!deferred_pixel(a.W, a.H, x, y)) return;
    const size_t p = (size_t)y * a.W + x;
    const float fw = (float)a.W, fh = (float)a.H;
    const float u = ((float)x + 0.5f) / fw, v = ((float)y + 0.5f) / fh;
    const float blend0 = 1.0f / (float)a.sampleCount;
    if (a.isNaive) {
        const float2 vel = __ldg(a.velocity + taa_nearest(a.color, u, v));
        const float hu = u - vel.x, hv = v - vel.y;
        const f3 current = post_bilinear(a.color, u, v, 0, 0);
        const f3 history = post_bilinear(a.history, hu, hv, 0, 0);
        a.out[p] = ssr_pack_half(mix3(history, current, blend0), 1.0f);
        return;
    }
    // GetResolveData: the 3x3 neighbourhood's colour bounds, the centre tap and the uv of the closest depth
    float minDepth = IDK_FLOAT_MAX;
    f3 nMin = mk3(IDK_FLOAT_MAX, IDK_FLOAT_MAX, IDK_FLOAT_MAX), nMax = mk3(-IDK_FLOAT_MAX, -IDK_FLOAT_MAX, -IDK_FLOAT_MAX);
    f3 current = mk3(0.0f, 0.0f, 0.0f);
    float bu = u, bv = v;                                            // GLSL leaves it undefined if no depth is below FLOAT_MAX
    for (int dy = -1; dy <= 1; dy++) {
        for (int dx = -1; dx <= 1; dx++) {
            const float nu = ((float)(x + dx) + 0.5f) / fw, nv = ((float)(y + dy) + 0.5f) / fh;
            const f3 c = post_bilinear(a.color, nu, nv, 0, 0);
            nMin = taa_min3(nMin, c);
            nMax = taa_max3(nMax, c);
            const float d = __ldg(a.depth + taa_nearest(a.color, nu, nv));
            if (d < minDepth) { minDepth = d; bu = nu; bv = nv; }
            if (dx == 0 && dy == 0) current = c;
        }
    }
    const float2 vel = __ldg(a.velocity + taa_nearest(a.color, bu, bv));
    const float hu = u - vel.x, hv = v - vel.y;
    if (hu >= 1.0f || hv >= 1.0f || hu < 0.0f || hv < 0.0f) {
        a.out[p] = ssr_pack_half(current, 1.0f);
        return;
    }
    f3 history = taa_catmull_rom(a.history, hu, hv);
    history = taa_min3(taa_max3(history, nMin), nMax);
    const float lx = fract1(hu * (float)a.history.w), ly = fract1(hv * (float)a.history.h_);
    const float pixelCenterDistance = fabsf(0.5f - lx) + fabsf(0.5f - ly);
    const float blend = mix1(blend0, 1.0f, pixelCenterDistance * a.preferAliasingOverBlur);
    a.out[p] = ssr_pack_half(mix3(history, current, blend), 1.0f);
}
