// The raster mode's G-buffer pass for sm_90a (RasterPipeline.Render's "Fill G-Buffer" draws, RasterPipeline.cs:364-414, with
// GBuffer/VertexPath/vertex.glsl and GBuffer/fragment.glsl), ray-cast at pixel centres instead of rasterised: the fragment GL
// keeps at a pixel centre after the depth test is the closest surface along the ray through that centre that the pass does
// not clip, cull or discard, and perspective-correct interpolation at that sample gives the hit's barycentrics.
//
//   k_gbuffer   one thread per pixel, 8x8 pixel tiles (four per CTA), the shared-memory traversal stack of k_trace_rays:
//               one closest-hit ray per pixel centre through trace_ray<false, false, AcceptGBuffer>, lights off; the
//               fragment shader's outputs at the hit, stored as the engine's attachment formats hold them (kept as fp32)
//
// The rules are spelled out in DESIGN.md 8f.1g and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_deferred.cuh"

// GpuMeshTransform rows: [0..2] ModelMatrix, [3..5] InvModelMatrix, [6..8] PrevModelMatrix.
// GLSL column-major mat4 (16 floats) times vec4(p, 1).
__device__ __forceinline__ float4 gbuffer_clip(const float* m, f3 p) {
    return make_float4(((m[0] * p.x + m[4] * p.y) + m[8] * p.z) + m[12],
                       ((m[1] * p.x + m[5] * p.y) + m[9] * p.z) + m[13],
                       ((m[2] * p.x + m[6] * p.y) + m[10] * p.z) + m[14],
                       ((m[3] * p.x + m[7] * p.y) + m[11] * p.z) + m[15]);
}
__device__ __forceinline__ f3 gbuffer_position(const float* positions, int v) {
    return mk3(__ldg(positions + 3 * (size_t)v), __ldg(positions + 3 * (size_t)v + 1), __ldg(positions + 3 * (size_t)v + 2));
}
// Rule 3: clip = projView * (model * p) per vertex (unjittered), depth = (sum b_i clip_i.z) / (sum b_i clip_i.w).
__device__ __forceinline__ float gbuffer_depth(const float* projView, const float* positions, const float4* model, int4 tri,
                                               float b0, float b1, float b2) {
    const float4 r0 = ldg4(model), r1 = ldg4(model + 1), r2 = ldg4(model + 2);
    const float4 c0 = gbuffer_clip(projView, xform_point(r0, r1, r2, gbuffer_position(positions, tri.x)));
    const float4 c1 = gbuffer_clip(projView, xform_point(r0, r1, r2, gbuffer_position(positions, tri.y)));
    const float4 c2 = gbuffer_clip(projView, xform_point(r0, r1, r2, gbuffer_position(positions, tri.z)));
    return ((c0.z * b0 + c1.z * b1) + c2.z * b2) / ((c0.w * b0 + c1.w * b1) + c2.w * b2);
}
// Front-facing (CCW, lower-left window origin): det(ModelMatrix) * dot(n_local, d_local) < 0, decided from the signs so that
// no product underflows.
__device__ __forceinline__ bool gbuffer_front(float det, f3 n, f3 ld) {
    const float dn = dot3(n, ld);
    return (det > 0.0f && dn < 0.0f) || (det < 0.0f && dn > 0.0f);
}
__device__ __forceinline__ float gbuffer_det(const float4* model) {
    const float4 m0 = ldg4(model), m1 = ldg4(model + 1), m2 = ldg4(model + 2);
    return (m0.x * (m1.y * m2.z - m1.z * m2.y) - m0.y * (m1.x * m2.z - m1.z * m2.x)) + m0.z * (m1.x * m2.y - m1.y * m2.x);
}

// The surface's alpha at barycentrics (b0, b1, b2), sampled as surface_textured samples it.
__device__ __forceinline__ float gbuffer_alpha(const DeviceScene& sc, const GpuMaterial& mat, int4 tri, float b0, float b1, float b2) {
    const float4 s0 = ldg4(sc.surfRec + 5 * (size_t)tri.w), s4 = ldg4(sc.surfRec + 5 * (size_t)tri.w + 4);
    float alpha = s0.w;
    if (__float_as_uint(s4.x) & 4u) {
        float u, v;
        interp_texcoord(sc, tri, b0, b1, b2, u, v);
        alpha = tex_sample(sc, mat.BaseColorTexture, u, v).w * ((float)((mat.BaseColorFactor >> 24) & 255u) / 255.0f);
    }
    return alpha;
}

// One instance's depth-test rules (rule 2): a triangle that beats the current t takes the hit unless it is clipped (depth
// outside [0, 1]), blended (AlphaCutoff == 2: culled from the pass), back-facing on a single-sided material (CullFace), or
// alpha-discarded (Alpha < AlphaCutoff, the base-colour alpha sampled as surface_textured does).
struct AcceptGBufferInstance {
    const float* projView;
    const float* positions;
    const float4* model;
    float det;
    f3 ld;
    __device__ __forceinline__ bool operator()(const DeviceScene& sc, uint32_t i, float bx, float by, float) const {
        const int4 tri = __ldg(sc.blasTris + i);
        const GpuMaterial& mat = sc.materials[sc.meshes[tri.w].MaterialId];
        const float alphaCutoff = mat.AlphaCutoff;
        if (alphaCutoff == 2.0f) return false;
        if (!mat.IsDoubleSided) {
            const float4 nr = ldg4(sc.triRec + 4 * (size_t)i + 2);
            if (!gbuffer_front(det, mk3(nr.y, nr.z, nr.w), ld)) return false;
        }
        const float b2 = 1.0f - bx - by;
        const float depth = gbuffer_depth(projView, positions, model, tri, bx, by, b2);
        if (!(depth >= 0.0f && depth <= 1.0f)) return false;
        return !(gbuffer_alpha(sc, mat, tri, bx, by, b2) < alphaCutoff);
    }
};
struct AcceptGBuffer {
    const float* projView;
    const float* positions;
    __device__ __forceinline__ AcceptGBufferInstance at(const DeviceScene& sc, uint32_t xf, f3 ld) const {
        const float4* model = sc.xforms + 9 * (size_t)xf;
        return AcceptGBufferInstance{projView, positions, model, gbuffer_det(model), ld};
    }
};

// Rule 4 at barycentrics (b0, b1, b2) of BLAS triangle triIndex (= tri) in transform mt, seen along world direction d: the
// surface (the per-mesh record, or the textures at level 0) into s, and the world normal: per-vertex world normal and tangent,
// interpolated, then GetTBN, the normal map mixed in by NormalMapStrength, negated on a back face.
__device__ __forceinline__ f3 gbuffer_surface(const DeviceScene& sc, uint32_t triIndex, int4 tri, const float4* mt, float b0, float b1,
                                              float b2, f3 d, Surface& s) {
    const float4 i0 = ldg4(mt + 3), i1 = ldg4(mt + 4), i2 = ldg4(mt + 5);
    const float4* vf = sc.vtxFrame;
    const float4 a0 = ldg4(vf + 2 * (size_t)tri.x), a1 = ldg4(vf + 2 * (size_t)tri.x + 1);
    const float4 c0 = ldg4(vf + 2 * (size_t)tri.y), c1 = ldg4(vf + 2 * (size_t)tri.y + 1);
    const float4 e0 = ldg4(vf + 2 * (size_t)tri.z), e1 = ldg4(vf + 2 * (size_t)tri.z + 1);
    const f3 wn0 = normalize3(xform_normal(i0, i1, i2, mk3(a0.x, a0.y, a0.z)));
    const f3 wn1 = normalize3(xform_normal(i0, i1, i2, mk3(c0.x, c0.y, c0.z)));
    const f3 wn2 = normalize3(xform_normal(i0, i1, i2, mk3(e0.x, e0.y, e0.z)));
    const f3 wt0 = normalize3(xform_normal(i0, i1, i2, mk3(a0.w, a1.x, a1.y)));
    const f3 wt1 = normalize3(xform_normal(i0, i1, i2, mk3(c0.w, c1.x, c1.y)));
    const f3 wt2 = normalize3(xform_normal(i0, i1, i2, mk3(e0.w, e1.x, e1.y)));
    const f3 interpNormal = normalize3((wn0 * b0 + wn1 * b1) + wn2 * b2);
    const f3 interpTangent = normalize3((wt0 * b0 + wt1 * b1) + wt2 * b2);

    const float4* sr = sc.surfRec + 5 * (size_t)tri.w;
    const float4 s0 = ldg4(sr), s1 = ldg4(sr + 1), s2 = ldg4(sr + 2), s3 = ldg4(sr + 3), s4 = ldg4(sr + 4);
    s.Albedo = mk3(s0.x, s0.y, s0.z); s.Alpha = s0.w;
    s.Normal = mk3(1.0f, 1.0f, 0.0f);
    s.Emissive = mk3(s1.x, s1.y, s1.z); s.Metallic = s1.w;
    s.Absorbance = mk3(s2.x, s2.y, s2.z); s.Roughness = s2.w;
    s.Transmission = s3.x; s.IOR = s3.y; s.AlphaCutoff = s3.z;
    s.IsVolumetric = false; s.TintOnTransmissive = false;
    if (__float_as_uint(s4.x) & 4u) {
        float tu, tv;
        interp_texcoord(sc, tri, b0, b1, b2, tu, tv);
        surface_textured(sc, tri.w, tu, tv, s);
    }
    const f3 N = normalize3(interpNormal);
    const f3 Tn = normalize3(interpTangent);
    const f3 B = normalize3(cross3(N, Tn));
    const f3 tbnN = (Tn * s.Normal.x + B * s.Normal.y) + N * s.Normal.z;
    f3 normal = normalize3(mix3(interpNormal, tbnN, s3.w));
    const float4 nr = ldg4(sc.triRec + 4 * (size_t)triIndex + 2);
    if (!gbuffer_front(gbuffer_det(mt), mk3(nr.y, nr.z, nr.w), xform_vector(i0, i1, i2, d))) normal = normal * -1.0f;
    return normal;
}

// Unsigned 11- / 10-bit float (R11G11B10F, GL core spec 2.3.4.3) with `mbits` mantissa bits, as fp32: nearest, ties to even,
// denormals below 2^-14; negative values, -0 and -inf store 0; finite values above the largest finite value (`maxv`: 65024
// with 6 bits, 64512 with 5) store it; +inf stays +inf and NaN stays NaN.
__device__ __forceinline__ float gbuffer_ufloat(float v, int mbits, float maxv) {
    if (v != v) return v;
    if (!(v > 0.0f)) return 0.0f;
    if (v == __int_as_float(0x7f800000)) return v;
    const int e = max((int)((__float_as_uint(v) >> 23) & 255u) - 127, -14);
    const float q = __uint_as_float((uint32_t)(e - mbits + 127) << 23);
    return fminf(rintf(v / q) * q, maxv);
}
__device__ __forceinline__ float gbuffer_unorm8(float v) { return (float)deferred_r8(v) / 255.0f; }
__device__ __forceinline__ float gbuffer_half(float v) { return __half2float(__float2half_rn(v)); }

struct GBufferArgs {
    DeviceScene sc;
    const float* positions;        // PackedVec3 per vertex: this frame's
    const float* prevPositions;    // and the previous frame's (prevVertexPositionSSBO)
    float projView[16], prevProjView[16], invProjView[16];
    float viewPos[3];
    float jitter[2];
    int w, h;
    float* depth;                  // planar [h][w] outputs
    float2* normalRG;
    float* albedo;                 // 3 floats per pixel
    float2* metallicRoughness;
    float* emissive;               // 3 floats per pixel
    float2* velocity;
};

__global__ void __launch_bounds__(IDK_BLOCK) k_gbuffer(GBufferArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    int x, y;
    if (!deferred_pixel(a.w, a.h, x, y)) return;
    const DeviceScene& sc = a.sc;
    // rule 1: the unjittered point the jittered geometry puts at the pixel centre, through InvProjView at the far plane
    const float ndcX = ((float)x + 0.5f) / (float)a.w * 2.0f - 1.0f - a.jitter[0];
    const float ndcY = ((float)y + 0.5f) / (float)a.h * 2.0f - 1.0f - a.jitter[1];
    const f3 o = mk3(a.viewPos[0], a.viewPos[1], a.viewPos[2]);
    const f3 d = normalize3(deferred_perspective(a.invProjView, ndcX, ndcY, 1.0f) - o);
    HitRec hit;
    uint32_t xf, S = 0, T = 0, I = 0;
    float cost = 0.0f;
    trace_ray<false, false>(sc, o, d, IDK_FLOAT_MAX, false, stack, hit, xf, S, T, I, cost, AcceptGBuffer{a.projView, a.positions});

    float depth = 1.0f, nx = 0.0f, ny = 0.0f, metallic = 0.0f, roughness = 0.0f, vx = 0.0f, vy = 0.0f;
    f3 albedo = mk3(0.0f, 0.0f, 0.0f), emissive = mk3(0.0f, 0.0f, 0.0f);
    if (hit.tri != ~0u) {
        const int4 tri = __ldg(sc.blasTris + hit.tri);
        const float4* mt = sc.xforms + 9 * (size_t)xf;
        const float b0 = hit.bx, b1 = hit.by, b2 = 1.0f - hit.bx - hit.by;
        depth = gbuffer_depth(a.projView, a.positions, mt, tri, b0, b1, b2);

        Surface s;
        const f3 normal = gbuffer_surface(sc, hit.tri, tri, mt, b0, b1, b2, d, s);

        // rule 5: the previous frame's clip position, interpolated
        const float4 p0 = ldg4(mt + 6), p1 = ldg4(mt + 7), p2 = ldg4(mt + 8);
        const float4 q0 = gbuffer_clip(a.prevProjView, xform_point(p0, p1, p2, gbuffer_position(a.prevPositions, tri.x)));
        const float4 q1 = gbuffer_clip(a.prevProjView, xform_point(p0, p1, p2, gbuffer_position(a.prevPositions, tri.y)));
        const float4 q2 = gbuffer_clip(a.prevProjView, xform_point(p0, p1, p2, gbuffer_position(a.prevPositions, tri.z)));
        const float pcx = (q0.x * b0 + q1.x * b1) + q2.x * b2;
        const float pcy = (q0.y * b0 + q1.y * b1) + q2.y * b2;
        const float pcw = (q0.w * b0 + q1.w * b1) + q2.w * b2;

        // rule 6: what the attachments hold
        float ex, ey;
        encode_unit_vec(normal, ex, ey);
        nx = gbuffer_unorm8(ex); ny = gbuffer_unorm8(ey);
        albedo = mk3(gbuffer_ufloat(s.Albedo.x, 6, 65024.0f), gbuffer_ufloat(s.Albedo.y, 6, 65024.0f), gbuffer_ufloat(s.Albedo.z, 5, 64512.0f));
        emissive = mk3(gbuffer_ufloat(s.Emissive.x, 6, 65024.0f), gbuffer_ufloat(s.Emissive.y, 6, 65024.0f), gbuffer_ufloat(s.Emissive.z, 5, 64512.0f));
        metallic = gbuffer_unorm8(s.Metallic); roughness = gbuffer_unorm8(s.Roughness);
        vx = gbuffer_half((ndcX - pcx / pcw) * 0.5f);
        vy = gbuffer_half((ndcY - pcy / pcw) * 0.5f);
    }
    const size_t p = (size_t)y * a.w + x;
    a.depth[p] = depth;
    a.normalRG[p] = make_float2(nx, ny);
    a.albedo[3 * p] = albedo.x; a.albedo[3 * p + 1] = albedo.y; a.albedo[3 * p + 2] = albedo.z;
    a.metallicRoughness[p] = make_float2(metallic, roughness);
    a.emissive[3 * p] = emissive.x; a.emissive[3 * p + 1] = emissive.y; a.emissive[3 * p + 2] = emissive.z;
    a.velocity[p] = make_float2(vx, vy);
}
