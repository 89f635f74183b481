// The raster mode's light spheres and skybox for sm_90a: RasterPipeline.Render's "Draw lights" and "Draw skybox" draws
// (RasterPipeline.cs:465-516, LightManager.Draw, Light/vertex.glsl + fragment.glsl, SkyBox/vertex.glsl + fragment.glsl), fused
// and ray-cast at pixel centres like the G-buffer pass. They run after deferred lighting and before transparency, and write the
// context's G-buffer images and deferred image in place.
//
//   k_lights_skybox   one thread per pixel, 8x8 pixel tiles (four per CTA), the scene's lights staged in shared memory per CTA:
//                     the ray of k_gbuffer against every triangle of every light's tessellated unit sphere (the mesh in
//                     constant memory), with the light draw's depth test (LESS, back faces culled) against the G-buffer depth;
//                     the winning fragment's colour, normal, emissive, velocity and depth; then the skybox (LEQUAL against the
//                     window depth 1) where the depth is still 1: the cube-map colour and the rotation-only velocity
//   k_lights_skybox_vrs the same draws under the shading-rate image (VariableRateShadingNV on both draws): the same kernel
//                     body (lights_skybox_pixel<true>), with coverage and depth per pixel and the fragment shaders' values at
//                     the centre of the pixel's coarse fragment
//
// The rules are spelled out in DESIGN.md 8f.1i and restated independently by the CPU oracle; the two agree bit for bit.
#pragma once
#include "idk_gbuffer.cuh"
#include "idk_vrs.cuh"

// LightManager's sphere: GeometricPrimitives.Sphere with 12 latitudes and 12 longitudes at radius 1.
#define IDK_SPHERE_SEGMENTS 12
#define IDK_SPHERE_VERTICES ((IDK_SPHERE_SEGMENTS + 1) * (IDK_SPHERE_SEGMENTS + 1))          // 169
#define IDK_SPHERE_TRIANGLES (2 * IDK_SPHERE_SEGMENTS * (IDK_SPHERE_SEGMENTS - 1))           // 264: one per pole cell

// The vertex table and the index buffer (three 8-bit vertex indices per triangle, the first in the low byte), written at context
// creation by sphere_mesh_tables. Every lane of a warp reads the same entry, so each read is a constant-cache broadcast.
__constant__ float3 c_sphere_vertices[IDK_SPHERE_VERTICES];
__constant__ uint32_t c_sphere_triangles[IDK_SPHERE_TRIANGLES];

// GenerateVertices / GenerateIndices (GeometricPrimitives.cs:16-83) in their statement order, fp32, with cos and sin taken as
// (float)cos((double)angle): what a correctly rounded cosf returns, independent of the host's libm.
static inline void sphere_mesh_tables(float3 vertices[IDK_SPHERE_VERTICES], uint32_t triangles[IDK_SPHERE_TRIANGLES]) {
    const int n = IDK_SPHERE_SEGMENTS;
    const float pi = 3.14159265358979323846f;
    const float deltaLatitude = pi / (float)n;
    const float deltaLongitude = 2.0f * pi / (float)n;
    int v = 0;
    for (int i = 0; i <= n; i++) {
        const float latitudeAngle = pi / 2.0f - (float)i * deltaLatitude;
        const float xy = 1.0f * (float)std::cos((double)latitudeAngle);
        const float z = 1.0f * (float)std::sin((double)latitudeAngle);
        for (int j = 0; j <= n; j++) {
            const float longitudeAngle = (float)j * deltaLongitude;
            vertices[v++] = make_float3(xy * (float)std::cos((double)longitudeAngle), xy * (float)std::sin((double)longitudeAngle), z);
        }
    }
    int t = 0;
    for (uint32_t i = 0; i < (uint32_t)n; i++) {
        uint32_t k1 = i * (uint32_t)(n + 1), k2 = k1 + (uint32_t)n + 1;
        for (int j = 0; j < n; j++, k1++, k2++) {
            if (i != 0) triangles[t++] = k1 | (k2 << 8) | ((k1 + 1) << 16);
            if (i != (uint32_t)n - 1) triangles[t++] = (k1 + 1) | (k2 << 8) | ((k2 + 1) << 16);
        }
    }
}

// Rule 3: world vertex Radius * p + Position of the unit-sphere vertex k.
__device__ __forceinline__ f3 light_vertex(float radius, f3 position, uint32_t k) {
    const float3 p = c_sphere_vertices[k];
    return mk3(radius * p.x + position.x, radius * p.y + position.y, radius * p.z + position.z);
}

// A light the ray certainly misses: its world vertices lie within |Radius| (1 + a few ulp) plus the rounding of
// Radius * p + Position of Position, and the triangle test accepts nothing farther from its triangle than a few ulp of the
// distances involved. The bound below is 1e-3 of the radius and 1e-4 of those distances wider, so it never rejects a ray that
// the triangle test accepts (no pixel changes), and rejects every ray that passes outside it or has the sphere behind it.
__device__ __forceinline__ bool light_missed(f3 o, f3 d, f3 position, float radius) {
    const f3 s = position - o;
    const f3 c = cross3(s, d);
    const float r = fabsf(radius) * 1.001f + (sqrtf(dot3(s, s)) + (fabsf(position.x) + fabsf(position.y)) + fabsf(position.z)) * 1e-4f;
    return dot3(c, c) > r * r || dot3(s, d) < -r;
}

struct LightsSkyboxArgs {
    DeviceScene sc;                // the sky (sample_sky)
    const GpuLight* lights;
    int lightCount;                // <= IDK_GPU_MAX_UBO_LIGHT_COUNT
    float projView[16], prevProjView[16], invProjView[16];
    float projection[16], invProjection[16], invView[16], prevView[16];
    float viewPos[3];
    float jitter[2];
    int w, h;
    float* depth;                  // the G-buffer planes [h][w], written in place
    float2* normalRG;
    float* emissive;               // 3 floats per pixel
    float2* velocity;
    float4* color;                 // the deferred image [h][w], written in place
};

// Rule 5's direction at NDC (sx, sy): (InvView * vec4(PerspectiveTransform((s, 1), InvProjection), 0)).xyz, as k_ssr's miss
// direction.
__device__ __forceinline__ f3 sky_direction(const LightsSkyboxArgs& a, float sx, float sy) {
    const f3 v = deferred_perspective(a.invProjection, sx, sy, 1.0f);
    const float* m = a.invView;
    return mk3(((m[0] * v.x + m[4] * v.y) + m[8] * v.z) + m[12] * 0.0f, ((m[1] * v.x + m[5] * v.y) + m[9] * v.z) + m[13] * 0.0f,
               ((m[2] * v.x + m[6] * v.y) + m[10] * v.z) + m[14] * 0.0f);
}

// One pixel of the two draws. kVrs: the draws under the rate image `rates` ([ceil(h/16)][ceil(w/16)] palette indices, 8f.1i's
// VRS paragraph): coverage, the depth test and the written depth stay the pixel's own; what the fragment shaders compute
// (FragPos, the normal, the velocity, the sky's TexCoord) is evaluated at the centre of the pixel's coarse fragment.
template <bool kVrs>
__device__ __forceinline__ void lights_skybox_pixel(const LightsSkyboxArgs& a, const GpuLight* s_lights, const uint8_t* rates) {
    int x, y;
    if (!deferred_pixel(a.w, a.h, x, y)) return;
    const size_t p = (size_t)y * a.w + x;
    float depth = a.depth[p];
    // rule 2: the ray of k_gbuffer
    const float ndcX = ((float)x + 0.5f) / (float)a.w * 2.0f - 1.0f - a.jitter[0];
    const float ndcY = ((float)y + 0.5f) / (float)a.h * 2.0f - 1.0f - a.jitter[1];
    const f3 o = mk3(a.viewPos[0], a.viewPos[1], a.viewPos[2]);
    const f3 d = normalize3(deferred_perspective(a.invProjView, ndcX, ndcY, 1.0f) - o);

    // rule 3: every triangle of every light in draw order; a front-facing, unclipped fragment below the current depth wins
    int best = -1, bestTri = 0;
    float b0 = 0.0f, b1 = 0.0f;
    for (int l = 0; l < a.lightCount; l++) {
        const GpuLight& light = s_lights[l];
        const f3 position = mk3(light.Position[0], light.Position[1], light.Position[2]);
        const float radius = light.Radius;
        if (light_missed(o, d, position, radius)) continue;
#pragma unroll 1
        for (int t = 0; t < IDK_SPHERE_TRIANGLES; t++) {
            const uint32_t k = c_sphere_triangles[t];
            const f3 w0 = light_vertex(radius, position, k & 255u);
            const f3 w1 = light_vertex(radius, position, (k >> 8) & 255u);
            const f3 w2 = light_vertex(radius, position, k >> 16);
            const f3 e1 = w1 - w0, e2 = w2 - w0, n = cross3(e1, e2);
            float bx, by, tHit;
            if (!ray_triangle(o, d, w0, e1, e2, n, bx, by, tHit)) continue;
            // front-facing: det(Model) = Radius^3 and d_local = d / Radius share their sign, so 8f.1g's rule is dot(n, d) < 0
            if (!gbuffer_front(1.0f, n, d)) continue;
            const float4 c0 = gbuffer_clip(a.projView, w0), c1 = gbuffer_clip(a.projView, w1), c2 = gbuffer_clip(a.projView, w2);
            const float bz = 1.0f - bx - by;
            const float fragDepth = ((c0.z * bx + c1.z * by) + c2.z * bz) / ((c0.w * bx + c1.w * by) + c2.w * bz);
            if (!(fragDepth >= 0.0f && fragDepth <= 1.0f && fragDepth < depth)) continue;
            depth = fragDepth; best = l; bestTri = t; b0 = bx; b1 = by;
        }
    }

    // VRS: the pixel's coarse fragment, cw x ch at (x - x mod cw, y - y mod ch) inside its 16x16 tile, and its centre in pixels
    float xc = 0.0f, yc = 0.0f;
    if constexpr (kVrs) {
        int cw, ch;
        vrs_fragment_size(rates[(size_t)(y / IDK_VRS_TILE) * ((a.w + IDK_VRS_TILE - 1) / IDK_VRS_TILE) + x / IDK_VRS_TILE], cw, ch);
        xc = (float)(x - x % cw) + 0.5f * (float)cw;
        yc = (float)(y - y % ch) + 0.5f * (float)ch;
    }

    if (best >= 0) {
        // rule 4: the light fragment's outputs
        const GpuLight& light = s_lights[best];
        const f3 position = mk3(light.Position[0], light.Position[1], light.Position[2]);
        const f3 prevPosition = mk3(light.PrevPosition[0], light.PrevPosition[1], light.PrevPosition[2]);
        const float radius = light.Radius;
        const uint32_t k = c_sphere_triangles[bestTri];
        const uint32_t i0 = k & 255u, i1 = (k >> 8) & 255u, i2 = k >> 16;
        float thisX = ndcX, thisY = ndcY;
        if constexpr (kVrs) {
            // the centre's ray against the winning triangle's plane: ray_triangle's arithmetic, its inside and t tests ignored
            thisX = xc / (float)a.w * 2.0f - 1.0f - a.jitter[0];
            thisY = yc / (float)a.h * 2.0f - 1.0f - a.jitter[1];
            const f3 dc = normalize3(deferred_perspective(a.invProjView, thisX, thisY, 1.0f) - o);
            const f3 w0 = light_vertex(radius, position, i0), w1 = light_vertex(radius, position, i1), w2 = light_vertex(radius, position, i2);
            const f3 e1 = w1 - w0, e2 = w2 - w0;
            float tHit;
            (void)ray_triangle(o, dc, w0, e1, e2, cross3(e1, e2), b0, b1, tHit);
        }
        const float b2 = 1.0f - b0 - b1;
        const f3 fragPos = (light_vertex(radius, position, i0) * b0 + light_vertex(radius, position, i1) * b1) + light_vertex(radius, position, i2) * b2;
        float ex, ey;
        encode_unit_vec((fragPos - position) / radius, ex, ey);
        const float4 q0 = gbuffer_clip(a.prevProjView, light_vertex(radius, prevPosition, i0));
        const float4 q1 = gbuffer_clip(a.prevProjView, light_vertex(radius, prevPosition, i1));
        const float4 q2 = gbuffer_clip(a.prevProjView, light_vertex(radius, prevPosition, i2));
        const float pcx = (q0.x * b0 + q1.x * b1) + q2.x * b2;
        const float pcy = (q0.y * b0 + q1.y * b1) + q2.y * b2;
        const float pcw = (q0.w * b0 + q1.w * b1) + q2.w * b2;
        a.depth[p] = depth;
        a.normalRG[p] = make_float2(gbuffer_unorm8(ex), gbuffer_unorm8(ey));
        a.emissive[3 * p] = gbuffer_ufloat(light.Color[0], 6, 65024.0f);
        a.emissive[3 * p + 1] = gbuffer_ufloat(light.Color[1], 6, 65024.0f);
        a.emissive[3 * p + 2] = gbuffer_ufloat(light.Color[2], 5, 64512.0f);
        a.velocity[p] = make_float2(gbuffer_half((thisX - pcx / pcw) * 0.5f), gbuffer_half((thisY - pcy / pcw) * 0.5f));
        a.color[p] = make_float4(light.Color[0], light.Color[1], light.Color[2], 1.0f);
    } else if (1.0f <= depth) {
        // rule 5: the skybox at the unjittered pixel centre, on the cube around the camera
        float sx = ((float)x + 0.5f) / (float)a.w * 2.0f - 1.0f, sy = ((float)y + 0.5f) / (float)a.h * 2.0f - 1.0f;
        const f3 dir = sky_direction(a, sx, sy);
        f3 c;
        if constexpr (kVrs) {
            // TexCoord on the pixel's own cube face (the axis of its largest |dir|, x before y before z), at the fragment centre
            const float ax = fabsf(dir.x), ay = fabsf(dir.y), az = fabsf(dir.z);
            const int axis = ax >= ay && ax >= az ? 0 : ay >= az ? 1 : 2;
            sx = xc / (float)a.w * 2.0f - 1.0f;
            sy = yc / (float)a.h * 2.0f - 1.0f;
            const f3 dc = sky_direction(a, sx, sy);
            c = dc * (0.5f / fabsf(axis == 0 ? dc.x : axis == 1 ? dc.y : dc.z));
        } else {
            c = dir * (0.5f / fmaxf(fmaxf(fabsf(dir.x), fabsf(dir.y)), fabsf(dir.z)));
        }
        const f3 sky = sample_sky(a.sc, c);
        const float* pv = a.prevView;                                // mat3(PrevView) * c, then Projection * (., 1)
        const f3 pc = mk3((pv[0] * c.x + pv[4] * c.y) + pv[8] * c.z, (pv[1] * c.x + pv[5] * c.y) + pv[9] * c.z, (pv[2] * c.x + pv[6] * c.y) + pv[10] * c.z);
        const float4 q = gbuffer_clip(a.projection, pc);
        a.velocity[p] = make_float2(gbuffer_half((sx - q.x / q.w) * 0.5f), gbuffer_half((sy - q.y / q.w) * 0.5f));
        a.color[p] = make_float4(sky.x, sky.y, sky.z, 1.0f);
    }
}

__global__ void __launch_bounds__(256) k_lights_skybox(LightsSkyboxArgs a) {
    __shared__ GpuLight s_lights[IDK_GPU_MAX_UBO_LIGHT_COUNT];
    for (int i = threadIdx.x; i < a.lightCount; i += blockDim.x) s_lights[i] = a.lights[i];
    __syncthreads();
    lights_skybox_pixel<false>(a, s_lights, nullptr);
}

// The same draws under the context's rate image: one thread per pixel as k_lights_skybox, each reading its tile's rate byte.
// Coverage is per pixel, so there is no fragment list (k_vrs_scan) to build.
__global__ void __launch_bounds__(256) k_lights_skybox_vrs(LightsSkyboxArgs a, const uint8_t* __restrict__ rates) {
    __shared__ GpuLight s_lights[IDK_GPU_MAX_UBO_LIGHT_COUNT];
    for (int i = threadIdx.x; i < a.lightCount; i += blockDim.x) s_lights[i] = a.lights[i];
    __syncthreads();
    lights_skybox_pixel<true>(a, s_lights, rates);
}
