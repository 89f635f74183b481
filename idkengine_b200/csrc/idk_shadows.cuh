// "Next" rows of the scope table (SURVEY.md 8f.1): any-hit traversal and the ray-traced point-light shadow pass, both on
// top of the path tracer's serial walk (trace_ray, idk_kernels.cuh).
//   k_trace_rays_any        TraceRayAny / IntersectBlasAny, include/BVHIntersect.glsl:107-181,299-411: trace_ray<false, true>
//   k_shadows_ray_traced    ShadowsRayTraced/compute.glsl (PointShadowManager.ComputeRayTracedShadowMaps, PointShadowManager.cs:53-75)
#pragma once
#include "idk_kernels.cuh"

__global__ void __launch_bounds__(IDK_BLOCK) k_trace_rays_any(TraceRaysArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(a.ticket, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= a.count) break;
        const uint32_t gid = base + lane;
        if (gid < a.count) {
            const float4 r0 = a.rays[2 * (size_t)gid], r1 = a.rays[2 * (size_t)gid + 1];
            uint32_t S = 0, T = 0, I = 0;
            float cost = 0.0f;
            HitRec hit;
            uint32_t xf;
            const bool any = trace_ray<false, true>(a.sc, mk3(r0.x, r0.y, r0.z), mk3(r1.x, r1.y, r1.z), r0.w, a.traceLights != 0, stack, hit, xf, S, T, I, cost);
            a.hits[2 * (size_t)gid] = make_uint4(__float_as_uint(hit.bx), __float_as_uint(hit.by), __float_as_uint(hit.t), hit.tri);
            a.hits[2 * (size_t)gid + 1] = make_uint4(xf, any ? 1u : 0u, 0u, 0u);
        }
    }
}

// Sampling.glsl:35-57 SampleSphere(toSphere, radius, rnd0, rnd1, ...) with SampleCone / ConstructBasis (Math.glsl:104-117)
__device__ __forceinline__ f3 sample_sphere_light(f3 toSphere, float sphereRadius, float rnd0, float rnd1, float& distanceToSphere) {
    const float radiusSq = sphereRadius * sphereRadius;
    const float distanceSq = dot3(toSphere, toSphere);
    const float sinThetaMaxSq = radiusSq / distanceSq;
    const float cosThetaMax = sqrtf(fmaxf(1.0f - sinThetaMaxSq, 0.0f));
    const float phiMax = 2.0f * IDK_PI;
    const float phi = phiMax * rnd0;
    const float cosTheta = mix1(cosThetaMax, 1.0f, fmaxf(rnd1, 0.001f));
    const float sinTheta = sqrtf(fmaxf(1.0f - cosTheta * cosTheta, 0.0f));
    distanceToSphere = sqrtf(dot3(toSphere, toSphere)) * cosTheta - sqrtf(radiusSq - distanceSq * sinTheta * sinTheta);
    const f3 normal = normalize3(toSphere);
    float sinPhi, cosPhi;
    det_sincos(phi, &sinPhi, &cosPhi);
    const f3 local = mk3(cosPhi * sinTheta, cosTheta, sinPhi * sinTheta);
    const f3 up = fabsf(normal.z) < 0.999f ? mk3(0.0f, 0.0f, 1.0f) : mk3(1.0f, 0.0f, 0.0f);
    const f3 tangent = normalize3(cross3(up, normal));
    const f3 bitangent = cross3(normal, tangent);
    return (tangent * local.x + normal * local.y) + bitangent * local.z;
}

__device__ __forceinline__ float ign_noise(float x, float y, uint32_t index) {
    x += (float)index * 5.588238f;
    y += (float)index * 5.588238f;
    return fract1(52.9829189f * fract1(0.06711056f * x + 0.00583715f * y));
}

struct ShadowArgs {
    DeviceScene sc;
    float invProjView[16];
    float jitter[2];
    const float* depth;
    const float2* normalRG;
    float* visibility;
    int width, height, lightIndex, samples;
    uint32_t noiseIndex;
};

__global__ void __launch_bounds__(IDK_BLOCK) k_shadows_ray_traced(ShadowArgs a) {
    extern __shared__ uint32_t s_stack[];
    uint32_t* stack = s_stack + threadIdx.x;
    const DeviceScene& sc = a.sc;
    const size_t n = (size_t)a.width * a.height;
    for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(p % a.width), y = (int)(p / a.width);
        const float d = a.depth[p];
        if (d == 1.0f) continue;
        const GpuLight& L = sc.lights[a.lightIndex];
        const f3 lightPos = mk3(L.Position[0], L.Position[1], L.Position[2]);
        const float u = ((float)x + 0.5f) / (float)a.width, v = ((float)y + 0.5f) / (float)a.height;
        const float nx = (u * 2.0f - 1.0f) - a.jitter[0], ny = (v * 2.0f - 1.0f) - a.jitter[1];
        const float* m = a.invProjView;
        const float wx = ((m[0] * nx + m[4] * ny) + m[8] * d) + m[12] * 1.0f;
        const float wy = ((m[1] * nx + m[5] * ny) + m[9] * d) + m[13] * 1.0f;
        const float wz = ((m[2] * nx + m[6] * ny) + m[10] * d) + m[14] * 1.0f;
        const float ww = ((m[3] * nx + m[7] * ny) + m[11] * d) + m[15] * 1.0f;
        const f3 fragPos = mk3(wx / ww, wy / ww, wz / ww);
        const float2 nrg = a.normalRG[p];
        const f3 normal = decode_unit_vec(nrg.x, nrg.y);
        const float cosTheta = dot3(normal, normalize3(lightPos - fragPos));
        if (cosTheta <= 0.0f) { a.visibility[p] = 0.0f; continue; }
        float visibility = 0.0f;
        uint32_t noiseIndex = a.noiseIndex;
        for (int i = 0; i < a.samples; i++) {
            const f3 biasedPosition = fragPos + normal * 0.01f;
            const float rnd0 = ign_noise((float)x, (float)y, noiseIndex + 0);
            const float rnd1 = ign_noise((float)x, (float)y, noiseIndex + 1);
            noiseIndex++;
            float distanceToLight;
            const f3 direction = sample_sphere_light(lightPos - biasedPosition, L.Radius, rnd0, rnd1, distanceToLight);
            f3 origin = biasedPosition;
            float thisVisibility = 1.0f;
            for (;;) {
                HitRec hit;
                uint32_t xf, S = 0, T = 0, I = 0;
                float cost = 0.0f;
                const float maxDist = distanceToLight - 0.001f;
                trace_ray<false, false>(sc, origin, direction, maxDist, true, stack, hit, xf, S, T, I, cost);
                if (!(hit.t != maxDist)) break;
                if (hit.tri == ~0u) {
                    if (xf != (uint32_t)a.lightIndex) thisVisibility = 0.0f;
                    break;
                }
                const int4 tri = __ldg(sc.blasTris + hit.tri);
                const float4* sr = sc.surfRec + 5 * (size_t)tri.w;
                float alpha = ldg4(sr).w;
                const float alphaCutoff = ldg4(sr + 3).z;
                if (__float_as_uint(ldg4(sr + 4).x) & 4u) {   // textured material: alpha = texture(BaseColor, uv).a * factor.a
                    float tu, tv;
                    interp_texcoord(sc, tri, hit.bx, hit.by, 1.0f - hit.bx - hit.by, tu, tv);
                    const GpuMaterial& m = sc.materials[sc.meshes[tri.w].MaterialId];
                    alpha = tex_sample(sc, m.BaseColorTexture, tu, tv).w * ((float)((m.BaseColorFactor >> 24) & 255u) / 255.0f);
                }
                if (alphaCutoff == 2.0f) thisVisibility *= 1.0f - alpha;
                else if (alpha > alphaCutoff) thisVisibility = 0.0f;
                if (thisVisibility < 0.01f) break;
                const float dist = hit.t + 0.001f;
                origin = origin + direction * dist;
                distanceToLight -= dist;
            }
            visibility += thisVisibility;
        }
        a.visibility[p] = visibility / (float)a.samples;
    }
}
