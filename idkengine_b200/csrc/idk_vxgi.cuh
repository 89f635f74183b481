// VXGI kernels for sm_90a over a linear rgba16f 3D grid in HBM (all mip levels in one allocation).
//
//   k_vx_voxelize_small / k_vx_voxelize_large   Voxelize/{vertex,geometry,fragment}.glsl + MergeIntermediates
//   k_vx_mipmap                                 Voxelize/Mipmap/compute.glsl
//   k_vx_cone_trace                             VXGI/ConeTraceGI/** + include/TraceCone.glsl
//
// Rasterisation rule, filtering rule and float semantics are spelled out in DESIGN.md section 8 and implemented
// independently by the CPU oracle (oracle/oracle_vxgi.inc); the two agree bit for bit.
#pragma once
#include <cuda_fp16.h>
#include "idk_device.cuh"
#include "idk_shadows.cuh"
#include "../../include/idk_gpu_types.h"

#define IDKVX_MAX_LEVELS 16
#define IDKVX_SMALL_LIMIT 16   // bounding boxes up to this many pixel centres are rasterised by the discovering thread
#define IDKVX_TILE 64          // larger boxes are cut into IDKVX_TILE^2 pixel tiles, one CTA each

struct VxGridDev {
    unsigned long long* level[IDKVX_MAX_LEVELS];   // 4 x half per texel
    int sx[IDKVX_MAX_LEVELS], sy[IDKVX_MAX_LEVELS], sz[IDKVX_MAX_LEVELS];
    int levels;
    float gmin[3], gmax[3];
    int z0, z1;                                    // voxelise only z in [z0, z1) (multi-GPU z-slab split; whole grid: 0, sz[0])
};

struct VxScene {
    const float* positions;        // PackedVec3
    const uint4* vertices;         // GpuVertex
    const int4* blasTris;          // GpuBlasTriangle
    const GpuBlasDesc* descs;
    const GpuBlasInstance* instances;
    const float4* xforms;          // 9 x float4 per GpuMeshTransform
    const GpuMesh* meshes;
    const GpuMaterial* materials;
    const GpuLight* lights;
    uint32_t lightCount;
    const TexRec* textures;        // material texture table (idkpt.h IdkPtTextureDesc), handle k = textures[k - 1]
    const float* srgbLut;
    DeviceScene occ;               // the path tracer's device scene: occluders of the point-shadowed lights (idkvx_set_shadow_tracer)
    int occValid;
};

__device__ __forceinline__ float det_tan(float x) { float s, c; det_sincos(x, &s, &c); return s / c; }

struct VxTri {
    f3 P[3], N[3];
    float U[3], V[3];             // TexCoord of the three vertices
    float qa[3], qb[3];
    float area;
    int a, b;
    int i0, i1, j0, j1;
    int meshId;
    bool valid;
};

__device__ __forceinline__ float vx_edge(float ax, float ay, float bx, float by, float cx, float cy) { return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax); }
__device__ __forceinline__ float f3get(f3 v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : v.z); }

__device__ __forceinline__ void vx_setup(const VxScene& sc, const VxGridDev& g, uint32_t inst, uint32_t triIndex, VxTri& t) {
    const GpuBlasInstance bi = sc.instances[inst];
    const float4* xf = sc.xforms + 9 * (size_t)bi.MeshTransformId;
    const float4 m0 = ldg4(xf), m1 = ldg4(xf + 1), m2 = ldg4(xf + 2), i0 = ldg4(xf + 3), i1 = ldg4(xf + 4), i2 = ldg4(xf + 5);
    const int4 tri = sc.blasTris[triIndex];
    const int vid[3] = {tri.x, tri.y, tri.z};
    const float ex = g.gmax[0] - g.gmin[0], ey = g.gmax[1] - g.gmin[1], ez = g.gmax[2] - g.gmin[2];
    f3 uvw[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const f3 p = mk3(sc.positions[3 * (size_t)vid[c]], sc.positions[3 * (size_t)vid[c] + 1], sc.positions[3 * (size_t)vid[c] + 2]);
        t.P[c] = xform_point(m0, m1, m2, p);
        t.N[c] = normalize3(xform_normal(i0, i1, i2, decompress_sr11g11b10(sc.vertices[vid[c]].w)));
        t.U[c] = __uint_as_float(sc.vertices[vid[c]].x);
        t.V[c] = __uint_as_float(sc.vertices[vid[c]].y);
        uvw[c] = mk3((t.P[c].x - g.gmin[0]) / ex, (t.P[c].y - g.gmin[1]) / ey, (t.P[c].z - g.gmin[2]) / ez);
    }
    const f3 n0 = mk3(uvw[0].x * 2.0f - 1.0f, uvw[0].y * 2.0f - 1.0f, uvw[0].z * 2.0f - 1.0f);
    const f3 n1 = mk3(uvw[1].x * 2.0f - 1.0f, uvw[1].y * 2.0f - 1.0f, uvw[1].z * 2.0f - 1.0f);
    const f3 n2 = mk3(uvw[2].x * 2.0f - 1.0f, uvw[2].y * 2.0f - 1.0f, uvw[2].z * 2.0f - 1.0f);
    const f3 cr = cross3(n1 - n0, n2 - n0);
    const float nw0 = fabsf(cr.x), nw1 = fabsf(cr.y), nw2 = fabsf(cr.z);
    int dom = nw1 > nw0 ? 1 : 0;
    dom = nw2 > (dom == 1 ? nw1 : nw0) ? 2 : dom;
    t.a = (dom + 1) % 3;
    t.b = (dom + 2) % 3;
    const int sa = t.a == 0 ? g.sx[0] : (t.a == 1 ? g.sy[0] : g.sz[0]);
    const int sb = t.b == 0 ? g.sx[0] : (t.b == 1 ? g.sy[0] : g.sz[0]);
#pragma unroll
    for (int c = 0; c < 3; c++) { t.qa[c] = f3get(uvw[c], t.a) * (float)sa; t.qb[c] = f3get(uvw[c], t.b) * (float)sb; }
    t.area = vx_edge(t.qa[0], t.qb[0], t.qa[1], t.qb[1], t.qa[2], t.qb[2]);
    t.valid = !(t.area == 0.0f || !(t.area == t.area));
    const float mina = fminf(t.qa[0], fminf(t.qa[1], t.qa[2])), maxa = fmaxf(t.qa[0], fmaxf(t.qa[1], t.qa[2]));
    const float minb = fminf(t.qb[0], fminf(t.qb[1], t.qb[2])), maxb = fmaxf(t.qb[0], fmaxf(t.qb[1], t.qb[2]));
    t.i0 = max(0, (int)ceilf(mina - 0.5f)); t.i1 = min(sa - 1, (int)floorf(maxa - 0.5f));
    t.j0 = max(0, (int)ceilf(minb - 0.5f)); t.j1 = min(sb - 1, (int)floorf(maxb - 0.5f));
    t.meshId = tri.w;
    if (t.i1 < t.i0 || t.j1 < t.j0) t.valid = false;
}

// one pixel centre (i, j) of the projection plane; returns true if a voxel was written
__device__ __forceinline__ bool vx_pixel(const VxScene& sc, const VxGridDev& g, const VxTri& t, int i, int j, uint32_t* stack) {
    const float cx = (float)i + 0.5f, cy = (float)j + 0.5f;
    const float w0 = vx_edge(t.qa[1], t.qb[1], t.qa[2], t.qb[2], cx, cy);
    const float w1 = vx_edge(t.qa[2], t.qb[2], t.qa[0], t.qb[0], cx, cy);
    const float w2 = vx_edge(t.qa[0], t.qb[0], t.qa[1], t.qb[1], cx, cy);
    const bool inside = t.area > 0.0f ? (w0 >= 0.0f && w1 >= 0.0f && w2 >= 0.0f) : (w0 <= 0.0f && w1 <= 0.0f && w2 <= 0.0f);
    if (!inside) return false;
    const float b0 = w0 / t.area, b1 = w1 / t.area, b2 = w2 / t.area;
    const f3 fragPos = (t.P[0] * b0 + t.P[1] * b1) + t.P[2] * b2;
    const f3 normal = (t.N[0] * b0 + t.N[1] * b1) + t.N[2] * b2;
    const float fu = (fragPos.x - g.gmin[0]) / (g.gmax[0] - g.gmin[0]);
    const float fv = (fragPos.y - g.gmin[1]) / (g.gmax[1] - g.gmin[1]);
    const float fw = (fragPos.z - g.gmin[2]) / (g.gmax[2] - g.gmin[2]);
    if (!(fu >= 0.0f && fv >= 0.0f && fw >= 0.0f)) return false;
    const int vx = (int)(fu * (float)g.sx[0]), vy = (int)(fv * (float)g.sy[0]), vz = (int)(fw * (float)g.sz[0]);
    if (vx >= g.sx[0] || vy >= g.sy[0] || vz >= g.sz[0]) return false;
    if (vz < g.z0 || vz >= g.z1) return false;                    // another rank's slab

    // fragment.glsl:31-79 (no point shadows). GetSurface(material, TexCoord): the fragment stage samples with implicit
    // derivatives / mip levels; here the base level is sampled bilinearly like everywhere else in this library.
    const GpuMesh& mesh = sc.meshes[t.meshId];
    const GpuMaterial& mat = sc.materials[mesh.MaterialId];
    const uint32_t c = mat.BaseColorFactor;
    f3 albedo = mk3((float)(c & 255u) / 255.0f, (float)((c >> 8) & 255u) / 255.0f, (float)((c >> 16) & 255u) / 255.0f);
    float alpha = (float)((c >> 24) & 255u) / 255.0f;
    f3 emissive = mk3(mat.EmissiveFactor[0], mat.EmissiveFactor[1], mat.EmissiveFactor[2]);
    if ((mat.BaseColorTexture | mat.MetallicRoughnessTexture | mat.NormalTexture | mat.EmissiveTexture | mat.TransmissionTexture) != 0) {
        const float tu = (t.U[0] * b0 + t.U[1] * b1) + t.U[2] * b2, tv = (t.V[0] * b0 + t.V[1] * b1) + t.V[2] * b2;
        const float4 base = tex_sample_raw(sc.textures, sc.srgbLut, mat.BaseColorTexture, tu, tv);
        albedo = mk3(base.x * albedo.x, base.y * albedo.y, base.z * albedo.z);
        alpha = base.w * alpha;
        const float4 et = tex_sample_raw(sc.textures, sc.srgbLut, mat.EmissiveTexture, tu, tv);
        emissive = mk3(et.x * emissive.x, et.y * emissive.y, et.z * emissive.z);
    }
    emissive = emissive + mesh.EmissiveBias * albedo;
    f3 direct = mk3(0.0f, 0.0f, 0.0f);
    for (uint32_t l = 0; l < sc.lightCount; l++) {
        const GpuLight& L = sc.lights[l];
        const f3 sampleToLight = mk3(L.Position[0], L.Position[1], L.Position[2]) - fragPos;
        const float dist = sqrtf(dot3(sampleToLight, sampleToLight));
        const f3 lightDir = sampleToLight / dist;
        const float cosTheta = dot3(normalize3(normal), lightDir);
        if (cosTheta > 0.0f) {
            const f3 diffuse = mk3(L.Color[0], L.Color[1], L.Color[2]) * cosTheta * albedo;
            const float lr = fmaxf(L.Radius, 0.0001f);
            const float dsq = fmaxf(dist * dist, 0.0001f);
            f3 contrib = diffuse * ((lr * lr) / dsq);
            if (L.PointShadowIndex >= 0 && sc.occValid) {
                // Visibility(pointShadow, -sampleToLight) (fragment.glsl:100-110): the shadow-map compare point sits 2 % of the way
                // towards the light; here that point is connected to the light by an any-hit ray instead of the PCF lookup
                const float bias = 0.02f;
                HitRec sh;
                uint32_t sx;
                const bool occluded = trace_any(sc.occ, fragPos + sampleToLight * bias, lightDir, dist * (1.0f - bias), false, stack, sh, sx);
                contrib = contrib * (occluded ? 0.0f : 1.0f);
            }
            direct = direct + contrib;
        }
    }
    direct = direct + albedo * 0.02f;
    direct = direct + emissive;
    const f3 val = direct * alpha;

    // imageAtomicMax per channel (+ alpha = 1 where written): 64-bit CAS on the packed rgba16f texel. Non-negative
    // halves order like unsigned shorts and RNE conversion is monotonic, so this equals max-then-convert.
    const uint32_t lo = (uint32_t)__half_as_ushort(__float2half_rn(val.x)) | ((uint32_t)__half_as_ushort(__float2half_rn(val.y)) << 16);
    const uint32_t hi = (uint32_t)__half_as_ushort(__float2half_rn(val.z)) | (0x3C00u << 16);
    unsigned long long* p = g.level[0] + (((size_t)vz * g.sy[0] + vy) * g.sx[0] + vx);
    unsigned long long old = *p;
    for (;;) {
        const uint32_t mlo = __vmaxu2((uint32_t)old, lo), mhi = __vmaxu2((uint32_t)(old >> 32), hi);
        const unsigned long long m = (unsigned long long)mlo | ((unsigned long long)mhi << 32);
        if (m == old) break;
        const unsigned long long prev = atomicCAS(p, old, m);
        if (prev == old) break;
        old = prev;
    }
    return true;
}

struct VxVoxelizeArgs {
    VxScene sc;
    VxGridDev g;
    uint32_t instance;
    uint32_t triFirst, triCount;     // BlasTriangles range of this instance's BLAS
    uint4* queue;                    // (instance, triangle, tile x, tile y) work items of large triangles
    uint32_t* queueCount;
    uint32_t queueCapacity;
    unsigned long long* fragments;
};

__global__ void __launch_bounds__(256) k_vx_voxelize_small(VxVoxelizeArgs a) {
    extern __shared__ uint32_t s_vxStack[];          // shadow-ray traversal stacks (only with point-shadowed lights)
    uint32_t* stack = s_vxStack + threadIdx.x;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t frags = 0;
    if (k < a.triCount) {
        VxTri t;
        vx_setup(a.sc, a.g, a.instance, a.triFirst + k, t);
        if (t.valid) {
            const int area = (t.i1 - t.i0 + 1) * (t.j1 - t.j0 + 1);
            if (area <= IDKVX_SMALL_LIMIT) {
                for (int j = t.j0; j <= t.j1; j++)
                    for (int i = t.i0; i <= t.i1; i++) frags += vx_pixel(a.sc, a.g, t, i, j, stack) ? 1u : 0u;
            } else {
                // cut the bounding box into tiles and queue one work item per tile (a wall-sized triangle becomes
                // dozens of CTAs instead of one); if the queue is full the thread rasterises the remainder itself
                const int tx = (t.i1 - t.i0) / IDKVX_TILE + 1, ty = (t.j1 - t.j0) / IDKVX_TILE + 1;
                const uint32_t slot = atomicAdd(a.queueCount, (uint32_t)(tx * ty));
                for (int q = 0; q < tx * ty; q++) {
                    const int ox = q % tx, oy = q / tx;
                    if (slot + (uint32_t)q < a.queueCapacity) {
                        a.queue[slot + q] = make_uint4(a.instance, a.triFirst + k, (uint32_t)ox, (uint32_t)oy);
                    } else {
                        const int i0 = t.i0 + ox * IDKVX_TILE, j0 = t.j0 + oy * IDKVX_TILE;
                        for (int j = j0; j <= min(t.j1, j0 + IDKVX_TILE - 1); j++)
                            for (int i = i0; i <= min(t.i1, i0 + IDKVX_TILE - 1); i++) frags += vx_pixel(a.sc, a.g, t, i, j, stack) ? 1u : 0u;
                    }
                }
            }
        }
    }
    for (int off = 16; off > 0; off >>= 1) frags += __shfl_down_sync(0xffffffffu, frags, off);
    if ((threadIdx.x & 31) == 0 && frags) atomicAdd(a.fragments, (unsigned long long)frags);
}

// one CTA per queued (triangle, tile) work item, threads stride over the tile's pixel centres
__global__ void __launch_bounds__(256) k_vx_voxelize_large(VxScene sc, VxGridDev g, const uint4* __restrict__ queue,
                                                           const uint32_t* __restrict__ queueCount, uint32_t queueCapacity,
                                                           unsigned long long* fragments) {
    extern __shared__ uint32_t s_vxStack[];
    uint32_t* stack = s_vxStack + threadIdx.x;
    const uint32_t n = min(*queueCount, queueCapacity);
    uint32_t frags = 0;
    for (uint32_t q = blockIdx.x; q < n; q += gridDim.x) {
        const uint4 e = queue[q];
        VxTri t;
        vx_setup(sc, g, e.x, e.y, t);
        const int i0 = t.i0 + (int)e.z * IDKVX_TILE, j0 = t.j0 + (int)e.w * IDKVX_TILE;
        const int w = min(t.i1, i0 + IDKVX_TILE - 1) - i0 + 1, h = min(t.j1, j0 + IDKVX_TILE - 1) - j0 + 1;
        for (int p = threadIdx.x; p < w * h; p += blockDim.x)
            frags += vx_pixel(sc, g, t, i0 + p % w, j0 + p / w, stack) ? 1u : 0u;
    }
    for (int off = 16; off > 0; off >>= 1) frags += __shfl_down_sync(0xffffffffu, frags, off);
    if ((threadIdx.x & 31) == 0 && frags) atomicAdd(fragments, (unsigned long long)frags);
}

// ------------------------------------------------------------------------------------------------ filtering
__device__ __forceinline__ float4 vx_fetch(const VxGridDev& g, int l, int x, int y, int z) {
    const unsigned long long t = __ldg(g.level[l] + (((size_t)z * g.sy[l] + y) * g.sx[l] + x));
    const uint32_t lo = (uint32_t)t, hi = (uint32_t)(t >> 32);
    return make_float4(__half2float(__ushort_as_half((unsigned short)(lo & 0xFFFFu))), __half2float(__ushort_as_half((unsigned short)(lo >> 16))),
                       __half2float(__ushort_as_half((unsigned short)(hi & 0xFFFFu))), __half2float(__ushort_as_half((unsigned short)(hi >> 16))));
}
__device__ __forceinline__ float4 lerp4(float4 a, float4 b, float t) {
    const float s = 1.0f - t;
    return make_float4(a.x * s + b.x * t, a.y * s + b.y * t, a.z * s + b.z * t, a.w * s + b.w * t);
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__device__ __forceinline__ float4 vx_trilinear(const VxGridDev& g, int l, float u, float v, float w, int ox, int oy, int oz) {
    const int sx = g.sx[l], sy = g.sy[l], sz = g.sz[l];
    const float px = u * (float)sx - 0.5f, py = v * (float)sy - 0.5f, pz = w * (float)sz - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py), fz0 = floorf(pz);
    const float fx = px - fx0, fy = py - fy0, fz = pz - fz0;
    const int x0 = clampi((int)fx0 + ox, 0, sx - 1), x1 = clampi((int)fx0 + 1 + ox, 0, sx - 1);
    const int y0 = clampi((int)fy0 + oy, 0, sy - 1), y1 = clampi((int)fy0 + 1 + oy, 0, sy - 1);
    const int z0 = clampi((int)fz0 + oz, 0, sz - 1), z1 = clampi((int)fz0 + 1 + oz, 0, sz - 1);
    const float4 c00 = lerp4(vx_fetch(g, l, x0, y0, z0), vx_fetch(g, l, x1, y0, z0), fx);
    const float4 c10 = lerp4(vx_fetch(g, l, x0, y1, z0), vx_fetch(g, l, x1, y1, z0), fx);
    const float4 c01 = lerp4(vx_fetch(g, l, x0, y0, z1), vx_fetch(g, l, x1, y0, z1), fx);
    const float4 c11 = lerp4(vx_fetch(g, l, x0, y1, z1), vx_fetch(g, l, x1, y1, z1), fx);
    return lerp4(lerp4(c00, c10, fy), lerp4(c01, c11, fy), fz);
}

__device__ __forceinline__ float4 vx_texture_lod(const VxGridDev& g, float u, float v, float w, float lod) {
    const int maxLevel = g.levels - 1;
    lod = clamp1(lod, 0.0f, (float)maxLevel);
    const float l0f = floorf(lod);
    const int l0 = (int)l0f;
    const float fl = lod - l0f;
    const float4 a = vx_trilinear(g, l0, u, v, w, 0, 0, 0);
    if (fl == 0.0f || l0 >= maxLevel) return a;
    return lerp4(a, vx_trilinear(g, l0 + 1, u, v, w, 0, 0, 0), fl);
}

__global__ void __launch_bounds__(256) k_vx_mipmap(VxGridDev g, int level) {
    const int sx = g.sx[level], sy = g.sy[level], sz = g.sz[level];
    const size_t n = (size_t)sx * sy * sz;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(idx % sx), y = (int)((idx / sx) % sy), z = (int)(idx / ((size_t)sx * sy));
        const float u = ((float)x + 0.5f) / (float)sx, v = ((float)y + 0.5f) / (float)sy, w = ((float)z + 0.5f) / (float)sz;
        float4 r = vx_trilinear(g, level - 1, u, v, w, 0, 0, 0);
        float4 s;
        s = vx_trilinear(g, level - 1, u, v, w, -1, 0, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
        s = vx_trilinear(g, level - 1, u, v, w, 1, 0, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
        s = vx_trilinear(g, level - 1, u, v, w, 0, -1, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
        s = vx_trilinear(g, level - 1, u, v, w, 0, 1, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
        s = vx_trilinear(g, level - 1, u, v, w, 0, 0, -1); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
        s = vx_trilinear(g, level - 1, u, v, w, 0, 0, 1); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
        const uint32_t lo = (uint32_t)__half_as_ushort(__float2half_rn(r.x / 7.0f)) | ((uint32_t)__half_as_ushort(__float2half_rn(r.y / 7.0f)) << 16);
        const uint32_t hi = (uint32_t)__half_as_ushort(__float2half_rn(r.z / 7.0f)) | ((uint32_t)__half_as_ushort(__float2half_rn(r.w / 7.0f)) << 16);
        g.level[level][idx] = (unsigned long long)lo | ((unsigned long long)hi << 32);
    }
}

// Tiled variant for the levels that halve exactly (source = 2 x destination on every axis, i.e. every big level of a
// power-of-two-ish grid): a CTA produces an 8 x 8 x 4 block of destination texels from the (2*8+2) x (2*8+2) x (2*4+2) source
// texels around it. The tile is fetched from HBM ONCE (coalesced rows), converted half -> float ONCE and kept in shared
// memory as float4; the 7 trilinear taps then read shared memory. The arithmetic of every destination texel -- coordinates,
// weights, lerp order, tap order, /7, RNE conversion -- is that of k_vx_mipmap, so the result is bit-identical; what changes
// is that a source texel is read and converted once per tile instead of ~7 times per neighbourhood (the r01 kernel ran at
// 21 % of the HBM rate, bound by the 56 global fetches + 224 half conversions per destination texel).
#define IDKVX_MT_X 8
#define IDKVX_MT_Y 8
#define IDKVX_MT_Z 4
#define IDKVX_MS_X (2 * IDKVX_MT_X + 2)
#define IDKVX_MS_Y (2 * IDKVX_MT_Y + 2)
#define IDKVX_MS_Z (2 * IDKVX_MT_Z + 2)
#define IDKVX_MIP_TILE_SMEM (IDKVX_MS_X * IDKVX_MS_Y * IDKVX_MS_Z * 16)

__device__ __forceinline__ float4 vx_tile_trilinear(const float4* tile, int bx, int by, int bz, int sx, int sy, int sz,
                                                    float u, float v, float w, int ox, int oy, int oz) {
    const float px = u * (float)sx - 0.5f, py = v * (float)sy - 0.5f, pz = w * (float)sz - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py), fz0 = floorf(pz);
    const float fx = px - fx0, fy = py - fy0, fz = pz - fz0;
    // tile entry (i, j, k) holds source texel (clamp(bx + i), clamp(by + j), clamp(bz + k)): indexing with the UNCLAMPED
    // coordinate relative to the tile origin returns exactly what clamp-then-fetch returns in vx_trilinear
    const int x0 = (int)fx0 + ox - bx, y0 = (int)fy0 + oy - by, z0 = (int)fz0 + oz - bz;
#define T_(i, j, k) tile[((k) * IDKVX_MS_Y + (j)) * IDKVX_MS_X + (i)]
    const float4 c00 = lerp4(T_(x0, y0, z0), T_(x0 + 1, y0, z0), fx);
    const float4 c10 = lerp4(T_(x0, y0 + 1, z0), T_(x0 + 1, y0 + 1, z0), fx);
    const float4 c01 = lerp4(T_(x0, y0, z0 + 1), T_(x0 + 1, y0, z0 + 1), fx);
    const float4 c11 = lerp4(T_(x0, y0 + 1, z0 + 1), T_(x0 + 1, y0 + 1, z0 + 1), fx);
#undef T_
    return lerp4(lerp4(c00, c10, fy), lerp4(c01, c11, fy), fz);
}

__global__ void __launch_bounds__(256) k_vx_mipmap_tiled(VxGridDev g, int level) {
    extern __shared__ __align__(16) float4 s_tile[];
    const int sx = g.sx[level], sy = g.sy[level], sz = g.sz[level];
    const int px_ = g.sx[level - 1], py_ = g.sy[level - 1], pz_ = g.sz[level - 1];      // source = 2 x destination on every axis
    const int tilesX = (sx + IDKVX_MT_X - 1) / IDKVX_MT_X, tilesY = (sy + IDKVX_MT_Y - 1) / IDKVX_MT_Y, tilesZ = (sz + IDKVX_MT_Z - 1) / IDKVX_MT_Z;
    const int nTiles = tilesX * tilesY * tilesZ;
    for (int tIdx = blockIdx.x; tIdx < nTiles; tIdx += gridDim.x) {
        const int tx = tIdx % tilesX, ty = (tIdx / tilesX) % tilesY, tz = tIdx / (tilesX * tilesY);
        const int X0 = tx * IDKVX_MT_X, Y0 = ty * IDKVX_MT_Y, Z0 = tz * IDKVX_MT_Z;
        const int bx = 2 * X0 - 1, by = 2 * Y0 - 1, bz = 2 * Z0 - 1;      // source coordinate of tile entry (0, 0, 0)
        __syncthreads();                                                    // the previous tile has been consumed
        for (int e = threadIdx.x; e < IDKVX_MS_X * IDKVX_MS_Y * IDKVX_MS_Z; e += blockDim.x) {
            const int i = e % IDKVX_MS_X, j = (e / IDKVX_MS_X) % IDKVX_MS_Y, k = e / (IDKVX_MS_X * IDKVX_MS_Y);
            s_tile[e] = vx_fetch(g, level - 1, clampi(bx + i, 0, px_ - 1), clampi(by + j, 0, py_ - 1), clampi(bz + k, 0, pz_ - 1));
        }
        __syncthreads();
        const int lx = threadIdx.x % IDKVX_MT_X, ly = (threadIdx.x / IDKVX_MT_X) % IDKVX_MT_Y, lz = threadIdx.x / (IDKVX_MT_X * IDKVX_MT_Y);
        const int x = X0 + lx, y = Y0 + ly, z = Z0 + lz;
        if (x < sx && y < sy && z < sz) {
            const float u = ((float)x + 0.5f) / (float)sx, v = ((float)y + 0.5f) / (float)sy, w = ((float)z + 0.5f) / (float)sz;
            float4 r = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, 0, 0, 0);
            float4 s;
            s = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, -1, 0, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
            s = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, 1, 0, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
            s = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, 0, -1, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
            s = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, 0, 1, 0); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
            s = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, 0, 0, -1); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
            s = vx_tile_trilinear(s_tile, bx, by, bz, px_, py_, pz_, u, v, w, 0, 0, 1); r = make_float4(r.x + s.x, r.y + s.y, r.z + s.z, r.w + s.w);
            const uint32_t lo = (uint32_t)__half_as_ushort(__float2half_rn(r.x / 7.0f)) | ((uint32_t)__half_as_ushort(__float2half_rn(r.y / 7.0f)) << 16);
            const uint32_t hi = (uint32_t)__half_as_ushort(__float2half_rn(r.z / 7.0f)) | ((uint32_t)__half_as_ushort(__float2half_rn(r.w / 7.0f)) << 16);
            g.level[level][((size_t)z * sy + y) * sx + x] = (unsigned long long)lo | ((unsigned long long)hi << 32);
        }
    }
}

// ------------------------------------------------------------------------------------------------ cone tracing
struct VxConeArgs {
    VxGridDev g;
    float invProjView[16];
    float viewPos[3];
    int maxSamples;
    float stepMultiplier, giBoost, giSkyBoxBoost, normalRayOffset;
    uint32_t noiseIndex;
    float sky[3];
    const float* depth;
    const float2* normalRG;
    const float2* metalRough;
    float4* out;
    int width, height;            // height = rows in this launch's arrays
    int fullHeight, rowFirst;     // the G-buffer's real height and the first row these arrays hold (screen-tiled cone tracing)
    unsigned long long* steps;
};

__device__ __forceinline__ float vx_ign(float x, float y, uint32_t index) {
    x += (float)index * 5.588238f;
    y += (float)index * 5.588238f;
    return fract1(52.9829189f * fract1(0.06711056f * x + 0.00583715f * y));
}

__device__ __forceinline__ float4 vx_trace_cone(const VxGridDev& g, f3 origin, f3 dir, f3 normal, float coneAngle, float stepMultiplier,
                                                float normalRayOffset, float alphaThreshold, uint32_t& steps) {
    const float vsx = (g.gmax[0] - g.gmin[0]) / (float)g.sx[0], vsy = (g.gmax[1] - g.gmin[1]) / (float)g.sy[0], vsz = (g.gmax[2] - g.gmin[2]) / (float)g.sz[0];
    const float voxelMaxLength = fmaxf(vsx, fmaxf(vsy, vsz));
    const float voxelMinLength = fminf(vsx, fminf(vsy, vsz));
    const float maxLevel = (float)(g.levels - 1);
    float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    origin = origin + normal * voxelMaxLength * normalRayOffset;
    float distFromStart = voxelMaxLength;
    const float tanA = det_tan(coneAngle);
    while (acc.w < alphaThreshold) {
        const float coneDiameter = 2.0f * tanA * distFromStart;
        const float sampleDiameter = fmaxf(voxelMinLength, coneDiameter);
        const float sampleLod = det_log2(sampleDiameter / voxelMinLength);
        const f3 worldPos = origin + dir * distFromStart;
        const float u = (worldPos.x - g.gmin[0]) / (g.gmax[0] - g.gmin[0]);
        const float v = (worldPos.y - g.gmin[1]) / (g.gmax[1] - g.gmin[1]);
        const float w = (worldPos.z - g.gmin[2]) / (g.gmax[2] - g.gmin[2]);
        if (u < 0.0f || v < 0.0f || w < 0.0f || u >= 1.0f || v >= 1.0f || w >= 1.0f || sampleLod > maxLevel || !(u == u) || !(v == v) || !(w == w)) break;
        const float4 s = vx_texture_lod(g, u, v, w, sampleLod);
        const float weight = 1.0f - acc.w;
        acc = make_float4(acc.x + s.x * weight, acc.y + s.y * weight, acc.z + s.z * weight, acc.w + s.w * weight);
        distFromStart += sampleDiameter * stepMultiplier;
        steps++;
    }
    return acc;
}

__global__ void __launch_bounds__(64) k_vx_cone_trace(VxConeArgs a) {
    const int x = blockIdx.x * 8 + threadIdx.x, yl = blockIdx.y * 8 + threadIdx.y;
    const int y = yl + a.rowFirst;
    uint32_t steps = 0;
    if (x < a.width && yl < a.height) {
        const size_t p = (size_t)yl * a.width + x;
        const float d = a.depth[p];
        if (d == 1.0f) {
            a.out[p] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        } else {
            const float u = ((float)x + 0.5f) / (float)a.width, v = ((float)y + 0.5f) / (float)a.fullHeight;
            const float nx = u * 2.0f - 1.0f, ny = v * 2.0f - 1.0f;
            const float* m = a.invProjView;
            const float wx = ((m[0] * nx + m[4] * ny) + m[8] * d) + m[12] * 1.0f;
            const float wy = ((m[1] * nx + m[5] * ny) + m[9] * d) + m[13] * 1.0f;
            const float wz = ((m[2] * nx + m[6] * ny) + m[10] * d) + m[14] * 1.0f;
            const float ww = ((m[3] * nx + m[7] * ny) + m[11] * d) + m[15] * 1.0f;
            const f3 fragPos = mk3(wx / ww, wy / ww, wz / ww);
            const float2 nrg = a.normalRG[p], mr = a.metalRough[p];
            const f3 normal = decode_unit_vec(nrg.x, nrg.y);
            const float metallic = mr.x;
            float roughness = mr.y;
            const f3 incomming = fragPos - mk3(a.viewPos[0], a.viewPos[1], a.viewPos[2]);
            roughness *= roughness;
            const float dc = 1.0f - metallic - 0.0f;
            const float materialVariance = dc + metallic * roughness + 0.0f * roughness;
            const uint32_t samples = (uint32_t)mix1(1.0f, (float)a.maxSamples, materialVariance);
            uint32_t noiseIndex = a.noiseIndex;
            f3 irradiance = mk3(0.0f, 0.0f, 0.0f);
            for (uint32_t i = 0; i < samples; i++) {
                const float rnd0 = vx_ign((float)x, (float)y, noiseIndex + 0);
                const float rnd1 = vx_ign((float)x, (float)y, noiseIndex + 1);
                const float rnd2 = vx_ign((float)x, (float)y, noiseIndex + 2);
                noiseIndex++;
                const f3 diffuseDir = normalize3(normal + sample_sphere(rnd0, rnd1));
                f3 dir;
                float coneAngle;
                if (metallic > rnd2) {
                    dir = normalize3(mix3(reflect3(incomming, normal), diffuseDir, roughness));
                    coneAngle = mix1(0.0f, 0.32f, roughness);
                } else {
                    dir = diffuseDir;
                    coneAngle = 0.32f;
                }
                const float4 c = vx_trace_cone(a.g, fragPos, dir, normal, coneAngle, a.stepMultiplier, a.normalRayOffset, 0.99f, steps);
                const float k = 1.0f - c.w;
                irradiance = irradiance + mk3(c.x + k * (a.sky[0] * a.giSkyBoxBoost), c.y + k * (a.sky[1] * a.giSkyBoxBoost), c.z + k * (a.sky[2] * a.giSkyBoxBoost));
            }
            irradiance = irradiance / (float)samples;
            a.out[p] = make_float4(irradiance.x * a.giBoost, irradiance.y * a.giBoost, irradiance.z * a.giBoost, 1.0f);
        }
    }
    for (int off = 16; off > 0; off >>= 1) steps += __shfl_down_sync(0xffffffffu, steps, off);
    if (((threadIdx.y * 8 + threadIdx.x) & 31) == 0 && steps) atomicAdd(a.steps, (unsigned long long)steps);
}
