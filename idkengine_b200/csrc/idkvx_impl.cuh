// libidkpt, VXGI part: C ABI of include/idkvx.h over the kernels of idk_vxgi.cuh. Included at the end of idkpt.cu (one
// translation unit), so that the voxeliser can trace shadow rays through the path tracer's device scene (idk_shadows.cuh).
// Host sequencing mirrors Voxelizer.Render (IDKEngine/Source/Render/VXGI/Voxelizer/Voxelizer.cs:109-228:
// ClearTextures -> Voxelize -> Mipmap levels 1..n-1) and ConeTracer.Compute (ConeTracing/ConeTracer.cs:37-50).
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>

#include "../../include/idkvx.h"
#include "idk_vxgi.cuh"
#include "idk_textures_host.h"
#pragma once

static thread_local std::string g_vxCreateError;

struct IdkVxCtx {
    int device = 0, smCount = 132;
    cudaStream_t stream = nullptr;
    std::string lastError;
    VxGridDev grid = {};
    void* gridMem = nullptr;
    size_t levelTexels[IDKVX_MAX_LEVELS] = {};
    bool haveScene = false;
    VxScene sc = {};
    IdkPtSceneDesc counts = {};
    std::vector<GpuBlasDesc> hostDescs;
    std::vector<GpuBlasInstance> hostInstances;
    void* dPositions = nullptr; void* dVertices = nullptr; void* dTris = nullptr; void* dDescs = nullptr; void* dInstances = nullptr;
    void* dXforms = nullptr; void* dMeshes = nullptr; void* dMaterials = nullptr; void* dLights = nullptr;
    void* dTexPixels = nullptr; void* dTexRecs = nullptr; void* dSrgbLut = nullptr;
    void* dQueue = nullptr; void* dQueueCount = nullptr; void* dCounters = nullptr;
    size_t queueCapacity = 0;
    bool slabMode = false;                // idkvx_set_slab: voxelise one z-slab, no mip chain (the host all-gathers the slabs first)
    IdkPtCtx* shadowTracer = nullptr;     // idkvx_set_shadow_tracer: visibility of point-shadowed lights by shadow rays through this scene
    bool shadowedLights = false;
};

#define VCK(call)                                                                                  \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            char buf_[512];                                                                        \
            snprintf(buf_, sizeof(buf_), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            ctx->lastError = buf_;                                                                 \
            return IDKPT_ERR_CUDA;                                                                 \
        }                                                                                          \
    } while (0)

static int vfail(IdkVxCtx* ctx, int code, const char* msg) {
    if (ctx) ctx->lastError = msg; else g_vxCreateError = msg;
    return code;
}

static int vupload(IdkVxCtx* ctx, void** dst, const void* src, size_t bytes) {
    if (*dst) { cudaFree(*dst); *dst = nullptr; }
    VCK(cudaMalloc(dst, std::max<size_t>(bytes, 16)));
    if (bytes) VCK(cudaMemcpyAsync(*dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return IDKPT_OK;
}

static void set_grid_bounds(IdkVxCtx* ctx, const float* mn, const float* mx) {
    // Voxelizer.GridMin / GridMax setters keep max >= min + 0.1 (Voxelizer.cs:16-33)
    for (int i = 0; i < 3; i++) {
        ctx->grid.gmin[i] = mn[i];
        ctx->grid.gmax[i] = std::max(mx[i], mn[i] + 0.1f);
    }
}

extern "C" {

IDKPT_API const char* idkvx_last_error(IdkVxCtx* ctx) { return ctx ? ctx->lastError.c_str() : g_vxCreateError.c_str(); }

IDKPT_API int idkvx_create(const IdkVxCreateInfo* ci, IdkVxCtx** out) {
    if (!ci || !out) return vfail(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_create: null argument");
    *out = nullptr;
    if (ci->Width < 1 || ci->Height < 1 || ci->Depth < 1 || ci->Width > 2048 || ci->Height > 2048 || ci->Depth > 2048)
        return vfail(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_create: invalid grid size");
    int deviceCount = 0;
    if (cudaGetDeviceCount(&deviceCount) != cudaSuccess || deviceCount == 0)
        return vfail(nullptr, IDKPT_ERR_NO_DEVICE, "idkvx_create: no CUDA device (libidkpt has no CPU fallback)");
    if (ci->Device < 0 || ci->Device >= deviceCount) return vfail(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_create: device ordinal out of range");
    if (cudaSetDevice(ci->Device) != cudaSuccess) return vfail(nullptr, IDKPT_ERR_CUDA, "idkvx_create: cudaSetDevice failed");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, ci->Device) != cudaSuccess) return vfail(nullptr, IDKPT_ERR_CUDA, "idkvx_create: cudaGetDeviceProperties failed");
    if (prop.major != 9 || prop.minor != 0) return vfail(nullptr, IDKPT_ERR_NO_DEVICE, "idkvx_create: libidkpt is built for sm_90a only");
    IdkVxCtx* ctx = new IdkVxCtx();
    ctx->device = ci->Device;
    ctx->smCount = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return vfail(nullptr, IDKPT_ERR_CUDA, "idkvx_create: stream creation failed"); }
    // Texture.GetMaxMipmapLevel: levels down to 1 texel of the largest extent
    const int mx = std::max(ci->Width, std::max(ci->Height, ci->Depth));
    int levels = 1;
    while ((mx >> levels) > 0) levels++;
    ctx->grid.levels = levels;
    ctx->grid.z0 = 0; ctx->grid.z1 = ci->Depth;
    size_t total = 0;
    for (int l = 0; l < levels; l++) {
        ctx->grid.sx[l] = std::max(1, ci->Width >> l);
        ctx->grid.sy[l] = std::max(1, ci->Height >> l);
        ctx->grid.sz[l] = std::max(1, ci->Depth >> l);
        ctx->levelTexels[l] = (size_t)ctx->grid.sx[l] * ctx->grid.sy[l] * ctx->grid.sz[l];
        total += ctx->levelTexels[l];
    }
    if (cudaMalloc(&ctx->gridMem, total * 8) != cudaSuccess) {
        cudaStreamDestroy(ctx->stream);
        delete ctx;
        return vfail(nullptr, IDKPT_ERR_OUT_OF_MEMORY, "idkvx_create: voxel grid allocation failed");
    }
    cudaMemsetAsync(ctx->gridMem, 0, total * 8, ctx->stream);   // ResultVoxels.Fill(0), Voxelizer.cs:258
    size_t off = 0;
    for (int l = 0; l < levels; l++) { ctx->grid.level[l] = (unsigned long long*)ctx->gridMem + off; off += ctx->levelTexels[l]; }
    set_grid_bounds(ctx, ci->GridMin, ci->GridMax);
    cudaMalloc(&ctx->dQueueCount, 16);
    cudaMalloc(&ctx->dCounters, 16);
    *out = ctx;
    return IDKPT_OK;
}

IDKPT_API void idkvx_destroy(IdkVxCtx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    void* all[] = {ctx->gridMem, ctx->dPositions, ctx->dVertices, ctx->dTris, ctx->dDescs, ctx->dInstances, ctx->dXforms, ctx->dMeshes,
                   ctx->dMaterials, ctx->dLights, ctx->dTexPixels, ctx->dTexRecs, ctx->dSrgbLut, ctx->dQueue, ctx->dQueueCount, ctx->dCounters};
    for (void* p : all) if (p) cudaFree(p);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

IDKPT_API int32_t idkvx_level_count(IdkVxCtx* ctx) { return ctx ? ctx->grid.levels : 0; }

IDKPT_API int idkvx_set_grid(IdkVxCtx* ctx, const float gridMin[3], const float gridMax[3]) {
    if (!ctx || !gridMin || !gridMax) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_grid: null argument");
    set_grid_bounds(ctx, gridMin, gridMax);
    return IDKPT_OK;
}

IDKPT_API int idkvx_set_scene(IdkVxCtx* ctx, const IdkPtSceneDesc* s) {
    if (!ctx || !s) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: null argument");
    VCK(cudaSetDevice(ctx->device));
    if (!s->BlasTriangles || !s->BlasDescs || !s->BlasInstances || !s->MeshTransforms || !s->Meshes || !s->Materials || !s->Vertices || !s->VertexPositions)
        return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: a required array is null");
    if (s->LightCount > IDK_GPU_MAX_UBO_LIGHT_COUNT) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: more than 256 lights");
    bool shadowed = false;
    for (uint64_t i = 0; i < s->LightCount; i++) shadowed = shadowed || s->Lights[i].PointShadowIndex >= 0;
    for (uint64_t i = 0; i < s->BlasInstanceCount; i++)
        if (s->BlasInstances[i].BlasId >= s->BlasDescCount || s->BlasInstances[i].MeshTransformId >= s->MeshTransformCount)
            return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: BlasInstance references a missing BLAS or transform");
    for (uint64_t i = 0; i < s->BlasDescCount; i++) {
        const GpuBlasDesc& d = s->BlasDescs[i];
        if (d.TriangleOffset < 0 || d.TriangleCount < 0 || (uint64_t)d.TriangleOffset + d.TriangleCount > s->BlasTriangleCount)
            return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: GpuBlasDesc triangle range outside the array");
    }
    const uint64_t lim = std::min(s->VertexPositionCount, s->VertexCount);
    for (uint64_t i = 0; i < s->BlasTriangleCount; i++) {
        const GpuBlasTriangle& t = s->BlasTriangles[i];
        if ((uint64_t)(uint32_t)t.X >= lim || (uint64_t)(uint32_t)t.Y >= lim || (uint64_t)(uint32_t)t.Z >= lim || t.MeshId < 0 || (uint64_t)t.MeshId >= s->MeshCount)
            return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: GpuBlasTriangle index out of range");
    }
    for (uint64_t i = 0; i < s->MeshCount; i++)
        if (s->Meshes[i].MaterialId < 0 || (uint64_t)s->Meshes[i].MaterialId >= s->MaterialCount)
            return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: GpuMesh.MaterialId out of range");
    if (const char* terr = idk_validate_textures(s)) {
        ctx->lastError = std::string("idkvx_set_scene: ") + terr;
        return strstr(terr, "not supported") ? IDKPT_ERR_UNSUPPORTED : IDKPT_ERR_INVALID_ARGUMENT;
    }
    int rc;
    if ((rc = vupload(ctx, &ctx->dPositions, s->VertexPositions, s->VertexPositionCount * sizeof(PackedVec3)))) return rc;
    if ((rc = vupload(ctx, &ctx->dVertices, s->Vertices, s->VertexCount * sizeof(GpuVertex)))) return rc;
    if ((rc = vupload(ctx, &ctx->dTris, s->BlasTriangles, s->BlasTriangleCount * sizeof(GpuBlasTriangle)))) return rc;
    if ((rc = vupload(ctx, &ctx->dDescs, s->BlasDescs, s->BlasDescCount * sizeof(GpuBlasDesc)))) return rc;
    if ((rc = vupload(ctx, &ctx->dInstances, s->BlasInstances, s->BlasInstanceCount * sizeof(GpuBlasInstance)))) return rc;
    if ((rc = vupload(ctx, &ctx->dXforms, s->MeshTransforms, s->MeshTransformCount * sizeof(GpuMeshTransform)))) return rc;
    if ((rc = vupload(ctx, &ctx->dMeshes, s->Meshes, s->MeshCount * sizeof(GpuMesh)))) return rc;
    if ((rc = vupload(ctx, &ctx->dMaterials, s->Materials, s->MaterialCount * sizeof(GpuMaterial)))) return rc;
    if ((rc = vupload(ctx, &ctx->dLights, s->Lights, s->LightCount * sizeof(GpuLight)))) return rc;
    {   // material textures (BaseColor / Emissive are the slots the voxeliser's fragment stage uses)
        const std::vector<size_t> off = idk_texture_offsets(s);
        std::vector<TexRec> recs;
        if (ctx->dTexPixels) { cudaFree(ctx->dTexPixels); ctx->dTexPixels = nullptr; }
        VCK(cudaMalloc(&ctx->dTexPixels, std::max<size_t>(off[s->TextureCount], 16)));
        VCK(idk_upload_texture_table(s->Textures, s->TextureCount, off, ctx->dTexPixels, ctx->stream, recs));
        if ((rc = vupload(ctx, &ctx->dTexRecs, recs.data(), recs.size() * sizeof(TexRec)))) return rc;
        float lut[256];
        idk_srgb_lut(lut);
        if ((rc = vupload(ctx, &ctx->dSrgbLut, lut, sizeof(lut)))) return rc;
        VCK(cudaStreamSynchronize(ctx->stream));   // packed / recs / lut are locals
    }
    size_t maxTris = 0;
    ctx->hostDescs.assign(s->BlasDescs, s->BlasDescs + s->BlasDescCount);
    ctx->hostInstances.assign(s->BlasInstances, s->BlasInstances + s->BlasInstanceCount);
    for (const GpuBlasInstance& bi : ctx->hostInstances) maxTris += (size_t)ctx->hostDescs[bi.BlasId].TriangleCount;
    if (ctx->dQueue) { cudaFree(ctx->dQueue); ctx->dQueue = nullptr; }
    ctx->queueCapacity = maxTris * 2 + (1u << 20);   // (triangle, tile) work items of large triangles
    VCK(cudaMalloc(&ctx->dQueue, ctx->queueCapacity * sizeof(uint4)));
    VxScene& sc = ctx->sc;
    sc.positions = (const float*)ctx->dPositions;
    sc.vertices = (const uint4*)ctx->dVertices;
    sc.blasTris = (const int4*)ctx->dTris;
    sc.descs = (const GpuBlasDesc*)ctx->dDescs;
    sc.instances = (const GpuBlasInstance*)ctx->dInstances;
    sc.xforms = (const float4*)ctx->dXforms;
    sc.meshes = (const GpuMesh*)ctx->dMeshes;
    sc.materials = (const GpuMaterial*)ctx->dMaterials;
    sc.lights = (const GpuLight*)ctx->dLights;
    sc.textures = (const TexRec*)ctx->dTexRecs;
    sc.srgbLut = (const float*)ctx->dSrgbLut;
    sc.lightCount = (uint32_t)s->LightCount;
    ctx->counts = *s;
    ctx->shadowedLights = shadowed;
    VCK(cudaStreamSynchronize(ctx->stream));
    ctx->haveScene = true;
    return IDKPT_OK;
}

IDKPT_API int idkvx_voxelize(IdkVxCtx* ctx, IdkVxStats* stats) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (!ctx->haveScene) return vfail(ctx, IDKPT_ERR_NO_SCENE, "idkvx_voxelize: idkvx_set_scene has not been called");
    // fragment.glsl:55-58: lights with PointShadowIndex >= 0 are multiplied by Visibility(), a PCF lookup into the shadow cube
    // map the rasteriser renders. Without a rasteriser the same question -- is the (2 % biased) sample point visible from the
    // light -- is answered by an any-hit shadow ray through the path tracer's BVH (idkvx_set_shadow_tracer).
    size_t shadowSmem = 0;
    ctx->sc.occValid = 0;
    if (ctx->shadowedLights) {
        IdkPtCtx* pt = ctx->shadowTracer;
        if (!pt || !pt->haveScene || pt->device != ctx->device)
            return vfail(ctx, IDKPT_ERR_UNSUPPORTED, "idkvx_voxelize: the scene has point-shadowed lights (PointShadowIndex >= 0): give the voxeliser a path-tracer context "
                                                     "with the same scene on the same device (idkvx_set_shadow_tracer) to trace their visibility");
        if (pt->asyncPending) { cudaSetDevice(pt->device); drain(pt); }
        ctx->sc.occ = pt->sc;
        ctx->sc.occValid = 1;
        shadowSmem = pt->stackBytes;
        VCK(cudaFuncSetAttribute(k_vx_voxelize_small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shadowSmem));
        VCK(cudaFuncSetAttribute(k_vx_voxelize_large, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shadowSmem));
    }
    VCK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    cudaEvent_t ev[4];
    for (auto& e : ev) VCK(cudaEventCreate(&e));
    uint32_t launches = 0;
    VCK(cudaEventRecord(ev[0], ctx->stream));
    // ClearTextures (Clear/compute.glsl): level 0 back to zero
    VCK(cudaMemsetAsync(ctx->grid.level[0], 0, ctx->levelTexels[0] * 8, ctx->stream));
    VCK(cudaMemsetAsync(ctx->dQueueCount, 0, 16, ctx->stream));
    VCK(cudaMemsetAsync(ctx->dCounters, 0, 16, ctx->stream));
    VCK(cudaEventRecord(ev[1], ctx->stream));
    for (size_t i = 0; i < ctx->hostInstances.size(); i++) {
        const GpuBlasDesc& d = ctx->hostDescs[ctx->hostInstances[i].BlasId];
        if (d.TriangleCount <= 0) continue;
        VxVoxelizeArgs a;
        a.sc = ctx->sc; a.g = ctx->grid; a.instance = (uint32_t)i;
        a.triFirst = (uint32_t)d.TriangleOffset; a.triCount = (uint32_t)d.TriangleCount;
        a.queue = (uint4*)ctx->dQueue; a.queueCount = (uint32_t*)ctx->dQueueCount; a.queueCapacity = (uint32_t)ctx->queueCapacity;
        a.fragments = (unsigned long long*)ctx->dCounters;
        k_vx_voxelize_small<<<(a.triCount + 255) / 256, 256, shadowSmem, ctx->stream>>>(a);
        launches++;
    }
    k_vx_voxelize_large<<<ctx->smCount * 8, 256, shadowSmem, ctx->stream>>>(ctx->sc, ctx->grid, (const uint4*)ctx->dQueue, (const uint32_t*)ctx->dQueueCount,
                                                                     (uint32_t)ctx->queueCapacity, (unsigned long long*)ctx->dCounters);
    launches++;
    VCK(cudaEventRecord(ev[2], ctx->stream));
    for (int l = 1; l < (ctx->slabMode ? 1 : ctx->grid.levels); l++) {
        const size_t n = ctx->levelTexels[l];
        const int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)ctx->smCount * 16);
        k_vx_mipmap<<<blocks, 256, 0, ctx->stream>>>(ctx->grid, l);
        launches++;
    }
    VCK(cudaEventRecord(ev[3], ctx->stream));
    VCK(cudaGetLastError());
    cudaError_t se = cudaStreamSynchronize(ctx->stream);
    if (se != cudaSuccess) { ctx->lastError = std::string("idkvx_voxelize: kernel execution failed: ") + cudaGetErrorString(se); return IDKPT_ERR_CUDA; }
    if (stats) {
        cudaEventElapsedTime(&stats->ClearMs, ev[0], ev[1]);
        cudaEventElapsedTime(&stats->VoxelizeMs, ev[1], ev[2]);
        cudaEventElapsedTime(&stats->MipmapMs, ev[2], ev[3]);
        unsigned long long f = 0;
        VCK(cudaMemcpy(&f, ctx->dCounters, 8, cudaMemcpyDeviceToHost));
        stats->Fragments = f;
        stats->KernelLaunches = launches;
    }
    for (auto& e : ev) cudaEventDestroy(e);
    return IDKPT_OK;
}

// ---- multi-GPU (SURVEY 8e): voxelise by z-slab, all-gather the slabs, then build the mip chain on every rank -------------------
IDKPT_API int idkvx_set_slab(IdkVxCtx* ctx, int32_t z0, int32_t z1) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    const int d = ctx->grid.sz[0];
    if (z0 < 0 || z1 > d || z0 >= z1) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_slab: need 0 <= z0 < z1 <= depth");
    ctx->grid.z0 = z0; ctx->grid.z1 = z1;
    ctx->slabMode = !(z0 == 0 && z1 == d);
    return IDKPT_OK;
}

IDKPT_API int idkvx_level_device_ptr(IdkVxCtx* ctx, int32_t level, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_level_device_ptr: null argument");
    if (level < 0 || level >= ctx->grid.levels) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_level_device_ptr: level out of range");
    *devPtr = ctx->grid.level[level];
    if (bytes) *bytes = ctx->levelTexels[level] * 8;
    return IDKPT_OK;
}

IDKPT_API int idkvx_mipmap(IdkVxCtx* ctx, IdkVxStats* stats) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    VCK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    cudaEvent_t e0, e1;
    VCK(cudaEventCreate(&e0)); VCK(cudaEventCreate(&e1));
    cudaEventRecord(e0, ctx->stream);
    uint32_t launches = 0;
    for (int l = 1; l < ctx->grid.levels; l++) {
        const size_t n = ctx->levelTexels[l];
        k_vx_mipmap<<<(int)std::min<size_t>((n + 255) / 256, (size_t)ctx->smCount * 16), 256, 0, ctx->stream>>>(ctx->grid, l);
        launches++;
    }
    cudaEventRecord(e1, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess && stats) { cudaEventElapsedTime(&stats->MipmapMs, e0, e1); stats->KernelLaunches = launches; }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (e != cudaSuccess) { ctx->lastError = std::string("idkvx_mipmap: ") + cudaGetErrorString(e); return IDKPT_ERR_CUDA; }
    return IDKPT_OK;
}

IDKPT_API int idkvx_set_shadow_tracer(IdkVxCtx* ctx, IdkPtCtx* pathTracer) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    ctx->shadowTracer = pathTracer;
    return IDKPT_OK;
}

IDKPT_API int idkvx_read_level(IdkVxCtx* ctx, int32_t level, void* dst, uint64_t bytes) {
    if (!ctx || !dst) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_read_level: null argument");
    if (level < 0 || level >= ctx->grid.levels) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_read_level: level out of range");
    if (bytes < ctx->levelTexels[level] * 8) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_read_level: buffer too small");
    VCK(cudaSetDevice(ctx->device));
    VCK(cudaMemcpyAsync(dst, ctx->grid.level[level], ctx->levelTexels[level] * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VCK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

IDKPT_API int idkvx_cone_trace_rows(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const float* depth,
                                    const float* normalRG, const float* metallicRoughness, int32_t width, int32_t fullHeight,
                                    int32_t rowFirst, int32_t height, const float skyColor[3], float* out, IdkVxStats* stats);

IDKPT_API int idkvx_cone_trace(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const float* depth,
                               const float* normalRG, const float* metallicRoughness, int32_t width, int32_t height,
                               const float skyColor[3], float* out, IdkVxStats* stats) {
    return idkvx_cone_trace_rows(ctx, frame, st, depth, normalRG, metallicRoughness, width, height, 0, height, skyColor, out, stats);
}

// Screen-tiled cone tracing (multi-GPU: the grid is replicated, every rank traces its rows): the arrays hold `height` rows starting
// at row `rowFirst` of a G-buffer that is `fullHeight` rows tall; pixel coordinates (noise, NDC) are those of the full image.
IDKPT_API int idkvx_cone_trace_rows(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const float* depth,
                                    const float* normalRG, const float* metallicRoughness, int32_t width, int32_t fullHeight,
                                    int32_t rowFirst, int32_t height, const float skyColor[3], float* out, IdkVxStats* stats) {
    if (!ctx || !frame || !st || !depth || !normalRG || !metallicRoughness || !skyColor || !out) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace: null argument");
    if (width < 1 || height < 1 || width > 16384 || fullHeight > 16384 || rowFirst < 0 || rowFirst + height > fullHeight) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace: invalid image size / row range");
    if (st->MaxSamples < 1 || st->MaxSamples > 64) return vfail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace: MaxSamples out of range");
    VCK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    const size_t n = (size_t)width * height;
    void *dDepth = nullptr, *dN = nullptr, *dMR = nullptr, *dOut = nullptr;
    int rc = IDKPT_OK;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    do {
        if (cudaMalloc(&dDepth, n * 4) != cudaSuccess || cudaMalloc(&dN, n * 8) != cudaSuccess || cudaMalloc(&dMR, n * 8) != cudaSuccess || cudaMalloc(&dOut, n * 16) != cudaSuccess) {
            rc = vfail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkvx_cone_trace: device allocation failed");
            break;
        }
        cudaMemcpyAsync(dDepth, depth, n * 4, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(dN, normalRG, n * 8, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(dMR, metallicRoughness, n * 8, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemsetAsync(ctx->dCounters, 0, 16, ctx->stream);
        VxConeArgs a;
        a.g = ctx->grid;
        memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
        memcpy(a.viewPos, frame->ViewPos, sizeof(a.viewPos));
        a.maxSamples = st->MaxSamples; a.stepMultiplier = st->StepMultiplier; a.giBoost = st->GIBoost; a.giSkyBoxBoost = st->GISkyBoxBoost;
        a.normalRayOffset = st->NormalRayOffset; a.noiseIndex = st->NoiseIndex;
        for (int i = 0; i < 3; i++) a.sky[i] = skyColor[i];
        a.depth = (const float*)dDepth; a.normalRG = (const float2*)dN; a.metalRough = (const float2*)dMR; a.out = (float4*)dOut;
        a.width = width; a.height = height; a.fullHeight = fullHeight; a.rowFirst = rowFirst; a.steps = (unsigned long long*)ctx->dCounters;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0, ctx->stream);
        k_vx_cone_trace<<<dim3((width + 7) / 8, (height + 7) / 8), dim3(8, 8), 0, ctx->stream>>>(a);
        cudaEventRecord(e1, ctx->stream);
        cudaMemcpyAsync(out, dOut, n * 16, cudaMemcpyDeviceToHost, ctx->stream);
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { ctx->lastError = std::string("idkvx_cone_trace: ") + cudaGetErrorString(e); rc = IDKPT_ERR_CUDA; break; }
        if (stats) {
            cudaEventElapsedTime(&stats->ConeTraceMs, e0, e1);
            unsigned long long s = 0;
            cudaMemcpy(&s, ctx->dCounters, 8, cudaMemcpyDeviceToHost);
            stats->ConeSteps = s;
            stats->KernelLaunches = 1;
        }
    } while (0);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    cudaFree(dDepth); cudaFree(dN); cudaFree(dMR); cudaFree(dOut);
    return rc;
}

} // extern "C"
