// libidkpt, VXGI part: C ABI of include/idkvx.h over the kernels of idk_vxgi.cuh. Included at the end of idkpt.cu (one
// translation unit), so that the voxeliser can trace shadow rays through the path tracer's device scene (idk_shadows.cuh).
// Host sequencing mirrors Voxelizer.Render (IDKEngine/Source/Render/VXGI/Voxelizer/Voxelizer.cs:109-228:
// ClearTextures -> Voxelize -> Mipmap levels 1..n-1) and ConeTracer.Compute (ConeTracing/ConeTracer.cs:37-50). It uses
// idkpt.cu's context base, buffers and helpers (CK, fail, ensure, upload, run_timed, validate_scene).
#include "../../include/idkvx.h"
#include "idk_vxgi.cuh"
#pragma once

struct IdkVxCtx : IdkCtxBase {
    static inline thread_local std::string createError;   // last failed idkvx_create (idkvx_last_error(NULL))
    VxGridDev grid = {};
    DevBuf gridMem;
    size_t levelTexels[IDKVX_MAX_LEVELS] = {};
    bool haveScene = false;               // idkvx_set_scene: the context holds its own copy of a scene
    // idkvx_set_scene_from: no copy; each idkvx_voxelize reads this path tracer's device scene as it stands (bind_source)
    IdkPtCtx* source = nullptr;
    uint64_t sourceGeneration = 0;        // source->sceneGeneration that queueCapacity was sized for
    VxScene sc = {};
    IdkPtSceneDesc counts = {};
    std::vector<GpuBlasDesc> hostDescs;
    std::vector<GpuBlasInstance> hostInstances;
    DevBuf positions, vertices, tris, descs, instances, xforms, meshes, materials, lights;
    TextureTable tex;
    DevBuf queue, queueCount, counters;
    size_t queueCapacity = 0;
    DevBuf stage;                         // the cone trace's host G-buffer arrays (stage_inputs_into), kept between calls
    RasterImage cone;                     // the rgba32f image of the last successful cone trace (width x rows traced)
    bool slabMode = false;                // idkvx_set_slab: voxelise one z-slab, no mip chain (the host all-gathers the slabs first)
    IdkPtCtx* shadowTracer = nullptr;     // idkvx_set_shadow_tracer: visibility of point-shadowed lights by shadow rays through this scene
    IdkPtCtx* shadowMaps = nullptr;       // idkvx_set_shadow_maps: visibility by the PCF lookup into this context's point-shadow cube maps
    bool shadowedLights = false;
    int32_t maxPointShadowIndex = -1;     // largest PointShadowIndex of the scene's lights
    // the grid holds a whole voxelisation with its mip chain (idkpt_transparency's cone trace reads it): set by a successful
    // idkvx_voxelize of the whole grid, or by idkvx_mipmap after a slab voxelisation (the multi-GPU flow all-gathers the slabs in
    // between); cleared by idkvx_set_grid, idkvx_set_scene, idkvx_set_scene_from and idkvx_set_slab
    bool voxelized = false;
    bool slabVoxelized = false;           // idkvx_voxelize ran in slab mode since the grid last changed
    bool conservative = false;            // idkvx_set_conservative_rasterization: coverage rule of the next idkvx_voxelize
    DevBuf debugImage, debugMask;         // idkvx_debug_render: the rgba32f image and the level-0 brick masks
    size_t debugBytes = 0;                // bytes of the last successful idkvx_debug_render's image (0: none yet)
};

static void set_grid_bounds(IdkVxCtx* ctx, const float* mn, const float* mx) {
    // Voxelizer.GridMin / GridMax setters keep max >= min + 0.1 (Voxelizer.cs:16-33)
    for (int i = 0; i < 3; i++) {
        ctx->grid.gmin[i] = mn[i];
        ctx->grid.gmax[i] = std::max(mx[i], mn[i] + 0.1f);
    }
}

static int allocate_grid(IdkVxCtx* ctx, size_t bytes) {
    if (ensure(ctx->gridMem, bytes) != cudaSuccess) return fail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkvx_create: voxel grid allocation failed");
    CK(cudaMemsetAsync(ctx->gridMem.p, 0, bytes, ctx->stream));   // ResultVoxels.Fill(0), Voxelizer.cs:258
    CK(ensure(ctx->queueCount, 16));
    CK(ensure(ctx->counters, 16));
    return IDKPT_OK;
}

// Removes the voxeliser from its path tracer's list of bound voxelisers (idkvx_set_scene_from).
static void unbind_source(IdkVxCtx* ctx) {
    if (!ctx->source) return;
    std::vector<IdkVxCtx*>& v = ctx->source->boundVoxelizers;
    v.erase(std::remove(v.begin(), v.end(), ctx), v.end());
    ctx->source = nullptr;
}

static void unbind_voxelizers(IdkPtCtx* pt) {
    for (IdkVxCtx* vx : pt->boundVoxelizers) vx->source = nullptr;
    pt->boundVoxelizers.clear();
}

// The scene arrays idkvx_set_scene copies, the texture table included.
static void release_scene(IdkVxCtx* ctx) {
    for (DevBuf* b : {&ctx->positions, &ctx->vertices, &ctx->tris, &ctx->descs, &ctx->instances, &ctx->xforms, &ctx->meshes,
                      &ctx->materials, &ctx->lights})
        release(*b);
    release_textures(ctx->tex);
}

// Work items of the large-triangle queue for a draw list: (triangle, tile) items of large triangles.
static int size_queue(IdkVxCtx* ctx, const std::vector<GpuBlasDesc>& descs, const std::vector<GpuBlasInstance>& instances) {
    size_t maxTris = 0;
    for (const GpuBlasInstance& bi : instances) maxTris += (size_t)descs[bi.BlasId].TriangleCount;
    ctx->queueCapacity = maxTris * 2 + (1u << 20);
    CK(ensure(ctx->queue, ctx->queueCapacity * sizeof(uint4)));
    return IDKPT_OK;
}

// idkvx_voxelize of a bound voxeliser: VxScene's pointers, the light count and the shadowed-light bound from the path tracer's
// scene as it stands now. Every path-tracer call that writes these arrays (idkpt_set_scene, idkpt_update_range,
// idkpt_set_textures, idkpt_skin_vertices, idkpt_blas_refit, idkpt_tlas_build) ends in a synchronise of its stream, and so
// does idkvx_voxelize; samples idkpt_compute has queued only read them. So the voxelisation reads a finished scene without
// waiting for the path tracer, and a pointer is never kept past the call that could reallocate it.
static int bind_source(IdkVxCtx* ctx) {
    IdkPtCtx* pt = ctx->source;
    if (!pt->haveScene)
        return fail(ctx, IDKPT_ERR_NO_SCENE, "idkvx_voxelize: the path-tracer context bound with idkvx_set_scene_from has no scene (idkpt_set_scene)");
    VxScene& sc = ctx->sc;
    sc.positions = (const float*)pt->positions.p;
    sc.vertices = (const uint4*)pt->vertices.p;
    sc.blasTris = (const int4*)pt->blasTris.p;
    sc.descs = (const GpuBlasDesc*)pt->descs.p;
    sc.instances = (const GpuBlasInstance*)pt->instances.p;
    sc.xforms = (const float4*)pt->xforms.p;
    sc.meshes = (const GpuMesh*)pt->meshes.p;
    sc.materials = (const GpuMaterial*)pt->materials.p;
    sc.lights = (const GpuLight*)pt->lights.p;
    sc.textures = (const TexRec*)pt->tex.recs.p;
    sc.srgbLut = (const float*)pt->tex.srgbLut.p;
    sc.lightCount = (uint32_t)pt->counts.LightCount;
    ctx->maxPointShadowIndex = -1;   // idkpt_update_range(LIGHTS) may have changed it
    for (const GpuLight& L : pt->hostLights) ctx->maxPointShadowIndex = std::max(ctx->maxPointShadowIndex, L.PointShadowIndex);
    ctx->shadowedLights = ctx->maxPointShadowIndex >= 0;
    if (ctx->sourceGeneration != pt->sceneGeneration) {
        CK(cudaSetDevice(ctx->device));
        if (int rc = size_queue(ctx, pt->hostDescs, pt->hostInstances)) return rc;
        ctx->sourceGeneration = pt->sceneGeneration;
    }
    return IDKPT_OK;
}

// Voxelizer.Mipmap: levels 1 .. n-1, each from the level below. Returns the number of launches.
static uint32_t launch_mips(IdkVxCtx* ctx) {
    for (int l = 1; l < ctx->grid.levels; l++) {
        const size_t n = ctx->levelTexels[l];
        k_vx_mipmap<<<(int)std::min<size_t>((n + 255) / 256, (size_t)ctx->smCount * 16), 256, 0, ctx->stream>>>(ctx->grid, l);
    }
    return (uint32_t)(ctx->grid.levels - 1);
}

extern "C" {

IDKPT_API const char* idkvx_last_error(IdkVxCtx* ctx) { return ctx ? ctx->lastError.c_str() : IdkVxCtx::createError.c_str(); }

IDKPT_API int idkvx_create(const IdkVxCreateInfo* ci, IdkVxCtx** out) {
    if (!ci || !out) return fail<IdkVxCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_create: null argument");
    *out = nullptr;
    if (ci->Width < 1 || ci->Height < 1 || ci->Depth < 1 || ci->Width > 2048 || ci->Height > 2048 || ci->Depth > 2048)
        return fail<IdkVxCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_create: invalid grid size");
    int deviceCount = 0;
    if (cudaGetDeviceCount(&deviceCount) != cudaSuccess || deviceCount == 0)
        return fail<IdkVxCtx>(nullptr, IDKPT_ERR_NO_DEVICE, "idkvx_create: no CUDA device (libidkpt has no CPU fallback)");
    if (ci->Device < 0 || ci->Device >= deviceCount) return fail<IdkVxCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_create: device ordinal out of range");
    if (cudaSetDevice(ci->Device) != cudaSuccess) return fail<IdkVxCtx>(nullptr, IDKPT_ERR_CUDA, "idkvx_create: cudaSetDevice failed");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, ci->Device) != cudaSuccess) return fail<IdkVxCtx>(nullptr, IDKPT_ERR_CUDA, "idkvx_create: cudaGetDeviceProperties failed");
    if (prop.major != 9 || prop.minor != 0) return fail<IdkVxCtx>(nullptr, IDKPT_ERR_NO_DEVICE, "idkvx_create: libidkpt is built for sm_90a only");
    IdkVxCtx* ctx = new IdkVxCtx();
    ctx->device = ci->Device;
    ctx->smCount = prop.multiProcessorCount;
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
    int rc = create_stream(ctx);
    if (rc == IDKPT_OK) rc = allocate_grid(ctx, total * 8);
    if (rc != IDKPT_OK) {
        IdkVxCtx::createError = ctx->lastError;
        idkvx_destroy(ctx);
        return rc;
    }
    size_t off = 0;
    for (int l = 0; l < levels; l++) { ctx->grid.level[l] = (unsigned long long*)ctx->gridMem.p + off; off += ctx->levelTexels[l]; }
    set_grid_bounds(ctx, ci->GridMin, ci->GridMax);
    *out = ctx;
    return IDKPT_OK;
}

IDKPT_API void idkvx_destroy(IdkVxCtx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    unbind_source(ctx);
    release_scene(ctx);
    DevBuf* all[] = {&ctx->gridMem, &ctx->queue, &ctx->queueCount, &ctx->counters, &ctx->stage, &ctx->cone.buf[0], &ctx->debugImage, &ctx->debugMask};
    for (DevBuf* b : all) release(*b);
    destroy_stream(ctx);
    delete ctx;
}

IDKPT_API int32_t idkvx_level_count(IdkVxCtx* ctx) { return ctx ? ctx->grid.levels : 0; }

IDKPT_API int idkvx_set_grid(IdkVxCtx* ctx, const float gridMin[3], const float gridMax[3]) {
    if (!ctx || !gridMin || !gridMax) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_grid: null argument");
    set_grid_bounds(ctx, gridMin, gridMax);
    ctx->voxelized = ctx->slabVoxelized = false;
    return IDKPT_OK;
}

IDKPT_API int idkvx_set_scene(IdkVxCtx* ctx, const IdkPtSceneDesc* s) {
    if (!ctx || !s) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_scene: null argument");
    CK(cudaSetDevice(ctx->device));
    if (int rc = validate_scene(ctx, "idkvx_set_scene", s)) return rc;
    unbind_source(ctx);
    ctx->voxelized = ctx->slabVoxelized = false;
    ctx->haveScene = false;   // the device arrays are overwritten from here on: a failure below leaves no scene
    ctx->shadowedLights = false;
    ctx->maxPointShadowIndex = -1;
    for (uint64_t i = 0; i < s->LightCount; i++) ctx->maxPointShadowIndex = std::max(ctx->maxPointShadowIndex, s->Lights[i].PointShadowIndex);
    ctx->shadowedLights = ctx->maxPointShadowIndex >= 0;
    int rc;
    if ((rc = upload(ctx, ctx->positions, s->VertexPositions, s->VertexPositionCount * sizeof(PackedVec3)))) return rc;
    if ((rc = upload(ctx, ctx->vertices, s->Vertices, s->VertexCount * sizeof(GpuVertex)))) return rc;
    if ((rc = upload(ctx, ctx->tris, s->BlasTriangles, s->BlasTriangleCount * sizeof(GpuBlasTriangle)))) return rc;
    if ((rc = upload(ctx, ctx->descs, s->BlasDescs, s->BlasDescCount * sizeof(GpuBlasDesc)))) return rc;
    if ((rc = upload(ctx, ctx->instances, s->BlasInstances, s->BlasInstanceCount * sizeof(GpuBlasInstance)))) return rc;
    if ((rc = upload(ctx, ctx->xforms, s->MeshTransforms, s->MeshTransformCount * sizeof(GpuMeshTransform)))) return rc;
    if ((rc = upload(ctx, ctx->meshes, s->Meshes, s->MeshCount * sizeof(GpuMesh)))) return rc;
    if ((rc = upload(ctx, ctx->materials, s->Materials, s->MaterialCount * sizeof(GpuMaterial)))) return rc;
    if ((rc = upload(ctx, ctx->lights, s->Lights, s->LightCount * sizeof(GpuLight)))) return rc;
    // material textures (BaseColor / Emissive are the slots the voxeliser's fragment stage uses)
    if ((rc = upload_textures(ctx, ctx->tex, s->Textures, s->TextureCount))) return rc;
    ctx->hostDescs.assign(s->BlasDescs, s->BlasDescs + s->BlasDescCount);
    ctx->hostInstances.assign(s->BlasInstances, s->BlasInstances + s->BlasInstanceCount);
    if ((rc = size_queue(ctx, ctx->hostDescs, ctx->hostInstances))) return rc;
    VxScene& sc = ctx->sc;
    sc.positions = (const float*)ctx->positions.p;
    sc.vertices = (const uint4*)ctx->vertices.p;
    sc.blasTris = (const int4*)ctx->tris.p;
    sc.descs = (const GpuBlasDesc*)ctx->descs.p;
    sc.instances = (const GpuBlasInstance*)ctx->instances.p;
    sc.xforms = (const float4*)ctx->xforms.p;
    sc.meshes = (const GpuMesh*)ctx->meshes.p;
    sc.materials = (const GpuMaterial*)ctx->materials.p;
    sc.lights = (const GpuLight*)ctx->lights.p;
    sc.textures = (const TexRec*)ctx->tex.recs.p;
    sc.srgbLut = (const float*)ctx->tex.srgbLut.p;
    sc.lightCount = (uint32_t)s->LightCount;
    ctx->counts = *s;
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->haveScene = true;
    return IDKPT_OK;
}

IDKPT_API int idkvx_set_scene_from(IdkVxCtx* ctx, IdkPtCtx* pathTracer) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (pathTracer && pathTracer->device != ctx->device)
        return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkvx_set_scene_from: the path-tracer context is on another device");
    CK(cudaSetDevice(ctx->device));
    unbind_source(ctx);
    release_scene(ctx);
    ctx->haveScene = false;
    ctx->hostDescs.clear();
    ctx->hostInstances.clear();
    ctx->counts = {};
    ctx->shadowedLights = false;
    ctx->maxPointShadowIndex = -1;
    ctx->voxelized = ctx->slabVoxelized = false;
    if (pathTracer) {
        ctx->source = pathTracer;
        ctx->sourceGeneration = pathTracer->sceneGeneration - 1;   // sizes the work queue at the first voxelisation
        pathTracer->boundVoxelizers.push_back(ctx);
    }
    return IDKPT_OK;
}

IDKPT_API int idkvx_voxelize(IdkVxCtx* ctx, IdkVxStats* stats) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (ctx->source) {
        if (int rc = bind_source(ctx)) return rc;
    } else if (!ctx->haveScene) {
        return fail(ctx, IDKPT_ERR_NO_SCENE, "idkvx_voxelize: idkvx_set_scene has not been called (or idkvx_set_scene_from's path-tracer "
                                             "context was unbound or destroyed)");
    }
    const std::vector<GpuBlasDesc>& descs = ctx->source ? ctx->source->hostDescs : ctx->hostDescs;
    const std::vector<GpuBlasInstance>& instances = ctx->source ? ctx->source->hostInstances : ctx->hostInstances;
    // fragment.glsl:55-58: lights with PointShadowIndex >= 0 are multiplied by Visibility(), a PCF lookup into the shadow cube
    // map. With shadow maps attached that lookup runs on the path tracer's traced cube maps (idkvx_set_shadow_maps); otherwise
    // the same question -- is the (2 % biased) sample point visible from the light -- is answered by an any-hit shadow ray
    // through the path tracer's BVH (idkvx_set_shadow_tracer).
    // Voxelizer.IsConservativeRasterization picks the coverage rule: pixel centres, or every pixel the triangle touches
    void (*const small)(VxVoxelizeArgs) = ctx->conservative ? k_vx_voxelize_small<true> : k_vx_voxelize_small<false>;
    void (*const large)(VxScene, VxGridDev, const uint4*, const uint32_t*, uint32_t, unsigned long long*) =
        ctx->conservative ? k_vx_voxelize_large<true> : k_vx_voxelize_large<false>;
    size_t shadowSmem = 0;
    ctx->sc.occValid = 0;
    ctx->sc.psmValid = 0;
    if (ctx->shadowedLights && ctx->shadowMaps) {
        IdkPtCtx* pt = ctx->shadowMaps;
        if (pt->device != ctx->device) return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkvx_voxelize: the shadow-map context is on another device");
        if ((size_t)ctx->maxPointShadowIndex >= pt->pointShadowRecs.size())
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_voxelize: a light's PointShadowIndex is not below the shadow-map context's shadow count (idkpt_set_point_shadows)");
        ctx->sc.psm.shadows = (const PointShadowDev*)pt->pointShadowDev.p;
        ctx->sc.psm.texels = (const uint16_t*)pt->pointShadowMaps.p;
        ctx->sc.psm.count = (uint32_t)pt->pointShadowRecs.size();
        ctx->sc.psmValid = 1;
    } else if (ctx->shadowedLights) {
        IdkPtCtx* pt = ctx->shadowTracer;
        if (!pt || !pt->haveScene || pt->device != ctx->device)
            return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkvx_voxelize: the scene has point-shadowed lights (PointShadowIndex >= 0): give the voxeliser a path-tracer context "
                                                     "with the same scene on the same device (idkvx_set_shadow_tracer) to trace their visibility");
        if (pt->asyncPending) { cudaSetDevice(pt->device); drain(pt); }
        ctx->sc.occ = pt->sc;
        ctx->sc.occValid = 1;
        shadowSmem = pt->stackBytes;
        CK(cudaFuncSetAttribute(small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shadowSmem));
        CK(cudaFuncSetAttribute(large, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shadowSmem));
    }
    CK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    uint32_t launches = 0;
    const int rc = run_timed(ctx, "idkvx_voxelize", nullptr, [&]() -> int {
        // ClearTextures (Clear/compute.glsl): level 0 back to zero
        CK(cudaMemsetAsync(ctx->grid.level[0], 0, ctx->levelTexels[0] * 8, ctx->stream));
        CK(cudaMemsetAsync(ctx->queueCount.p, 0, 16, ctx->stream));
        CK(cudaMemsetAsync(ctx->counters.p, 0, 16, ctx->stream));
        CK(cudaEventRecord(ctx->timing[2], ctx->stream));
        for (size_t i = 0; i < instances.size(); i++) {
            const GpuBlasDesc& d = descs[instances[i].BlasId];
            if (d.TriangleCount <= 0) continue;
            VxVoxelizeArgs a;
            a.sc = ctx->sc; a.g = ctx->grid; a.instance = (uint32_t)i;
            a.triFirst = (uint32_t)d.TriangleOffset; a.triCount = (uint32_t)d.TriangleCount;
            a.queue = (uint4*)ctx->queue.p; a.queueCount = (uint32_t*)ctx->queueCount.p; a.queueCapacity = (uint32_t)ctx->queueCapacity;
            a.fragments = (unsigned long long*)ctx->counters.p;
            small<<<(a.triCount + 255) / 256, 256, shadowSmem, ctx->stream>>>(a);
            launches++;
        }
        large<<<ctx->smCount * 8, 256, shadowSmem, ctx->stream>>>(ctx->sc, ctx->grid, (const uint4*)ctx->queue.p, (const uint32_t*)ctx->queueCount.p,
                                                           (uint32_t)ctx->queueCapacity, (unsigned long long*)ctx->counters.p);
        launches++;
        CK(cudaEventRecord(ctx->timing[3], ctx->stream));
        if (!ctx->slabMode) launches += launch_mips(ctx);
        return IDKPT_OK;
    });
    if (rc) return rc;
    ctx->voxelized = !ctx->slabMode;
    ctx->slabVoxelized = ctx->slabMode;
    if (stats) {
        CK(cudaEventElapsedTime(&stats->ClearMs, ctx->timing[0], ctx->timing[2]));
        CK(cudaEventElapsedTime(&stats->VoxelizeMs, ctx->timing[2], ctx->timing[3]));
        CK(cudaEventElapsedTime(&stats->MipmapMs, ctx->timing[3], ctx->timing[1]));
        unsigned long long f = 0;
        CK(cudaMemcpy(&f, ctx->counters.p, 8, cudaMemcpyDeviceToHost));
        stats->Fragments = f;
        stats->KernelLaunches = launches;
    }
    return IDKPT_OK;
}

// ---- multi-GPU (SURVEY 8e): voxelise by z-slab, all-gather the slabs, then build the mip chain on every rank -------------------
IDKPT_API int idkvx_set_slab(IdkVxCtx* ctx, int32_t z0, int32_t z1) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    const int d = ctx->grid.sz[0];
    if (z0 < 0 || z1 > d || z0 >= z1) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_slab: need 0 <= z0 < z1 <= depth");
    ctx->grid.z0 = z0; ctx->grid.z1 = z1;
    ctx->voxelized = ctx->slabVoxelized = false;
    ctx->slabMode = !(z0 == 0 && z1 == d);
    return IDKPT_OK;
}

IDKPT_API int idkvx_level_device_ptr(IdkVxCtx* ctx, int32_t level, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_level_device_ptr: null argument");
    if (level < 0 || level >= ctx->grid.levels) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_level_device_ptr: level out of range");
    *devPtr = ctx->grid.level[level];
    if (bytes) *bytes = ctx->levelTexels[level] * 8;
    return IDKPT_OK;
}

IDKPT_API int idkvx_mipmap(IdkVxCtx* ctx, IdkVxStats* stats) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    CK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    uint32_t launches = 0;
    const int rc = run_timed(ctx, "idkvx_mipmap", stats ? &stats->MipmapMs : nullptr, [&]() -> int {
        launches = launch_mips(ctx);
        return IDKPT_OK;
    });
    if (rc == IDKPT_OK && stats) stats->KernelLaunches = launches;
    if (rc == IDKPT_OK && ctx->slabVoxelized) ctx->voxelized = true;
    return rc;
}

IDKPT_API int idkvx_set_conservative_rasterization(IdkVxCtx* ctx, int32_t enable) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (enable != 0 && enable != 1) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_set_conservative_rasterization: enable must be 0 or 1");
    ctx->conservative = enable == 1;   // takes effect at the next idkvx_voxelize; the current grid is left as it is
    return IDKPT_OK;
}

IDKPT_API int idkvx_set_shadow_tracer(IdkVxCtx* ctx, IdkPtCtx* pathTracer) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    ctx->shadowTracer = pathTracer;
    return IDKPT_OK;
}

IDKPT_API int idkvx_set_shadow_maps(IdkVxCtx* ctx, IdkPtCtx* pathTracer) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    ctx->shadowMaps = pathTracer;
    return IDKPT_OK;
}

IDKPT_API int idkvx_read_level(IdkVxCtx* ctx, int32_t level, void* dst, uint64_t bytes) {
    if (!ctx || !dst) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_read_level: null argument");
    if (level < 0 || level >= ctx->grid.levels) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_read_level: level out of range");
    if (bytes < ctx->levelTexels[level] * 8) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_read_level: buffer too small");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(dst, ctx->grid.level[level], ctx->levelTexels[level] * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

// ConeTracer.Compute for every entry point, into ctx->cone: g (Depth, NormalRG and MetallicRoughness, read in place when
// g->OnDevice is 1; its arguments checked by the caller) holds g->Height rows starting at row `rowFirst` of a G-buffer that is
// `fullHeight` rows tall; pixel coordinates (noise, NDC) are those of the full image. out (may be null) gets a copy.
static int cone_trace(IdkVxCtx* ctx, const char* who, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const IdkPtGBuffer* g,
                      int32_t fullHeight, int32_t rowFirst, const float skyColor[3], float* out, IdkVxStats* stats) {
    const int width = g->Width, height = g->Height;
    CK(cudaSetDevice(ctx->device));
    const float* in[3];
    if (int rc = stage_inputs_into(ctx, ctx->stage, who, width, height, g->OnDevice,
                              {attachment(g->Depth, 1), attachment(g->NormalRG, 2), attachment(g->MetallicRoughness, 2)}, in)) return rc;
    if (stats) memset(stats, 0, sizeof(*stats));
    const size_t n = (size_t)width * height;
    ctx->cone.invalidate();        // the image may be reallocated and is overwritten: valid again only when the call succeeds
    if (ensure(ctx->cone.buf[0], n * 16) != cudaSuccess) return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    CK(cudaMemsetAsync(ctx->counters.p, 0, 16, ctx->stream));
    VxConeArgs a;
    a.g = ctx->grid;
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    memcpy(a.viewPos, frame->ViewPos, sizeof(a.viewPos));
    a.maxSamples = st->MaxSamples; a.stepMultiplier = st->StepMultiplier; a.giBoost = st->GIBoost; a.giSkyBoxBoost = st->GISkyBoxBoost;
    a.normalRayOffset = st->NormalRayOffset; a.noiseIndex = st->NoiseIndex;
    for (int i = 0; i < 3; i++) a.sky[i] = skyColor[i];
    a.depth = in[0]; a.normalRG = (const float2*)in[1]; a.metalRough = (const float2*)in[2]; a.out = (float4*)ctx->cone.buf[0].p;
    a.width = width; a.height = height; a.fullHeight = fullHeight; a.rowFirst = rowFirst; a.steps = (unsigned long long*)ctx->counters.p;
    const int rc = run_timed(ctx, who, stats ? &stats->ConeTraceMs : nullptr, [&]() -> int {
        k_vx_cone_trace<<<dim3((width + 7) / 8, (height + 7) / 8), dim3(8, 8), 0, ctx->stream>>>(a);
        return IDKPT_OK;
    }, out, ctx->cone.buf[0].p, out ? n * 16 : 0);
    if (rc) return rc;
    ctx->cone.publish(width, height);
    if (stats) {
        unsigned long long s = 0;
        CK(cudaMemcpy(&s, ctx->counters.p, 8, cudaMemcpyDeviceToHost));
        stats->ConeSteps = s;
        stats->KernelLaunches = 1;
    }
    return IDKPT_OK;
}

IDKPT_API int idkvx_cone_trace(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const float* depth,
                               const float* normalRG, const float* metallicRoughness, int32_t width, int32_t height,
                               const float skyColor[3], float* out, IdkVxStats* stats) {
    return idkvx_cone_trace_rows(ctx, frame, st, depth, normalRG, metallicRoughness, width, height, 0, height, skyColor, out, stats);
}

// Screen-tiled cone tracing (multi-GPU: the grid is replicated, every rank traces its rows) from host arrays of `height` rows.
IDKPT_API int idkvx_cone_trace_rows(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const float* depth,
                                    const float* normalRG, const float* metallicRoughness, int32_t width, int32_t fullHeight,
                                    int32_t rowFirst, int32_t height, const float skyColor[3], float* out, IdkVxStats* stats) {
    if (!ctx || !frame || !st || !depth || !normalRG || !metallicRoughness || !skyColor || !out) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace: null argument");
    if (width < 1 || height < 1 || width > 16384 || fullHeight > 16384 || rowFirst < 0 || rowFirst + height > fullHeight) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace: invalid image size / row range");
    if (st->MaxSamples < 1 || st->MaxSamples > 64) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace: MaxSamples out of range");
    const IdkPtGBuffer g{width, height, 0, depth, normalRG, nullptr, metallicRoughness, nullptr};
    return cone_trace(ctx, "idkvx_cone_trace", frame, st, &g, fullHeight, rowFirst, skyColor, out, stats);
}

IDKPT_API int idkvx_cone_trace_gbuffer(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* st, const IdkPtGBuffer* g,
                                       const float skyColor[3], float* out, IdkVxStats* stats) {
    static const char* who = "idkvx_cone_trace_gbuffer";
    if (!ctx || !frame || !st || !g || !skyColor) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace_gbuffer: null argument");
    if (!g->Depth || !g->NormalRG || !g->MetallicRoughness) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "null argument");
    if (int rc = gbuffer_shape_check(ctx, who, g)) return rc;
    if (st->MaxSamples < 1 || st->MaxSamples > 64) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "MaxSamples outside 1..64");
    return cone_trace(ctx, who, frame, st, g, g->Height, 0, skyColor, out, stats);
}

IDKPT_API int idkvx_cone_trace_device_ptr(IdkVxCtx* ctx, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_cone_trace_device_ptr: null argument");
    if (!ctx->cone.valid()) return fail(ctx, "idkvx_cone_trace_device_ptr", IDKPT_ERR_INVALID_ARGUMENT, "call idkvx_cone_trace_gbuffer first");
    *devPtr = ctx->cone.buf[0].p;
    if (bytes) *bytes = (uint64_t)ctx->cone.w * ctx->cone.h * 16;
    return IDKPT_OK;
}

// Voxelizer.DebugRender (Voxelizer.cs:230-244): the grid as it is now, marched per pixel and blended over the sky of `sky`.
IDKPT_API int idkvx_debug_render(IdkVxCtx* ctx, IdkPtCtx* sky, const GpuPerFrameData* frame, float stepMultiplier, float coneAngle,
                                 int32_t width, int32_t height, float* out, IdkVxStats* stats) {
    static const char* who = "idkvx_debug_render";
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (!sky || !frame) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "null argument");
    if (sky->device != ctx->device) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "the sky's path-tracer context is on another device");
    if (width < 1 || height < 1 || width > 16384 || height > 16384) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "width or height outside 1..16384");
    if (!std::isfinite(coneAngle) || coneAngle < 0.0f || coneAngle > 1.5f) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "cone angle not finite or outside [0, 1.5]");
    if (!std::isfinite(stepMultiplier) || !(stepMultiplier > 0.0f)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "step multiplier not finite or not > 0");
    // every march ends within (|GridMax - GridMin| + voxelMaxLength) / (voxelMinLength * stepMultiplier) steps (DESIGN.md 8f.1k)
    const VxGridDev& g = ctx->grid;
    double diag2 = 0.0, vmin = 0.0, vmax = 0.0;
    for (int i = 0; i < 3; i++) {
        const float e = g.gmax[i] - g.gmin[i];
        const double vs = (double)(e / (float)(i == 0 ? g.sx[0] : (i == 1 ? g.sy[0] : g.sz[0])));
        diag2 += (double)e * (double)e;
        vmin = i == 0 ? vs : std::min(vmin, vs);
        vmax = i == 0 ? vs : std::max(vmax, vs);
    }
    const double bound = (std::sqrt(diag2) + vmax) / (vmin * (double)stepMultiplier);
    if (!(bound <= 65536.0)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "step multiplier too small for the grid: the march would take more than 65536 steps");
    CK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));

    // the skip pays for its mask only where the march reads level 0 alone: at cone angle 0 (DESIGN.md 8f.1k)
    const bool skip = IDKVX_DEBUG_SKIP && coneAngle == 0.0f;
    VxBrickGrid bg;
    bg.nx = (g.sx[0] + 3) >> IDKVX_BRICK_SHIFT; bg.ny = (g.sy[0] + 3) >> IDKVX_BRICK_SHIFT; bg.nz = (g.sz[0] + 3) >> IDKVX_BRICK_SHIFT;
    const uint32_t bricks = (uint32_t)bg.nx * bg.ny * bg.nz;
    bg.words = (bricks + 31) / 32;
    if (skip && ensure(ctx->debugMask, 2 * (size_t)bg.words * 4) != cudaSuccess) return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    // a larger image goes into a fresh allocation that replaces the old one only once the kernel has succeeded
    const size_t n = (size_t)width * height, bytes = n * 16;
    DevBuf fresh;
    if (bytes > ctx->debugImage.bytes && ensure(fresh, bytes) != cudaSuccess) {
        release(fresh);
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    }
    float4* image = (float4*)(fresh.p ? fresh.p : ctx->debugImage.p);
    VxDebugArgs a;
    a.g = g;
    a.bg = bg;
    a.mask = (const uint32_t*)ctx->debugMask.p + bg.words;
    a.sky = sky->sc;
    a.invProjection[0] = frame->InvProjection[0]; a.invProjection[1] = frame->InvProjection[1];
    a.invProjection[2] = frame->InvProjection[4]; a.invProjection[3] = frame->InvProjection[5];
    memcpy(a.invView, frame->InvView, sizeof(a.invView));
    memcpy(a.viewPos, frame->ViewPos, sizeof(a.viewPos));
    a.coneAngle = coneAngle; a.stepMultiplier = stepMultiplier;
    a.out = image;
    a.width = width; a.height = height;
    a.steps = (unsigned long long*)ctx->counters.p;
    uint32_t launches = 0;
    const int rc = run_timed(ctx, who, stats ? &stats->ConeTraceMs : nullptr, [&]() -> int {
        CK(cudaMemsetAsync(ctx->counters.p, 0, 16, ctx->stream));
        if (skip) {
            const unsigned blocks = (unsigned)(((size_t)bg.words * 32 + 255) / 256);
            k_vx_debug_bricks<<<blocks, 256, 0, ctx->stream>>>(g, bg, (uint32_t*)ctx->debugMask.p);
            k_vx_debug_dilate<<<blocks, 256, 0, ctx->stream>>>(bg, (const uint32_t*)ctx->debugMask.p, (uint32_t*)ctx->debugMask.p + bg.words);
            launches += 2;
        }
        (skip ? k_vx_debug_render<true> : k_vx_debug_render<false>)<<<dim3((width + 7) / 8, (height + 7) / 8), dim3(8, 8), 0, ctx->stream>>>(a);
        launches++;
        return IDKPT_OK;
    }, out, image, out ? bytes : 0);
    if (rc) { release(fresh); return rc; }
    if (fresh.p) { release(ctx->debugImage); ctx->debugImage = fresh; }
    ctx->debugBytes = bytes;
    if (stats) {
        unsigned long long s = 0;
        CK(cudaMemcpy(&s, ctx->counters.p, 8, cudaMemcpyDeviceToHost));
        stats->ConeSteps = s;
        stats->KernelLaunches = launches;
    }
    return IDKPT_OK;
}

IDKPT_API int idkvx_debug_device_ptr(IdkVxCtx* ctx, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkvx_debug_device_ptr: null argument");
    *devPtr = ctx->debugBytes ? ctx->debugImage.p : nullptr;
    if (bytes) *bytes = ctx->debugBytes;
    return IDKPT_OK;
}

} // extern "C"
