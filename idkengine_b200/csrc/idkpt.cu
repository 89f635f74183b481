// libidkpt: C ABI (include/idkpt.h) over the sm_90a wavefront kernels (idk_kernels.cuh).
// Host sequencing mirrors PathTracer.Compute(), IDKEngine/Source/Render/PathTracer.cs:214-297, with
// every GL dispatch replaced by a CUDA launch on one stream and no CPU read-back inside the loop
// (alive counts stay on the device, like the reference's indirect dispatch).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include <cmath>

#include "../../include/idkpt.h"
#include "idk_kernels.cuh"
#include "idk_sort.cuh"
#include "idk_shadows.cuh"
#include "idk_dynamic.cuh"
#include "idk_post.cuh"
#include "idk_point_shadows.cuh"
#include "idk_volumetric.cuh"
#include "idk_deferred.cuh"
#include "idk_ssr_taa.cuh"
#include "idk_vrs.cuh"
#include "idk_gbuffer.cuh"
#include "idk_transparency.cuh"
#include "idk_lights_skybox.cuh"
#include "idk_sky.cuh"
#include "idk_blas_build.cuh"
#include "idk_scene_add.cuh"
#include "idk_textures_host.h"

#define IDKPT_ABI_VERSION 4u   // 2: IdkPtSceneDesc gained Textures / TextureCount; 3: IdkPtStats gained CompactMs / AccumulateMs, host-buffer registration;
                               // 4: gather handle blob is 5 IPC handles (320 bytes), IDKPT_CREATE_GLOBAL_SLOTS, idkpt_gather_connect.
                               // Entry points added since (point-shadow cube maps, idkvx_set_shadow_maps, volumetric lighting, SSAO
                               // and deferred lighting, SSR and the TAA resolve, the shading-rate classifier, the G-buffer pass,
                               // transparency, the light spheres and the skybox) are
                               // additive and keep 4;
                               // IdkPtDeferredSettings grew a trailing IsVariableRateShading.

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
};

// What the path tracer (IdkPtCtx) and the voxeliser (IdkVxCtx) contexts share: device, stream, last error, and the events
// run_timed brackets synchronous work with.
struct IdkCtxBase {
    int device = 0;
    int smCount = 132;
    cudaStream_t stream = nullptr;
    std::string lastError;
    cudaEvent_t timing[4] = {};    // [0], [1]: start and end of run_timed's work; [2], [3]: marks inside it (idkvx_voxelize's spans)
};

// Material textures: their base levels, their records, the sRGB decode table. pools[0] holds every image of the last
// idkpt_set_scene / idkpt_set_textures; each idkpt_add_models with textures appends a pool of its own, which the records of
// its textures point into.
struct TextureTable {
    std::vector<DevBuf> pools;
    DevBuf recs, srgbLut;
};

// An output of a raster pass: its device buffer(s) and the size of the image they hold. A call invalidates the record before
// it may reallocate or overwrite the buffers and publishes it only when it succeeds, so the *_device_ptr exports and the passes
// that read the image never see a stale or half-written one.
struct RasterImage {
    DevBuf buf[2];
    int w = 0, h = 0;
    int last = -1;                 // the buffer the last successful call wrote; -1: none since the scene was set, or a later call failed
    void invalidate() { last = -1; }
    void publish(int width, int height, int written = 0) { w = width; h = height; last = written; }
    bool valid() const { return last >= 0; }
    bool valid_at(int width, int height) const { return valid() && w == width && h == height; }
};

// What the raster passes keep between calls; idkpt_set_scene drops all of it (release_raster).
struct RasterState {
    DevBuf stage;                  // the host inputs of a call (stage_inputs)
    DevBuf rtPtrs;                 // deferred lighting: the device pointer table of the ray-traced visibility images
    DevBuf volMarch, volDepth;     // volumetric lighting: the render-size march (rgba16f) and its depth (r32f)
    DevBuf vrsOffsets;             // variable-rate deferred lighting: the per-tile coarse-fragment offsets
    DevBuf gbPrev;                 // the G-buffer pass: the previous vertex positions' upload
    RasterImage vol;               // rgba16f at the presentation size
    RasterImage ssao;              // R8Unorm
    RasterImage deferred;          // rgba32f lit image
    RasterImage ssr;               // [0] the rgba32f merged image, [1] the rgba16f SSR image
    RasterImage vrs;               // [0] R8 rates, [1] r32f debug image, one texel per 16x16 tile; w x h is the render size
    RasterImage gb;                // the six planar fp32 attachments in one allocation (gbuffer_planes)
    RasterImage taa;               // the two rgba16f presentation-size history images (TAAResolve's ping-pong); w x h: their size
    int taaFrame = 0;              // TAAResolve.frame: Result = taa.buf[taaFrame % 2], PrevResult the other one
    // the ray-traced visibility (r32f) of each idkpt_shadows_ray_traced_gbuffer slot; the extra last one is the image the
    // host-array idkpt_shadows_ray_traced seeds with the caller's array
    RasterImage rtShadow[IDKPT_MAX_POINT_SHADOWS + 1];
};

#define IDK_MAX_LANES 16

struct Lane {
    cudaStream_t stream = nullptr;
    cudaEvent_t radianceReady = nullptr;   // recorded on the lane stream after the last shade of a sample
    cudaEvent_t accDone = nullptr;         // recorded on the main stream after that sample's FinalDraw consumed `radiance`
    bool accPending = false;
    bool allocated = false;
    DevBuf state, aov, alive[2], survivors, keysTmp, sortedAlive, hits, hitXform, debugCost, radiance, aovAlbedoFinal, aovNormalFinal;
    DevBuf countsDev;              // uint32 counts[IDKPT_MAX_RAY_DEPTH + 1]
    DevBuf tickets;                // uint32 tickets[2 * (IDKPT_MAX_RAY_DEPTH + 1)] (traverse, compact)
    DevBuf tileStatus;             // u64 per tile
    uint32_t epoch = 0;            // compaction epoch of this lane's status words: 1 .. IDK_EPOCH_MASK, cleared on wrap
    DevBuf keys;                   // ray sorting: key per slot of the compacted alive list
    IdkSortScratch sortScratch;
    DevBuf slotDelta;              // global slots: per local stripe, global - local slot of the current bounce (k_slot_exchange)
    uint32_t slotEpoch = 0;        // exchanges issued on this lane since the peers were connected (identical on every rank)
};

struct IdkPtCtx : IdkCtxBase {
    static inline thread_local std::string createError;   // last failed idkpt_create (idkpt_last_error(NULL))

    // image / tile geometry
    int width = 0, height = 0;
    int stripeH = 8, tileIndex = 0, tileCount = 1;
    std::vector<int> rows;         // owned rows, ascending
    uint32_t nLocal = 0;           // rows.size() * width
    uint32_t accumulatedSamples = 0;

    // scene
    bool haveScene = false;
    DeviceScene sc = {};
    IdkPtSceneDesc counts = {};    // element counts only (pointers unused)
    DevBuf nodes, triRec, blasTris, positions, descs, instances, xforms, meshes, materials, vertices, lights, tlas, vtxFrame, surfRec;
    std::vector<GpuLight> hostLights;   // host mirror of `lights` (idkpt_set_scene, idkpt_update_range): shadow-index checks
    float sky[3] = {0.0f, 0.0f, 0.0f};
    DevBuf skyFaces;
    int skyFaceSize = 0;
    TextureTable tex;
    std::vector<uint64_t> hostMaterialMaxHandle;   // per material: largest texture handle it uses (validation of later edits)

    // idkpt_trace_rays / idkpt_trace_rays_any: device staging buffers, kept between calls
    DevBuf scratch[3];

    // point-shadow cube maps (idkpt_set_point_shadows): host copies of the records and sizes, device records, one D16 allocation
    std::vector<GpuPointShadow> pointShadows;
    std::vector<int32_t> pointShadowSizes;
    std::vector<PointShadowDev> pointShadowRecs;
    DevBuf pointShadowDev, pointShadowMaps;
    DevBuf pointShadowLights;      // int32 LightIndex per shadow (the volumetric pass's Lights[shadow.LightIndex])

    RasterState raster;            // the raster passes (volumetric lighting .. the light spheres and the skybox)

    // present chain: bloom mip chains (rgba16f), AgX constants, RGBA8 frame
    DevBuf bloomDown, bloomUp, postConsts, ldr;
    // denoise hand-off: OIDN-layout packed RGB buffers (beauty, albedo, normal, output), a-trous ping-pong, denoised rgba32f image
    DevBuf oidn[4], denoiseWork[2], denoised;
    bool haveDenoised = false;

    // dynamic geometry: unskinned vertices, joint matrices, refit scratch (parents + locks of the largest BLAS)
    DevBuf unskinned, joints, refitParents, refitLocks, tlasScratch;
    DevBuf sahScratch;             // idkpt_blas_sah: the walk's stack and the per-BLAS results
    uint64_t unskinnedCount = 0;
    std::vector<uint32_t> unskinnedMaxJoint;   // per vertex max(JointIndices), host copy for range validation
    std::vector<GpuBlasDesc> hostDescs;
    std::vector<GpuBlasInstance> hostInstances;   // host mirror of `instances` (idkpt_set_scene): a bound voxeliser's draw list
    size_t nodeBytes = 0;
    // prevVertexPositionSSBO (ModelManager.cs:620): the positions before the last skin of each range. Created from the
    // positions at the first idkpt_skin_vertices or idkpt_prev_positions_device_ptr after idkpt_set_scene or idkpt_add_models,
    // which release it.
    DevBuf prevPositions;

    // voxelisers reading this scene (idkvx_set_scene_from); idkpt_destroy unbinds them. sceneGeneration counts idkpt_set_scene,
    // idkpt_blas_rebuild and idkpt_add_models calls, so that a bound voxeliser knows when the instance list or the BLAS triangle counts, and
    // with them its work-queue size, may have changed.
    std::vector<IdkVxCtx*> boundVoxelizers;
    uint64_t sceneGeneration = 0;

    // wavefront buffers: one set per lane. A lane is one sample in flight (ray-gen .. last shade) on its own stream; with
    // several lanes the latency-bound tail bounces of one sample overlap the throughput-bound head of the next
    // Lane 0 also serves the synchronous path (stats, export, debug).
    Lane lanes[IDK_MAX_LANES];
    int laneCount = 8;             // lanes used by asynchronous idkpt_compute (stats == NULL); IDKPT_LANES / CreateInfo.Flags
    int nextLane = 0;
    bool asyncPending = false;     // work issued on lane streams / main stream that no host call has waited for yet
    DevBuf images[3];
    DevBuf counters;               // TraceCounters
    DevBuf countLog;               // per-sample copies of the alive counts (stats only)
    uint32_t epochStart = 0;       // IDKPT_DEBUG_EPOCH_START: first compaction epoch of a fresh lane (wrap-around test hook)
    uint32_t slotEpochStart = 0;   // IDKPT_DEBUG_SLOT_EPOCH_START: slot-exchange epoch right after the peers are connected (wrap-around test hook)
    bool exportEnabled = false;

    // launch configuration
    int traverseBlocks = 0, traverseBlocksStats = 0, shadeBlocks = 0, traceRaysBlocks = 0, compactBlocks = 0;
    int firstHitBlocks[2][2] = {};  // k_first_hit grids of this scene's TLAS mode, [STATS][TEX]
    int traverseBlocksLane = 0, firstHitBlocksLane[2] = {};   // grids of the asynchronous path ([TEX]): the resident-block budget split between the lanes
    size_t stackBytes = 0;
    size_t traverse2Smem = 0;      // k_traverse2 stacks (IDK_T2_BLOCK columns)

    std::vector<cudaEvent_t> events;
    cudaStreamAttrValue l2Window = {};   // persisting-L2 window over [nodes | triRec]; applied to the main stream and every lane stream

    // multi-GPU gather over NVLink peer memory (CUDA IPC): full-size images (double-buffered) + arrival flags per rank
    int gatherWorld = 0, gatherRank = 0;
    DevBuf gatherImage[2], gatherFlags[2], gatherRows, gatherScratch;     // own buffers (exported)
    void* peerImage[2][IDK_MAX_PEERS] = {};                               // mapped peers (own entries = own buffers)
    void* peerFlags[2][IDK_MAX_PEERS] = {};
    bool peerMapped[IDK_MAX_PEERS] = {};
    uint32_t gatherEpoch = 0;
    double gatherTimeoutMs = 30000.0;                                     // arrival wait bound (IDKPT_GATHER_TIMEOUT_MS); a dead peer becomes an error, not a hung GPU
    int clockKHz = 1980000;
    int gatherCurrent = -1;                                               // buffer holding the last completed frame
    bool peerIsIpc = false;                                               // peers mapped with cudaIpcOpenMemHandle (else: same-process pointers)
    // global slots (IDKPT_CREATE_GLOBAL_SLOTS): per-stripe alive counts exchanged every bounce; table = [lane][parity][stripe] u64
    bool globalSlots = false;
    int nStripes = 0, nLocalStripes = 0;
    DevBuf slotTable;                                                     // own table (exported)
    void* peerSlotTable[IDK_MAX_PEERS] = {};

    // asynchronous presentation (device snapshot + D2H on a second stream, overlapping the next Compute)
    cudaStream_t copyStream = nullptr;
    cudaEvent_t snapDone = nullptr, copyDone = nullptr;
    DevBuf presentSnap;
    bool copyPending = false;
};

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            char buf_[512];                                                                        \
            snprintf(buf_, sizeof(buf_), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            ctx->lastError = buf_;                                                                 \
            return IDKPT_ERR_CUDA;                                                                 \
        }                                                                                          \
    } while (0)

// Without a context the message goes to the last create error of that context type.
template <class Ctx> static int fail(Ctx* ctx, int code, const char* msg) {
    (ctx ? ctx->lastError : Ctx::createError) = msg;
    return code;
}

static int fail(IdkCtxBase* ctx, const char* who, int code, const char* what) {
    ctx->lastError = std::string(who) + ": " + what;
    return code;
}

static cudaError_t ensure(DevBuf& b, size_t bytes) {
    if (bytes <= b.bytes && b.p) return cudaSuccess;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.bytes = 0;
    if (bytes == 0) return cudaSuccess;
    cudaError_t e = cudaMalloc(&b.p, bytes);
    if (e == cudaSuccess) b.bytes = bytes;
    return e;
}

static void release(DevBuf& b) {
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.bytes = 0;
}

static void release_textures(TextureTable& t) {
    for (DevBuf& b : t.pools) release(b);
    t.pools.clear();
    release(t.recs);
    release(t.srgbLut);
}

static void release_raster(RasterState& r) {
    for (DevBuf* b : {&r.stage, &r.rtPtrs, &r.volMarch, &r.volDepth, &r.vrsOffsets, &r.gbPrev}) release(*b);
    for (RasterImage* img : {&r.vol, &r.ssao, &r.deferred, &r.ssr, &r.vrs, &r.gb, &r.taa})
        for (DevBuf& b : img->buf) release(b);
    for (RasterImage& img : r.rtShadow) release(img.buf[0]);
    r = RasterState{};
}

static int upload(IdkCtxBase* ctx, DevBuf& b, const void* src, size_t bytes) {
    CK(ensure(b, std::max<size_t>(bytes, 16)));
    if (bytes) CK(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return IDKPT_OK;
}

static int create_stream(IdkCtxBase* ctx) {
    CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : ctx->timing) CK(cudaEventCreate(&e));
    return IDKPT_OK;
}

static void destroy_stream(IdkCtxBase* ctx) {
    for (cudaEvent_t e : ctx->timing) if (e) cudaEventDestroy(e);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
}

// Synchronous, timed work on the context's stream: `work` enqueues it between the start and end events and returns IDKPT_OK
// or an error code. The result's copy to the host (dst, if given) follows the end event, outside the timing. Waits for the
// stream, reports a launch or execution error as "<who>: <CUDA error>", and writes the elapsed time to *ms only on success.
template <class Work>
static int run_timed(IdkCtxBase* ctx, const char* who, float* ms, Work&& work, void* dst = nullptr, const void* src = nullptr, size_t bytes = 0) {
    CK(cudaEventRecord(ctx->timing[0], ctx->stream));
    if (int rc = work()) return rc;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        CK(cudaEventRecord(ctx->timing[1], ctx->stream));
        if (dst) CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        e = cudaStreamSynchronize(ctx->stream);
    }
    if (e != cudaSuccess) return fail(ctx, who, IDKPT_ERR_CUDA, cudaGetErrorString(e));
    if (ms) CK(cudaEventElapsedTime(ms, ctx->timing[0], ctx->timing[1]));
    return IDKPT_OK;
}

static void compute_tile_rows(IdkPtCtx* ctx) {
    ctx->rows.clear();
    for (int y = 0; y < ctx->height; y++)
        if (ctx->tileCount <= 1 || ((y / ctx->stripeH) % ctx->tileCount) == ctx->tileIndex) ctx->rows.push_back(y);
    ctx->nLocal = (uint32_t)(ctx->rows.size() * (size_t)ctx->width);
    ctx->nStripes = (ctx->height + ctx->stripeH - 1) / ctx->stripeH;
    ctx->nLocalStripes = 0;
    for (int s = 0; s < ctx->nStripes; s++)
        if (ctx->tileCount <= 1 || (s % ctx->tileCount) == ctx->tileIndex) ctx->nLocalStripes++;
}

// k_first_hit<STATS, TLAS, TEX> by [TLAS][STATS][TEX]
using FirstHitKernel = void (*)(FirstHitArgs);
static const FirstHitKernel kFirstHit[2][2][2] = {
    {{k_first_hit<false, false, false>, k_first_hit<false, false, true>}, {k_first_hit<true, false, false>, k_first_hit<true, false, true>}},
    {{k_first_hit<false, true, false>, k_first_hit<false, true, true>}, {k_first_hit<true, true, false>, k_first_hit<true, true, true>}}};

static int configure_launches(IdkPtCtx* ctx) {
    const int stackSize = std::max(1, ctx->sc.stackSize);
    ctx->stackBytes = (size_t)stackSize * IDK_BLOCK * sizeof(uint32_t);
    if (ctx->stackBytes > 200 * 1024) return fail(ctx, IDKPT_ERR_UNSUPPORTED, "BlasStackSize too large for the shared-memory traversal stack");
    CK(cudaFuncSetAttribute(k_trace_rays, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    CK(cudaFuncSetAttribute(k_trace_rays_any, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    CK(cudaFuncSetAttribute(k_shadows_ray_traced, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    CK(cudaFuncSetAttribute(k_point_shadow_faces, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    CK(cudaFuncSetAttribute(k_gbuffer, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    CK(cudaFuncSetAttribute(k_transparency<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    CK(cudaFuncSetAttribute(k_transparency<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
    ctx->traverse2Smem = (size_t)stackSize * IDK_T2_BLOCK * sizeof(uint32_t);
    CK(cudaFuncSetAttribute(k_traverse2<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->traverse2Smem));
    CK(cudaFuncSetAttribute(k_traverse2<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->traverse2Smem));
    CK(cudaFuncSetAttribute(k_traverse2<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->traverse2Smem));
    CK(cudaFuncSetAttribute(k_traverse2<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->traverse2Smem));
    int n = 0;
    // both TEX variants: idkpt_set_textures may switch between them without coming back here
    for (int stats = 0; stats < 2; stats++)
        for (int tex = 0; tex < 2; tex++) {
            const FirstHitKernel k = kFirstHit[ctx->sc.useTlas ? 1 : 0][stats][tex];
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->stackBytes));
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k, IDK_BLOCK, ctx->stackBytes));
            ctx->firstHitBlocks[stats][tex] = std::max(1, n) * ctx->smCount;
        }
    if (ctx->sc.useTlas) {
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_traverse2<false, true>, IDK_T2_BLOCK, ctx->traverse2Smem));
        ctx->traverseBlocks = std::max(1, n) * ctx->smCount;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_traverse2<true, true>, IDK_T2_BLOCK, ctx->traverse2Smem));
        ctx->traverseBlocksStats = std::max(1, n) * ctx->smCount;
    } else {
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_traverse2<false, false>, IDK_T2_BLOCK, ctx->traverse2Smem));
        ctx->traverseBlocks = std::max(1, n) * ctx->smCount;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_traverse2<true, false>, IDK_T2_BLOCK, ctx->traverse2Smem));
        ctx->traverseBlocksStats = std::max(1, n) * ctx->smCount;
    }
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_trace_rays, IDK_BLOCK, ctx->stackBytes));
    ctx->traceRaysBlocks = std::max(1, n) * ctx->smCount;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_shade<false>, IDK_BLOCK, 0));
    ctx->shadeBlocks = std::max(1, n) * ctx->smCount;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_compact, IDK_BLOCK, 0));
    ctx->compactBlocks = std::max(1, std::min(n, 4)) * ctx->smCount;
    // asynchronous path: `laneCount` samples in flight share the SMs; each lane's persistent traversal grid takes its share of
    // the resident-block budget
    {
        const int lanes = std::max(1, ctx->laneCount);
        const int perSm2 = (ctx->traverseBlocks / ctx->smCount + lanes - 1) / lanes;
        ctx->traverseBlocksLane = std::max(1, perSm2) * ctx->smCount;
        for (int tex = 0; tex < 2; tex++)
            ctx->firstHitBlocksLane[tex] = std::max(1, (ctx->firstHitBlocks[0][tex] / ctx->smCount + lanes - 1) / lanes) * ctx->smCount;
    }
    return IDKPT_OK;
}

static int allocate_lane(IdkPtCtx* ctx, Lane& ln) {
    const size_t n = std::max<uint32_t>(ctx->nLocal, 1);
    CK(ensure(ln.state, n * sizeof(PathState)));
    CK(ensure(ln.aov, n * 32));
    for (int i = 0; i < 2; i++) CK(ensure(ln.alive[i], n * 4));
    CK(ensure(ln.survivors, n * 4));
    CK(ensure(ln.hits, n * 16));
    CK(ensure(ln.hitXform, n * 4));
    CK(ensure(ln.debugCost, n * 4));
    CK(ensure(ln.radiance, n * 16));
    CK(ensure(ln.aovAlbedoFinal, n * 16));
    CK(ensure(ln.aovNormalFinal, n * 16));
    CK(ensure(ln.countsDev, (IDKPT_MAX_RAY_DEPTH + 1) * sizeof(uint32_t)));
    CK(ensure(ln.tickets, 2 * (IDKPT_MAX_RAY_DEPTH + 1) * sizeof(uint32_t)));
    CK(ensure(ln.tileStatus, ((n + IDK_BLOCK * IDK_COMPACT_ITEMS - 1) / (IDK_BLOCK * IDK_COMPACT_ITEMS) + 1) * sizeof(unsigned long long)));
    if (ctx->globalSlots && ctx->tileCount > 1) CK(ensure(ln.slotDelta, (size_t)std::max(1, ctx->nLocalStripes) * sizeof(uint32_t)));
    CK(cudaMemsetAsync(ln.tileStatus.p, 0, ln.tileStatus.bytes, ctx->stream));
    if (!ln.stream) CK(cudaStreamCreateWithFlags(&ln.stream, cudaStreamNonBlocking));
    if (!ln.radianceReady) CK(cudaEventCreateWithFlags(&ln.radianceReady, cudaEventDisableTiming));
    if (!ln.accDone) CK(cudaEventCreateWithFlags(&ln.accDone, cudaEventDisableTiming));
    CK(cudaStreamSynchronize(ctx->stream));   // the status words are cleared before any lane stream touches them
    ln.epoch = ctx->epochStart;
    CK(cudaStreamSetAttribute(ln.stream, cudaStreamAttributeAccessPolicyWindow, &ctx->l2Window));   // BVH persistence on the lane streams too
    ln.accPending = false;
    ln.allocated = true;
    return IDKPT_OK;
}

static void release_lane(Lane& ln, bool keepStream) {
    DevBuf* all[] = {&ln.state, &ln.aov, &ln.alive[0], &ln.alive[1], &ln.survivors, &ln.keysTmp, &ln.sortedAlive, &ln.hits, &ln.hitXform, &ln.debugCost,
                     &ln.radiance, &ln.aovAlbedoFinal, &ln.aovNormalFinal, &ln.countsDev, &ln.tickets, &ln.tileStatus, &ln.keys, &ln.slotDelta};
    for (DevBuf* b : all) release(*b);
    idk_sort_release(ln.sortScratch);
    ln.allocated = false;
    ln.accPending = false;
    if (!keepStream) {
        if (ln.stream) { cudaStreamDestroy(ln.stream); ln.stream = nullptr; }
        if (ln.radianceReady) { cudaEventDestroy(ln.radianceReady); ln.radianceReady = nullptr; }
        if (ln.accDone) { cudaEventDestroy(ln.accDone); ln.accDone = nullptr; }
    }
}

// Wait for everything issued so far: every lane stream and the main (image) stream. Every entry point that reads or
// changes device data other than idkpt_compute / idkpt_present_async starts with this.
static cudaError_t drain(IdkPtCtx* ctx) {
    cudaError_t first = cudaSuccess;
    for (int i = 0; i < IDK_MAX_LANES; i++)
        if (ctx->lanes[i].stream) { cudaError_t e = cudaStreamSynchronize(ctx->lanes[i].stream); if (first == cudaSuccess) first = e; }
    if (ctx->stream) { cudaError_t e = cudaStreamSynchronize(ctx->stream); if (first == cudaSuccess) first = e; }
    for (int i = 0; i < IDK_MAX_LANES; i++) ctx->lanes[i].accPending = false;
    ctx->asyncPending = false;
    return first;
}

// Errors that only the device knows about (a kernel fault, a peer rank that never delivered its tile) surface at the
// next host-synchronising call.
static int check_device_errors(IdkPtCtx* ctx, cudaError_t se, const char* who) {
    if (se != cudaSuccess) {
        ctx->lastError = std::string(who) + ": kernel execution failed: " + cudaGetErrorString(se);
        return IDKPT_ERR_CUDA;
    }
    if (ctx->gatherWorld > 1) {
        uint32_t timedOut = 0;
        CK(cudaMemcpy(&timedOut, (uint32_t*)ctx->gatherScratch.p + 1, 4, cudaMemcpyDeviceToHost));
        if (timedOut) {
            cudaMemset((uint32_t*)ctx->gatherScratch.p + 1, 0, 4);
            return fail(ctx, IDKPT_ERR_CUDA, timedOut == 2u ? "idkpt_compute: timed out waiting for a peer rank's per-stripe alive counts (multi-GPU global slots)"
                                                            : "idkpt_compute: timed out waiting for a peer rank's tile (multi-GPU gather)");
        }
    }
    return IDKPT_OK;
}

// Entry points that change or expose device data wait for the samples in flight first.
#define DRAIN_PENDING(who)                                                         \
    do {                                                                           \
        if (ctx->asyncPending) {                                                   \
            cudaSetDevice(ctx->device);                                            \
            int rc_ = check_device_errors(ctx, drain(ctx), who);                   \
            if (rc_) return rc_;                                                   \
        }                                                                          \
    } while (0)

static int allocate_wavefront(IdkPtCtx* ctx) {
    const size_t n = std::max<uint32_t>(ctx->nLocal, 1);
    for (int i = 1; i < IDK_MAX_LANES; i++) if (ctx->lanes[i].allocated) release_lane(ctx->lanes[i], true);   // re-created on demand at the new size
    int rc = allocate_lane(ctx, ctx->lanes[0]);
    if (rc) return rc;
    for (int i = 0; i < 3; i++) {
        CK(ensure(ctx->images[i], n * 16));
        CK(cudaMemsetAsync(ctx->images[i].p, 0, n * 16, ctx->stream));   // Result.Fill(0), PathTracer.cs:305
    }
    CK(ensure(ctx->counters, sizeof(TraceCounters)));
    return IDKPT_OK;
}

static const char* validate_material_textures(const GpuMaterial& m, uint64_t textureCount, const char* msg) {
    const uint64_t h[5] = {m.BaseColorTexture, m.MetallicRoughnessTexture, m.NormalTexture, m.EmissiveTexture, m.TransmissionTexture};
    for (int i = 0; i < 5; i++) if (h[i] > textureCount) return msg;
    return nullptr;
}

static uint64_t material_max_handle(const GpuMaterial& m) {
    return std::max(std::max(std::max(m.BaseColorTexture, m.MetallicRoughnessTexture), std::max(m.NormalTexture, m.EmissiveTexture)), m.TransmissionTexture);
}

// Material textures: all base levels in one allocation, 256-byte aligned; 32-byte records point into it.
static int upload_textures(IdkCtxBase* ctx, TextureTable& t, const IdkPtTextureDesc* textures, uint64_t count) {
    IdkPtSceneDesc tmp = {};
    tmp.Textures = textures; tmp.TextureCount = count;
    const std::vector<size_t> off = idk_texture_offsets(&tmp);
    if (t.pools.empty()) t.pools.emplace_back();
    for (size_t i = 1; i < t.pools.size(); i++) release(t.pools[i]);   // the pools idkpt_add_models appended
    t.pools.resize(1);
    CK(ensure(t.pools[0], std::max<size_t>(off[count], 16)));
    std::vector<TexRec> recs;
    CK(idk_upload_texture_table(textures, count, off, t.pools[0].p, ctx->stream, recs));
    int rc;
    if ((rc = upload(ctx, t.recs, recs.data(), recs.size() * sizeof(TexRec)))) return rc;
    float lut[256];
    idk_srgb_lut(lut);
    if ((rc = upload(ctx, t.srgbLut, lut, sizeof(lut)))) return rc;
    CK(cudaStreamSynchronize(ctx->stream));   // recs / lut are locals
    return IDKPT_OK;
}

// idk_validate_textures's verdict: formats the decoder lacks are unsupported, anything else is an invalid argument.
static int texture_error(IdkCtxBase* ctx, const char* who, const char* terr) {
    return fail(ctx, who, strstr(terr, "not supported") ? IDKPT_ERR_UNSUPPORTED : IDKPT_ERR_INVALID_ARGUMENT, terr);
}

// Checks idkpt_set_scene and idkvx_set_scene share: every index the kernels chase must be in range (a malformed host array
// must become an error code, never a device fault).
static int validate_scene(IdkCtxBase* ctx, const char* who, const IdkPtSceneDesc* s) {
    if (!s->BlasTriangles || !s->BlasDescs || !s->BlasInstances || !s->MeshTransforms || !s->Meshes || !s->Materials || !s->Vertices || !s->VertexPositions)
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a required array is null");
    if (s->LightCount > IDK_GPU_MAX_UBO_LIGHT_COUNT) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "more than 256 lights");
    for (uint64_t i = 0; i < s->BlasInstanceCount; i++)
        if (s->BlasInstances[i].BlasId >= s->BlasDescCount || s->BlasInstances[i].MeshTransformId >= s->MeshTransformCount)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "BlasInstance references a missing BLAS or transform");
    for (uint64_t i = 0; i < s->BlasDescCount; i++) {
        const GpuBlasDesc& d = s->BlasDescs[i];
        if (d.TriangleOffset < 0 || d.TriangleCount < 0 || (uint64_t)d.TriangleOffset + d.TriangleCount > s->BlasTriangleCount)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "GpuBlasDesc triangle range outside the array");
    }
    // triangle vertex ids must index the position / vertex arrays (checked on the host copy: cheap relative to the BVH build
    // that produced it)
    const uint64_t lim = std::min(s->VertexPositionCount, s->VertexCount);
    for (uint64_t i = 0; i < s->BlasTriangleCount; i++) {
        const GpuBlasTriangle& t = s->BlasTriangles[i];
        if ((uint64_t)(uint32_t)t.X >= lim || (uint64_t)(uint32_t)t.Y >= lim || (uint64_t)(uint32_t)t.Z >= lim || t.MeshId < 0 || (uint64_t)t.MeshId >= s->MeshCount)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "GpuBlasTriangle index out of range");
    }
    for (uint64_t i = 0; i < s->MeshCount; i++)
        if (s->Meshes[i].MaterialId < 0 || (uint64_t)s->Meshes[i].MaterialId >= s->MaterialCount) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "GpuMesh.MaterialId out of range");
    if (const char* terr = idk_validate_textures(s)) return texture_error(ctx, who, terr);
    return IDKPT_OK;
}

// TLAS.AllocateRequiredNodes (TLAS.cs:266-269): children adjacent and behind their parent, leaves name an existing instance.
// `t` holds nodes [first, first + count) of a TLAS with nodeCount nodes.
static bool tlas_nodes_valid(const GpuTlasNode* t, uint64_t first, uint64_t count, uint64_t nodeCount, uint64_t instanceCount) {
    for (uint64_t i = 0; i < count; i++) {
        const uint32_t w = t[i].IsLeafAndChildOrInstanceId, id = w & 0x7FFFFFFFu;
        if ((w >> 31) ? (id >= instanceCount) : (id <= first + i || (uint64_t)id + 1 >= nodeCount)) return false;
    }
    return true;
}

// Structural validation of one BLAS before its arrays reach the kernels: child pairs in range, even, and behind their parent
// (the builder emits DFS order, which also rules out cycles); leaf ranges inside the BLAS's triangle range; and the
// traversal stack the kernels will need (BLAS.ComputeRequiredStackSize, Bvh/BLAS.cs:672-702) must fit BlasStackSize.
// Returns nullptr or an error text.
static const char* validate_blas(const GpuBlasNode* nodes, const GpuBlasDesc& d, int blasStackSize) {
    const int n = d.NodeCount;
    if (n < 4 || (n & 1)) return "idkpt_set_scene: BLAS node count must be even and >= 4";
    if (nodes[1].TriCount != 0 || nodes[1].TriStartOrChild != 2) return "idkpt_set_scene: BLAS root must be interior with children at 2 (BLAS.cs:16-22)";
    std::vector<int> req((size_t)n / 2, 0);
    for (int p = n / 2 - 1; p >= 1; p--) {
        int need[2] = {-1, -1};
        for (int c = 0; c < 2; c++) {
            const GpuBlasNode& nd = nodes[2 * p + c];
            if (nd.TriCount > 0) {
                if (nd.TriStartOrChild < 0 || (int64_t)nd.TriStartOrChild + nd.TriCount > d.TriangleCount) return "idkpt_set_scene: BLAS leaf triangle range outside the BLAS";
            } else if (nd.TriCount == 0) {
                const int ch = nd.TriStartOrChild;
                if (ch <= 2 * p || (ch & 1) || ch + 1 >= n) return "idkpt_set_scene: BLAS child index out of range / not in DFS order";
                need[c] = req[(size_t)ch / 2];
            } else {
                return "idkpt_set_scene: negative TriCount in a BLAS node";
            }
        }
        req[p] = (need[0] >= 0 && need[1] >= 0) ? std::max(need[0], need[1]) + 1 : std::max(need[0], std::max(need[1], 0));
    }
    if (req[1] > blasStackSize) return "idkpt_set_scene: BlasStackSize smaller than the traversal stack this BLAS needs";
    return nullptr;
}

// Height of a host-provided TLAS (= stack entries the walk needs); children follow their parent (validated before).
static int tlas_height(const GpuTlasNode* t, uint64_t count) {
    std::vector<int> need(count, 0);
    for (int64_t i = (int64_t)count - 1; i >= 0; i--) {
        const uint32_t w = t[i].IsLeafAndChildOrInstanceId, c = w & 0x7FFFFFFFu;
        need[i] = (w >> 31) ? 0 : 1 + std::max(need[c], need[c + 1]);
    }
    return count ? need[0] : 0;
}

static void gather_teardown(IdkPtCtx* ctx) {
    for (int b = 0; b < 2; b++)
        for (int p = 0; p < IDK_MAX_PEERS; p++) {
            if (ctx->peerMapped[p] && p != ctx->gatherRank && ctx->peerIsIpc) {
                if (ctx->peerImage[b][p]) cudaIpcCloseMemHandle(ctx->peerImage[b][p]);
                if (ctx->peerFlags[b][p]) cudaIpcCloseMemHandle(ctx->peerFlags[b][p]);
            }
            ctx->peerImage[b][p] = nullptr;
            ctx->peerFlags[b][p] = nullptr;
        }
    for (int p = 0; p < IDK_MAX_PEERS; p++) {
        if (ctx->peerMapped[p] && p != ctx->gatherRank && ctx->peerIsIpc && ctx->peerSlotTable[p]) cudaIpcCloseMemHandle(ctx->peerSlotTable[p]);
        ctx->peerSlotTable[p] = nullptr;
        ctx->peerMapped[p] = false;
    }
    ctx->peerIsIpc = false;
    release(ctx->slotTable);
    for (int i = 0; i < IDK_MAX_LANES; i++) ctx->lanes[i].slotEpoch = 0;
    for (int b = 0; b < 2; b++) { release(ctx->gatherImage[b]); release(ctx->gatherFlags[b]); }
    release(ctx->gatherRows);
    release(ctx->gatherScratch);
    ctx->gatherWorld = 0;
    ctx->gatherCurrent = -1;
    ctx->gatherEpoch = 0;
}

// The light spheres' mesh (k_lights_skybox's constant tables) on the context's device. Every context writes the same bytes.
static int upload_sphere_mesh(IdkPtCtx* ctx) {
    float3 vertices[IDK_SPHERE_VERTICES];
    uint32_t triangles[IDK_SPHERE_TRIANGLES];
    sphere_mesh_tables(vertices, triangles);
    CK(cudaMemcpyToSymbolAsync(c_sphere_vertices, vertices, sizeof(vertices), 0, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyToSymbolAsync(c_sphere_triangles, triangles, sizeof(triangles), 0, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

// The kept previous positions, created on first need as a copy of the positions (ModelManager.cs:620 creates
// prevVertexPositionSSBO from the uploaded positions; only skinning moves them afterwards). Ordered on the context stream.
static int keep_prev_positions(IdkPtCtx* ctx) {
    if (ctx->prevPositions.p) return IDKPT_OK;
    const size_t bytes = ctx->counts.VertexPositionCount * sizeof(PackedVec3);
    CK(ensure(ctx->prevPositions, std::max<size_t>(bytes, 16)));
    const cudaError_t e = bytes ? cudaMemcpyAsync(ctx->prevPositions.p, ctx->positions.p, bytes, cudaMemcpyDeviceToDevice, ctx->stream) : cudaSuccess;
    if (e != cudaSuccess) release(ctx->prevPositions);
    CK(e);
    return IDKPT_OK;
}

// Keep the BVH resident in the 50 MB L2: persisting access-policy window over [nodes | triRec] (bvhBytes from `base`) on the
// render stream and every lane stream. The wavefront buffers (hundreds of MB per frame) stream through the rest of the cache
// without evicting the tree.
static int set_l2_window(IdkPtCtx* ctx, void* base, size_t bvhBytes) {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, ctx->device));
    cudaStreamAttrValue& attr = ctx->l2Window;
    memset(&attr, 0, sizeof(attr));
    if (prop.persistingL2CacheMaxSize > 0 && prop.accessPolicyMaxWindowSize > 0) {
        const size_t setAside = std::min<size_t>((size_t)prop.persistingL2CacheMaxSize, std::max<size_t>(bvhBytes, 1 << 20));
        CK(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, setAside));
        const size_t window = std::min<size_t>(bvhBytes, (size_t)prop.accessPolicyMaxWindowSize);
        attr.accessPolicyWindow.base_ptr = base;
        attr.accessPolicyWindow.num_bytes = window;
        attr.accessPolicyWindow.hitRatio = window <= setAside ? 1.0f : (float)((double)setAside / (double)window);
        attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    } else {
        attr.accessPolicyWindow.num_bytes = 0;
    }
    CK(cudaStreamSetAttribute(ctx->stream, cudaStreamAttributeAccessPolicyWindow, &attr));
    for (int i = 0; i < IDK_MAX_LANES; i++)    // the asynchronous path launches traverse / shade on the lane streams
        if (ctx->lanes[i].stream) CK(cudaStreamSetAttribute(ctx->lanes[i].stream, cudaStreamAttributeAccessPolicyWindow, &attr));
    return IDKPT_OK;
}

// IdkPtBlasBuildSettings (NULL: the engine's defaults) as the builder's parameters. Rejects non-finite values and
// StopSplittingThreshold < 1 (a node of 0 fragments would read as an interior node, GpuBlasNode.TriCount == 0).
static int blas_build_params(IdkPtCtx* ctx, const char* who, const IdkPtBlasBuildSettings* settings, idkbvh::Params& p) {
    const idkbvh::Params d;
    const IdkPtBlasBuildSettings s = settings ? *settings : IdkPtBlasBuildSettings{d.stopSplittingThreshold, d.maxLeafTriangleCount,
        d.triangleCost, d.stackOptThreshold, d.stackOptSahIncreaseAcceptance, d.splitFactor, d.doPreSplit};
    if (!std::isfinite(s.TriangleCost) || !std::isfinite(s.StackOptSahIncreaseAcceptance) || !std::isfinite(s.SplitFactor))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "non-finite setting");
    if (s.StopSplittingThreshold < 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "StopSplittingThreshold must be at least 1");
    p = {s.StopSplittingThreshold, s.MaxLeafTriangleCount, s.TriangleCost, s.StackOptThreshold, s.StackOptSahIncreaseAcceptance,
         s.SplitFactor, s.DoPreSplit ? 1 : 0};
    return IDKPT_OK;
}

// idkvx_impl.cuh: forgets this context in every voxeliser bound to it (idkvx_set_scene_from), before it goes away.
static void unbind_voxelizers(IdkPtCtx* ctx);

extern "C" {

IDKPT_API uint32_t idkpt_abi_version(void) { return IDKPT_ABI_VERSION; }

IDKPT_API const char* idkpt_last_error(IdkPtCtx* ctx) { return ctx ? ctx->lastError.c_str() : IdkPtCtx::createError.c_str(); }

IDKPT_API int idkpt_create(const IdkPtCreateInfo* ci, IdkPtCtx** out) {
    if (!ci || !out) return fail<IdkPtCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_create: null argument");
    *out = nullptr;
    if (ci->Width <= 0 || ci->Height <= 0 || ci->Width > 4096 * 4 || ci->Height > 4096 * 4)
        return fail<IdkPtCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_create: invalid image size");
    int stripe = ci->TileStripeHeight > 0 ? ci->TileStripeHeight : 8;
    int tcount = ci->TileCount > 1 ? ci->TileCount : 1;
    if ((ci->Flags & IDKPT_CREATE_GLOBAL_SLOTS) && tcount > 1 && (ci->Height + stripe - 1) / stripe > IDK_MAX_STRIPES)
        return fail<IdkPtCtx>(nullptr, IDKPT_ERR_UNSUPPORTED, "idkpt_create: IDKPT_CREATE_GLOBAL_SLOTS supports at most 4096 stripes (raise TileStripeHeight)");
    if (tcount > 1 && (ci->TileIndex < 0 || ci->TileIndex >= tcount))
        return fail<IdkPtCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_create: TileIndex out of range");
    int deviceCount = 0;
    cudaError_t e = cudaGetDeviceCount(&deviceCount);
    if (e != cudaSuccess || deviceCount == 0)
        return fail<IdkPtCtx>(nullptr, IDKPT_ERR_NO_DEVICE, "idkpt_create: no CUDA device (libidkpt has no CPU fallback)");
    if (ci->Device < 0 || ci->Device >= deviceCount)
        return fail<IdkPtCtx>(nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_create: device ordinal out of range");
    if (cudaSetDevice(ci->Device) != cudaSuccess) return fail<IdkPtCtx>(nullptr, IDKPT_ERR_CUDA, "idkpt_create: cudaSetDevice failed");
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, ci->Device) != cudaSuccess) return fail<IdkPtCtx>(nullptr, IDKPT_ERR_CUDA, "idkpt_create: cudaGetDeviceProperties failed");
    if (prop.major != 9 || prop.minor != 0) {
        char buf[512];
        snprintf(buf, sizeof(buf), "idkpt_create: device '%s' is sm_%d%d; libidkpt is built for sm_90a only", prop.name, prop.major, prop.minor);
        return fail<IdkPtCtx>(nullptr, IDKPT_ERR_NO_DEVICE, buf);
    }
    IdkPtCtx* ctx = new IdkPtCtx();
    ctx->device = ci->Device;
    ctx->smCount = prop.multiProcessorCount;
    ctx->width = ci->Width;
    ctx->height = ci->Height;
    ctx->stripeH = stripe;
    ctx->tileIndex = tcount > 1 ? ci->TileIndex : 0;
    ctx->tileCount = tcount;
    if (const int fl = (ci->Flags >> 8) & 15) ctx->laneCount = std::min(IDK_MAX_LANES, fl);   // IDKPT_CREATE_LANES(n)
    ctx->globalSlots = (ci->Flags & IDKPT_CREATE_GLOBAL_SLOTS) != 0;
    if (const char* v = getenv("IDKPT_LANES")) ctx->laneCount = std::max(1, std::min(IDK_MAX_LANES, atoi(v)));
    if (const char* v = getenv("IDKPT_DEBUG_EPOCH_START")) ctx->epochStart = (uint32_t)strtoul(v, nullptr, 0) & IDK_EPOCH_MASK;
    if (const char* v = getenv("IDKPT_DEBUG_SLOT_EPOCH_START")) ctx->slotEpochStart = (uint32_t)strtoul(v, nullptr, 0) & ~1u;   // even: keeps the parity sequence
    if (const char* v = getenv("IDKPT_GATHER_TIMEOUT_MS")) ctx->gatherTimeoutMs = std::max(1.0, atof(v));
    ctx->clockKHz = prop.clockRate;
    compute_tile_rows(ctx);
    int rc = create_stream(ctx);
    if (rc == IDKPT_OK) rc = allocate_wavefront(ctx);
    if (rc == IDKPT_OK) rc = upload_sphere_mesh(ctx);
    if (rc != IDKPT_OK) {
        IdkPtCtx::createError = ctx->lastError;
        idkpt_destroy(ctx);
        return rc;
    }
    ctx->sky[0] = ctx->sky[1] = ctx->sky[2] = 0.0f;
    *out = ctx;
    return IDKPT_OK;
}

IDKPT_API void idkpt_destroy(IdkPtCtx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    drain(ctx);
    unbind_voxelizers(ctx);
    DevBuf* all[] = {&ctx->nodes, &ctx->triRec, &ctx->blasTris, &ctx->positions, &ctx->descs, &ctx->instances, &ctx->xforms,
                     &ctx->meshes, &ctx->materials, &ctx->vertices, &ctx->lights, &ctx->tlas, &ctx->vtxFrame, &ctx->surfRec,
                     &ctx->images[0], &ctx->images[1], &ctx->images[2], &ctx->counters, &ctx->countLog, &ctx->skyFaces,
                     &ctx->bloomDown, &ctx->bloomUp, &ctx->postConsts, &ctx->ldr,
                     &ctx->unskinned, &ctx->joints, &ctx->refitParents, &ctx->refitLocks, &ctx->scratch[0], &ctx->scratch[1], &ctx->scratch[2],
                     &ctx->tlasScratch, &ctx->sahScratch, &ctx->oidn[0], &ctx->oidn[1], &ctx->oidn[2], &ctx->oidn[3], &ctx->denoiseWork[0], &ctx->denoiseWork[1], &ctx->denoised,
                     &ctx->pointShadowDev, &ctx->pointShadowMaps, &ctx->pointShadowLights, &ctx->prevPositions};
    for (DevBuf* b : all) release(*b);
    release_textures(ctx->tex);
    release_raster(ctx->raster);
    for (int i = 0; i < IDK_MAX_LANES; i++) release_lane(ctx->lanes[i], false);
    for (cudaEvent_t ev : ctx->events) cudaEventDestroy(ev);
    gather_teardown(ctx);
    if (ctx->copyStream) { cudaStreamSynchronize(ctx->copyStream); cudaStreamDestroy(ctx->copyStream); }
    if (ctx->snapDone) cudaEventDestroy(ctx->snapDone);
    if (ctx->copyDone) cudaEventDestroy(ctx->copyDone);
    release(ctx->presentSnap);
    destroy_stream(ctx);
    delete ctx;
}

IDKPT_API int idkpt_set_scene(IdkPtCtx* ctx, const IdkPtSceneDesc* s) {
    if (!ctx || !s) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: null argument");
    DRAIN_PENDING("idkpt_set_scene");
    CK(cudaSetDevice(ctx->device));
    if (!s->BlasNodes) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: a required array is null");
    if (int rc = validate_scene(ctx, "idkpt_set_scene", s)) return rc;
    if (s->UseTlas) {
        // TLAS.AllocateRequiredNodes: 2n-1 nodes, root at 0 (TLAS.cs:266-269)
        if (!s->TlasNodes || s->BlasInstanceCount == 0 || s->TlasNodeCount != 2 * s->BlasInstanceCount - 1)
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: UseTlas needs 2*instances-1 TLAS nodes");
        if (!tlas_nodes_valid(s->TlasNodes, 0, s->TlasNodeCount, s->TlasNodeCount, s->BlasInstanceCount))
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: malformed TLAS node (child / instance id out of range)");
        if (tlas_height(s->TlasNodes, s->TlasNodeCount) > IDK_TLAS_STACK_SIZE)
            return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_set_scene: TLAS deeper than the 24-entry traversal stack of the TLAS walk (BVHIntersect.glsl:4)");
    }
    if (s->BlasTriangleCount >= (1ull << 31) || s->BlasNodeCount >= (1ull << 31)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: scene too large");
    for (uint64_t i = 0; i < s->BlasDescCount; i++) {
        const GpuBlasDesc& d = s->BlasDescs[i];
        if (d.NodeOffset < 0 || d.NodeCount < 4 || (uint64_t)d.NodeOffset + d.NodeCount > s->BlasNodeCount)
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: GpuBlasDesc range outside the node array");
        if (d.RequiredStackSize > s->BlasStackSize)
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_scene: BlasStackSize smaller than a BLAS's RequiredStackSize");
        if (const char* err = validate_blas(s->BlasNodes + d.NodeOffset, d, s->BlasStackSize)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, err);
    }
    if ((size_t)std::max(1, s->BlasStackSize) * IDK_BLOCK * sizeof(uint32_t) > 200 * 1024)
        return fail(ctx, IDKPT_ERR_UNSUPPORTED, "BlasStackSize too large for the shared-memory traversal stack");

    // Every host-side check has passed; from here on device arrays are overwritten / reallocated. Until the new scene is
    // complete the context has NO scene: a failure below (CUDA error, out of memory) must not leave the previous scene's
    // pointers and counts looking valid.
    ctx->haveScene = false;
    ctx->sceneGeneration++;
    ctx->pointShadows.clear(); ctx->pointShadowSizes.clear(); ctx->pointShadowRecs.clear();   // the shadows belong to the old scene
    release(ctx->pointShadowDev); release(ctx->pointShadowMaps); release(ctx->pointShadowLights);
    release(ctx->prevPositions);
    release_raster(ctx->raster);   // the raster images belong to the old scene too
    int rc;
    // nodes and triangle records share one allocation ("bvh"): [nodes | triRec], so that one L2 access-policy window covers both
    const size_t nodeBytes = ((s->BlasNodeCount * sizeof(GpuBlasNode)) + 255) & ~(size_t)255;
    const size_t triRecBytes = std::max<size_t>(s->BlasTriangleCount, 1) * 64;
    CK(ensure(ctx->nodes, nodeBytes + triRecBytes));
    CK(cudaMemcpyAsync(ctx->nodes.p, s->BlasNodes, s->BlasNodeCount * sizeof(GpuBlasNode), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = upload(ctx, ctx->blasTris, s->BlasTriangles, s->BlasTriangleCount * sizeof(GpuBlasTriangle)))) return rc;
    if ((rc = upload(ctx, ctx->positions, s->VertexPositions, s->VertexPositionCount * sizeof(PackedVec3)))) return rc;
    if ((rc = upload(ctx, ctx->descs, s->BlasDescs, s->BlasDescCount * sizeof(GpuBlasDesc)))) return rc;
    if ((rc = upload(ctx, ctx->instances, s->BlasInstances, s->BlasInstanceCount * sizeof(GpuBlasInstance)))) return rc;
    if ((rc = upload(ctx, ctx->xforms, s->MeshTransforms, s->MeshTransformCount * sizeof(GpuMeshTransform)))) return rc;
    if ((rc = upload(ctx, ctx->meshes, s->Meshes, s->MeshCount * sizeof(GpuMesh)))) return rc;
    if ((rc = upload(ctx, ctx->materials, s->Materials, s->MaterialCount * sizeof(GpuMaterial)))) return rc;
    if ((rc = upload(ctx, ctx->vertices, s->Vertices, s->VertexCount * sizeof(GpuVertex)))) return rc;
    if ((rc = upload(ctx, ctx->lights, s->Lights, s->LightCount * sizeof(GpuLight)))) return rc;
    if ((rc = upload(ctx, ctx->tlas, s->TlasNodes, s->UseTlas ? s->TlasNodeCount * sizeof(GpuTlasNode) : 0))) return rc;
    if ((rc = upload_textures(ctx, ctx->tex, s->Textures, s->TextureCount))) return rc;
    ctx->hostMaterialMaxHandle.assign(s->MaterialCount, 0);
    for (uint64_t i = 0; i < s->MaterialCount; i++) ctx->hostMaterialMaxHandle[i] = material_max_handle(s->Materials[i]);

    CK(ensure(ctx->vtxFrame, std::max<size_t>(s->VertexCount, 1) * 32));
    CK(ensure(ctx->surfRec, std::max<size_t>(s->MeshCount, 1) * 80));
    if (s->VertexCount) {
        const uint32_t nv = (uint32_t)s->VertexCount;
        k_prepare_vertices<<<(nv + 255) / 256, 256, 0, ctx->stream>>>((const uint4*)ctx->vertices.p, (float4*)ctx->vtxFrame.p, nv);
    }
    if (s->MeshCount) {
        const uint32_t nm = (uint32_t)s->MeshCount;
        k_prepare_surfaces<<<(nm + 255) / 256, 256, 0, ctx->stream>>>((const GpuMesh*)ctx->meshes.p, (const GpuMaterial*)ctx->materials.p, (float4*)ctx->surfRec.p, nm);
    }
    CK(cudaGetLastError());
    if (s->BlasTriangleCount) {
        const uint32_t n = (uint32_t)s->BlasTriangleCount;
        k_prepare_triangles<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const int4*)ctx->blasTris.p, (const float*)ctx->positions.p, (float4*)((char*)ctx->nodes.p + nodeBytes), n);
        CK(cudaGetLastError());
    }

    DeviceScene& sc = ctx->sc;
    sc.nodes = (const float4*)ctx->nodes.p;
    sc.triRec = (const float4*)((char*)ctx->nodes.p + nodeBytes);
    sc.blasTris = (const int4*)ctx->blasTris.p;
    sc.descs = (const GpuBlasDesc*)ctx->descs.p;
    sc.instances = (const GpuBlasInstance*)ctx->instances.p;
    sc.xforms = (const float4*)ctx->xforms.p;
    sc.meshes = (const GpuMesh*)ctx->meshes.p;
    sc.materials = (const GpuMaterial*)ctx->materials.p;
    sc.vertices = (const uint4*)ctx->vertices.p;
    sc.lights = (const GpuLight*)ctx->lights.p;
    sc.instanceCount = (uint32_t)s->BlasInstanceCount;
    sc.lightCount = (uint32_t)s->LightCount;
    sc.skyR = ctx->sky[0]; sc.skyG = ctx->sky[1]; sc.skyB = ctx->sky[2];
    sc.skyFaces = ctx->skyFaceSize ? (const float4*)ctx->skyFaces.p : nullptr;
    sc.skyFaceSize = ctx->skyFaceSize;
    sc.stackSize = std::max(1, s->BlasStackSize);
    sc.tlasNodes = (const float4*)ctx->tlas.p;
    sc.useTlas = s->UseTlas ? 1 : 0;
    sc.vtxFrame = (const float4*)ctx->vtxFrame.p;
    sc.surfRec = (const float4*)ctx->surfRec.p;
    sc.textures = (const TexRec*)ctx->tex.recs.p;
    sc.textureCount = (uint32_t)s->TextureCount;
    sc.srgbLut = (const float*)ctx->tex.srgbLut.p;
    ctx->counts = *s;
    ctx->hostLights.assign(s->Lights, s->Lights + s->LightCount);
    ctx->hostDescs.assign(s->BlasDescs, s->BlasDescs + s->BlasDescCount);
    ctx->hostInstances.assign(s->BlasInstances, s->BlasInstances + s->BlasInstanceCount);
    ctx->nodeBytes = nodeBytes;
    if ((rc = configure_launches(ctx))) return rc;
    if ((rc = set_l2_window(ctx, ctx->nodes.p, nodeBytes + triRecBytes))) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->haveScene = true;
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

IDKPT_API int idkpt_update_range(IdkPtCtx* ctx, IdkPtArrayId which, uint64_t first, uint64_t count, const void* data) {
    if (!ctx || !data) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_update_range: null argument");
    DRAIN_PENDING("idkpt_update_range");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_update_range: no scene");
    CK(cudaSetDevice(ctx->device));
    DevBuf* b = nullptr;
    size_t elem = 0;
    uint64_t limit = 0;
    switch (which) {
        case IDKPT_ARRAY_MESH_TRANSFORMS: b = &ctx->xforms; elem = sizeof(GpuMeshTransform); limit = ctx->counts.MeshTransformCount; break;
        case IDKPT_ARRAY_MESHES: b = &ctx->meshes; elem = sizeof(GpuMesh); limit = ctx->counts.MeshCount; break;
        case IDKPT_ARRAY_MATERIALS: b = &ctx->materials; elem = sizeof(GpuMaterial); limit = ctx->counts.MaterialCount; break;
        case IDKPT_ARRAY_LIGHTS: b = &ctx->lights; elem = sizeof(GpuLight); limit = ctx->counts.LightCount; break;
        case IDKPT_ARRAY_TLAS_NODES: b = &ctx->tlas; elem = sizeof(GpuTlasNode); limit = ctx->counts.UseTlas ? ctx->counts.TlasNodeCount : 0; break;
        default: return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_update_range: unknown array id");
    }
    if (first > limit || count > limit - first) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_update_range: range outside the array");
    if (which == IDKPT_ARRAY_MESHES) {
        const GpuMesh* m = (const GpuMesh*)data;
        for (uint64_t i = 0; i < count; i++)
            if (m[i].MaterialId < 0 || (uint64_t)m[i].MaterialId >= ctx->counts.MaterialCount)
                return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_update_range: GpuMesh.MaterialId out of range");
    }
    if (which == IDKPT_ARRAY_TLAS_NODES) {
        const GpuTlasNode* t = (const GpuTlasNode*)data;
        if (!tlas_nodes_valid(t, first, count, ctx->counts.TlasNodeCount, ctx->counts.BlasInstanceCount))
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_update_range: malformed TLAS node (child / instance id out of range)");
        if (first == 0 && count == ctx->counts.TlasNodeCount && tlas_height(t, count) > IDK_TLAS_STACK_SIZE)
            return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_update_range: TLAS deeper than the 24-entry traversal stack of the TLAS walk (BVHIntersect.glsl:4)");
    }
    if (which == IDKPT_ARRAY_MATERIALS) {
        const GpuMaterial* m = (const GpuMaterial*)data;
        for (uint64_t i = 0; i < count; i++)
            if (const char* err = validate_material_textures(m[i], ctx->counts.TextureCount, "idkpt_update_range: material texture handle outside the texture table"))
                return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, err);
        for (uint64_t i = 0; i < count; i++) ctx->hostMaterialMaxHandle[first + i] = material_max_handle(m[i]);
    }
    CK(cudaMemcpyAsync((char*)b->p + first * elem, data, count * elem, cudaMemcpyHostToDevice, ctx->stream));
    if (which == IDKPT_ARRAY_LIGHTS) std::copy((const GpuLight*)data, (const GpuLight*)data + count, ctx->hostLights.begin() + first);
    if ((which == IDKPT_ARRAY_MESHES || which == IDKPT_ARRAY_MATERIALS) && ctx->counts.MeshCount) {
        const uint32_t nm = (uint32_t)ctx->counts.MeshCount;   // refresh the per-mesh surface records
        k_prepare_surfaces<<<(nm + 255) / 256, 256, 0, ctx->stream>>>((const GpuMesh*)ctx->meshes.p, (const GpuMaterial*)ctx->materials.p, (float4*)ctx->surfRec.p, nm);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

IDKPT_API int idkpt_set_sky(IdkPtCtx* ctx, const IdkPtSkyDesc* sky) {
    if (!ctx || !sky) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_sky: null argument");
    DRAIN_PENDING("idkpt_set_sky");
    if (sky->FaceSize < 0 || sky->FaceSize > 8192) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_sky: invalid FaceSize");
    CK(cudaSetDevice(ctx->device));
    if (sky->FaceSize > 0) {
        const size_t faceBytes = (size_t)sky->FaceSize * sky->FaceSize * 16;
        for (int i = 0; i < 6; i++) if (!sky->Faces[i]) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_sky: a cubemap face is null");
        CK(ensure(ctx->skyFaces, 6 * faceBytes));
        for (int i = 0; i < 6; i++) CK(cudaMemcpyAsync((char*)ctx->skyFaces.p + i * faceBytes, sky->Faces[i], faceBytes, cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    ctx->skyFaceSize = sky->FaceSize;
    for (int i = 0; i < 3; i++) ctx->sky[i] = sky->Color[i];
    ctx->sc.skyR = ctx->sky[0]; ctx->sc.skyG = ctx->sky[1]; ctx->sc.skyB = ctx->sky[2];
    ctx->sc.skyFaces = ctx->skyFaceSize ? (const float4*)ctx->skyFaces.p : nullptr;
    ctx->sc.skyFaceSize = ctx->skyFaceSize;
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

} // extern "C"

// ---- the sky generated on the device (SkyBoxManager: AtmosphericScatterer.Compute, LoadSkyBoxEquirectangular) -----------------
// Runs `launch(faces)` over the 6 x n x n grid into the sky's allocation when it is large enough, else into a new one that
// replaces it only once the kernel has succeeded, then leaves the context as idkpt_set_sky would with those faces.
template <class Launch>
static int sky_generate(IdkPtCtx* ctx, const char* who, int n, float* kernelMs, Launch&& launch) {
    const size_t bytes = 6 * (size_t)n * n * 16;
    DevBuf fresh;
    if (bytes > ctx->skyFaces.bytes && ensure(fresh, bytes) != cudaSuccess) {
        release(fresh);
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    }
    float4* faces = (float4*)(fresh.p ? fresh.p : ctx->skyFaces.p);
    const dim3 grid((unsigned)((n + 7) / 8), (unsigned)((n + 7) / 8), 6), block(8, 8);
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int { launch(grid, block, faces); return IDKPT_OK; });
    if (rc != IDKPT_OK) { release(fresh); return rc; }
    if (fresh.p) { release(ctx->skyFaces); ctx->skyFaces = fresh; }
    ctx->skyFaceSize = n;
    ctx->sc.skyFaces = (const float4*)ctx->skyFaces.p;
    ctx->sc.skyFaceSize = n;
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

extern "C" {

IDKPT_API int idkpt_sky_atmosphere(IdkPtCtx* ctx, const IdkPtAtmosphereSettings* s, int32_t faceSize, float* kernelMs) {
    static const char* who = "idkpt_sky_atmosphere";
    if (!ctx || !s) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_sky_atmosphere: null argument");
    DRAIN_PENDING(who);
    if (faceSize < 1 || faceSize > 8192) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "face size outside 1..8192");
    if (s->ISteps < 1 || s->ISteps > 1024 || s->JSteps < 1 || s->JSteps > 1024)
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "ISteps or JSteps outside 1..1024");
    if (!std::isfinite(s->LightIntensity) || !std::isfinite(s->Azimuth) || !std::isfinite(s->Elevation))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a setting is not finite");
    CK(cudaSetDevice(ctx->device));
    if (kernelMs) *kernelMs = 0.0f;
    SkyAtmosphereArgs a;
    a.n = faceSize;
    a.iSteps = s->ISteps; a.jSteps = s->JSteps;
    a.lightIntensity = std::max(s->LightIntensity, 0.0f);   // AtmosphericScatterer.Compute
    a.azimuth = s->Azimuth; a.elevation = s->Elevation;
    return sky_generate(ctx, who, faceSize, kernelMs, [&](dim3 grid, dim3 block, float4* faces) {
        a.faces = faces;
        k_sky_atmosphere<<<grid, block, 0, ctx->stream>>>(a);
    });
}

IDKPT_API int idkpt_sky_equirectangular(IdkPtCtx* ctx, const float* rgb, int32_t width, int32_t height, float* kernelMs) {
    static const char* who = "idkpt_sky_equirectangular";
    if (!ctx || !rgb) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_sky_equirectangular: null argument");
    DRAIN_PENDING(who);
    if (width < 4 || height < 1 || width / 4 > 8192)
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "width outside 4..32771 (face size width / 4 in 1..8192) or height below 1");
    CK(cudaSetDevice(ctx->device));
    if (kernelMs) *kernelMs = 0.0f;
    const size_t srcBytes = (size_t)width * height * 12;
    DevBuf src;                    // the source lives for this call only: an import is a one-off, and it can be large
    if (ensure(src, srcBytes) != cudaSuccess) { release(src); return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed"); }
    cudaError_t e = cudaMemcpyAsync(src.p, rgb, srcBytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) { release(src); return fail(ctx, who, IDKPT_ERR_CUDA, cudaGetErrorString(e)); }
    SkyEquirectArgs a;
    a.rgb = (const float*)src.p;
    a.w = width; a.h = height;
    a.n = width / 4;               // SkyBoxManager.cs:124
    const int rc = sky_generate(ctx, who, a.n, kernelMs, [&](dim3 grid, dim3 block, float4* faces) {
        a.faces = faces;
        k_sky_equirect<<<grid, block, 0, ctx->stream>>>(a);
    });
    release(src);                  // run_timed synchronised the stream (or the call failed)
    return rc;
}

IDKPT_API int idkpt_read_sky(IdkPtCtx* ctx, int32_t* faceSize, float* dst, uint64_t bytes) {
    if (!ctx || !faceSize) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_sky: null argument");
    DRAIN_PENDING("idkpt_read_sky");
    const uint64_t need = 6 * (uint64_t)ctx->skyFaceSize * (uint64_t)ctx->skyFaceSize * 16;
    if (dst && bytes < need) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_sky: buffer smaller than 6 * FaceSize^2 * 16 bytes");
    *faceSize = ctx->skyFaceSize;
    if (dst && need) {
        CK(cudaSetDevice(ctx->device));
        CK(cudaMemcpyAsync(dst, ctx->skyFaces.p, need, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return IDKPT_OK;
}

// Replaces the texture table (SURVEY 8b idkpt_set_textures): e.g. streamed-in higher-resolution images. Handles already
// stored in the materials must stay valid.
IDKPT_API int idkpt_set_textures(IdkPtCtx* ctx, const IdkPtTextureDesc* textures, uint64_t count) {
    if (!ctx || (!textures && count)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_textures: null argument");
    DRAIN_PENDING("idkpt_set_textures");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_set_textures: no scene");
    IdkPtSceneDesc tmp = {};
    tmp.Textures = textures; tmp.TextureCount = count;
    if (const char* terr = idk_validate_textures(&tmp)) return texture_error(ctx, "idkpt_set_textures", terr);
    for (uint64_t h : ctx->hostMaterialMaxHandle)
        if (h > count) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_textures: a material references a texture beyond the new table");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    int rc = upload_textures(ctx, ctx->tex, textures, count);
    if (rc) return rc;
    ctx->sc.textures = (const TexRec*)ctx->tex.recs.p;
    ctx->sc.textureCount = (uint32_t)count;
    ctx->sc.srgbLut = (const float*)ctx->tex.srgbLut.p;
    ctx->counts.TextureCount = count;
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

IDKPT_API int idkpt_resize(IdkPtCtx* ctx, int32_t width, int32_t height) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    DRAIN_PENDING("idkpt_resize");
    if (width <= 0 || height <= 0 || width > 16384 || height > 16384) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_resize: invalid size");
    if (ctx->globalSlots && ctx->tileCount > 1 && (height + ctx->stripeH - 1) / ctx->stripeH > IDK_MAX_STRIPES)
        return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_resize: IDKPT_CREATE_GLOBAL_SLOTS supports at most 4096 stripes");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    if (ctx->copyPending) { CK(cudaEventSynchronize(ctx->copyDone)); ctx->copyPending = false; }
    gather_teardown(ctx);   // the exported full-frame buffers have the old size: peers must export / import again
    ctx->haveDenoised = false;
    for (int i = 0; i < 4; i++) release(ctx->oidn[i]);
    release(ctx->denoiseWork[0]); release(ctx->denoiseWork[1]); release(ctx->denoised);
    ctx->width = width;
    ctx->height = height;
    compute_tile_rows(ctx);
    int rc = allocate_wavefront(ctx);
    if (rc) return rc;
    for (int i = 0; i < IDK_MAX_LANES; i++) {
        release(ctx->lanes[i].keys);
        release(ctx->lanes[i].keysTmp);
        release(ctx->lanes[i].sortedAlive);
    }
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

IDKPT_API int idkpt_reset_accumulation(IdkPtCtx* ctx) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

IDKPT_API uint32_t idkpt_accumulated_samples(IdkPtCtx* ctx) { return ctx ? ctx->accumulatedSamples : 0; }

IDKPT_API int idkpt_set_accumulated_samples(IdkPtCtx* ctx, uint32_t n) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    ctx->accumulatedSamples = n;
    return IDKPT_OK;
}

struct EventPool {
    IdkPtCtx* ctx;
    size_t used = 0;
    struct Span { size_t a, b; int cat; int bounce; };
    std::vector<Span> spans;
    bool enabled;
    cudaEvent_t get() {
        if (used == ctx->events.size()) {
            cudaEvent_t e;
            cudaEventCreate(&e);
            ctx->events.push_back(e);
        }
        return ctx->events[used++];
    }
    size_t begin() {
        if (!enabled) return 0;
        size_t i = used;
        cudaEventRecord(get(), ctx->stream);
        return i;
    }
    void end(size_t a, int cat, int bounce = -1) {
        if (!enabled) return;
        size_t i = used;
        cudaEventRecord(get(), ctx->stream);
        spans.push_back({a, i, cat, bounce});
    }
};

IDKPT_API int idkpt_stream_handle(IdkPtCtx* ctx, void** stream) {
    if (!ctx || !stream) return IDKPT_ERR_INVALID_ARGUMENT;
    *stream = (void*)ctx->stream;
    return IDKPT_OK;
}

IDKPT_API int idkpt_sync(IdkPtCtx* ctx) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    CK(cudaSetDevice(ctx->device));
    return check_device_errors(ctx, drain(ctx), "idkpt_sync");
}

IDKPT_API int idkpt_compute(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtSettings* st, IdkPtStats* stats) {
    if (!ctx || !frame || !st) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_compute: null argument");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_compute: idkpt_set_scene has not been called");
    if (st->RayDepth < 1 || st->RayDepth > IDKPT_MAX_RAY_DEPTH) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_compute: RayDepth out of range");
    if (st->SamplesPerPixel < 1) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_compute: SamplesPerPixel must be >= 1");
    CK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(*stats));
    const uint32_t n = ctx->nLocal;
    if (n == 0) { ctx->accumulatedSamples += st->SamplesPerPixel; return IDKPT_OK; }

    const bool wantStats = st->CollectStats != 0 || st->Gpu.DoDebugBVHTraversal != 0;
    const bool sorting = st->DoRaySorting != 0;
    const bool aovs = st->OutputAOVs != 0;
    // stats == NULL: asynchronous. Samples are issued round-robin onto the lanes and the call returns without waiting
    // (idkpt_sync, or any call that reads device data, waits). With stats the call is synchronous and runs one sample at
    // a time on lane 0, exactly the sequence the per-kernel timings describe.
    const bool async = stats == nullptr && !wantStats && !ctx->exportEnabled && ctx->laneCount > 1;
    const bool globalSlots = ctx->globalSlots && ctx->tileCount > 1;
    if (globalSlots && ctx->gatherWorld < 2)
        return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_compute: IDKPT_CREATE_GLOBAL_SLOTS needs the peers connected (idkpt_gather_import / idkpt_gather_connect)");
    if (globalSlots && sorting)
        return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_compute: ray sorting reorders the slots by a tile-local key sort; not available with IDKPT_CREATE_GLOBAL_SLOTS");
    if (!async && ctx->asyncPending) {
        int rc = check_device_errors(ctx, drain(ctx), "idkpt_compute");
        if (rc) return rc;
    }

    FrameParams f;
    memcpy(f.invProj, frame->InvProjection, sizeof(f.invProj));
    memcpy(f.invView, frame->InvView, sizeof(f.invView));
    memcpy(f.viewPos, frame->ViewPos, sizeof(f.viewPos));
    f.focalLength = st->Gpu.FocalLength;
    f.lenseRadius = st->Gpu.LenseRadius;
    f.width = ctx->width; f.height = ctx->height;
    f.stripeH = ctx->stripeH; f.tileIndex = ctx->tileIndex; f.tileCount = ctx->tileCount;
    f.doDebugTraversal = st->Gpu.DoDebugBVHTraversal;
    f.doTraceLights = st->Gpu.DoTraceLights;
    f.doRussianRoulette = st->Gpu.DoRussianRoulette;

    EventPool ev{ctx, 0, {}, stats != nullptr};
    const size_t evTotal = ev.begin();
    uint32_t launches = 0, traverseLaunches = 0;
    std::vector<uint32_t> hostCounts(stats ? (size_t)st->SamplesPerPixel * (IDKPT_MAX_RAY_DEPTH + 1) : 0, 0);
    DevBuf& countLog = ctx->countLog;   // per-sample copy of counts for the stats (device-side, read once at the end)
    if (stats) CK(ensure(countLog, hostCounts.size() * sizeof(uint32_t)));
    if (wantStats) CK(cudaMemsetAsync(ctx->counters.p, 0, sizeof(TraceCounters), ctx->stream));

    const int accBlocks = std::min<int>((int)((n + IDK_BLOCK - 1) / IDK_BLOCK), ctx->smCount * 8);

    for (int s = 0; s < st->SamplesPerPixel; s++) {
        Lane& ln = ctx->lanes[async ? ctx->nextLane : 0];
        if (async) {
            ctx->nextLane = (ctx->nextLane + 1) % ctx->laneCount;
            if (!ln.allocated)   // first asynchronous call (or first after a resize): bring up every lane now, not one per call
                for (int i = 0; i < ctx->laneCount; i++)
                    if (!ctx->lanes[i].allocated) { int rc = allocate_lane(ctx, ctx->lanes[i]); if (rc) return rc; }
            if (ln.accPending) CK(cudaStreamWaitEvent(ln.stream, ln.accDone, 0));   // its previous sample's radiance has been consumed
        }
        const cudaStream_t ls = async ? ln.stream : ctx->stream;   // the wavefront chain of this sample
        if (sorting) {
            CK(ensure(ln.keys, (size_t)n * 4));
            CK(ensure(ln.keysTmp, (size_t)n * 4));
            CK(ensure(ln.sortedAlive, (size_t)n * 4));
            if (idk_sort_prepare(ln.sortScratch, n)) return fail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkpt_compute: sort scratch allocation failed");
        }
        uint32_t* counts = (uint32_t*)ln.countsDev.p;
        uint32_t* tickets = (uint32_t*)ln.tickets.p;
        f.accumulatedSamples = ctx->accumulatedSamples;
        // zero the alive counts and work tickets, counts[0] = n (every pixel of the tile traces a primary ray)
        k_init_sample<<<1, 256, 0, ls>>>(counts, IDKPT_MAX_RAY_DEPTH + 1, tickets, 2 * (IDKPT_MAX_RAY_DEPTH + 1), n);
        launches++;

        size_t e0 = 0;
        for (int j = 0; j < st->RayDepth; j++) {
            const bool first = j == 0;
            const bool last = j == st->RayDepth - 1;
            // alive list of this bounce: slot -> tile pixel (none for the first hit: its slot is the tile pixel)
            const uint32_t* alive = first ? nullptr : (const uint32_t*)ln.alive[j & 1].p;
            if (sorting && j > 1) {
                // PathTracer.RaySorting(), PathTracer.cs:273-297: stable sort of the alive list by cached key
                e0 = ev.begin();
                int nl = idk_sort_by_key(ln.sortScratch, (const uint32_t*)ln.keys.p, alive, (uint32_t*)ln.sortedAlive.p, counts + j, n, ctx->smCount, ls);
                ev.end(e0, 2);
                if (nl < 0) return fail(ctx, IDKPT_ERR_CUDA, "idkpt_compute: sort launch failed");
                launches += (uint32_t)nl;
                alive = (const uint32_t*)ln.sortedAlive.p;
            }

            if (globalSlots && !first) {
                // per-stripe alive counts of this bounce to every peer, everybody's counts back: global slot = local slot + delta[stripe]
                SlotExchangeArgs xa;
                memset(&xa, 0, sizeof(xa));
                // 32-bit epoch (~20 days at 2,400 exchanges per second and lane). Wrap: 0 means "nothing published" and the parity
                // must keep alternating (0xFFFFFFFF is odd), so the successor of 0xFFFFFFFF is 2. A table word always holds the
                // epoch of two exchanges ago, so a reused value can never be mistaken for the current one.
                if (++ln.slotEpoch == 0u) ln.slotEpoch = 2u;
                const uint32_t epoch = ln.slotEpoch;
                const size_t laneIdx = (size_t)(&ln - ctx->lanes);
                for (int p = 0; p < ctx->gatherWorld; p++)
                    xa.peerTable[p] = (unsigned long long*)ctx->peerSlotTable[p] + (laneIdx * 2 + (epoch & 1u)) * (size_t)ctx->nStripes;
                xa.alive = alive; xa.count = counts + j;
                xa.delta = (uint32_t*)ln.slotDelta.p;
                xa.timedOut = (uint32_t*)ctx->gatherScratch.p + 1;
                xa.timeoutCycles = (long long)(ctx->gatherTimeoutMs * (double)ctx->clockKHz);
                xa.epoch = epoch;
                xa.world = ctx->gatherWorld; xa.rank = ctx->gatherRank;
                xa.stripePixels = (uint32_t)ctx->stripeH * (uint32_t)ctx->width;
                xa.nLocalStripes = (uint32_t)ctx->nLocalStripes; xa.nStripes = (uint32_t)ctx->nStripes;
                k_slot_exchange<<<1, 256, 0, ls>>>(xa);
                launches++;
            }

            ShadeArgs sa;
            sa.sc = ctx->sc;
            sa.f = f;
            sa.state = (PathState*)ln.state.p;
            sa.aov = (float4*)ln.aov.p;
            sa.alive = alive;
            sa.hits = (const HitRec*)ln.hits.p;
            sa.hitXform = (const uint32_t*)ln.hitXform.p;
            sa.count = counts + j;
            sa.survivors = (uint32_t*)ln.survivors.p;
            sa.keysTmp = sorting ? (uint32_t*)ln.keysTmp.p : nullptr;
            sa.radiance = (float4*)ln.radiance.p;
            sa.aovAlbedoFinal = (float4*)ln.aovAlbedoFinal.p;
            sa.aovNormalFinal = (float4*)ln.aovNormalFinal.p;
            sa.slotDelta = (globalSlots && !first) ? (const uint32_t*)ln.slotDelta.p : nullptr;
            sa.stripePixels = (uint32_t)ctx->stripeH * (uint32_t)ctx->width;
            sa.exportState = ctx->exportEnabled ? 1 : 0;
            sa.lastBounce = last ? 1 : 0;
            sa.outputAovs = aovs ? 1 : 0;
            const int tex = ctx->sc.textureCount ? 1 : 0;

            // bounce 0 is one kernel (camera rays, closest hit, FirstHit shading), timed as its traversal
            e0 = ev.begin();
            if (first) {
                FirstHitArgs fa;
                fa.s = sa;
                fa.ticket = tickets;
                fa.counters = (TraceCounters*)ctx->counters.p;
                fa.rows = n / (uint32_t)ctx->width;
                const int fb = wantStats ? ctx->firstHitBlocks[1][tex] : async ? ctx->firstHitBlocksLane[tex] : ctx->firstHitBlocks[0][tex];
                kFirstHit[ctx->sc.useTlas ? 1 : 0][wantStats ? 1 : 0][tex]<<<fb, IDK_BLOCK, ctx->stackBytes, ls>>>(fa);
            } else {         // every later bounce: phase-scheduled warps
                TraverseArgs ta;
                ta.sc = ctx->sc;
                ta.state = (const PathState*)ln.state.p;
                ta.perm = alive;
                ta.count = counts + j;
                ta.ticket = tickets + 2 * j;
                ta.hits = (HitRec*)ln.hits.p;
                ta.hitXform = (uint32_t*)ln.hitXform.p;
                ta.debugCost = (float*)ln.debugCost.p;
                ta.counters = (TraceCounters*)ctx->counters.p;
                ta.traceLights = st->Gpu.DoTraceLights;
                ta.bounce = j;
                const int tb = async ? ctx->traverseBlocksLane : ctx->traverseBlocks;
                const TraverseTuning tune = {IDK_T2_SETUP_THRESHOLD, IDK_T2_LEAF_THRESHOLD, async ? 1 : 0};
                if (ctx->sc.useTlas) {       // the TLAS walk is a fourth phase of the production kernel (BVHIntersect.glsl:205-272)
                    if (wantStats) k_traverse2<true, true><<<ctx->traverseBlocksStats, IDK_T2_BLOCK, ctx->traverse2Smem, ls>>>(ta, tune);
                    else k_traverse2<false, true><<<tb, IDK_T2_BLOCK, ctx->traverse2Smem, ls>>>(ta, tune);
                } else {
                    if (wantStats) k_traverse2<true, false><<<ctx->traverseBlocksStats, IDK_T2_BLOCK, ctx->traverse2Smem, ls>>>(ta, tune);
                    else k_traverse2<false, false><<<tb, IDK_T2_BLOCK, ctx->traverse2Smem, ls>>>(ta, tune);
                }
            }
            ev.end(e0, 0, j);
            launches++;
            traverseLaunches++;

            e0 = ev.begin();
            if (!first) {
                if (tex) k_shade<true><<<ctx->shadeBlocks, IDK_BLOCK, 0, ls>>>(sa);
                else k_shade<false><<<ctx->shadeBlocks, IDK_BLOCK, 0, ls>>>(sa);
                launches++;
            }
            if (!last) {
                CompactArgs ca;
                ca.survivors = (const uint32_t*)ln.survivors.p;
                ca.keysTmp = sorting ? (const uint32_t*)ln.keysTmp.p : nullptr;
                ca.count = counts + j;
                ca.aliveOut = (uint32_t*)ln.alive[(j + 1) & 1].p;
                ca.keysOut = sorting ? (uint32_t*)ln.keys.p : nullptr;
                ca.countOut = counts + j + 1;
                ca.ticket = tickets + 2 * j + 1;
                ca.tileStatus = (unsigned long long*)ln.tileStatus.p;
                if (ln.epoch >= IDK_EPOCH_MASK) {   // 30-bit epoch wrapped: clear this lane's status words (ordered on its stream) and restart at 1
                    CK(cudaMemsetAsync(ln.tileStatus.p, 0, ln.tileStatus.bytes, ls));
                    ln.epoch = 0;
                }
                ca.epoch = ++ln.epoch;
                const size_t ec = ev.begin();
                k_compact<<<ctx->compactBlocks, IDK_BLOCK, 0, ls>>>(ca);
                ev.end(ec, 5);
                launches++;
            }
            ev.end(e0, 1, j);
        }

        // FinalDraw runs on the main (image) stream in issue order: samples accumulate in the order they were submitted
        // whichever lane finishes first, and presents / read-backs queued on the main stream see a consistent image.
        if (async) {
            CK(cudaEventRecord(ln.radianceReady, ls));
            CK(cudaStreamWaitEvent(ctx->stream, ln.radianceReady, 0));
        }
        e0 = ev.begin();
        const bool gatherNow = ctx->gatherWorld > 1 && s == st->SamplesPerPixel - 1;
        if (gatherNow) {
            // FinalDraw fused with the all-gather: Result pixels go straight to every rank's full image over NVLink
            const int b = (int)((ctx->gatherEpoch + 1) & 1u);
            GatherArgs g;
            memset(&g, 0, sizeof(g));
            for (int p = 0; p < ctx->gatherWorld; p++) { g.peerImage[p] = (float4*)ctx->peerImage[b][p]; g.peerFlags[p] = (uint32_t*)ctx->peerFlags[b][p]; }
            g.tileRows = (const int*)ctx->gatherRows.p;
            g.doneCounter = (uint32_t*)ctx->gatherScratch.p;
            g.world = ctx->gatherWorld; g.rank = ctx->gatherRank; g.width = ctx->width;
            g.epoch = ++ctx->gatherEpoch;
            CK(cudaMemsetAsync(ctx->gatherScratch.p, 0, 4, ctx->stream));
            k_accumulate_scatter<<<accBlocks, IDK_BLOCK, 0, ctx->stream>>>((const float4*)ln.radiance.p, (float4*)ctx->images[0].p, n,
                                                                           ctx->accumulatedSamples, st->Gpu.DoDebugBVHTraversal, g);
            if (aovs)   // AOV images stay local to the tile (only Result is gathered)
                k_accumulate_aov<<<accBlocks, IDK_BLOCK, 0, ctx->stream>>>((const float4*)ln.aovAlbedoFinal.p, (const float4*)ln.aovNormalFinal.p,
                                                                           (float4*)ctx->images[1].p, (float4*)ctx->images[2].p, n, ctx->accumulatedSamples);
            if (async) { CK(cudaEventRecord(ln.accDone, ctx->stream)); ln.accPending = true; }   // before the arrival wait: the lane may go on
            k_gather_wait<<<1, 32, 0, ctx->stream>>>((const uint32_t*)ctx->gatherFlags[b].p, ctx->gatherWorld, g.epoch, (uint32_t*)ctx->gatherScratch.p + 1,
                                                     (long long)(ctx->gatherTimeoutMs * (double)ctx->clockKHz));
            ctx->gatherCurrent = b;
            launches += aovs ? 3 : 2;
        } else {
            k_accumulate<<<accBlocks, IDK_BLOCK, 0, ctx->stream>>>((const float4*)ln.radiance.p, (const float4*)ln.aovAlbedoFinal.p,
                                                                   (const float4*)ln.aovNormalFinal.p, (float4*)ctx->images[0].p,
                                                                   (float4*)ctx->images[1].p, (float4*)ctx->images[2].p, n,
                                                                   ctx->accumulatedSamples, st->Gpu.DoDebugBVHTraversal, aovs ? 1 : 0);
            if (async) { CK(cudaEventRecord(ln.accDone, ctx->stream)); ln.accPending = true; }
            launches++;
        }
        ev.end(e0, 3);
        ev.end(e0, 6);
        if (stats) CK(cudaMemcpyAsync((uint32_t*)countLog.p + (size_t)s * (IDKPT_MAX_RAY_DEPTH + 1), counts,
                                      (IDKPT_MAX_RAY_DEPTH + 1) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
        ctx->accumulatedSamples++;   // PathTracer.cs:269
    }
    ev.end(evTotal, 4);
    CK(cudaGetLastError());
    if (async) {
        ctx->asyncPending = true;
        return IDKPT_OK;
    }
    {
        int rc = check_device_errors(ctx, cudaStreamSynchronize(ctx->stream), "idkpt_compute");
        if (rc) return rc;
    }
    if (stats) {
        CK(cudaMemcpy(hostCounts.data(), countLog.p, hostCounts.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        for (int s = 0; s < st->SamplesPerPixel; s++)
            for (int j = 0; j < st->RayDepth; j++) {
                const uint64_t c = hostCounts[(size_t)s * (IDKPT_MAX_RAY_DEPTH + 1) + j];
                stats->BounceRays[j] += c;
                stats->Rays += c;
            }
        if (wantStats) {
            TraceCounters tc;
            CK(cudaMemcpy(&tc, ctx->counters.p, sizeof(tc), cudaMemcpyDeviceToHost));
            stats->NodePairFetches = tc.steps;
            stats->TriangleTests = tc.tris;
            stats->InstanceVisits = tc.instances;
            stats->Hits = tc.hits;
            for (int j = 0; j < IDKPT_MAX_RAY_DEPTH; j++) stats->BounceMaxSteps[j] = tc.maxSteps[j];
        }
        for (const EventPool::Span& sp : ev.spans) {
            float ms = 0.0f;
            cudaEventElapsedTime(&ms, ctx->events[sp.a], ctx->events[sp.b]);
            switch (sp.cat) {
                case 0: stats->TraverseMs += ms; if (sp.bounce >= 0) stats->BounceTraverseMs[sp.bounce] += ms; break;
                case 1: stats->ShadeMs += ms; if (sp.bounce >= 0) stats->BounceShadeMs[sp.bounce] += ms; break;
                case 2: stats->SortMs += ms; break;
                case 3: stats->OtherMs += ms; break;
                case 5: stats->CompactMs += ms; break;
                case 6: stats->AccumulateMs += ms; break;
                default: stats->TotalMs = ms; break;
            }
        }
        stats->KernelLaunches = launches;
        stats->TraverseLaunches = traverseLaunches;
    }
    return IDKPT_OK;
}

static int image_copy(IdkPtCtx* ctx, IdkPtImage which, void* host, uint64_t bytes, bool toHost) {
    if (!ctx || !host) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt image copy: null argument");
    if (which == IDKPT_IMAGE_DENOISED) {
        if (!toHost || !ctx->haveDenoised) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt image copy: no denoised image (call idkpt_denoise)");
        if (bytes < (uint64_t)ctx->width * ctx->height * 16) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt image copy: buffer smaller than width*height*16");
        CK(cudaSetDevice(ctx->device));
        CK(cudaMemcpyAsync(host, ctx->denoised.p, (size_t)ctx->width * ctx->height * 16, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        return IDKPT_OK;
    }
    if ((int)which < 0 || (int)which > 2) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt image copy: unknown image");
    if (bytes < (uint64_t)ctx->width * ctx->height * 16) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt image copy: buffer smaller than width*height*16");
    CK(cudaSetDevice(ctx->device));
    const size_t rowBytes = (size_t)ctx->width * 16;
    // owned rows are stored compactly; copy stripe by stripe into the full-image layout
    size_t i = 0;
    while (i < ctx->rows.size()) {
        size_t j = i;
        while (j + 1 < ctx->rows.size() && ctx->rows[j + 1] == ctx->rows[j] + 1) j++;
        char* h = (char*)host + (size_t)ctx->rows[i] * rowBytes;
        char* d = (char*)ctx->images[which].p + i * rowBytes;
        if (toHost) CK(cudaMemcpyAsync(h, d, (j - i + 1) * rowBytes, cudaMemcpyDeviceToHost, ctx->stream));
        else CK(cudaMemcpyAsync(d, h, (j - i + 1) * rowBytes, cudaMemcpyHostToDevice, ctx->stream));
        i = j + 1;
    }
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

IDKPT_API int idkpt_read_result(IdkPtCtx* ctx, IdkPtImage which, void* dst, uint64_t bytes) { return image_copy(ctx, which, dst, bytes, true); }
IDKPT_API int idkpt_write_result(IdkPtCtx* ctx, IdkPtImage which, const void* src, uint64_t bytes) { return image_copy(ctx, which, (void*)src, bytes, false); }

// Present without stalling the renderer: snapshot the image on the device (ordered after the Compute that produced it)
// and copy the snapshot to (ideally pinned) host memory on a second stream, so the transfer overlaps the next Compute.
IDKPT_API int idkpt_present_async(IdkPtCtx* ctx, IdkPtImage which, void* dstHost, uint64_t bytes) {
    if (!ctx || !dstHost) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_present_async: null argument");
    if ((int)which < 0 || (int)which > 3) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_present_async: unknown image");
    if (bytes < (uint64_t)ctx->width * ctx->height * 16) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_present_async: buffer smaller than width*height*16");
    CK(cudaSetDevice(ctx->device));
    // IDKPT_IMAGE_GATHERED is the full multi-GPU frame. It is snapshot on the main stream too: with several frames in flight a
    // peer may start scattering frame k+2 into this buffer as soon as every rank has finished frame k+1, and that is ordered
    // after this snapshot (main stream: wait(k) -> snapshot(k) -> scatter(k+1)) but not after a slow D2H copy.
    const bool gathered = (int)which == 3;
    if (gathered && (ctx->gatherWorld < 2 || ctx->gatherCurrent < 0)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_present_async: no gathered frame yet");
    if (!ctx->copyStream) {
        CK(cudaStreamCreateWithFlags(&ctx->copyStream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&ctx->snapDone, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&ctx->copyDone, cudaEventDisableTiming));
    }
    const size_t n = gathered ? (size_t)ctx->width * ctx->height * 16 : (size_t)ctx->nLocal * 16;
    CK(ensure(ctx->presentSnap, std::max<size_t>(n, 16)));
    if (ctx->copyPending) CK(cudaStreamWaitEvent(ctx->stream, ctx->copyDone, 0));   // previous transfer still reads the snapshot
    CK(cudaMemcpyAsync(ctx->presentSnap.p, gathered ? ctx->gatherImage[ctx->gatherCurrent].p : ctx->images[which].p, n, cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaEventRecord(ctx->snapDone, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->copyStream, ctx->snapDone, 0));
    // The tile's rows are stored compactly, stripe after stripe; in the full-frame host layout its stripes are tileCount stripes
    // apart: ONE strided (2-D) copy moves all complete stripes, a second one the partial last stripe of the image if it is ours.
    // With a host frame shared by all ranks (idkpt_register_host_buffer on the same mapping in every process) each GPU
    // delivers its own 1/N of the frame over its own PCIe link -- no rank has to download the whole gathered image.
    const size_t rowBytes = (size_t)ctx->width * 16;
    if (gathered) {
        CK(cudaMemcpyAsync(dstHost, ctx->presentSnap.p, n, cudaMemcpyDeviceToHost, ctx->copyStream));
    } else if (!ctx->rows.empty()) {
        const size_t stripeBytes = (size_t)ctx->stripeH * rowBytes;
        const size_t fullStripes = ctx->rows.size() / (size_t)ctx->stripeH, tailRows = ctx->rows.size() % (size_t)ctx->stripeH;
        char* h0 = (char*)dstHost + (size_t)ctx->rows[0] * rowBytes;
        if (fullStripes)
            CK(cudaMemcpy2DAsync(h0, stripeBytes * (size_t)ctx->tileCount, ctx->presentSnap.p, stripeBytes, stripeBytes, fullStripes,
                                 cudaMemcpyDeviceToHost, ctx->copyStream));
        if (tailRows)
            CK(cudaMemcpyAsync((char*)dstHost + (size_t)ctx->rows[fullStripes * ctx->stripeH] * rowBytes, (char*)ctx->presentSnap.p + fullStripes * stripeBytes,
                               tailRows * rowBytes, cudaMemcpyDeviceToHost, ctx->copyStream));
    }
    CK(cudaEventRecord(ctx->copyDone, ctx->copyStream));
    ctx->copyPending = true;
    return IDKPT_OK;
}

IDKPT_API int idkpt_present_wait(IdkPtCtx* ctx) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (ctx->copyPending) {
        CK(cudaSetDevice(ctx->device));
        CK(cudaEventSynchronize(ctx->copyDone));
        ctx->copyPending = false;
    }
    return IDKPT_OK;
}

// Page-lock a host buffer the engine owns (e.g. the POSIX shared-memory frame all ranks present into) so that
// idkpt_present_async's copies are truly asynchronous. The C# host has no CUDA runtime of its own to call cudaHostRegister.
IDKPT_API int idkpt_register_host_buffer(IdkPtCtx* ctx, void* hostPtr, uint64_t bytes) {
    if (!ctx || !hostPtr || !bytes) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_register_host_buffer: null argument");
    CK(cudaSetDevice(ctx->device));
    CK(cudaHostRegister(hostPtr, bytes, cudaHostRegisterPortable));
    return IDKPT_OK;
}

IDKPT_API int idkpt_unregister_host_buffer(IdkPtCtx* ctx, void* hostPtr) {
    if (!ctx || !hostPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_unregister_host_buffer: null argument");
    CK(cudaSetDevice(ctx->device));
    if (ctx->copyPending) { CK(cudaEventSynchronize(ctx->copyDone)); ctx->copyPending = false; }   // a transfer may still target it
    CK(cudaHostUnregister(hostPtr));
    return IDKPT_OK;
}

// ---- multi-GPU gather over peer memory -----------------------------------------------------------------------------
// Step 1 (every rank): allocate the exported buffers and return their CUDA IPC handles (4 x 64 bytes:
// image[0], image[1], flags[0], flags[1]). Step 2: exchange the handles (any transport) and import all ranks' handles.
// The buffers peers write into: full-size images + arrival flags (double-buffered), the per-stripe count tables of the
// global-slot exchange. Stand-alone cudaMalloc allocations (IPC export needs that).
// CUDA loads kernels lazily, and loading one may have to wait for the kernels that are running. Once contexts wait for each
// other ON THE DEVICE (arrival wait, slot exchange) a first launch from the host thread that still has to submit the peer's
// work would deadlock against them -- so everything a connected context can launch is loaded before the first wait exists.
__global__ void k_denoise_import(const float* __restrict__ rgb, float4* __restrict__ out, int count);
static int preload_kernels(IdkPtCtx* ctx) {
    cudaFuncAttributes fa;
#define IDK_PRELOAD(k) CK(cudaFuncGetAttributes(&fa, k))
    IDK_PRELOAD(k_init_sample); IDK_PRELOAD(k_prepare_triangles); IDK_PRELOAD(k_prepare_vertices); IDK_PRELOAD(k_prepare_surfaces);
    for (const auto& byStats : kFirstHit)
        for (const auto& byTex : byStats)
            for (FirstHitKernel k : byTex) IDK_PRELOAD(k);
    IDK_PRELOAD((k_traverse2<false, false>)); IDK_PRELOAD((k_traverse2<true, false>));
    IDK_PRELOAD((k_traverse2<false, true>)); IDK_PRELOAD((k_traverse2<true, true>));
    IDK_PRELOAD(k_shade<false>); IDK_PRELOAD(k_shade<true>); IDK_PRELOAD(k_compact); IDK_PRELOAD(k_slot_exchange);
    IDK_PRELOAD(k_accumulate); IDK_PRELOAD(k_accumulate_aov); IDK_PRELOAD(k_accumulate_scatter); IDK_PRELOAD(k_gather_wait);
    IDK_PRELOAD(k_sort_histogram); IDK_PRELOAD(k_sort_scan); IDK_PRELOAD(k_sort_scatter);
    IDK_PRELOAD(k_trace_rays); IDK_PRELOAD(k_trace_rays_any); IDK_PRELOAD(k_shadows_ray_traced);
    IDK_PRELOAD(k_skin_vertices); IDK_PRELOAD(k_refit_prepare); IDK_PRELOAD(k_refit_climb); IDK_PRELOAD(k_tlas_build);
    IDK_PRELOAD(k_tlas_leaves); IDK_PRELOAD(k_tlas_bounds); IDK_PRELOAD(k_tlas_keys); IDK_PRELOAD(k_tlas_ploc);
    IDK_PRELOAD(k_bloom_down); IDK_PRELOAD(k_bloom_up); IDK_PRELOAD(k_agx_matrices); IDK_PRELOAD(k_tonemap);
    IDK_PRELOAD(k_denoise_prepare); IDK_PRELOAD(k_denoise_atrous); IDK_PRELOAD(k_denoise_finish); IDK_PRELOAD(k_denoise_import);
    IDK_PRELOAD(k_bcn_decode); IDK_PRELOAD(k_point_shadow_faces); IDK_PRELOAD(k_volumetric_march); IDK_PRELOAD(k_volumetric_upscale);
    IDK_PRELOAD(k_ssao); IDK_PRELOAD(k_deferred_lighting); IDK_PRELOAD(k_ssr); IDK_PRELOAD(k_taa_resolve);
    IDK_PRELOAD(k_shading_rate); IDK_PRELOAD(k_vrs_scan); IDK_PRELOAD(k_deferred_lighting_vrs); IDK_PRELOAD(k_gbuffer);
    IDK_PRELOAD(k_transparency<false>); IDK_PRELOAD(k_transparency<true>); IDK_PRELOAD(k_lights_skybox);
    IDK_PRELOAD(k_sky_atmosphere); IDK_PRELOAD(k_sky_equirect);
#undef IDK_PRELOAD
    return IDKPT_OK;
}

static size_t slot_table_words(const IdkPtCtx* ctx) { return (size_t)IDK_MAX_LANES * 2 * (size_t)std::max(1, ctx->nStripes); }
static int gather_allocate(IdkPtCtx* ctx) {
    { int rc = preload_kernels(ctx); if (rc) return rc; }
    const size_t imgBytes = (size_t)ctx->width * ctx->height * 16;
    for (int b = 0; b < 2; b++) {
        CK(ensure(ctx->gatherImage[b], imgBytes));
        CK(ensure(ctx->gatherFlags[b], IDK_MAX_PEERS * sizeof(uint32_t)));
        CK(cudaMemsetAsync(ctx->gatherImage[b].p, 0, imgBytes, ctx->stream));
        CK(cudaMemsetAsync(ctx->gatherFlags[b].p, 0, IDK_MAX_PEERS * sizeof(uint32_t), ctx->stream));
    }
    // every lane is brought up NOW: once peers wait for each other on the device, a later allocation (an implicit device
    // synchronisation in the worst case) from the thread that still has to submit a peer's work could deadlock
    if (ctx->laneCount > 1)
        for (int i = 0; i < ctx->laneCount; i++)
            if (!ctx->lanes[i].allocated) { int rc = allocate_lane(ctx, ctx->lanes[i]); if (rc) return rc; }
    CK(ensure(ctx->slotTable, slot_table_words(ctx) * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(ctx->slotTable.p, 0, ctx->slotTable.bytes, ctx->stream));   // epoch 0 = nothing published
    CK(ensure(ctx->gatherScratch, 16));
    CK(cudaMemsetAsync(ctx->gatherScratch.p, 0, 16, ctx->stream));
    CK(ensure(ctx->gatherRows, std::max<size_t>(ctx->rows.size(), 1) * sizeof(int)));
    if (!ctx->rows.empty()) CK(cudaMemcpyAsync(ctx->gatherRows.p, ctx->rows.data(), ctx->rows.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

IDKPT_API int idkpt_gather_export(IdkPtCtx* ctx, void* handlesOut, uint64_t bytes) {
    if (!ctx || !handlesOut) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_export: null argument");
    DRAIN_PENDING("idkpt_gather_export");
    if (bytes < IDKPT_GATHER_HANDLE_BYTES) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_export: need IDKPT_GATHER_HANDLE_BYTES (320) bytes");
    CK(cudaSetDevice(ctx->device));
    { int rc = gather_allocate(ctx); if (rc) return rc; }
    cudaIpcMemHandle_t* out = (cudaIpcMemHandle_t*)handlesOut;
    for (int b = 0; b < 2; b++) {
        CK(cudaIpcGetMemHandle(&out[b], ctx->gatherImage[b].p));
        CK(cudaIpcGetMemHandle(&out[2 + b], ctx->gatherFlags[b].p));
    }
    CK(cudaIpcGetMemHandle(&out[4], ctx->slotTable.p));
    return IDKPT_OK;
}

// allHandles = world x 256 bytes in rank order (this rank's own entry is ignored and replaced by the local pointers).
IDKPT_API int idkpt_gather_import(IdkPtCtx* ctx, int32_t rank, int32_t world, const void* allHandles, uint64_t bytes) {
    if (!ctx || !allHandles) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_import: null argument");
    DRAIN_PENDING("idkpt_gather_import");
    if (world < 2 || world > IDK_MAX_PEERS || rank < 0 || rank >= world) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_import: invalid rank / world");
    if (world != ctx->tileCount || rank != ctx->tileIndex) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_import: rank / world must equal TileIndex / TileCount");
    if (bytes < (uint64_t)world * IDKPT_GATHER_HANDLE_BYTES) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_import: handle buffer too small");
    if (!ctx->gatherImage[0].p) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_import: call idkpt_gather_export first");
    if (ctx->gatherWorld > 1) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_import: peers are already connected (idkpt_resize disconnects them)");
    CK(cudaSetDevice(ctx->device));
    const cudaIpcMemHandle_t* hs = (const cudaIpcMemHandle_t*)allHandles;
    ctx->peerIsIpc = true;
    for (int p = 0; p < world; p++) {
        for (int b = 0; b < 2; b++) {
            if (p == rank) {
                ctx->peerImage[b][p] = ctx->gatherImage[b].p;
                ctx->peerFlags[b][p] = ctx->gatherFlags[b].p;
            } else {
                CK(cudaIpcOpenMemHandle(&ctx->peerImage[b][p], hs[5 * p + b], cudaIpcMemLazyEnablePeerAccess));
                CK(cudaIpcOpenMemHandle(&ctx->peerFlags[b][p], hs[5 * p + 2 + b], cudaIpcMemLazyEnablePeerAccess));
            }
        }
        if (p == rank) ctx->peerSlotTable[p] = ctx->slotTable.p;
        else CK(cudaIpcOpenMemHandle(&ctx->peerSlotTable[p], hs[5 * p + 4], cudaIpcMemLazyEnablePeerAccess));
        ctx->peerMapped[p] = true;
    }
    ctx->gatherWorld = world;
    ctx->gatherRank = rank;
    ctx->gatherEpoch = 0;
    ctx->gatherCurrent = -1;
    for (int i = 0; i < IDK_MAX_LANES; i++) ctx->lanes[i].slotEpoch = ctx->slotEpochStart;
    return IDKPT_OK;
}

// The same wiring for a host that drives all GPUs from ONE process (the reference engine is a single process): contexts
// [0, world) in tile order, each created with TileIndex = its position and TileCount = world. No IPC: the contexts hand each
// other their device pointers; peer access between different devices is enabled here.
IDKPT_API int idkpt_gather_connect(IdkPtCtx** ctxs, int32_t world) {
    if (!ctxs || world < 2 || world > IDK_MAX_PEERS) return fail(ctxs && world > 0 ? ctxs[0] : nullptr, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_connect: invalid argument");
    for (int r = 0; r < world; r++) {
        IdkPtCtx* ctx = ctxs[r];
        if (!ctx) return fail(ctxs[0], IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_connect: null context");
        if (ctx->tileCount != world || ctx->tileIndex != r) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_connect: context r must have TileIndex r and TileCount world");
        if (ctx->width != ctxs[0]->width || ctx->height != ctxs[0]->height || ctx->stripeH != ctxs[0]->stripeH || ctx->laneCount != ctxs[0]->laneCount ||
            ctx->globalSlots != ctxs[0]->globalSlots)
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_connect: contexts differ in size, stripe height, lanes or flags");
        DRAIN_PENDING("idkpt_gather_connect");
        if (ctx->gatherWorld > 1) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_connect: peers are already connected");
        CK(cudaSetDevice(ctx->device));
        int rc = gather_allocate(ctx);
        if (rc) return rc;
    }
    for (int r = 0; r < world; r++) {
        IdkPtCtx* ctx = ctxs[r];
        CK(cudaSetDevice(ctx->device));
        for (int p = 0; p < world; p++) {
            if (ctxs[p]->device != ctx->device) {
                int can = 0;
                CK(cudaDeviceCanAccessPeer(&can, ctx->device, ctxs[p]->device));
                if (!can) return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_gather_connect: no peer access between two of the devices");
                const cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[p]->device, 0);
                if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
                else CK(e);
            }
            for (int b = 0; b < 2; b++) {
                ctx->peerImage[b][p] = ctxs[p]->gatherImage[b].p;
                ctx->peerFlags[b][p] = ctxs[p]->gatherFlags[b].p;
            }
            ctx->peerSlotTable[p] = ctxs[p]->slotTable.p;
            ctx->peerMapped[p] = true;
        }
        ctx->peerIsIpc = false;
        ctx->gatherWorld = world;
        ctx->gatherRank = r;
        ctx->gatherEpoch = 0;
        ctx->gatherCurrent = -1;
        for (int i = 0; i < IDK_MAX_LANES; i++) ctx->lanes[i].slotEpoch = ctx->slotEpochStart;
    }
    return IDKPT_OK;
}

// Full image (all ranks' tiles) of the last idkpt_compute; valid until the compute after next (double-buffered).
IDKPT_API int idkpt_gather_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_device_ptr: null argument");
    DRAIN_PENDING("idkpt_gather_device_ptr");
    if (ctx->gatherWorld < 2 || ctx->gatherCurrent < 0) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gather_device_ptr: no gathered frame yet");
    *devPtr = ctx->gatherImage[ctx->gatherCurrent].p;
    if (bytes) *bytes = (uint64_t)ctx->width * ctx->height * 16;
    return IDKPT_OK;
}

IDKPT_API int idkpt_result_device_ptr(IdkPtCtx* ctx, IdkPtImage which, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr || (int)which < 0 || (int)which > 2) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_result_device_ptr: invalid argument");
    DRAIN_PENDING("idkpt_result_device_ptr");
    *devPtr = ctx->images[which].p;
    if (bytes) *bytes = (uint64_t)ctx->nLocal * 16;
    return IDKPT_OK;
}

IDKPT_API int idkpt_tile_rows(IdkPtCtx* ctx, int32_t* rowCount, int32_t* rowsOut, int32_t capacity) {
    if (!ctx || !rowCount) return IDKPT_ERR_INVALID_ARGUMENT;
    *rowCount = (int32_t)ctx->rows.size();
    if (rowsOut) for (int i = 0; i < capacity && i < (int)ctx->rows.size(); i++) rowsOut[i] = ctx->rows[i];
    return IDKPT_OK;
}

IDKPT_API int idkpt_read_wavefront_rays(IdkPtCtx* ctx, GpuWavefrontRay* dst, uint64_t count) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    DRAIN_PENDING("idkpt_read_wavefront_rays");
    if (!dst) {   // dst == NULL arms the export for subsequent idkpt_compute calls (debug / parity feature)
        ctx->exportEnabled = count != 0;
        return IDKPT_OK;
    }
    if (!ctx->exportEnabled) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_wavefront_rays: arm the export first (dst = NULL, count = 1) and call idkpt_compute");
    if (count < (uint64_t)ctx->width * ctx->height) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_wavefront_rays: buffer smaller than width*height");
    CK(cudaSetDevice(ctx->device));
    std::vector<PathState> tmp(ctx->nLocal);
    CK(cudaMemcpyAsync(tmp.data(), ctx->lanes[0].state.p, (size_t)ctx->nLocal * sizeof(PathState), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < ctx->rows.size(); i++) {
        for (int x = 0; x < ctx->width; x++) {
            const PathState& s = tmp[i * (size_t)ctx->width + x];
            GpuWavefrontRay& w = dst[(size_t)ctx->rows[i] * ctx->width + x];
            w.Origin[0] = s.ox; w.Origin[1] = s.oy; w.Origin[2] = s.oz; w.PreviousIOROrTraverseCost = s.prevIor;
            w.Throughput[0] = s.tx; w.Throughput[1] = s.ty; w.Throughput[2] = s.tz; w.PackedDirectionX = s.pdx;
            w.Radiance[0] = s.rx; w.Radiance[1] = s.ry; w.Radiance[2] = s.rz; w.PackedDirectionY = s.pdy;
        }
    }
    return IDKPT_OK;
}

// ---- present chain (SURVEY.md 8f.3) ----------------------------------------------------------------------------------------

static inline int ilogb_int(int v) { int r = 0; while (v > 1) { v >>= 1; r++; } return r; }

IDKPT_API int idkpt_post_process(IdkPtCtx* ctx, const IdkPtPostSettings* s, IdkPtImage source, uint8_t* rgba8Out, float* kernelMs) {
    if (!ctx || !s) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: null argument");
    if (kernelMs) *kernelMs = 0.0f;
    const int w = ctx->width, h = ctx->height;
    const float4* src = nullptr;
    if (source == IDKPT_IMAGE_GATHERED) {
        if (ctx->gatherWorld < 2 || ctx->gatherCurrent < 0) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: no gathered frame yet");
        src = (const float4*)ctx->gatherImage[ctx->gatherCurrent].p;
    } else if (source == IDKPT_IMAGE_DENOISED) {
        if (!ctx->haveDenoised) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: no denoised image (call idkpt_denoise)");
        src = (const float4*)ctx->denoised.p;
    } else if ((int)source >= 0 && (int)source <= 2) {
        if (ctx->tileCount != 1) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: a tiled context holds only its own rows; use IDKPT_IMAGE_GATHERED");
        src = (const float4*)ctx->images[source].p;
    } else return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: unknown image");
    if (s->IsBloom && (w < 2 || h < 2)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: bloom needs an image of at least 2x2");
    if (s->IsBloom && (s->BloomMinusLods < 0 || s->BloomMinusLods > 30)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_post_process: BloomMinusLods out of range");
    CK(cudaSetDevice(ctx->device));
    CK(ensure(ctx->ldr, (size_t)w * h * 4));
    CK(ensure(ctx->postConsts, sizeof(PostTonemapConsts)));
    const dim3 blk(256);
    auto grid = [](int gw, int gh) { return dim3((unsigned)((gw + 31) / 32), (unsigned)((gh + 7) / 8)); };
    return run_timed(ctx, "idkpt_post_process", kernelMs, [&]() -> int {
        PostImage bloomResult = {nullptr, nullptr, 0, 0};
        if (s->IsBloom) {
            // Bloom.SetSize (Bloom.cs:132-150): half resolution, levels = max(MaxMipmapLevel - MinusLods, 2); the upsample chain has one level less
            const int w2 = w / 2, h2 = h / 2;
            const int levels = std::max(ilogb_int(std::max(w2, h2)) + 1 - s->BloomMinusLods, 2);
            std::vector<size_t> off(levels + 1, 0);
            std::vector<int> lw(levels), lh(levels);
            for (int l = 0; l < levels; l++) {
                lw[l] = std::max(1, w2 / (1 << std::min(l, 30))); lh[l] = std::max(1, h2 / (1 << std::min(l, 30)));
                off[l + 1] = off[l] + (size_t)lw[l] * lh[l];
            }
            cudaError_t ce = ensure(ctx->bloomDown, off[levels] * 8);
            if (ce == cudaSuccess) ce = ensure(ctx->bloomUp, off[levels - 1] * 8);
            if (ce != cudaSuccess) return fail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkpt_post_process: bloom allocation failed");
            uint2* down = (uint2*)ctx->bloomDown.p;
            uint2* up = (uint2*)ctx->bloomUp.p;
            // Bloom.cs:62-93. The shader prefilters when its Lod uniform is 0, and Lod is 0 for the dispatch that writes level 0
            // and again for the one that writes level 1 (that one uploads currentWriteLod - 1): both levels are prefiltered.
            for (int l = 0; l < levels; l++) {
                BloomDownArgs a;
                a.src = l == 0 ? PostImage{src, nullptr, w, h} : PostImage{nullptr, down + off[l - 1], lw[l - 1], lh[l - 1]};
                a.dst = down + off[l]; a.dw = lw[l]; a.dh = lh[l];
                a.prefilter = l <= 1; a.maxColor = s->BloomMaxColor; a.threshold = s->BloomThreshold;
                k_bloom_down<<<grid(a.dw, a.dh), blk, 0, ctx->stream>>>(a);
            }
            for (int l = levels - 2; l >= 0; l--) {
                BloomUpArgs a;
                a.up = l == levels - 2 ? PostImage{nullptr, down + off[l + 1], lw[l + 1], lh[l + 1]} : PostImage{nullptr, up + off[l + 1], lw[l + 1], lh[l + 1]};
                a.down = PostImage{nullptr, down + off[l + 1], lw[l + 1], lh[l + 1]};
                a.dst = up + off[l]; a.dw = lw[l]; a.dh = lh[l];
                k_bloom_up<<<grid(a.dw, a.dh), blk, 0, ctx->stream>>>(a);
            }
            bloomResult = PostImage{nullptr, up, lw[0], lh[0]};
        }
        k_agx_matrices<<<1, 1, 0, ctx->stream>>>(s->Exposure, s->Compression, (PostTonemapConsts*)ctx->postConsts.p);
        TonemapArgs t;
        t.src0 = PostImage{src, nullptr, w, h};
        t.src1 = bloomResult;
        t.dst = (uchar4*)ctx->ldr.p; t.w = w; t.h = h;
        t.saturation = s->Saturation; t.linear = s->Linear; t.peak = s->Peak; t.doTonemap = s->DoTonemapAndSrgbTransform ? 1 : 0;
        t.consts = (const PostTonemapConsts*)ctx->postConsts.p;
        k_tonemap<<<grid(w, h), blk, 0, ctx->stream>>>(t);
        return IDKPT_OK;
    }, rgba8Out, ctx->ldr.p, (size_t)w * h * 4);
}

IDKPT_API int idkpt_ldr_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_ldr_device_ptr: null argument");
    DRAIN_PENDING("idkpt_ldr_device_ptr");
    if (!ctx->ldr.p) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_ldr_device_ptr: call idkpt_post_process first");
    *devPtr = ctx->ldr.p;
    if (bytes) *bytes = (uint64_t)ctx->width * ctx->height * 4;
    return IDKPT_OK;
}

// ---- denoise hand-off (SURVEY.md 8f.3) ---------------------------------------------------------------------------------------
static int denoise_alloc(IdkPtCtx* ctx) {
    const size_t n = (size_t)ctx->width * ctx->height;
    for (int i = 0; i < 4; i++) CK(ensure(ctx->oidn[i], n * 12));
    for (int i = 0; i < 2; i++) CK(ensure(ctx->denoiseWork[i], n * 16));
    CK(ensure(ctx->denoised, n * 16));
    return IDKPT_OK;
}

IDKPT_API int idkpt_denoise(IdkPtCtx* ctx, const IdkPtDenoiseSettings* s, float* kernelMs) {
    if (!ctx || !s) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_denoise: null argument");
    if (kernelMs) *kernelMs = 0.0f;
    if (ctx->tileCount != 1) return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_denoise: the AOV images of a tiled context hold only its own rows");
    if (s->Iterations < 0 || s->Iterations > 12 || !(s->SigmaColor > 0.0f) || !(s->SigmaNormal > 0.0f) || !(s->SigmaAlbedo > 0.0f))
        return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_denoise: Iterations must be 0..12 and the sigmas positive");
    DRAIN_PENDING("idkpt_denoise");
    CK(cudaSetDevice(ctx->device));
    int rc = denoise_alloc(ctx);
    if (rc) return rc;
    const int w = ctx->width, h = ctx->height, n = w * h;
    rc = run_timed(ctx, "idkpt_denoise", kernelMs, [&]() -> int {
        DenoisePrepareArgs pa;
        pa.result = (const float4*)ctx->images[0].p; pa.albedo = (const float4*)ctx->images[1].p; pa.normal = (const float4*)ctx->images[2].p;
        pa.oidnBeauty = (float*)ctx->oidn[0].p; pa.oidnAlbedo = (float*)ctx->oidn[1].p; pa.oidnNormal = (float*)ctx->oidn[2].p;
        pa.work = (float4*)ctx->denoiseWork[0].p; pa.count = n; pa.demodulate = s->Demodulate ? 1 : 0;
        k_denoise_prepare<<<(n + 255) / 256, 256, 0, ctx->stream>>>(pa);
        int cur = 0;
        for (int it = 0; it < s->Iterations; it++) {
            const int step = 1 << it;
            const float sc = s->SigmaColor / (float)step;
            DenoiseAtrousArgs a;
            a.in = (const float4*)ctx->denoiseWork[cur].p; a.out = (float4*)ctx->denoiseWork[cur ^ 1].p;
            a.albedo = pa.albedo; a.normal = pa.normal; a.w = w; a.h = h; a.step = step;
            a.invSigmaColor2 = 1.0f / (sc * sc); a.invSigmaNormal2 = 1.0f / (s->SigmaNormal * s->SigmaNormal);
            a.invSigmaAlbedo2 = 1.0f / (s->SigmaAlbedo * s->SigmaAlbedo); a.invStep2 = 1.0f / ((float)step * (float)step);
            k_denoise_atrous<<<dim3((unsigned)((w + 31) / 32), (unsigned)((h + 7) / 8)), 256, 0, ctx->stream>>>(a);
            cur ^= 1;
        }
        if (s->Iterations > 0) {
            DenoiseFinishArgs fa;
            fa.filtered = (const float4*)ctx->denoiseWork[cur].p; fa.albedo = pa.albedo; fa.denoised = (float4*)ctx->denoised.p;
            fa.oidnOutput = (float*)ctx->oidn[3].p; fa.count = n; fa.demodulate = pa.demodulate;
            k_denoise_finish<<<(n + 255) / 256, 256, 0, ctx->stream>>>(fa);
        }
        return IDKPT_OK;
    });
    if (rc == IDKPT_OK && s->Iterations > 0) ctx->haveDenoised = true;
    return rc;
}

IDKPT_API int idkpt_denoise_device_ptrs(IdkPtCtx* ctx, void** beauty, void** albedo, void** normal, void** output, uint64_t* bytesEach) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    DRAIN_PENDING("idkpt_denoise_device_ptrs");
    CK(cudaSetDevice(ctx->device));
    int rc = denoise_alloc(ctx);
    if (rc) return rc;
    if (beauty) *beauty = ctx->oidn[0].p;
    if (albedo) *albedo = ctx->oidn[1].p;
    if (normal) *normal = ctx->oidn[2].p;
    if (output) *output = ctx->oidn[3].p;
    if (bytesEach) *bytesEach = (uint64_t)ctx->width * ctx->height * 12;
    return IDKPT_OK;
}

// The OIDN output buffer (written by the host's OIDN CUDA device) becomes the denoised image.
__global__ void __launch_bounds__(256) k_denoise_import(const float* __restrict__ rgb, float4* __restrict__ out, int count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = make_float4(rgb[3 * (size_t)i], rgb[3 * (size_t)i + 1], rgb[3 * (size_t)i + 2], 1.0f);
}

IDKPT_API int idkpt_denoise_import_output(IdkPtCtx* ctx) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    DRAIN_PENDING("idkpt_denoise_import_output");
    if (!ctx->oidn[3].p || !ctx->denoised.p) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_denoise_import_output: call idkpt_denoise_device_ptrs / idkpt_denoise first");
    CK(cudaSetDevice(ctx->device));
    const int n = ctx->width * ctx->height;
    k_denoise_import<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const float*)ctx->oidn[3].p, (float4*)ctx->denoised.p, n);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->haveDenoised = true;
    return IDKPT_OK;
}

// ---- dynamic geometry (SURVEY.md 8f.2) -----------------------------------------------------------------------------------

IDKPT_API int idkpt_set_skinning_data(IdkPtCtx* ctx, const GpuUnskinnedVertex* vertices, uint64_t count) {
    if (!ctx || (!vertices && count)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_skinning_data: null argument");
    DRAIN_PENDING("idkpt_set_skinning_data");
    CK(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = upload(ctx, ctx->unskinned, vertices, count * sizeof(GpuUnskinnedVertex)))) return rc;
    ctx->unskinnedMaxJoint.resize(count);
    for (uint64_t i = 0; i < count; i++) {
        const uint32_t* j = vertices[i].JointIndices;
        ctx->unskinnedMaxJoint[i] = std::max(std::max(j[0], j[1]), std::max(j[2], j[3]));
    }
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->unskinnedCount = count;
    return IDKPT_OK;
}

IDKPT_API int idkpt_skin_vertices(IdkPtCtx* ctx, const float* jointMatrices, uint64_t jointCount, const IdkPtSkinningCmd* cmds, uint32_t cmdCount, float* kernelMs) {
    if (!ctx || (!jointMatrices && jointCount) || (!cmds && cmdCount)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_skin_vertices: null argument");
    DRAIN_PENDING("idkpt_skin_vertices");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_skin_vertices: no scene");
    if (kernelMs) *kernelMs = 0.0f;
    const uint64_t vtxLimit = std::min(ctx->counts.VertexPositionCount, ctx->counts.VertexCount);
    for (uint32_t c = 0; c < cmdCount; c++) {
        const IdkPtSkinningCmd& k = cmds[c];
        if ((uint64_t)k.InputVertexOffset + k.VertexCount > ctx->unskinnedCount) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_skin_vertices: input range outside the unskinned vertices (idkpt_set_skinning_data)");
        if ((uint64_t)k.OutputVertexOffset + k.VertexCount > vtxLimit) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_skin_vertices: output range outside the vertex arrays");
        uint32_t maxJoint = 0;
        for (uint64_t i = k.InputVertexOffset; i < (uint64_t)k.InputVertexOffset + k.VertexCount; i++) maxJoint = std::max(maxJoint, ctx->unskinnedMaxJoint[i]);
        if (k.VertexCount && (uint64_t)k.JointMatricesOffset + maxJoint >= jointCount) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_skin_vertices: a joint index points past the joint matrices");
    }
    CK(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = upload(ctx, ctx->joints, jointMatrices, jointCount * 48))) return rc;   // jointMatricesBuffer.UploadElements (ModelManager.cs:277)
    if ((rc = keep_prev_positions(ctx))) return rc;
    rc = run_timed(ctx, "idkpt_skin_vertices", kernelMs, [&]() -> int {
        for (uint32_t c = 0; c < cmdCount; c++) {
            if (!cmds[c].VertexCount) continue;
            // Skinning/compute.glsl:42, prevVertexPositionSSBO = vertexPositionSSBO over the command's output range, dispatch by
            // dispatch: with overlapping commands the kept positions are those the previous command left, as in the engine
            const size_t off = (size_t)cmds[c].OutputVertexOffset * sizeof(PackedVec3), n = (size_t)cmds[c].VertexCount * sizeof(PackedVec3);
            CK(cudaMemcpyAsync((char*)ctx->prevPositions.p + off, (const char*)ctx->positions.p + off, n, cudaMemcpyDeviceToDevice, ctx->stream));
            SkinArgs a;
            a.unskinned = (const uint32_t*)ctx->unskinned.p; a.joints = (const float4*)ctx->joints.p;
            a.positions = (float*)ctx->positions.p; a.vertices = (uint4*)ctx->vertices.p; a.vtxFrame = (float4*)ctx->vtxFrame.p;
            a.inOffset = cmds[c].InputVertexOffset; a.outOffset = cmds[c].OutputVertexOffset; a.jointOffset = cmds[c].JointMatricesOffset; a.count = cmds[c].VertexCount;
            k_skin_vertices<<<(a.count + 255) / 256, 256, 0, ctx->stream>>>(a);
        }
        return IDKPT_OK;
    });
    if (rc == IDKPT_OK) ctx->accumulatedSamples = 0;
    return rc;
}

IDKPT_API int idkpt_blas_refit(IdkPtCtx* ctx, uint32_t first, uint32_t count, float* kernelMs) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    DRAIN_PENDING("idkpt_blas_refit");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_blas_refit: no scene");
    if ((uint64_t)first + count > ctx->hostDescs.size()) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_refit: BLAS range outside BlasDescs");
    if (kernelMs) *kernelMs = 0.0f;
    CK(cudaSetDevice(ctx->device));
    int maxNodes = 0;
    for (uint32_t b = first; b < first + count; b++) maxNodes = std::max(maxNodes, ctx->hostDescs[b].NodeCount);
    CK(ensure(ctx->refitParents, std::max<size_t>((size_t)maxNodes, 4) * 4));   // blasRefitLockBuffer sizing, BVH.cs:451
    CK(ensure(ctx->refitLocks, std::max<size_t>((size_t)maxNodes, 4) * 4));
    const int rc = run_timed(ctx, "idkpt_blas_refit", kernelMs, [&]() -> int {
        for (uint32_t b = first; b < first + count; b++) {
            const GpuBlasDesc& d = ctx->hostDescs[b];
            RefitArgs a;
            a.nodes = (float4*)ctx->nodes.p + 2 * (size_t)d.NodeOffset;
            a.blasTris = (const int4*)ctx->blasTris.p; a.positions = (const float*)ctx->positions.p;
            a.triRec = (float4*)((char*)ctx->nodes.p + ctx->nodeBytes);
            a.parents = (int32_t*)ctx->refitParents.p; a.locks = (uint32_t*)ctx->refitLocks.p;
            a.nodeCount = (uint32_t)d.NodeCount; a.triOffset = (uint32_t)d.TriangleOffset; a.triCount = (uint32_t)d.TriangleCount;
            k_refit_prepare<<<(a.nodeCount + 255) / 256, 256, 0, ctx->stream>>>(a);
            k_refit_climb<<<(a.nodeCount + 255) / 256, 256, 0, ctx->stream>>>(a);
        }
        return IDKPT_OK;
    });
    if (rc == IDKPT_OK) ctx->accumulatedSamples = 0;
    return rc;
}

// The TLAS build of n >= 1 instances over the given device arrays into `out` (2n - 1 nodes), with its scratch in the context's
// tlasScratch. Up to IDK_TLAS_SINGLE_CTA_MAX instances k_tlas_build, above it the grid build (k_tlas_ploc): four kernels, the
// radix sort and one cooperative launch. Neither synchronises with the host. On return
// *need is the device address of the built tree's height (valid once the stream has finished); a value above
// IDK_TLAS_STACK_SIZE means the build stopped at the first parent deeper than the walk's stack, and -1 that an iteration
// merged nothing (a box that is not finite); in both cases `out` is not a tree.
static int enqueue_tlas_build(IdkPtCtx* ctx, const void* blasNodes, const void* descs, const void* instances, const void* xforms,
                              void* out, uint64_t n, int searchRadius, int** need) {
    if (n <= IDK_TLAS_SINGLE_CTA_MAX) {                   // one launch beats the grid build's nine at a few dozen instances
        const size_t nodeCount = 2 * n - 1;
        const size_t tempOff = 0, leavesOff = nodeCount * 32, keysOff = leavesOff + n * 32, prefOff = keysOff + n * 4, needOff = prefOff + n * 4;
        CK(ensure(ctx->tlasScratch, needOff + nodeCount * 4 + 64));
        TlasBuildArgs a;
        a.blasNodes = (const float4*)blasNodes; a.descs = (const GpuBlasDesc*)descs; a.instances = (const GpuBlasInstance*)instances;
        a.xforms = (const float4*)xforms; a.nodes = (float4*)out;
        a.temp = (float4*)((char*)ctx->tlasScratch.p + tempOff); a.leaves = (float4*)((char*)ctx->tlasScratch.p + leavesOff);
        a.keys = (uint32_t*)((char*)ctx->tlasScratch.p + keysOff); a.pref = (int*)((char*)ctx->tlasScratch.p + prefOff);
        a.need = (int*)((char*)ctx->tlasScratch.p + needOff);
        a.n = (int)n; a.searchRadius = searchRadius;
        k_tlas_build<<<1, 1024, 0, ctx->stream>>>(a);
        *need = a.need;
        return IDKPT_OK;
    }
    const int T = IDK_TLAS_BLOCK;
    const size_t nodeCount = 2 * n - 1, leafBlocks = (n + T - 1) / T;
    const int smem = (T + 2 * searchRadius) * 6 * (int)sizeof(float);
    CK(cudaFuncSetAttribute(k_tlas_ploc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int perSm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, k_tlas_ploc, T, smem));
    if (perSm < 1) return fail(ctx, IDKPT_ERR_CUDA, "TLAS build: k_tlas_ploc does not fit on an SM");
    const int G = (int)std::min<size_t>((size_t)perSm * ctx->smCount, leafBlocks);   // co-resident, as grid.sync needs
    size_t sortBytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr,
                                       (int*)nullptr, (int)n, 0, 30, ctx->stream));
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const size_t oA = take(nodeCount * 32), oB = take(nodeCount * 32), ohA = take(nodeCount * 4), ohB = take(nodeCount * 4);
    const size_t oKeys = take(n * 4), oKeysSorted = take(n * 4), oOrder = take(n * 4), oOrderSorted = take(n * 4), oPref = take(n * 4);
    const size_t oPartial = take(leafBlocks * 24), oGlobal = take(24), oSums = take((size_t)G * 8), oStatus = take(8), oSort = take(sortBytes);
    CK(ensure(ctx->tlasScratch, off));
    char* s = (char*)ctx->tlasScratch.p;
    TlasGridArgs a;
    a.blasNodes = (const float4*)blasNodes; a.descs = (const GpuBlasDesc*)descs; a.instances = (const GpuBlasInstance*)instances;
    a.xforms = (const float4*)xforms; a.nodes = (float4*)out;
    a.bufA = (float4*)(s + oA); a.bufB = (float4*)(s + oB); a.hA = (int*)(s + ohA); a.hB = (int*)(s + ohB);
    a.keys = (uint32_t*)(s + oKeys); a.keysSorted = (uint32_t*)(s + oKeysSorted);
    a.order = (int*)(s + oOrder); a.orderSorted = (int*)(s + oOrderSorted); a.pref = (int*)(s + oPref);
    a.partial = (float*)(s + oPartial); a.global = (float*)(s + oGlobal); a.blockSums = (int*)(s + oSums); a.status = (int*)(s + oStatus);
    a.n = (int)n; a.searchRadius = searchRadius; a.partialCount = (int)leafBlocks;
    k_tlas_leaves<<<(unsigned)leafBlocks, T, 0, ctx->stream>>>(a);
    k_tlas_bounds<<<1, 1024, 0, ctx->stream>>>(a);
    k_tlas_keys<<<(unsigned)leafBlocks, T, 0, ctx->stream>>>(a);
    CK(cub::DeviceRadixSort::SortPairs(s + oSort, sortBytes, a.keys, a.keysSorted, a.order, a.orderSorted, (int)n, 0, 30, ctx->stream));
    void* args[] = {&a};
    CK(cudaLaunchCooperativeKernel((const void*)k_tlas_ploc, dim3(G), dim3(T), args, (size_t)smem, ctx->stream));
    *need = a.status + 1;
    return IDKPT_OK;
}

// BVH.TlasBuild on the device (BVH.cs:278-298, TLAS.cs:28-141): see k_tlas_ploc.
IDKPT_API int idkpt_tlas_build(IdkPtCtx* ctx, int32_t searchRadius, float* kernelMs) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    DRAIN_PENDING("idkpt_tlas_build");
    if (kernelMs) *kernelMs = 0.0f;
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_tlas_build: no scene");
    if (!ctx->counts.UseTlas) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_tlas_build: the scene was set without UseTlas (no TLAS node array to fill)");
    if (searchRadius < 1 || searchRadius > 1024) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_tlas_build: search radius out of range (TLAS.BuildSettings.SearchRadius, default 15)");
    const uint64_t n = ctx->counts.BlasInstanceCount;
    if (2 * n - 1 >= (1ull << 31)) return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_tlas_build: more than 2^30 instances (TLAS child and instance ids are 31 bits)");
    CK(cudaSetDevice(ctx->device));
    int* needDev = nullptr;
    const int rc = run_timed(ctx, "idkpt_tlas_build", kernelMs, [&]() -> int {
        return enqueue_tlas_build(ctx, ctx->nodes.p, ctx->descs.p, ctx->instances.p, ctx->xforms.p, ctx->tlas.p, n, searchRadius, &needDev);
    });
    if (rc) return rc;
    ctx->accumulatedSamples = 0;
    int need = 0;
    CK(cudaMemcpy(&need, needDev, 4, cudaMemcpyDeviceToHost));
    if (need < 0) {                       // the PLOC loop merged nothing: the node array is not a tree
        ctx->haveScene = false;
        return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_tlas_build: an instance's world box is not finite or its half area overflows (ModelMatrix or BLAS root); scene invalidated; set it again");
    }
    if (need > IDK_TLAS_STACK_SIZE) {     // the walk's stack is fixed (BVHIntersect.glsl:4): refuse to trace through a TLAS it cannot hold
        ctx->haveScene = false;
        return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_tlas_build: the built TLAS is deeper than the 24-entry traversal stack of the TLAS walk (scene invalidated; set it again)");
    }
    return IDKPT_OK;
}

// idkbb::build's status as the library's
static int blas_build_fail(IdkPtCtx* ctx, const char* who, int rc, const std::string& err) {
    if (rc == idkbb::BB_CUDA) cudaStreamSynchronize(ctx->stream);
    return fail(ctx, who, rc == idkbb::BB_CUDA ? IDKPT_ERR_CUDA : IDKPT_ERR_UNSUPPORTED, err.c_str());
}

// BLAS.Build + PreSplitting.PreSplit on the device (BVH.BlasesBuild's loop body, BVH.cs:315-377): a batch of one, see
// idk_blas_build.cuh.
IDKPT_API int idkpt_blas_build(IdkPtCtx* ctx, const PackedVec3* positions, uint64_t vertexCount, const GpuBlasTriangle* triangles,
                               uint64_t triangleCount, const IdkPtBlasBuildSettings* settings, IdkPtBlasBuild** out, float* kernelMs) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (out) *out = nullptr;
    if (kernelMs) *kernelMs = 0.0f;
    if (!positions || !triangles || !out) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_build: null argument");
    if (triangleCount == 0) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_build: no triangles");
    idkbvh::Params p;
    if (int rc = blas_build_params(ctx, "idkpt_blas_build", settings, p)) return rc;
    if (triangleCount > (uint64_t)idkbb::MAX_FRAGMENTS)
        return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_blas_build: more than 2^24 triangles");
    for (uint64_t i = 0; i < triangleCount; i++) {
        const GpuBlasTriangle& t = triangles[i];
        if ((uint64_t)(uint32_t)t.X >= vertexCount || (uint64_t)(uint32_t)t.Y >= vertexCount || (uint64_t)(uint32_t)t.Z >= vertexCount)
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_build: vertex id out of range");
    }
    DRAIN_PENDING("idkpt_blas_build");
    CK(cudaSetDevice(ctx->device));
    IdkPtBlasBuild* b = new IdkPtBlasBuild();
    std::string err;
    float ms = 0.0f;
    const std::vector<idkbb::Input> in = {{0, (int)triangleCount, p.doPreSplit}};
    const int rc = idkbb::build(ctx->stream, positions, vertexCount, triangles, triangleCount, in, std::vector<GpuBlasDesc>(1), p, *b, ms, err);
    if (rc != idkbb::BB_OK) {
        delete b;
        return blas_build_fail(ctx, "idkpt_blas_build", rc, err);
    }
    *out = b;
    if (kernelMs) *kernelMs = ms;
    return IDKPT_OK;
}

// BVH.BlasesBuild's parallel loop (BVH.cs:315-377) as one batch: see idk_blas_build.cuh.
IDKPT_API int idkpt_blas_build_batch(IdkPtCtx* ctx, const PackedVec3* positions, uint64_t vertexCount, const GpuBlasTriangle* triangles,
                                     uint64_t triangleCount, const GpuBlasDesc* descs, uint32_t descCount,
                                     const IdkPtBlasBuildSettings* settings, IdkPtBlasBuild** out, float* kernelMs) {
    const char* who = "idkpt_blas_build_batch";
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (out) *out = nullptr;
    if (kernelMs) *kernelMs = 0.0f;
    if (!positions || !triangles || !descs || !out) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "null argument");
    if (descCount == 0) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "no BLASes");
    idkbvh::Params p;
    if (int rc = blas_build_params(ctx, who, settings, p)) return rc;
    std::vector<idkbb::Input> in(descCount);
    std::vector<int> counts(descCount);
    for (uint32_t s = 0; s < descCount; s++) {
        const GpuBlasDesc& d = descs[s];
        if (d.TriangleCount <= 0) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a BLAS without triangles");
        if (d.TriangleOffset < 0 || (uint64_t)d.TriangleOffset + (uint64_t)d.TriangleCount > triangleCount)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "GpuBlasDesc triangle range outside the array");
        if (d.TriangleCount > idkbb::MAX_FRAGMENTS) return fail(ctx, who, IDKPT_ERR_UNSUPPORTED, "a BLAS of more than 2^24 triangles");
        in[s] = {d.TriangleOffset, d.TriangleCount, d.IsRefittable ? 0 : 1};   // BVH.cs:325
        counts[s] = d.TriangleCount;
    }
    if (idkbb::nodeIdCount(counts, descCount) < 0) return fail(ctx, who, IDKPT_ERR_UNSUPPORTED, "the batch needs 2^31 or more node ids");
    for (uint32_t s = 0; s < descCount; s++) {
        for (int i = 0; i < descs[s].TriangleCount; i++) {
            const GpuBlasTriangle& t = triangles[(size_t)descs[s].TriangleOffset + i];
            if ((uint64_t)(uint32_t)t.X >= vertexCount || (uint64_t)(uint32_t)t.Y >= vertexCount || (uint64_t)(uint32_t)t.Z >= vertexCount)
                return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "vertex id out of range");
        }
    }
    DRAIN_PENDING("idkpt_blas_build_batch");
    CK(cudaSetDevice(ctx->device));
    IdkPtBlasBuild* b = new IdkPtBlasBuild();
    std::string err;
    float ms = 0.0f;
    const int rc = idkbb::build(ctx->stream, positions, vertexCount, triangles, triangleCount, in,
                                std::vector<GpuBlasDesc>(descs, descs + descCount), p, *b, ms, err);
    if (rc != idkbb::BB_OK) {
        delete b;
        return blas_build_fail(ctx, who, rc, err);
    }
    *out = b;
    if (kernelMs) *kernelMs = ms;
    return IDKPT_OK;
}

// Totals over the batch: the largest RequiredStackSize (BVH.UpdateBlasStackSize) and the SAHs added in BLAS order.
IDKPT_API int idkpt_blas_build_info(const IdkPtBlasBuild* b, uint64_t* nodeCount, uint64_t* triangleCount, int32_t* requiredStackSize,
                                    int32_t* fragmentCount, double* sah) {
    if (!b) return IDKPT_ERR_INVALID_ARGUMENT;
    int32_t stack = 0, fragments = 0;
    double total = 0.0;
    for (size_t s = 0; s < b->descs.size(); s++) {
        stack = std::max(stack, b->descs[s].RequiredStackSize);
        fragments += b->fragmentCounts[s];
        total += b->sahs[s];
    }
    if (nodeCount) *nodeCount = b->nodes.size();
    if (triangleCount) *triangleCount = b->tris.size();
    if (requiredStackSize) *requiredStackSize = stack;
    if (fragmentCount) *fragmentCount = fragments;
    if (sah) *sah = total;
    return IDKPT_OK;
}

IDKPT_API int idkpt_blas_build_copy(const IdkPtBlasBuild* b, GpuBlasNode* nodes, GpuBlasTriangle* triangles) {
    if (!b || !nodes || !triangles) return IDKPT_ERR_INVALID_ARGUMENT;
    memcpy(nodes, b->nodes.data(), b->nodes.size() * sizeof(GpuBlasNode));
    memcpy(triangles, b->tris.data(), b->tris.size() * sizeof(GpuBlasTriangle));
    return IDKPT_OK;
}

IDKPT_API int idkpt_blas_build_batch_copy(const IdkPtBlasBuild* b, GpuBlasDesc* descs, GpuBlasNode* nodes, GpuBlasTriangle* triangles,
                                          int32_t* fragmentCounts, double* sahs) {
    if (!b) return IDKPT_ERR_INVALID_ARGUMENT;
    const size_t B = b->descs.size();
    if (descs) memcpy(descs, b->descs.data(), B * sizeof(GpuBlasDesc));
    if (nodes) memcpy(nodes, b->nodes.data(), b->nodes.size() * sizeof(GpuBlasNode));
    if (triangles) memcpy(triangles, b->tris.data(), b->tris.size() * sizeof(GpuBlasTriangle));
    if (fragmentCounts) memcpy(fragmentCounts, b->fragmentCounts.data(), B * sizeof(int32_t));
    if (sahs) memcpy(sahs, b->sahs.data(), B * sizeof(double));
    return IDKPT_OK;
}

IDKPT_API void idkpt_blas_build_free(IdkPtBlasBuild* b) { delete b; }

static int64_t nodes_end(const GpuBlasDesc& d) { return (int64_t)d.NodeOffset + d.NodeCount; }
static int64_t triangles_end(const GpuBlasDesc& d) { return (int64_t)d.TriangleOffset + d.TriangleCount; }

// BVH.BlasesBuild(first, count) (BVH.cs:300-470) on the scene in place: the BLASes of the range are built by one batched
// idkbb::build_device from their current triangle records and the device positions, into staging memory. When it succeeded, the new nodes
// and triangles replace the old ones in new allocations: the data before the range (up to the end of desc first - 1) and the
// data after it move unchanged, and the descs from `first` on are repacked behind each other (BVH.cs:378-441).
IDKPT_API int idkpt_blas_rebuild(IdkPtCtx* ctx, uint32_t first, uint32_t count, const IdkPtBlasBuildSettings* settings, float* kernelMs) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (kernelMs) *kernelMs = 0.0f;
    DRAIN_PENDING("idkpt_blas_rebuild");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_blas_rebuild: no scene");
    const std::vector<GpuBlasDesc>& old = ctx->hostDescs;
    const size_t nd = old.size();
    if ((uint64_t)first + count > nd) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_rebuild: BLAS range outside BlasDescs");
    idkbvh::Params p;
    if (int rc = blas_build_params(ctx, "idkpt_blas_rebuild", settings, p)) return rc;
    if (count == 0) return IDKPT_OK;   // BVH.cs:302
    // The layout BlasesBuild and host.Scene.add produce: from `first` on, each BLAS starts where the previous one ends, and the
    // last one ends the arrays. The BLASes before the range keep their data, so none may reach past the end of desc first - 1.
    const int64_t keepNodes = first ? nodes_end(old[first - 1]) : 0, keepTris = first ? triangles_end(old[first - 1]) : 0;
    for (size_t i = 0; i < nd; i++) {
        const bool ok = i < first ? nodes_end(old[i]) <= keepNodes && triangles_end(old[i]) <= keepTris
                                  : i == first || (old[i].NodeOffset == nodes_end(old[i - 1]) && old[i].TriangleOffset == triangles_end(old[i - 1]));
        if (!ok) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_rebuild: the BLASes are not packed behind each other from the first one rebuilt");
    }
    if (nodes_end(old[nd - 1]) != (int64_t)ctx->counts.BlasNodeCount || triangles_end(old[nd - 1]) != (int64_t)ctx->counts.BlasTriangleCount)
        return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_rebuild: the last BLAS does not end the node and triangle arrays");
    std::vector<idkbb::Input> in(count);
    for (uint32_t k = 0; k < count; k++) {
        const GpuBlasDesc& d = old[first + k];
        if (d.TriangleCount > idkbb::MAX_FRAGMENTS) return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_blas_rebuild: a BLAS of more than 2^24 triangles");
        in[k] = {d.TriangleOffset, d.TriangleCount, d.IsRefittable ? 0 : 1};   // BVH.cs:325
    }
    CK(cudaSetDevice(ctx->device));

    std::vector<GpuBlasDesc> descs = old;
    idkbb::Arena staged;                                  // the rebuilt BLASes, until they are committed
    idkbb::DeviceResult built;
    DevBuf bvh, tris, descBuf;                            // the new [nodes | triRec], triangles and descs
    struct Drop { DevBuf* b[3]; ~Drop() { for (DevBuf* x : b) release(*x); } } drop = {{&bvh, &tris, &descBuf}};
    size_t nodeBytes = 0, triRecBytes = 0;
    int stackSize = 0;
    int rc = run_timed(ctx, "idkpt_blas_rebuild", kernelMs, [&]() -> int {
        idkbb::StageTimer tm(ctx->stream);
        tm.mark("start");
        std::string err;
        const int brc = idkbb::build_device(ctx->stream, (const PackedVec3*)ctx->positions.p, (const GpuBlasTriangle*)ctx->blasTris.p,
                                            in, p, staged, built, tm, err);
        if (brc != idkbb::BB_OK) return blas_build_fail(ctx, "idkpt_blas_rebuild", brc, err);
        long long fragments = 0;
        for (int c : built.fragmentCount) fragments += c;
        tm.print((int)count, fragments);
        for (uint32_t k = 0; k < count; k++) {
            GpuBlasDesc& d = descs[first + k];
            d.NodeCount = built.nodeStart[k + 1] - built.nodeStart[k];
            d.TriangleCount = built.triStart[k + 1] - built.triStart[k];
            d.RequiredStackSize = built.requiredStackSize[k];
        }
        int64_t nodeEnd = 0, triEnd = 0;
        for (size_t i = first; i < nd; i++) {
            const int64_t no = i ? nodes_end(descs[i - 1]) : 0, to = i ? triangles_end(descs[i - 1]) : 0;
            nodeEnd = no + descs[i].NodeCount;
            triEnd = to + descs[i].TriangleCount;
            if (nodeEnd >= (1ll << 31) || triEnd >= (1ll << 31)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_rebuild: scene too large");
            descs[i].NodeOffset = (int32_t)no;
            descs[i].TriangleOffset = (int32_t)to;
        }
        for (const GpuBlasDesc& d : descs) stackSize = std::max(stackSize, d.RequiredStackSize);   // BVH.UpdateBlasStackSize
        if ((size_t)std::max(1, stackSize) * IDK_BLOCK * sizeof(uint32_t) > 200 * 1024)
            return fail(ctx, IDKPT_ERR_UNSUPPORTED, "idkpt_blas_rebuild: BlasStackSize too large for the shared-memory traversal stack");

        // the new arrays: the kept prefix, the rebuilt BLASes, the moved tail
        const GpuBlasDesc &r0 = descs[first], &rl = descs[first + count - 1];
        const int64_t oldEndN = nodes_end(old[first + count - 1]), oldEndT = triangles_end(old[first + count - 1]);
        const int64_t tailN = (int64_t)ctx->counts.BlasNodeCount - oldEndN, tailT = (int64_t)ctx->counts.BlasTriangleCount - oldEndT;
        nodeBytes = (((size_t)nodeEnd * sizeof(GpuBlasNode)) + 255) & ~(size_t)255;
        triRecBytes = std::max<size_t>((size_t)triEnd, 1) * 64;
        if (ensure(bvh, nodeBytes + triRecBytes) != cudaSuccess || ensure(tris, std::max<size_t>((size_t)triEnd * sizeof(GpuBlasTriangle), 16)) != cudaSuccess ||
            ensure(descBuf, std::max<size_t>(nd * sizeof(GpuBlasDesc), 16)) != cudaSuccess)
            return fail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkpt_blas_rebuild: device allocation failed");
        GpuBlasNode* nodesNew = (GpuBlasNode*)bvh.p;
        const GpuBlasNode* nodesOld = (const GpuBlasNode*)ctx->nodes.p;
        float4* recNew = (float4*)((char*)bvh.p + nodeBytes);
        const float4* recOld = (const float4*)((const char*)ctx->nodes.p + ctx->nodeBytes);
        GpuBlasTriangle* trisNew = (GpuBlasTriangle*)tris.p;
        const GpuBlasTriangle* trisOld = (const GpuBlasTriangle*)ctx->blasTris.p;
        auto d2d = [&](void* dst, const void* src, size_t bytes) { return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream) : cudaSuccess; };
        CK(d2d(nodesNew, nodesOld, (size_t)keepNodes * sizeof(GpuBlasNode)));
        CK(d2d(trisNew, trisOld, (size_t)keepTris * sizeof(GpuBlasTriangle)));
        CK(d2d(recNew, recOld, (size_t)keepTris * 64));
        CK(d2d(nodesNew + r0.NodeOffset, built.nodes, (size_t)built.nodeStart[count] * sizeof(GpuBlasNode)));   // the batch's ranges
        CK(d2d(trisNew + r0.TriangleOffset, built.tris, (size_t)built.triStart[count] * sizeof(GpuBlasTriangle)));  // are packed already
        CK(d2d(nodesNew + nodes_end(rl), nodesOld + oldEndN, (size_t)tailN * sizeof(GpuBlasNode)));
        CK(d2d(trisNew + triangles_end(rl), trisOld + oldEndT, (size_t)tailT * sizeof(GpuBlasTriangle)));
        CK(d2d(recNew + 4 * triangles_end(rl), recOld + 4 * oldEndT, (size_t)tailT * 64));
        if (const uint32_t n = (uint32_t)(triangles_end(rl) - r0.TriangleOffset))   // the rebuilt BLASes' triangle records
            k_prepare_triangles<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const int4*)(trisNew + r0.TriangleOffset), (const float*)ctx->positions.p,
                                                                          recNew + 4 * (size_t)r0.TriangleOffset, n);
        CK(cudaMemcpyAsync(descBuf.p, descs.data(), nd * sizeof(GpuBlasDesc), cudaMemcpyHostToDevice, ctx->stream));
        return IDKPT_OK;
    });
    if (rc) return rc;

    // commit: launch configuration and L2 window for the new arrays first (restored if either fails), then the swap
    const int oldStack = ctx->sc.stackSize;
    ctx->sc.stackSize = std::max(1, stackSize);
    if ((rc = configure_launches(ctx)) || (rc = set_l2_window(ctx, bvh.p, nodeBytes + triRecBytes))) {
        const std::string err = ctx->lastError;
        ctx->sc.stackSize = oldStack;
        configure_launches(ctx);
        set_l2_window(ctx, ctx->nodes.p, ctx->nodeBytes + std::max<size_t>(ctx->counts.BlasTriangleCount, 1) * 64);
        ctx->lastError = err;
        return rc;
    }
    std::swap(ctx->nodes, bvh);
    std::swap(ctx->blasTris, tris);
    std::swap(ctx->descs, descBuf);                      // `drop` frees the old arrays
    ctx->nodeBytes = nodeBytes;
    ctx->sc.nodes = (const float4*)ctx->nodes.p;
    ctx->sc.triRec = (const float4*)((char*)ctx->nodes.p + nodeBytes);
    ctx->sc.blasTris = (const int4*)ctx->blasTris.p;
    ctx->sc.descs = (const GpuBlasDesc*)ctx->descs.p;
    ctx->counts.BlasNodeCount = (uint64_t)nodes_end(descs[nd - 1]);
    ctx->counts.BlasTriangleCount = (uint64_t)triangles_end(descs[nd - 1]);
    ctx->counts.BlasStackSize = stackSize;
    ctx->hostDescs = std::move(descs);
    ctx->sceneGeneration++;                              // a bound voxeliser re-sizes its work queue for the new triangle counts
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

// validate_scene's checks for idkpt_add_models's own arrays, every id local to them: O(model), never O(scene).
static int validate_add_models(IdkPtCtx* ctx, const char* who, const IdkPtAddModelsDesc* m) {
    auto invalid = [&](const char* what) { return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, what); };
    if ((!m->Triangles && m->TriangleCount) || (!m->BlasDescs && m->BlasDescCount) || (!m->BlasInstances && m->BlasInstanceCount) ||
        (!m->MeshTransforms && m->MeshTransformCount) || (!m->Meshes && m->MeshCount) || (!m->Materials && m->MaterialCount) ||
        ((!m->Vertices || !m->VertexPositions) && m->VertexCount) || (!m->UnskinnedVertices && m->UnskinnedVertexCount))
        return invalid("a required array is null");
    const IdkPtSceneDesc& c = ctx->counts;
    if (c.VertexCount != c.VertexPositionCount) return invalid("the scene's vertex and position counts differ");
    const uint64_t lim = 1ull << 31;
    if (m->TriangleCount >= lim || c.BlasTriangleCount + m->TriangleCount >= lim || m->VertexCount >= lim || c.VertexCount + m->VertexCount >= lim ||
        m->MeshCount >= lim || c.MeshCount + m->MeshCount >= lim || m->MaterialCount >= lim || c.MaterialCount + m->MaterialCount >= lim ||
        m->BlasDescCount >= lim || c.BlasDescCount + m->BlasDescCount >= lim || m->MeshTransformCount >= lim ||
        c.MeshTransformCount + m->MeshTransformCount >= lim || m->BlasInstanceCount >= lim || c.BlasInstanceCount + m->BlasInstanceCount >= lim)
        return invalid("scene too large");
    for (uint64_t i = 0; i < m->BlasInstanceCount; i++)
        if (m->BlasInstances[i].BlasId >= m->BlasDescCount || m->BlasInstances[i].MeshTransformId >= m->MeshTransformCount)
            return invalid("BlasInstance references a BLAS or transform outside the call's arrays");
    for (uint64_t i = 0; i < m->BlasDescCount; i++) {
        const GpuBlasDesc& d = m->BlasDescs[i];
        if (d.TriangleCount <= 0) return invalid("a BLAS without triangles");
        if (d.TriangleOffset < 0 || (uint64_t)d.TriangleOffset + (uint64_t)d.TriangleCount > m->TriangleCount)
            return invalid("GpuBlasDesc triangle range outside the call's triangles");
        if (d.TriangleCount > idkbb::MAX_FRAGMENTS) return fail(ctx, who, IDKPT_ERR_UNSUPPORTED, "a BLAS of more than 2^24 triangles");
    }
    for (uint64_t i = 0; i < m->TriangleCount; i++) {
        const GpuBlasTriangle& t = m->Triangles[i];
        if ((uint64_t)(uint32_t)t.X >= m->VertexCount || (uint64_t)(uint32_t)t.Y >= m->VertexCount || (uint64_t)(uint32_t)t.Z >= m->VertexCount ||
            t.MeshId < 0 || (uint64_t)t.MeshId >= m->MeshCount)
            return invalid("GpuBlasTriangle index outside the call's vertices or meshes");
    }
    for (uint64_t i = 0; i < m->MeshCount; i++)
        if (m->Meshes[i].MaterialId < 0 || (uint64_t)m->Meshes[i].MaterialId >= m->MaterialCount)
            return invalid("GpuMesh.MaterialId outside the call's materials");
    IdkPtSceneDesc tex = {};                             // idk_validate_textures over the call's table and materials
    tex.Textures = m->Textures; tex.TextureCount = m->TextureCount;
    tex.Materials = m->Materials; tex.MaterialCount = m->MaterialCount;
    if (const char* terr = idk_validate_textures(&tex)) return texture_error(ctx, who, terr);
    if (c.UseTlas && 2 * (c.BlasInstanceCount + m->BlasInstanceCount) - 1 >= (1ull << 31))
        return fail(ctx, who, IDKPT_ERR_UNSUPPORTED, "more than 2^30 instances under UseTlas (TLAS child and instance ids are 31 bits)");
    return IDKPT_OK;
}

// ModelManager.Add(models) (ModelManager.cs:128-216) on the scene in place: see idkpt.h and DESIGN.md 8f.5 "Adding models".
// Everything is built into staging allocations first -- the grown arrays, the new BLASes, the new TLAS -- and swapped in only
// when all of it succeeded; until then the context's arrays are only read.
IDKPT_API int idkpt_add_models(IdkPtCtx* ctx, const IdkPtAddModelsDesc* m, const IdkPtBlasBuildSettings* settings, float* kernelMs) {
    static const char* who = "idkpt_add_models";
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (kernelMs) *kernelMs = 0.0f;
    if (!m) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "null argument");
    DRAIN_PENDING(who);
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    idkbvh::Params p;
    if (int rc = blas_build_params(ctx, who, settings, p)) return rc;
    if (int rc = validate_add_models(ctx, who, m)) return rc;
    if (!m->TriangleCount && !m->BlasDescCount && !m->BlasInstanceCount && !m->MeshTransformCount && !m->MeshCount && !m->MaterialCount &&
        !m->VertexCount && !m->TextureCount && !m->UnskinnedVertexCount)
        return IDKPT_OK;
    CK(cudaSetDevice(ctx->device));

    const IdkPtSceneDesc old = ctx->counts;
    const uint64_t nV = old.VertexCount + m->VertexCount, nX = old.MeshTransformCount + m->MeshTransformCount;
    const uint64_t nM = old.MeshCount + m->MeshCount, nMat = old.MaterialCount + m->MaterialCount;
    const uint64_t nI = old.BlasInstanceCount + m->BlasInstanceCount, nB = old.BlasDescCount + m->BlasDescCount;
    const uint64_t nTex = old.TextureCount + m->TextureCount, nU = ctx->unskinnedCount + m->UnskinnedVertexCount;
    const uint32_t B = (uint32_t)m->BlasDescCount;
    std::vector<idkbb::Input> in(B);
    for (uint32_t k = 0; k < B; k++) {
        const GpuBlasDesc& d = m->BlasDescs[k];
        in[k] = {d.TriangleOffset, d.TriangleCount, d.IsRefittable ? 0 : 1};   // BVH.cs:325
    }

    // the grown arrays ([nodes | triRec] in `bvh`), the new texture pool and records, and the staged records with ids
    DevBuf positions, vertices, xforms, meshes, materials, instances, vtxFrame, surfRec, descBuf, tris, bvh, tlas, recs, pool, unskinned, stage;
    struct Drop {
        DevBuf* b[16];
        ~Drop() { for (DevBuf* x : b) release(*x); }
    } drop = {{&positions, &vertices, &xforms, &meshes, &materials, &instances, &vtxFrame, &surfRec, &descBuf, &tris, &bvh, &tlas, &recs,
               &pool, &unskinned, &stage}};
    std::vector<GpuBlasDesc> descs = ctx->hostDescs;
    std::vector<TexRec> newRecs;
    idkbb::Arena staged;                                  // the new BLASes, until they are copied into `bvh`
    idkbb::DeviceResult built;
    size_t nodeBytes = 0, triRecBytes = 0;
    uint64_t nN = old.BlasNodeCount, nT = old.BlasTriangleCount;
    int stackSize = 0;
    int* needDev = nullptr;
    int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        auto alloc = [](DevBuf& b, size_t bytes) { return ensure(b, std::max<size_t>(bytes, 16)) == cudaSuccess; };
        auto d2d = [&](void* dst, const void* src, size_t bytes) { return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream) : cudaSuccess; };
        auto h2d = [&](void* dst, const void* src, size_t bytes) { return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream) : cudaSuccess; };
        auto at = [](const DevBuf& b, size_t off) { return (void*)((char*)b.p + off); };
        auto a256 = [](size_t x) { return (x + 255) & ~(size_t)255; };
        const size_t stTris = 0, stMeshes = a256(m->TriangleCount * sizeof(GpuBlasTriangle)), stMaterials = stMeshes + a256(m->MeshCount * sizeof(GpuMesh));
        const size_t stInstances = stMaterials + a256(m->MaterialCount * sizeof(GpuMaterial)), stEnd = stInstances + m->BlasInstanceCount * sizeof(GpuBlasInstance);
        if (!alloc(stage, stEnd) || !alloc(positions, nV * sizeof(PackedVec3)) || !alloc(vertices, nV * sizeof(GpuVertex)) ||
            !alloc(xforms, nX * sizeof(GpuMeshTransform)) || !alloc(meshes, nM * sizeof(GpuMesh)) || !alloc(materials, nMat * sizeof(GpuMaterial)) ||
            !alloc(instances, nI * sizeof(GpuBlasInstance)) || !alloc(vtxFrame, std::max<uint64_t>(nV, 1) * 32) || !alloc(surfRec, std::max<uint64_t>(nM, 1) * 80) ||
            !alloc(descBuf, nB * sizeof(GpuBlasDesc)) || (m->UnskinnedVertexCount && !alloc(unskinned, nU * sizeof(GpuUnskinnedVertex))))
            return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");

        // the scene's arrays move device to device; the call's arrays come over once, those with ids into the staging buffer
        CK(d2d(positions.p, ctx->positions.p, old.VertexCount * sizeof(PackedVec3)));
        CK(d2d(vertices.p, ctx->vertices.p, old.VertexCount * sizeof(GpuVertex)));
        CK(d2d(vtxFrame.p, ctx->vtxFrame.p, old.VertexCount * 32));
        CK(d2d(xforms.p, ctx->xforms.p, old.MeshTransformCount * sizeof(GpuMeshTransform)));
        CK(d2d(meshes.p, ctx->meshes.p, old.MeshCount * sizeof(GpuMesh)));
        CK(d2d(surfRec.p, ctx->surfRec.p, old.MeshCount * 80));
        CK(d2d(materials.p, ctx->materials.p, old.MaterialCount * sizeof(GpuMaterial)));
        CK(d2d(instances.p, ctx->instances.p, old.BlasInstanceCount * sizeof(GpuBlasInstance)));
        CK(h2d(at(positions, old.VertexCount * sizeof(PackedVec3)), m->VertexPositions, m->VertexCount * sizeof(PackedVec3)));
        CK(h2d(at(vertices, old.VertexCount * sizeof(GpuVertex)), m->Vertices, m->VertexCount * sizeof(GpuVertex)));
        CK(h2d(at(xforms, old.MeshTransformCount * sizeof(GpuMeshTransform)), m->MeshTransforms, m->MeshTransformCount * sizeof(GpuMeshTransform)));
        CK(h2d(at(stage, stTris), m->Triangles, m->TriangleCount * sizeof(GpuBlasTriangle)));
        CK(h2d(at(stage, stMeshes), m->Meshes, m->MeshCount * sizeof(GpuMesh)));
        CK(h2d(at(stage, stMaterials), m->Materials, m->MaterialCount * sizeof(GpuMaterial)));
        CK(h2d(at(stage, stInstances), m->BlasInstances, m->BlasInstanceCount * sizeof(GpuBlasInstance)));
        if (m->UnskinnedVertexCount) {
            CK(d2d(unskinned.p, ctx->unskinned.p, ctx->unskinnedCount * sizeof(GpuUnskinnedVertex)));
            CK(h2d(at(unskinned, ctx->unskinnedCount * sizeof(GpuUnskinnedVertex)), m->UnskinnedVertices, m->UnskinnedVertexCount * sizeof(GpuUnskinnedVertex)));
        }
        SceneAddArgs a;
        a.tris = (GpuBlasTriangle*)at(stage, stTris);
        a.meshesIn = (const GpuMesh*)at(stage, stMeshes); a.meshesOut = (GpuMesh*)meshes.p + old.MeshCount;
        a.materialsIn = (const GpuMaterial*)at(stage, stMaterials); a.materialsOut = (GpuMaterial*)materials.p + old.MaterialCount;
        a.instancesIn = (const GpuBlasInstance*)at(stage, stInstances); a.instancesOut = (GpuBlasInstance*)instances.p + old.BlasInstanceCount;
        a.triCount = m->TriangleCount; a.meshCount = m->MeshCount; a.materialCount = m->MaterialCount; a.instanceCount = m->BlasInstanceCount;
        a.vertexOffset = (int32_t)old.VertexCount; a.meshOffset = (int32_t)old.MeshCount; a.materialOffset = (int32_t)old.MaterialCount;
        a.blasOffset = (uint32_t)old.BlasDescCount; a.transformOffset = (uint32_t)old.MeshTransformCount; a.textureOffset = old.TextureCount;
        if (const uint64_t total = a.triCount + a.meshCount + a.materialCount + a.instanceCount)
            k_scene_add_rebase<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(a);
        if (const uint32_t n = (uint32_t)m->VertexCount)      // per element: a launch over the appended range equals the full one
            k_prepare_vertices<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const uint4*)vertices.p + old.VertexCount, (float4*)vtxFrame.p + 2 * old.VertexCount, n);
        if (const uint32_t n = (uint32_t)m->MeshCount)
            k_prepare_surfaces<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const GpuMesh*)meshes.p + old.MeshCount, (const GpuMaterial*)materials.p,
                                                                         (float4*)surfRec.p + 5 * old.MeshCount, n);
        CK(cudaGetLastError());

        if (m->TextureCount) {                            // decoded once, into a pool of their own; the old records keep theirs
            IdkPtSceneDesc tmp = {};
            tmp.Textures = m->Textures; tmp.TextureCount = m->TextureCount;
            const std::vector<size_t> off = idk_texture_offsets(&tmp);
            if (!alloc(pool, off[m->TextureCount]) || !alloc(recs, nTex * sizeof(TexRec)))
                return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
            CK(idk_upload_texture_table(m->Textures, m->TextureCount, off, pool.p, ctx->stream, newRecs));
            CK(d2d(recs.p, ctx->tex.recs.p, old.TextureCount * sizeof(TexRec)));
            CK(h2d(at(recs, old.TextureCount * sizeof(TexRec)), newRecs.data(), m->TextureCount * sizeof(TexRec)));
        }

        // the new BLASes: one batch over the staged, rebased triangles and the grown positions
        if (B) {
            idkbb::StageTimer tm(ctx->stream);
            tm.mark("start");
            std::string err;
            const int brc = idkbb::build_device(ctx->stream, (const PackedVec3*)positions.p, (const GpuBlasTriangle*)at(stage, stTris), in, p,
                                                staged, built, tm, err);
            if (brc != idkbb::BB_OK) return blas_build_fail(ctx, who, brc, err);
            long long fragments = 0;
            for (int c : built.fragmentCount) fragments += c;
            tm.print((int)B, fragments);
            nN += (uint64_t)built.nodeStart[B];
            nT += (uint64_t)built.triStart[B];
            if (nN >= (1ull << 31) || nT >= (1ull << 31)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "scene too large");
            for (uint32_t k = 0; k < B; k++) {            // BVH.cs:363-386
                GpuBlasDesc d = m->BlasDescs[k];
                d.NodeOffset = (int32_t)(old.BlasNodeCount + built.nodeStart[k]);
                d.NodeCount = built.nodeStart[k + 1] - built.nodeStart[k];
                d.TriangleOffset = (int32_t)(old.BlasTriangleCount + built.triStart[k]);
                d.TriangleCount = built.triStart[k + 1] - built.triStart[k];
                d.RequiredStackSize = built.requiredStackSize[k];
                descs.push_back(d);
            }
        }
        for (const GpuBlasDesc& d : descs) stackSize = std::max(stackSize, d.RequiredStackSize);   // BVH.UpdateBlasStackSize
        if ((size_t)std::max(1, stackSize) * IDK_BLOCK * sizeof(uint32_t) > 200 * 1024)
            return fail(ctx, who, IDKPT_ERR_UNSUPPORTED, "BlasStackSize too large for the shared-memory traversal stack");
        nodeBytes = ((nN * sizeof(GpuBlasNode)) + 255) & ~(size_t)255;
        triRecBytes = std::max<size_t>(nT, 1) * 64;
        if (!alloc(bvh, nodeBytes + triRecBytes) || !alloc(tris, nT * sizeof(GpuBlasTriangle)))
            return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
        float4* recNew = (float4*)at(bvh, nodeBytes);
        CK(d2d(bvh.p, ctx->nodes.p, old.BlasNodeCount * sizeof(GpuBlasNode)));
        CK(d2d(recNew, (const char*)ctx->nodes.p + ctx->nodeBytes, old.BlasTriangleCount * 64));
        CK(d2d(tris.p, ctx->blasTris.p, old.BlasTriangleCount * sizeof(GpuBlasTriangle)));
        CK(d2d(descBuf.p, ctx->descs.p, old.BlasDescCount * sizeof(GpuBlasDesc)));
        if (B) {
            CK(d2d((GpuBlasNode*)bvh.p + old.BlasNodeCount, built.nodes, (size_t)built.nodeStart[B] * sizeof(GpuBlasNode)));
            CK(d2d((GpuBlasTriangle*)tris.p + old.BlasTriangleCount, built.tris, (size_t)built.triStart[B] * sizeof(GpuBlasTriangle)));
            if (const uint32_t n = (uint32_t)built.triStart[B])
                k_prepare_triangles<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const int4*)tris.p + old.BlasTriangleCount, (const float*)positions.p,
                                                                              recNew + 4 * old.BlasTriangleCount, n);
            CK(h2d(at(descBuf, old.BlasDescCount * sizeof(GpuBlasDesc)), descs.data() + old.BlasDescCount, B * sizeof(GpuBlasDesc)));
        }

        // BVH.TlasBuild(true) in ModelManager.Add: the device PLOC build over every instance, TLAS.BuildSettings.SearchRadius 15
        if (old.UseTlas) {
            if (!alloc(tlas, (2 * nI - 1) * sizeof(GpuTlasNode))) return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
            if (int trc = enqueue_tlas_build(ctx, bvh.p, descBuf.p, instances.p, xforms.p, tlas.p, nI, 15, &needDev)) return trc;
        }
        return IDKPT_OK;
    });
    if (rc) return rc;
    if (needDev) {
        int need = 0;
        CK(cudaMemcpy(&need, needDev, 4, cudaMemcpyDeviceToHost));
        if (need < 0)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "an instance's world box is not finite or its half area overflows (ModelMatrix or BLAS root)");
        if (need > IDK_TLAS_STACK_SIZE)
            return fail(ctx, who, IDKPT_ERR_UNSUPPORTED, "the TLAS is deeper than the 24-entry traversal stack of the TLAS walk (BVHIntersect.glsl:4)");
    }

    // commit: launch configuration and L2 window for the new arrays first (restored if either fails), then the swap
    const int oldStack = ctx->sc.stackSize;
    ctx->sc.stackSize = std::max(1, stackSize);
    if ((rc = configure_launches(ctx)) || (rc = set_l2_window(ctx, bvh.p, nodeBytes + triRecBytes))) {
        const std::string err = ctx->lastError;
        ctx->sc.stackSize = oldStack;
        configure_launches(ctx);
        set_l2_window(ctx, ctx->nodes.p, ctx->nodeBytes + std::max<size_t>(ctx->counts.BlasTriangleCount, 1) * 64);
        ctx->lastError = err;
        return rc;
    }
    std::swap(ctx->positions, positions);                // `drop` frees the old arrays
    std::swap(ctx->vertices, vertices);
    std::swap(ctx->xforms, xforms);
    std::swap(ctx->meshes, meshes);
    std::swap(ctx->materials, materials);
    std::swap(ctx->instances, instances);
    std::swap(ctx->vtxFrame, vtxFrame);
    std::swap(ctx->surfRec, surfRec);
    std::swap(ctx->descs, descBuf);
    std::swap(ctx->blasTris, tris);
    std::swap(ctx->nodes, bvh);
    if (old.UseTlas) std::swap(ctx->tlas, tlas);
    if (m->TextureCount) {
        std::swap(ctx->tex.recs, recs);
        ctx->tex.pools.push_back(pool);
        pool = DevBuf{};
    }
    if (m->UnskinnedVertexCount) std::swap(ctx->unskinned, unskinned);
    release(ctx->prevPositions);                         // re-created from the positions at its next use (ModelManager.cs:620)

    DeviceScene& sc = ctx->sc;
    sc.nodes = (const float4*)ctx->nodes.p;
    sc.triRec = (const float4*)((char*)ctx->nodes.p + nodeBytes);
    sc.blasTris = (const int4*)ctx->blasTris.p;
    sc.descs = (const GpuBlasDesc*)ctx->descs.p;
    sc.instances = (const GpuBlasInstance*)ctx->instances.p;
    sc.xforms = (const float4*)ctx->xforms.p;
    sc.meshes = (const GpuMesh*)ctx->meshes.p;
    sc.materials = (const GpuMaterial*)ctx->materials.p;
    sc.vertices = (const uint4*)ctx->vertices.p;
    sc.instanceCount = (uint32_t)nI;
    sc.tlasNodes = (const float4*)ctx->tlas.p;
    sc.vtxFrame = (const float4*)ctx->vtxFrame.p;
    sc.surfRec = (const float4*)ctx->surfRec.p;
    sc.textures = (const TexRec*)ctx->tex.recs.p;
    sc.textureCount = (uint32_t)nTex;
    IdkPtSceneDesc& c = ctx->counts;
    c.BlasNodeCount = nN; c.BlasTriangleCount = nT; c.BlasDescCount = nB; c.BlasInstanceCount = nI;
    if (old.UseTlas) c.TlasNodeCount = 2 * nI - 1;
    c.MeshTransformCount = nX; c.MeshCount = nM; c.MaterialCount = nMat; c.VertexCount = nV; c.VertexPositionCount = nV;
    c.BlasStackSize = stackSize; c.TextureCount = nTex;
    ctx->nodeBytes = nodeBytes;
    ctx->hostDescs = std::move(descs);
    for (uint64_t i = 0; i < m->BlasInstanceCount; i++)
        ctx->hostInstances.push_back({m->BlasInstances[i].BlasId + (uint32_t)old.BlasDescCount, m->BlasInstances[i].MeshTransformId + (uint32_t)old.MeshTransformCount});
    for (uint64_t i = 0; i < m->MaterialCount; i++) {
        const uint64_t h = material_max_handle(m->Materials[i]);
        ctx->hostMaterialMaxHandle.push_back(h ? h + old.TextureCount : 0);
    }
    for (uint64_t i = 0; i < m->UnskinnedVertexCount; i++) {
        const uint32_t* j = m->UnskinnedVertices[i].JointIndices;
        ctx->unskinnedMaxJoint.push_back(std::max(std::max(j[0], j[1]), std::max(j[2], j[3])));
    }
    ctx->unskinnedCount = nU;
    ctx->sceneGeneration++;                              // a bound voxeliser re-sizes its work queue for the new draw list
    ctx->accumulatedSamples = 0;
    return IDKPT_OK;
}

// BLAS.ComputeGlobalSAH (BLAS.cs:629-656) of each BLAS in [first, first + count) as the device holds it now: k_global_sah.
IDKPT_API int idkpt_blas_sah(IdkPtCtx* ctx, uint32_t first, uint32_t count, const IdkPtBlasBuildSettings* settings, double* sahOut) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (!sahOut && count) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_sah: null argument");
    DRAIN_PENDING("idkpt_blas_sah");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_blas_sah: no scene");
    if ((uint64_t)first + count > ctx->hostDescs.size()) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_sah: BLAS range outside BlasDescs");
    const float triangleCost = settings ? settings->TriangleCost : idkbvh::Params().triangleCost;
    if (!std::isfinite(triangleCost)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_blas_sah: non-finite TriangleCost");
    if (count == 0) return IDKPT_OK;
    CK(cudaSetDevice(ctx->device));
    int maxNodes = 0;
    for (uint32_t b = first; b < first + count; b++) maxNodes = std::max(maxNodes, ctx->hostDescs[b].NodeCount);
    CK(ensure(ctx->sahScratch, (size_t)count * sizeof(double) + (size_t)maxNodes * sizeof(int)));
    double* out = (double*)ctx->sahScratch.p;
    int* stack = (int*)(out + count);
    return run_timed(ctx, "idkpt_blas_sah", nullptr, [&]() -> int {
        for (uint32_t k = 0; k < count; k++)
            idkbb::k_global_sah<<<1, 1, 0, ctx->stream>>>((const GpuBlasNode*)ctx->nodes.p + ctx->hostDescs[first + k].NodeOffset, stack, triangleCost, out + k);
        return IDKPT_OK;
    }, sahOut, out, (size_t)count * sizeof(double));
}

IDKPT_API int idkpt_read_range(IdkPtCtx* ctx, IdkPtArrayId which, uint64_t first, uint64_t count, void* out) {
    if (!ctx || (!out && count)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_range: null argument");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_read_range: no scene");
    const DevBuf* b = nullptr;
    size_t elem = 0;
    uint64_t limit = 0;
    switch (which) {
        case IDKPT_ARRAY_BLAS_NODES: b = &ctx->nodes; elem = sizeof(GpuBlasNode); limit = ctx->counts.BlasNodeCount; break;
        case IDKPT_ARRAY_VERTEX_POSITIONS: b = &ctx->positions; elem = sizeof(PackedVec3); limit = ctx->counts.VertexPositionCount; break;
        case IDKPT_ARRAY_VERTICES: b = &ctx->vertices; elem = sizeof(GpuVertex); limit = ctx->counts.VertexCount; break;
        case IDKPT_ARRAY_TLAS_NODES: b = &ctx->tlas; elem = sizeof(GpuTlasNode); limit = ctx->counts.UseTlas ? ctx->counts.TlasNodeCount : 0; break;
        case IDKPT_ARRAY_BLAS_TRIANGLES: b = &ctx->blasTris; elem = sizeof(GpuBlasTriangle); limit = ctx->counts.BlasTriangleCount; break;
        case IDKPT_ARRAY_BLAS_DESCS: b = &ctx->descs; elem = sizeof(GpuBlasDesc); limit = ctx->counts.BlasDescCount; break;
        default: return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_range: array id not readable");
    }
    if (first > limit || count > limit - first) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_range: range outside the array");
    CK(cudaSetDevice(ctx->device));
    if (count) CK(cudaMemcpyAsync(out, (const char*)b->p + first * elem, count * elem, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

static int trace_rays_impl(IdkPtCtx* ctx, const IdkPtRay* rays, uint64_t count, int32_t traceLights, IdkPtHit* hitsOut, float* kernelMs, bool anyHit) {
    if (!ctx || (!rays && count) || (!hitsOut && count)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_trace_rays: null argument");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_trace_rays: no scene");
    if (count >= (1ull << 31)) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_trace_rays: too many rays");
    if (kernelMs) *kernelMs = 0.0f;
    if (count == 0) return IDKPT_OK;
    CK(cudaSetDevice(ctx->device));
    DevBuf &dr = ctx->scratch[0], &dh = ctx->scratch[1], &dt = ctx->scratch[2];
    if (ensure(dr, count * 32) != cudaSuccess || ensure(dh, count * 32) != cudaSuccess || ensure(dt, 16) != cudaSuccess)
        return fail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkpt_trace_rays: device allocation failed");
    CK(cudaMemcpyAsync(dr.p, rays, count * 32, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(dt.p, 0, 16, ctx->stream));
    TraceRaysArgs a;
    a.sc = ctx->sc;
    a.rays = (const float4*)dr.p;
    a.hits = (uint4*)dh.p;
    a.count = (uint32_t)count;
    a.ticket = (uint32_t*)dt.p;
    a.traceLights = traceLights;
    return run_timed(ctx, "idkpt_trace_rays", kernelMs, [&]() -> int {
        if (anyHit) k_trace_rays_any<<<ctx->traceRaysBlocks, IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        else k_trace_rays<<<ctx->traceRaysBlocks, IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        return IDKPT_OK;
    }, hitsOut, dh.p, count * 32);
}

IDKPT_API int idkpt_trace_rays(IdkPtCtx* ctx, const IdkPtRay* rays, uint64_t count, int32_t traceLights, IdkPtHit* hitsOut, float* kernelMs) {
    return trace_rays_impl(ctx, rays, count, traceLights, hitsOut, kernelMs, false);
}

IDKPT_API int idkpt_trace_rays_any(IdkPtCtx* ctx, const IdkPtRay* rays, uint64_t count, int32_t traceLights, IdkPtHit* hitsOut, float* kernelMs) {
    return trace_rays_impl(ctx, rays, count, traceLights, hitsOut, kernelMs, true);
}

// ---- point-shadow cube maps (PointShadowManager.UpdateBuffer / RenderShadowMaps) ----------------------------------------------
IDKPT_API int idkpt_set_point_shadows(IdkPtCtx* ctx, const GpuPointShadow* shadows, const int32_t* sizes, uint32_t count) {
    if (!ctx || (count && (!shadows || !sizes))) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_point_shadows: null argument");
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_set_point_shadows: no scene");
    if (count > IDKPT_MAX_POINT_SHADOWS) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_point_shadows: more than IDKPT_MAX_POINT_SHADOWS shadows");
    for (uint32_t i = 0; i < count; i++) {
        if (sizes[i] < 1 || sizes[i] > 16384) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_point_shadows: size outside 1..16384");
        if (!(shadows[i].NearPlane > 0.0f) || !std::isfinite(shadows[i].NearPlane))
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_point_shadows: NearPlane must be > 0");
        if (!(shadows[i].FarPlane > shadows[i].NearPlane) || !std::isfinite(shadows[i].FarPlane))
            return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_set_point_shadows: FarPlane must be > NearPlane");
    }
    CK(cudaSetDevice(ctx->device));
    std::vector<PointShadowDev> recs(count);
    std::vector<int32_t> lightIndex(count);   // checked against the light count where it is read (idkpt_volumetric_lighting)
    size_t texels = 0;
    for (uint32_t i = 0; i < count; i++) {
        lightIndex[i] = shadows[i].LightIndex;
        PointShadowDev& r = recs[i];
        for (int k = 0; k < 3; k++) r.pos[k] = shadows[i].Position[k];
        r.nearPlane = shadows[i].NearPlane; r.farPlane = shadows[i].FarPlane;
        r.size = sizes[i];
        r.offset = texels;
        texels += 6 * (size_t)sizes[i] * (size_t)sizes[i];
    }
    if (std::vector<int32_t>(sizes, sizes + count) != ctx->pointShadowSizes) {
        // new layout: the maps start cleared to 65535 (ShadowMap.Fill(1.0))
        ctx->pointShadowSizes.clear();
        ctx->pointShadows.clear();
        ctx->pointShadowRecs.clear();
        release(ctx->pointShadowMaps);
        if (ensure(ctx->pointShadowMaps, std::max<size_t>(texels, 1) * 2) != cudaSuccess)
            return fail(ctx, IDKPT_ERR_OUT_OF_MEMORY, "idkpt_set_point_shadows: cube-map allocation failed");
        CK(cudaMemsetAsync(ctx->pointShadowMaps.p, 0xFF, texels * 2, ctx->stream));
    }
    if (int rc = upload(ctx, ctx->pointShadowDev, recs.data(), recs.size() * sizeof(PointShadowDev))) return rc;
    if (int rc = upload(ctx, ctx->pointShadowLights, lightIndex.data(), lightIndex.size() * sizeof(int32_t))) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->pointShadows.assign(shadows, shadows + count);
    ctx->pointShadowSizes.assign(sizes, sizes + count);
    ctx->pointShadowRecs = recs;
    return IDKPT_OK;
}

IDKPT_API int idkpt_render_point_shadows(IdkPtCtx* ctx, uint32_t first, uint32_t count, const uint32_t* faceMasks, float* kernelMs) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    if (!ctx->haveScene) return fail(ctx, IDKPT_ERR_NO_SCENE, "idkpt_render_point_shadows: no scene");
    const uint32_t have = (uint32_t)ctx->pointShadowRecs.size();
    if (first > have || count > have - first) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_render_point_shadows: shadow range outside the set shadows");
    for (uint32_t i = 0; faceMasks && i < count; i++)
        if (faceMasks[i] > 0x3Fu) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_render_point_shadows: face mask has bits above the six faces");
    if (kernelMs) *kernelMs = 0.0f;
    if (count == 0) return IDKPT_OK;
    CK(cudaSetDevice(ctx->device));
    return run_timed(ctx, "idkpt_render_point_shadows", kernelMs, [&]() -> int {
        for (uint32_t i = first; i < first + count; i++) {
            const PointShadowDev& r = ctx->pointShadowRecs[i];
            const uint32_t mask = faceMasks ? faceMasks[i - first] : 0x3Fu;
            PointShadowRenderArgs a;
            a.sc = ctx->sc;
            for (int k = 0; k < 3; k++) a.pos[k] = r.pos[k];
            a.nearPlane = r.nearPlane; a.farPlane = r.farPlane; a.size = r.size;
            a.map = (uint16_t*)ctx->pointShadowMaps.p + r.offset;
            int faces = 0;
            for (int f = 0; f < 6; f++) if (mask & (1u << f)) a.faces[faces++] = f;
            if (faces == 0) continue;
            const size_t tilesX = ((size_t)r.size + 7) / 8, tiles = tilesX * tilesX;
            const dim3 grid((unsigned)((tiles + IDK_BLOCK / 64 - 1) / (IDK_BLOCK / 64)), (unsigned)faces);
            k_point_shadow_faces<<<grid, IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        }
        return IDKPT_OK;
    });
}

IDKPT_API int idkpt_point_shadow_device_ptr(IdkPtCtx* ctx, int32_t index, void** devPtr, uint64_t* bytes) {
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_point_shadow_device_ptr: null argument");
    if (index < 0 || (size_t)index >= ctx->pointShadowRecs.size()) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_point_shadow_device_ptr: shadow index out of range");
    const PointShadowDev& r = ctx->pointShadowRecs[index];
    *devPtr = (uint16_t*)ctx->pointShadowMaps.p + r.offset;
    if (bytes) *bytes = 6 * (uint64_t)r.size * (uint64_t)r.size * 2;
    return IDKPT_OK;
}

IDKPT_API int idkpt_read_point_shadow(IdkPtCtx* ctx, int32_t index, uint16_t* dst, uint64_t bytes) {
    if (!ctx || !dst) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_point_shadow: null argument");
    if (index < 0 || (size_t)index >= ctx->pointShadowRecs.size()) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_point_shadow: shadow index out of range");
    const PointShadowDev& r = ctx->pointShadowRecs[index];
    const uint64_t need = 6 * (uint64_t)r.size * (uint64_t)r.size * 2;
    if (bytes < need) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_read_point_shadow: buffer too small");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(dst, (const uint16_t*)ctx->pointShadowMaps.p + r.offset, need, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

// ---- the raster passes: their shared checks, input stage and output images ----------------------------------------------------
// Their messages read "<entry point>: <what>" (fail(ctx, who, ...)); a null context goes through the template fail, so that
// idkpt_last_error(NULL) reports it.

static int size_check(IdkCtxBase* ctx, const char* who, int w, int h) {
    if (w < 1 || h < 1 || w > 16384 || h > 16384) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "size outside 1..16384");
    return IDKPT_OK;
}

// The shadowed lighting modes read the point shadow of every light whose PointShadowIndex is not -1.
static int shadow_index_check(IdkPtCtx* ctx, const char* who) {
    for (const GpuLight& L : ctx->hostLights)
        if (L.PointShadowIndex != -1 && (L.PointShadowIndex < 0 || (size_t)L.PointShadowIndex >= ctx->pointShadowRecs.size()))
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a light's PointShadowIndex is neither -1 nor below the point-shadow count");
    return IDKPT_OK;
}

// The TAA jitter of a call in NDC units: taaJitter[0..1], or none without the array. Returns whether both are finite.
static bool read_jitter(const float* taaJitter, float jitter[2]) {
    jitter[0] = taaJitter ? taaJitter[0] : 0.0f;
    jitter[1] = taaJitter ? taaJitter[1] : 0.0f;
    return std::isfinite(jitter[0]) && std::isfinite(jitter[1]);
}

// The grid of a raster kernel over 8x8-pixel tiles, four tiles per block.
static unsigned tile_blocks(int w, int h) {
    const size_t tiles = (size_t)((w + 7) / 8) * (size_t)((h + 7) / 8);
    return (unsigned)((tiles + 3) / 4);
}

// One input image of a raster call: the caller's array of `floats` floats per pixel, or (floats 0) an image of the context,
// read in place. The caller's arrays are read in place when the call's OnDevice is 1: each must then be device memory on the
// context's device, aligned to the width of the kernels' loads of it (`align` bytes), else the call fails with `misaligned`.
struct StageInput {
    const float* src;
    size_t floats;
    size_t align;
    const char* misaligned;
};

// A G-buffer attachment: loaded as float2 when it has two floats per pixel, as floats otherwise.
static StageInput attachment(const float* src, size_t floats) {
    return floats == 2 ? StageInput{src, 2, 8, "OnDevice NormalRG / MetallicRoughness pointer not 8-byte aligned"}
                       : StageInput{src, floats, 4, "OnDevice pointer not 4-byte aligned"};
}

static StageInput velocity_input(const float* src) { return {src, 2, 8, "OnDevice VelocityRG pointer not 8-byte aligned"}; }

// The input stage of a raster call over w x h pixels. Checks every OnDevice array first, so that a rejected pointer is never
// read and nothing has been allocated or invalidated; then uploads the host arrays into `stage`, each at a 256-byte aligned
// offset. Writes the device pointer of every input to dev[], in order (null for a null src: an input the call does not use).
static int stage_inputs_into(IdkCtxBase* ctx, DevBuf& stageBuf, const char* who, int w, int h, int onDevice, const std::vector<StageInput>& in,
                             const float** dev) {
    const size_t pixels = (size_t)w * h;
    size_t bytes = 0;
    for (const StageInput& i : in) {
        if (!i.src || !i.floats) continue;
        if (!onDevice) {
            bytes += (pixels * i.floats * 4 + 255) & ~(size_t)255;
            continue;
        }
        cudaPointerAttributes attr;
        const cudaError_t e = cudaPointerGetAttributes(&attr, i.src);
        if (e != cudaSuccess) cudaGetLastError();   // not a pointer CUDA knows: clear the error, reject below
        if (e != cudaSuccess || !(attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) || attr.device != ctx->device)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "OnDevice = 1 with a pointer that is not device memory on the context's device");
        if ((uintptr_t)i.src % i.align != 0) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, i.misaligned);
    }
    if (bytes && ensure(stageBuf, bytes) != cudaSuccess) return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    char* stage = (char*)stageBuf.p;
    for (const StageInput& i : in) {
        *dev = i.src;
        if (i.src && i.floats && !onDevice) {
            CK(cudaMemcpyAsync(stage, i.src, pixels * i.floats * 4, cudaMemcpyHostToDevice, ctx->stream));
            *dev = (const float*)stage;
            stage += (pixels * i.floats * 4 + 255) & ~(size_t)255;
        }
        dev++;
    }
    return IDKPT_OK;
}

// The raster passes of the path-tracer context stage into its raster stage.
static int stage_inputs(IdkPtCtx* ctx, const char* who, int w, int h, int onDevice, const std::vector<StageInput>& in, const float** dev) {
    return stage_inputs_into(ctx, ctx->raster.stage, who, w, h, onDevice, in, dev);
}

// A G-buffer's size and OnDevice; the callers check the attachments they read.
static int gbuffer_shape_check(IdkCtxBase* ctx, const char* who, const IdkPtGBuffer* g) {
    if (int rc = size_check(ctx, who, g->Width, g->Height)) return rc;
    if (g->OnDevice != 0 && g->OnDevice != 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "OnDevice is neither 0 nor 1");
    return IDKPT_OK;
}

static int gbuffer_check(IdkCtxBase* ctx, const char* who, const IdkPtGBuffer* g, bool all) {
    if (!g->Depth || !g->NormalRG || (all && (!g->AlbedoRGB || !g->MetallicRoughness || !g->EmissiveRGB)))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "null argument");
    return gbuffer_shape_check(ctx, who, g);
}

// The lit-image selector (IdkPtLitSource), checked before anything is allocated: a caller array, or a context image of w x h.
static int lit_source_check(IdkPtCtx* ctx, const char* who, int32_t source, bool allowMerged, const float* color, int w, int h) {
    if (source != IDKPT_LIT_SOURCE_ARRAY && source != IDKPT_LIT_SOURCE_DEFERRED && (!allowMerged || source != IDKPT_LIT_SOURCE_MERGED))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, allowMerged ? "source is not ARRAY, DEFERRED or MERGED" : "source is neither ARRAY nor DEFERRED");
    if (source == IDKPT_LIT_SOURCE_ARRAY && !color) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "ARRAY source without a colour array");
    if (source == IDKPT_LIT_SOURCE_DEFERRED && !ctx->raster.deferred.valid_at(w, h))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "DEFERRED source needs an idkpt_deferred_lighting image of the render size");
    if (source == IDKPT_LIT_SOURCE_MERGED && !ctx->raster.ssr.valid_at(w, h))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "MERGED source needs an idkpt_ssr image of the render size");
    return IDKPT_OK;
}

// The input entry of that lit image: the caller's rgba32f array, or the context's deferred or merged image.
static StageInput lit_input(IdkPtCtx* ctx, int32_t source, const float* color) {
    if (source == IDKPT_LIT_SOURCE_DEFERRED) return {(const float*)ctx->raster.deferred.buf[0].p, 0, 0, nullptr};
    if (source == IDKPT_LIT_SOURCE_MERGED) return {(const float*)ctx->raster.ssr.buf[0].p, 0, 0, nullptr};
    return {color, 4, 16, "OnDevice colour pointer not 16-byte aligned"};
}

// The checks of the *_device_ptr exports: a context, somewhere to write, and the image `img` as its pass (`producer`) left it
// after a successful call. Returns the image, or null with the error (IDKPT_ERR_INVALID_ARGUMENT) set.
static const RasterImage* published_image(IdkPtCtx* ctx, const char* who, bool haveOut, RasterImage RasterState::*img, const char* producer) {
    if (!ctx || !haveOut) {
        fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, (std::string(who) + ": null argument").c_str());
        return nullptr;
    }
    const RasterImage& r = ctx->raster.*img;
    if (!r.valid()) {
        fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, (std::string("call ") + producer + " first").c_str());
        return nullptr;
    }
    return &r;
}

// A one-image *_device_ptr export: the image's device pointer and its size in bytes, `texelBytes` per texel, one texel per
// tile x tile pixels.
static int image_device_ptr(IdkPtCtx* ctx, const char* who, RasterImage RasterState::*img, const char* producer, uint64_t texelBytes,
                            int tile, void** devPtr, uint64_t* bytes) {
    const RasterImage* r = published_image(ctx, who, devPtr != nullptr, img, producer);
    if (!r) return IDKPT_ERR_INVALID_ARGUMENT;
    *devPtr = r->buf[r->last].p;
    if (bytes) *bytes = (uint64_t)((r->w + tile - 1) / tile) * ((r->h + tile - 1) / tile) * texelBytes;
    return IDKPT_OK;
}

// ---- volumetric lighting (VolumetricLighting.Compute: march + depth-aware upscale) ---------------------------------------------
// Both entry points: g's Depth (g->Width x g->Height, the other attachments unused), read in place when g->OnDevice is 1.
static int volumetric_lighting(IdkPtCtx* ctx, const char* who, const GpuPerFrameData* frame, const IdkPtVolumetricSettings* s,
                               const IdkPtGBuffer* g, int32_t width, int32_t height, const float* taaJitter, uint16_t* outRgba16f,
                               float* kernelMs) {
    const int depthWidth = g->Width, depthHeight = g->Height;
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = gbuffer_shape_check(ctx, who, g)) return rc;
    if (int rc = size_check(ctx, who, width, height)) return rc;
    if (s->SampleCount < 1 || s->SampleCount > 1024) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "SampleCount outside 1..1024");
    if (!(s->ResolutionScale > 0.0f && s->ResolutionScale <= 1.0f)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "ResolutionScale not in (0, 1]");
    // VolumetricLighting.SetSize: (Vector2i)((Vector2)PresentationResolution * ResolutionScale), truncated
    const int w = (int)((float)width * s->ResolutionScale), h = (int)((float)height * s->ResolutionScale);
    if (w < 1 || h < 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "render size of 0 (ResolutionScale too small for the size)");
    for (const GpuPointShadow& ps : ctx->pointShadows)
        if (ps.LightIndex < 0 || (uint64_t)ps.LightIndex >= ctx->counts.LightCount)
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a shadow's LightIndex is not below the scene's light count");
    CK(cudaSetDevice(ctx->device));
    const float* gdepth;
    if (int rc = stage_inputs(ctx, who, depthWidth, depthHeight, g->OnDevice, {attachment(g->Depth, 1)}, &gdepth)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    RasterState& r = ctx->raster;
    const size_t nRender = (size_t)w * h, nOut = (size_t)width * height;
    r.vol.invalidate();            // the image may be reallocated and is overwritten: valid again only when the call succeeds
    if (ensure(r.volMarch, nRender * 8) != cudaSuccess || ensure(r.volDepth, nRender * 4) != cudaSuccess || ensure(r.vol.buf[0], nOut * 8) != cudaSuccess)
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    VolumetricMarchArgs a;
    a.shadows = (const PointShadowDev*)ctx->pointShadowDev.p; a.lightIndex = (const int32_t*)ctx->pointShadowLights.p;
    a.lights = ctx->sc.lights; a.maps = (const uint16_t*)ctx->pointShadowMaps.p; a.count = (int)ctx->pointShadowRecs.size();
    a.gdepth = gdepth; a.gw = depthWidth; a.gh = depthHeight;
    a.color = (uint2*)r.volMarch.p; a.depth = (float*)r.volDepth.p; a.w = w; a.h = h;
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    for (int k = 0; k < 3; k++) { a.viewPos[k] = frame->ViewPos[k]; a.absorbance[k] = s->Absorbance[k]; }
    read_jitter(taaJitter, a.jitter);
    a.sampleCount = s->SampleCount; a.scattering = s->Scattering; a.strength = s->Strength; a.maxDist = s->MaxDist;
    VolumetricUpscaleArgs b;
    b.gdepth = a.gdepth; b.gw = depthWidth; b.gh = depthHeight;
    b.march = PostImage{nullptr, (const uint2*)r.volMarch.p, w, h};
    b.depth = (const float*)r.volDepth.p;
    b.out = (uint2*)r.vol.buf[0].p; b.W = width; b.H = height;
    b.nearPlane = frame->NearPlane; b.farPlane = frame->FarPlane;
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_volumetric_march<<<tile_blocks(w, h), 256, 0, ctx->stream>>>(a);
        k_volumetric_upscale<<<dim3((unsigned)((width + 31) / 32), (unsigned)((height + 7) / 8)), 256, 0, ctx->stream>>>(b);
        return IDKPT_OK;
    }, outRgba16f, r.vol.buf[0].p, outRgba16f ? nOut * 8 : 0);
    if (rc == IDKPT_OK) r.vol.publish(width, height);
    return rc;
}

IDKPT_API int idkpt_volumetric_lighting(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtVolumetricSettings* s, const float* depth,
                                        int32_t depthWidth, int32_t depthHeight, int32_t width, int32_t height, const float* taaJitter,
                                        uint16_t* outRgba16f, float* kernelMs) {
    if (!ctx || !frame || !s || !depth) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_volumetric_lighting: null argument");
    const IdkPtGBuffer g{depthWidth, depthHeight, 0, depth, nullptr, nullptr, nullptr, nullptr};
    return volumetric_lighting(ctx, "idkpt_volumetric_lighting", frame, s, &g, width, height, taaJitter, outRgba16f, kernelMs);
}

IDKPT_API int idkpt_volumetric_lighting_gbuffer(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtVolumetricSettings* s, const IdkPtGBuffer* g,
                                                int32_t width, int32_t height, const float* taaJitter, uint16_t* outRgba16f, float* kernelMs) {
    if (!ctx || !frame || !s || !g || !g->Depth) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_volumetric_lighting_gbuffer: null argument");
    return volumetric_lighting(ctx, "idkpt_volumetric_lighting_gbuffer", frame, s, g, width, height, taaJitter, outRgba16f, kernelMs);
}

IDKPT_API int idkpt_volumetric_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    return image_device_ptr(ctx, "idkpt_volumetric_device_ptr", &RasterState::vol, "idkpt_volumetric_lighting", 8, 1, devPtr, bytes);
}

// ---- G-buffer lighting (SSAO.Compute, the deferred lighting draw) -------------------------------------------------------------
IDKPT_API int idkpt_ssao(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtSsaoSettings* s, const IdkPtGBuffer* g, uint8_t* outR8, float* kernelMs) {
    static const char* who = "idkpt_ssao";
    if (!ctx || !frame || !s || !g) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_ssao: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = gbuffer_check(ctx, who, g, false)) return rc;
    if (s->SampleCount < 1 || s->SampleCount > 1024) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "SampleCount outside 1..1024");
    CK(cudaSetDevice(ctx->device));
    const float* in[2];
    if (int rc = stage_inputs(ctx, who, g->Width, g->Height, g->OnDevice, {attachment(g->Depth, 1), attachment(g->NormalRG, 2)}, in)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    RasterImage& out = ctx->raster.ssao;
    const size_t n = (size_t)g->Width * g->Height;
    out.invalidate();              // the image may be reallocated and is overwritten: valid again only when the call succeeds
    if (ensure(out.buf[0], n) != cudaSuccess) return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    SsaoArgs a;
    a.g = DeferredGBuffer{in[0], (const float2*)in[1], nullptr, nullptr, nullptr, g->Width, g->Height};
    a.out = (uint8_t*)out.buf[0].p;
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    memcpy(a.projView, frame->ProjView, sizeof(a.projView));
    a.sampleCount = s->SampleCount; a.radius = s->Radius; a.strength = s->Strength; a.noiseIndex = s->NoiseIndex;
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_ssao<<<tile_blocks(g->Width, g->Height), 256, 0, ctx->stream>>>(a);
        return IDKPT_OK;
    }, outR8, out.buf[0].p, outR8 ? n : 0);
    if (rc == IDKPT_OK) out.publish(g->Width, g->Height);
    return rc;
}

IDKPT_API int idkpt_ssao_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    return image_device_ptr(ctx, "idkpt_ssao_device_ptr", &RasterState::ssao, "idkpt_ssao", 1, 1, devPtr, bytes);
}

// The RayTraced mode's visibility images (PointShadowManager.ComputeRayTracedShadowMaps for one light) into the image of `slot`
// (ctx->raster.rtShadow). Pixels with depth == 1 keep what the image held, as the shader returns early there: the caller's
// array with `seed` (uploaded first), else the last successful call's values when the image has the G-buffer's size, else 0.
// The deferred pass never reads those pixels (DeferredLighting/fragment.glsl returns early on them too).
static int shadows_ray_traced(IdkPtCtx* ctx, const char* who, const GpuPerFrameData* frame, const IdkPtGBuffer* g, int32_t lightIndex,
                              int32_t samples, uint32_t noiseIndex, const float* taaJitter, int slot, const float* seed,
                              float* visibilityOut, float* kernelMs) {
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = gbuffer_check(ctx, who, g, false)) return rc;
    if (samples < 1 || samples > 1024) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "samples outside 1..1024");
    if (lightIndex < 0 || (uint64_t)lightIndex >= ctx->counts.LightCount) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "light index out of range");
    CK(cudaSetDevice(ctx->device));
    const float* in[2];
    if (int rc = stage_inputs(ctx, who, g->Width, g->Height, g->OnDevice, {attachment(g->Depth, 1), attachment(g->NormalRG, 2)}, in)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    RasterImage& out = ctx->raster.rtShadow[slot];
    const size_t bytes = (size_t)g->Width * g->Height * 4;
    const bool keep = out.valid_at(g->Width, g->Height);
    out.invalidate();              // the image may be reallocated and is overwritten: valid again only when the call succeeds
    if (ensure(out.buf[0], bytes) != cudaSuccess) return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    if (seed) CK(cudaMemcpyAsync(out.buf[0].p, seed, bytes, cudaMemcpyHostToDevice, ctx->stream));
    else if (!keep) CK(cudaMemsetAsync(out.buf[0].p, 0, bytes, ctx->stream));
    ShadowArgs a;
    a.sc = ctx->sc;
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    read_jitter(taaJitter, a.jitter);
    a.depth = in[0]; a.normalRG = (const float2*)in[1]; a.visibility = (float*)out.buf[0].p;
    a.width = g->Width; a.height = g->Height; a.lightIndex = lightIndex; a.samples = samples; a.noiseIndex = noiseIndex;
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_shadows_ray_traced<<<ctx->traceRaysBlocks, IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        return IDKPT_OK;
    }, visibilityOut, out.buf[0].p, visibilityOut ? bytes : 0);
    if (rc == IDKPT_OK) out.publish(g->Width, g->Height);
    return rc;
}

// From host arrays: visibility_out is read-modify-write, through the context's own image (the slot after the last public one).
IDKPT_API int idkpt_shadows_ray_traced(IdkPtCtx* ctx, const GpuPerFrameData* frame, const float* depth, const float* normalRG, int32_t width,
                                       int32_t height, int32_t lightIndex, int32_t samples, uint32_t noiseIndex, const float* taaJitter,
                                       float* visibilityOut, float* kernelMs) {
    static const char* who = "idkpt_shadows_ray_traced";
    if (!ctx || !frame || !depth || !normalRG || !visibilityOut) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_shadows_ray_traced: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (width < 1 || height < 1 || width > 16384 || height > 16384 || samples < 1 || samples > 1024) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "invalid size / sample count");
    const IdkPtGBuffer g{width, height, 0, depth, normalRG, nullptr, nullptr, nullptr};
    return shadows_ray_traced(ctx, who, frame, &g, lightIndex, samples, noiseIndex, taaJitter, IDKPT_MAX_POINT_SHADOWS, visibilityOut,
                              visibilityOut, kernelMs);
}

IDKPT_API int idkpt_shadows_ray_traced_gbuffer(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtGBuffer* g, int32_t lightIndex,
                                               int32_t samples, uint32_t noiseIndex, const float* taaJitter, int32_t slot, float* visibilityOut,
                                               float* kernelMs) {
    static const char* who = "idkpt_shadows_ray_traced_gbuffer";
    if (!ctx || !frame || !g) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_shadows_ray_traced_gbuffer: null argument");
    if (slot < 0 || slot >= IDKPT_MAX_POINT_SHADOWS) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "slot outside 0..IDKPT_MAX_POINT_SHADOWS - 1");
    return shadows_ray_traced(ctx, who, frame, g, lightIndex, samples, noiseIndex, taaJitter, slot, nullptr, visibilityOut, kernelMs);
}

IDKPT_API int idkpt_shadows_device_ptr(IdkPtCtx* ctx, int32_t slot, void** devPtr, uint64_t* bytes) {
    static const char* who = "idkpt_shadows_device_ptr";
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_shadows_device_ptr: null argument");
    if (slot < 0 || slot >= IDKPT_MAX_POINT_SHADOWS) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "slot outside 0..IDKPT_MAX_POINT_SHADOWS - 1");
    const RasterImage& r = ctx->raster.rtShadow[slot];
    if (!r.valid()) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "call idkpt_shadows_ray_traced_gbuffer for the slot first");
    *devPtr = r.buf[0].p;
    if (bytes) *bytes = (uint64_t)r.w * r.h * 4;
    return IDKPT_OK;
}

IDKPT_API int idkpt_deferred_lighting(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtDeferredSettings* s, const IdkPtGBuffer* g,
                                      const float* taaJitter, const float* indirect, const float* const* rtVisibility, uint32_t rtCount,
                                      float* outRgba32f, float* kernelMs) {
    static const char* who = "idkpt_deferred_lighting";
    if (!ctx || !frame || !s || !g) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_deferred_lighting: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = gbuffer_check(ctx, who, g, true)) return rc;
    if (s->ShadowMode < 0 || s->ShadowMode > 2) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "ShadowMode outside 0..2");
    if (s->IsVariableRateShading != 0 && s->IsVariableRateShading != 1)
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVariableRateShading is neither 0 nor 1");
    RasterState& r = ctx->raster;
    if (s->IsVariableRateShading && !r.vrs.valid_at(g->Width, g->Height))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVariableRateShading needs an idkpt_shading_rate image of the G-buffer's size");
    if (s->IsVXGI && !indirect) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVXGI without an indirect-light image");
    if (s->IsSSAO && !r.ssao.valid_at(g->Width, g->Height))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsSSAO needs an idkpt_ssao image of the G-buffer's size");
    if (s->ShadowMode != 0)
        if (int rc = shadow_index_check(ctx, who)) return rc;
    const uint32_t shadowCount = (uint32_t)ctx->pointShadowRecs.size();
    if (s->ShadowMode == 2) {
        if (rtCount < shadowCount || (rtCount && !rtVisibility))
            return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "RayTraced needs a visibility image per point shadow");
        for (uint32_t i = 0; i < rtCount; i++)
            if (!rtVisibility[i]) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a visibility image is null");
    }
    CK(cudaSetDevice(ctx->device));
    const uint32_t rtUsed = s->ShadowMode == 2 ? shadowCount : 0;
    std::vector<StageInput> inputs = {attachment(g->Depth, 1), attachment(g->NormalRG, 2), attachment(g->AlbedoRGB, 3),
                                      attachment(g->MetallicRoughness, 2), attachment(g->EmissiveRGB, 3),
                                      {s->IsVXGI ? indirect : nullptr, 4, 16, "OnDevice indirect-light pointer not 16-byte aligned"}};
    for (uint32_t i = 0; i < rtUsed; i++) inputs.push_back(attachment(rtVisibility[i], 1));
    std::vector<const float*> in(inputs.size());   // the G-buffer, the indirect light, the visibility images
    if (int rc = stage_inputs(ctx, who, g->Width, g->Height, g->OnDevice, inputs, in.data())) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    const size_t n = (size_t)g->Width * g->Height;
    const int tilesX = (g->Width + IDK_VRS_TILE - 1) / IDK_VRS_TILE, vrsTiles = tilesX * ((g->Height + IDK_VRS_TILE - 1) / IDK_VRS_TILE);
    r.deferred.invalidate();       // the image may be reallocated and is overwritten: valid again only when the call succeeds
    if (ensure(r.deferred.buf[0], n * 16) != cudaSuccess || (s->IsVariableRateShading && ensure(r.vrsOffsets, ((size_t)vrsTiles + 1) * 4) != cudaSuccess))
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    if (rtUsed)
        if (int rc = upload(ctx, r.rtPtrs, in.data() + 6, rtUsed * sizeof(const float*))) return rc;
    DeferredArgs a;
    a.g = DeferredGBuffer{in[0], (const float2*)in[1], in[2], (const float2*)in[3], in[4], g->Width, g->Height};
    a.ssao = s->IsSSAO ? (const uint8_t*)r.ssao.buf[0].p : nullptr;
    a.indirect = (const float4*)in[5];
    a.rtVisibility = rtUsed ? (const float* const*)r.rtPtrs.p : nullptr;
    a.lights = ctx->sc.lights; a.lightCount = (int)ctx->counts.LightCount;
    a.shadows = PointShadowMapsDev{(const PointShadowDev*)ctx->pointShadowDev.p, (const uint16_t*)ctx->pointShadowMaps.p, shadowCount};
    a.out = (float4*)r.deferred.buf[0].p;
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    for (int k = 0; k < 3; k++) a.viewPos[k] = frame->ViewPos[k];
    read_jitter(taaJitter, a.jitter);
    a.shadowMode = s->ShadowMode;
    const VrsTiles v{(const uint8_t*)r.vrs.buf[0].p, (uint32_t*)r.vrsOffsets.p, g->Width, g->Height, tilesX, vrsTiles};
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        if (s->IsVariableRateShading) {   // the fragment list, then one thread per coarse fragment (grid sized for all 1x1)
            k_vrs_scan<<<1, 1024, 0, ctx->stream>>>(v);
            k_deferred_lighting_vrs<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(a, v);
        } else {
            k_deferred_lighting<<<tile_blocks(g->Width, g->Height), 256, 0, ctx->stream>>>(a);
        }
        return IDKPT_OK;
    }, outRgba32f, r.deferred.buf[0].p, outRgba32f ? n * 16 : 0);
    if (rc == IDKPT_OK) r.deferred.publish(g->Width, g->Height);
    return rc;
}

IDKPT_API int idkpt_deferred_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    return image_device_ptr(ctx, "idkpt_deferred_device_ptr", &RasterState::deferred, "idkpt_deferred_lighting", 16, 1, devPtr, bytes);
}

// ---- the end of the raster frame (SSR.Compute, "Merge Textures", TaaResolve.Compute) --------------------------------------------
IDKPT_API int idkpt_ssr(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtSsrSettings* s, const IdkPtGBuffer* g, int32_t source,
                        const float* color, float* mergedOut, uint16_t* ssrOut, float* kernelMs) {
    static const char* who = "idkpt_ssr";
    if (!ctx || !frame || !s || !g) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_ssr: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = gbuffer_check(ctx, who, g, false)) return rc;
    if (!g->AlbedoRGB || !g->MetallicRoughness) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "null argument");
    if (s->SampleCount < 1 || s->SampleCount > 1024) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "SampleCount outside 1..1024");
    if (s->BinarySearchCount < 0 || s->BinarySearchCount > 64) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "BinarySearchCount outside 0..64");
    if (!std::isfinite(s->MaxDist)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "MaxDist not finite");
    CK(cudaSetDevice(ctx->device));
    if (int rc = lit_source_check(ctx, who, source, false, color, g->Width, g->Height)) return rc;
    const float* in[5];            // the lit image, the G-buffer
    if (int rc = stage_inputs(ctx, who, g->Width, g->Height, g->OnDevice, {lit_input(ctx, source, color), attachment(g->Depth, 1),
                              attachment(g->NormalRG, 2), attachment(g->AlbedoRGB, 3), attachment(g->MetallicRoughness, 2)}, in)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    RasterImage& out = ctx->raster.ssr;
    const size_t n = (size_t)g->Width * g->Height;
    out.invalidate();              // the images may be reallocated and are overwritten: valid again only when the call succeeds
    if (ensure(out.buf[0], n * 16) != cudaSuccess || ensure(out.buf[1], n * 8) != cudaSuccess)
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    SsrArgs a;
    a.g = DeferredGBuffer{in[1], (const float2*)in[2], in[3], (const float2*)in[4], nullptr, g->Width, g->Height};
    a.src = (const float4*)in[0];
    a.ssr = (uint2*)out.buf[1].p;
    a.merged = (float4*)out.buf[0].p;
    a.sc = ctx->sc;
    memcpy(a.projection, frame->Projection, sizeof(a.projection));
    memcpy(a.invProjection, frame->InvProjection, sizeof(a.invProjection));
    memcpy(a.invView, frame->InvView, sizeof(a.invView));
    a.sampleCount = s->SampleCount; a.binarySearchCount = s->BinarySearchCount; a.maxDist = s->MaxDist;
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_ssr<<<tile_blocks(g->Width, g->Height), 256, 0, ctx->stream>>>(a);
        return IDKPT_OK;
    }, mergedOut, out.buf[0].p, mergedOut ? n * 16 : 0);
    if (rc != IDKPT_OK) return rc;
    if (ssrOut) {
        CK(cudaMemcpyAsync(ssrOut, out.buf[1].p, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    out.publish(g->Width, g->Height);
    return IDKPT_OK;
}

IDKPT_API int idkpt_ssr_device_ptrs(IdkPtCtx* ctx, void** mergedDevPtr, void** ssrDevPtr, uint64_t* mergedBytes, uint64_t* ssrBytes) {
    const RasterImage* r = published_image(ctx, "idkpt_ssr_device_ptrs", mergedDevPtr || ssrDevPtr, &RasterState::ssr, "idkpt_ssr");
    if (!r) return IDKPT_ERR_INVALID_ARGUMENT;
    const uint64_t n = (uint64_t)r->w * r->h;
    if (mergedDevPtr) *mergedDevPtr = r->buf[0].p;
    if (ssrDevPtr) *ssrDevPtr = r->buf[1].p;
    if (mergedBytes) *mergedBytes = n * 16;
    if (ssrBytes) *ssrBytes = n * 8;
    return IDKPT_OK;
}

IDKPT_API int idkpt_taa_resolve(IdkPtCtx* ctx, const IdkPtTaaSettings* s, const IdkPtTaaInputs* in, int width, int height, uint16_t* out,
                                float* kernelMs) {
    static const char* who = "idkpt_taa_resolve";
    if (!ctx || !s || !in || !in->Depth || !in->VelocityRG) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_taa_resolve: null argument");
    if (int rc = size_check(ctx, who, in->Width, in->Height)) return rc;
    if (int rc = size_check(ctx, who, width, height)) return rc;
    if (in->OnDevice != 0 && in->OnDevice != 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "OnDevice is neither 0 nor 1");
    if (s->IsNaiveTaa != 0 && s->IsNaiveTaa != 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsNaiveTaa is neither 0 nor 1");
    if (s->SampleCount < 1 || s->SampleCount > 1024) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "SampleCount outside 1..1024");
    if (!std::isfinite(s->PreferAliasingOverBlur)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "PreferAliasingOverBlur not finite");
    CK(cudaSetDevice(ctx->device));
    if (int rc = lit_source_check(ctx, who, in->Source, true, in->ColorRgba32f, in->Width, in->Height)) return rc;
    const float* src[3];           // the lit image, depth, velocity
    if (int rc = stage_inputs(ctx, who, in->Width, in->Height, in->OnDevice, {lit_input(ctx, in->Source, in->ColorRgba32f),
                              attachment(in->Depth, 1), velocity_input(in->VelocityRG)}, src)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    RasterState& r = ctx->raster;
    r.taa.invalidate();            // valid again only when the call succeeds
    const size_t bytes = (size_t)width * height * 8;
    if (width != r.taa.w || height != r.taa.h) {   // a new presentation size restarts from a zero history
        r.taa.w = r.taa.h = 0;
        if (ensure(r.taa.buf[0], bytes) != cudaSuccess || ensure(r.taa.buf[1], bytes) != cudaSuccess)
            return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
        CK(cudaMemsetAsync(r.taa.buf[0].p, 0, bytes, ctx->stream));
        CK(cudaMemsetAsync(r.taa.buf[1].p, 0, bytes, ctx->stream));
        r.taa.w = width; r.taa.h = height;
    }
    r.taaFrame++;
    const int dst = r.taaFrame % 2 == 0 ? 0 : 1;
    TaaArgs a;
    a.color = PostImage{(const float4*)src[0], nullptr, in->Width, in->Height};
    a.depth = src[1];
    a.velocity = (const float2*)src[2];
    a.history = PostImage{nullptr, (const uint2*)r.taa.buf[1 - dst].p, width, height};
    a.out = (uint2*)r.taa.buf[dst].p;
    a.W = width; a.H = height;
    a.isNaive = s->IsNaiveTaa; a.sampleCount = s->SampleCount; a.preferAliasingOverBlur = s->PreferAliasingOverBlur;
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_taa_resolve<<<tile_blocks(width, height), 256, 0, ctx->stream>>>(a);
        return IDKPT_OK;
    }, out, r.taa.buf[dst].p, out ? bytes : 0);
    if (rc == IDKPT_OK) r.taa.publish(width, height, dst);
    return rc;
}

IDKPT_API int idkpt_taa_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    return image_device_ptr(ctx, "idkpt_taa_device_ptr", &RasterState::taa, "idkpt_taa_resolve", 8, 1, devPtr, bytes);
}

// ---- variable-rate deferred lighting (LightingShadingRateClassifier.Compute) ---------------------------------------------------
IDKPT_API int idkpt_shading_rate(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtShadingRateSettings* s, const IdkPtShadingRateInputs* in,
                                 uint8_t* outRates, float* debugOut, float* kernelMs) {
    static const char* who = "idkpt_shading_rate";
    if (!ctx || !frame || !s || !in || !in->VelocityRG) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_shading_rate: null argument");
    if (int rc = size_check(ctx, who, in->Width, in->Height)) return rc;
    if (in->OnDevice != 0 && in->OnDevice != 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "OnDevice is neither 0 nor 1");
    if (s->DebugMode < 0 || s->DebugMode > 4) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "DebugMode outside 0..4");
    if (debugOut && s->DebugMode < 2) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "a debug image needs DebugMode 2, 3 or 4");
    if (!std::isfinite(s->SpeedFactor) || !std::isfinite(s->LumVarianceFactor))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "SpeedFactor or LumVarianceFactor not finite");
    CK(cudaSetDevice(ctx->device));
    if (int rc = lit_source_check(ctx, who, in->Source, false, in->ColorRgba32f, in->Width, in->Height)) return rc;
    const float* src[2];           // the lit image, velocity
    if (int rc = stage_inputs(ctx, who, in->Width, in->Height, in->OnDevice, {lit_input(ctx, in->Source, in->ColorRgba32f),
                              velocity_input(in->VelocityRG)}, src)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    const unsigned tilesX = (unsigned)(in->Width + IDK_VRS_TILE - 1) / IDK_VRS_TILE, tilesY = (unsigned)(in->Height + IDK_VRS_TILE - 1) / IDK_VRS_TILE;
    const size_t tiles = (size_t)tilesX * tilesY;
    RasterImage& out = ctx->raster.vrs;
    out.invalidate();              // the images may be reallocated and are overwritten: valid again only when the call succeeds
    const bool debug = s->DebugMode >= 2;
    if (ensure(out.buf[0], tiles) != cudaSuccess || (debug && ensure(out.buf[1], tiles * 4) != cudaSuccess))
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    ShadingRateArgs a;
    a.color = (const float4*)src[0];
    a.velocity = (const float2*)src[1];
    a.w = in->Width; a.h = in->Height;
    a.deltaRenderTime = frame->DeltaRenderTime; a.speedFactor = s->SpeedFactor; a.lumVarianceFactor = s->LumVarianceFactor;
    a.debugMode = s->DebugMode;
    a.rates = (uint8_t*)out.buf[0].p;
    a.debug = debug ? (float*)out.buf[1].p : nullptr;
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_shading_rate<<<dim3(tilesX, tilesY), 256, 0, ctx->stream>>>(a);
        return IDKPT_OK;
    }, outRates, out.buf[0].p, outRates ? tiles : 0);
    if (rc != IDKPT_OK) return rc;
    if (debugOut) {
        CK(cudaMemcpyAsync(debugOut, out.buf[1].p, tiles * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    out.publish(in->Width, in->Height);
    return IDKPT_OK;
}

IDKPT_API int idkpt_shading_rate_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    return image_device_ptr(ctx, "idkpt_shading_rate_device_ptr", &RasterState::vrs, "idkpt_shading_rate", 1, IDK_VRS_TILE, devPtr, bytes);
}

// ---- the G-buffer pass (RasterPipeline.Render's "Fill G-Buffer" draws) --------------------------------------------------------
// The six attachments' planes in one allocation, each 256-byte aligned: Depth 1, NormalRG 2, AlbedoRGB 3, MetallicRoughness 2,
// EmissiveRGB 3, VelocityRG 2 floats per pixel. Returns the total size.
static size_t gbuffer_planes(int w, int h, size_t offsets[6]) {
    static const size_t floats[6] = {1, 2, 3, 2, 3, 2};
    size_t n = 0;
    for (int i = 0; i < 6; i++) {
        offsets[i] = n;
        n += (((size_t)w * h * floats[i] * 4) + 255) & ~(size_t)255;
    }
    return n;
}

IDKPT_API int idkpt_gbuffer(IdkPtCtx* ctx, const GpuPerFrameData* frame, int32_t width, int32_t height, const float* taaJitter,
                            const PackedVec3* prevPositions, float* kernelMs) {
    static const char* who = "idkpt_gbuffer";
    if (!ctx || !frame) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_gbuffer: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = size_check(ctx, who, width, height)) return rc;
    GBufferArgs a;
    if (!read_jitter(taaJitter, a.jitter)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "jitter not finite");
    CK(cudaSetDevice(ctx->device));
    if (kernelMs) *kernelMs = 0.0f;
    RasterState& r = ctx->raster;
    size_t off[6];
    const size_t bytes = gbuffer_planes(width, height, off);
    const size_t prevBytes = ctx->counts.VertexPositionCount * sizeof(PackedVec3);
    // idkpt_prev_positions_device_ptr's buffer is read in place; any other pointer is a host array
    const bool kept = prevPositions && (const void*)prevPositions == ctx->prevPositions.p;
    const bool hostPrev = prevPositions && !kept;
    r.gb.invalidate();             // the images may be reallocated and are overwritten: valid again only when the call succeeds
    if (ensure(r.gb.buf[0], bytes) != cudaSuccess || (hostPrev && ensure(r.gbPrev, std::max<size_t>(prevBytes, 16)) != cudaSuccess))
        return fail(ctx, who, IDKPT_ERR_OUT_OF_MEMORY, "device allocation failed");
    if (hostPrev && prevBytes) CK(cudaMemcpyAsync(r.gbPrev.p, prevPositions, prevBytes, cudaMemcpyHostToDevice, ctx->stream));
    char* base = (char*)r.gb.buf[0].p;
    a.sc = ctx->sc;
    a.positions = (const float*)ctx->positions.p;
    a.prevPositions = kept ? (const float*)ctx->prevPositions.p : hostPrev ? (const float*)r.gbPrev.p : a.positions;
    memcpy(a.projView, frame->ProjView, sizeof(a.projView));
    memcpy(a.prevProjView, frame->PrevProjView, sizeof(a.prevProjView));
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    for (int k = 0; k < 3; k++) a.viewPos[k] = frame->ViewPos[k];
    a.w = width; a.h = height;
    a.depth = (float*)(base + off[0]); a.normalRG = (float2*)(base + off[1]); a.albedo = (float*)(base + off[2]);
    a.metallicRoughness = (float2*)(base + off[3]); a.emissive = (float*)(base + off[4]); a.velocity = (float2*)(base + off[5]);
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        k_gbuffer<<<tile_blocks(width, height), IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        return IDKPT_OK;
    });
    if (rc == IDKPT_OK) r.gb.publish(width, height);
    return rc;
}

IDKPT_API int idkpt_gbuffer_device_ptrs(IdkPtCtx* ctx, IdkPtGBuffer* gbufferOut, const float** velocityOut) {
    const RasterImage* r = published_image(ctx, "idkpt_gbuffer_device_ptrs", gbufferOut || velocityOut, &RasterState::gb, "idkpt_gbuffer");
    if (!r) return IDKPT_ERR_INVALID_ARGUMENT;
    size_t off[6];
    gbuffer_planes(r->w, r->h, off);
    const char* base = (const char*)r->buf[0].p;
    if (gbufferOut)
        *gbufferOut = IdkPtGBuffer{r->w, r->h, 1, (const float*)(base + off[0]), (const float*)(base + off[1]),
                                   (const float*)(base + off[2]), (const float*)(base + off[3]), (const float*)(base + off[4])};
    if (velocityOut) *velocityOut = (const float*)(base + off[5]);
    return IDKPT_OK;
}

IDKPT_API int idkpt_prev_positions_device_ptr(IdkPtCtx* ctx, void** devPtr, uint64_t* bytes) {
    static const char* who = "idkpt_prev_positions_device_ptr";
    if (!ctx || !devPtr) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_prev_positions_device_ptr: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    CK(cudaSetDevice(ctx->device));
    if (!ctx->prevPositions.p) {
        if (int rc = keep_prev_positions(ctx)) return rc;
        CK(cudaStreamSynchronize(ctx->stream));    // the copy is complete before the pointer is handed out
    }
    *devPtr = ctx->prevPositions.p;
    if (bytes) *bytes = ctx->counts.VertexPositionCount * sizeof(PackedVec3);
    return IDKPT_OK;
}

IDKPT_API int idkpt_read_gbuffer(IdkPtCtx* ctx, float* depth, float* normalRG, float* albedoRGB, float* metallicRoughness,
                                 float* emissiveRGB, float* velocityRG) {
    if (!ctx) return IDKPT_ERR_INVALID_ARGUMENT;
    const RasterImage& gb = ctx->raster.gb;
    if (!gb.valid()) return fail(ctx, "idkpt_read_gbuffer", IDKPT_ERR_INVALID_ARGUMENT, "call idkpt_gbuffer first");
    CK(cudaSetDevice(ctx->device));
    size_t off[6];
    gbuffer_planes(gb.w, gb.h, off);
    float* dst[6] = {depth, normalRG, albedoRGB, metallicRoughness, emissiveRGB, velocityRG};
    static const size_t floats[6] = {1, 2, 3, 2, 3, 2};
    const size_t n = (size_t)gb.w * gb.h;
    for (int i = 0; i < 6; i++)
        if (dst[i]) CK(cudaMemcpyAsync(dst[i], (const char*)gb.buf[0].p + off[i], n * floats[i] * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

} // extern "C"

#include "idkvx_impl.cuh"

// ---- transparency (RasterPipeline.Render's "Record transparent fragments" + "Resolve transparent fragments") -------------------
// After the voxeliser's context (idkvx_impl.cuh): the VXGI path cone-traces that context's grid.
extern "C" {

IDKPT_API int idkpt_transparency(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtTransparencySettings* s, const IdkPtGBuffer* g,
                                 const float* taaJitter, IdkVxCtx* voxels, const IdkVxConeSettings* cone, int32_t source, float* color,
                                 float* outRgba32f, float* kernelMs) {
    static const char* who = "idkpt_transparency";
    if (!ctx || !frame || !s || !g || !g->Depth) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_transparency: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    if (int rc = size_check(ctx, who, g->Width, g->Height)) return rc;
    if (g->OnDevice != 0 && g->OnDevice != 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "OnDevice is neither 0 nor 1");
    if (s->ShadowMode < 0 || s->ShadowMode > 2) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "ShadowMode outside 0..2");
    if (s->IsVXGI != 0 && s->IsVXGI != 1) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVXGI is neither 0 nor 1");
    if (s->IsVXGI) {
        if (!voxels || !cone) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVXGI without a voxeliser context or cone settings");
        if (!voxels->voxelized) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVXGI with a voxeliser context that has not voxelised its grid");
        if (voxels->device != ctx->device) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "IsVXGI with a voxeliser context on another device");
        if (cone->MaxSamples < 1 || cone->MaxSamples > 64) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "cone MaxSamples out of range");
    }
    TransparencyArgs a;
    if (!read_jitter(taaJitter, a.jitter)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "jitter not finite");
    if (s->ShadowMode == 1)
        if (int rc = shadow_index_check(ctx, who)) return rc;
    CK(cudaSetDevice(ctx->device));
    if (int rc = lit_source_check(ctx, who, source, false, color, g->Width, g->Height)) return rc;
    const float* in[2];            // the lit image (the stage copy, the caller's device array or the context's deferred image), depth
    if (int rc = stage_inputs(ctx, who, g->Width, g->Height, g->OnDevice, {lit_input(ctx, source, color), attachment(g->Depth, 1)}, in)) return rc;
    if (kernelMs) *kernelMs = 0.0f;
    const size_t n = (size_t)g->Width * g->Height;
    const bool hostArray = source == IDKPT_LIT_SOURCE_ARRAY && !g->OnDevice;
    a.sc = ctx->sc;
    a.positions = (const float*)ctx->positions.p;
    memcpy(a.projView, frame->ProjView, sizeof(a.projView));
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    for (int k = 0; k < 3; k++) a.viewPos[k] = frame->ViewPos[k];
    a.w = g->Width; a.h = g->Height;
    a.depth = in[1];
    a.color = (float4*)in[0];      // written in place
    a.shadowMode = s->ShadowMode;
    a.shadows = PointShadowMapsDev{(const PointShadowDev*)ctx->pointShadowDev.p, (const uint16_t*)ctx->pointShadowMaps.p,
                                   (uint32_t)ctx->pointShadowRecs.size()};
    a.g = s->IsVXGI ? voxels->grid : VxGridDev{};
    a.cone = s->IsVXGI ? VxConeParams{cone->MaxSamples, cone->StepMultiplier, cone->GIBoost, cone->GISkyBoxBoost, cone->NormalRayOffset, cone->NoiseIndex}
                       : VxConeParams{1, 0.0f, 0.0f, 0.0f, 0.0f, 0u};
    const int rc = run_timed(ctx, who, kernelMs, [&]() -> int {
        if (s->IsVXGI) k_transparency<true><<<tile_blocks(g->Width, g->Height), IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        else k_transparency<false><<<tile_blocks(g->Width, g->Height), IDK_BLOCK, ctx->stackBytes, ctx->stream>>>(a);
        return IDKPT_OK;
    });
    if (rc != IDKPT_OK) return rc;
    if (hostArray) CK(cudaMemcpyAsync(color, in[0], n * 16, cudaMemcpyDeviceToHost, ctx->stream));
    if (outRgba32f) CK(cudaMemcpyAsync(outRgba32f, in[0], n * 16, cudaMemcpyDeviceToHost, ctx->stream));
    if (hostArray || outRgba32f) CK(cudaStreamSynchronize(ctx->stream));
    return IDKPT_OK;
}

// ---- the light spheres and the skybox (RasterPipeline.Render's "Draw lights" + "Draw skybox") ---------------------------------
IDKPT_API int idkpt_lights_and_skybox(IdkPtCtx* ctx, const GpuPerFrameData* frame, const float* taaJitter, float* outRgba32f,
                                      float* kernelMs) {
    static const char* who = "idkpt_lights_and_skybox";
    if (!ctx || !frame) return fail(ctx, IDKPT_ERR_INVALID_ARGUMENT, "idkpt_lights_and_skybox: null argument");
    if (!ctx->haveScene) return fail(ctx, who, IDKPT_ERR_NO_SCENE, "no scene");
    const RasterState& r = ctx->raster;
    if (!r.gb.valid()) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "call idkpt_gbuffer first");
    if (!r.deferred.valid_at(r.gb.w, r.gb.h))
        return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "needs an idkpt_deferred_lighting image of the G-buffer's size");
    LightsSkyboxArgs a;
    if (!read_jitter(taaJitter, a.jitter)) return fail(ctx, who, IDKPT_ERR_INVALID_ARGUMENT, "jitter not finite");
    CK(cudaSetDevice(ctx->device));
    if (kernelMs) *kernelMs = 0.0f;
    const int w = r.gb.w, h = r.gb.h;
    size_t off[6];
    gbuffer_planes(w, h, off);
    char* base = (char*)r.gb.buf[0].p;
    a.sc = ctx->sc;
    a.lights = ctx->sc.lights; a.lightCount = (int)ctx->counts.LightCount;
    memcpy(a.projView, frame->ProjView, sizeof(a.projView));
    memcpy(a.prevProjView, frame->PrevProjView, sizeof(a.prevProjView));
    memcpy(a.invProjView, frame->InvProjView, sizeof(a.invProjView));
    memcpy(a.projection, frame->Projection, sizeof(a.projection));
    memcpy(a.invProjection, frame->InvProjection, sizeof(a.invProjection));
    memcpy(a.invView, frame->InvView, sizeof(a.invView));
    memcpy(a.prevView, frame->PrevView, sizeof(a.prevView));
    for (int k = 0; k < 3; k++) a.viewPos[k] = frame->ViewPos[k];
    a.w = w; a.h = h;
    a.depth = (float*)(base + off[0]); a.normalRG = (float2*)(base + off[1]); a.emissive = (float*)(base + off[4]);
    a.velocity = (float2*)(base + off[5]);
    a.color = (float4*)r.deferred.buf[0].p;
    return run_timed(ctx, who, kernelMs, [&]() -> int {
        k_lights_skybox<<<tile_blocks(w, h), 256, 0, ctx->stream>>>(a);
        return IDKPT_OK;
    }, outRgba32f, r.deferred.buf[0].p, outRgba32f ? (size_t)w * h * 16 : 0);
}

} // extern "C"
