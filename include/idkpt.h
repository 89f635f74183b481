/*
 * idkpt.h -- C ABI of libidkpt, the H100-native replacement for the body of
 * IDKEngine.Render.PathTracer (reference: IDKEngine/Source/Render/PathTracer.cs).
 *
 * The C# class keeps its public surface (ctor / Compute / SetSize /
 * ResetAccumulation / properties, PathTracer.cs:10-125,170-346); its GL
 * dispatch sequence (PathTracer.cs:214-297) is replaced by P/Invoke calls into
 * the functions below (binding shown in INTEGRATION.md). Scene data that the
 * reference binds implicitly to fixed SSBO/UBO slots (ModelManager.cs:103-119,
 * BVH.cs:145-152, LightManager.cs:80) is handed over explicitly, in the same
 * struct layouts (idk_gpu_types.h).
 *
 * Conventions (mirroring the reference's own native interop, SRC/OIDN/OIDN.cs:
 * opaque handles, plain pointers + sizes, error string getter):
 *   - every function returns IDKPT_OK (0) or a negative IdkPtStatus;
 *   - idkpt_last_error() returns a UTF-8 string owned by the library;
 *   - host arrays are borrowed only for the duration of the call (copied);
 *   - a context is single-threaded (the engine's render thread);
 *   - there is NO CPU fallback: without a usable CUDA device idkpt_create fails.
 */
#ifndef IDKPT_H
#define IDKPT_H

#include "idk_gpu_types.h"

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define IDKPT_API __declspec(dllexport)
#else
#define IDKPT_API __attribute__((visibility("default")))
#endif

typedef struct IdkPtCtx IdkPtCtx;

typedef enum IdkPtStatus {
    IDKPT_OK = 0,
    IDKPT_ERR_INVALID_ARGUMENT = -1,
    IDKPT_ERR_NO_DEVICE = -2,
    IDKPT_ERR_CUDA = -3,
    IDKPT_ERR_NO_SCENE = -4,
    IDKPT_ERR_OUT_OF_MEMORY = -5,
    IDKPT_ERR_UNSUPPORTED = -6
} IdkPtStatus;

#define IDKPT_MAX_RAY_DEPTH 64

/* Replaces: new PathTracer(width, height, settings)   (PathTracer.cs:170-212).
 * Tile fields implement the multi-GPU screen split (one context per GPU):
 * image rows are cut into stripes of TileStripeHeight rows, stripe s belongs to
 * context (s % TileCount) == TileIndex. TileCount <= 1 => the whole image. */
#define IDKPT_CREATE_LANES(n) (((uint32_t)(n) & 15u) << 8)
/* Multi-GPU, strict parity: NHit seeds a ray's random numbers with its slot in the alive list (NHit/compute.glsl:
 * gl_GlobalInvocationID.x). By default a tile numbers its own alive rays (the N-GPU image is then a valid, but different,
 * Monte-Carlo estimate than the 1-GPU image, reproducible per GPU count). With this flag the ranks exchange their per-stripe
 * alive counts over NVLink once per bounce so that every ray gets its WHOLE-IMAGE slot: the N-GPU image is bit-identical to
 * the 1-GPU image. Needs the peers connected (idkpt_gather_import / idkpt_gather_connect) and every rank issuing the same
 * idkpt_compute calls; not available together with DoRaySorting. Ignored when TileCount <= 1. */
#define IDKPT_CREATE_GLOBAL_SLOTS (1u << 12)

typedef struct IdkPtCreateInfo {
    int32_t Device;            /* CUDA device ordinal */
    int32_t Width;
    int32_t Height;
    int32_t TileStripeHeight;  /* rows per stripe (multiple of 8), 0 => 8 */
    int32_t TileIndex;
    int32_t TileCount;
    uint32_t Flags;            /* 0, IDKPT_CREATE_LANES(n): samples in flight for asynchronous idkpt_compute (default 8, 1 = off), IDKPT_CREATE_GLOBAL_SLOTS */
} IdkPtCreateInfo;

/* Replaces the implicit SSBO bindings 4,5(vertices),8,9..: ModelManager.cs:103-119
 * (meshes, materials, vertices, positions, transforms) and BVH.cs:145-152,445-451
 * (nodes, triangles, descs, instances, tlas) plus LightManager.cs:80 (UBO 2). */
/* Material textures. The reference stores 64-bit GL bindless sampler handles in GpuMaterial (GpuMaterial.cs:8-67); here a
 * handle is an index into this table: 0 = the 1x1 white fallback (ModelLoader.cs:1855-1870), k > 0 = Textures[k-1]. Base
 * level only: the path tracer's compute shaders sample lod 0 (Surface.glsl:57-60). Uncompressed RGBA8 as the loader
 * creates for non-KTX images (BaseColor/Emissive sRGB, ModelLoader.cs:938-945), or the BC7 / BC5 / BC4 level-0 block stream of
 * a KTX2 image as it comes out of the loader's transcoder (decoded on the GPU at upload).
 * Channel use as in Surface.glsl:49-77: BaseColor rgba, MetallicRoughness r = metallic g = roughness, Normal rg,
 * Emissive rgb, Transmission r. */
typedef enum IdkPtTextureFormat {
    IDKPT_TEX_RGBA8_UNORM = 0, IDKPT_TEX_RGBA8_SRGB = 1,   /* what the loader creates for PNG / JPG images (ModelLoader.cs:938-945) */
    /* ABI 3: the KTX2 formats of ModelLoader.cs:954-968, handed over as the level-0 block stream exactly as the loader gives it
     * to glCompressedTextureSubImage2D: ceil(W/4) x ceil(H/4) blocks, row-major. Decoded once at upload (csrc/idk_bcn.cuh). */
    IDKPT_TEX_BC7_UNORM = 2, IDKPT_TEX_BC7_SRGB = 3,       /* 16-byte blocks -> exact RGBA8 */
    IDKPT_TEX_BC5_RG_UNORM = 4,                            /* 16-byte blocks (RGTC2) -> (R, G, 0, 1) in fp32 */
    IDKPT_TEX_BC4_R_UNORM = 5,                             /* 8-byte blocks (RGTC1) -> (R, 0, 0, 1) in fp32 */
    IDKPT_TEX_RG32F = 6, IDKPT_TEX_R32F = 7, IDKPT_TEX_RGBA32F = 8   /* uncompressed float texels (e.g. the R11G11B10F metallic-roughness image) */
} IdkPtTextureFormat;
#define IDKPT_TEX_FLAG_R_FROM_B 1   /* texture.SetSwizzleR(Swizzle.B): BC7 / RGBA metallic-roughness images keep metallic in B (ModelLoader.cs:989-994) */
#define IDKPT_TEX_FLAG_MAG_NEAREST 2 /* the glTF sampler's magFilter is NEAREST (9728; ModelLoader.cs:1166-1196): compute shaders sample at lod 0, i.e.
                                      * under MAGNIFICATION, so the sampler's MagFilter decides between this and bilinear (the default, LINEAR 9729) */
typedef struct IdkPtTextureDesc {
    const void* Pixels;       /* level 0, row 0 first (v = 0): Width*Height texels of the format, or its block stream for BCn */
    int32_t Width, Height;
    int32_t Format;           /* IdkPtTextureFormat */
    int32_t WrapS, WrapT;     /* GL enums as in the glTF sampler: 10497 REPEAT, 33071 CLAMP_TO_EDGE, 33648 MIRRORED_REPEAT */
    int32_t Flags;            /* IDKPT_TEX_FLAG_* (was padding before ABI 3: 0 keeps the old meaning) */
} IdkPtTextureDesc;

typedef struct IdkPtSceneDesc {
    const GpuBlasNode*      BlasNodes;       uint64_t BlasNodeCount;
    const GpuBlasTriangle*  BlasTriangles;   uint64_t BlasTriangleCount;
    const GpuBlasDesc*      BlasDescs;       uint64_t BlasDescCount;
    const GpuBlasInstance*  BlasInstances;   uint64_t BlasInstanceCount;
    const GpuTlasNode*      TlasNodes;       uint64_t TlasNodeCount;     /* may be NULL/0 */
    const GpuMeshTransform* MeshTransforms;  uint64_t MeshTransformCount;
    const GpuMesh*          Meshes;          uint64_t MeshCount;
    const GpuMaterial*      Materials;       uint64_t MaterialCount;
    const GpuVertex*        Vertices;        uint64_t VertexCount;
    const PackedVec3*       VertexPositions; uint64_t VertexPositionCount;
    const GpuLight*         Lights;          uint64_t LightCount;        /* <= 256 */
    int32_t UseTlas;        /* BVH.GpuUseTlas (BVH.cs:18-27); default 0 */
    int32_t BlasStackSize;  /* BVH.BlasStackSize (BVH.cs:29-45,559-567) = max RequiredStackSize */
    const IdkPtTextureDesc* Textures; uint64_t TextureCount;             /* may be NULL/0: every material handle must then be 0 */
} IdkPtSceneDesc;

typedef enum IdkPtArrayId {
    IDKPT_ARRAY_MESH_TRANSFORMS = 0,
    IDKPT_ARRAY_MESHES = 1,
    IDKPT_ARRAY_MATERIALS = 2,
    IDKPT_ARRAY_LIGHTS = 3,
    IDKPT_ARRAY_TLAS_NODES = 4,        /* update + read: BVH.TlasBuild re-upload (BVH.cs:278-283); needs a scene set with UseTlas */
    IDKPT_ARRAY_BLAS_NODES = 5,        /* read only (idkpt_read_range): refitted boxes for the host-side TLAS build */
    IDKPT_ARRAY_VERTEX_POSITIONS = 6,  /* read only: skinned positions (the download behind fenceCopiedSkinnedVerticesToHost, ModelManager.cs:282) */
    IDKPT_ARRAY_VERTICES = 7,          /* read only: skinned normals / tangents */
    IDKPT_ARRAY_BLAS_TRIANGLES = 8,    /* read only: GpuBlasTriangle records (the CPU copy for BVH.Intersect after idkpt_blas_rebuild) */
    IDKPT_ARRAY_BLAS_DESCS = 9         /* read only: GpuBlasDesc records; the last one's ends are the node and triangle totals */
} IdkPtArrayId;

/* Replaces SkyBoxManager's bindless samplerCube in UBO 5 (SkyBoxManager.cs:87):
 * either a constant colour or six rgba32f faces (+X,-X,+Y,-Y,+Z,-Z), FaceSize^2
 * texels each (row-major, GL face orientation), sampled with GL face selection +
 * bilinear filtering inside the face (clamp to edge). */
typedef struct IdkPtSkyDesc {
    float        Color[3];
    int32_t      FaceSize;       /* 0 => constant Color */
    const float* Faces[6];
} IdkPtSkyDesc;

/* PathTracer's runtime-mutable properties (PathTracer.cs:12-125). */
typedef struct IdkPtSettings {
    IdkPtGpuSettings Gpu;        /* FocalLength.. DoRussianRoulette */
    int32_t RayDepth;            /* default 7 (PathTracer.cs:211) */
    int32_t SamplesPerPixel;     /* default 1 (PathTracer.cs:12) */
    int32_t DoRaySorting;        /* default 0 (PathTracer.cs:173) */
    int32_t OutputAOVs;          /* default 0 (PathTracer.cs:174) */
    int32_t CollectStats;        /* count node-pair fetches / triangle tests (debugCost semantics, BVHIntersect.glsl:45,60) */
} IdkPtSettings;

typedef struct IdkPtStats {
    uint64_t Rays;                               /* TraceRay invocations of this call */
    uint64_t BounceRays[IDKPT_MAX_RAY_DEPTH];    /* per bounce, summed over samples */
    uint64_t NodePairFetches;                    /* S (valid if CollectStats) */
    uint64_t TriangleTests;                      /* T (valid if CollectStats) */
    uint64_t InstanceVisits;                     /* I (valid if CollectStats) */
    uint64_t Hits;                               /* rays that hit scene geometry (valid if CollectStats) */
    float    TotalMs;                            /* CUDA-event time of the whole call */
    float    TraverseMs;                         /* sum over traversal launches (bounce 0's includes ray-gen and FirstHit shading) */
    float    ShadeMs;                            /* sum over shade launches (bounces >= 1) + compaction */
    float    SortMs;
    float    OtherMs;                            /* accumulate */
    uint32_t KernelLaunches;
    uint32_t TraverseLaunches;
    float    BounceTraverseMs[IDKPT_MAX_RAY_DEPTH];   /* per bounce, summed over samples */
    float    BounceShadeMs[IDKPT_MAX_RAY_DEPTH];      /* shade + compaction */
    uint32_t BounceMaxSteps[IDKPT_MAX_RAY_DEPTH];     /* longest ray (node-pair fetches) per bounce (valid if CollectStats) */
    float    CompactMs;                          /* ABI 3: the ordered compaction launches alone (also contained in ShadeMs / BounceShadeMs) */
    float    AccumulateMs;                       /* ABI 3: FinalDraw (+ fused peer scatter and arrival wait) alone (also contained in OtherMs) */
} IdkPtStats;

typedef enum IdkPtImage {
    IDKPT_IMAGE_RESULT = 0,   /* PathTracer.Result        (PathTracer.cs:143) */
    IDKPT_IMAGE_ALBEDO = 1,   /* PathTracer.AlbedoTexture (PathTracer.cs:167) */
    IDKPT_IMAGE_NORMAL = 2,   /* PathTracer.NormalTexture (PathTracer.cs:168) */
    IDKPT_IMAGE_GATHERED = 3, /* full multi-GPU Result (idkpt_present_async only; needs idkpt_gather_import) */
    IDKPT_IMAGE_DENOISED = 4  /* PathTracerPipeline's denoised output texture (idkpt_denoise; untiled contexts) */
} IdkPtImage;

/* One ray / hit record of the stand-alone closest-hit query (the GPU analogue of
 * BVH.Intersect(in Ray, out RayHitInfo), SRC/Bvh/BVH.cs:162-193, with the GLSL
 * acceptance rules of SH/include/BVHIntersect.glsl:183-291). */
typedef struct IdkPtRay {
    float Origin[3];
    float TMax;
    float Direction[3];
    float _pad0;
} IdkPtRay;
IDK_STATIC_ASSERT(sizeof(IdkPtRay) == 32, "IdkPtRay must be 32 bytes");

typedef struct IdkPtHit {
    float    BaryX, BaryY;      /* HitInfo.BaryXY (BVHIntersect.glsl:10-16) */
    float    T;                 /* == TMax on miss */
    uint32_t TriangleId;        /* global index into BlasTriangles, ~0u on miss / light */
    uint32_t MeshTransformId;   /* or light index when TriangleId == ~0u and T < TMax */
    uint32_t NodePairFetches;   /* per-ray S */
    uint32_t TriangleTests;     /* per-ray T */
    uint32_t _pad0;
} IdkPtHit;
IDK_STATIC_ASSERT(sizeof(IdkPtHit) == 32, "IdkPtHit must be 32 bytes");

IDKPT_API int idkpt_create(const IdkPtCreateInfo* ci, IdkPtCtx** out);
IDKPT_API void idkpt_destroy(IdkPtCtx* ctx);                                  /* PathTracer.Dispose, PathTracer.cs:344 */
IDKPT_API const char* idkpt_last_error(IdkPtCtx* ctx);                        /* ctx may be NULL: error of the last failed create */

IDKPT_API int idkpt_set_scene(IdkPtCtx* ctx, const IdkPtSceneDesc* scene);    /* ModelManager.Add -> UpdateBuffers + BVH.BlasesBuild uploads (ModelManager.cs:207-213, BVH.cs:445-451) */
IDKPT_API int idkpt_update_range(IdkPtCtx* ctx, IdkPtArrayId which, uint64_t first, uint64_t count, const void* data); /* dirty-range uploads, ModelManager.cs:236-261; LightManager.cs:363-380 */
IDKPT_API int idkpt_set_sky(IdkPtCtx* ctx, const IdkPtSkyDesc* sky);

/* ---- the sky generated on the device (SkyBoxManager's two compute passes; DESIGN.md 8f.1j) ----
 * Both write the context's sky in place, in the layout idkpt_set_sky fills, and leave the context as idkpt_set_sky would with
 * those faces: the face size changes, Color is kept, the accumulation is reset. No scene is needed. Every argument is checked
 * before anything is launched, so a failed call changes no byte of the sky. They are synchronous and ordered after the samples
 * idkpt_compute has queued. kernel_ms (may be NULL): the kernel's CUDA-event time.
 * idkpt_sky_atmosphere: AtmosphericScattering/compute.glsl (the engine's default sky, 128^2) at face_size 1..8192; ISteps and
 *   JSteps 1..1024, every setting finite; LightIntensity is clamped to >= 0 as AtmosphericScatterer.Compute does.
 * idkpt_sky_equirectangular: UnprojectEquirectangular/compute.glsl over a host image of width*height*3 floats, row 0 first
 *   (ImageLoader.Load(path, RGB, true)), uploaded as RGB16F; face size width / 4 (integer division), width 4..32771, height >= 1.
 *   The faces hold RGBA16F values (alpha 1).
 * idkpt_read_sky: the face size (0 for a constant sky) and, when dst is not NULL, the 6 * n^2 * 16 bytes of the faces. */
typedef struct IdkPtAtmosphereSettings {   /* AtmosphericScatterer.GpuSettings (AtmosphericScatterer.cs:9-20) */
    int32_t ISteps;          /* 40 */
    int32_t JSteps;          /* 8 */
    float   LightIntensity;  /* 15 */
    float   Azimuth;         /* 0 */
    float   Elevation;       /* 0 = sun at the zenith (PolarToCartesian, Math.glsl:139-153) */
} IdkPtAtmosphereSettings;
IDKPT_API int idkpt_sky_atmosphere(IdkPtCtx* ctx, const IdkPtAtmosphereSettings* settings, int32_t face_size, float* kernel_ms);
IDKPT_API int idkpt_sky_equirectangular(IdkPtCtx* ctx, const float* rgb, int32_t width, int32_t height, float* kernel_ms);
IDKPT_API int idkpt_read_sky(IdkPtCtx* ctx, int32_t* face_size, float* dst_rgba32f, uint64_t bytes);
/* Replace the material texture table of the current scene (same rules as IdkPtSceneDesc.Textures); every handle stored in
 * a material must remain inside the new table. Resets the accumulation. */
IDKPT_API int idkpt_set_textures(IdkPtCtx* ctx, const IdkPtTextureDesc* textures, uint64_t count);

IDKPT_API int idkpt_resize(IdkPtCtx* ctx, int32_t width, int32_t height);     /* PathTracer.SetSize, PathTracer.cs:299-332 */
IDKPT_API int idkpt_reset_accumulation(IdkPtCtx* ctx);                        /* PathTracer.ResetAccumulation, PathTracer.cs:334 */
IDKPT_API uint32_t idkpt_accumulated_samples(IdkPtCtx* ctx);                  /* PathTracer.AccumulatedSamples, PathTracer.cs:27-37 */
IDKPT_API int idkpt_set_accumulated_samples(IdkPtCtx* ctx, uint32_t n);       /* restore a snapshot taken with idkpt_read_result */

/* PathTracer.Compute(), PathTracer.cs:214-271. Images stay on the device.
 * With stats: synchronous, one sample at a time, per-kernel CUDA-event times filled in.
 * With stats == NULL (and CollectStats / DoDebugBVHTraversal / the wavefront export off): ASYNCHRONOUS. The call queues its
 * samples and returns; up to `lanes` samples are in flight on separate streams, so the few-ray tail bounces of one sample
 * overlap the next sample's first bounces. Each sample's values, and the order in which samples are folded into the
 * images, are exactly those of the synchronous path. idkpt_present_async / idkpt_post_process / idkpt_read_result are
 * ordered after every queued sample; calls that change the scene or hand out device pointers wait for the queue to
 * drain; idkpt_sync waits explicitly and reports device-side errors (kernel fault, multi-GPU gather time-out). */
IDKPT_API int idkpt_compute(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtSettings* settings, IdkPtStats* stats);
IDKPT_API int idkpt_sync(IdkPtCtx* ctx);
/* The context's main (image) stream as a cudaStream_t: FinalDraw of every sample, presents and post-processing run on it in
 * submission order, so an event recorded on it after N idkpt_compute calls completes when those N samples are in the image. */
IDKPT_API int idkpt_stream_handle(IdkPtCtx* ctx, void** stream);

/* Host read-back / restore of an rgba32f image of this context's tile rows in
 * full-image layout (rows not owned by the tile are left untouched). */
IDKPT_API int idkpt_read_result(IdkPtCtx* ctx, IdkPtImage which, void* dst_rgba32f, uint64_t bytes);
IDKPT_API int idkpt_write_result(IdkPtCtx* ctx, IdkPtImage which, const void* src_rgba32f, uint64_t bytes);

/* Asynchronous presentation: snapshot the image (ordered after the Compute that produced it) and copy it to host memory
 * (pinned for full overlap) on a second stream while the next idkpt_compute runs; idkpt_present_wait blocks until the
 * most recent transfer has landed. The GL-free analogue of handing Result to the presenter each frame. */
IDKPT_API int idkpt_present_async(IdkPtCtx* ctx, IdkPtImage which, void* dst_rgba32f_host, uint64_t bytes);
IDKPT_API int idkpt_present_wait(IdkPtCtx* ctx);
/* Page-lock (cudaHostRegister) a host buffer owned by the engine so that idkpt_present_async into it is asynchronous, e.g.
 * ONE frame in POSIX shared memory registered by every rank: each rank's idkpt_present_async(IDKPT_IMAGE_RESULT) then
 * delivers its own stripes to their final position over its own PCIe link (multi-GPU presentation without a root copy). */
IDKPT_API int idkpt_register_host_buffer(IdkPtCtx* ctx, void* host_ptr, uint64_t bytes);
IDKPT_API int idkpt_unregister_host_buffer(IdkPtCtx* ctx, void* host_ptr);

/* Multi-GPU tile gather over NVLink peer memory (no NCCL in the data path). Every rank calls idkpt_gather_export
 * (allocates a double-buffered full-size image + arrival flags + the global-slot table and returns 5 CUDA IPC handles =
 * 320 bytes; 4 handles / 256 bytes before ABI 4), the ranks
 * exchange the handles (torch.distributed, MPI, a socket...) and call idkpt_gather_import with all of them in rank
 * order. From then on the FinalDraw of every idkpt_compute also stores this rank's pixels into every rank's full image
 * at their final position and idkpt_compute returns once all ranks' tiles of that frame have arrived (or fails after
 * IDKPT_GATHER_TIMEOUT_MS, default 30 s, if a peer never delivers). idkpt_resize drops the mappings: export / exchange /
 * import again afterwards.
 * idkpt_gather_connect does the same for a host that drives every GPU from ONE process (like the reference engine): pass
 * the contexts in tile order (context r created with TileIndex r, TileCount world); no IPC, peer access is enabled here.
 * With ONE host thread feeding all contexts only queue work afterwards (idkpt_compute with stats == NULL): a synchronous call
 * would wait for peers whose work has not been submitted yet (and fail after the time-out). Resizing or destroying one
 * context invalidates what its peers hold of it: resize all, then connect again. */
#define IDKPT_GATHER_HANDLE_BYTES 320
IDKPT_API int idkpt_gather_export(IdkPtCtx* ctx, void* handles_out, uint64_t bytes);
IDKPT_API int idkpt_gather_import(IdkPtCtx* ctx, int32_t rank, int32_t world, const void* all_handles, uint64_t bytes);
IDKPT_API int idkpt_gather_connect(IdkPtCtx** ctxs, int32_t world);
IDKPT_API int idkpt_gather_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* Device-side access for zero-copy hand-over (GL interop / NCCL gather):
 * pointer to this tile's compact rgba32f rows (TileRowCount*Width float4). */
IDKPT_API int idkpt_result_device_ptr(IdkPtCtx* ctx, IdkPtImage which, void** dev_ptr, uint64_t* bytes);
IDKPT_API int idkpt_tile_rows(IdkPtCtx* ctx, int32_t* row_count, int32_t* rows_out, int32_t capacity);

/* Export the wavefront state of the last compute() call in the reference's
 * per-pixel layout (GpuWavefrontRay[W*H], SSBO 30) for inspection / parity. */
IDKPT_API int idkpt_read_wavefront_rays(IdkPtCtx* ctx, GpuWavefrontRay* dst, uint64_t count);

/* Stand-alone closest-hit batch with host buffers (H2D + kernel + D2H inside). */
IDKPT_API int idkpt_trace_rays(IdkPtCtx* ctx, const IdkPtRay* rays, uint64_t count, int32_t trace_lights, IdkPtHit* hits_out, float* kernel_ms);

/* ---- "next" rows of the scope table (SURVEY.md 8f.1), built on the same traversal code ----
 * Any-hit (occlusion) batch: TraceRayAny / IntersectBlasAny (BVHIntersect.glsl:107-181,299-411). hits_out[i].NodePairFetches
 * is 1 if the ray is occluded, 0 otherwise; T/TriangleId/Bary describe the first accepted (not the closest) hit. */
IDKPT_API int idkpt_trace_rays_any(IdkPtCtx* ctx, const IdkPtRay* rays, uint64_t count, int32_t trace_lights, IdkPtHit* hits_out, float* kernel_ms);

/* Ray-traced point-light shadows: ShadowsRayTraced/compute.glsl for one light (PointShadowManager.ComputeRayTracedShadowMaps,
 * Source/Render/PointShadowManager.cs:53-75). Host arrays: depth [w*h], octahedral normal rg [w*h*2]; visibility_out [w*h] is
 * read-modify-write (pixels with depth == 1 are left untouched, as the shader returns early). noise_index = the
 * (Frame % SampleCount) * samples term (0 without TAA); taa_jitter may be NULL. idkpt_shadows_ray_traced_gbuffer (below, with
 * the G-buffer passes) runs the same pass on an IdkPtGBuffer into a context image. */
IDKPT_API int idkpt_shadows_ray_traced(IdkPtCtx* ctx, const GpuPerFrameData* frame, const float* depth, const float* normalRG,
                                       int32_t width, int32_t height, int32_t light_index, int32_t samples, uint32_t noise_index,
                                       const float* taa_jitter, float* visibility_out, float* kernel_ms);

/* ---- point-shadow cube maps (PointShadowManager.UpdateBuffer / RenderShadowMaps, CpuPointShadow.RenderShadowMap) ----
 * idkpt_set_point_shadows: the engine's GpuPointShadow array (count <= IDKPT_MAX_POINT_SHADOWS) and the face size of each
 *   shadow's cube map (1..16384). Position, NearPlane (> 0), FarPlane (> NearPlane) and LightIndex are read; LightIndex is
 *   used only by idkpt_volumetric_lighting, which checks it against the scene's light count. The maps are one device
 *   allocation of 6*size^2 uint16 (D16) per shadow, face-major (+X,-X,+Y,-Y,+Z,-Z), row y = t of GL table 8.19, x fastest.
 *   A call whose sizes equal the previous call's keeps the maps; otherwise they are reallocated and every texel is 65535.
 * idkpt_render_point_shadows: shadows [first, first + count). Texel (x, y) of face f stores the D16 depth of the closest
 *   surface along the ray through its centre (GetLogarithmicDepth, Math.glsl:59-66, near/far clipped; 65535 = nothing),
 *   which is what the engine's raster pass stores there. face_masks[i] (bit f = face f, NULL = all six) selects the faces
 *   written for shadow first + i; the other faces keep their texels (the camera-frustum face culling of
 *   CpuPointShadow.RenderShadowMap:125-145 is the host's). Synchronous; kernel_ms may be NULL.
 * idkpt_read_point_shadow copies one shadow's 6*size^2*2 bytes to the host; idkpt_point_shadow_device_ptr hands the device
 *   copy over for interop (valid until the next idkpt_set_point_shadows with other sizes, or idkpt_set_scene).
 * The scene must be set first, and idkpt_set_scene drops the shadows. The maps show the scene as it was at the last render:
 * re-render after idkpt_blas_refit / idkpt_tlas_build, as the engine does every frame. */
#define IDKPT_MAX_POINT_SHADOWS 128   /* GPU_MAX_UBO_POINT_SHADOW_COUNT */
IDKPT_API int idkpt_set_point_shadows(IdkPtCtx* ctx, const GpuPointShadow* shadows, const int32_t* sizes, uint32_t count);
IDKPT_API int idkpt_render_point_shadows(IdkPtCtx* ctx, uint32_t first, uint32_t count, const uint32_t* face_masks, float* kernel_ms);
IDKPT_API int idkpt_read_point_shadow(IdkPtCtx* ctx, int32_t index, uint16_t* dst, uint64_t bytes);
IDKPT_API int idkpt_point_shadow_device_ptr(IdkPtCtx* ctx, int32_t index, void** dev_ptr, uint64_t* bytes);

/* ---- volumetric lighting (VolumetricLighting.Compute: VolumetricLight/compute.glsl + VolumetricLight/Upscale/compute.glsl) ----
 * Ray-marched in-scattering of every point shadow's light through the cube maps of idkpt_set_point_shadows /
 * idkpt_render_point_shadows (NEAREST lookup, no bias), at the render size w = (int)(width * ResolutionScale),
 * h = (int)(height * ResolutionScale), then upscaled to width x height with four depth-weighted bilinear taps.
 * depth: the G-buffer depth [depth_height][depth_width] (host array, sampled NEAREST; idkpt_volumetric_lighting_gbuffer, below
 * with the G-buffer passes, takes it from an IdkPtGBuffer); taa_jitter may be NULL.
 * out_rgba16f: width*height*4 halves (rgba16f, alpha 1), or NULL to keep the image on the device
 * (idkpt_volumetric_device_ptr: valid until the next call with other sizes, idkpt_set_scene or idkpt_destroy).
 * Synchronous; ordered after the samples idkpt_compute has queued. With no shadows set the image is 0.
 * Every shadow's LightIndex must be below the scene's light count. */
typedef struct IdkPtVolumetricSettings {   /* VolumetricLighting.GpuSettings (VolumetricLighting.cs:10-21) + ResolutionScale */
    float   Absorbance[3];                 /* 0.025, 0.025, 0.025 */
    int32_t SampleCount;                   /* 5 (1..1024) */
    float   Scattering;                    /* 0.758: Henyey-Greenstein g */
    float   MaxDist;                       /* 50 */
    float   Strength;                      /* 0.1 */
    float   ResolutionScale;               /* 0.6, in (0, 1] */
} IdkPtVolumetricSettings;
IDKPT_API int idkpt_volumetric_lighting(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtVolumetricSettings* settings, const float* depth,
                                        int32_t depth_width, int32_t depth_height, int32_t width, int32_t height, const float* taa_jitter,
                                        uint16_t* out_rgba16f, float* kernel_ms);
IDKPT_API int idkpt_volumetric_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* ---- G-buffer lighting (RasterPipeline.Render: SSAO.Compute, then the "Deferred Lighting" draw) ----
 * IdkPtGBuffer: the G-buffer attachments as float arrays [Height][Width] in the engine's channel layout. OnDevice = 0: host
 *   arrays, uploaded per call. OnDevice = 1: every pointer is device memory on the context's device and is read in place
 *   (checked with cudaPointerGetAttributes), aligned to the kernels' loads: NormalRG and MetallicRoughness to 8 bytes, the
 *   indirect-light image to 16 bytes, the other arrays to 4 bytes (cudaMalloc'd buffers always are). Any other OnDevice
 *   value, or a pointer that is not device memory or not so aligned, is IDKPT_ERR_INVALID_ARGUMENT, before anything runs.
 *   SSAO reads Depth and NormalRG; deferred lighting reads all five.
 * idkpt_ssao: SSAO/compute.glsl at the G-buffer size into an R8Unorm image (out_r8: Width*Height bytes, or NULL to keep it on
 *   the device: idkpt_ssao_device_ptr).
 * idkpt_deferred_lighting: DeferredLighting/fragment.glsl at the G-buffer size into an rgba32f image (alpha 1; the engine's
 *   beforeTAATexture is R11G11B10F, packing to it is the caller's business). out_rgba32f: Width*Height*4 floats, or NULL to
 *   keep it on the device (idkpt_deferred_device_ptr). taa_jitter may be NULL (0, 0). IsSSAO reads the image of the last
 *   idkpt_ssao call, which must have the G-buffer's size. indirect_rgba32f (IsVXGI; the cone trace's image, [Height][Width]
 *   rgba32f) and the ShadowMode 2 visibility images (rt_visibility[k]: shadow k's float [Height][Width] image, as
 *   idkpt_shadows_ray_traced writes it or idkpt_shadows_device_ptr hands it over; read through the R8Unorm store rule;
 *   idkvx_cone_trace_device_ptr hands over the indirect light) are host or device arrays as gbuffer->OnDevice
 *   says. In ShadowMode 1 and 2 every light's PointShadowIndex must be -1 or below the idkpt_set_point_shadows count, and
 *   ShadowMode 2 needs rt_count >= that count with no NULL entry; ShadowMode 0 ignores the index.
 * Both calls are synchronous and ordered after the samples idkpt_compute has queued. Their images are context allocations,
 * reused by calls with the same size, valid until the next call with another size, idkpt_set_scene or idkpt_destroy. */
typedef struct IdkPtGBuffer {
    int32_t Width;
    int32_t Height;
    int32_t OnDevice;                      /* 0: host arrays, 1: device arrays on the context's device */
    const float* Depth;                    /* D32F: 1 float per pixel */
    const float* NormalRG;                 /* octahedral normal (EncodeUnitVec): 2 floats */
    const float* AlbedoRGB;                /* 3 floats */
    const float* MetallicRoughness;        /* 2 floats */
    const float* EmissiveRGB;              /* 3 floats */
} IdkPtGBuffer;
typedef struct IdkPtSsaoSettings {         /* SSAO.GpuSettings (SSAO.cs:10-15) + the noise index */
    int32_t  SampleCount;                  /* 10 (1..1024) */
    float    Radius;                       /* 0.2 */
    float    Strength;                     /* 1.3 */
    uint32_t NoiseIndex;                   /* (Frame % TAASamples) * SampleCount * 3 with TAA, 0 without */
} IdkPtSsaoSettings;
typedef struct IdkPtDeferredSettings {     /* the deferred lighting program's uniforms (RasterPipeline.cs:454-458) */
    int32_t ShadowMode;                    /* 1: 0 None, 1 Pcf, 2 RayTraced (RasterPipeline.ShadowMode) */
    int32_t IsSSAO;                        /* 1 */
    int32_t IsVXGI;                        /* 0 */
    int32_t IsVariableRateShading;         /* 0 (RasterPipeline.IsVariableRateShading): 1 shades under the rate image of the last
                                              idkpt_shading_rate call, which must have the G-buffer's size (see below) */
} IdkPtDeferredSettings;
IDKPT_API int idkpt_ssao(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtSsaoSettings* settings, const IdkPtGBuffer* gbuffer,
                         uint8_t* out_r8, float* kernel_ms);
IDKPT_API int idkpt_ssao_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);
IDKPT_API int idkpt_deferred_lighting(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtDeferredSettings* settings, const IdkPtGBuffer* gbuffer,
                                      const float* taa_jitter, const float* indirect_rgba32f, const float* const* rt_visibility, uint32_t rt_count,
                                      float* out_rgba32f, float* kernel_ms);
IDKPT_API int idkpt_deferred_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* ---- the deferred pass's other inputs from an IdkPtGBuffer: ray-traced shadows and volumetric light ----
 * Read the G-buffer as idkpt_ssao does (OnDevice 0: host arrays uploaded per call; 1: device arrays read in place, checked and
 * aligned alike), so that a frame whose G-buffer comes from idkpt_gbuffer_device_ptrs never leaves the device. Every argument
 * is checked before anything is uploaded or launched: a rejected call (IDKPT_ERR_INVALID_ARGUMENT) leaves every image as it
 * was. Both calls are synchronous and ordered after the samples idkpt_compute has queued.
 * idkpt_shadows_ray_traced_gbuffer: idkpt_shadows_ray_traced's pass for light light_index (samples 1..1024) over Depth and
 *   NormalRG (the other attachments may be NULL), into the context's float [Height][Width] visibility image of `slot`
 *   (0 <= slot < IDKPT_MAX_POINT_SHADOWS; one per point shadow). Pixels with depth == 1 keep what the image held, as the
 *   shader returns early there: the last successful call's values for the slot if it had the G-buffer's size, else 0 (the
 *   slot's first call, a new size, after a failed call or idkpt_set_scene). The deferred pass returns early on those pixels
 *   too, so it never reads them. visibility_out: Width*Height floats, or NULL to keep the image on the device only.
 * idkpt_shadows_device_ptr: that image of `slot` (Width*Height*4 bytes, 256-byte aligned) for idkpt_deferred_lighting's
 *   rt_visibility[k] with OnDevice = 1; valid until the slot's next call with another size, a failed call for the slot,
 *   idkpt_set_scene or idkpt_destroy. Fails before the slot's first successful call.
 * idkpt_volumetric_lighting_gbuffer: idkpt_volumetric_lighting with the depth gbuffer->Depth [Height][Width] (the other
 *   attachments are not read and may be NULL); same image, same idkpt_volumetric_device_ptr. */
IDKPT_API int idkpt_shadows_ray_traced_gbuffer(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtGBuffer* gbuffer, int32_t light_index,
                                               int32_t samples, uint32_t noise_index, const float* taa_jitter, int32_t slot,
                                               float* visibility_out, float* kernel_ms);
IDKPT_API int idkpt_shadows_device_ptr(IdkPtCtx* ctx, int32_t slot, void** dev_ptr, uint64_t* bytes);
IDKPT_API int idkpt_volumetric_lighting_gbuffer(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtVolumetricSettings* settings,
                                                const IdkPtGBuffer* gbuffer, int32_t width, int32_t height, const float* taa_jitter,
                                                uint16_t* out_rgba16f, float* kernel_ms);

/* ---- the end of the raster frame (RasterPipeline.Render: SSR.Compute, "Merge Textures", TaaResolve.Compute) ----
 * The lit image both calls read (`source`): IDKPT_LIT_SOURCE_ARRAY, a caller rgba32f [Height][Width] array (host or device as
 *   the call's OnDevice says; a host that keeps the light, skybox and transparency draws in GL passes its composited buffer);
 *   IDKPT_LIT_SOURCE_DEFERRED, the context's lit image as the last idkpt_deferred_lighting call left it, composited by any
 *   idkpt_transparency since; IDKPT_LIT_SOURCE_MERGED (TAA only), the
 *   merged image of the last idkpt_ssr call. A context image must exist and have the render size.
 * idkpt_ssr: SSR/compute.glsl at the G-buffer size (reads Depth, NormalRG, AlbedoRGB and MetallicRoughness; EmissiveRGB may be
 *   NULL), then MergeTextures/compute.glsl: merged = source.rgb + SSR.rgb (alpha 1). The sky is the context's (idkpt_set_sky).
 *   merged_out_rgba32f: Width*Height*4 floats; ssr_out_rgba16f: Width*Height*4 halves (alpha 0 where the shader's early out
 *   stores vec4(0), else 1). Either may be NULL to keep that image on the device (idkpt_ssr_device_ptrs).
 * idkpt_taa_resolve: TAAResolve/compute.glsl at the presentation size width x height over the render-size inputs (the sizes
 *   are independent: upscaling TAA). The context keeps two rgba16f presentation-size images and a frame counter (TAAResolve's
 *   ping-pong): each call increments the counter, writes Result and reads PrevResult. Both images are zero-filled whenever
 *   the presentation size changes (and on the first call); idkpt_set_scene drops them. out_rgba16f: width*height*4 halves
 *   (alpha 1), or NULL (idkpt_taa_device_ptr: the image the last call wrote).
 * OnDevice arrays must be device memory on the context's device, aligned to 4 bytes (depth), 8 bytes (velocity and the float2
 * G-buffer attachments) and 16 bytes (colour arrays). Both calls are synchronous and ordered after the samples idkpt_compute
 * has queued. Their images are context allocations, valid until the next call with another size, idkpt_set_scene or
 * idkpt_destroy. */
#define IDKPT_LIT_SOURCE_ARRAY    0
#define IDKPT_LIT_SOURCE_DEFERRED 1
#define IDKPT_LIT_SOURCE_MERGED   2
typedef struct IdkPtSsrSettings {          /* SSR.GpuSettings (SSR.cs:10-19) */
    int32_t SampleCount;                   /* 30 (1..1024) */
    int32_t BinarySearchCount;             /* 8 (0..64) */
    float   MaxDist;                       /* 50 (finite) */
} IdkPtSsrSettings;
typedef struct IdkPtTaaSettings {          /* TAAResolve.GpuSettings (TAAResolve.cs:10-18) + GpuTaaData.SampleCount */
    int32_t IsNaiveTaa;                    /* 0 */
    float   PreferAliasingOverBlur;        /* 0.25 */
    int32_t SampleCount;                   /* 6 (1..1024) */
} IdkPtTaaSettings;
typedef struct IdkPtTaaInputs {            /* the render-size images TAAResolve/compute.glsl samples */
    int32_t Width;                         /* render size */
    int32_t Height;
    int32_t OnDevice;                      /* 0: host arrays, 1: device arrays on the context's device */
    int32_t Source;                        /* IDKPT_LIT_SOURCE_*: the colour */
    const float* Depth;                    /* D32F: 1 float per pixel */
    const float* VelocityRG;               /* 2 floats per pixel (R16G16F in the engine) */
    const float* ColorRgba32f;             /* Source ARRAY: 4 floats per pixel, else ignored */
} IdkPtTaaInputs;
IDKPT_API int idkpt_ssr(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtSsrSettings* settings, const IdkPtGBuffer* gbuffer,
                        int32_t source, const float* color_rgba32f, float* merged_out_rgba32f, uint16_t* ssr_out_rgba16f, float* kernel_ms);
IDKPT_API int idkpt_ssr_device_ptrs(IdkPtCtx* ctx, void** merged_dev_ptr, void** ssr_dev_ptr, uint64_t* merged_bytes, uint64_t* ssr_bytes);
IDKPT_API int idkpt_taa_resolve(IdkPtCtx* ctx, const IdkPtTaaSettings* settings, const IdkPtTaaInputs* inputs, int width, int height,
                                uint16_t* out_rgba16f, float* kernel_ms);
IDKPT_API int idkpt_taa_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* ---- variable-rate deferred lighting (LightingShadingRateClassifier.Compute; the deferred lighting draw under its image) ----
 * idkpt_shading_rate: ShadingRateClassification/compute.glsl over a render-size lit image (Source ARRAY: a caller rgba32f
 *   [Height][Width] array; DEFERRED: the image of the last idkpt_deferred_lighting call, which must have the render size;
 *   MERGED is rejected: the engine classifies the image before SSR) and the velocity (RG float [Height][Width]). Every 16x16
 *   tile gets a palette index of the engine's palette {1x1, 2x1, 2x2, 4x2, 4x4} from its mean speed (/ frame->DeltaRenderTime)
 *   and its luminance's coefficient of variation. out_rates: ceil(Height/16) * ceil(Width/16) bytes, or NULL to keep the
 *   image on the device (idkpt_shading_rate_device_ptr). debug_out_r32f (DebugMode 2 Speed, 3 Luminance, 4 LuminanceVariance):
 *   the mean speed, mean luminance or coefficient of variation per tile, same size; it must be NULL in DebugMode 0 and 1 and
 *   may be NULL in the others. The sums are taken in a pinned order and the rate conversion is pinned too (DESIGN.md 8f.1f).
 * With IdkPtDeferredSettings.IsVariableRateShading = 1, idkpt_deferred_lighting shades each pixel under NV_shading_rate_image's
 *   rules with the context's rate image: the fragment shader runs once per coarse fragment, at its centre, and its result is
 *   written to every pixel of the fragment. The image of frame N's classification drives frame N+1's lighting.
 * OnDevice arrays must be device memory on the context's device, aligned to 8 bytes (velocity) and 16 bytes (colour). The call
 * is synchronous and ordered after the samples idkpt_compute has queued. Its image is a context allocation, valid until the
 * next call with another size, a failed call, idkpt_set_scene or idkpt_destroy. */
typedef struct IdkPtShadingRateSettings {  /* LightingShadingRateClassifier.GpuSettings */
    int32_t DebugMode;                     /* 0: 0 None, 1 ShadingRate, 2 Speed, 3 Luminance, 4 LuminanceVariance */
    float   SpeedFactor;                   /* 0.2 (finite) */
    float   LumVarianceFactor;             /* 0.04 (finite) */
} IdkPtShadingRateSettings;
typedef struct IdkPtShadingRateInputs {    /* the render-size images the classifier reads */
    int32_t Width;
    int32_t Height;
    int32_t OnDevice;                      /* 0: host arrays, 1: device arrays on the context's device */
    int32_t Source;                        /* IDKPT_LIT_SOURCE_ARRAY or _DEFERRED */
    const float* VelocityRG;               /* 2 floats per pixel (R16G16F in the engine) */
    const float* ColorRgba32f;             /* Source ARRAY: 4 floats per pixel, else ignored */
} IdkPtShadingRateInputs;
IDKPT_API int idkpt_shading_rate(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtShadingRateSettings* settings,
                                 const IdkPtShadingRateInputs* inputs, uint8_t* out_rates, float* debug_out_r32f, float* kernel_ms);
IDKPT_API int idkpt_shading_rate_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* ---- the G-buffer pass (RasterPipeline.Render: the "Fill G-Buffer" draws, GBuffer/VertexPath/vertex.glsl + fragment.glsl) ----
 * idkpt_gbuffer: renders the pass at the render size width x height into context images, ray-cast at pixel centres: each pixel
 *   holds the closest surface along the ray through its centre that the pass does not clip (depth outside [0, 1]), cull
 *   (blended materials; back faces of single-sided materials) or discard (alpha test). Six planar fp32 arrays [Height][Width],
 *   each 256-byte aligned: Depth 1 float per pixel, NormalRG 2, AlbedoRGB 3, MetallicRoughness 2, EmissiveRGB 3, VelocityRG 2,
 *   holding exactly what the engine's attachments hold (R11G11B10F albedo and emissive, RG8 normal and metallic/roughness,
 *   RG16F velocity, D32F depth); pixels without a surface hold the clears (depth 1, everything else 0). The rules are in
 *   DESIGN.md 8f.1g. taa_jitter: taaDataUBO.Jitter in NDC units, NULL = (0, 0). prev_positions: the previous frame's vertex
 *   positions (prevVertexPositionSSBO, VertexPositionCount entries): idkpt_prev_positions_device_ptr's pointer, read in place
 *   (what idkpt_skin_vertices keeps, so an animated frame uploads nothing), any other pointer a host array, NULL = this
 *   frame's (static geometry). Lights and the skybox are separate draws: idkpt_lights_and_skybox draws them into these
 *   images afterwards.
 * idkpt_gbuffer_device_ptrs: the images of the last successful call: an IdkPtGBuffer with OnDevice = 1 that idkpt_ssao,
 *   idkpt_deferred_lighting and idkpt_ssr take as it is, and the velocity for IdkPtTaaInputs / IdkPtShadingRateInputs.
 *   Either output may be NULL.
 * idkpt_read_gbuffer: downloads the images of the last successful call; any argument may be NULL.
 * idkpt_prev_positions_device_ptr: the context's previous positions (PackedVec3 [VertexPositionCount], *bytes their size), as
 *   idkpt_skin_vertices keeps them. Created at the first idkpt_skin_vertices or idkpt_prev_positions_device_ptr after
 *   idkpt_set_scene or idkpt_add_models as a copy of the positions at that moment; valid until idkpt_set_scene,
 *   idkpt_add_models or idkpt_destroy. Needs a scene.
 * The call is synchronous and ordered after the samples idkpt_compute has queued. Its images are context allocations, reused
 * by calls with the same size, valid until the next call with another size, a failed call, idkpt_set_scene or idkpt_destroy. */
IDKPT_API int idkpt_gbuffer(IdkPtCtx* ctx, const GpuPerFrameData* frame, int32_t width, int32_t height, const float* taa_jitter,
                            const PackedVec3* prev_positions, float* kernel_ms);
IDKPT_API int idkpt_gbuffer_device_ptrs(IdkPtCtx* ctx, IdkPtGBuffer* gbuffer_out, const float** velocity_rg_out);
IDKPT_API int idkpt_read_gbuffer(IdkPtCtx* ctx, float* depth, float* normal_rg, float* albedo_rgb, float* metallic_roughness,
                                 float* emissive_rgb, float* velocity_rg);
IDKPT_API int idkpt_prev_positions_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* ---- transparency (RasterPipeline.Render: "Record transparent fragments" + "Resolve transparent fragments") ----
 * idkpt_transparency: the blended surfaces (AlphaCutoff == 2) the G-buffer pass culls, ray-cast at pixel centres along
 *   idkpt_gbuffer's rays and composited front to back over the lit image, in place. A fragment is kept where its material is
 *   blended, it is front-facing or double-sided, its depth is in [0, 1] and below gbuffer->Depth, and its alpha is not 0;
 *   per pixel the 10 (TRANSPARENT_LAYERS) with the smallest depth are kept, ties broken by BLAS triangle, then
 *   MeshTransformId. Each is lit as the record shader lights it: every light through GGX with the surface's IOR, shadowed by
 *   the PCF filter (ShadowMode 1; ShadowMode 2 leaves transparents unshadowed, as the engine does), plus VXGI indirect light
 *   traced from `voxels` with the context's sky (IsVXGI) or 0.015 * albedo; premultiplied and rounded to rgba16f. The result
 *   is acc.rgb of ResolveTransparent's blend with alpha 1; a pixel without a layer keeps its bytes. The rules are in DESIGN.md
 *   8f.1h.
 * gbuffer: Width, Height, OnDevice and Depth are read; the other attachments may be NULL. source: IDKPT_LIT_SOURCE_DEFERRED
 *   composites the context's deferred image (later DEFERRED reads see it); IDKPT_LIT_SOURCE_ARRAY composites color_rgba32f
 *   (host or device as OnDevice says; a host array is uploaded and downloaded back into itself); MERGED is rejected (the engine
 *   resolves before SSR). out_rgba32f: an optional download of the result (Width*Height*4 floats). taa_jitter: NULL = (0, 0).
 *   voxels / cone: IsVXGI only; the grid must be voxelised, on the context's device. Every argument is checked before anything
 *   is uploaded or launched, so a failed call leaves the target unchanged. The call is synchronous and ordered after the
 *   samples idkpt_compute has queued. */
struct IdkVxCtx;
struct IdkVxConeSettings;
typedef struct IdkPtTransparencySettings { /* the record program's uniforms (RasterPipeline.cs:555-558) */
    int32_t ShadowMode;                    /* 1: 0 None, 1 Pcf, 2 RayTraced (no shadow on transparents, as in the engine) */
    int32_t IsVXGI;                        /* 0 */
} IdkPtTransparencySettings;
IDKPT_API int idkpt_transparency(IdkPtCtx* ctx, const GpuPerFrameData* frame, const IdkPtTransparencySettings* settings,
                                 const IdkPtGBuffer* gbuffer, const float* taa_jitter, struct IdkVxCtx* voxels,
                                 const struct IdkVxConeSettings* cone, int32_t source, float* color_rgba32f, float* out_rgba32f,
                                 float* kernel_ms);

/* ---- the light spheres and the skybox (RasterPipeline.Render: "Draw lights" + "Draw skybox") ----
 * idkpt_lights_and_skybox: the two draws the engine runs between deferred lighting and transparency, ray-cast at pixel centres
 *   along idkpt_gbuffer's rays and written in place into the context's images: the G-buffer of the last successful
 *   idkpt_gbuffer (Depth, NormalRG, EmissiveRGB, VelocityRG) and the deferred image of idkpt_deferred_lighting, which must have
 *   the G-buffer's size. So later DEFERRED reads, idkpt_gbuffer_device_ptrs and idkpt_read_gbuffer see the result.
 *   Lights: each scene light is LightManager's 12 x 12 sphere mesh scaled by Radius at Position, depth-tested LESS against the
 *   G-buffer depth with back faces culled; the nearest fragment wins, ties keep the first in draw order (light, then triangle).
 *   It writes the light's Color to the lit image (alpha 1) and to EmissiveRGB, the encoded sphere normal, the velocity
 *   against PrevPosition and PrevProjView, and its depth. A camera inside a sphere sees none of it.
 *   Skybox: every pixel whose depth is still 1 gets the context's sky (idkpt_set_sky) seen through the unjittered pixel
 *   centre (alpha 1) and the rotation-only velocity between View and PrevView; its depth stays 1.
 *   AlbedoRGB and MetallicRoughness are never written. The rules are in DESIGN.md 8f.1i.
 * taa_jitter: NULL = (0, 0). out_rgba32f: an optional download of the lit image (Width*Height*4 floats). Every argument is
 * checked before anything is launched, so a failed call changes no byte. A second call with the same arguments changes nothing.
 * The call is synchronous and ordered after the samples idkpt_compute has queued. */
IDKPT_API int idkpt_lights_and_skybox(IdkPtCtx* ctx, const GpuPerFrameData* frame, const float* taa_jitter, float* out_rgba32f,
                                      float* kernel_ms);

/* ---- dynamic geometry (SURVEY.md 8f.2): ModelManager.Update = skin -> refit -> TLAS (ModelManager.cs:236-261) ----
 * idkpt_set_skinning_data: unskinnedVertexSSBO upload (52-byte GpuUnskinnedVertex records).
 * idkpt_skin_vertices: uploads the joint matrices (row-major mat4x3 = 3 x vec4 each, ModelManager.cs:272-277) and runs
 *   Skinning/compute.glsl once per command; positions, normals and tangents are rewritten in place on the device. Before
 *   each command skins its output range, the call copies that range of the positions into the context's previous positions
 *   (Skinning/compute.glsl:42, idkpt_prev_positions_device_ptr), so overlapping commands keep what the earlier command
 *   left. Every argument is checked first: a rejected call changes neither. kernel_ms covers the copies and the kernels.
 * idkpt_blas_refit: BVH.GpuBlasesRefit(first, count) (BVH.cs:472-489, BLASRefit/compute.glsl); also refreshes the derived
 *   triangle records of the refitted BLASes. Call it for every BLAS whose vertices moved.
 * idkpt_read_range: device -> host read-back (refitted BLAS nodes for the host TLAS build, skinned vertices, and after
 *   idkpt_blas_rebuild the BLAS nodes, triangles and descs for the host's CPU copy).
 * All of them reset the accumulation like any other scene edit. */
typedef struct IdkPtSkinningCmd {     /* ModelManager.SkinningCmd, Skinning/compute.glsl:9-12 uniforms */
    uint32_t InputVertexOffset;
    uint32_t OutputVertexOffset;
    uint32_t JointMatricesOffset;
    uint32_t VertexCount;
} IdkPtSkinningCmd;

IDKPT_API int idkpt_set_skinning_data(IdkPtCtx* ctx, const GpuUnskinnedVertex* vertices, uint64_t count);
IDKPT_API int idkpt_skin_vertices(IdkPtCtx* ctx, const float* joint_matrices, uint64_t joint_count, const IdkPtSkinningCmd* cmds, uint32_t cmd_count, float* kernel_ms);
IDKPT_API int idkpt_blas_refit(IdkPtCtx* ctx, uint32_t first_blas, uint32_t count, float* kernel_ms);
IDKPT_API int idkpt_read_range(IdkPtCtx* ctx, IdkPtArrayId which, uint64_t first, uint64_t count, void* out);
/* BVH.TlasBuild() on the device (BVH.cs:278-298 + TLAS.Build, TLAS.cs:28-141, serial PLOC with TLAS.BuildSettings.SearchRadius = 15):
 * world bounds of every instance from the (refitted) BLAS roots and the current mesh transforms, both already in HBM; fills the
 * scene's TLAS node array (UseTlas scenes) with exactly the nodes the host build produces -- a moving scene reads nothing back.
 * Any instance count the node format holds (31-bit child and instance ids: 2n - 1 < 2^31; above, IDKPT_ERR_UNSUPPORTED). Up
 * to 64 instances one CTA builds the tree; above, the build is spread over the GPU. search_radius: 1..1024.
 * The TLAS walk's stack has 24 entries (BVHIntersect.glsl:4), so a tree deeper than 24 is refused with IDKPT_ERR_UNSUPPORTED
 * and invalidates the scene (set it again). Large scenes can reach that depth: the radius-15 tree of 262144 uniformly
 * scattered boxes is 25 deep, of 1 M boxes in 64 clusters 35. Identical boxes make a chain and are refused after 25 PLOC
 * iterations, not after n. An instance box that is not finite (a NaN or infinite ModelMatrix or BLAS root) stops the build
 * with IDKPT_ERR_INVALID_ARGUMENT and also invalidates the scene. */
IDKPT_API int idkpt_tlas_build(IdkPtCtx* ctx, int32_t search_radius, float* kernel_ms);

/* BLAS.Build + PreSplitting.PreSplit on the device (the loop body of BVH.BlasesBuild, BVH.cs:315-377): the SweepSAH build of
 * one BLAS with early split clipping, node for node and triangle for triangle equal to the host build (idkhost_blas_build),
 * with the same required stack size, fragment count and SAH bits. Host arrays in and out, like the host build: the engine
 * keeps a CPU copy of every BLAS for BVH.Intersect and hands the arrays to idkpt_set_scene. Needs no scene and leaves the
 * context's scene, sky and accumulation alone; synchronous, ordered after queued idkpt_compute samples.
 * IDKPT_ERR_INVALID_ARGUMENT: a NULL pointer, no triangles, a vertex id >= vertex_count, a non-finite setting, or
 * StopSplittingThreshold < 1. IDKPT_ERR_UNSUPPORTED: more than 2^24 fragments after pre-splitting (the host's float
 * counters saturate there). kernel_ms (may be NULL): device time of the whole build, copies included. */
typedef struct IdkPtBlasBuildSettings {      /* BLAS.BuildSettings + PreSplitting.Settings; = IdkBlasBuildSettings without Threads */
    int32_t StopSplittingThreshold;          /* 1 */
    int32_t MaxLeafTriangleCount;            /* 2 */
    float   TriangleCost;                    /* 1.1 */
    int32_t StackOptThreshold;               /* 16 */
    float   StackOptSahIncreaseAcceptance;   /* 0.0009745 */
    float   SplitFactor;                     /* 0.3 */
    int32_t DoPreSplit;                      /* 1 (= !IsRefittable) */
} IdkPtBlasBuildSettings;
typedef struct IdkPtBlasBuild IdkPtBlasBuild;
IDKPT_API int idkpt_blas_build(IdkPtCtx* ctx, const PackedVec3* positions, uint64_t vertex_count,
                               const GpuBlasTriangle* triangles, uint64_t triangle_count,
                               const IdkPtBlasBuildSettings* settings /* NULL = defaults */,
                               IdkPtBlasBuild** out, float* kernel_ms);
IDKPT_API int  idkpt_blas_build_info(const IdkPtBlasBuild* b, uint64_t* node_count, uint64_t* triangle_count,
                                     int32_t* required_stack_size, int32_t* fragment_count, double* sah);
/* nodes: node_count GpuBlasNode (node 0 the pad, node 1 the root); triangles: triangle_count GpuBlasTriangle */
IDKPT_API int  idkpt_blas_build_copy(const IdkPtBlasBuild* b, GpuBlasNode* nodes, GpuBlasTriangle* triangles);
IDKPT_API void idkpt_blas_build_free(IdkPtBlasBuild* b);

/* BVH.BlasesBuild's parallel loop (BVH.cs:315-377) in one call: builds every BLAS of `descs` -- a model load's or a rebuild's --
 * together on the device, each node for node and triangle for triangle equal to building it alone with idkpt_blas_build (and
 * so to the host build), with the same required stack size, fragment count and SAH bits. Per desc only TriangleOffset,
 * TriangleCount and IsRefittable are read: the BLAS's triangles are triangles[TriangleOffset, +TriangleCount), anywhere in
 * the array, and it is pre-split exactly when !IsRefittable (BVH.cs:325); the settings' DoPreSplit is ignored. The batch
 * pays for its launches and host synchronisations once, not once per BLAS, which is what makes a load of many small BLASes
 * fast. Needs no scene and leaves the context's scene, sky and accumulation alone; synchronous, ordered after queued
 * idkpt_compute samples.
 * The handle works with idkpt_blas_build_info (totals: nodes, triangles, the largest RequiredStackSize as
 * BVH.UpdateBlasStackSize takes it, fragments, and the BLASes' SAHs added in desc order as BVH.cs:460-468 logs them),
 * idkpt_blas_build_copy (the BLASes' nodes and triangles one after another) and idkpt_blas_build_batch_copy.
 * IDKPT_ERR_INVALID_ARGUMENT, before anything runs and with *out NULL: a NULL pointer, desc_count == 0, a desc without
 * triangles or with a range outside `triangles`, a vertex id >= vertex_count in any BLAS, a non-finite setting, or
 * StopSplittingThreshold < 1. IDKPT_ERR_UNSUPPORTED: more than 2^24 fragments in one BLAS after pre-splitting, or a batch
 * whose node ids (the sum of max(2 * fragments, 4) over its BLASes) reach 2^31; both are found before any fragment is
 * written. kernel_ms (may be NULL): device time of the whole batch, copies included. */
IDKPT_API int idkpt_blas_build_batch(IdkPtCtx* ctx, const PackedVec3* positions, uint64_t vertex_count,
                                     const GpuBlasTriangle* triangles, uint64_t triangle_count,
                                     const GpuBlasDesc* descs, uint32_t desc_count,
                                     const IdkPtBlasBuildSettings* settings /* NULL = defaults; DoPreSplit ignored */,
                                     IdkPtBlasBuild** out, float* kernel_ms);
/* Per BLAS of a batch (desc_count entries each): its desc as BVH.cs:363-386 fills it (NodeOffset and TriangleOffset from 0
 * over the copied arrays, NodeCount, TriangleCount and RequiredStackSize from the build, the other fields as handed in), its
 * fragment count and its SAH. nodes and triangles as idkpt_blas_build_copy. Any output pointer may be NULL. */
IDKPT_API int idkpt_blas_build_batch_copy(const IdkPtBlasBuild* b, GpuBlasDesc* descs, GpuBlasNode* nodes,
                                          GpuBlasTriangle* triangles, int32_t* fragment_counts, double* sahs);

/* BVH.BlasesBuild(first, count) (BVH.cs:300-470) on the scene in place: rebuilds BLASes [first, first + count) from the scene's
 * current device arrays -- each BLAS's triangle records BlasTriangles[TriangleOffset, +TriangleCount) and the device vertex
 * positions, including whatever idkpt_skin_vertices last wrote -- with the same builder as idkpt_blas_build. Nothing is uploaded.
 * A BLAS is pre-split exactly when !IsRefittable (BVH.cs:325); the settings' DoPreSplit is ignored, the other fields mean what
 * they mean for idkpt_blas_build. A pre-split BLAS is pre-split again from its current, already duplicated triangle list, as
 * the engine does, so its triangle count can grow with every rebuild.
 * The new nodes and triangles replace the old ones: NodeOffset and TriangleOffset of every desc from `first` to the end become
 * the previous desc's end and the data behind them moves along; the rebuilt descs get the new NodeCount, TriangleCount and
 * RequiredStackSize, and keep IsRefittable and the LeafIndices / ParentIndices fields the host handed over. BlasStackSize
 * becomes the largest RequiredStackSize (BVH.UpdateBlasStackSize). Everything else -- instances, transforms, meshes,
 * materials, textures, lights, sky, point-shadow maps, kept previous positions, raster images, TAA history -- stays. The TLAS
 * is not rebuilt, as after idkpt_blas_refit: call idkpt_tlas_build (or upload TLAS nodes) next. Resets the accumulation.
 * All or nothing: the BLASes are built as one batch (as idkpt_blas_build_batch builds them) into staging memory and committed
 * only when the whole batch succeeded; a failed call leaves every scene array, desc, the stack size and the image as they were. Synchronous, ordered after queued idkpt_compute samples.
 * IDKPT_ERR_INVALID_ARGUMENT: a NULL context, first + count past the descs, a non-finite setting, StopSplittingThreshold < 1,
 * or a layout other than the one BlasesBuild and host.Scene.add produce (from `first` on each desc's nodes and triangles
 * start where the previous desc's end and the last desc ends both arrays; the descs before `first` end at or before the end
 * of desc first - 1). IDKPT_ERR_UNSUPPORTED: more than 2^24 fragments in one build, or a new BlasStackSize beyond the
 * shared-memory traversal stack (the limit idkpt_set_scene applies). count == 0 does nothing. kernel_ms (may be NULL): device
 * time of the builds and the commit's copies. */
IDKPT_API int idkpt_blas_rebuild(IdkPtCtx* ctx, uint32_t first, uint32_t count, const IdkPtBlasBuildSettings* settings /* NULL = defaults */,
                                 float* kernel_ms);
/* BLAS.ComputeGlobalSAH (BLAS.cs:629-656) of BLASes [first, first + count) as the device holds them now (built, refitted or
 * rebuilt): the engine's pre-order walk, left child first, with the double sum in that order. Equals the build's sah for a
 * BLAS the builder just produced. Only settings->TriangleCost is read (NULL = 1.1). sah_out: count doubles. A host refits most
 * frames and rebuilds (idkpt_blas_rebuild) when the SAH has drifted far enough from the built one. */
IDKPT_API int idkpt_blas_sah(IdkPtCtx* ctx, uint32_t first, uint32_t count, const IdkPtBlasBuildSettings* settings, double* sah_out);

/* ModelManager.Add(models) (ModelManager.cs:128-216) on the scene in place: appends the call's arrays behind the scene's,
 * builds the new BLASes on the device and, for a scene set with UseTlas, rebuilds the TLAS. Loading a model costs what the
 * model costs: nothing already on the device crosses PCIe again, no texture is decoded again, and nothing the renderer keeps
 * between frames is dropped. Every id is local to this call's arrays; several models are concatenated by the caller, as
 * ModelManager.Add(params models) does.
 * Append order and offsets: the call's arrays go behind the scene's, in order, with the scene's old counts added:
 *   GpuBlasTriangle X/Y/Z + old VertexCount, MeshId + old MeshCount; GpuMesh.MaterialId + old MaterialCount; a material
 *   texture handle k > 0 + old TextureCount (0, the white fallback, stays 0); GpuBlasInstance.BlasId + old BlasDescCount,
 *   MeshTransformId + old MeshTransformCount. Every other field (GpuMesh.MeshletsOffset and the like) is copied as given.
 * BLASes: built as one idkpt_blas_build_batch batch over the rebased triangles, each pre-split exactly when !IsRefittable
 *   (settings->DoPreSplit is ignored), so each equals idkpt_blas_build_batch's and the host build's node for node. Their
 *   descs are filled as BVH.cs:363-386 fills them: NodeOffset and TriangleOffset behind the scene's current ends, NodeCount,
 *   TriangleCount and RequiredStackSize from the build, every other field as handed in. BlasStackSize becomes the largest
 *   RequiredStackSize of all descs (BVH.UpdateBlasStackSize).
 * TLAS: with UseTlas the node array grows to 2n - 1 nodes and is rebuilt over every instance by idkpt_tlas_build's PLOC build
 *   with search radius 15 (BVH.TlasBuild(true) in ModelManager.Add). A scene without UseTlas stays without it.
 * Kept as they are: lights, sky, point-shadow maps and records, every raster image (G-buffer, SSAO, deferred, shadow
 *   visibility slots, volumetric, SSR, shading rate), the TAA history and its frame counter, the existing texture records;
 *   their *_device_ptr exports stay valid. The kept previous positions are released, so that they equal the current
 *   positions of every vertex, old and new (ModelManager.cs:620); a pointer idkpt_prev_positions_device_ptr returned before is
 *   no longer valid. UnskinnedVertices are appended behind idkpt_set_skinning_data's; the skinning commands stay the host's.
 * The call bumps the scene generation (a voxeliser bound with idkvx_set_scene_from re-sizes its work queue at its next
 * voxelisation), resets the accumulation, and is synchronous and ordered after queued idkpt_compute samples.
 * All or nothing: every check runs on the host over the call's arrays only, before anything runs on the device. The grown
 * arrays, the BLASes and the TLAS are built into staging memory (old and new arrays exist together until the commit) and
 * swapped in only when all of it succeeded; a failed call leaves every array, count, desc, image, exported pointer and the
 * accumulation as they were. A call whose counts are all 0 does nothing and returns IDKPT_OK.
 * IDKPT_ERR_NO_SCENE: no scene. IDKPT_ERR_INVALID_ARGUMENT: a NULL pointer with a count, an id outside its call-local range,
 * an instance world box under UseTlas that is not finite (see idkpt_tlas_build),
 * a desc without triangles or with a range outside Triangles, a non-finite setting, StopSplittingThreshold < 1, a scene whose
 * VertexCount and VertexPositionCount differ, or 2^31 or more nodes, triangles, vertices, meshes, materials, descs,
 * transforms or instances in total. IDKPT_ERR_UNSUPPORTED: a texture format the decoder lacks, more than 2^24 fragments in
 * one BLAS, a BlasStackSize beyond the shared-memory traversal stack, or with UseTlas more than 2^30 instances (31-bit TLAS
 * node ids) or a TLAS deeper than 24 entries (see idkpt_tlas_build). kernel_ms (may be NULL): device time of the whole call. */
typedef struct IdkPtAddModelsDesc {
    const GpuBlasTriangle*    Triangles;         uint64_t TriangleCount;        /* BVH.Add's source triangles: X/Y/Z index this call's vertices, MeshId its meshes */
    const GpuBlasDesc*        BlasDescs;         uint64_t BlasDescCount;        /* per new BLAS: TriangleOffset/TriangleCount into Triangles, IsRefittable */
    const GpuBlasInstance*    BlasInstances;     uint64_t BlasInstanceCount;    /* BlasId into BlasDescs, MeshTransformId into MeshTransforms */
    const GpuMeshTransform*   MeshTransforms;    uint64_t MeshTransformCount;
    const GpuMesh*            Meshes;            uint64_t MeshCount;            /* MaterialId into Materials */
    const GpuMaterial*        Materials;         uint64_t MaterialCount;        /* texture handle 0 = white fallback, k > 0 = Textures[k-1] */
    const GpuVertex*          Vertices;
    const PackedVec3*         VertexPositions;   uint64_t VertexCount;          /* both arrays VertexCount long */
    const IdkPtTextureDesc*   Textures;          uint64_t TextureCount;         /* may be NULL/0 */
    const GpuUnskinnedVertex* UnskinnedVertices; uint64_t UnskinnedVertexCount; /* may be NULL/0 */
} IdkPtAddModelsDesc;
IDK_STATIC_ASSERT(sizeof(IdkPtAddModelsDesc) == 152, "IdkPtAddModelsDesc must be 152 bytes");
IDKPT_API int idkpt_add_models(IdkPtCtx* ctx, const IdkPtAddModelsDesc* models,
                               const IdkPtBlasBuildSettings* settings /* NULL = defaults; DoPreSplit ignored */, float* kernel_ms);

/* ---- present chain (SURVEY.md 8f.3): Bloom.Compute(Result) + TonemapAndGamma.Compute(Result, Bloom.Result)
 * (Application.cs:217-223) -> the RGBA8 frame the reference copies to the swapchain, produced on the device. ---- */
typedef struct IdkPtPostSettings {
    float   Exposure;                    /* TonemapAndGammaCorrect.GpuSettings (TonemapAndGammaCorrecter.cs:10-22): 0.45 */
    float   Saturation;                  /* 1.06 */
    float   Linear;                      /* 0.18 */
    float   Peak;                        /* 1.0 */
    float   Compression;                 /* 0.1 */
    int32_t DoTonemapAndSrgbTransform;   /* 1 */
    int32_t IsBloom;                     /* Application.IsBloom, default 1 */
    float   BloomThreshold;              /* Bloom.GpuSettings (Bloom.cs:10-19): 1.5 */
    float   BloomMaxColor;               /* 3.8 */
    int32_t BloomMinusLods;              /* Bloom.MinusLods, default 3 */
} IdkPtPostSettings;

/* source: IDKPT_IMAGE_RESULT/ALBEDO/NORMAL of an untiled context, or IDKPT_IMAGE_GATHERED (full multi-GPU frame).
 * rgba8_out: host buffer of width*height*4 bytes (row-major, R8G8B8A8Unorm), or NULL to keep the frame on the device
 * (idkpt_ldr_device_ptr). */
IDKPT_API int idkpt_post_process(IdkPtCtx* ctx, const IdkPtPostSettings* settings, IdkPtImage source, uint8_t* rgba8_out, float* kernel_ms);
IDKPT_API int idkpt_ldr_device_ptr(IdkPtCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* ---- denoise hand-off (SURVEY.md 8f.3): PathTracerPipeline.Denoise (PathTracerPipeline.cs:165-194) without the host round trip.
 * idkpt_denoise packs Result / AlbedoTexture / NormalTexture into OIDN-layout buffers on the device (packed RGB floats,
 * Format.Float3: what Texture.Download(PixelFormat.RGB, Float) fills today) and runs the built-in guided a-trous filter into
 * the denoised image (IDKPT_IMAGE_DENOISED: idkpt_read_result, idkpt_post_process source) and into the OIDN output buffer.
 * A host that links OIDN's CUDA device wraps the four pointers of idkpt_denoise_device_ptrs with oidnNewSharedBuffer, calls
 * idkpt_denoise with Iterations = 0 (pack only), executes its filters, and then idkpt_denoise_import_output takes the
 * output buffer over as the denoised image -- nothing crosses PCIe. Needs OutputAOVs samples in the AOV images. ---- */
typedef struct IdkPtDenoiseSettings {
    int32_t Iterations;      /* a-trous passes (step 1, 2, 4, ...); 5 = default; 0 = only pack the OIDN buffers */
    float   SigmaColor;      /* 3.0: colour edge-stopping on the (demodulated) radiance, halved every pass */
    float   SigmaNormal;     /* 0.35 */
    float   SigmaAlbedo;     /* 0.25 */
    int32_t Demodulate;      /* 1: filter colour / max(albedo, 1e-3) and re-apply the albedo afterwards */
} IdkPtDenoiseSettings;
IDKPT_API int idkpt_denoise(IdkPtCtx* ctx, const IdkPtDenoiseSettings* settings, float* kernel_ms);
IDKPT_API int idkpt_denoise_device_ptrs(IdkPtCtx* ctx, void** beauty, void** albedo, void** normal, void** output, uint64_t* bytes_each);
IDKPT_API int idkpt_denoise_import_output(IdkPtCtx* ctx);

IDKPT_API uint32_t idkpt_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* IDKPT_H */
