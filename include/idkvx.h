/*
 * idkvx.h -- C ABI of the VXGI passes of libidkpt: voxelise, mipmap and cone-trace GI as sm_90a kernels over a
 * linear 3D rgba16f grid in HBM (BASELINE.json configs[4]).
 *
 * Replaces (reference paths relative to IDKEngine/):
 *   Source/Render/VXGI/Voxelizer/Voxelizer.cs:109-228   Voxelizer.Render = ClearTextures + Voxelize (+Merge) + Mipmap
 *   Source/Render/VXGI/ConeTracing/ConeTracer.cs:37-50  ConeTracer.Compute
 *   Resource/Shaders/VXGI/Voxelize/{Clear,Voxelize,MergeIntermediates,Mipmap}, VXGI/ConeTraceGI (all files), include/TraceCone.glsl
 * Call sites in the engine: RasterPipeline.Render (Source/Render/RasterPipeline.cs:306-327,436-439).
 *
 * The reference voxelises with the GL rasteriser (one draw per dominant axis via NV passthrough geometry shader +
 * viewport swizzle, Voxelize/geometry.glsl); this library rasterises the same projection in a compute kernel
 * (pixel-centre coverage, DESIGN.md section 8), which matches GL to tolerance and its own CPU oracle bit for bit.
 * Same conventions as idkpt.h: status codes, idkvx_last_error, borrowed host arrays, no CPU fallback.
 */
#ifndef IDKVX_H
#define IDKVX_H

#include "idkpt.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct IdkVxCtx IdkVxCtx;

/* new Voxelizer(width, height, depth, gridMin, gridMax) -- Voxelizer.cs:57-107; defaults 256^3 over
 * [-28,-3,-17]..[28,20,17] (RasterPipeline.cs:213). */
typedef struct IdkVxCreateInfo {
    int32_t Device;
    int32_t Width, Height, Depth;
    float   GridMin[3];
    float   GridMax[3];
} IdkVxCreateInfo;

/* ConeTraceGISettings (VXGI/ConeTraceGI/include/Impl.glsl:7-15) with ConeTracer.cs:10-22 defaults
 * {4, 0.16, 1.3, 1/1.3, 1.0, true}; NoiseIndex = the (Frame % SampleCount) * MaxSamples term of Impl.glsl:37
 * (0 when temporal accumulation / TAA is off). */
typedef struct IdkVxConeSettings {
    int32_t MaxSamples;
    float   StepMultiplier;
    float   GIBoost;
    float   GISkyBoxBoost;
    float   NormalRayOffset;
    uint32_t NoiseIndex;
} IdkVxConeSettings;

typedef struct IdkVxStats {
    float ClearMs, VoxelizeMs, MipmapMs, ConeTraceMs;
    uint64_t Fragments;      /* pixel-centre samples that wrote a voxel */
    uint64_t ConeSteps;      /* texture sample steps of the cone trace  */
    uint32_t KernelLaunches;
    uint32_t _pad0;
} IdkVxStats;

IDKPT_API int idkvx_create(const IdkVxCreateInfo* ci, IdkVxCtx** out);
IDKPT_API void idkvx_destroy(IdkVxCtx* ctx);
IDKPT_API const char* idkvx_last_error(IdkVxCtx* ctx);

/* Geometry + materials + lights of the scene (same arrays as idkpt_set_scene; the BVH members are used only for the
 * triangle list and the instance -> transform map). */
IDKPT_API int idkvx_set_scene(IdkVxCtx* ctx, const IdkPtSceneDesc* scene);
IDKPT_API int idkvx_set_grid(IdkVxCtx* ctx, const float gridMin[3], const float gridMax[3]);   /* Voxelizer.GridMin/GridMax, Voxelizer.cs:16-33 */
IDKPT_API int32_t idkvx_level_count(IdkVxCtx* ctx);                                           /* Texture.GetMaxMipmapLevel */

/* Voxelizer.Render(): clear + voxelise + mip chain. */
IDKPT_API int idkvx_voxelize(IdkVxCtx* ctx, IdkVxStats* stats);

/* rgba16f texels of one mip level, x fastest (size = w*h*d*8 bytes). */
/* Lights with PointShadowIndex >= 0 are attenuated by Visibility() in the fragment stage (Voxelize/fragment.glsl:55-58,100-115),
 * a PCF lookup into the shadow cube map the rasteriser renders (PointShadowManager). Without a rasteriser the voxeliser asks the
 * same question with an any-hit shadow ray from the 2 %-biased sample point to the light through the BVH of a path-tracer
 * context holding the same scene on the same device (hard shadows instead of the PCF-filtered lookup). NULL detaches.
 * A scene with such lights cannot be voxelised without it (IDKPT_ERR_UNSUPPORTED). */
struct IdkPtCtx;
IDKPT_API int idkvx_set_shadow_tracer(IdkVxCtx* ctx, struct IdkPtCtx* path_tracer);
IDKPT_API int idkvx_read_level(IdkVxCtx* ctx, int32_t level, void* dst_rgba16f, uint64_t bytes);

/* ConeTracer.Compute(): per pixel of a width x height G-buffer (host arrays: depth [w*h], normal = octahedral rg
 * [w*h*2], metallicRoughness = rg [w*h*2]) -> rgba32f indirect light [w*h*4]. skyColor = constant sky albedo. */
IDKPT_API int idkvx_cone_trace(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* settings,
                               const float* depth, const float* normalRG, const float* metallicRoughness,
                               int32_t width, int32_t height, const float skyColor[3], float* out_rgba32f, IdkVxStats* stats);

/* ---- multi-GPU (SURVEY.md 8e): voxelise by z-slab, all-gather, cone-trace screen tiles ----
 * Rank r of N: idkvx_set_slab(r * D / N, (r + 1) * D / N), idkvx_voxelize (writes only that slab of level 0, no mip chain),
 * one all-gather of the slabs straight into the grid (a z-slab of the linear x-fastest level is one contiguous range:
 * idkvx_level_device_ptr(0) + z0 * W * H * 8; with equal slabs an in-place ncclAllGather), idkvx_mipmap on every rank, then
 * idkvx_cone_trace_rows over the rank's rows of the G-buffer. The merge is max per channel, so the gathered grid equals the
 * single-GPU grid bit for bit. idkvx_set_slab(0, D) returns to the single-GPU behaviour. */
IDKPT_API int idkvx_set_slab(IdkVxCtx* ctx, int32_t z0, int32_t z1);
IDKPT_API int idkvx_level_device_ptr(IdkVxCtx* ctx, int32_t level, void** dev_ptr, uint64_t* bytes);
IDKPT_API int idkvx_mipmap(IdkVxCtx* ctx, IdkVxStats* stats);
IDKPT_API int idkvx_cone_trace_rows(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* settings,
                                    const float* depth, const float* normalRG, const float* metallicRoughness,
                                    int32_t width, int32_t full_height, int32_t row_first, int32_t row_count,
                                    const float skyColor[3], float* out_rgba32f, IdkVxStats* stats);

#ifdef __cplusplus
}
#endif
#endif /* IDKVX_H */
