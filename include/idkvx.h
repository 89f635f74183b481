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
 * (pixel-centre coverage, DESIGN.md section 8), which matches GL to tolerance and its own CPU oracle bit for bit. The engine's
 * conservative-raster option (Voxelizer.IsConservativeRasterization, GL_NV_conservative_raster) is built too:
 * idkvx_set_conservative_rasterization switches the kernels to an exact square-against-triangle coverage test (DESIGN.md
 * section 7).
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

/* Voxelizer.Render(modelManager) reads the scene the engine binds globally; this is that binding. After the call the voxeliser
 * holds no scene of its own (idkvx_set_scene's copies are released) and every idkvx_voxelize reads path_tracer's device arrays
 * as they stand at that moment: positions, normals and tangents after idkpt_skin_vertices, MESH_TRANSFORMS, MESHES,
 * MATERIALS and LIGHTS after idkpt_update_range, textures after idkpt_set_textures, and a new idkpt_set_scene all reach the
 * next voxelisation with no copy. The kernels, their launches, slab mode, both coverage rules and the point-shadow rules
 * (idkvx_set_shadow_maps / idkvx_set_shadow_tracer) are those of a voxeliser with its own scene.
 * path_tracer must be on the voxeliser's device (else IDKPT_ERR_UNSUPPORTED); it may have no scene yet: idkvx_voxelize then
 * fails with IDKPT_ERR_NO_SCENE until it has one. NULL unbinds and leaves no scene. The grid's voxelised state is cleared, as
 * idkvx_set_scene clears it. A later idkvx_set_scene returns to an owned copy.
 * Lifetime: idkpt_destroy unbinds every voxeliser bound to the path tracer (their next idkvx_voxelize fails with
 * IDKPT_ERR_NO_SCENE); idkvx_destroy, a rebind, idkvx_set_scene or an unbind ends the binding from the voxeliser's side.
 * Ordering: every path-tracer call that writes scene arrays, and idkvx_voxelize, is synchronous, and samples idkpt_compute has
 * queued only read the scene; so idkvx_voxelize needs no idkpt_sync. */
IDKPT_API int idkvx_set_scene_from(IdkVxCtx* ctx, struct IdkPtCtx* path_tracer);
IDKPT_API int idkvx_set_grid(IdkVxCtx* ctx, const float gridMin[3], const float gridMax[3]);   /* Voxelizer.GridMin/GridMax, Voxelizer.cs:16-33 */
IDKPT_API int32_t idkvx_level_count(IdkVxCtx* ctx);                                           /* Texture.GetMaxMipmapLevel */

/* Voxelizer.Render(): clear + voxelise + mip chain. */
IDKPT_API int idkvx_voxelize(IdkVxCtx* ctx, IdkVxStats* stats);

/* Voxelizer.IsConservativeRasterization (Voxelizer.cs:41-56,142): 0 (the default after idkvx_create) = a triangle covers the
 * pixels whose centre it contains; 1 = it covers every pixel whose closed square it touches, with attributes extrapolated to
 * the pixel centre, so that geometry thinner than a voxel voxelises without gaps (DESIGN.md section 7). `enable` other than
 * 0 or 1 fails with IDKPT_ERR_INVALID_ARGUMENT and leaves the setting as it was. The setting belongs to the context: it
 * survives idkvx_set_scene / idkvx_set_grid / idkvx_set_slab, applies from the next idkvx_voxelize on, and does not touch
 * the current grid. */
IDKPT_API int idkvx_set_conservative_rasterization(IdkVxCtx* ctx, int32_t enable);

/* rgba16f texels of one mip level, x fastest (size = w*h*d*8 bytes). */
/* Lights with PointShadowIndex >= 0 are attenuated by Visibility() in the fragment stage (Voxelize/fragment.glsl:55-58,100-117),
 * a PCF lookup into the shadow cube map the rasteriser renders (PointShadowManager). The voxeliser evaluates it in one of two
 * modes, each taking a path-tracer context on the same device (NULL detaches):
 *   shadow maps (idkvx_set_shadow_maps): the PCF lookup itself -- 2 % biased reference depth, seamless bilinear footprint,
 *     compare LESS -- into the cube maps of that context (idkpt_set_point_shadows / idkpt_render_point_shadows), at the
 *     light's PointShadowIndex. An index >= the context's shadow count fails with IDKPT_ERR_INVALID_ARGUMENT.
 *   shadow tracer (idkvx_set_shadow_tracer): an any-hit shadow ray from the 2 %-biased sample point to the light through the
 *     BVH of a context holding the same scene (hard 0/1 shadows instead of the filtered lookup; needs no cube-map memory).
 * Shadow maps take precedence when both are attached. A scene with such lights cannot be voxelised with neither
 * (IDKPT_ERR_UNSUPPORTED). */
struct IdkPtCtx;
IDKPT_API int idkvx_set_shadow_tracer(IdkVxCtx* ctx, struct IdkPtCtx* path_tracer);
IDKPT_API int idkvx_set_shadow_maps(IdkVxCtx* ctx, struct IdkPtCtx* path_tracer);
IDKPT_API int idkvx_read_level(IdkVxCtx* ctx, int32_t level, void* dst_rgba16f, uint64_t bytes);

/* ConeTracer.Compute(): per pixel of a width x height G-buffer (host arrays: depth [w*h], normal = octahedral rg
 * [w*h*2], metallicRoughness = rg [w*h*2]) -> rgba32f indirect light [w*h*4]. skyColor = constant sky albedo. */
IDKPT_API int idkvx_cone_trace(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* settings,
                               const float* depth, const float* normalRG, const float* metallicRoughness,
                               int32_t width, int32_t height, const float skyColor[3], float* out_rgba32f, IdkVxStats* stats);

/* The same trace on an IdkPtGBuffer: Depth, NormalRG and MetallicRoughness (the other attachments may be NULL), host arrays with
 * OnDevice = 0, device arrays on the context's device read in place with OnDevice = 1 (aligned to 4 bytes for Depth, 8 for the
 * other two; as idkpt.h's G-buffer passes check them), e.g. idkpt_gbuffer_device_ptrs' G-buffer. out_rgba32f: Width*Height*4
 * floats, or NULL to keep the image on the device only. Every argument is checked before anything is uploaded or launched:
 * a rejected call (IDKPT_ERR_INVALID_ARGUMENT) leaves the image as it was.
 * idkvx_cone_trace_device_ptr: the rgba32f image of the last successful idkvx_cone_trace* call (width * rows traced * 16 bytes,
 * 256-byte aligned: idkpt_deferred_lighting's indirect_rgba32f with OnDevice = 1); valid until the next cone trace or
 * idkvx_destroy. Fails before the first successful trace and after a failed one. */
IDKPT_API int idkvx_cone_trace_gbuffer(IdkVxCtx* ctx, const GpuPerFrameData* frame, const IdkVxConeSettings* settings,
                                       const IdkPtGBuffer* gbuffer, const float skyColor[3], float* out_rgba32f, IdkVxStats* stats);
IDKPT_API int idkvx_cone_trace_device_ptr(IdkVxCtx* ctx, void** dev_ptr, uint64_t* bytes);

/* Voxelizer.DebugRender (Voxelizer.cs:230-244, VXGI/Voxelize/DebugVisualization/compute.glsl): the grid-configuration view
 * (RasterPipeline.Render's IsConfigureGridMode branch). Per pixel of a width x height image, the camera ray of `frame`
 * (InvProjection, InvView, ViewPos; pixel centres, no jitter) is clipped to [GridMin, GridMax]; a ray that misses the box, or
 * has it behind the camera, stores the sky (rgb, 1). Otherwise a cone of `cone_angle` is marched through the context's
 * current grid (every level, whatever it holds; a fresh context's cleared grid renders as sky) from where the ray enters the
 * grid, or from ViewPos inside it, with steps of step_multiplier x the sample diameter, until alpha reaches 1 or the cone
 * leaves the grid; the result c is blended over the sky: (c.rgb + (1 - c.a) * sky.rgb, c.a + (1 - c.a)). The sky is that of
 * the path-tracer context `sky` on the same device (idkpt_set_sky, idkpt_sky_atmosphere, idkpt_sky_equirectangular; a
 * constant sky works the same way); every sky the library holds is opaque, so the blend takes its alpha as 1.
 * out_rgba32f: width*height*4 floats, row 0 first, not rounded (the engine's target is rgba16f or R11G11B10F: the host rounds
 * when it copies into its texture). out_rgba32f may be NULL: the image then stays on the device only, where
 * idkvx_debug_device_ptr finds it; either way the context keeps the image of the last successful call, in an allocation that
 * calls of the same or a smaller size reuse. stats (may be NULL): ConeTraceMs = CUDA-event time of the kernels, ConeSteps =
 * samples the marches took, KernelLaunches. Synchronous. Fails with IDKPT_ERR_INVALID_ARGUMENT, before anything is launched
 * (the previous image keeps every byte), on a NULL ctx, sky or frame; a sky context on another device; width or height
 * outside 1..16384; cone_angle not finite or outside [0, 1.5]; step_multiplier not finite or not > 0; and a grid and
 * step_multiplier for which (|GridMax - GridMin| + voxelMaxLength) / (voxelMinLength * step_multiplier) > 65536, the most
 * steps a march may take (DESIGN.md 8f.1k). */
IDKPT_API int idkvx_debug_render(IdkVxCtx* ctx, struct IdkPtCtx* sky, const GpuPerFrameData* frame, float step_multiplier,
                                 float cone_angle, int32_t width, int32_t height, float* out_rgba32f, IdkVxStats* stats);
/* The device image of the last successful idkvx_debug_render (rgba32f, width*height*16 bytes); NULL and 0 bytes before the
 * first. The pointer stays valid until the next idkvx_debug_render with a larger image, or idkvx_destroy. */
IDKPT_API int idkvx_debug_device_ptr(IdkVxCtx* ctx, void** dev_ptr, uint64_t* bytes);

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
