// idkpt.hpp -- header-only C++17 host mirror of IDKEngine.Render.PathTracer over the C ABI of idkpt.h.
//
// The reference host is compiled C#; .NET is not available in this image, so the class a maintainer would write as
// `PathTracerNative : IDisposable` (INTEGRATION.md) is provided here in C++ with the reference's member names, argument
// meaning and reset-on-set behaviour (PathTracer.cs:12-125,170-346). Errors become idk::Error carrying the IdkPtStatus and
// idkpt_last_error(). Link with -lidkpt (no torch, no CUDA headers needed on the host side).
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "idkpt.h"
#include "idkvx.h"

namespace idk {

class Error : public std::runtime_error {
public:
    Error(int status, const std::string& what) : std::runtime_error(what), status_(status) {}
    int status() const { return status_; }

private:
    int status_;
};

// new PathTracer.GpuSettings() defaults (PathTracer.cs:127-138) + the class defaults (RayDepth 7, 1 spp; :12,211)
inline IdkPtSettings DefaultSettings() {
    IdkPtSettings s = {};
    s.Gpu.FocalLength = 8.0f;
    s.Gpu.LenseRadius = 0.0f;
    s.Gpu.DoDebugBVHTraversal = 0;
    s.Gpu.DoTraceLights = 0;
    s.Gpu.DoRussianRoulette = 1;
    s.RayDepth = 7;
    s.SamplesPerPixel = 1;
    return s;
}

// TonemapAndGammaCorrect.GpuSettings + Bloom.GpuSettings + Application.IsBloom defaults
inline IdkPtPostSettings DefaultPostSettings() {
    IdkPtPostSettings p = {};
    p.Exposure = 0.45f; p.Saturation = 1.06f; p.Linear = 0.18f; p.Peak = 1.0f; p.Compression = 0.1f;
    p.DoTonemapAndSrgbTransform = 1;
    p.IsBloom = 1; p.BloomThreshold = 1.5f; p.BloomMaxColor = 3.8f; p.BloomMinusLods = 3;
    return p;
}

struct Tile {
    int StripeHeight = 8, Index = 0, Count = 1;   // multi-GPU screen split: one PathTracer per GPU
    bool GlobalSlots = false;                     // IDKPT_CREATE_GLOBAL_SLOTS: the N tiles reproduce the untiled image bit for bit
};

class PathTracer {
public:
    // PathTracer(int width, int height, in GpuSettings settings)   PathTracer.cs:170
    PathTracer(int width, int height, const IdkPtGpuSettings& gpuSettings = DefaultSettings().Gpu, int device = 0, Tile tile = Tile(), int lanes = 0)
        : settings_(DefaultSettings()), width_(width), height_(height) {
        settings_.Gpu = gpuSettings;
        IdkPtCreateInfo ci = {};
        ci.Device = device; ci.Width = width; ci.Height = height;
        ci.TileStripeHeight = tile.StripeHeight; ci.TileIndex = tile.Index; ci.TileCount = tile.Count;
        ci.Flags = IDKPT_CREATE_LANES(lanes) | (tile.GlobalSlots ? IDKPT_CREATE_GLOBAL_SLOTS : 0u);
        const int rc = idkpt_create(&ci, &ctx_);
        if (rc != IDKPT_OK) {
            const char* msg = idkpt_last_error(nullptr);
            throw Error(rc, std::string("idkpt_create failed: ") + (msg ? msg : ""));
        }
    }
    ~PathTracer() { Dispose(); }
    PathTracer(const PathTracer&) = delete;
    PathTracer& operator=(const PathTracer&) = delete;
    PathTracer(PathTracer&& o) noexcept : ctx_(o.ctx_), settings_(o.settings_), width_(o.width_), height_(o.height_) { o.ctx_ = nullptr; }
    PathTracer& operator=(PathTracer&& o) noexcept {
        if (this != &o) { Dispose(); ctx_ = o.ctx_; settings_ = o.settings_; width_ = o.width_; height_ = o.height_; o.ctx_ = nullptr; }
        return *this;
    }
    void Dispose() {   // PathTracer.cs:344
        if (ctx_) { idkpt_destroy(ctx_); ctx_ = nullptr; }
    }

    // ---- the reference's public surface -------------------------------------------------------------------------------
    // Compute(): PathTracer.cs:214-271. Asynchronous (several samples in flight); pass `stats` for the synchronous, timed form.
    void Compute(const GpuPerFrameData& frame, IdkPtStats* stats = nullptr) { check(idkpt_compute(ctx_, &frame, &settings_, stats), "idkpt_compute"); }
    void Sync() { check(idkpt_sync(ctx_), "idkpt_sync"); }
    void SetSize(int width, int height) {   // :299-332
        check(idkpt_resize(ctx_, width, height), "idkpt_resize");
        width_ = width; height_ = height;
    }
    void ResetAccumulation() { check(idkpt_reset_accumulation(ctx_), "idkpt_reset_accumulation"); }   // :334
    const IdkPtGpuSettings& GetGpuSettings() const { return settings_.Gpu; }                           // :339
    uint32_t AccumulatedSamples() const { return idkpt_accumulated_samples(ctx_); }                    // :27-37
    int Width() const { return width_; }
    int Height() const { return height_; }

    // properties; the setters that reset the accumulation in the reference do so here (:16-25, :39-97)
    int RayDepth() const { return settings_.RayDepth; }
    void RayDepth(int v) { settings_.RayDepth = v; ResetAccumulation(); }
    float FocalLength() const { return settings_.Gpu.FocalLength; }
    void FocalLength(float v) { settings_.Gpu.FocalLength = v; ResetAccumulation(); }
    float LenseRadius() const { return settings_.Gpu.LenseRadius; }
    void LenseRadius(float v) { settings_.Gpu.LenseRadius = v; ResetAccumulation(); }
    bool DoDebugBVHTraversal() const { return settings_.Gpu.DoDebugBVHTraversal != 0; }
    void DoDebugBVHTraversal(bool v) { settings_.Gpu.DoDebugBVHTraversal = v; ResetAccumulation(); }
    bool DoTraceLights() const { return settings_.Gpu.DoTraceLights != 0; }
    void DoTraceLights(bool v) { settings_.Gpu.DoTraceLights = v; ResetAccumulation(); }
    bool DoRussianRoulette() const { return settings_.Gpu.DoRussianRoulette != 0; }
    void DoRussianRoulette(bool v) { settings_.Gpu.DoRussianRoulette = v; ResetAccumulation(); }
    int SamplesPerPixel() const { return settings_.SamplesPerPixel; }        // :12
    void SamplesPerPixel(int v) { settings_.SamplesPerPixel = v; }
    bool DoRaySorting() const { return settings_.DoRaySorting != 0; }        // :101-111
    void DoRaySorting(bool v) { settings_.DoRaySorting = v; }
    bool OutputAOVs() const { return settings_.OutputAOVs != 0; }            // :113-125
    void OutputAOVs(bool v) { settings_.OutputAOVs = v; }
    bool CollectStats() const { return settings_.CollectStats != 0; }
    void CollectStats(bool v) { settings_.CollectStats = v; }

    // Result / AlbedoTexture / NormalTexture (:143,167-168): rgba32f, width*height*4 floats, full-image layout
    std::vector<float> Result() const { return read(IDKPT_IMAGE_RESULT); }
    std::vector<float> AlbedoTexture() const { return read(IDKPT_IMAGE_ALBEDO); }
    std::vector<float> NormalTexture() const { return read(IDKPT_IMAGE_NORMAL); }

    // ---- what the reference passes implicitly through bound buffers ------------------------------------------------------
    void SetScene(const IdkPtSceneDesc& scene) { check(idkpt_set_scene(ctx_, &scene), "idkpt_set_scene"); }
    void UpdateRange(IdkPtArrayId which, uint64_t first, uint64_t count, const void* data) { check(idkpt_update_range(ctx_, which, first, count, data), "idkpt_update_range"); }
    void SetTextures(const IdkPtTextureDesc* textures, uint64_t count) { check(idkpt_set_textures(ctx_, textures, count), "idkpt_set_textures"); }
    void SetSky(const IdkPtSkyDesc& sky) { check(idkpt_set_sky(ctx_, &sky), "idkpt_set_sky"); }
    // The sky generated on the device (DESIGN.md 8f.1j): AtmosphericScatterer.Compute at faceSize (the engine's is 128), or the
    // unprojection of an equirectangular RGB float image (width * height * 3, row 0 first) at face size width / 4.
    // Each returns the kernel time in ms.
    float SkyAtmosphere(const IdkPtAtmosphereSettings& settings, int32_t faceSize = 128) {
        float ms = 0.0f;
        check(idkpt_sky_atmosphere(ctx_, &settings, faceSize, &ms), "idkpt_sky_atmosphere");
        return ms;
    }
    float SkyEquirectangular(const float* rgb, int32_t width, int32_t height) {
        float ms = 0.0f;
        check(idkpt_sky_equirectangular(ctx_, rgb, width, height, &ms), "idkpt_sky_equirectangular");
        return ms;
    }
    // The sky's faces, 6 * n * n rgba32f (+X,-X,+Y,-Y,+Z,-Z); empty for a constant sky.
    std::vector<float> ReadSky(int32_t* faceSize = nullptr) const {
        int32_t n = 0;
        check(idkpt_read_sky(ctx_, &n, nullptr, 0), "idkpt_read_sky");
        std::vector<float> faces((size_t)6 * n * n * 4);
        if (n) check(idkpt_read_sky(ctx_, &n, faces.data(), faces.size() * sizeof(float)), "idkpt_read_sky");
        if (faceSize) *faceSize = n;
        return faces;
    }

    // ---- presentation / interop -------------------------------------------------------------------------------------------
    void PresentAsync(void* pinnedHostRgba32f, uint64_t bytes, IdkPtImage which = IDKPT_IMAGE_RESULT) { check(idkpt_present_async(ctx_, which, pinnedHostRgba32f, bytes), "idkpt_present_async"); }
    void PresentWait() { check(idkpt_present_wait(ctx_), "idkpt_present_wait"); }
    float TlasBuild(int searchRadius = 15) { float ms = 0.0f; check(idkpt_tlas_build(ctx_, searchRadius, &ms), "idkpt_tlas_build"); return ms; }   // BVH.TlasBuild on the device
    // BLAS.Build + PreSplitting.PreSplit on the device (one BLAS of BVH.BlasesBuild); equal to the host build
    struct BlasBuildResult {
        std::vector<GpuBlasNode> nodes;
        std::vector<GpuBlasTriangle> triangles;
        int32_t requiredStackSize = 0, fragmentCount = 0;
        double sah = 0.0;
        float kernelMs = 0.0f;
    };
    BlasBuildResult BuildBlas(const PackedVec3* positions, uint64_t vertexCount, const GpuBlasTriangle* triangles, uint64_t triangleCount,
                              const IdkPtBlasBuildSettings* settings = nullptr) {
        BlasBuildResult r;
        IdkPtBlasBuild* b = nullptr;
        check(idkpt_blas_build(ctx_, positions, vertexCount, triangles, triangleCount, settings, &b, &r.kernelMs), "idkpt_blas_build");
        uint64_t nodeCount = 0, triCount = 0;
        idkpt_blas_build_info(b, &nodeCount, &triCount, &r.requiredStackSize, &r.fragmentCount, &r.sah);
        r.nodes.resize(nodeCount);
        r.triangles.resize(triCount);
        idkpt_blas_build_copy(b, r.nodes.data(), r.triangles.data());
        idkpt_blas_build_free(b);
        return r;
    }
    // BVH.BlasesBuild's loop over `descs` in one device call (idkpt_blas_build_batch): each BLAS equal to BuildBlas of it
    struct BlasBatchResult {
        std::vector<GpuBlasDesc> descs;   // offsets into nodes / triangles, as BVH.cs:363-386 fills them
        std::vector<GpuBlasNode> nodes;
        std::vector<GpuBlasTriangle> triangles;
        std::vector<int32_t> fragmentCounts;
        std::vector<double> sahs;
        float kernelMs = 0.0f;
    };
    BlasBatchResult BuildBlases(const PackedVec3* positions, uint64_t vertexCount, const GpuBlasTriangle* triangles, uint64_t triangleCount,
                                const GpuBlasDesc* descs, uint32_t descCount, const IdkPtBlasBuildSettings* settings = nullptr) {
        BlasBatchResult r;
        IdkPtBlasBuild* b = nullptr;
        check(idkpt_blas_build_batch(ctx_, positions, vertexCount, triangles, triangleCount, descs, descCount, settings, &b, &r.kernelMs),
              "idkpt_blas_build_batch");
        uint64_t nodeCount = 0, triCount = 0;
        idkpt_blas_build_info(b, &nodeCount, &triCount, nullptr, nullptr, nullptr);
        r.descs.resize(descCount);
        r.nodes.resize(nodeCount);
        r.triangles.resize(triCount);
        r.fragmentCounts.resize(descCount);
        r.sahs.resize(descCount);
        idkpt_blas_build_batch_copy(b, r.descs.data(), r.nodes.data(), r.triangles.data(), r.fragmentCounts.data(), r.sahs.data());
        idkpt_blas_build_free(b);
        return r;
    }
    // ModelManager.Add(models) on the device scene in place (idkpt_add_models): every id of `models` local to its arrays.
    // Returns the device time of the call.
    float AddModels(const IdkPtAddModelsDesc& models, const IdkPtBlasBuildSettings* settings = nullptr) {
        float ms = 0.0f;
        check(idkpt_add_models(ctx_, &models, settings, &ms), "idkpt_add_models");
        return ms;
    }
    // ModelManager.Update on the device (idkpt_set_animations .. idkpt_update_models)
    void SetAnimations(const IdkPtAnimationDesc& desc) { check(idkpt_set_animations(ctx_, &desc), "idkpt_set_animations"); }
    void EnableAnimations(uint32_t first, uint32_t count, const uint8_t* enabled) {
        check(idkpt_enable_animations(ctx_, first, count, enabled), "idkpt_enable_animations");
    }
    void SetNodeTransforms(uint32_t first, uint32_t count, const IdkPtNode* nodes) {
        check(idkpt_set_node_transforms(ctx_, first, count, nodes), "idkpt_set_node_transforms");
    }
    // Returns the moved bits (1 anyNodeMoved, 2 anyMeshInstanceMoved); *kernelMs (may be null) the device time
    uint32_t UpdateModels(float animationTime, int32_t searchRadius = 15, float* kernelMs = nullptr) {
        uint32_t moved = 0;
        check(idkpt_update_models(ctx_, animationTime, searchRadius, &moved, kernelMs), "idkpt_update_models");
        return moved;
    }
    float Denoise(const IdkPtDenoiseSettings& s) { float ms = 0.0f; check(idkpt_denoise(ctx_, &s, &ms), "idkpt_denoise"); return ms; }   // PathTracerPipeline.Denoise
    std::vector<float> Denoised() const { return read(IDKPT_IMAGE_DENOISED); }
    void RegisterHostBuffer(void* hostPtr, uint64_t bytes) { check(idkpt_register_host_buffer(ctx_, hostPtr, bytes), "idkpt_register_host_buffer"); }
    void UnregisterHostBuffer(void* hostPtr) { check(idkpt_unregister_host_buffer(ctx_, hostPtr), "idkpt_unregister_host_buffer"); }
    // Bloom + TonemapAndGammaCorrect -> RGBA8 (Application.cs:217-223); out may be null to keep the frame on the device
    float PostProcess(const IdkPtPostSettings& post, uint8_t* rgba8Out, IdkPtImage source = IDKPT_IMAGE_RESULT) {
        float ms = 0.0f;
        check(idkpt_post_process(ctx_, &post, source, rgba8Out, &ms), "idkpt_post_process");
        return ms;
    }
    void* StreamHandle() const { void* s = nullptr; check(idkpt_stream_handle(ctx_, &s), "idkpt_stream_handle"); return s; }
    std::pair<void*, uint64_t> ResultDevicePtr(IdkPtImage which = IDKPT_IMAGE_RESULT) const {
        void* p = nullptr; uint64_t n = 0;
        check(idkpt_result_device_ptr(ctx_, which, &p, &n), "idkpt_result_device_ptr");
        return {p, n};
    }
    std::vector<int32_t> TileRows() const {
        int32_t n = 0;
        check(idkpt_tile_rows(ctx_, &n, nullptr, 0), "idkpt_tile_rows");
        std::vector<int32_t> rows((size_t)n);
        check(idkpt_tile_rows(ctx_, &n, rows.data(), n), "idkpt_tile_rows");
        return rows;
    }

    // ---- neighbours of the path (SURVEY 8f) ------------------------------------------------------------------------------------
    std::vector<IdkPtHit> TraceRays(const std::vector<IdkPtRay>& rays, bool traceLights = false, bool anyHit = false) {
        std::vector<IdkPtHit> hits(rays.size());
        float ms = 0.0f;
        check((anyHit ? idkpt_trace_rays_any : idkpt_trace_rays)(ctx_, rays.data(), rays.size(), traceLights, hits.data(), &ms), "idkpt_trace_rays");
        return hits;
    }
    void ShadowsRayTraced(const GpuPerFrameData& frame, const float* depth, const float* normalRG, int width, int height, int lightIndex, int samples,
                          uint32_t noiseIndex, const float* taaJitter, float* visibilityInOut) {
        check(idkpt_shadows_ray_traced(ctx_, &frame, depth, normalRG, width, height, lightIndex, samples, noiseIndex, taaJitter, visibilityInOut, nullptr), "idkpt_shadows_ray_traced");
    }
    // PointShadowManager.UpdateBuffer / RenderShadowMaps: traced D16 cube maps, 6 * size^2 uint16 per shadow (idkpt.h)
    void SetPointShadows(const GpuPointShadow* shadows, const int32_t* sizes, uint32_t count) {
        check(idkpt_set_point_shadows(ctx_, shadows, sizes, count), "idkpt_set_point_shadows");
    }
    float RenderPointShadows(uint32_t first, uint32_t count, const uint32_t* faceMasks = nullptr) {
        float ms = 0.0f;
        check(idkpt_render_point_shadows(ctx_, first, count, faceMasks, &ms), "idkpt_render_point_shadows");
        return ms;
    }
    void ReadPointShadow(int32_t index, uint16_t* dst, uint64_t bytes) { check(idkpt_read_point_shadow(ctx_, index, dst, bytes), "idkpt_read_point_shadow"); }
    void* PointShadowDevicePtr(int32_t index, uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_point_shadow_device_ptr(ctx_, index, &p, bytes), "idkpt_point_shadow_device_ptr");
        return p;
    }
    // VolumetricLighting.Compute through the point-shadow cube maps: out = width * height * 4 halves, or nullptr to keep the
    // image on the device (VolumetricDevicePtr). Returns the kernel time in ms.
    float VolumetricLighting(const GpuPerFrameData& frame, const IdkPtVolumetricSettings& settings, const float* depth, int depthWidth, int depthHeight,
                             int width, int height, const float* taaJitter, uint16_t* outRgba16f) {
        float ms = 0.0f;
        check(idkpt_volumetric_lighting(ctx_, &frame, &settings, depth, depthWidth, depthHeight, width, height, taaJitter, outRgba16f, &ms),
              "idkpt_volumetric_lighting");
        return ms;
    }
    void* VolumetricDevicePtr(uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_volumetric_device_ptr(ctx_, &p, bytes), "idkpt_volumetric_device_ptr");
        return p;
    }
    // The two passes above on a host or device G-buffer (GBufferDevicePtrs' as it is). ShadowsRayTracedGBuffer writes the
    // context's visibility image of `slot` (ShadowsDevicePtr: DeferredLighting's rtVisibility[k]); visibilityOut may be nullptr.
    float ShadowsRayTracedGBuffer(const GpuPerFrameData& frame, const IdkPtGBuffer& gbuffer, int lightIndex, int samples, uint32_t noiseIndex,
                                  const float* taaJitter, int32_t slot, float* visibilityOut) {
        float ms = 0.0f;
        check(idkpt_shadows_ray_traced_gbuffer(ctx_, &frame, &gbuffer, lightIndex, samples, noiseIndex, taaJitter, slot, visibilityOut, &ms),
              "idkpt_shadows_ray_traced_gbuffer");
        return ms;
    }
    void* ShadowsDevicePtr(int32_t slot, uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_shadows_device_ptr(ctx_, slot, &p, bytes), "idkpt_shadows_device_ptr");
        return p;
    }
    float VolumetricLightingGBuffer(const GpuPerFrameData& frame, const IdkPtVolumetricSettings& settings, const IdkPtGBuffer& gbuffer,
                                    int width, int height, const float* taaJitter, uint16_t* outRgba16f) {
        float ms = 0.0f;
        check(idkpt_volumetric_lighting_gbuffer(ctx_, &frame, &settings, &gbuffer, width, height, taaJitter, outRgba16f, &ms),
              "idkpt_volumetric_lighting_gbuffer");
        return ms;
    }
    // SSAO.Compute on a host or device G-buffer: out = Width * Height bytes (R8Unorm), or nullptr to keep the image on the device
    // (SsaoDevicePtr; DeferredLighting's IsSSAO reads it). Returns the kernel time in ms.
    float Ssao(const GpuPerFrameData& frame, const IdkPtSsaoSettings& settings, const IdkPtGBuffer& gbuffer, uint8_t* outR8) {
        float ms = 0.0f;
        check(idkpt_ssao(ctx_, &frame, &settings, &gbuffer, outR8, &ms), "idkpt_ssao");
        return ms;
    }
    void* SsaoDevicePtr(uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_ssao_device_ptr(ctx_, &p, bytes), "idkpt_ssao_device_ptr");
        return p;
    }
    // The deferred lighting draw: out = Width * Height * 4 floats (rgba32f), or nullptr to keep the image on the device
    // (DeferredDevicePtr). indirect and rtVisibility follow gbuffer.OnDevice. Returns the kernel time in ms.
    float DeferredLighting(const GpuPerFrameData& frame, const IdkPtDeferredSettings& settings, const IdkPtGBuffer& gbuffer, const float* taaJitter,
                           const float* indirectRgba32f, const float* const* rtVisibility, uint32_t rtCount, float* outRgba32f) {
        float ms = 0.0f;
        check(idkpt_deferred_lighting(ctx_, &frame, &settings, &gbuffer, taaJitter, indirectRgba32f, rtVisibility, rtCount, outRgba32f, &ms),
              "idkpt_deferred_lighting");
        return ms;
    }
    void* DeferredDevicePtr(uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_deferred_device_ptr(ctx_, &p, bytes), "idkpt_deferred_device_ptr");
        return p;
    }
    // SSR.Compute + "Merge Textures": source = IDKPT_LIT_SOURCE_ARRAY (colorRgba32f, host or device as gbuffer.OnDevice says)
    // or IDKPT_LIT_SOURCE_DEFERRED. mergedOut = Width * Height * 4 floats, ssrOut = Width * Height * 4 halves; either may be
    // nullptr to keep that image on the device (SsrDevicePtrs). Returns the kernel time in ms.
    float Ssr(const GpuPerFrameData& frame, const IdkPtSsrSettings& settings, const IdkPtGBuffer& gbuffer, int32_t source,
              const float* colorRgba32f, float* mergedOutRgba32f, uint16_t* ssrOutRgba16f) {
        float ms = 0.0f;
        check(idkpt_ssr(ctx_, &frame, &settings, &gbuffer, source, colorRgba32f, mergedOutRgba32f, ssrOutRgba16f, &ms), "idkpt_ssr");
        return ms;
    }
    void SsrDevicePtrs(void** merged, void** ssr, uint64_t* mergedBytes = nullptr, uint64_t* ssrBytes = nullptr) {
        check(idkpt_ssr_device_ptrs(ctx_, merged, ssr, mergedBytes, ssrBytes), "idkpt_ssr_device_ptrs");
    }
    // TaaResolve.Compute at width x height over the render-size inputs, against the context's history: out = width * height * 4
    // halves, or nullptr to keep the result on the device (TaaDevicePtr). Returns the kernel time in ms.
    float TaaResolve(const IdkPtTaaSettings& settings, const IdkPtTaaInputs& inputs, int width, int height, uint16_t* outRgba16f) {
        float ms = 0.0f;
        check(idkpt_taa_resolve(ctx_, &settings, &inputs, width, height, outRgba16f, &ms), "idkpt_taa_resolve");
        return ms;
    }
    void* TaaDevicePtr(uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_taa_device_ptr(ctx_, &p, bytes), "idkpt_taa_device_ptr");
        return p;
    }
    // LightingShadingRateClassifier.Compute over the render-size inputs: outRates = ceil(h/16) * ceil(w/16) palette indices, or
    // nullptr to keep the image on the device (ShadingRateDevicePtr; DeferredLighting with IsVariableRateShading reads it);
    // debugOutR32f (DebugMode 2..4 only) the same size, or nullptr. Returns the kernel time in ms.
    float ShadingRate(const GpuPerFrameData& frame, const IdkPtShadingRateSettings& settings, const IdkPtShadingRateInputs& inputs,
                      uint8_t* outRates, float* debugOutR32f = nullptr) {
        float ms = 0.0f;
        check(idkpt_shading_rate(ctx_, &frame, &settings, &inputs, outRates, debugOutR32f, &ms), "idkpt_shading_rate");
        return ms;
    }
    void* ShadingRateDevicePtr(uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_shading_rate_device_ptr(ctx_, &p, bytes), "idkpt_shading_rate_device_ptr");
        return p;
    }
    // The G-buffer pass at width x height into context images (DESIGN.md 8f.1g); taaJitter and prevPositions may be nullptr.
    // prevPositions may be PrevPositionsDevicePtr(), read in place. Returns the kernel time in ms.
    float GBuffer(const GpuPerFrameData& frame, int32_t width, int32_t height, const float* taaJitter = nullptr,
                  const PackedVec3* prevPositions = nullptr) {
        float ms = 0.0f;
        check(idkpt_gbuffer(ctx_, &frame, width, height, taaJitter, prevPositions, &ms), "idkpt_gbuffer");
        return ms;
    }
    // The images of the last GBuffer call: an OnDevice G-buffer for Ssao / DeferredLighting / Ssr, and the velocity.
    IdkPtGBuffer GBufferDevicePtrs(const float** velocityRG = nullptr) {
        IdkPtGBuffer g = {};
        check(idkpt_gbuffer_device_ptrs(ctx_, &g, velocityRG), "idkpt_gbuffer_device_ptrs");
        return g;
    }
    void ReadGBuffer(float* depth, float* normalRG, float* albedoRGB, float* metallicRoughness, float* emissiveRGB, float* velocityRG) {
        check(idkpt_read_gbuffer(ctx_, depth, normalRG, albedoRGB, metallicRoughness, emissiveRGB, velocityRG), "idkpt_read_gbuffer");
    }
    // prevVertexPositionSSBO: the positions SkinVertices keeps from before each skin, valid until SetScene or Dispose
    const PackedVec3* PrevPositionsDevicePtr(uint64_t* bytes = nullptr) {
        void* p = nullptr;
        check(idkpt_prev_positions_device_ptr(ctx_, &p, bytes), "idkpt_prev_positions_device_ptr");
        return (const PackedVec3*)p;
    }
    // The blended layers composited over the lit image in place (DESIGN.md 8f.1h): the context's deferred image (source
    // IDKPT_LIT_SOURCE_DEFERRED) or `color` (IDKPT_LIT_SOURCE_ARRAY); only gbuffer.Depth is read. voxels / cone: IsVXGI only.
    // Returns the kernel time in ms.
    float Transparency(const GpuPerFrameData& frame, const IdkPtTransparencySettings& settings, const IdkPtGBuffer& gbuffer,
                       int32_t source, float* color = nullptr, const float* taaJitter = nullptr, IdkVxCtx* voxels = nullptr,
                       const IdkVxConeSettings* cone = nullptr, float* outRgba32f = nullptr) {
        float ms = 0.0f;
        check(idkpt_transparency(ctx_, &frame, &settings, &gbuffer, taaJitter, voxels, cone, source, color, outRgba32f, &ms), "idkpt_transparency");
        return ms;
    }
    // The light spheres and the skybox, in place into the last GBuffer's images and the deferred image (DESIGN.md 8f.1i);
    // taaJitter and outRgba32f may be nullptr. Returns the kernel time in ms.
    float LightsAndSkybox(const GpuPerFrameData& frame, const float* taaJitter = nullptr, float* outRgba32f = nullptr) {
        float ms = 0.0f;
        check(idkpt_lights_and_skybox(ctx_, &frame, taaJitter, outRgba32f, &ms), "idkpt_lights_and_skybox");
        return ms;
    }
    // The same draws with IsVariableRateShading, under the rate image of the last ShadingRate call (DESIGN.md 8f.1i).
    float LightsAndSkyboxVrs(const GpuPerFrameData& frame, const float* taaJitter = nullptr, float* outRgba32f = nullptr) {
        float ms = 0.0f;
        check(idkpt_lights_and_skybox_vrs(ctx_, &frame, taaJitter, outRgba32f, &ms), "idkpt_lights_and_skybox_vrs");
        return ms;
    }
    void SetSkinningData(const GpuUnskinnedVertex* vertices, uint64_t count) { check(idkpt_set_skinning_data(ctx_, vertices, count), "idkpt_set_skinning_data"); }
    void SkinVertices(const float* jointMatrices3x4, uint64_t jointCount, const IdkPtSkinningCmd* cmds, uint32_t cmdCount) {
        check(idkpt_skin_vertices(ctx_, jointMatrices3x4, jointCount, cmds, cmdCount, nullptr), "idkpt_skin_vertices");
    }
    void BlasRefit(uint32_t firstBlas, uint32_t count = 1) { check(idkpt_blas_refit(ctx_, firstBlas, count, nullptr), "idkpt_blas_refit"); }
    // BVH.BlasesBuild(first, count) on the scene in place, from the current device positions; returns the device ms
    float RebuildBlases(uint32_t firstBlas, uint32_t count = 1, const IdkPtBlasBuildSettings* settings = nullptr) {
        float ms = 0.0f;
        check(idkpt_blas_rebuild(ctx_, firstBlas, count, settings, &ms), "idkpt_blas_rebuild");
        return ms;
    }
    // BLAS.ComputeGlobalSAH of each BLAS in [first, first + count) as the device holds it now
    std::vector<double> BlasSah(uint32_t firstBlas, uint32_t count = 1, const IdkPtBlasBuildSettings* settings = nullptr) const {
        std::vector<double> sah(count);
        check(idkpt_blas_sah(ctx_, firstBlas, count, settings, sah.data()), "idkpt_blas_sah");
        return sah;
    }
    void ReadRange(IdkPtArrayId which, uint64_t first, uint64_t count, void* out) const { check(idkpt_read_range(ctx_, which, first, count, out), "idkpt_read_range"); }

    IdkPtCtx* Handle() const { return ctx_; }

    // One process driving N GPUs (like the engine): tracers in tile order (tracer r created with Tile{.., r, N}). Afterwards every
    // Compute() also delivers this tile into every tracer's full frame over peer memory (PresentAsync(.., IDKPT_IMAGE_GATHERED)).
    // With one host thread only queue work (Compute without stats): a synchronous call would wait for peers not yet submitted.
    static void ConnectPeers(const std::vector<PathTracer*>& tracers) {
        std::vector<IdkPtCtx*> ctxs;
        for (PathTracer* t : tracers) ctxs.push_back(t->ctx_);
        const int rc = idkpt_gather_connect(ctxs.data(), (int32_t)ctxs.size());
        if (rc != IDKPT_OK) {
            std::string msg;
            for (IdkPtCtx* c : ctxs) { const char* m = idkpt_last_error(c); if (m && *m) { msg = m; break; } }
            throw Error(rc, "idkpt_gather_connect failed: " + msg);
        }
    }

private:
    void check(int rc, const char* what) const {
        if (rc != IDKPT_OK) {
            const char* msg = idkpt_last_error(ctx_);
            throw Error(rc, std::string(what) + " failed: " + (msg ? msg : ""));
        }
    }
    std::vector<float> read(IdkPtImage which) const {
        std::vector<float> img((size_t)width_ * height_ * 4);
        check(idkpt_read_result(ctx_, which, img.data(), img.size() * sizeof(float)), "idkpt_read_result");
        return img;
    }

    IdkPtCtx* ctx_ = nullptr;
    IdkPtSettings settings_;
    int width_, height_;
};

// Voxelizer.Render() + ConeTracer.Compute() (Source/Render/VXGI/Voxelizer/Voxelizer.cs:57-114, ConeTracing/ConeTracer.cs:10-50)
class Voxelizer {
public:
    Voxelizer(int width, int height, int depth, const float gridMin[3], const float gridMax[3], int device = 0) {
        IdkVxCreateInfo ci = {};
        ci.Device = device; ci.Width = width; ci.Height = height; ci.Depth = depth;
        for (int i = 0; i < 3; i++) { ci.GridMin[i] = gridMin[i]; ci.GridMax[i] = gridMax[i]; }
        const int rc = idkvx_create(&ci, &ctx_);
        if (rc != IDKPT_OK) {
            const char* msg = idkvx_last_error(nullptr);
            throw Error(rc, std::string("idkvx_create failed: ") + (msg ? msg : ""));
        }
    }
    ~Voxelizer() { Dispose(); }
    Voxelizer(const Voxelizer&) = delete;
    Voxelizer& operator=(const Voxelizer&) = delete;
    void Dispose() { if (ctx_) { idkvx_destroy(ctx_); ctx_ = nullptr; } }

    void SetScene(const IdkPtSceneDesc& scene) { check(idkvx_set_scene(ctx_, &scene), "idkvx_set_scene"); }
    // Voxelise pt's device scene as it stands at each Render, with no copy (idkvx_set_scene_from); SetScene ends the binding
    void SetSceneFrom(PathTracer& pt) { check(idkvx_set_scene_from(ctx_, pt.Handle()), "idkvx_set_scene_from"); }
    void SetGrid(const float gridMin[3], const float gridMax[3]) { check(idkvx_set_grid(ctx_, gridMin, gridMax), "idkvx_set_grid"); }   // GridMin / GridMax setters
    int LevelCount() const { return idkvx_level_count(ctx_); }
    IdkVxStats Render() { IdkVxStats st = {}; check(idkvx_voxelize(ctx_, &st), "idkvx_voxelize"); return st; }
    // IsConservativeRasterization setter: every pixel a triangle touches instead of the pixel centres it covers, from the next Render on
    void SetConservativeRasterization(bool enable) {
        check(idkvx_set_conservative_rasterization(ctx_, enable ? 1 : 0), "idkvx_set_conservative_rasterization");
    }
    // point-shadowed lights: PCF lookup into a path tracer's cube maps, or shadow rays through its BVH (idkvx.h); nullptr detaches
    void SetShadowMaps(const PathTracer* pt) { check(idkvx_set_shadow_maps(ctx_, pt ? pt->Handle() : nullptr), "idkvx_set_shadow_maps"); }
    void SetShadowTracer(const PathTracer* pt) { check(idkvx_set_shadow_tracer(ctx_, pt ? pt->Handle() : nullptr), "idkvx_set_shadow_tracer"); }
    // ConeTracer.Compute: G-buffer attachments in, rgba32f indirect light out (width * height * 4 floats)
    std::vector<float> ConeTrace(const GpuPerFrameData& frame, const IdkVxConeSettings& settings, const float* depth, const float* normalRG,
                                 const float* metallicRoughness, int width, int height, const float skyColor[3], IdkVxStats* stats = nullptr) {
        std::vector<float> out((size_t)width * height * 4);
        check(idkvx_cone_trace(ctx_, &frame, &settings, depth, normalRG, metallicRoughness, width, height, skyColor, out.data(), stats), "idkvx_cone_trace");
        return out;
    }
    // ConeTracer.Compute on a host or device G-buffer (PathTracer::GBufferDevicePtrs' as it is): out may be nullptr to keep the
    // image on the device (ConeTraceDevicePtr: DeferredLighting's indirect light)
    void ConeTraceGBuffer(const GpuPerFrameData& frame, const IdkVxConeSettings& settings, const IdkPtGBuffer& gbuffer, const float skyColor[3],
                          float* outRgba32f, IdkVxStats* stats = nullptr) {
        check(idkvx_cone_trace_gbuffer(ctx_, &frame, &settings, &gbuffer, skyColor, outRgba32f, stats), "idkvx_cone_trace_gbuffer");
    }
    void* ConeTraceDevicePtr(uint64_t* bytes = nullptr) const {
        void* p = nullptr;
        check(idkvx_cone_trace_device_ptr(ctx_, &p, bytes), "idkvx_cone_trace_device_ptr");
        return p;
    }
    // ConeTracer.GpuSettings defaults (ConeTracer.cs:10-22)
    static IdkVxConeSettings DefaultConeSettings() {
        IdkVxConeSettings c = {};
        c.MaxSamples = 4; c.StepMultiplier = 0.16f; c.GIBoost = 1.3f; c.GISkyBoxBoost = 1.0f / 1.3f; c.NormalRayOffset = 1.0f; c.NoiseIndex = 0;
        return c;
    }
    // DebugRender's settings, with the constructor defaults of Voxelizer.cs:68
    float DebugStepMultiplier = 0.4f;
    float DebugConeAngle = 0.0f;
    // Voxelizer.DebugRender: the grid marched per pixel over the sky of `sky`, rgba32f out (width * height * 4 floats)
    std::vector<float> DebugRender(const PathTracer& sky, const GpuPerFrameData& frame, int width, int height, IdkVxStats* stats = nullptr) {
        std::vector<float> out((size_t)width * height * 4);
        check(idkvx_debug_render(ctx_, sky.Handle(), &frame, DebugStepMultiplier, DebugConeAngle, width, height, out.data(), stats), "idkvx_debug_render");
        return out;
    }
    // the last DebugRender's image on the device (nullptr before the first)
    void* DebugDevicePtr(uint64_t* bytes = nullptr) const {
        void* p = nullptr;
        check(idkvx_debug_device_ptr(ctx_, &p, bytes), "idkvx_debug_device_ptr");
        return p;
    }

private:
    void check(int rc, const char* what) const {
        if (rc != IDKPT_OK) {
            const char* msg = idkvx_last_error(ctx_);
            throw Error(rc, std::string(what) + " failed: " + (msg ? msg : ""));
        }
    }
    IdkVxCtx* ctx_ = nullptr;
};

}  // namespace idk
