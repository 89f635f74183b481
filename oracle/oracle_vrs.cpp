// ORACLE (TEST INFRASTRUCTURE ONLY) -- variable-rate deferred lighting: the lighting shading-rate classifier and the deferred
// lighting draw under its rate image.
//
// Built as its own library (tests/vrs_oracle.py -> oracle/liboracle_vrs.so). It compiles oracle_deferred.cpp (and with it
// oracle_point_shadows.cpp and oracle.cpp) into the same translation unit and reuses EvaluateLighting, DfVisibility,
// DfPerspective, DfStoreR8, DecodeUnitVec and mixf unchanged; what it adds is restated here from the shaders and from
// NV_shading_rate_image.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/ShadingRateClassification/compute.glsl            the classifier (GetTileData, GetLuminance)
//   Resource/Shaders/ShadingRateClassification/include/Constants.glsl  TILE_SIZE 16, the rate and debug-mode enums
//   Source/Render/LightingShadingRateClassifier.cs                     settings, the palette, the R8UI / r32f images
//   Resource/Shaders/DeferredLighting/fragment.glsl                    the fragment shader, once per coarse fragment
//   Source/Render/RasterPipeline.cs:441-463, 590-593                   the draw under the rate image; the classification
//
// The rules DESIGN.md 8f.1f pins: the per-warp xor butterfly (16, 8, 4, 2, 1) and the in-order sum of the eight warp sums;
// round() half to even; uint() as cvt.rzi.sat.u32 (NaN and negatives 0, overflow UINT_MAX); edge lanes read colour 0 and
// velocity 0 and still count in the 256; a coarse fragment's sample at the centre of its area with imgCoord clamped to the image.
#include "oracle_deferred.cpp"

#include <cfenv>

namespace {

// subgroupAdd over 32 lanes in the pinned order: lane i adds lane i ^ o for o = 16, 8, 4, 2, 1. Returns lane 0's sum.
static float VrsButterfly(const float* lanes) {
    float v[32];
    for (int i = 0; i < 32; i++) v[i] = lanes[i];
    for (int o = 16; o >= 1; o >>= 1) {
        float n[32];
        for (int i = 0; i < 32; i++) n[i] = v[i] + v[i ^ o];
        for (int i = 0; i < 32; i++) v[i] = n[i];
    }
    return v[0];
}

// uint(x) as the hardware converts: truncation with saturation, NaN -> 0
static uint32_t VrsUint(float x) {
    if (x != x || x <= 0.0f) return 0u;
    if (x >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)x;
}

// round() half to even in the default rounding mode
static float VrsRoundEven(float x) { return std::nearbyint(x); }

// The coarse fragment of palette index r: {1x1, 2x1, 2x2, 4x2, 4x4}
static void VrsFragmentSize(int r, int& cw, int& ch) {
    static const int W[5] = {1, 2, 2, 4, 4}, H[5] = {1, 1, 2, 2, 4};
    cw = W[r]; ch = H[r];
}

// ShadingRateClassification/compute.glsl over a w x h image: one 16x16 tile per workgroup
static void ShadingRate(const GpuPerFrameData& f, const IdkPtShadingRateSettings& st, const float* color, const float* velocity, int w, int h,
                        uint8_t* rates, float* debug) {
    const int tilesX = (w + 15) / 16, tilesY = (h + 15) / 16;
    for (int ty = 0; ty < tilesY; ty++)
        for (int tx = 0; tx < tilesX; tx++) {
            float speed[256], lum[256], lumSq[256];
            for (int i = 0; i < 256; i++) {   // gl_LocalInvocationIndex = lx + 16 ly
                const int x = tx * 16 + i % 16, y = ty * 16 + i / 16;
                float c[3] = {0.0f, 0.0f, 0.0f}, v[2] = {0.0f, 0.0f};
                if (x < w && y < h) {
                    const size_t p = (size_t)y * w + x;
                    for (int k = 0; k < 3; k++) c[k] = color[4 * p + k];
                    v[0] = velocity[2 * p]; v[1] = velocity[2 * p + 1];
                }
                lum[i] = ((c[0] + c[1]) + c[2]) * (1.0f / 3.0f);
                speed[i] = std::sqrt(v[0] * v[0] + v[1] * v[1]);
                lumSq[i] = lum[i] * lum[i];
            }
            float ss = 0.0f, ls = 0.0f, lq = 0.0f;
            for (int wp = 0; wp < 8; wp++) {   // SharedSums[0] += SharedSums[i], i = 1..7
                const float a = VrsButterfly(speed + 32 * wp), b = VrsButterfly(lum + 32 * wp), c = VrsButterfly(lumSq + 32 * wp);
                if (wp == 0) { ss = a; ls = b; lq = c; }
                else { ss += a; ls += b; lq += c; }
            }
            float meanSpeed = ss / 256.0f;
            meanSpeed /= f.DeltaRenderTime;
            const float luminanceMean = ls / 256.0f;
            uint32_t rate;
            float coeffOfVariation;
            if (luminanceMean <= 0.001f) {
                rate = 4u;
                coeffOfVariation = 0.0f;
            } else {
                const float luminanceSquaredMean = lq / 256.0f;
                const float variance = luminanceSquaredMean - luminanceMean * luminanceMean;
                const float stdDev = std::sqrt(variance);
                coeffOfVariation = stdDev / luminanceMean;
                const float velocityShadingRate = mixf(0.0f, 4.0f, meanSpeed * st.SpeedFactor);
                const float varianceShadingRate = mixf(0.0f, 4.0f, st.LumVarianceFactor / coeffOfVariation);
                const float combinedShadingRate = velocityShadingRate + varianceShadingRate;
                rate = std::min(VrsUint(VrsRoundEven(combinedShadingRate)), 4u);
            }
            const size_t t = (size_t)ty * tilesX + tx;
            rates[t] = (uint8_t)rate;
            if (debug) debug[t] = st.DebugMode == 2 ? meanSpeed : st.DebugMode == 3 ? luminanceMean : coeffOfVariation;
        }
}

// DeferredLighting/fragment.glsl at one sample: every G-buffer read at texel p (imgCoord), the NDC from uv. The statements are
// oracle_deferred.cpp's DeferredLighting loop body with (p, uv) as inputs instead of the pixel; that file stays as it is, and
// tests/test_vrs.py checks that rate 0 everywhere reproduces its image bit for bit.
static void DfShadeSample(const GpuPerFrameData& f, int shadowMode, const DfInputs& in, const std::vector<size_t>& offsets, size_t p,
                          float uvx, float uvy, const float* jitter, float* o) {
    const float depth = in.depth[p];
    if (depth == 1.0f) { o[0] = o[1] = o[2] = 0.0f; o[3] = 1.0f; return; }
    const vec3 ndc = V(uvx * 2.0f - 1.0f, uvy * 2.0f - 1.0f, depth);
    const vec3 fragPos = DfPerspective(f.InvProjView, ndc.x, ndc.y, ndc.z);
    const vec3 unjitteredFragPos = DfPerspective(f.InvProjView, ndc.x - jitter[0], ndc.y - jitter[1], ndc.z);
    const float ambientOcclusion = in.ssao ? (float)in.ssao[p] / 255.0f : 0.0f;
    DfSurface surface;
    surface.Albedo = V(in.albedo + 3 * p);
    surface.Normal = DecodeUnitVec(in.nrg[2 * p], in.nrg[2 * p + 1]);
    surface.Metallic = in.mr[2 * p];
    surface.Roughness = in.mr[2 * p + 1];
    surface.Emissive = V(in.emissive + 3 * p);
    surface.IOR = 1.0f;
    vec3 directLighting = V(0, 0, 0);
    for (uint64_t i = 0; i < in.lightCount; i++) {
        const GpuLight& light = in.lights[i];
        vec3 contribution = EvaluateLighting(light, surface, fragPos, V(f.ViewPos), ambientOcclusion);
        if (contribution.x != 0.0f || contribution.y != 0.0f || contribution.z != 0.0f) {
            const int k = light.PointShadowIndex;
            if (k == -1) {
            } else if (shadowMode == 1) {
                const vec3 lightToSample = unjitteredFragPos - V(light.Position);
                contribution = contribution * DfVisibility(in.shadows[k], in.sizes[k], in.texels + offsets[k], lightToSample);
            } else if (shadowMode == 2) {
                contribution = contribution * ((float)DfStoreR8(in.rt[k][p]) / 255.0f);
            }
        }
        directLighting = directLighting + contribution;
    }
    vec3 indirectLight;
    if (in.indirect) indirectLight = V(in.indirect + 4 * p) * surface.Albedo;
    else indirectLight = V(0.015f, 0.015f, 0.015f) * surface.Albedo;
    const vec3 c = (directLighting + indirectLight) + surface.Emissive;
    o[0] = c.x; o[1] = c.y; o[2] = c.z; o[3] = 1.0f;
}

static std::vector<size_t> DfShadowOffsets(const DfInputs& in) {
    std::vector<size_t> offsets(std::max(in.shadowCount, 0), 0);
    for (int i = 1; i < in.shadowCount; i++) offsets[i] = offsets[i - 1] + 6 * (size_t)in.sizes[i - 1] * (size_t)in.sizes[i - 1];
    return offsets;
}

// The draw under the rate image (NV_shading_rate_image): tile (x / 16, y / 16)'s palette entry gives cw x ch; fragments are
// aligned to multiples of (cw, ch); each runs the shader once at the centre of its area, uv = ((x0 + cw / 2) / W, ...) and
// imgCoord = (x0 + cw / 2, y0 + ch / 2) in integers, clamped to the image, and its result fills its in-image pixels.
static void DeferredLightingVrs(const GpuPerFrameData& f, int shadowMode, const DfInputs& in, int w, int h, const float* jitter,
                                const uint8_t* rates, float* out) {
    const std::vector<size_t> offsets = DfShadowOffsets(in);
    const int tilesX = (w + 15) / 16;
    for (int ty = 0; ty * 16 < h; ty++)
        for (int tx = 0; tx * 16 < w; tx++) {
            int cw, ch;
            VrsFragmentSize(rates[(size_t)ty * tilesX + tx], cw, ch);
            for (int y0 = ty * 16; y0 < std::min(ty * 16 + 16, h); y0 += ch)
                for (int x0 = tx * 16; x0 < std::min(tx * 16 + 16, w); x0 += cw) {
                    const int ix = std::min(x0 + cw / 2, w - 1), iy = std::min(y0 + ch / 2, h - 1);
                    const float uvx = ((float)x0 + 0.5f * (float)cw) / (float)w, uvy = ((float)y0 + 0.5f * (float)ch) / (float)h;
                    float c[4];
                    DfShadeSample(f, shadowMode, in, offsets, (size_t)iy * w + ix, uvx, uvy, jitter, c);
                    for (int y = y0; y < std::min(y0 + ch, h); y++)
                        for (int x = x0; x < std::min(x0 + cw, w); x++)
                            for (int k = 0; k < 4; k++) out[4 * ((size_t)y * w + x) + k] = c[k];
                }
        }
}

} // namespace

extern "C" {

// LightingShadingRateClassifier.Compute (idkpt_shading_rate): color rgba32f [h][w], velocity [h][w][2] -> rates
// [ceil(h/16)][ceil(w/16)] and, when debug is not null (DebugMode 2..4), the debug value per tile. Returns 0, or -1 for an
// argument the library rejects.
ORACLE_API int oracle_shading_rate(const GpuPerFrameData* frame, const IdkPtShadingRateSettings* st, const float* color, const float* velocity,
                                   int w, int h, uint8_t* rates, float* debug) {
    if (w < 1 || h < 1 || st->DebugMode < 0 || st->DebugMode > 4 || (debug && st->DebugMode < 2)) return -1;
    if (!std::isfinite(st->SpeedFactor) || !std::isfinite(st->LumVarianceFactor)) return -1;
    if (std::fegetround() != FE_TONEAREST) return -1;
    ShadingRate(*frame, *st, color, velocity, w, h, rates, debug);
    return 0;
}

// The deferred lighting draw under a rate image (idkpt_deferred_lighting with IsVariableRateShading): oracle_deferred_lighting's
// arguments plus rates [ceil(h/16)][ceil(w/16)] (palette indices 0..4). Returns 0, or -1 for an argument the library rejects.
ORACLE_API int oracle_deferred_lighting_vrs(const GpuLight* lights, uint64_t lightCount, const GpuPerFrameData* frame, int shadowMode,
                                            const GpuPointShadow* shadows, const int32_t* sizes, const uint16_t* texels, int shadowCount,
                                            const float* depth, const float* nrg, const float* albedo, const float* mr, const float* emissive,
                                            int w, int h, const float* jitter, const uint8_t* ssao, const float* indirect,
                                            const float* const* rt, int rtCount, const uint8_t* rates, float* out) {
    if (shadowMode < 0 || shadowMode > 2 || w < 1 || h < 1) return -1;
    if (shadowMode != 0)
        for (uint64_t i = 0; i < lightCount; i++)
            if (lights[i].PointShadowIndex != -1 && (lights[i].PointShadowIndex < 0 || lights[i].PointShadowIndex >= shadowCount)) return -1;
    if (shadowMode == 2 && rtCount < shadowCount) return -1;
    for (size_t t = 0; t < (size_t)((w + 15) / 16) * ((h + 15) / 16); t++)
        if (rates[t] > 4) return -1;
    const float noJitter[2] = {0.0f, 0.0f};
    const DfInputs in = {lights, lightCount, shadows, sizes, texels, shadowCount, depth, nrg, albedo, mr, emissive, ssao, indirect, rt};
    DeferredLightingVrs(*frame, shadowMode, in, w, h, jitter ? jitter : noJitter, rates, out);
    return 0;
}

// The fragment shader at n samples: imgCoord img[2 i], img[2 i + 1] (in the image) and uv uv[2 i], uv[2 i + 1], with
// oracle_deferred_lighting's scene and G-buffer arguments. out: n * 4 floats.
ORACLE_API int oracle_deferred_samples(const GpuLight* lights, uint64_t lightCount, const GpuPerFrameData* frame, int shadowMode,
                                       const GpuPointShadow* shadows, const int32_t* sizes, const uint16_t* texels, int shadowCount,
                                       const float* depth, const float* nrg, const float* albedo, const float* mr, const float* emissive,
                                       int w, int h, const float* jitter, const uint8_t* ssao, const float* indirect,
                                       const float* const* rt, int rtCount, const int32_t* img, const float* uv, uint64_t n, float* out) {
    if (shadowMode < 0 || shadowMode > 2 || w < 1 || h < 1 || (shadowMode == 2 && rtCount < shadowCount)) return -1;
    for (uint64_t i = 0; i < n; i++)
        if (img[2 * i] < 0 || img[2 * i] >= w || img[2 * i + 1] < 0 || img[2 * i + 1] >= h) return -1;
    const float noJitter[2] = {0.0f, 0.0f};
    const DfInputs in = {lights, lightCount, shadows, sizes, texels, shadowCount, depth, nrg, albedo, mr, emissive, ssao, indirect, rt};
    const std::vector<size_t> offsets = DfShadowOffsets(in);
    for (uint64_t i = 0; i < n; i++)
        DfShadeSample(*frame, shadowMode, in, offsets, (size_t)img[2 * i + 1] * w + img[2 * i], uv[2 * i], uv[2 * i + 1],
                      jitter ? jitter : noJitter, out + 4 * i);
    return 0;
}

} // extern "C"
