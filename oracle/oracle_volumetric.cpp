// ORACLE (TEST INFRASTRUCTURE ONLY) -- the volumetric lighting pass: a ray march through the point-shadow cube maps and its
// depth-aware upscale.
//
// Built as its own library (tests/volumetric_oracle.py -> oracle/liboracle_volumetric.so). It compiles
// oracle_point_shadows.cpp (and with it oracle.cpp) into the same translation unit and reuses its GetLogarithmicDepth, the
// det_exp / det_log2 polynomials and the present chain's PostTex / PostBilinear / half conversions unchanged; what it adds
// is restated here, including its own NEAREST cube-map lookup.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/VolumetricLight/compute.glsl             the march at the render size (Shadow(), UniformScatter(),
//                                                            ComputeScattering(), the 4x4 dither table)
//   Resource/Shaders/VolumetricLight/Upscale/compute.glsl     the depth-aware upscale to the presentation size
//   Source/Render/VolumetricLighting.cs:57-105                 dispatch sizes, texture formats and samplers
//   Resource/Shaders/include/Math.glsl:68-73, Pbr.glsl:9-17    LogarithmicDepthToLinearViewDepth, GetAttenuationFactor
//   Source/Render/CpuPointShadow.cs:220-230                    the shadow map's plain sampler (NEAREST, no compare)
//   OpenGL 4.6 spec 8.13 (table 8.19)                          cube-map face selection
#include "oracle_point_shadows.cpp"

namespace {

// ---- volumetric lighting (VolumetricLight/compute.glsl, VolumetricLight/Upscale/compute.glsl) -------------------------------

// Texel of texture(sampler, uv) along one axis of n texels with NEAREST filtering and clamp to edge; clamped in float, so a
// NaN coordinate gives texel 0.
static inline int VolNearest(float u, int n) { return (int)fminf(fmaxf(floorf(u * (float)n), 0.0f), (float)(n - 1)); }

// texture(samplerCube, dir).r with the shadow map's plain sampler (CpuPointShadow.cs:220-230: NEAREST, no compare): face and
// (s, t) per table 8.19 (major axis, ties x >= y >= z), texel clamp(floor(s * N), 0, N - 1); no seamless filtering under
// NEAREST. D16 reads as D / 65535.
static float CubeNearestDepth(const uint16_t* map, int size, vec3 d) {
    const float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
    int face;
    float sc, tc, ma;
    if (ax >= ay && ax >= az) { face = d.x >= 0.0f ? 0 : 1; sc = d.x >= 0.0f ? -d.z : d.z; tc = -d.y; ma = ax; }
    else if (ay >= az) { face = d.y >= 0.0f ? 2 : 3; sc = d.x; tc = d.y >= 0.0f ? d.z : -d.z; ma = ay; }
    else { face = d.z >= 0.0f ? 4 : 5; sc = d.z >= 0.0f ? d.x : -d.x; tc = -d.y; ma = az; }
    const float s = 0.5f * (sc / ma + 1.0f), t = 0.5f * (tc / ma + 1.0f);
    return (float)map[((size_t)face * size + VolNearest(t, size)) * size + VolNearest(s, size)] / 65535.0f;
}

static inline vec3 ExpNeg(const float* absorbance, float len) {   // exp(-Absorbance * len)
    return V(det_exp(-absorbance[0] * len), det_exp(-absorbance[1] * len), det_exp(-absorbance[2] * len));
}

// ComputeScattering: Henyey-Greenstein; pow(x, 1.5) = exp(log2(x) * ln2 * 1.5) like the present chain's pow
static inline float HenyeyGreenstein(float cosTheta, float g) {
    const float p = det_exp((det_log2(1.0f + g * g - 2.0f * g * cosTheta) * 0.69314718f) * 1.5f);
    return (1.0f - g * g) / (4.0f * PI_F * p);
}

// VolumetricLight/compute.glsl over the render size w x h: rgb (rounded through rgba16f) into `vol`, depth into `lowDepth`.
static void VolumetricMarch(const GpuLight* lights, const GpuPerFrameData& f, const IdkPtVolumetricSettings& st, const GpuPointShadow* shadows,
                            const int32_t* sizes, const uint16_t* texels, int count, const float* depth, int dw, int dh, const float* jitter,
                            PostTex& vol, std::vector<float>& lowDepth) {
    static const float Dither[4][4] = {{0.0f, 0.5f, 0.125f, 0.625f}, {0.75f, 0.22f, 0.875f, 0.375f},
                                       {0.1875f, 0.6875f, 0.0625f, 0.5625f}, {0.9375f, 0.4375f, 0.8125f, 0.3125f}};
    std::vector<size_t> offsets(std::max(count, 0), 0);
    for (int i = 1; i < count; i++) offsets[i] = offsets[i - 1] + 6 * (size_t)sizes[i - 1] * (size_t)sizes[i - 1];
    const int w = vol.w, h = vol.h;
    const vec3 viewPos = V(f.ViewPos);
    const float* m = f.InvProjView;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const float u = ((float)x + 0.5f) / (float)w, v = ((float)y + 0.5f) / (float)h;
            const float d = depth[(size_t)VolNearest(v, dh) * dw + VolNearest(u, dw)];
            const float nx = (u * 2.0f - 1.0f) - jitter[0], ny = (v * 2.0f - 1.0f) - jitter[1];
            const float wx = ((m[0] * nx + m[4] * ny) + m[8] * d) + m[12] * 1.0f;
            const float wy = ((m[1] * nx + m[5] * ny) + m[9] * d) + m[13] * 1.0f;
            const float wz = ((m[2] * nx + m[6] * ny) + m[10] * d) + m[14] * 1.0f;
            const float ww = ((m[3] * nx + m[7] * ny) + m[11] * d) + m[15] * 1.0f;
            vec3 viewToFrag = V(wx / ww, wy / ww, wz / ww) - viewPos;
            const float viewToFragLen = sqrtf(dot(viewToFrag, viewToFrag));
            const vec3 viewDir = viewToFrag / viewToFragLen;
            if (viewToFragLen > st.MaxDist) viewToFrag = viewDir * st.MaxDist;
            const vec3 deltaStep = viewToFrag / (float)st.SampleCount;
            const vec3 origin = viewPos + deltaStep * Dither[x % 4][y % 4];
            vec3 scattered = V(0, 0, 0);
            for (int i = 0; i < count; i++) {   // UniformScatter
                const GpuPointShadow& ps = shadows[i];
                const GpuLight& light = lights[ps.LightIndex];
                const uint16_t* map = texels + offsets[i];
                vec3 sum = V(0, 0, 0);
                vec3 samplePoint = origin;
                for (int k = 0; k < st.SampleCount; k++) {
                    const vec3 lightToSample = samplePoint - V(light.Position);
                    const float dist = fmaxf(fabsf(lightToSample.x), fmaxf(fabsf(lightToSample.y), fabsf(lightToSample.z)));
                    const bool shadowed = GetLogarithmicDepth(ps.NearPlane, ps.FarPlane, dist) > CubeNearestDepth(map, sizes[i], lightToSample);
                    if (!shadowed) {
                        const float lengthToLight = sqrtf(dot(lightToSample, lightToSample));
                        const float lr = fmaxf(light.Radius, 0.0001f), dsq = fmaxf(lengthToLight * lengthToLight, 0.0001f);
                        const float attenuation = (lr * lr) / dsq;
                        const vec3 absorbed = ExpNeg(st.Absorbance, lengthToLight);
                        const vec3 lightDir = lightToSample / lengthToLight;
                        const float cosTheta = dot(lightDir, -viewDir);
                        sum = sum + ((V(light.Color) * HenyeyGreenstein(cosTheta, st.Scattering)) * attenuation) * absorbed;
                    }
                    samplePoint = samplePoint + deltaStep;
                }
                sum = sum / (float)st.SampleCount;
                const vec3 e = origin - samplePoint;
                sum = sum * ExpNeg(st.Absorbance, sqrtf(dot(e, e)));
                scattered = scattered + sum;
            }
            StoreHalf(vol, x, y, scattered * st.Strength);
            lowDepth[(size_t)y * w + x] = d;
        }
}

// LogarithmicDepthToLinearViewDepth (Math.glsl:68-73) / FarPlane
static inline float VolLinearDepth(float n, float f, float z) { return ((2.0f * n) * f) / ((f + n) - z * (f - n)) / f; }

// VolumetricLight/Upscale/compute.glsl: W x H rgba16f (alpha 1) from the render-size image and depth.
static void VolumetricUpscale(const GpuPerFrameData& f, const float* depth, int dw, int dh, const PostTex& vol, const std::vector<float>& lowDepth,
                              int W, int H, uint16_t* out) {
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            const float u = ((float)x + 0.5f) / (float)W, v = ((float)y + 0.5f) / (float)H;
            const float high = VolLinearDepth(f.NearPlane, f.FarPlane, depth[(size_t)VolNearest(v, dh) * dw + VolNearest(u, dw)]);
            const int xo = x % 2 == 0 ? -1 : 1, yo = y % 2 == 0 ? -1 : 1;
            const int offsets[4][2] = {{0, 0}, {0, yo}, {xo, 0}, {xo, yo}};
            vec3 color = V(0, 0, 0);
            float totalWeight = 0.0f;
            for (int i = 0; i < 4; i++) {
                const float su = ((float)(x + offsets[i][0]) + 0.5f) / (float)W, sv = ((float)(y + offsets[i][1]) + 0.5f) / (float)H;
                const vec3 c = PostBilinear(vol, su, sv, 0, 0);
                const float low = VolLinearDepth(f.NearPlane, f.FarPlane, lowDepth[(size_t)VolNearest(sv, vol.h) * vol.w + VolNearest(su, vol.w)]);
                const float wt = fmaxf(1.0f - 0.05f * fabsf(low - high), 0.0f);
                color = color + c * wt;
                totalWeight = totalWeight + wt;
            }
            color = color / (totalWeight + 0.0001f);
            uint16_t* o = out + 4 * ((size_t)y * W + x);
            o[0] = f32_to_f16(color.x); o[1] = f32_to_f16(color.y); o[2] = f32_to_f16(color.z); o[3] = f32_to_f16(1.0f);
        }
}

} // namespace

extern "C" {

// VolumetricLighting.Compute (idkpt_volumetric_lighting): `count` shadows with their face sizes and maps back to back, lights
// indexed by each shadow's LightIndex (must be < lightCount). out: W*H*4 halves. march (w*h*4 halves) and marchDepth (w*h)
// receive the render-size images when not null. Returns 0, or -1 for an argument the library rejects.
ORACLE_API int oracle_volumetric_lighting(const GpuLight* lights, uint64_t lightCount, const GpuPerFrameData* frame, const IdkPtVolumetricSettings* st,
                                          const GpuPointShadow* shadows, const int32_t* sizes, const uint16_t* texels, int count,
                                          const float* depth, int dw, int dh, int W, int H, const float* jitter, uint16_t* out,
                                          uint16_t* march, float* marchDepth) {
    if (st->SampleCount < 1 || !(st->ResolutionScale > 0.0f && st->ResolutionScale <= 1.0f)) return -1;
    for (int i = 0; i < count; i++)
        if (shadows[i].LightIndex < 0 || (uint64_t)shadows[i].LightIndex >= lightCount) return -1;
    const float noJitter[2] = {0.0f, 0.0f};
    PostTex vol;
    vol.w = (int)((float)W * st->ResolutionScale); vol.h = (int)((float)H * st->ResolutionScale);
    if (vol.w < 1 || vol.h < 1) return -1;
    vol.px.assign(3 * (size_t)vol.w * vol.h, 0.0f);
    std::vector<float> lowDepth((size_t)vol.w * vol.h);
    VolumetricMarch(lights, *frame, *st, shadows, sizes, texels, count, depth, dw, dh, jitter ? jitter : noJitter, vol, lowDepth);
    VolumetricUpscale(*frame, depth, dw, dh, vol, lowDepth, W, H, out);
    for (size_t i = 0; march && i < (size_t)vol.w * vol.h; i++) {
        for (int c = 0; c < 3; c++) march[4 * i + c] = f32_to_f16(vol.px[3 * i + c]);
        march[4 * i + 3] = f32_to_f16(1.0f);
    }
    if (marchDepth) memcpy(marchDepth, lowDepth.data(), lowDepth.size() * 4);
    return 0;
}

// The volumetric pass's NEAREST cube lookup on its own, for n directions into one map.
ORACLE_API void oracle_cube_nearest(const uint16_t* map, int size, const float* dirs, uint64_t n, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = CubeNearestDepth(map, size, V(dirs + 3 * i));
}

// The upscale dispatch on its own: render-size rgba16f `march` and r32f `marchDepth` (w x h) to W x H halves.
ORACLE_API void oracle_volumetric_upscale(const GpuPerFrameData* frame, const float* depth, int dw, int dh, const uint16_t* march,
                                          const float* marchDepth, int w, int h, int W, int H, uint16_t* out) {
    PostTex vol;
    vol.w = w; vol.h = h;
    vol.px.resize(3 * (size_t)w * h);
    for (size_t i = 0; i < (size_t)w * h; i++)
        for (int c = 0; c < 3; c++) vol.px[3 * i + c] = f16_to_f32(march[4 * i + c]);
    VolumetricUpscale(*frame, depth, dw, dh, vol, std::vector<float>(marchDepth, marchDepth + (size_t)w * h), W, H, out);
}

} // extern "C"
