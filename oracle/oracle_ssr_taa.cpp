// ORACLE (TEST INFRASTRUCTURE ONLY) -- the end of the raster frame: screen-space reflections, the lighting merge and one TAA
// resolve step.
//
// Built as its own library (tests/ssr_taa_oracle.py -> oracle/liboracle_ssr_taa.so). It compiles oracle_deferred.cpp (and
// with it oracle_point_shadows.cpp and oracle.cpp) into the same translation unit and reuses SampleSky, PostBilinear /
// PostTex, the rgba16f conversions, DfPerspective, DfNearest, DecodeUnitVec, normalize, reflect, mixf and fractf unchanged;
// what it adds is restated here from the shaders. The TAA history is the caller's: each call is one resolve step.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/SSR/compute.glsl                 SSR, BinarySearch; Source/Render/SSR.cs (settings, rgba16f, LINEAR)
//   Resource/Shaders/MergeTextures/compute.glsl       the merge of the lit image and SSR
//   Resource/Shaders/TAAResolve/compute.glsl          the resolve, GetResolveData, SampleTextureCatmullRom;
//                                                      Source/Render/TAAResolve.cs (rgba16f ping-pong, LINEAR, clamp to edge)
//   Source/Render/RasterPipeline.cs:672-676            the velocity texture (R16G16F, NEAREST)
#include "oracle_deferred.cpp"

namespace {

// min, max and clamp in the one form DESIGN.md 8f.1e states
static inline float TaMin(float x, float y) { return y < x ? y : x; }
static inline float TaMax(float x, float y) { return y > x ? y : x; }
static inline float TaClamp(float x, float lo, float hi) { return TaMin(TaMax(x, lo), hi); }

// An rgba32f image as the PostTex of its rgb
static PostTex TaFromRgba32f(const float* px, int w, int h) {
    PostTex t;
    t.w = w; t.h = h; t.px.resize((size_t)w * h * 3);
    for (size_t i = 0; i < (size_t)w * h; i++)
        for (int c = 0; c < 3; c++) t.px[3 * i + c] = px[4 * i + c];
    return t;
}

// An rgba16f image as the PostTex of its rgb
static PostTex TaFromRgba16f(const uint16_t* px, int w, int h) {
    PostTex t;
    t.w = w; t.h = h; t.px.resize((size_t)w * h * 3);
    for (size_t i = 0; i < (size_t)w * h; i++)
        for (int c = 0; c < 3; c++) t.px[3 * i + c] = f16_to_f32(px[4 * i + c]);
    return t;
}

static inline void TaStoreHalf(uint16_t* o, vec3 c, float alpha) {
    o[0] = f32_to_f16(c.x); o[1] = f32_to_f16(c.y); o[2] = f32_to_f16(c.z); o[3] = f32_to_f16(alpha);
}

struct SsrInputs {
    const GpuPerFrameData* f;
    const IdkPtSsrSettings* st;
    const IdkPtSkyDesc* sky;
    const float *depth, *nrg, *albedo, *mr;
    const PostTex* src;
    int w, h;
};

// PerspectiveTransform(p, Projection), xy * 0.5 + 0.5
static inline vec3 SsrProject(const float* m, vec3 p) {
    vec3 q = DfPerspective(m, p.x, p.y, p.z);
    q.x = q.x * 0.5f + 0.5f;
    q.y = q.y * 0.5f + 0.5f;
    return q;
}

static inline float SsrDepth(const SsrInputs& in, vec3 q) {
    return in.depth[(size_t)DfNearest(q.y, in.h) * in.w + DfNearest(q.x, in.w)];
}

// BinarySearch(samplePoint, deltaStep, inout projectedSample)
static void SsrBinarySearch(const SsrInputs& in, vec3 samplePoint, vec3 deltaStep, vec3& projectedSample) {
    deltaStep = deltaStep * 0.5f;
    samplePoint = samplePoint - deltaStep * 0.5f;
    for (int i = 1; i < in.st->BinarySearchCount; i++) {
        projectedSample = SsrProject(in.f->Projection, samplePoint);
        const float depth = SsrDepth(in, projectedSample);
        deltaStep = deltaStep * 0.5f;
        if (projectedSample.z > depth) samplePoint = samplePoint - deltaStep;
        else samplePoint = samplePoint + deltaStep;
    }
}

// SSR(normal, fragPos)
static vec3 SsrTrace(const SsrInputs& in, vec3 normal, vec3 fragPos) {
    const vec3 reflectDir = reflect(normalize(fragPos), normal);
    const vec3 maxReflectPoint = fragPos + reflectDir * in.st->MaxDist;
    const vec3 deltaStep = (maxReflectPoint - fragPos) / (float)in.st->SampleCount;
    vec3 samplePoint = fragPos;
    for (int i = 0; i < in.st->SampleCount; i++) {
        samplePoint = samplePoint + deltaStep;
        vec3 projectedSample = SsrProject(in.f->Projection, samplePoint);
        if (projectedSample.x >= 1.0f || projectedSample.y >= 1.0f || projectedSample.x < 0.0f || projectedSample.y < 0.0f ||
            projectedSample.z > 1.0f)
            return V(0.0f, 0.0f, 0.0f);
        const float depth = SsrDepth(in, projectedSample);
        if (projectedSample.z > depth) {
            SsrBinarySearch(in, samplePoint, deltaStep, projectedSample);
            return PostBilinear(*in.src, projectedSample.x, projectedSample.y, 0, 0);
        }
    }
    const float* m = in.f->InvView;
    const vec3 r = reflectDir;
    const vec3 world = V(((m[0] * r.x + m[4] * r.y) + m[8] * r.z) + m[12] * 0.0f, ((m[1] * r.x + m[5] * r.y) + m[9] * r.z) + m[13] * 0.0f,
                         ((m[2] * r.x + m[6] * r.y) + m[10] * r.z) + m[14] * 0.0f);
    const float* faces[6];
    for (int i = 0; i < 6; i++) faces[i] = in.sky->Faces[i];
    return SampleSky(faces, in.sky->FaceSize, in.sky->Color, world);
}

// SSR/compute.glsl into rgba16f, then MergeTextures/compute.glsl into rgba32f
static void Ssr(const SsrInputs& in, const float* srcRgba, uint16_t* ssrOut, float* mergedOut) {
    for (int y = 0; y < in.h; y++)
        for (int x = 0; x < in.w; x++) {
            const size_t p = (size_t)y * in.w + x;
            uint16_t* o = ssrOut + 4 * p;
            const float specular = in.mr[2 * p];
            const float depth = in.depth[p];
            if (specular < 0.001f || depth == 1.0f) {
                TaStoreHalf(o, V(0.0f, 0.0f, 0.0f), 0.0f);
            } else {
                const float uvx = ((float)x + 0.5f) / (float)in.w, uvy = ((float)y + 0.5f) / (float)in.h;
                const vec3 fragPos = DfPerspective(in.f->InvProjection, uvx * 2.0f - 1.0f, uvy * 2.0f - 1.0f, depth);
                const vec3 n = DecodeUnitVec(in.nrg[2 * p], in.nrg[2 * p + 1]);
                const float* m = in.f->InvView;   // mat3(transpose(InvView)): row i of the upper 3x3 is column i of InvView
                const vec3 normal = V((m[0] * n.x + m[1] * n.y) + m[2] * n.z, (m[4] * n.x + m[5] * n.y) + m[6] * n.z,
                                      (m[8] * n.x + m[9] * n.y) + m[10] * n.z);
                vec3 color = SsrTrace(in, normal, fragPos) * specular;
                color = color * V(in.albedo + 3 * p);
                TaStoreHalf(o, color, 1.0f);
            }
            float* mo = mergedOut + 4 * p;
            for (int c = 0; c < 3; c++) mo[c] = srcRgba[4 * p + c] + f16_to_f32(o[c]);
            mo[3] = 1.0f;
        }
}

// SampleTextureCatmullRom, one axis' weights and positions
struct CrAxis { float w0, w12, w3, t0, t12, t3; };
static CrAxis CatmullRomAxis(float uv, int size) {
    const float texelSize = 1.0f / (float)size;
    const float samplePos = uv / texelSize;
    const float texPos1 = floorf(samplePos - 0.5f) + 0.5f;
    const float f = samplePos - texPos1;
    const float w0 = f * (-0.5f + f * (1.0f - 0.5f * f));
    const float w1 = 1.0f + f * f * (-2.5f + 1.5f * f);
    const float w2 = f * (0.5f + f * (2.0f - 1.5f * f));
    const float w3 = f * f * (-0.5f + 0.5f * f);
    const float w12 = w1 + w2;
    const float offset12 = w2 / (w1 + w2);
    float texPos0 = texPos1 - 1.0f, texPos3 = texPos1 + 2.0f, texPos12 = texPos1 + offset12;
    texPos0 *= texelSize; texPos3 *= texelSize; texPos12 *= texelSize;
    return {w0, w12, w3, texPos0, texPos12, texPos3};
}

static vec3 SampleTextureCatmullRom(const PostTex& src, float u, float v) {
    const CrAxis X = CatmullRomAxis(u, src.w), Y = CatmullRomAxis(v, src.h);
    vec3 result = PostBilinear(src, X.t0, Y.t0, 0, 0) * X.w0 * Y.w0;
    result = result + PostBilinear(src, X.t12, Y.t0, 0, 0) * X.w12 * Y.w0;
    result = result + PostBilinear(src, X.t3, Y.t0, 0, 0) * X.w3 * Y.w0;
    result = result + PostBilinear(src, X.t0, Y.t12, 0, 0) * X.w0 * Y.w12;
    result = result + PostBilinear(src, X.t12, Y.t12, 0, 0) * X.w12 * Y.w12;
    result = result + PostBilinear(src, X.t3, Y.t12, 0, 0) * X.w3 * Y.w12;
    result = result + PostBilinear(src, X.t0, Y.t3, 0, 0) * X.w0 * Y.w3;
    result = result + PostBilinear(src, X.t12, Y.t3, 0, 0) * X.w12 * Y.w3;
    result = result + PostBilinear(src, X.t3, Y.t3, 0, 0) * X.w3 * Y.w3;
    return result;
}

// TAAResolve/compute.glsl at W x H: color, depth and velocity at rw x rh, history rgba16f at W x H. rgb only: alpha is 1 on
// every path (DESIGN.md 8f.1e).
static void TaaResolve(const IdkPtTaaSettings& st, const PostTex& color, const float* depth, const float* velocity, int rw, int rh,
                       const PostTex& history, int W, int H, uint16_t* out) {
    auto nearest = [&](float u, float v) { return (size_t)DfNearest(v, rh) * rw + DfNearest(u, rw); };
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            uint16_t* o = out + 4 * ((size_t)y * W + x);
            const float uvx = ((float)x + 0.5f) / (float)W, uvy = ((float)y + 0.5f) / (float)H;
            if (st.IsNaiveTaa) {
                const size_t k = nearest(uvx, uvy);
                const float hx = uvx - velocity[2 * k], hy = uvy - velocity[2 * k + 1];
                const vec3 currentColor = PostBilinear(color, uvx, uvy, 0, 0);
                const vec3 historyColor = PostBilinear(history, hx, hy, 0, 0);
                const float blend = 1.0f / (float)st.SampleCount;
                TaStoreHalf(o, mix(historyColor, currentColor, blend), 1.0f);
                continue;
            }
            // GetResolveData
            float minDepth = 3.4028235e+38f;
            vec3 nMin = V(3.4028235e+38f, 3.4028235e+38f, 3.4028235e+38f), nMax = V(-3.4028235e+38f, -3.4028235e+38f, -3.4028235e+38f);
            vec3 currentColor = V(0.0f, 0.0f, 0.0f);
            float bestX = uvx, bestY = uvy;      // undefined in GLSL when no depth is below FLOAT_MAX; the pixel's own uv here
            for (int dy = -1; dy <= 1; dy++)
                for (int dx = -1; dx <= 1; dx++) {
                    const float nx = ((float)(x + dx) + 0.5f) / (float)W, ny = ((float)(y + dy) + 0.5f) / (float)H;
                    const vec3 c = PostBilinear(color, nx, ny, 0, 0);
                    nMin = V(TaMin(nMin.x, c.x), TaMin(nMin.y, c.y), TaMin(nMin.z, c.z));
                    nMax = V(TaMax(nMax.x, c.x), TaMax(nMax.y, c.y), TaMax(nMax.z, c.z));
                    const float inputDepth = depth[nearest(nx, ny)];
                    if (inputDepth < minDepth) { minDepth = inputDepth; bestX = nx; bestY = ny; }
                    if (dx == 0 && dy == 0) currentColor = c;
                }
            const size_t k = nearest(bestX, bestY);
            const float hx = uvx - velocity[2 * k], hy = uvy - velocity[2 * k + 1];
            if (hx >= 1.0f || hy >= 1.0f || hx < 0.0f || hy < 0.0f) {
                TaStoreHalf(o, currentColor, 1.0f);
                continue;
            }
            vec3 historyColor = SampleTextureCatmullRom(history, hx, hy);
            historyColor = V(TaClamp(historyColor.x, nMin.x, nMax.x), TaClamp(historyColor.y, nMin.y, nMax.y), TaClamp(historyColor.z, nMin.z, nMax.z));
            float blend = 1.0f / (float)st.SampleCount;
            const float lx = fractf(hx * (float)history.w), ly = fractf(hy * (float)history.h);
            const float pixelCenterDistance = fabsf(0.5f - lx) + fabsf(0.5f - ly);
            blend = mixf(blend, 1.0f, pixelCenterDistance * st.PreferAliasingOverBlur);
            TaStoreHalf(o, mix(historyColor, currentColor, blend), 1.0f);
        }
}

} // namespace

extern "C" {

// SSR.Compute + Merge Textures (idkpt_ssr): G-buffer (depth [h][w], normal [h][w][2], albedo [h][w][3], metallic/roughness
// [h][w][2]), source rgba32f [h][w], the sky -> ssr rgba16f [h][w][4] (raw halves) and merged rgba32f [h][w][4]. Returns 0,
// or -1 for an argument the library rejects.
ORACLE_API int oracle_ssr(const GpuPerFrameData* frame, const IdkPtSsrSettings* st, const IdkPtSkyDesc* sky, const float* depth, const float* nrg,
                          const float* albedo, const float* mr, const float* src, int w, int h, uint16_t* ssrOut, float* mergedOut) {
    if (st->SampleCount < 1 || st->SampleCount > 1024 || st->BinarySearchCount < 0 || st->BinarySearchCount > 64 || !std::isfinite(st->MaxDist) ||
        w < 1 || h < 1)
        return -1;
    const PostTex s = TaFromRgba32f(src, w, h);
    const SsrInputs in = {frame, st, sky, depth, nrg, albedo, mr, &s, w, h};
    Ssr(in, src, ssrOut, mergedOut);
    return 0;
}

// One TaaResolve.Compute step (idkpt_taa_resolve): colour rgba32f, depth, velocity [rh][rw][2] at the render size, history
// rgba16f [H][W][4] (raw halves, the previous step's output) -> out rgba16f [H][W][4]. Returns 0, or -1 for an argument the
// library rejects.
ORACLE_API int oracle_taa_resolve(const IdkPtTaaSettings* st, const float* color, const float* depth, const float* velocity, int rw, int rh,
                                  const uint16_t* history, int W, int H, uint16_t* out) {
    if ((st->IsNaiveTaa != 0 && st->IsNaiveTaa != 1) || st->SampleCount < 1 || st->SampleCount > 1024 || rw < 1 || rh < 1 || W < 1 || H < 1)
        return -1;
    const PostTex c = TaFromRgba32f(color, rw, rh), hist = TaFromRgba16f(history, W, H);
    TaaResolve(*st, c, depth, velocity, rw, rh, hist, W, H, out);
    return 0;
}

} // extern "C"
