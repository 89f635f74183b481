// ORACLE (TEST INFRASTRUCTURE ONLY) -- the sky cube map generated on the device: atmospheric scattering and the
// equirectangular import.
//
// Built as its own library (tests/sky_oracle.py -> oracle/liboracle_sky.so). It compiles oracle.cpp into the same translation
// unit and reuses its normalize, det_sincos / det_exp / det_log2 polynomials and the half conversion unchanged; the two
// shaders, GetWorldSpaceDirection and the atan2 / asin polynomials are restated here.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/AtmosphericScattering/compute.glsl        main, Rsi, Atmosphere
//   Resource/Shaders/UnprojectEquirectangular/compute.glsl     main, SampleSphericalMap, SrgbToLinear
//   Resource/Shaders/include/Math.glsl:17-39,139-153           GetWorldSpaceDirection(ndc, face), PolarToCartesian
//   Source/Render/AtmosphericScatterer.cs:9-49                 the settings, LightIntensity = max(LightIntensity, 0)
//   Source/Render/SkyBoxManager.cs:115-146                     face size Width / 4, the RGB16F source, the RGBA16F faces
//   OpenGL 4.6 spec 8.14.2                                     LINEAR filtering with REPEAT on the texel indices
//
// DESIGN.md 8f.1j pins the rules.
#include "oracle.cpp"

namespace {

// atan on [0, 1]: around pi/4 above tan(pi/8), then t + t^3 P(t^2) (Cephes atanf).
float SkyAtan01(float t) {
    float base = 0.0f;
    if (t > 0.41421356f) {
        t = (t - 1.0f) / (t + 1.0f);
        base = 0.78539816f;
    }
    const float z = t * t;
    const float poly = (((8.05374449538e-2f * z - 1.38776856032e-1f) * z + 1.99777106478e-1f) * z - 3.33329491539e-1f) * z * t;
    return base + (poly + t);
}

// atan2 with C's signed-zero cases; NaN in, NaN out.
float SkyAtan2(float y, float x) {
    if (std::isnan(x) || std::isnan(y)) return x + y;
    const float ax = std::fabs(x), ay = std::fabs(y);
    float a = 0.0f;
    if (ay != 0.0f) a = ay <= ax ? SkyAtan01(ay / ax) : 1.57079637f - SkyAtan01(ax / ay);
    if (std::signbit(x)) a = 3.14159274f - a;
    return std::copysign(a, y);
}

// asin (Cephes asinf); |x| > 1 gives the NaN 0x7fffffff.
float SkyAsin(float x) {
    const float a = std::fabs(x);
    if (a > 1.0f) { const uint32_t bits = 0x7fffffffu; float nan; memcpy(&nan, &bits, 4); return nan; }
    if (a < 1e-4f) return x;
    const bool upper = a > 0.5f;
    const float z = upper ? 0.5f * (1.0f - a) : a * a;
    const float s = upper ? sqrtf(z) : a;
    float r = ((((4.2163199048e-2f * z + 2.4181311049e-2f) * z + 4.5470025998e-2f) * z + 7.4953002686e-2f) * z + 1.6666752422e-1f) * z * s + s;
    if (upper) r = 1.57079637f - (r + r);
    return std::copysign(r, x);
}

// GetWorldSpaceDirection(ndc, face) of texel (x, y) of an n x n face.
vec3 SkyTexelDir(int n, int face, int x, int y) {
    const float ndcX = ((float)x + 0.5f) / (float)n * 2.0f - 1.0f;
    const float ndcY = ((float)y + 0.5f) / (float)n * 2.0f - 1.0f;
    static const float table[6][3][3] = {   // rows: the x, y, z of the direction as (constant, ndcX, ndcY) coefficients
        {{1, 0, 0}, {0, 0, -1}, {0, -1, 0}}, {{-1, 0, 0}, {0, 0, -1}, {0, 1, 0}}, {{0, 1, 0}, {1, 0, 0}, {0, 0, 1}},
        {{0, 1, 0}, {-1, 0, 0}, {0, 0, -1}}, {{0, 1, 0}, {0, 0, -1}, {1, 0, 0}}, {{0, -1, 0}, {0, 0, -1}, {-1, 0, 0}}};
    float c[3];
    for (int k = 0; k < 3; k++) {
        const float* t = table[face][k];
        c[k] = t[0] != 0.0f ? t[0] : t[1] != 0.0f ? t[1] * ndcX : t[2] * ndcY;
    }
    return normalize(V(c[0], c[1], c[2]));
}

struct Hit2 { float x, y; };

Hit2 Rsi(vec3 r0, vec3 rd, float sr) {
    const float a = dot(rd, rd);
    const float b = 2.0f * dot(rd, r0);
    const float c = dot(r0, r0) - sr * sr;
    const float d = b * b - 4.0f * a * c;
    if (d < 0.0f) return {1e5f, -1e5f};
    return {(-b - sqrtf(d)) / (2.0f * a), (-b + sqrtf(d)) / (2.0f * a)};
}

inline float Length(vec3 v) { return sqrtf(dot(v, v)); }

vec3 Atmosphere(vec3 r, vec3 r0, vec3 pSun, float iSun, float rPlanet, float rAtmos, vec3 kRlh, float kMie, float shRlh, float shMie,
                float g, int iSteps, int jSteps) {
    pSun = normalize(pSun);
    r = normalize(r);
    Hit2 p = Rsi(r0, r, rAtmos);
    if (p.x > p.y) return V(0.0f, 0.0f, 0.0f);
    p.y = fminf(p.y, Rsi(r0, r, rPlanet).x);
    const float iStepSize = (p.y - p.x) / (float)iSteps;
    float iTime = 0.0f;
    vec3 totalRlh = V(0.0f, 0.0f, 0.0f), totalMie = V(0.0f, 0.0f, 0.0f);
    float iOdRlh = 0.0f, iOdMie = 0.0f;
    const float mu = dot(r, pSun);
    const float mumu = mu * mu;
    const float gg = g * g;
    const float pRlh = 3.0f / (16.0f * PI_F) * (1.0f + mumu);
    const float pw = det_exp((det_log2(1.0f + gg - 2.0f * mu * g) * 0.69314718f) * 1.5f);   // pow(., 1.5)
    const float pMie = 3.0f / (8.0f * PI_F) * ((1.0f - gg) * (mumu + 1.0f)) / (pw * (2.0f + gg));
    for (int i = 0; i < iSteps; i++) {
        const vec3 iPos = r0 + r * (iTime + iStepSize * 0.5f);
        const float iHeight = Length(iPos) - rPlanet;
        const float odStepRlh = det_exp(-iHeight / shRlh) * iStepSize;
        const float odStepMie = det_exp(-iHeight / shMie) * iStepSize;
        iOdRlh += odStepRlh;
        iOdMie += odStepMie;
        const float jStepSize = Rsi(iPos, pSun, rAtmos).y / (float)jSteps;
        float jTime = 0.0f, jOdRlh = 0.0f, jOdMie = 0.0f;
        for (int j = 0; j < jSteps; j++) {
            const vec3 jPos = iPos + pSun * (jTime + jStepSize * 0.5f);
            const float jHeight = Length(jPos) - rPlanet;
            jOdRlh += det_exp(-jHeight / shRlh) * jStepSize;
            jOdMie += det_exp(-jHeight / shMie) * jStepSize;
            jTime += jStepSize;
        }
        const float m = kMie * (iOdMie + jOdMie);
        const vec3 rl = kRlh * (iOdRlh + jOdRlh);
        const vec3 attn = V(det_exp(-(m + rl.x)), det_exp(-(m + rl.y)), det_exp(-(m + rl.z)));
        totalRlh = totalRlh + attn * odStepRlh;
        totalMie = totalMie + attn * odStepMie;
        iTime += iStepSize;
    }
    return (kRlh * pRlh * totalRlh + totalMie * (pMie * kMie)) * iSun;
}

// SrgbToLinear of one channel; NaN passes through.
float SrgbToLinear(float s) {
    if (std::isnan(s)) return s;
    const float lower = s / 12.92f;
    const float higher = det_exp((det_log2((s + 0.055f) / 1.055f) * 0.69314718f) * 2.4f);
    return s < 0.04045f ? lower : higher;
}

int Repeat(int i, int n) { const int m = i % n; return m < 0 ? m + n : m; }

} // namespace

extern "C" {

// AtmosphericScatterer.Compute into faces [6][n][n][4].
ORACLE_API int oracle_sky_atmosphere(const IdkPtAtmosphereSettings* s, int n, float* faces, int threads) {
    if (!s || !faces || n < 1 || s->ISteps < 1 || s->JSteps < 1) return 1;
    const float iSun = fmaxf(s->LightIntensity, 0.0f);
    float sinTheta, cosTheta, sinPhi, cosPhi;
    det_sincos(s->Elevation, &sinTheta, &cosTheta);
    det_sincos(s->Azimuth, &sinPhi, &cosPhi);
    const vec3 lightPos = V(sinTheta * cosPhi, cosTheta, sinTheta * sinPhi) * 1.0f;
    parallel_for((size_t)6 * n * n, threads, [&](size_t begin, size_t end, int) {
        for (size_t t = begin; t < end; t++) {
            const int face = (int)(t / ((size_t)n * n)), y = (int)(t / n % n), x = (int)(t % n);
            const vec3 c = Atmosphere(SkyTexelDir(n, face, x, y), V(0.0f, 6376e3f, 0.0f), lightPos, iSun, 6371e3f, 6471e3f,
                                      V(5.5e-6f, 13.0e-6f, 22.4e-6f), 21e-6f, 8e3f, 1.2e3f, 0.758f, s->ISteps, s->JSteps);
            float* o = faces + 4 * t;
            o[0] = c.x; o[1] = c.y; o[2] = c.z; o[3] = 1.0f;
        }
    });
    return 0;
}

// LoadSkyBoxEquirectangular: rgb [h][w][3] -> faces [6][w/4][w/4][4].
ORACLE_API int oracle_sky_equirect(const float* rgb, int w, int h, float* faces, int threads) {
    if (!rgb || !faces || w < 4 || h < 1) return 1;
    const int n = w / 4;
    std::vector<float> src((size_t)w * h * 3);   // the RGB16F texture
    for (size_t i = 0; i < src.size(); i++) src[i] = to_half_and_back(rgb[i]);
    parallel_for((size_t)6 * n * n, threads, [&](size_t begin, size_t end, int) {
        for (size_t t = begin; t < end; t++) {
            const int face = (int)(t / ((size_t)n * n)), y = (int)(t / n % n), x = (int)(t % n);
            const vec3 v = SkyTexelDir(n, face, x, y);
            const float u = SkyAtan2(v.z, v.x) * 0.1591f + 0.5f;
            const float tv = SkyAsin(v.y) * 0.3183f + 0.5f;
            const float px = u * (float)w - 0.5f, py = tv * (float)h - 0.5f;
            const float i0 = floorf(px), j0 = floorf(py);
            const float a = px - i0, b = py - j0;
            const int xs[2] = {Repeat((int)i0, w), Repeat((int)i0 + 1, w)}, ys[2] = {Repeat((int)j0, h), Repeat((int)j0 + 1, h)};
            float* o = faces + 4 * t;
            for (int c = 0; c < 3; c++) {
                float tex[2][2];
                for (int j = 0; j < 2; j++)
                    for (int i = 0; i < 2; i++) tex[j][i] = src[((size_t)ys[j] * w + xs[i]) * 3 + c];
                const float row0 = tex[0][0] * (1.0f - a) + tex[0][1] * a;
                const float row1 = tex[1][0] * (1.0f - a) + tex[1][1] * a;
                o[c] = to_half_and_back(SrgbToLinear(row0 * (1.0f - b) + row1 * b));
            }
            o[3] = 1.0f;
        }
    });
    return 0;
}

// The texel directions of an n x n cube: dirs [6][n][n][3].
ORACLE_API void oracle_sky_directions(int n, float* dirs) {
    for (int face = 0; face < 6; face++)
        for (int y = 0; y < n; y++)
            for (int x = 0; x < n; x++) {
                const vec3 d = SkyTexelDir(n, face, x, y);
                float* o = dirs + 3 * (((size_t)face * n + y) * n + x);
                o[0] = d.x; o[1] = d.y; o[2] = d.z;
            }
}

ORACLE_API void oracle_det_atan2(const float* y, const float* x, uint64_t n, float* out) { for (uint64_t i = 0; i < n; i++) out[i] = SkyAtan2(y[i], x[i]); }
ORACLE_API void oracle_det_asin(const float* x, uint64_t n, float* out) { for (uint64_t i = 0; i < n; i++) out[i] = SkyAsin(x[i]); }

} // extern "C"
