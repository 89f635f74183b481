// Device-side math for libidkpt (sm_90a). Float semantics contract (DESIGN.md):
// fp32, left-to-right evaluation, NO fused multiply-add (the TU is compiled with
// -fmad=false), IEEE divide / sqrt (-prec-div=true -prec-sqrt=true), fminf/fmaxf
// return the non-NaN operand. normalize(v) = v * (1/sqrt(dot)), pow(x,5) by
// squaring, sin/cos/exp = the polynomial routines below.
//
// GLSL sources restated (relative to the reference repository's IDKEngine/Resource/Shaders):
//   include/IntersectionRoutines.glsl:6-69, include/Random.glsl:16-33,
//   include/Sampling.glsl:4-19,59-68,86-114, include/Compression.glsl:11-73,
//   include/Math.glsl:6-15,41-57,104-137
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define IDK_PI 3.14159265f
#define IDK_FLOAT_MAX 3.4028235e+38f

struct f3 { float x, y, z; };

__device__ __forceinline__ f3 mk3(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ f3 operator+(f3 a, f3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ f3 operator-(f3 a, f3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ f3 operator-(f3 a) { return mk3(-a.x, -a.y, -a.z); }
__device__ __forceinline__ f3 operator*(f3 a, f3 b) { return mk3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ f3 operator*(f3 a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ f3 operator*(float s, f3 a) { return mk3(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ f3 operator/(f3 a, float s) { return mk3(a.x / s, a.y / s, a.z / s); }
__device__ __forceinline__ float dot3(f3 a, f3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ f3 cross3(f3 a, f3 b) { return mk3(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y); }
__device__ __forceinline__ f3 normalize3(f3 v) { float inv = 1.0f / sqrtf(dot3(v, v)); return v * inv; }
__device__ __forceinline__ float mix1(float x, float y, float a) { return x * (1.0f - a) + y * a; }
__device__ __forceinline__ f3 mix3(f3 x, f3 y, float a) { return mk3(mix1(x.x, y.x, a), mix1(x.y, y.y, a), mix1(x.z, y.z, a)); }
__device__ __forceinline__ float clamp1(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ float fract1(float x) { return x - floorf(x); }
__device__ __forceinline__ f3 reflect3(f3 I, f3 N) { return I - (2.0f * dot3(N, I)) * N; }
__device__ __forceinline__ f3 refract3(f3 I, f3 N, float eta) {
    float d = dot3(N, I);
    float k = 1.0f - eta * eta * (1.0f - d * d);
    if (k < 0.0f) return mk3(0.0f, 0.0f, 0.0f);
    return eta * I - (eta * d + sqrtf(k)) * N;
}
__device__ __forceinline__ float pow5f(float x) { float x2 = x * x; return (x2 * x2) * x; }

// ---- deterministic sin/cos on [0, 2pi]: quadrant reduction (two-term pi/2) + Cephes sinf/cosf polynomials
__device__ __forceinline__ void det_sincos(float x, float* s, float* c) {
    float q = floorf(x * 0.63661977236758134f + 0.5f);
    int n = (int)q;
    float r = (x - q * 1.5703125f) - q * 4.83826794897e-4f;
    float z = r * r;
    float sp = ((-1.9515295891e-4f * z + 8.3321608736e-3f) * z - 1.6666654611e-1f) * z * r + r;
    float cp = ((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z + 4.166664568298827e-2f) * z * z - 0.5f * z + 1.0f;
    switch (n & 3) {
        case 0: *s = sp; *c = cp; break;
        case 1: *s = cp; *c = -sp; break;
        case 2: *s = -sp; *c = -cp; break;
        default: *s = -cp; *c = sp; break;
    }
}

// ---- deterministic exp: n = round(x*log2e), two-term ln2 reduction, Cephes expf polynomial, 2^n by exponent bits
__device__ __forceinline__ float det_exp(float x) {
    if (x < -87.0f) return 0.0f;
    if (x > 88.0f) return __int_as_float(0x7f800000);
    float fn = floorf(x * 1.44269504088896341f + 0.5f);
    float r = (x - fn * 0.693359375f) - fn * -2.12194440e-4f;
    float z = r * r;
    float p = ((((1.9875691500e-4f * r + 1.3981999507e-3f) * r + 8.3334519073e-3f) * r + 4.1665795894e-2f) * r + 1.6666665459e-1f) * r + 5.0000001201e-1f;
    float e = p * z + r + 1.0f;
    int n = (int)fn;
    return e * __int_as_float((n + 127) << 23);
}

// ---- deterministic log2: Cephes logf polynomial on [sqrt(1/2), sqrt(2)), then * log2(e) + exponent
__device__ __forceinline__ float det_log2(float x) {
    const uint32_t bits = __float_as_uint(x);
    int e = (int)((bits >> 23) & 255u) - 126;
    float m = __uint_as_float((bits & 0x807FFFFFu) | 0x3F000000u);
    if (m < 0.70710678f) { m = m + m; e -= 1; }
    m = m - 1.0f;
    const float z = m * m;
    float y = ((((((((7.0376836292e-2f * m - 1.1514610310e-1f) * m + 1.1676998740e-1f) * m - 1.2420140846e-1f) * m + 1.4249322787e-1f) * m - 1.6668057665e-1f) * m + 2.0000714765e-1f) * m - 2.4999993993e-1f) * m + 3.3333331174e-1f) * m * z;
    y = y - 0.5f * z;
    return (m + y) * 1.44269504f + (float)e;
}

// One 2-D RGBA8 texture, base level only: compute shaders sample lod 0 (Surface.glsl:57-60).
struct TexRec {
    const void* px;               // decoded level 0: uchar4 (kind 0), float2 (1), float (2) or float4 (3) texels
    int w, h;
    int wrapS, wrapT;             // GL enums: 10497 REPEAT, 33071 CLAMP_TO_EDGE, 33648 MIRRORED_REPEAT
    int srgb;                     // rgb decoded through srgbLut before filtering (GL_SRGB8_ALPHA8 / BC7 sRGB)
    int kind;                     // bits 0-7: texel storage kind, bit 8: R channel reads B (IDKPT_TEX_FLAG_R_FROM_B), bit 9: MagFilter NEAREST
};

// ---- material textures: texture(sampler2D, uv) at lod 0 = bilinear on the base level, evaluated explicitly in fp32
// (same rule as the sky faces / VXGI grid), wrap modes of the glTF sampler (ModelLoader.cs:1166-1196).
__device__ __forceinline__ int tex_wrap(int i, int n, int mode) {
    if (mode == 33071) return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
    if (mode == 33648) { int m = i % (2 * n); if (m < 0) m += 2 * n; return m < n ? m : 2 * n - 1 - m; }
    int m = i % n;
    return m < 0 ? m + n : m;
}
__device__ __forceinline__ float4 tex_fetch(const TexRec& t, const float* lut, int x, int y) {
    const size_t i = (size_t)y * t.w + x;
    const int kind = t.kind & 255;
    float4 r;
    if (kind == 0) {
        const uchar4 c = __ldg((const uchar4*)t.px + i);
        if (t.srgb) r = make_float4(__ldg(lut + c.x), __ldg(lut + c.y), __ldg(lut + c.z), (float)c.w / 255.0f);
        else r = make_float4((float)c.x / 255.0f, (float)c.y / 255.0f, (float)c.z / 255.0f, (float)c.w / 255.0f);
    } else if (kind == 1) {       // GL returns (R, G, 0, 1) for a two-channel texture
        const float2 c = __ldg((const float2*)t.px + i);
        r = make_float4(c.x, c.y, 0.0f, 1.0f);
    } else if (kind == 2) {
        r = make_float4(__ldg((const float*)t.px + i), 0.0f, 0.0f, 1.0f);
    } else {
        r = __ldg((const float4*)t.px + i);
    }
    if (t.kind & 256) r.x = r.z;
    return r;
}
__device__ __forceinline__ float4 tex_lerp(float4 a, float4 b, float t) {
    const float s = 1.0f - t;
    return make_float4(a.x * s + b.x * t, a.y * s + b.y * t, a.z * s + b.z * t, a.w * s + b.w * t);
}
__device__ __forceinline__ float4 tex_sample_raw(const TexRec* textures, const float* lut, unsigned long long handle, float u, float v) {
    if (handle == 0) return make_float4(1.0f, 1.0f, 1.0f, 1.0f);
    const TexRec& t = textures[handle - 1];
    if (t.wrapS == 10497) u = u - floorf(u);
    if (t.wrapT == 10497) v = v - floorf(v);
    if (t.kind & 512)             // GL_NEAREST magnification: the texel that contains (u, v)
        return tex_fetch(t, lut, tex_wrap((int)floorf(u * (float)t.w), t.w, t.wrapS), tex_wrap((int)floorf(v * (float)t.h), t.h, t.wrapT));
    const float px = u * (float)t.w - 0.5f, py = v * (float)t.h - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    const float fx = px - fx0, fy = py - fy0;
    const int x0 = tex_wrap((int)fx0, t.w, t.wrapS), x1 = tex_wrap((int)fx0 + 1, t.w, t.wrapS);
    const int y0 = tex_wrap((int)fy0, t.h, t.wrapT), y1 = tex_wrap((int)fy0 + 1, t.h, t.wrapT);
    const float4 a = tex_lerp(tex_fetch(t, lut, x0, y0), tex_fetch(t, lut, x1, y0), fx);
    const float4 b = tex_lerp(tex_fetch(t, lut, x0, y1), tex_fetch(t, lut, x1, y1), fx);
    return tex_lerp(a, b, fy);
}

// ---- RNG (Random.glsl:16-33)
__device__ __forceinline__ uint32_t pcg_hash(uint32_t& seed) {
    seed = seed * 747796405u + 2891336453u;
    uint32_t word = ((seed >> ((seed >> 28u) + 4u)) ^ seed) * 277803737u;
    return (word >> 22u) ^ word;
}
__device__ __forceinline__ float rnd01(uint32_t& seed) { return __uint2float_rn(pcg_hash(seed)) / 4294967296.0f; }

// ---- Sampling.glsl
__device__ __forceinline__ f3 sample_sphere(float rnd0, float rnd1) {
    float cosTheta = rnd0 * 2.0f - 1.0f;
    float phi = rnd1 * 2.0f * IDK_PI;
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    float sinPhi, cosPhi;
    det_sincos(phi, &sinPhi, &cosPhi);
    return mk3(sinTheta * cosPhi, sinTheta * sinPhi, cosTheta);
}
__device__ __forceinline__ void sample_disk(uint32_t& seed, float& px, float& py) {
    float dist;
    float lastRnd = rnd01(seed);
    do {
        float thisRnd = rnd01(seed);
        px = lastRnd;
        py = thisRnd;
        dist = px * px + py * py;
        lastRnd = thisRnd;
    } while (dist > 1.0f);
    px = px * 2.0f - 1.0f;
    py = py * 2.0f - 1.0f;
}

// ---- Compression.glsl
__device__ __forceinline__ f3 decompress_sr11g11b10(uint32_t data) {
    float r = (float)((data >> 0) & 2047u);
    float g = (float)((data >> 11) & 2047u);
    float b = (float)((data >> 22) & 1023u);
    r /= 2047.0f;
    g /= 2047.0f;
    b /= 1023.0f;
    return mk3(r * 2.0f - 1.0f, g * 2.0f - 1.0f, b * 2.0f - 1.0f);
}
__device__ __forceinline__ void encode_unit_vec(f3 n, float& ex, float& ey) {
    float l1 = (fabsf(n.x) + fabsf(n.y)) + fabsf(n.z);
    n = n / l1;
    float nx = n.x, ny = n.y;
    if (!(n.z > 0.0f)) {
        float wx = 1.0f - fabsf(n.y);
        float wy = 1.0f - fabsf(n.x);
        if (n.x < 0.0f) wx = -wx;
        if (n.y < 0.0f) wy = -wy;
        nx = wx;
        ny = wy;
    }
    ex = nx * 0.5f + 0.5f;
    ey = ny * 0.5f + 0.5f;
}
__device__ __forceinline__ f3 decode_unit_vec(float fx, float fy) {
    fx = fx * 2.0f - 1.0f;
    fy = fy * 2.0f - 1.0f;
    f3 n = mk3(fx, fy, 1.0f - fabsf(fx) - fabsf(fy));
    float t = fmaxf(-n.z, 0.0f);
    n.x += n.x >= 0.0f ? -t : t;
    n.y += n.y >= 0.0f ? -t : t;
    return normalize3(n);
}
__device__ __forceinline__ float sign1(float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); }
__device__ __forceinline__ f3 cubemap_face_normal(f3 dir) {
    f3 a = mk3(fabsf(dir.x), fabsf(dir.y), fabsf(dir.z));
    float mx = a.x >= fmaxf(a.y, a.z) ? 1.0f : 0.0f;
    float my = a.y >= fmaxf(a.z, a.x) ? 1.0f : 0.0f;
    float mz = a.z >= fmaxf(a.x, a.y) ? 1.0f : 0.0f;
    return mk3(mx * -sign1(dir.x), my * -sign1(dir.y), mz * -sign1(dir.z));
}

// ---- matrices
// GpuMeshTransform 3x4 (rows act on column vectors): point and vector transforms (Ray.glsl:7-12)
__device__ __forceinline__ f3 xform_point(const float4 r0, const float4 r1, const float4 r2, f3 p) {
    return mk3(((r0.x * p.x + r0.y * p.y) + r0.z * p.z) + r0.w,
               ((r1.x * p.x + r1.y * p.y) + r1.z * p.z) + r1.w,
               ((r2.x * p.x + r2.y * p.y) + r2.z * p.z) + r2.w);
}
__device__ __forceinline__ f3 xform_vector(const float4 r0, const float4 r1, const float4 r2, f3 v) {
    return mk3((r0.x * v.x + r0.y * v.y) + r0.z * v.z,
               (r1.x * v.x + r1.y * v.y) + r1.z * v.z,
               (r2.x * v.x + r2.y * v.y) + r2.z * v.z);
}
// mat3(transpose(InvModel)) * v  (FirstHit/compute.glsl:148)
__device__ __forceinline__ f3 xform_normal(const float4 r0, const float4 r1, const float4 r2, f3 v) {
    return mk3((r0.x * v.x + r1.x * v.y) + r2.x * v.z,
               (r0.y * v.x + r1.y * v.y) + r2.y * v.z,
               (r0.z * v.x + r1.z * v.y) + r2.z * v.z);
}
// GLSL column-major mat4 (16 floats) times vec4 -> xyz
__device__ __forceinline__ f3 mat4_mul_xyz(const float* m, float x, float y, float z, float w) {
    return mk3(((m[0] * x + m[4] * y) + m[8] * z) + m[12] * w,
               ((m[1] * x + m[5] * y) + m[9] * z) + m[13] * w,
               ((m[2] * x + m[6] * y) + m[10] * z) + m[14] * w);
}

// ---- intersectors (IntersectionRoutines.glsl)
__device__ __forceinline__ bool ray_box(f3 o, f3 inv, float4 nA, float4 nB, float& tNear) {
    // nA = (Min.xyz, TriStartOrChild), nB = (Max.xyz, TriCount)
    float t0x = (nA.x - o.x) * inv.x, t0y = (nA.y - o.y) * inv.y, t0z = (nA.z - o.z) * inv.z;
    float t1x = (nB.x - o.x) * inv.x, t1y = (nB.y - o.y) * inv.y, t1z = (nB.z - o.z) * inv.z;
    float sx = fminf(t0x, t1x), sy = fminf(t0y, t1y), sz = fminf(t0z, t1z);
    float bx = fmaxf(t0x, t1x), by = fmaxf(t0y, t1y), bz = fmaxf(t0z, t1z);
    tNear = fmaxf(sx, fmaxf(sy, fmaxf(sz, 0.0f)));
    float tFar = fminf(bx, fminf(by, bz));
    return tNear <= tFar;
}

// Triangle record prepared at scene upload: p0, e1 = p1-p0, e2 = p2-p0, n = cross(e1,e2) -- the first four
// statements of RayTriangleIntersect, hoisted out of the traversal loop (same fp32 operations, same bits).
__device__ __forceinline__ bool ray_triangle(f3 o, f3 d, f3 p0, f3 e1, f3 e2, f3 n, float& bx, float& by, float& t) {
    f3 rop0 = o - p0;
    f3 q = cross3(rop0, d);
    float invDet = 1.0f / dot3(d, n);
    t = dot3(-n, rop0) * invDet;
    float b1 = dot3(-q, e2) * invDet;
    float b2 = dot3(q, e1) * invDet;
    float b0 = 1.0f - b1 - b2;
    bx = b0;
    by = b1;
    return b0 >= 0.0f && b1 >= 0.0f && b2 >= 0.0f && t >= 0.0f;
}

__device__ __forceinline__ bool ray_sphere(f3 o, f3 d, f3 position, float radius, float& t1, float& t2) {
    t1 = IDK_FLOAT_MAX;
    t2 = IDK_FLOAT_MAX;
    f3 sphereToRay = o - position;
    float b = dot3(d, sphereToRay);
    float c = dot3(sphereToRay, sphereToRay) - radius * radius;
    float discriminant = b * b - c;
    if (discriminant < 0.0f) return false;
    float squareRoot = sqrtf(discriminant);
    t1 = -b - squareRoot;
    t2 = -b + squareRoot;
    return t1 <= t2 && t2 > 0.0f;
}

__device__ __forceinline__ float4 ldg4(const float4* p) { return __ldg(p); }

// ---- experiment switches (defaults = the measured best; scripts/variant_probe.py builds and times the alternatives)
#ifndef IDK_TRI_STRIDE
#define IDK_TRI_STRIDE 4     // float4s per device-private triangle record: 3 = packed 48 B, 4 = 64 B (never straddles a 128-B line)
#endif
#ifndef IDK_REG_STACK
#define IDK_REG_STACK 0      // k_traverse2: top N entries of the traversal stack live in registers (0 = all in shared memory)
#endif

#ifndef IDK_STAGED_FETCH
#define IDK_STAGED_FETCH 0   // k_traverse2: rays are prefetched into shared memory one batch ahead (cp.async) instead of fetched in the SETUP round
#endif
#ifndef IDK_FAST_VOTE
#define IDK_FAST_VOTE 0      // k_traverse2: one ballot instead of four when (nearly) every lane is in the BOX phase
#endif
#ifndef IDK_BOX_LOOP
#define IDK_BOX_LOOP 0       // k_traverse2: stay in the BOX phase with one ballot per round while >= 33 - min(thresholds) lanes are in it
#endif
#ifndef IDK_LEAF_LOOP
#define IDK_LEAF_LOOP 0      // k_traverse2: a LEAF round tests a lane's whole pending range instead of one triangle
#endif

// One GpuBlasNode sibling pair (64 bytes, children are adjacent: BLAS.cs:16-22) / two adjacent GpuTlasNodes.
struct NodePair { float4 lA, lB, rA, rB; };

// 4 x 128-bit read-only loads (the widest global load sm_90 has)
__device__ __forceinline__ NodePair ldg_pair(const float4* np) {
    NodePair r;
    r.lA = ldg4(np); r.lB = ldg4(np + 1); r.rA = ldg4(np + 2); r.rB = ldg4(np + 3);
    return r;
}

// Device-private triangle record i: (p0.xyz,e1.x) (e1.yz,e2.xy) (e2.z,n.xyz) [pad]
__device__ __forceinline__ void ldg_tri(const float4* triRec, size_t i, float4& a, float4& b, float4& c) {
    const float4* tr = triRec + IDK_TRI_STRIDE * i;
    a = ldg4(tr); b = ldg4(tr + 1); c = ldg4(tr + 2);
}
