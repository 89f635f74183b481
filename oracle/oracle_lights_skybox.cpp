// ORACLE (TEST INFRASTRUCTURE ONLY) -- the light spheres and the skybox, ray-cast at pixel centres.
//
// Part of liboracle.so (wrapped by tests/lights_skybox_oracle.py). It includes the G-buffer oracle (and with it oracle.cpp)
// and reuses its clip transform, front-face rule and attachment
// conversions, and oracle.cpp's RayTriangleIntersect, EncodeUnitVec, SampleSky and half conversion unchanged. The sphere mesh,
// the brute-force light draw (every triangle of every light, no rejection) and the skybox draw are restated here.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Source/Utils/GeometricPrimitives.cs:16-83                  Sphere.GenerateVertices / GenerateIndices
//   Source/Render/LightManager.cs:82-117                       the 12 x 12 unit sphere, one instance per light
//   Resource/Shaders/Light/vertex.glsl, fragment.glsl          model matrix Radius * p + Position, the four outputs
//   Resource/Shaders/SkyBox/vertex.glsl, fragment.glsl         the cube around the camera, xyww, the rotation-only velocity
//   Source/Render/RasterPipeline.cs:465-516                    the two draws: LESS + CullFace, then LEQUAL without culling
//
// DESIGN.md 8f.1i pins the rules.
#pragma once
#include "oracle_gbuffer.cpp"

namespace {

const int kSegments = 12, kVertices = 169, kTriangles = 264;

struct SphereMesh {
    vec3 v[kVertices];
    uint32_t idx[kTriangles][3];
    SphereMesh() {
        const float pi = 3.14159265358979323846f;
        const float dLat = pi / (float)kSegments, dLon = 2.0f * pi / (float)kSegments;
        int k = 0;
        for (int i = 0; i <= kSegments; i++) {
            const float lat = pi / 2.0f - (float)i * dLat;
            const float xy = 1.0f * (float)std::cos((double)lat), z = 1.0f * (float)std::sin((double)lat);
            for (int j = 0; j <= kSegments; j++) {
                const float lon = (float)j * dLon;
                v[k++] = {xy * (float)std::cos((double)lon), xy * (float)std::sin((double)lon), z};
            }
        }
        int t = 0;
        for (uint32_t i = 0; i < (uint32_t)kSegments; i++) {
            uint32_t k1 = i * (kSegments + 1), k2 = k1 + kSegments + 1;
            for (int j = 0; j < kSegments; j++, k1++, k2++) {
                if (i != 0) { idx[t][0] = k1; idx[t][1] = k2; idx[t][2] = k1 + 1; t++; }
                if (i != (uint32_t)kSegments - 1) { idx[t][0] = k1 + 1; idx[t][1] = k2; idx[t][2] = k2 + 1; t++; }
            }
        }
    }
};
const SphereMesh& Mesh() { static const SphereMesh m; return m; }

// mat4x3(Radius I, Position) * vec4(p, 1)
inline vec3 LsWorld(const GpuLight& L, const float* position, vec3 p) {
    return {L.Radius * p.x + position[0], L.Radius * p.y + position[1], L.Radius * p.z + position[2]};
}

struct LsPixel { float depth, normal[2], emissive[3], velocity[2], color[4]; int winner; bool light, sky; };

ORACLE_INLINE LsPixel LsShadePixel(const Scene& s, const GpuPerFrameData& f, int x, int y, int w, int h, const float jitter[2], float gDepth) {
    LsPixel px = {};
    px.depth = gDepth;
    px.winner = -1;
    const float ndcX = ((float)x + 0.5f) / (float)w * 2.0f - 1.0f - jitter[0];
    const float ndcY = ((float)y + 0.5f) / (float)h * 2.0f - 1.0f - jitter[1];
    const float* m = f.InvProjView;
    const float hx = ((m[0] * ndcX + m[4] * ndcY) + m[8] * 1.0f) + m[12] * 1.0f;
    const float hy = ((m[1] * ndcX + m[5] * ndcY) + m[9] * 1.0f) + m[13] * 1.0f;
    const float hz = ((m[2] * ndcX + m[6] * ndcY) + m[10] * 1.0f) + m[14] * 1.0f;
    const float hw = ((m[3] * ndcX + m[7] * ndcY) + m[11] * 1.0f) + m[15] * 1.0f;
    const vec3 eye = V(f.ViewPos);
    const Ray ray{eye, normalize(V(hx / hw, hy / hw, hz / hw) - eye)};

    const SphereMesh& mesh = Mesh();
    float bb0 = 0.0f, bb1 = 0.0f;
    for (uint64_t l = 0; l < s.d.LightCount; l++) {
        const GpuLight& L = s.d.Lights[l];
        for (int t = 0; t < kTriangles; t++) {
            const vec3 w0 = LsWorld(L, L.Position, mesh.v[mesh.idx[t][0]]);
            const vec3 w1 = LsWorld(L, L.Position, mesh.v[mesh.idx[t][1]]);
            const vec3 w2 = LsWorld(L, L.Position, mesh.v[mesh.idx[t][2]]);
            vec3 bary;
            float tHit;
            if (!RayTriangleIntersect(ray, w0, w1, w2, bary, tHit)) continue;
            // CullFace: in world space the winding is the window-space winding (det(Radius I) and d / Radius share a sign)
            if (!GbFrontFacing(1.0f, cross(w1 - w0, w2 - w0), ray.d)) continue;
            const Vec4f c0 = GbClip(f.ProjView, w0), c1 = GbClip(f.ProjView, w1), c2 = GbClip(f.ProjView, w2);
            const float b0 = bary.x, b1 = bary.y, b2 = 1.0f - bary.x - bary.y;
            const float depth = ((c0.z * b0 + c1.z * b1) + c2.z * b2) / ((c0.w * b0 + c1.w * b1) + c2.w * b2);
            if (!(depth >= 0.0f && depth <= 1.0f)) continue;   // clipped
            if (!(depth < px.depth)) continue;                  // LESS
            px.depth = depth;
            px.winner = (int)l * kTriangles + t;
            bb0 = b0; bb1 = b1;
        }
    }
    if (px.winner >= 0) {
        const GpuLight& L = s.d.Lights[px.winner / kTriangles];
        const uint32_t* id = mesh.idx[px.winner % kTriangles];
        const float b0 = bb0, b1 = bb1, b2 = 1.0f - bb0 - bb1;
        const vec3 fragPos = (LsWorld(L, L.Position, mesh.v[id[0]]) * b0 + LsWorld(L, L.Position, mesh.v[id[1]]) * b1) +
                             LsWorld(L, L.Position, mesh.v[id[2]]) * b2;
        float ex, ey;
        EncodeUnitVec((fragPos - V(L.Position)) / L.Radius, ex, ey);
        px.normal[0] = GbUnorm8(ex); px.normal[1] = GbUnorm8(ey);
        for (int c = 0; c < 3; c++) {
            px.emissive[c] = c < 2 ? GbUnsignedFloat(L.Color[c], 6, 65024.0f) : GbUnsignedFloat(L.Color[c], 5, 64512.0f);
            px.color[c] = L.Color[c];
        }
        px.color[3] = 1.0f;
        Vec4f q[3];
        for (int i = 0; i < 3; i++) q[i] = GbClip(f.PrevProjView, LsWorld(L, L.PrevPosition, mesh.v[id[i]]));
        const float pcx = (q[0].x * b0 + q[1].x * b1) + q[2].x * b2;
        const float pcy = (q[0].y * b0 + q[1].y * b1) + q[2].y * b2;
        const float pcw = (q[0].w * b0 + q[1].w * b1) + q[2].w * b2;
        px.velocity[0] = to_half_and_back((ndcX - pcx / pcw) * 0.5f);
        px.velocity[1] = to_half_and_back((ndcY - pcy / pcw) * 0.5f);
        px.light = true;
    } else if (1.0f <= px.depth) {   // LEQUAL against the skybox's window depth 1
        const float sx = ((float)x + 0.5f) / (float)w * 2.0f - 1.0f, sy = ((float)y + 0.5f) / (float)h * 2.0f - 1.0f;
        const float* ip = f.InvProjection;
        const float vw = ((ip[3] * sx + ip[7] * sy) + ip[11] * 1.0f) + ip[15] * 1.0f;
        const vec3 v = {(((ip[0] * sx + ip[4] * sy) + ip[8] * 1.0f) + ip[12] * 1.0f) / vw,
                        (((ip[1] * sx + ip[5] * sy) + ip[9] * 1.0f) + ip[13] * 1.0f) / vw,
                        (((ip[2] * sx + ip[6] * sy) + ip[10] * 1.0f) + ip[14] * 1.0f) / vw};
        const float* iv = f.InvView;
        const vec3 dir = {((iv[0] * v.x + iv[4] * v.y) + iv[8] * v.z) + iv[12] * 0.0f, ((iv[1] * v.x + iv[5] * v.y) + iv[9] * v.z) + iv[13] * 0.0f,
                          ((iv[2] * v.x + iv[6] * v.y) + iv[10] * v.z) + iv[14] * 0.0f};
        const vec3 c = dir * (0.5f / fmaxf(fmaxf(fabsf(dir.x), fabsf(dir.y)), fabsf(dir.z)));   // TexCoord on the cube
        const vec3 sky = SampleSky(s.skyFaces, s.skyFaceSize, s.skyColor, c);
        const float* pv = f.PrevView;
        const vec3 pc = {(pv[0] * c.x + pv[4] * c.y) + pv[8] * c.z, (pv[1] * c.x + pv[5] * c.y) + pv[9] * c.z, (pv[2] * c.x + pv[6] * c.y) + pv[10] * c.z};
        const Vec4f q = GbClip(f.Projection, pc);
        px.velocity[0] = to_half_and_back((sx - q.x / q.w) * 0.5f);
        px.velocity[1] = to_half_and_back((sy - q.y / q.w) * 0.5f);
        px.color[0] = sky.x; px.color[1] = sky.y; px.color[2] = sky.z; px.color[3] = 1.0f;
        px.sky = true;
    }
    return px;
}

} // namespace

extern "C" {

// idkpt_lights_and_skybox, in place: depth [h][w], normal [h][w][2], emissive [h][w][3], velocity [h][w][2] (the G-buffer)
// and color [h][w][4] (the lit image). jitter and sky may be null ((0, 0); a black constant sky). winner (optional) receives
// per pixel light * 264 + triangle of the light fragment drawn, -2 for a sky pixel, -1 for a pixel neither draw touched.
ORACLE_API int oracle_lights_skybox(const IdkPtSceneDesc* scene, const IdkPtSkyDesc* sky, const GpuPerFrameData* frame, int w, int h,
                                    const float* jitter, float* depth, float* normal, float* emissive, float* velocity, float* color,
                                    int32_t* winner, int threads) {
    if (!scene || !frame || w < 1 || h < 1) return 1;
    Scene s; s.d = *scene;
    for (int i = 0; i < 3; i++) s.skyColor[i] = sky ? sky->Color[i] : 0.0f;
    if (sky && sky->FaceSize > 0) { s.skyFaceSize = sky->FaceSize; for (int i = 0; i < 6; i++) s.skyFaces[i] = sky->Faces[i]; }
    const float jit[2] = {jitter ? jitter[0] : 0.0f, jitter ? jitter[1] : 0.0f};
    parallel_for((size_t)w * h, threads, [&](size_t begin, size_t end, int) {
        for (size_t p = begin; p < end; p++) {
            const LsPixel px = LsShadePixel(s, *frame, (int)(p % w), (int)(p / w), w, h, jit, depth[p]);
            if (winner) winner[p] = px.light ? px.winner : px.sky ? -2 : -1;
            if (px.light) {
                depth[p] = px.depth;
                for (int c = 0; c < 2; c++) normal[2 * p + c] = px.normal[c];
                for (int c = 0; c < 3; c++) emissive[3 * p + c] = px.emissive[c];
            }
            if (px.light || px.sky) {
                for (int c = 0; c < 2; c++) velocity[2 * p + c] = px.velocity[c];
                for (int c = 0; c < 4; c++) color[4 * p + c] = px.color[c];
            }
        }
    });
    return 0;
}

// The unit-sphere mesh: vertices [169][3] and the index buffer [264][3].
ORACLE_API void oracle_sphere_mesh(float* vertices, uint32_t* indices) {
    const SphereMesh& m = Mesh();
    for (int i = 0; i < kVertices; i++) { vertices[3 * i] = m.v[i].x; vertices[3 * i + 1] = m.v[i].y; vertices[3 * i + 2] = m.v[i].z; }
    for (int t = 0; t < kTriangles; t++) for (int c = 0; c < 3; c++) indices[3 * t + c] = m.idx[t][c];
}

} // extern "C"
