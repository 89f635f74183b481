// ORACLE (TEST INFRASTRUCTURE ONLY) -- the light spheres and the skybox under the shading-rate image (idkpt_lights_and_skybox_vrs).
//
// The root of its own library, liboracle_lights_skybox_vrs.so, which tests/lights_skybox_vrs_oracle.py builds and wraps. It
// includes the per-pixel oracle (oracle_lights_skybox.cpp, and with it oracle_gbuffer.cpp and oracle.cpp) and the
// variable-rate deferred oracle (oracle_vrs.cpp) and reuses LsShadePixel's coverage, depth test and winner, the sphere mesh,
// RayTriangleIntersect, EncodeUnitVec, SampleSky, the attachment conversions and VrsFragmentSize unchanged. What the fragment
// shaders compute at the coarse fragment's centre is restated here.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Source/Render/RasterPipeline.cs:465-516                    "Draw lights" and "Draw skybox" with VariableRateShadingNV
//   Resource/Shaders/Light/fragment.glsl, SkyBox/fragment.glsl the fragment shaders, once per coarse fragment
//
// DESIGN.md 8f.1i (the variable-rate paragraph) pins the rules.
#pragma once
#include "oracle_lights_skybox.cpp"
#include "oracle_vrs.cpp"

namespace {

// The draws under a rate image (RasterPipeline.cs:465-516 with VariableRateShadingNV): GL runs the fragment shader once per
// (primitive, coarse fragment) at the fragment's centre, while coverage and the depth test stay per pixel. So the pixel keeps
// LsShadePixel's winner, depth, emissive and colour, and what the shaders interpolate is taken at the centre (xc, yc): for a
// light, the centre ray's barycentrics on the plane of the pixel's winning triangle (RayTriangleIntersect's arithmetic, its
// inside and t tests ignored: outside the triangle this is the line-plane intersection, t < 0 included); for the sky, TexCoord
// on the cube face the pixel's own direction leaves through (axis x if |x| >= |y|, |z|, else y if |y| >= |z|, else z).
void LsShadeAtCentre(const Scene& s, const GpuPerFrameData& f, int x, int y, int w, int h, const float jitter[2], float xc, float yc,
                     LsPixel& px) {
    if (px.light) {
        const float ndcX = xc / (float)w * 2.0f - 1.0f - jitter[0];
        const float ndcY = yc / (float)h * 2.0f - 1.0f - jitter[1];
        const float* m = f.InvProjView;
        const float hx = ((m[0] * ndcX + m[4] * ndcY) + m[8] * 1.0f) + m[12] * 1.0f;
        const float hy = ((m[1] * ndcX + m[5] * ndcY) + m[9] * 1.0f) + m[13] * 1.0f;
        const float hz = ((m[2] * ndcX + m[6] * ndcY) + m[10] * 1.0f) + m[14] * 1.0f;
        const float hw = ((m[3] * ndcX + m[7] * ndcY) + m[11] * 1.0f) + m[15] * 1.0f;
        const vec3 eye = V(f.ViewPos);
        const Ray ray{eye, normalize(V(hx / hw, hy / hw, hz / hw) - eye)};
        const SphereMesh& mesh = Mesh();
        const GpuLight& L = s.d.Lights[px.winner / kTriangles];
        const uint32_t* id = mesh.idx[px.winner % kTriangles];
        const vec3 w0 = LsWorld(L, L.Position, mesh.v[id[0]]), w1 = LsWorld(L, L.Position, mesh.v[id[1]]), w2 = LsWorld(L, L.Position, mesh.v[id[2]]);
        vec3 bary;
        float tHit;
        (void)RayTriangleIntersect(ray, w0, w1, w2, bary, tHit);
        const float b0 = bary.x, b1 = bary.y, b2 = 1.0f - bary.x - bary.y;
        const vec3 fragPos = (w0 * b0 + w1 * b1) + w2 * b2;
        float ex, ey;
        EncodeUnitVec((fragPos - V(L.Position)) / L.Radius, ex, ey);
        px.normal[0] = GbUnorm8(ex); px.normal[1] = GbUnorm8(ey);
        Vec4f q[3];
        for (int i = 0; i < 3; i++) q[i] = GbClip(f.PrevProjView, LsWorld(L, L.PrevPosition, mesh.v[id[i]]));
        const float pcx = (q[0].x * b0 + q[1].x * b1) + q[2].x * b2;
        const float pcy = (q[0].y * b0 + q[1].y * b1) + q[2].y * b2;
        const float pcw = (q[0].w * b0 + q[1].w * b1) + q[2].w * b2;
        px.velocity[0] = to_half_and_back((ndcX - pcx / pcw) * 0.5f);
        px.velocity[1] = to_half_and_back((ndcY - pcy / pcw) * 0.5f);
    } else if (px.sky) {
        const float* ip = f.InvProjection;
        const float* iv = f.InvView;
        auto dirAt = [&](float sx, float sy) {   // rule 5's direction at an unjittered NDC
            const float vw = ((ip[3] * sx + ip[7] * sy) + ip[11] * 1.0f) + ip[15] * 1.0f;
            const vec3 v = {(((ip[0] * sx + ip[4] * sy) + ip[8] * 1.0f) + ip[12] * 1.0f) / vw,
                            (((ip[1] * sx + ip[5] * sy) + ip[9] * 1.0f) + ip[13] * 1.0f) / vw,
                            (((ip[2] * sx + ip[6] * sy) + ip[10] * 1.0f) + ip[14] * 1.0f) / vw};
            return vec3{((iv[0] * v.x + iv[4] * v.y) + iv[8] * v.z) + iv[12] * 0.0f, ((iv[1] * v.x + iv[5] * v.y) + iv[9] * v.z) + iv[13] * 0.0f,
                        ((iv[2] * v.x + iv[6] * v.y) + iv[10] * v.z) + iv[14] * 0.0f};
        };
        const vec3 dp = dirAt(((float)x + 0.5f) / (float)w * 2.0f - 1.0f, ((float)y + 0.5f) / (float)h * 2.0f - 1.0f);
        const float ax = fabsf(dp.x), ay = fabsf(dp.y), az = fabsf(dp.z);
        const int axis = (ax >= ay && ax >= az) ? 0 : (ay >= az ? 1 : 2);
        const float sx = xc / (float)w * 2.0f - 1.0f, sy = yc / (float)h * 2.0f - 1.0f;
        const vec3 dir = dirAt(sx, sy);
        const vec3 c = dir * (0.5f / fabsf(axis == 0 ? dir.x : axis == 1 ? dir.y : dir.z));
        const vec3 sky = SampleSky(s.skyFaces, s.skyFaceSize, s.skyColor, c);
        const float* pv = f.PrevView;
        const vec3 pc = {(pv[0] * c.x + pv[4] * c.y) + pv[8] * c.z, (pv[1] * c.x + pv[5] * c.y) + pv[9] * c.z, (pv[2] * c.x + pv[6] * c.y) + pv[10] * c.z};
        const Vec4f q = GbClip(f.Projection, pc);
        px.velocity[0] = to_half_and_back((sx - q.x / q.w) * 0.5f);
        px.velocity[1] = to_half_and_back((sy - q.y / q.w) * 0.5f);
        px.color[0] = sky.x; px.color[1] = sky.y; px.color[2] = sky.z;
    }
}

} // namespace

// idkpt_lights_and_skybox_vrs: oracle_lights_skybox's arguments and, before `threads`, rates [ceil(h/16)][ceil(w/16)] (palette
// indices 0..4). Returns 0, or 1 for an argument the library rejects. Its ctypes signature is declared with its wrapper,
// tests/lights_skybox_vrs_oracle.py, which also builds this library.
extern "C" ORACLE_API int oracle_lights_skybox_vrs(const IdkPtSceneDesc* scene, const IdkPtSkyDesc* sky, const GpuPerFrameData* frame,
                                                   int w, int h, const float* jitter, float* depth, float* normal, float* emissive,
                                                   float* velocity, float* color, int32_t* winner, const uint8_t* rates, int threads) {
    if (!scene || !frame || !rates || w < 1 || h < 1) return 1;
    const int tilesX = (w + 15) / 16;
    for (size_t t = 0; t < (size_t)tilesX * ((h + 15) / 16); t++)
        if (rates[t] > 4) return 1;
    Scene s; s.d = *scene;
    for (int i = 0; i < 3; i++) s.skyColor[i] = sky ? sky->Color[i] : 0.0f;
    if (sky && sky->FaceSize > 0) { s.skyFaceSize = sky->FaceSize; for (int i = 0; i < 6; i++) s.skyFaces[i] = sky->Faces[i]; }
    const float jit[2] = {jitter ? jitter[0] : 0.0f, jitter ? jitter[1] : 0.0f};
    parallel_for((size_t)w * h, threads, [&](size_t begin, size_t end, int) {
        for (size_t p = begin; p < end; p++) {
            const int x = (int)(p % w), y = (int)(p / w);
            LsPixel px = LsShadePixel(s, *frame, x, y, w, h, jit, depth[p]);   // coverage, depth test and winner per pixel
            int cw, ch;                                                          // the pixel's coarse fragment and its centre
            VrsFragmentSize(rates[(size_t)(y / 16) * tilesX + x / 16], cw, ch);
            LsShadeAtCentre(s, *frame, x, y, w, h, jit, (float)(x - x % cw) + 0.5f * (float)cw, (float)(y - y % ch) + 0.5f * (float)ch, px);
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
