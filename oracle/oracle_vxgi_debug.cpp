// ORACLE (TEST INFRASTRUCTURE ONLY) -- the VXGI grid visualisation, Voxelizer.DebugRender.
//
// Built as its own library (tests/vxgi_debug_oracle.py -> oracle/liboracle_vxgi_debug.so). It compiles oracle.cpp (and with it
// oracle_vxgi.inc) into the same translation unit and reuses its SampleSky, vx_trace_cone and the half conversion unchanged.
// The march here fetches every sample: the device kernel's empty-space skipping is exact (DESIGN.md 8f.1k), so it has no
// counterpart in the oracle.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Resource/Shaders/VXGI/Voxelize/DebugVisualization/compute.glsl   the whole pass
//   Resource/Shaders/include/Math.glsl:6-15                          GetWorldSpaceDirection
//   Resource/Shaders/include/IntersectionRoutines.glsl:25-40         RayBoxIntersect with t1 and t2
//   Resource/Shaders/include/TraceCone.glsl:41-46                    the four-argument TraceCone
//   Source/Render/VXGI/Voxelizer/Voxelizer.cs:230-244                DebugRender
#include "oracle.cpp"

namespace {

// RayBoxIntersect(ray, box, t1, t2): invDir = 1 / dir (a zero component gives +-inf); min / max are fminf / fmaxf, which
// return the other operand when one is NaN (0 * inf on a face plane)
static bool DbgRayBox(vec3 o, vec3 d, const float* bmin, const float* bmax, float& t1, float& t2) {
    const vec3 invDir = V(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    const vec3 t0s = (V(bmin) - o) * invDir;
    const vec3 t1s = (V(bmax) - o) * invDir;
    const vec3 tsmaller = V(fminf(t0s.x, t1s.x), fminf(t0s.y, t1s.y), fminf(t0s.z, t1s.z));
    const vec3 tbigger = V(fmaxf(t0s.x, t1s.x), fmaxf(t0s.y, t1s.y), fmaxf(t0s.z, t1s.z));
    t1 = fmaxf(tsmaller.x, fmaxf(tsmaller.y, fmaxf(tsmaller.z, 0.0f)));
    t2 = fminf(tbigger.x, fminf(tbigger.y, tbigger.z));
    return t1 <= t2;
}

struct DbgSky {
    const float* faces[6];
    int size;
    const float* color;
};

// one pixel of DebugVisualization/compute.glsl: rgba into out, cone samples added to steps
static void DbgPixel(const VxGrid& g, const DbgSky& sky, const GpuPerFrameData& f, float stepMultiplier, float coneAngle, int x, int y,
                     int w, int h, float* out, uint64_t& steps) {
    const float ndcx = ((float)x + 0.5f) / (float)w * 2.0f - 1.0f;
    const float ndcy = ((float)y + 0.5f) / (float)h * 2.0f - 1.0f;
    const float* ip = f.InvProjection;
    const float rvx = ip[0] * ndcx + ip[4] * ndcy;          // mat2(inverseProj) * ndc
    const float rvy = ip[1] * ndcx + ip[5] * ndcy;
    const float* iv = f.InvView;                            // (inverseView * vec4(rv, -1, 0)).xyz
    const vec3 rw = V(((iv[0] * rvx + iv[4] * rvy) + iv[8] * -1.0f) + iv[12] * 0.0f,
                      ((iv[1] * rvx + iv[5] * rvy) + iv[9] * -1.0f) + iv[13] * 0.0f,
                      ((iv[2] * rvx + iv[6] * rvy) + iv[10] * -1.0f) + iv[14] * 0.0f);
    const vec3 dir = normalize(rw);
    const vec3 viewPos = V(f.ViewPos);
    const vec3 skyColor = SampleSky(sky.faces, sky.size, sky.color, dir);
    float t1, t2;
    if (!(DbgRayBox(viewPos, dir, g.gmin, g.gmax, t1, t2) && t2 > 0.0f)) {
        out[0] = skyColor.x; out[1] = skyColor.y; out[2] = skyColor.z; out[3] = 1.0f;   // every sky the library holds has alpha 1
        return;
    }
    const bool isInsideGrid = t1 < 0.0f && t2 > 0.0f;       // never: t1 >= 0
    const vec3 origin = isInsideGrid ? viewPos : viewPos + dir * t1;
    const f4 c = vx_trace_cone(g, origin, dir, V(0.0f, 0.0f, 0.0f), coneAngle, stepMultiplier, 0.0f, 1.0f, steps);
    const float k = 1.0f - c.w;
    out[0] = c.x + k * skyColor.x; out[1] = c.y + k * skyColor.y; out[2] = c.z + k * skyColor.z; out[3] = c.w + k * 1.0f;
}

} // namespace

extern "C" {

// Voxelizer.DebugRender on the CPU. levels: the grid's rgba16f levels back to back (level 0 first), bounds from ci (GridMax
// kept >= GridMin + 0.1 as idkvx_set_grid keeps it); sky: NULL is black. out: rgba32f [h][w]; steps: the cone samples.
ORACLE_API int oracle_vx_debug_render(const IdkVxCreateInfo* ci, const uint16_t* levels, const IdkPtSkyDesc* sky, const GpuPerFrameData* frame,
                                      float stepMultiplier, float coneAngle, int w, int h, float* out, uint64_t* stepsOut, int threads) {
    if (!ci || !levels || !frame || !out || w < 1 || h < 1) return -1;
    VxGrid g;
    g.size[0] = ci->Width; g.size[1] = ci->Height; g.size[2] = ci->Depth;
    for (int i = 0; i < 3; i++) { g.gmin[i] = ci->GridMin[i]; g.gmax[i] = std::max(ci->GridMax[i], ci->GridMin[i] + 0.1f); }
    const int mx = std::max(g.size[0], std::max(g.size[1], g.size[2]));
    g.levels = 1;
    while ((mx >> g.levels) > 0) g.levels++;
    g.mip.resize(g.levels);
    uint64_t off = 0;
    for (int l = 0; l < g.levels; l++) {
        const size_t n = (size_t)g.lsize(l, 0) * g.lsize(l, 1) * g.lsize(l, 2);
        g.mip[l].assign(levels + off * 4, levels + (off + n) * 4);
        off += n;
    }
    const float black[3] = {0.0f, 0.0f, 0.0f};
    DbgSky s;
    for (int i = 0; i < 6; i++) s.faces[i] = sky ? sky->Faces[i] : nullptr;
    s.size = sky ? sky->FaceSize : 0;
    s.color = sky ? sky->Color : black;
    const int T = std::max(1, threads);
    std::vector<uint64_t> stepAcc(T, 0);
    parallel_for((size_t)w * h, T, [&](size_t b, size_t e, int tid) {
        for (size_t p = b; p < e; p++) DbgPixel(g, s, *frame, stepMultiplier, coneAngle, (int)(p % w), (int)(p / w), w, h, out + 4 * p, stepAcc[tid]);
    });
    if (stepsOut) { *stepsOut = 0; for (uint64_t v : stepAcc) *stepsOut += v; }
    return 0;
}

} // extern "C"
