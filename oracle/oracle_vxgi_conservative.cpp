// ORACLE (TEST INFRASTRUCTURE ONLY) -- the voxeliser under Voxelizer.IsConservativeRasterization.
//
// Part of liboracle.so (wrapped by tests/vxgi_conservative_oracle.py). It includes oracle_point_shadows.cpp (and with it
// oracle.cpp and oracle_vxgi.inc) and reuses the
// projection, both fragment stages (vx_fragment: shadow rays; vx_fragment_pcf: the PCF lookup), the merge and the mip chain
// unchanged; what it adds is the coverage rule, stated in DESIGN.md section 7 and restated here.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Source/Render/VXGI/Voxelizer/Voxelizer.cs:41-56,142     IsConservativeRasterization -> GL_NV_conservative_raster
//   Resource/Shaders/VXGI/Voxelize/Voxelize/{vertex,geometry,fragment}.glsl   as in oracle_vxgi.inc
#pragma once
#include "oracle_point_shadows.cpp"

#include <climits>

namespace {

// The conservative coverage rule: a pixel is covered when its closed square [i, i+1] x [j, j+1] meets the projected triangle.
// Exact separating-axis test on the fp32 window coordinates: the square's two normals are the bounding-box restriction of
// the visited pixels, each edge normal is the edge function at the pixel centre widened by r_k = 0.5 (|da_k| + |db_k|), the
// most it gains anywhere in the square. Attributes stay at the pixel centre (extrapolated outside the triangle, like GL's
// non-centroid inputs).
struct VxConservativeRule {
    float r[3] = {0.0f, 0.0f, 0.0f};
    // the pixels whose closed square meets the closed bounding box, clamped to the plane; and the per-edge widening
    void setup(const float qa[3], const float qb[3], int sa, int sb, int& i0, int& i1, int& j0, int& j1) {
        const float mina = fminf(qa[0], fminf(qa[1], qa[2])), maxa = fmaxf(qa[0], fmaxf(qa[1], qa[2]));
        const float minb = fminf(qb[0], fminf(qb[1], qb[2])), maxb = fmaxf(qb[0], fmaxf(qb[1], qb[2]));
        i0 = std::max(0, (int)(ceilf(mina) - 1.0f)); i1 = std::min(sa - 1, (int)floorf(maxa));
        j0 = std::max(0, (int)(ceilf(minb) - 1.0f)); j1 = std::min(sb - 1, (int)floorf(maxb));
        r[0] = 0.5f * (fabsf(qa[2] - qa[1]) + fabsf(qb[2] - qb[1]));
        r[1] = 0.5f * (fabsf(qa[0] - qa[2]) + fabsf(qb[0] - qb[2]));
        r[2] = 0.5f * (fabsf(qa[1] - qa[0]) + fabsf(qb[1] - qb[0]));
    }
    // w0..w2: the edge functions at the pixel centre, in the order of the centre rule
    bool covers(float area, float w0, float w1, float w2) const {
        return area > 0.0f ? (w0 + r[0] >= 0.0f && w1 + r[1] >= 0.0f && w2 + r[2] >= 0.0f)
                           : (w0 - r[0] <= 0.0f && w1 - r[1] <= 0.0f && w2 - r[2] <= 0.0f);
    }
};

// int(f) of a voxel coordinate f >= 0 as the device's cvt.rzi.s32.f32 computes it: saturated at INT_MAX (an extrapolated
// FragPos can lie arbitrarily far outside the grid; x86's conversion would wrap it to a negative index)
static inline int vx_voxel_coord(float f) { return f < 2147483648.0f ? (int)f : INT_MAX; }

// vx_voxelize (oracle_vxgi.inc) with the conservative rule; `fragment(mat, emissiveBias, fragPos, normal, tu, tv, alpha)`
// is the fragment stage (vx_fragment or vx_fragment_pcf).
template <class Fragment>
static void vx_voxelize_conservative(const Scene& s, VxGrid& g, uint64_t* fragments, const Fragment& fragment) {
    const size_t n0 = (size_t)g.size[0] * g.size[1] * g.size[2];
    std::vector<uint32_t> rb(n0 * 3, 0);   // float bits, atomicMax semantics
    std::vector<uint8_t> written(n0, 0);
    uint64_t frags = 0;
    const float ext[3] = {g.gmax[0] - g.gmin[0], g.gmax[1] - g.gmin[1], g.gmax[2] - g.gmin[2]};
    for (uint64_t ii = 0; ii < s.d.BlasInstanceCount; ii++) {
        const GpuBlasInstance& inst = s.d.BlasInstances[ii];
        const GpuBlasDesc& desc = s.d.BlasDescs[inst.BlasId];
        const GpuMeshTransform& mt = s.d.MeshTransforms[inst.MeshTransformId];
        auto toWorldN = [&](vec3 v) {
            const float (*im)[4] = mt.InvModelMatrix;
            return vec3{(im[0][0] * v.x + im[1][0] * v.y) + im[2][0] * v.z, (im[0][1] * v.x + im[1][1] * v.y) + im[2][1] * v.z,
                        (im[0][2] * v.x + im[1][2] * v.y) + im[2][2] * v.z};
        };
        for (int32_t k = desc.TriangleOffset; k < desc.TriangleOffset + desc.TriangleCount; k++) {
            const GpuBlasTriangle& tri = s.d.BlasTriangles[k];
            const int32_t vid[3] = {tri.X, tri.Y, tri.Z};
            vec3 P[3], N[3];
            float uvw[3][3];
            for (int c = 0; c < 3; c++) {
                Ray tmp = RayTransform(Ray{pos(s, vid[c]), V(0, 0, 0)}, mt.ModelMatrix);
                P[c] = tmp.o;
                N[c] = normalize(toWorldN(DecompressSR11G11B10(s.d.Vertices[vid[c]].Normal)));
                uvw[c][0] = (P[c].x - g.gmin[0]) / ext[0];
                uvw[c][1] = (P[c].y - g.gmin[1]) / ext[1];
                uvw[c][2] = (P[c].z - g.gmin[2]) / ext[2];
            }
            // geometry.glsl: dominant axis of the NDC-space normal
            vec3 n0v = {uvw[0][0] * 2.0f - 1.0f, uvw[0][1] * 2.0f - 1.0f, uvw[0][2] * 2.0f - 1.0f};
            vec3 n1v = {uvw[1][0] * 2.0f - 1.0f, uvw[1][1] * 2.0f - 1.0f, uvw[1][2] * 2.0f - 1.0f};
            vec3 n2v = {uvw[2][0] * 2.0f - 1.0f, uvw[2][1] * 2.0f - 1.0f, uvw[2][2] * 2.0f - 1.0f};
            vec3 cr = cross(n1v - n0v, n2v - n0v);
            float nw[3] = {fabsf(cr.x), fabsf(cr.y), fabsf(cr.z)};
            int dom = nw[1] > nw[0] ? 1 : 0;
            dom = nw[2] > nw[dom] ? 2 : dom;
            const int a = (dom + 1) % 3, b = (dom + 2) % 3;
            float qa[3], qb[3];
            for (int c = 0; c < 3; c++) { qa[c] = uvw[c][a] * (float)g.size[a]; qb[c] = uvw[c][b] * (float)g.size[b]; }
            auto edge = [](float ax, float ay, float bx, float by, float cx, float cy) { return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax); };
            const float area = edge(qa[0], qb[0], qa[1], qb[1], qa[2], qb[2]);
            if (area == 0.0f || !(area == area)) continue;
            int i0, i1, j0, j1;
            VxConservativeRule rule;
            rule.setup(qa, qb, g.size[a], g.size[b], i0, i1, j0, j1);
            const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
            const GpuMaterial& mat = s.d.Materials[mesh.MaterialId];
            for (int j = j0; j <= j1; j++) {
                for (int i = i0; i <= i1; i++) {
                    const float cx = (float)i + 0.5f, cy = (float)j + 0.5f;
                    const float w0 = edge(qa[1], qb[1], qa[2], qb[2], cx, cy);
                    const float w1 = edge(qa[2], qb[2], qa[0], qb[0], cx, cy);
                    const float w2 = edge(qa[0], qb[0], qa[1], qb[1], cx, cy);
                    if (!rule.covers(area, w0, w1, w2)) continue;
                    const float b0 = w0 / area, b1 = w1 / area, b2 = w2 / area;
                    vec3 fragPos = (P[0] * b0 + P[1] * b1) + P[2] * b2;
                    vec3 normal = (N[0] * b0 + N[1] * b1) + N[2] * b2;
                    const float fu = (fragPos.x - g.gmin[0]) / ext[0], fv = (fragPos.y - g.gmin[1]) / ext[1], fw = (fragPos.z - g.gmin[2]) / ext[2];
                    if (!(fu >= 0.0f && fv >= 0.0f && fw >= 0.0f)) continue;
                    const int vx = vx_voxel_coord(fu * (float)g.size[0]), vy = vx_voxel_coord(fv * (float)g.size[1]), vz = vx_voxel_coord(fw * (float)g.size[2]);
                    if (vx >= g.size[0] || vy >= g.size[1] || vz >= g.size[2]) continue;
                    float alpha;
                    const GpuVertex& tv0 = s.d.Vertices[vid[0]]; const GpuVertex& tv1 = s.d.Vertices[vid[1]]; const GpuVertex& tv2 = s.d.Vertices[vid[2]];
                    const float tu = (tv0.TexCoord[0] * b0 + tv1.TexCoord[0] * b1) + tv2.TexCoord[0] * b2;
                    const float tv = (tv0.TexCoord[1] * b0 + tv1.TexCoord[1] * b1) + tv2.TexCoord[1] * b2;
                    vec3 val = fragment(mat, mesh.EmissiveBias, fragPos, normal, tu, tv, alpha);
                    const size_t vi = ((size_t)vz * g.size[1] + vy) * g.size[0] + vx;
                    uint32_t bits[3];
                    memcpy(&bits[0], &val.x, 4); memcpy(&bits[1], &val.y, 4); memcpy(&bits[2], &val.z, 4);
                    for (int c = 0; c < 3; c++) rb[vi * 3 + c] = std::max(rb[vi * 3 + c], bits[c]);
                    written[vi] = 1;
                    frags++;
                }
            }
        }
    }
    g.mip[0].assign(n0 * 4, 0);
    for (size_t vi = 0; vi < n0; vi++) {
        if (!written[vi]) continue;
        for (int c = 0; c < 3; c++) { float f; memcpy(&f, &rb[vi * 3 + c], 4); g.mip[0][vi * 4 + c] = f32_to_f16(f); }
        g.mip[0][vi * 4 + 3] = f32_to_f16(1.0f);
    }
    if (fragments) *fragments = frags;
}

static VxGrid vx_grid(const IdkVxCreateInfo* ci) {
    VxGrid g;
    g.size[0] = ci->Width; g.size[1] = ci->Height; g.size[2] = ci->Depth;
    for (int i = 0; i < 3; i++) { g.gmin[i] = ci->GridMin[i]; g.gmax[i] = ci->GridMax[i]; }
    const int mx = std::max(g.size[0], std::max(g.size[1], g.size[2]));
    g.levels = 1;
    while ((mx >> g.levels) > 0) g.levels++;
    g.mip.resize(g.levels);
    return g;
}

static int vx_copy_out(const VxGrid& g, uint16_t* levelsOut, uint64_t capacityTexels) {
    uint64_t off = 0;
    for (int l = 0; l < g.levels; l++) {
        if (off + g.mip[l].size() / 4 > capacityTexels) return -1;
        memcpy(levelsOut + off * 4, g.mip[l].data(), g.mip[l].size() * 2);
        off += g.mip[l].size() / 4;
    }
    return g.levels;
}

} // namespace

extern "C" {

// Voxelizer.Render() with IsConservativeRasterization on; point-shadowed lights by shadow rays (idkvx_set_shadow_tracer).
// levelsOut: rgba16f levels concatenated (level 0 first). Returns the level count.
ORACLE_API int oracle_vx_voxelize_conservative(const IdkPtSceneDesc* scene, const IdkVxCreateInfo* ci, uint16_t* levelsOut,
                                               uint64_t capacityTexels, uint64_t* fragments, int threads) {
    Scene s; s.d = *scene;
    VxGrid g = vx_grid(ci);
    vx_voxelize_conservative(s, g, fragments, [&](const GpuMaterial& mat, float bias, vec3 p, vec3 n, float tu, float tv, float& alpha) {
        return vx_fragment(s, mat, bias, p, n, tu, tv, alpha);
    });
    vx_mipmap(g, threads);
    return vx_copy_out(g, levelsOut, capacityTexels);
}

// The same with the voxeliser's shadow-map mode (idkvx_set_shadow_maps), arguments as oracle_vx_voxelize_shadow_maps.
ORACLE_API int oracle_vx_voxelize_conservative_shadow_maps(const IdkPtSceneDesc* scene, const IdkVxCreateInfo* ci, const GpuPointShadow* shadows,
                                                           const int32_t* sizes, const uint16_t* texels, int count, uint16_t* levelsOut,
                                                           uint64_t capacityTexels, uint64_t* fragments, int threads) {
    for (uint64_t i = 0; i < scene->LightCount; i++)
        if (scene->Lights[i].PointShadowIndex >= count) return -2;
    Scene s; s.d = *scene;
    ShadowMaps m = {shadows, sizes, texels, std::vector<size_t>(std::max(count, 0), 0)};
    for (int i = 1; i < count; i++) m.offsets[i] = m.offsets[i - 1] + 6 * (size_t)sizes[i - 1] * (size_t)sizes[i - 1];
    VxGrid g = vx_grid(ci);
    vx_voxelize_conservative(s, g, fragments, [&](const GpuMaterial& mat, float bias, vec3 p, vec3 n, float tu, float tv, float& alpha) {
        return vx_fragment_pcf(s, m, mat, bias, p, n, tu, tv, alpha);
    });
    vx_mipmap(g, threads);
    return vx_copy_out(g, levelsOut, capacityTexels);
}

} // extern "C"
