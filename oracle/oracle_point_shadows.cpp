// ORACLE (TEST INFRASTRUCTURE ONLY) -- point-shadow cube maps and the voxeliser's PCF lookup into them.
//
// Built as its own library (tests/point_shadow_oracle.py -> oracle/liboracle_point_shadows.so). It compiles oracle.cpp into
// the same translation unit and reuses its scene access, TraceRay, GetSurface and VXGI helpers unchanged; what it adds is
// restated here.
//
// Restated sources (relative to the reference repository's IDKEngine):
//   Source/Render/CpuPointShadow.cs:116-232                 the raster pass (depth test only, no culling, D16Unorm, Fill(1.0)),
//                                                            sampled at texel centres; the shadow sampler (LINEAR, compare LESS)
//   Resource/Shaders/include/Math.glsl:59-66                GetLogarithmicDepth
//   Resource/Shaders/VXGI/Voxelize/Voxelize/fragment.glsl:31-117   fragment stage incl. Visibility() / GetLightSpaceDepth
//   OpenGL 4.6 spec 8.13 (table 8.19), 8.14.2, 8.17 (seamless cube maps), 8.23.1 (depth compare)
#include "oracle.cpp"

namespace {

// GetLogarithmicDepth (Math.glsl:59-66)
static inline float GetLogarithmicDepth(float nearPlane, float farPlane, float viewZ) {
    return (1.0f / viewZ - 1.0f / nearPlane) / (1.0f / farPlane - 1.0f / nearPlane);
}

// Direction of table 8.19's (face, sc, tc) with major component 1.
static inline vec3 CubeDir(int face, float sc, float tc) {
    switch (face) {
        case 0: return V(1.0f, -tc, -sc);
        case 1: return V(-1.0f, -tc, sc);
        case 2: return V(sc, 1.0f, tc);
        case 3: return V(sc, -1.0f, -tc);
        case 4: return V(sc, -tc, 1.0f);
        default: return V(-sc, -tc, -1.0f);
    }
}

// One shadow's cube map as the engine's raster pass draws it, sampled at texel centres: texel (x, y) of face f of size N looks
// along (sc, tc) = ((2x+1)/N - 1, (2y+1)/N - 1), so that the ray parameter is the face's view depth. Near clipping: the ray
// starts at Position + dir * NearPlane; far clipping: TMax = Far - Near. Only faces in faceMask are written.
static void PointShadowRender(const Scene& s, const GpuPointShadow& ps, int size, uint32_t faceMask, uint16_t* map) {
    const float nearPlane = ps.NearPlane, farPlane = ps.FarPlane;
    for (int f = 0; f < 6; f++) {
        if (!(faceMask & (1u << f))) continue;
        for (int y = 0; y < size; y++)
            for (int x = 0; x < size; x++) {
                const float sc = (float)(2 * x + 1) / (float)size - 1.0f, tc = (float)(2 * y + 1) / (float)size - 1.0f;
                const vec3 dir = CubeDir(f, sc, tc);
                const Ray ray = {V(ps.Position) + dir * nearPlane, dir};
                HitInfo hit;
                Counters cnt = {0, 0, 0, 0.0f};
                uint16_t v = 65535;
                if (TraceRay(s, ray, hit, cnt, false, farPlane - nearPlane)) {
                    const float d = GetLogarithmicDepth(nearPlane, farPlane, nearPlane + hit.T);
                    v = (uint16_t)floorf(clampf(d, 0.0f, 1.0f) * 65535.0f + 0.5f);
                }
                map[((size_t)f * size + y) * size + x] = v;
            }
    }
}

// Bilinear footprint of a cube-map lookup: face selection and (s,t) per table 8.19 (major axis; ties x >= y >= z), the four
// texels (x fastest) and the weights. A texel beyond an edge is taken from the face across it (8.17); texel centres are kept
// as odd integers c = 2*texel + 1 - size on the cube [-size, size]^3, so crossing an edge is an exact integer fold. The tap
// that lies outside in both directions at a cube corner has no texel (corner = its index, else -1).
struct CubeTaps { int face[4], x[4], y[4]; float fx, fy; int corner; };
static CubeTaps CubeFootprint(int size, vec3 d) {
    const float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
    int face;
    float sc, tc, ma;
    if (ax >= ay && ax >= az) { face = d.x >= 0.0f ? 0 : 1; sc = d.x >= 0.0f ? -d.z : d.z; tc = -d.y; ma = ax; }
    else if (ay >= az) { face = d.y >= 0.0f ? 2 : 3; sc = d.x; tc = d.y >= 0.0f ? d.z : -d.z; ma = ay; }
    else { face = d.z >= 0.0f ? 4 : 5; sc = d.z >= 0.0f ? d.x : -d.x; tc = -d.y; ma = az; }
    const float s = 0.5f * (sc / ma + 1.0f), t = 0.5f * (tc / ma + 1.0f);
    const float px = s * (float)size - 0.5f, py = t * (float)size - 0.5f;
    const float fx0 = floorf(px), fy0 = floorf(py);
    CubeTaps r;
    r.fx = px - fx0; r.fy = py - fy0;
    const int x0 = (int)fx0, y0 = (int)fy0;
    r.corner = -1;
    for (int k = 0; k < 4; k++) {
        const int x = x0 + (k & 1), y = y0 + (k >> 1);
        r.face[k] = face; r.x[k] = x; r.y[k] = y;
        const bool outX = x < 0 || x >= size, outY = y < 0 || y >= size;
        if (outX && outY) { r.corner = k; r.x[k] = r.y[k] = 0; continue; }
        if (!outX && !outY) continue;
        const int s2 = 2 * x + 1 - size, t2 = 2 * y + 1 - size;
        int P[3];
        switch (face) {
            case 0: P[0] = size; P[1] = -t2; P[2] = -s2; break;
            case 1: P[0] = -size; P[1] = -t2; P[2] = s2; break;
            case 2: P[0] = s2; P[1] = size; P[2] = t2; break;
            case 3: P[0] = s2; P[1] = -size; P[2] = -t2; break;
            case 4: P[0] = s2; P[1] = -t2; P[2] = size; break;
            default: P[0] = -s2; P[1] = -t2; P[2] = -size; break;
        }
        const int major = face >> 1;                       // axis of the face we came from
        int over = -1;
        for (int c = 0; c < 3; c++) if (P[c] > size || P[c] < -size) over = c;
        P[over] = P[over] > 0 ? size : -size;              // the overhanging coordinate lands on the neighbouring face ...
        P[major] += P[major] > 0 ? -1 : 1;                 // ... one half-texel step in from the shared edge
        int nf, ns, nt;
        if (over == 0) { nf = P[0] > 0 ? 0 : 1; ns = P[0] > 0 ? -P[2] : P[2]; nt = -P[1]; }
        else if (over == 1) { nf = P[1] > 0 ? 2 : 3; ns = P[0]; nt = P[1] > 0 ? P[2] : -P[2]; }
        else { nf = P[2] > 0 ? 4 : 5; ns = P[2] > 0 ? P[0] : -P[0]; nt = -P[1]; }
        r.face[k] = nf; r.x[k] = (ns + size - 1) / 2; r.y[k] = (nt + size - 1) / 2;
    }
    return r;
}

// Visibility(pointShadow, lightToSample) (fragment.glsl:100-117) = texture(samplerCubeShadow, vec4(lightToSample, depth)) with
// the engine's shadow sampler (CpuPointShadow.SetSizeShadowMap:211-218: LINEAR, CompareRefToTexture, LESS) and seamless
// filtering. Reference depth: GetLightSpaceDepth of lightToSample * (1 - 0.02), clamped to [0, 1] (fixed-point depth format,
// 8.23.1). Texel selection first (CubeFootprint of the unbiased direction; at a cube corner the missing depth is the mean of
// the three defined ones), then each texel compares ref < D16 / 65535, then the results are filtered with the bilinear weights
// (mix order). A sample at the light itself is visible.
static float PointShadowVisibility(const GpuPointShadow& ps, int size, const uint16_t* map, vec3 lightToSample) {
    const float bias = 0.02f;
    const vec3 b = lightToSample * (1.0f - bias);
    const float dist = fmaxf(fabsf(b.x), fmaxf(fabsf(b.y), fabsf(b.z)));
    if (!(dist > 0.0f)) return 1.0f;
    const float ref = clampf(GetLogarithmicDepth(ps.NearPlane, ps.FarPlane, dist), 0.0f, 1.0f);
    const CubeTaps f = CubeFootprint(size, lightToSample);
    float d[4];
    for (int k = 0; k < 4; k++) d[k] = k == f.corner ? 0.0f : (float)map[((size_t)f.face[k] * size + f.y[k]) * size + f.x[k]] / 65535.0f;
    if (f.corner >= 0) d[f.corner] = ((d[0] + d[1]) + (d[2] + d[3])) / 3.0f;
    float c[4];
    for (int k = 0; k < 4; k++) c[k] = ref < d[k] ? 1.0f : 0.0f;
    return mixf(mixf(c[0], c[1], f.fx), mixf(c[2], c[3], f.fx), f.fy);
}

// The cube maps of the voxeliser's shadow-map mode: `count` shadows, their face sizes, the maps back to back.
struct ShadowMaps {
    const GpuPointShadow* shadows;
    const int32_t* sizes;
    const uint16_t* texels;
    std::vector<size_t> offsets;
};

// Voxelize/fragment.glsl:31-79 as vx_fragment (oracle_vxgi.inc), with the point-shadowed lights multiplied by the PCF lookup.
static vec3 vx_fragment_pcf(const Scene& s, const ShadowMaps& m, const GpuMaterial& mat, float emissiveBias, vec3 fragPos, vec3 normal,
                            float tu, float tv, float& alpha) {
    Surface surf = GetSurface(s.d, mat, tu, tv);
    surf.Emissive = surf.Emissive + emissiveBias * surf.Albedo;
    vec3 direct = V(0, 0, 0);
    for (uint64_t i = 0; i < s.d.LightCount; i++) {
        const GpuLight& L = s.d.Lights[i];
        vec3 sampleToLight = V(L.Position) - fragPos;
        float dist = sqrtf(dot(sampleToLight, sampleToLight));
        vec3 lightDir = sampleToLight / dist;
        float cosTheta = dot(normalize(normal), lightDir);
        if (cosTheta > 0.0f) {
            vec3 diffuse = V(L.Color) * cosTheta * surf.Albedo;
            float lr = fmaxf(L.Radius, 0.0001f);
            float dsq = fmaxf(dist * dist, 0.0001f);
            float attenuation = (lr * lr) / dsq;
            vec3 contrib = diffuse * attenuation;
            if (L.PointShadowIndex >= 0) {   // Visibility(pointShadow, -sampleToLight), fragment.glsl:55-58
                const int k = L.PointShadowIndex;
                contrib = contrib * PointShadowVisibility(m.shadows[k], m.sizes[k], m.texels + m.offsets[k], -sampleToLight);
            }
            direct = direct + contrib;
        }
    }
    direct = direct + surf.Albedo * 0.02f;
    direct = direct + surf.Emissive;
    alpha = surf.Alpha;
    return direct * surf.Alpha;
}

// vx_voxelize (oracle_vxgi.inc) under the product's coverage rule, with vx_fragment_pcf as the fragment stage.
static void vx_voxelize_pcf(const Scene& s, const ShadowMaps& m, VxGrid& g, uint64_t* fragments) {
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
                for (int a = 0; a < 3; a++) uvw[c][a] = ((a == 0 ? P[c].x : a == 1 ? P[c].y : P[c].z) - g.gmin[a]) / ext[a];
            }
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
            const float mina = fminf(qa[0], fminf(qa[1], qa[2])), maxa = fmaxf(qa[0], fmaxf(qa[1], qa[2]));
            const float minb = fminf(qb[0], fminf(qb[1], qb[2])), maxb = fmaxf(qb[0], fmaxf(qb[1], qb[2]));
            const int i0 = std::max(0, (int)ceilf(mina - 0.5f)), i1 = std::min(g.size[a] - 1, (int)floorf(maxa - 0.5f));
            const int j0 = std::max(0, (int)ceilf(minb - 0.5f)), j1 = std::min(g.size[b] - 1, (int)floorf(maxb - 0.5f));
            const GpuMesh& mesh = s.d.Meshes[tri.MeshId];
            const GpuMaterial& mat = s.d.Materials[mesh.MaterialId];
            for (int j = j0; j <= j1; j++)
                for (int i = i0; i <= i1; i++) {
                    const float cx = (float)i + 0.5f, cy = (float)j + 0.5f;
                    const float w0 = edge(qa[1], qb[1], qa[2], qb[2], cx, cy);
                    const float w1 = edge(qa[2], qb[2], qa[0], qb[0], cx, cy);
                    const float w2 = edge(qa[0], qb[0], qa[1], qb[1], cx, cy);
                    const bool inside = area > 0.0f ? (w0 >= 0.0f && w1 >= 0.0f && w2 >= 0.0f) : (w0 <= 0.0f && w1 <= 0.0f && w2 <= 0.0f);
                    if (!inside) continue;
                    const float b0 = w0 / area, b1 = w1 / area, b2 = w2 / area;
                    vec3 fragPos = (P[0] * b0 + P[1] * b1) + P[2] * b2;
                    vec3 normal = (N[0] * b0 + N[1] * b1) + N[2] * b2;
                    const float fu = (fragPos.x - g.gmin[0]) / ext[0], fv = (fragPos.y - g.gmin[1]) / ext[1], fw = (fragPos.z - g.gmin[2]) / ext[2];
                    if (!(fu >= 0.0f && fv >= 0.0f && fw >= 0.0f)) continue;
                    const int vx = (int)(fu * (float)g.size[0]), vy = (int)(fv * (float)g.size[1]), vz = (int)(fw * (float)g.size[2]);
                    if (vx >= g.size[0] || vy >= g.size[1] || vz >= g.size[2]) continue;
                    float alpha;
                    const GpuVertex& tv0 = s.d.Vertices[vid[0]]; const GpuVertex& tv1 = s.d.Vertices[vid[1]]; const GpuVertex& tv2 = s.d.Vertices[vid[2]];
                    const float tu = (tv0.TexCoord[0] * b0 + tv1.TexCoord[0] * b1) + tv2.TexCoord[0] * b2;
                    const float tv = (tv0.TexCoord[1] * b0 + tv1.TexCoord[1] * b1) + tv2.TexCoord[1] * b2;
                    vec3 val = vx_fragment_pcf(s, m, mat, mesh.EmissiveBias, fragPos, normal, tu, tv, alpha);
                    const size_t vi = ((size_t)vz * g.size[1] + vy) * g.size[0] + vx;
                    uint32_t bits[3];
                    memcpy(&bits[0], &val.x, 4); memcpy(&bits[1], &val.y, 4); memcpy(&bits[2], &val.z, 4);
                    for (int c = 0; c < 3; c++) rb[vi * 3 + c] = std::max(rb[vi * 3 + c], bits[c]);
                    written[vi] = 1;
                    frags++;
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

} // namespace

extern "C" {

// One shadow's cube map (6 * size^2 D16 texels, face-major), faces outside faceMask untouched (idkpt_render_point_shadows).
ORACLE_API void oracle_point_shadow_render(const IdkPtSceneDesc* scene, const GpuPointShadow* shadow, int size, uint32_t faceMask, uint16_t* inout) {
    Scene s; s.d = *scene;
    PointShadowRender(s, *shadow, size, faceMask, inout);
}

// The PCF lookup on its own, for n directions into one map.
ORACLE_API void oracle_point_shadow_visibility(const GpuPointShadow* shadow, int size, const uint16_t* map, const float* lightToSample,
                                               uint64_t n, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = PointShadowVisibility(*shadow, size, map, V(lightToSample + 3 * i));
}

// Voxelizer.Render() with the voxeliser's shadow-map mode (idkvx_set_shadow_maps): `count` shadows with their face sizes and
// maps back to back; every light's PointShadowIndex must be < count. levelsOut: rgba16f levels concatenated (level 0 first).
ORACLE_API int oracle_vx_voxelize_shadow_maps(const IdkPtSceneDesc* scene, const IdkVxCreateInfo* ci, const GpuPointShadow* shadows,
                                              const int32_t* sizes, const uint16_t* texels, int count, uint16_t* levelsOut,
                                              uint64_t capacityTexels, uint64_t* fragments, int threads) {
    for (uint64_t i = 0; i < scene->LightCount; i++)
        if (scene->Lights[i].PointShadowIndex >= count) return -2;
    Scene s; s.d = *scene;
    ShadowMaps m = {shadows, sizes, texels, std::vector<size_t>(std::max(count, 0), 0)};
    for (int i = 1; i < count; i++) m.offsets[i] = m.offsets[i - 1] + 6 * (size_t)sizes[i - 1] * (size_t)sizes[i - 1];
    VxGrid g;
    g.size[0] = ci->Width; g.size[1] = ci->Height; g.size[2] = ci->Depth;
    for (int i = 0; i < 3; i++) { g.gmin[i] = ci->GridMin[i]; g.gmax[i] = ci->GridMax[i]; }
    const int mx = std::max(g.size[0], std::max(g.size[1], g.size[2]));
    g.levels = 1;
    while ((mx >> g.levels) > 0) g.levels++;
    g.mip.resize(g.levels);
    vx_voxelize_pcf(s, m, g, fragments);
    vx_mipmap(g, threads);
    uint64_t off = 0;
    for (int l = 0; l < g.levels; l++) {
        if (off + g.mip[l].size() / 4 > capacityTexels) return -1;
        memcpy(levelsOut + off * 4, g.mip[l].data(), g.mip[l].size() * 2);
        off += g.mip[l].size() / 4;
    }
    return g.levels;
}

} // extern "C"
