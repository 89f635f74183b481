"""Point-shadow cube maps and the voxeliser's PCF lookup: the oracle against independent float64 definitions (no GPU).

1. the traced cube map against a float64 brute-force ray cast over every world-space triangle;
2. the PCF lookup against a float64 restatement of GL 4.6 face selection (8.13), seamless bilinear filtering (8.14.2, 8.17)
   and depth compare LESS (8.23.1);
3. the face layout against the engine's own face matrices (CpuPointShadow.UpdateViewMatrices + CreatePerspectiveFieldOfView-
   DepthZeroToOne), i.e. the map is the one its raster pass draws, addressed the way its samplerCubeShadow addresses it;
4. the voxeliser's shadow-map mode against its shadow-ray mode on the lit Cornell box.
"""
import numpy as np

import oracle_lib as ol
import point_shadow_oracle as pso
from idkengine_b200 import host, scenes, vxgi
from raster_lib import GRID_MAX, GRID_MIN, lit_cornell


def face_dirs64(n):
    """[6, n, n, 3] float64 texel-centre directions, GL table 8.19 inverted with major component 1."""
    c = (2.0 * np.arange(n) + 1.0) / n - 1.0
    tc, sc = np.meshgrid(c, c, indexing="ij")          # [y, x]
    one = np.ones_like(sc)
    return np.stack([np.stack([one, -tc, -sc], -1), np.stack([-one, -tc, sc], -1), np.stack([sc, one, tc], -1),
                     np.stack([sc, -one, -tc], -1), np.stack([sc, -tc, one], -1), np.stack([-sc, -tc, -one], -1)])


def world_triangles(scene):
    """[T, 3, 3] float64 world-space triangles of every instance."""
    P = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float64)
    out = []
    for inst in scene.blas_instances:
        d = scene.blas_descs[inst["BlasId"]]
        tri = scene.blas_triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]]
        v = P[np.stack([tri["X"], tri["Y"], tri["Z"]], 1)]
        m = scene.mesh_transforms["ModelMatrix"][inst["MeshTransformId"]].astype(np.float64)
        out.append(v @ m[:, :3].T + m[:, 3])
    return np.concatenate(out)


def log_depth64(near, far, z):
    return (1.0 / z - 1.0 / near) / (1.0 / far - 1.0 / near)


def cast64(tris, origins, dirs, tmax, eps):
    """Closest double-sided hit t per ray (inf = none) and a flag for rays that pass within eps (barycentric) of a triangle
    edge or within eps of the clip range's ends."""
    p0, e1, e2 = tris[:, 0], tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0]
    best = np.full(len(origins), np.inf)
    near_edge = np.zeros(len(origins), bool)
    for a in range(0, len(origins), 512):
        o, d = origins[a:a + 512, None], dirs[a:a + 512, None]
        pv = np.cross(d, e2)
        det = np.einsum("rtk,tk->rt", pv, e1)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            tv = o - p0
            u = np.einsum("rtk,rtk->rt", tv, pv) * inv
            qv = np.cross(tv, e1)
            v = np.einsum("rtk,rtk->rt", d, qv) * inv
            t = np.einsum("tk,rtk->rt", e2, qv) * inv
        w = 1.0 - u - v
        mb = np.minimum(np.minimum(u, v), w)
        inrange = (t >= -eps) & (t <= tmax + eps) & np.isfinite(t)
        hit = (mb >= 0) & (t >= 0) & (t < tmax) & np.isfinite(t)
        best[a:a + 512] = np.where(hit, t, np.inf).min(1)
        near_edge[a:a + 512] = (inrange & (np.abs(mb) < eps)).any(1) | (inrange & (mb >= -eps) & ((np.abs(t) < eps) | (np.abs(t - tmax) < eps))).any(1)
    return best, near_edge


def test_cube_map_matches_float64_ray_cast():
    """A light inside the Cornell box: near = 0.35 clips the top of the metal sphere (0.3 below the light), so its inside
    shows; far = 1.25 puts the red wall (1.3 away along -X) beyond the far plane while the floor and ceiling of that face stay."""
    scene, cam = scenes.cornell_1k(threads=1)
    pos, near, far, n = (0.3, 1.1, 0.2), 0.35, 1.25, 32
    m = pso.point_shadow_render(scene, scenes.point_shadows([(pos, near, far, 0)]), n)
    dirs = face_dirs64(n).reshape(-1, 3)
    origins = np.asarray(pos, np.float64) + dirs * near
    t, flagged = cast64(world_triangles(scene), origins, dirs, far - near, 1e-5)
    hit = np.isfinite(t)
    d = np.clip(log_depth64(near, far, near + np.where(hit, t, 1.0)), 0.0, 1.0) * 65535.0 + 0.5
    ref = np.where(hit, np.floor(d), 65535).astype(np.uint16)
    frac = d - np.floor(d)
    # within the fp32 pipeline's rounding of a D16 boundary: near the near plane a D16 step is ~5e-6 in distance, so the
    # float32 origin and hit distance (relative error ~1e-7) move the depth by up to ~0.02 of a step
    flagged |= hit & ((frac < 0.05) | (frac > 1 - 0.05))
    got = m.ravel()
    bad = got != ref
    assert not (bad & ~flagged).any(), np.flatnonzero(bad & ~flagged)[:10]
    # the scene reaches every case: clipped sphere top, clipped far wall, plain hits, misses
    assert 0.5 < hit.mean() < 0.99 and (got == 65535).sum() > 100
    # measured: 319 of 6144 texels flagged (most on the diagonals of the quads), 7 of them differ from the float64 value
    assert flagged.sum() <= 400 and bad.sum() <= 12, (int(flagged.sum()), int(bad.sum()))


def gl_lookup64(m, l, ref):
    """texture(samplerCubeShadow, vec4(l, ref)) from the GL 4.6 spec in float64: 8.13 face selection (table 8.19, ties to the
    lower axis), 8.14.2 bilinear footprint, seamless filtering (8.17: a texel beyond an edge is the adjacent face's texel
    under that position, the corner texel is the mean of the other three), 8.23.1 compare LESS per texel, then filtering."""
    n = m.shape[1]

    def select(v):
        a = np.abs(v)
        if a[0] >= a[1] and a[0] >= a[2]:
            return (0, -v[2], -v[1], a[0]) if v[0] >= 0 else (1, v[2], -v[1], a[0])
        if a[1] >= a[2]:
            return (2, v[0], v[2], a[1]) if v[1] >= 0 else (3, v[0], -v[2], a[1])
        return (4, v[0], -v[1], a[2]) if v[2] >= 0 else (5, -v[0], -v[1], a[2])

    def to_dir(f, sc, tc):
        return [np.array([1, -tc, -sc]), np.array([-1, -tc, sc]), np.array([sc, 1, tc]), np.array([sc, -1, -tc]),
                np.array([sc, -tc, 1]), np.array([-sc, -tc, -1])][f]

    f, sc, tc, ma = select(l)
    u, v = 0.5 * (sc / ma + 1.0) * n - 0.5, 0.5 * (tc / ma + 1.0) * n - 0.5
    i0, j0 = int(np.floor(u)), int(np.floor(v))
    a, b = u - i0, v - j0
    depth = {}
    for (i, j) in [(i0, j0), (i0 + 1, j0), (i0, j0 + 1), (i0 + 1, j0 + 1)]:
        oi, oj = not 0 <= i < n, not 0 <= j < n
        if oi and oj:
            continue
        if not (oi or oj):
            depth[(i, j)] = m[f, j, i] / 65535.0
            continue
        g, s2, t2, ma2 = select(to_dir(f, (2 * i + 1) / n - 1, (2 * j + 1) / n - 1))
        x, y = int(np.floor(0.5 * (s2 / ma2 + 1.0) * n)), int(np.floor(0.5 * (t2 / ma2 + 1.0) * n))
        depth[(i, j)] = m[g, y, x] / 65535.0
    taps = [(i0, j0), (i0 + 1, j0), (i0, j0 + 1), (i0 + 1, j0 + 1)]
    missing = [k for k in taps if k not in depth]
    if missing:
        depth[missing[0]] = sum(depth.values()) / 3.0
    c = [1.0 if ref < depth[k] else 0.0 for k in taps]
    return (c[0] * (1 - a) + c[1] * a) * (1 - b) + (c[2] * (1 - a) + c[3] * a) * b, [depth[k] for k in taps]


def test_pcf_lookup_matches_gl_rules():
    rng = np.random.default_rng(7)
    n = 8
    m = rng.integers(20000, 60000, (6, n, n)).astype(np.uint16)
    near, far = 0.1, 10.0
    sh = scenes.point_shadows([((0.0, 0.0, 0.0), near, far, 0)])
    dirs = [rng.normal(size=(400, 3))]
    # aimed at face edges and cube corners, and exactly on them
    e = rng.uniform(-1, 1, (300, 3))
    k = rng.integers(0, 3, 300)
    e[np.arange(300), k] = np.sign(e[np.arange(300), (k + 1) % 3]) * np.abs(e[np.arange(300), (k + 1) % 3]) * rng.choice([1.0, 1 + 1e-3, 1 - 1e-3], 300)
    dirs.append(e)
    corners = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float64)
    dirs.append(np.repeat(corners, 25, 0) * (1 + rng.uniform(-0.05, 0.05, (200, 3))))
    dirs.append(corners)
    dirs = np.concatenate(dirs).astype(np.float32)
    # references: the 2 %-biased distance maps to depths across the map's range
    dist = rng.uniform(0.15, 9.0, len(dirs)).astype(np.float32)
    l = (dirs / np.abs(dirs).max(1, keepdims=True) * dist[:, None]).astype(np.float32)
    got = pso.point_shadow_visibility(sh, m, l)
    checked = agree = 0
    for i in range(len(l)):
        lv = l[i].astype(np.float64)
        ref = np.clip(log_depth64(near, far, np.abs(lv * (1 - 0.02)).max()), 0, 1)
        want, taps = gl_lookup64(m, lv, ref)
        if min(abs(ref - t) for t in taps) < 1e-5:        # compare too close to call in fp32 vs float64
            continue
        checked += 1
        assert abs(got[i] - want) <= 1e-6, (i, l[i], got[i], want)
        if all(ref < t for t in taps) or all(ref >= t for t in taps):
            agree += 1
            assert got[i] in (0.0, 1.0), (i, got[i])
    assert checked >= 0.95 * len(l) and agree > 100


def test_face_layout_matches_engine_face_matrices():
    """CpuPointShadow.UpdateViewMatrices (CpuPointShadow.cs:187-195) with MyMath.CreatePerspectiveFieldOfViewDepthZeroToOne(90 deg,
    1, near, far): every texel-centre direction projects into its own texel, and its window depth is GetLogarithmicDepth."""
    pos, near, far, n = np.array([0.3, -1.2, 2.0]), 0.25, 60.0, 16
    proj = host.perspective_zero_to_one(np.pi / 2, 1.0, near, far)
    looks = [((1, 0, 0), (0, -1, 0)), ((-1, 0, 0), (0, -1, 0)), ((0, 1, 0), (0, 0, 1)), ((0, -1, 0), (0, 0, -1)),
             ((0, 0, 1), (0, -1, 0)), ((0, 0, -1), (0, -1, 0))]
    dirs = face_dirs64(n)
    xs, ys = np.meshgrid(np.arange(n), np.arange(n))
    for f, (fwd, up) in enumerate(looks):
        pv = host.look_at(pos, pos + np.array(fwd, float), up) @ proj       # OpenTK row vectors: clip = [p, 1] @ View @ Proj
        for z in (near, 1.0, 7.5, far):
            p = pos + dirs[f] * z
            clip = np.concatenate([p, np.ones(p.shape[:2] + (1,))], -1) @ pv
            ndc = clip[..., :3] / clip[..., 3:]
            wx, wy = (ndc[..., 0] * 0.5 + 0.5) * n, (ndc[..., 1] * 0.5 + 0.5) * n
            assert np.array_equal(np.floor(wx), xs) and np.array_equal(np.floor(wy), ys), f
            assert np.allclose(wx - xs, 0.5) and np.allclose(wy - ys, 0.5)
            assert np.abs(ndc[..., 2] - log_depth64(near, far, z)).max() < 1e-6, f


def lit_cornell_shadowed():
    scene, _ = lit_cornell()
    scene.lights["PointShadowIndex"][:] = [0, 1]
    shadows = scenes.point_shadows([(l["Position"], l["Radius"], 60.0, 0) for l in scene.lights])
    return scene, shadows


def test_pcf_mode_against_shadow_rays():
    scene, shadows = lit_cornell_shadowed()
    ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    maps = [pso.point_shadow_render(scene, s, 512) for s in shadows]       # the engine's size for its startup lights
    pcf = pso.vx_voxelize_shadow_maps(scene, ci, shadows, maps)[0][0].astype(np.float32)
    dark = pso.vx_voxelize_shadow_maps(scene, ci, shadows, [np.zeros_like(m) for m in maps])[0][0].astype(np.float32)
    rays = ol.vx_voxelize(scene, ci)[0][0].astype(np.float32)
    plain = scene.lights.copy()
    scene.lights["PointShadowIndex"][:] = -1
    unshadowed = ol.vx_voxelize(scene, ci)[0][0].astype(np.float32)
    scene.lights = plain
    occ = unshadowed[..., 3] == 1.0
    for g in (pcf, dark, rays):
        assert np.array_equal(g[..., 3], unshadowed[..., 3])                       # coverage is identical
    assert (dark[..., :3] <= pcf[..., :3]).all() and (pcf[..., :3] <= unshadowed[..., :3]).all()
    assert (dark[..., :3] < unshadowed[..., :3]).any(-1).mean() > 0.0
    differ = (pcf[..., :3] != rays[..., :3]).any(-1) & occ
    frac = differ.sum() / occ.sum()
    assert 0 < frac < 0.02, frac                                                     # measured: 87 of 10,162
    # the voxels where the two modes disagree lie at shadow boundaries, where the filtered lookup blends and the ray does not:
    # some voxel of their 3x3x3 neighbourhood is darker under the shadow rays than unshadowed. The rest (measured: 13 of 87)
    # are surfaces the light grazes, where a texel's depth footprint exceeds the 2 % bias and the lookup self-shadows a little
    # -- as the engine's does.
    shaded = np.pad((rays[..., :3] < unshadowed[..., :3]).any(-1), 1)
    near_shadow = np.zeros_like(occ)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                near_shadow |= shaded[1 + dz:shaded.shape[0] - 1 + dz, 1 + dy:shaded.shape[1] - 1 + dy, 1 + dx:shaded.shape[2] - 1 + dx]
    assert (near_shadow[differ]).mean() > 0.8, near_shadow[differ].mean()
