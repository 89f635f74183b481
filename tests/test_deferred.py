"""SSAO (SSAO/compute.glsl) and deferred lighting (DeferredLighting/fragment.glsl): the oracle against float64 restatements and
exact properties of both passes (no GPU).

1. the GGX terms (GGXBrdf with DistributionGGX, SmithGGXCorrelated, FresnelSchlick) on random inputs, to 1e-3 relative;
2. SSAO: a flat wall facing the camera is exactly 0; the inside of a depth step (a corner) is occluded; a large Strength
   saturates to 255;
3. PCF: all-65535 maps equal ShadowMode None bit for bit for points inside far; all-zero maps make every shadowed light add
   exactly 0;
4. the R8Unorm rule the SSAO store and the ray-traced visibility read use;
5. the whole pass (IsSSAO, IsVXGI, lights with and without shadows, ShadowMode None) against float64, to 2e-3 relative.
"""
import numpy as np

import deferred_oracle as do
import raster_lib as rl
from idkengine_b200 import capi, scenes, vxgi

W, H = 48, 32


def lit_cornell():
    """Three lights; lights 0 and 1 shadowed (crossed indices), light 2 not."""
    scene, cam = rl.lit_cornell(3)
    return scene, cam, rl.crossed_shadows(scene, 0.1, 0.1)


def frame_of(cam):
    f = scenes.camera_frame(cam, W, H)
    return f, (f[0] if f.ndim else f)


def unproject(f, ndc_x, ndc_y, depth):
    M = np.asarray(f["InvProjView"], np.float64).reshape(4, 4)
    wp = np.stack([ndc_x, ndc_y, depth, np.ones_like(depth)], -1) @ M
    return wp[..., :3] / wp[..., 3:]


def camera_basis(f):
    """Camera position and forward direction of the frame."""
    a, b = unproject(f, np.zeros(1), np.zeros(1), np.full(1, 0.5)), unproject(f, np.zeros(1), np.zeros(1), np.full(1, 0.9))
    fwd = (b - a)[0]
    return np.asarray(f["ViewPos"], np.float64).reshape(3), fwd / np.linalg.norm(fwd)


def depth_at(f, p):
    clip = np.append(p, 1.0) @ np.asarray(f["ProjView"], np.float64).reshape(4, 4)
    return np.float32(clip[2] / clip[3])


def decode_unit_vec64(e):
    e = e.astype(np.float64) * 2 - 1
    n = np.stack([e[..., 0], e[..., 1], 1 - np.abs(e[..., 0]) - np.abs(e[..., 1])], -1)
    t = np.maximum(-n[..., 2], 0)
    n[..., 0] += np.where(n[..., 0] >= 0, -t, t)
    n[..., 1] += np.where(n[..., 1] >= 0, -t, t)
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


def walls(f, dist_left, dist_right):
    """G-buffer depth of a wall facing the camera at dist_left (left half of the image) and dist_right (right half), with the
    normal facing the camera."""
    pos, fwd = camera_basis(f)
    depth = np.empty((H, W), np.float32)
    depth[:, : W // 2] = depth_at(f, pos + fwd * dist_left)
    depth[:, W // 2:] = depth_at(f, pos + fwd * dist_right)
    nrg = np.broadcast_to(vxgi.encode_unit_vec(-fwd), (H, W, 2)).copy()
    return depth, nrg


def surfaces(seed=5):
    rng = np.random.default_rng(seed)
    albedo = rng.random((H, W, 3), dtype=np.float32)
    mr = rng.random((H, W, 2), dtype=np.float32)
    mr[..., 1] = 0.2 + 0.8 * mr[..., 1]
    emissive = np.where(rng.random((H, W, 1)) < 0.3, rng.random((H, W, 3)) * 0.5, 0.0).astype(np.float32)
    return albedo, mr, emissive


def ggx64(albedo, metallic, roughness, N, V, L):
    r = roughness ** 2
    f0 = albedo * metallic[:, None]
    Hv = V + L
    Hv /= np.linalg.norm(Hv, axis=1, keepdims=True)
    NoV = np.abs(np.sum(N * V, 1))
    NoL = np.clip(np.sum(N * L, 1), 0, 1)
    NoH = np.clip(np.sum(N * Hv, 1), 0, 1)
    LoH = np.clip(np.sum(L * Hv, 1), 0, 1)
    rD = np.maximum(r, 0.005)
    k = rD / (1 - NoH * NoH + (NoH * rD) ** 2)
    D = k * k / np.pi
    rG = np.maximum(r, 0.0001)
    G = 0.5 / (NoL * np.sqrt((-NoV * rG + NoV) * NoV + rG) + NoV * np.sqrt((-NoL * rG + NoL) * NoL + rG))
    F = f0 + (1 - f0) * ((1 - LoH) ** 5)[:, None]
    return (D * G)[:, None] * F, F


def test_ggx_terms_against_float64():
    rng = np.random.default_rng(11)
    n = 4000

    def unit(k):
        v = rng.normal(size=(k, 3))
        return v / np.linalg.norm(v, axis=1, keepdims=True)
    N, V, L = unit(n), unit(n), unit(n)
    V = np.where((np.sum(N * V, 1) < 0)[:, None], -V, V)
    L = np.where((np.sum(N * L, 1) < 0)[:, None], -L, L)
    albedo, metallic, roughness = rng.random((n, 3)), rng.random(n), 0.3 + 0.7 * rng.random(n)
    keep = (np.sum(N * V, 1) > 0.1) & (np.sum(N * L, 1) > 0.1)
    args = [a[keep].astype(np.float32) for a in (albedo, metallic, roughness, N, V, L)]
    spec, F = do.ggx_brdf(*args)
    spec64, F64 = ggx64(*[a.astype(np.float64) for a in args])
    np.testing.assert_allclose(F, F64, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(spec, spec64, rtol=1e-3)
    assert keep.sum() > 1000


def test_ssao_flat_wall_is_zero_and_corner_is_occluded():
    _, cam, _ = lit_cornell()
    frame, f = frame_of(cam)
    st = capi.IdkPtSsaoSettings(16, 0.5, 1.3, 7)
    depth, nrg = walls(f, 2.0, 2.0)
    assert np.all(do.ssao(frame, st, depth, nrg) == 0)                         # every sample lies in front of the wall
    depth, nrg = walls(f, 2.0, 1.8)                                             # the right half steps 0.2 towards the camera
    ao = do.ssao(frame, st, depth, nrg)
    assert np.all(ao[:, W // 2 + 2:] == 0)                                     # the near wall sees only the far wall behind it
    assert np.all(ao[:, W // 2 - 1] > 0)                                       # the far wall next to the step is occluded
    depth[3, 5] = 1.0
    assert do.ssao(frame, st, depth, nrg)[3, 5] == 0                           # sky stores 0
    sat = do.ssao(frame, capi.IdkPtSsaoSettings(16, 0.5, 1e4, 7), depth, nrg)
    assert np.all((sat == 255) == (ao > 0)) and np.all(sat[ao == 0] == 0)      # Strength saturates to 255


def gbuffer_corner(f):
    depth, nrg = walls(f, 2.0, 1.8)
    rng = np.random.default_rng(3)
    _, fwd = camera_basis(f)
    n = -fwd + rng.normal(scale=0.3, size=(H, W, 3))                           # normals around the camera direction
    nrg = vxgi.encode_unit_vec(n / np.linalg.norm(n, axis=-1, keepdims=True))
    depth[0, 0] = 1.0
    return (depth, nrg) + surfaces()


def test_pcf_all_far_maps_equal_no_shadows_and_all_zero_maps_add_nothing():
    scene, cam, shadows = lit_cornell()
    frame, f = frame_of(cam)
    g = gbuffer_corner(f)
    ao = do.ssao(frame, capi.IdkPtSsaoSettings(10, 0.2, 1.3, 0), g[0], g[1])
    far_maps = [np.full((6, n, n), 65535, np.uint16) for n in (8, 5)]
    none = do.deferred_lighting(scene.lights, frame, 0, shadows, far_maps, g, (0.01, -0.02), ao)
    pcf = do.deferred_lighting(scene.lights, frame, 1, shadows, far_maps, g, (0.01, -0.02), ao)
    assert np.array_equal(none.view(np.uint32), pcf.view(np.uint32))
    rng = np.random.default_rng(2)
    v = rng.normal(size=(500, 3))
    v *= (rng.random((500, 1)) * 50 + 0.2) / np.linalg.norm(v, axis=1, keepdims=True)
    assert np.all(do.visibility(shadows[0], far_maps[0], v) == 1.0)
    assert np.all(do.visibility(shadows[0], np.zeros((6, 8, 8), np.uint16), v) == 0.0)
    lit = scene.lights.copy()
    lit["PointShadowIndex"][:] = [1, 0, 0]                                     # every light shadowed
    zero_maps = [np.zeros((6, n, n), np.uint16) for n in (8, 5)]
    gi = rng.random((H, W, 4)).astype(np.float32)
    dark = do.deferred_lighting(lit, frame, 1, shadows, zero_maps, g, None, ao, gi)
    unlit = do.deferred_lighting(lit[:0], frame, 1, shadows, zero_maps, g, None, ao, gi)
    assert np.array_equal(dark.view(np.uint32), unlit.view(np.uint32))
    assert not np.array_equal(do.deferred_lighting(lit, frame, 0, shadows, zero_maps, g, None, ao, gi), dark)


def test_r8_rule():
    v = np.concatenate([np.linspace(-0.5, 1.5, 2001), (np.arange(256) + 0.5) / 255, [np.nan, np.inf, -np.inf, 0.0, 1.0]]).astype(np.float32)
    want = np.where(np.isnan(v), 0, np.floor(np.clip(v, 0, 1).astype(np.float32) * np.float32(255) + np.float32(0.5))).astype(np.uint8)
    assert np.array_equal(do.store_r8(v), want)
    scene, cam, shadows = lit_cornell()                                         # the RayTraced read goes through the same rule
    frame, f = frame_of(cam)
    g = gbuffer_corner(f)
    maps = [np.full((6, 4, 4), 65535, np.uint16)] * 2
    one_light = scene.lights[:1].copy()                                         # light 0, shadow 1
    vis = np.random.default_rng(4).random((H, W)).astype(np.float32) * 1.2 - 0.1
    rt = do.deferred_lighting(one_light, frame, 2, shadows, maps, g, None, rt=[np.zeros((H, W), np.float32), vis])
    none = do.deferred_lighting(one_light, frame, 0, shadows, maps, g, None)
    amb = do.deferred_lighting(one_light[:0], frame, 0, shadows, maps, g, None)
    scale = (do.store_r8(vis).reshape(H, W) / np.float32(255)).astype(np.float32)
    direct = none[..., :3] - amb[..., :3]
    np.testing.assert_allclose(rt[..., :3] - amb[..., :3], direct * scale[..., None], rtol=1e-4, atol=1e-6)


def deferred64(lights, f, g, ao, gi):
    depth, nrg, albedo, mr, emissive = [a.astype(np.float64) for a in g]
    y, x = np.mgrid[0:H, 0:W]
    frag = unproject(f, (x + 0.5) / W * 2 - 1, (y + 0.5) / H * 2 - 1, depth)
    N = decode_unit_vec64(nrg)
    V = np.asarray(f["ViewPos"], np.float64).reshape(3) - frag
    V /= np.linalg.norm(V, axis=-1, keepdims=True)
    occ = ao.astype(np.float64) / 255
    metallic, r = mr[..., 0], mr[..., 1] ** 2
    f0 = albedo * metallic[..., None]
    direct = np.zeros((H, W, 3))
    for L in lights:
        s2l = np.asarray(L["Position"], np.float64) - frag
        dist2 = np.sum(s2l * s2l, -1)
        Ld = s2l / np.sqrt(dist2)[..., None]
        att = max(float(L["Radius"]), 1e-4) ** 2 / np.maximum(dist2, 1e-4)
        Hv = V + Ld
        Hv /= np.linalg.norm(Hv, axis=-1, keepdims=True)
        NoV = np.abs(np.sum(N * V, -1))
        NoL = np.clip(np.sum(N * Ld, -1), 0, 1)
        NoH = np.clip(np.sum(N * Hv, -1), 0, 1)
        LoH = np.clip(np.sum(Ld * Hv, -1), 0, 1)
        rD, rG = np.maximum(r, 0.005), np.maximum(r, 1e-4)
        k = rD / (1 - NoH ** 2 + (NoH * rD) ** 2)
        G = 0.5 / (NoL * np.sqrt((-NoV * rG + NoV) * NoV + rG) + NoV * np.sqrt((-NoL * rG + NoL) * NoL + rG))
        F = f0 + (1 - f0) * ((1 - LoH) ** 5)[..., None]
        comb = (k * k / np.pi * G)[..., None] * F + albedo * (1 - occ)[..., None] * (1 - F) * (1 - metallic)[..., None]
        direct += comb * (att * NoL)[..., None] * np.asarray(L["Color"], np.float64)
    out = direct + gi[..., :3].astype(np.float64) * albedo + emissive
    return np.where((depth == 1.0)[..., None], 0.0, out)


def test_whole_pass_against_float64():
    scene, cam, shadows = lit_cornell()
    frame, f = frame_of(cam)
    g = gbuffer_corner(f)
    ao = do.ssao(frame, capi.IdkPtSsaoSettings(10, 0.5, 1.3, 0), g[0], g[1])
    assert ao.any()
    gi = np.random.default_rng(9).random((H, W, 4)).astype(np.float32)
    maps = [np.full((6, 4, 4), 65535, np.uint16)] * 2
    got = do.deferred_lighting(scene.lights, frame, 0, shadows, maps, g, (0.01, 0.02), ao, gi)
    want = deferred64(scene.lights, f, g, ao, gi)
    assert np.all(got[..., 3] == 1.0) and np.all(got[0, 0, :3] == 0)
    np.testing.assert_allclose(got[..., :3], want, rtol=2e-3, atol=1e-6 * np.abs(want).max())
    no_vxgi = do.deferred_lighting(scene.lights, frame, 0, shadows, maps, g, None, None, None)   # ambient 0.015 * albedo, no AO
    gi015 = np.full((H, W, 4), 0.015, np.float32)
    np.testing.assert_allclose(no_vxgi[..., :3], deferred64(scene.lights, f, g, np.zeros((H, W), np.uint8), gi015), rtol=2e-3,
                               atol=1e-6 * np.abs(want).max())


def test_wrapper_rejects_mismatched_gbuffer_shapes():
    """PathTracer's G-buffer wrapper raises ValueError (not an assert, which `python -O` drops) before the library could copy
    W * H * c floats out of a smaller array."""
    import pytest
    from idkengine_b200.pathtracer import PathTracer
    d, n = np.zeros((H, W), np.float32), np.zeros((H, W, 2), np.float32)
    g, ptrs, _ = PathTracer._gbuffer([d, n, None], [1, 2, 3])
    assert (g.Width, g.Height, g.OnDevice) == (W, H, 0) and ptrs == [d.ctypes.data, n.ctypes.data, None]
    assert (g.Depth, g.NormalRG, g.AlbedoRGB) == (d.ctypes.data, n.ctypes.data, None)
    for arrays, channels in (([d, n[:-1]], [1, 2]),                      # fewer rows
                             ([d, n[..., :1]], [1, 2]),                   # one channel where two are read
                             ([d[..., None], n], [1, 2]),                 # depth not 2-D
                             ([d.ravel(), n], [1, 2]),
                             ([d, n, np.zeros((H, W // 2, 3), np.float32)], [1, 2, 3]),
                             ([n, np.zeros((H, W - 1, 4), np.float32)], [2, 4]),   # ShadingRate: velocity first
                             ([n[..., 0], np.zeros((H, W, 4), np.float32)], [2, 4])):
        with pytest.raises(ValueError, match="G-buffer array of shape"):
            PathTracer._gbuffer(arrays, channels)
