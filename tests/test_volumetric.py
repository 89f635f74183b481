"""Volumetric lighting (VolumetricLight/compute.glsl + Upscale/compute.glsl): the oracle against an independent float64
restatement of both dispatches (no GPU).

1. march + upscale with every map at 65535 (nothing occludes) on the lit Cornell box, to half precision;
2. every map at 0: each sample beyond a light's near plane is shadowed, so a camera whose samples all stay beyond it sees 0;
3. the NEAREST cube lookup: the direction through each texel centre selects that texel;
4. the upscale: a constant image stays constant, and the depth weights follow the float64 restatement across a depth step.
"""
import numpy as np

import oracle_lib as ol
import raster_lib as rl
import volumetric_oracle as vo
from idkengine_b200 import capi, scenes

DITHER = np.array([[0.0, 0.5, 0.125, 0.625], [0.75, 0.22, 0.875, 0.375], [0.1875, 0.6875, 0.0625, 0.5625], [0.9375, 0.4375, 0.8125, 0.3125]])


def lit_cornell():
    """Two lights, each with a point shadow; shadow 0 belongs to light 1 and shadow 1 to light 0."""
    scene, cam = rl.lit_cornell(2)
    return scene, cam, rl.crossed_shadows(scene, 0.1, 0.1)


def nearest64(u, n):
    return np.clip(np.floor(u * n), 0, n - 1).astype(np.int64)


def cube_nearest64(m, d):
    """texture(samplerCube, d).r, NEAREST: table 8.19 face selection (ties x >= y >= z), texel clamp(floor(s N), 0, N - 1)."""
    n = m.shape[1]
    a = np.abs(d)
    fx = (a[:, 0] >= a[:, 1]) & (a[:, 0] >= a[:, 2])
    fy = ~fx & (a[:, 1] >= a[:, 2])
    px, py, pz = d[:, 0] >= 0, d[:, 1] >= 0, d[:, 2] >= 0
    face = np.where(fx, np.where(px, 0, 1), np.where(fy, np.where(py, 2, 3), np.where(pz, 4, 5)))
    sc = np.where(fx, np.where(px, -d[:, 2], d[:, 2]), np.where(fy, d[:, 0], np.where(pz, d[:, 0], -d[:, 0])))
    tc = np.where(fx, -d[:, 1], np.where(fy, np.where(py, d[:, 2], -d[:, 2]), -d[:, 1]))
    ma = np.where(fx, a[:, 0], np.where(fy, a[:, 1], a[:, 2]))
    s, t = 0.5 * (sc / ma + 1.0), 0.5 * (tc / ma + 1.0)
    return m[face, nearest64(t, n), nearest64(s, n)] / 65535.0


def march64(lights, frame, st, shadows, maps, depth, w, h, jitter):
    """VolumetricLight/compute.glsl in float64 over the render size: (rgb [h, w, 3], depth [h, w], min over samples and shadows
    of max|lightToSample| / NearPlane)."""
    f = frame[0] if frame.ndim else frame
    hg, wg = depth.shape
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    u, v = (x + 0.5) / w, (y + 0.5) / h
    d = depth[nearest64(v, hg), nearest64(u, wg)].astype(np.float64)
    M = np.asarray(f["InvProjView"], np.float64).reshape(4, 4)          # column c = M[c]
    ndc = np.stack([u * 2 - 1 - jitter[0], v * 2 - 1 - jitter[1], d, np.ones_like(d)], -1)
    wp = ndc @ M
    frag = wp[..., :3] / wp[..., 3:]
    vp = np.asarray(f["ViewPos"], np.float64).reshape(3)
    vtf = frag - vp
    ln = np.linalg.norm(vtf, axis=-1, keepdims=True)
    vdir = vtf / ln
    vtf = np.where(ln > st.MaxDist, vdir * st.MaxDist, vtf)
    n = st.SampleCount
    step = vtf / n
    origin = vp + step * DITHER[x % 4, y % 4][..., None]
    A = np.array(st.Absorbance[:], np.float64)
    g = np.float64(st.Scattering)
    out = np.zeros((h, w, 3))
    closest = np.inf
    for i, sh in enumerate(shadows):
        L = lights[sh["LightIndex"]]
        lp = np.asarray(L["Position"], np.float64)
        acc = np.zeros((h, w, 3))
        for k in range(n):
            p = origin + step * k
            l = (p - lp).reshape(-1, 3)
            dist = np.abs(l).max(1)
            closest = min(closest, (dist / sh["NearPlane"]).min())
            ld = (1 / dist - 1 / sh["NearPlane"]) / (1 / sh["FarPlane"] - 1 / sh["NearPlane"])
            lit = ~(ld > cube_nearest64(maps[i], l))
            length = np.linalg.norm(l, axis=1)
            att = max(L["Radius"], 1e-4) ** 2 / np.maximum(length ** 2, 1e-4)
            cos = np.sum(l / length[:, None] * -vdir.reshape(-1, 3), 1)
            phase = (1 - g * g) / (4 * np.pi * (1 + g * g - 2 * g * cos) ** 1.5)
            c = np.asarray(L["Color"], np.float64) * (phase * att)[:, None] * np.exp(-A * length[:, None])
            acc += np.where(lit[:, None], c, 0.0).reshape(h, w, 3)
        end = origin + step * n
        acc = acc / n * np.exp(-A * np.linalg.norm(origin - end, axis=-1, keepdims=True))
        out += acc
    return out * st.Strength, d, closest


def upscale64(frame, depth, col, low_depth, W, H):
    """VolumetricLight/Upscale/compute.glsl in float64: (rgb [H, W, 3], weights [H, W, 4])."""
    f = frame[0] if frame.ndim else frame
    near, far = np.float64(f["NearPlane"]), np.float64(f["FarPlane"])
    lin = lambda z: (2 * near * far) / (far + near - z * (far - near)) / far  # noqa: E731
    hg, wg = depth.shape
    h, w = low_depth.shape
    x, y = np.meshgrid(np.arange(W), np.arange(H))
    high = lin(depth[nearest64((y + 0.5) / H, hg), nearest64((x + 0.5) / W, wg)].astype(np.float64))
    ox, oy = np.where(x % 2 == 0, -1, 1), np.where(y % 2 == 0, -1, 1)
    color, weights = np.zeros((H, W, 3)), []
    for dx, dy in ((0, 0), (0, 1), (1, 0), (1, 1)):
        su, sv = (x + dx * ox + 0.5) / W, (y + dy * oy + 0.5) / H
        px, py = su * w - 0.5, sv * h - 0.5
        x0, y0 = np.floor(px), np.floor(py)
        fx, fy = (px - x0)[..., None], (py - y0)[..., None]
        xi0, xi1 = np.clip(x0, 0, w - 1).astype(int), np.clip(x0 + 1, 0, w - 1).astype(int)
        yi0, yi1 = np.clip(y0, 0, h - 1).astype(int), np.clip(y0 + 1, 0, h - 1).astype(int)
        c = (col[yi0, xi0] * (1 - fx) + col[yi0, xi1] * fx) * (1 - fy) + (col[yi1, xi0] * (1 - fx) + col[yi1, xi1] * fx) * fy
        wt = np.maximum(1 - 0.05 * np.abs(lin(low_depth[nearest64(sv, h), nearest64(su, w)].astype(np.float64)) - high), 0)
        color += c * wt[..., None]
        weights.append(wt)
    weights = np.stack(weights, -1)
    return color / (weights.sum(-1, keepdims=True) + 1e-4), weights


def halves(a):
    return a.view(np.float16).astype(np.float64)


def test_unoccluded_march_and_upscale_match_float64():
    scene, cam, shadows = lit_cornell()
    W, H = 45, 31
    frame = scenes.camera_frame(cam, W, H)
    depth = ol.synth_gbuffer(scene, frame, 40, 28)[0]
    assert (depth == 1.0).any() and (depth < 1.0).mean() > 0.5
    st = capi.default_volumetric_settings()
    st.Absorbance[:] = [0.025, 0.05, 0.1]
    jitter = (0.013, -0.021)
    maps = [np.full((6, 8, 8), 65535, np.uint16), np.full((6, 16, 16), 65535, np.uint16)]
    out, march, low = vo.volumetric_lighting(scene.lights, frame, st, shadows, maps, depth, W, H, jitter)
    w, h = vo.render_size(W, H, st.ResolutionScale)
    assert (w, h) == (27, 18) and march.shape == (h, w, 4)
    col64, d64, _ = march64(scene.lights, frame, st, shadows, maps, depth, w, h, jitter)
    assert np.array_equal(low, d64.astype(np.float32))
    got = halves(march)
    assert np.all(got[..., 3] == 1.0) and np.all(halves(out)[..., 3] == 1.0)
    assert np.all(np.abs(got[..., :3] - col64) <= 2e-3 * np.abs(col64) + 1e-7)
    up64, _ = upscale64(frame, depth, col64, d64, W, H)
    assert np.all(np.abs(halves(out)[..., :3] - up64) <= 2e-3 * np.abs(up64) + 1e-7)
    assert col64.min() > 0 and col64.max() / col64.min() > 3                        # every sample lit, and a real gradient


def test_all_zero_maps_shadow_every_sample_beyond_the_near_plane():
    scene, cam, shadows = lit_cornell()
    shadows["NearPlane"] = 0.01
    W, H = 37, 23
    frame = scenes.camera_frame(cam, W, H)
    depth = ol.synth_gbuffer(scene, frame, W, H)[0]
    st = capi.default_volumetric_settings()
    st.ResolutionScale = 1.0
    maps = [np.zeros((6, 4, 4), np.uint16), np.zeros((6, 5, 5), np.uint16)]
    w, h = vo.render_size(W, H, 1.0)
    _, _, closest = march64(scene.lights, frame, st, shadows, maps, depth, w, h, (0.0, 0.0))
    assert closest > 1.5                                    # no sample comes near the near plane, so none is in front of it
    out, march, _ = vo.volumetric_lighting(scene.lights, frame, st, shadows, maps, depth, W, H)
    assert np.all(halves(out)[..., :3] == 0.0) and np.all(halves(march)[..., :3] == 0.0)
    # the same with 65535 maps is lit: the zeros come from the shadow test
    lit = vo.volumetric_lighting(scene.lights, frame, st, shadows, [np.full_like(m, 65535) for m in maps], depth, W, H)[0]
    assert (halves(lit)[..., :3] > 0).all()


def test_nearest_lookup_selects_the_texel_through_its_centre():
    for n in (1, 2, 7, 16):
        m = np.arange(6 * n * n, dtype=np.uint16).reshape(6, n, n) * 7 + 3
        c = (2.0 * np.arange(n) + 1.0) / n - 1.0
        tc, sc = np.meshgrid(c, c, indexing="ij")
        one = np.ones_like(sc)
        dirs = np.stack([np.stack([one, -tc, -sc], -1), np.stack([-one, -tc, sc], -1), np.stack([sc, one, tc], -1),
                         np.stack([sc, -one, -tc], -1), np.stack([sc, -tc, one], -1), np.stack([-sc, -tc, -one], -1)])
        for scale in (1.0, 0.37, 25.0):
            got = vo.cube_nearest(m, dirs.reshape(-1, 3) * scale)
            assert np.array_equal(got, (m.ravel() / np.float32(65535.0)).astype(np.float32)), (n, scale)
            assert np.array_equal(got, cube_nearest64(m, dirs.reshape(-1, 3) * scale).astype(np.float32))


def test_upscale_constant_and_depth_step_weights():
    scene, cam, _ = lit_cornell()
    W, H = 50, 34
    frame = scenes.camera_frame(cam, W, H)
    w, h = vo.render_size(W, H, 0.6)
    rng = np.random.default_rng(3)
    depth = np.where(np.arange(40)[None, :] < 17, np.float32(0.2), np.float32(0.9999)).repeat(25, 0).astype(np.float32)
    depth[:, 30:] = 1.0                                                                   # sky
    low = np.where(np.arange(w)[None, :] < w // 2, np.float32(0.97), np.float32(0.0)).repeat(h, 0).astype(np.float32)
    const = np.zeros((h, w, 4), np.float16)
    const[..., :3] = (0.3, 1.5, 0.0625)
    const[..., 3] = 1.0
    out = halves(vo.volumetric_upscale(frame, depth, const.view(np.uint16), low, W, H))
    assert np.all(np.abs(out[..., :3] - np.array([0.3, 1.5, 0.0625], np.float16)) <= np.array([0.3, 1.5, 0.0625]) * 1e-3)
    col = np.zeros((h, w, 4), np.float16)
    col[..., :3] = rng.uniform(0.0, 4.0, (h, w, 3))
    col[..., 3] = 1.0
    out = halves(vo.volumetric_upscale(frame, depth, col.view(np.uint16), low, W, H))
    up64, weights = upscale64(frame, depth, col[..., :3].astype(np.float64), low, W, H)
    assert np.all(np.abs(out[..., :3] - up64) <= 2e-3 * np.abs(up64) + 1e-6)
    # for depths in [0, 1] the linear depth / far stays in [0, 1]: the weights stay >= 0.95, a near-plain 4-tap blend
    assert weights.min() >= 0.95 and weights.max() <= 1.0 and weights.min() < 0.999
