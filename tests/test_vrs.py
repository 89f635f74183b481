"""Variable-rate deferred lighting (DESIGN 8f.1f): the classifier oracle against a float64 restatement and its pinned order and
conversions, and the coarse deferred oracle against the per-pixel one and the per-sample evaluation (no GPU).

1. the classifier's rates and debug values on seeded images against float64 (the butterfly emulated in numpy);
2. a tile whose sequential float32 sum differs from the butterfly's: the oracle gives the butterfly's;
3. the special tiles: lumMean <= 0.001 (rate 4, cov 0), a flat non-zero tile (cov 0 -> NaN -> rate 0), DeltaRenderTime 0,
   a rounded-negative variance, and zero-padded edge tiles at 17x9;
4. coarse lighting at rate 0 everywhere equals oracle_deferred_lighting bit for bit;
5. every coarse fragment is constant over its in-image pixels and equals the fragment shader at its (imgCoord, uv), at
   odd sizes where imgCoord is clamped.
"""
import numpy as np
import pytest

import deferred_oracle as do
import raster_lib as rl
import vrs_oracle as vo
from idkengine_b200 import capi, scenes

SPEED, LUM, COV = capi.VRS_DEBUG_SPEED, capi.VRS_DEBUG_LUMINANCE, capi.VRS_DEBUG_LUMINANCE_VARIANCE


def frame_with_dt(w, h, dt):
    _, cam = scenes.cornell_1k(threads=1)
    frame = scenes.camera_frame(cam, w, h).copy()
    frame["DeltaRenderTime"] = dt
    return frame


def settings(mode=0, speed_factor=0.2, lum_variance_factor=0.04):
    return capi.IdkPtShadingRateSettings(mode, speed_factor, lum_variance_factor)


def tile_lanes(a, w, h, c):
    """[tilesY, tilesX, 256, c] lanes of each tile (lx + 16 ly), zero outside the image."""
    ty, tx = vo.tiles_of(w, h)
    pad = np.zeros((ty * 16, tx * 16, c), a.dtype)
    pad[:h, :w] = a.reshape(h, w, c)
    return pad.reshape(ty, 16, tx, 16, c).transpose(0, 2, 1, 3, 4).reshape(ty, tx, 256, c)


def butterfly(lanes):
    """Per warp xor butterfly (16, 8, 4, 2, 1) on [..., 256], then the eight warp sums in order -> [...] (dtype kept)."""
    v = lanes.reshape(lanes.shape[:-1] + (8, 32)).copy()
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    s = v[..., 0, 0]
    for i in range(1, 8):
        s = s + v[..., i, 0]
    return s


def classify64(frame, st, color, velocity):
    """compute.glsl in float64: (pre-round rate, rate, meanSpeed, lumMean, cov) per tile."""
    h, w = velocity.shape[:2]
    c = tile_lanes(color[..., :3].astype(np.float64), w, h, 3)
    v = tile_lanes(velocity.astype(np.float64), w, h, 2)
    lum = (c[..., 0] + c[..., 1] + c[..., 2]) / 3.0
    speed = np.sqrt(v[..., 0] ** 2 + v[..., 1] ** 2)
    dt = float(frame["DeltaRenderTime"].reshape(-1)[0])
    mean_speed = butterfly(speed) / 256.0 / dt
    lum_mean = butterfly(lum) / 256.0
    with np.errstate(all="ignore"):
        cov = np.sqrt(butterfly(lum * lum) / 256.0 - lum_mean ** 2) / lum_mean
        pre = 4.0 * mean_speed * st.SpeedFactor + 4.0 * st.LumVarianceFactor / cov
    dark = lum_mean <= 0.001
    rate = np.where(dark, 4, np.clip(np.round(np.nan_to_num(pre, nan=0.0)), 0, 4)).astype(np.uint8)
    return np.where(dark, 4.0, pre), rate, mean_speed, lum_mean, np.where(dark, 0.0, cov)


def seeded_inputs(w, h, seed):
    rng = np.random.default_rng(seed)
    ty, tx = vo.tiles_of(w, h)
    # per-tile brightness and contrast, so tiles spread over every rate: some dark, some flat-ish, some busy
    bright = np.repeat(np.repeat(rng.choice([0.0005, 0.05, 0.5, 2.0], (ty, tx)), 16, 0), 16, 1)[:h, :w]
    contrast = np.repeat(np.repeat(rng.choice([0.01, 0.5, 1.0, 2.0], (ty, tx)), 16, 0), 16, 1)[:h, :w]
    color = np.empty((h, w, 4), np.float32)
    color[..., :3] = bright[..., None] * (1.0 + contrast[..., None] * (rng.random((h, w, 3)) - 0.5))
    color[..., 3] = 1.0
    speed = np.repeat(np.repeat(rng.choice([0.0, 0.02, 0.05, 0.2], (ty, tx)), 16, 0), 16, 1)[:h, :w]
    velocity = (speed[..., None] * (rng.random((h, w, 2)) - 0.5)).astype(np.float32)
    return color, velocity


@pytest.mark.parametrize("w, h, seed", [(64, 48, 1), (37, 23, 2), (200, 120, 3)])
def test_classifier_matches_float64(w, h, seed):
    frame = frame_with_dt(w, h, 1.0 / 60.0)
    color, velocity = seeded_inputs(w, h, seed)
    pre, want, mean_speed, lum_mean, cov = classify64(frame, settings(), color, velocity)
    got = vo.shading_rate(frame, settings(), color, velocity)
    near_half = np.abs(pre - np.floor(pre) - 0.5) < 1e-4
    assert np.array_equal(got[~near_half], want[~near_half])
    assert len(np.unique(got)) >= 3
    # debug values to 1e-5 relative; cov where it is at least 0.05 (below that the float32 one-pass variance cancels: a tile with
    # cov 0.005 keeps about 2 of its variance's significant digits), to 1e-3 relative
    for mode, ref, ok, tol in ((SPEED, mean_speed, np.isfinite(mean_speed), 1e-5), (LUM, lum_mean, np.isfinite(lum_mean), 1e-5),
                               (COV, cov, cov >= 0.05, 1e-3)):
        rates, dbg = vo.shading_rate(frame, settings(mode), color, velocity, debug=True)
        assert np.array_equal(rates, got)
        assert ok.sum() >= ok.size // 4
        np.testing.assert_allclose(dbg[ok], ref[ok], rtol=tol, atol=1e-7)


def test_pinned_butterfly_order_not_sequential():
    """Luminances of widely different magnitudes: the float32 butterfly and the float32 sequential sum differ; the oracle's
    mean luminance is the butterfly's, exactly."""
    rng = np.random.default_rng(5)
    color = np.zeros((16, 16, 4), np.float32)
    color[..., 0] = np.where(rng.random((16, 16)) < 0.1, 3.0e7, 1.0) * (1.0 + rng.random((16, 16))).astype(np.float32)
    velocity = np.zeros((16, 16, 2), np.float32)
    lanes = tile_lanes(color[..., :3], 16, 16, 3)[0, 0]
    lum = ((lanes[:, 0] + lanes[:, 1]) + lanes[:, 2]) * np.float32(1.0 / 3.0)
    bf = butterfly(lum[None])[0]
    seq = np.float32(0.0)
    for x in lum:
        seq = np.float32(seq + x)
    assert bf != seq
    frame = frame_with_dt(16, 16, 1.0)
    _, dbg = vo.shading_rate(frame, settings(LUM), color, velocity, debug=True)
    assert dbg[0, 0] == np.float32(bf / np.float32(256.0))


def special_tiles():
    """A 64x16 image of four tiles: dark (lumMean <= 0.001), flat non-zero, busy and moving, busy and still."""
    rng = np.random.default_rng(3)
    color = np.zeros((16, 64, 4), np.float32)
    color[:, 0:16, :3] = 0.0009
    color[:, 16:32, :3] = 0.5
    color[:, 32:64, :3] = rng.random((16, 32, 3)).astype(np.float32)
    velocity = np.zeros((16, 64, 2), np.float32)
    velocity[:, 32:48] = 0.01
    return color, velocity


def test_special_tiles():
    color, velocity = special_tiles()
    frame = frame_with_dt(64, 16, 1.0 / 60.0)
    rates, cov = vo.shading_rate(frame, settings(COV), color, velocity, debug=True)
    assert rates[0, 0] == 4 and cov[0, 0] == 0.0                    # dark: 4x4, cov 0 as written
    assert cov[0, 1] == 0.0 and rates[0, 1] == 0                    # flat: cov 0 -> LumVarianceFactor / 0 = inf -> mix NaN -> 0
    assert 0 < cov[0, 2] < 1 and 0 < cov[0, 3] < 1
    _, lum = vo.shading_rate(frame, settings(LUM), color, velocity, debug=True)
    assert 0.0008 < lum[0, 0] <= 0.001                               # the dark branch still stores lumMean
    # DeltaRenderTime 0: a moving tile's mean speed is inf, a still one's 0 / 0 = NaN; both mix to NaN -> rate 0
    frame0 = frame_with_dt(64, 16, 0.0)
    rates0, speed0 = vo.shading_rate(frame0, settings(SPEED), color, velocity, debug=True)
    assert np.isinf(speed0[0, 2]) and np.isnan(speed0[0, 3])
    assert rates0[0, 2] == 0 and rates0[0, 3] == 0 and rates0[0, 0] == 4


def test_negative_rounded_variance_gives_full_rate():
    """A tile of one luminance whose squared mean rounds below the square of its mean: sqrt(negative) = NaN -> cov NaN -> 0."""
    frame = frame_with_dt(16, 16, 1.0)
    for v in np.linspace(0.1, 3.0, 400, dtype=np.float32):
        color = np.zeros((16, 16, 4), np.float32)
        color[..., 0] = v * 3
        lanes = tile_lanes(color[..., :3], 16, 16, 3)[0, 0]
        lum = ((lanes[:, 0] + lanes[:, 1]) + lanes[:, 2]) * np.float32(1.0 / 3.0)
        m = butterfly(lum[None])[0] / np.float32(256)
        q = butterfly((lum * lum)[None])[0] / np.float32(256)
        if np.float32(q - m * m) < 0:
            rates, cov = vo.shading_rate(frame, settings(COV), color, np.zeros((16, 16, 2), np.float32), debug=True)
            assert np.isnan(cov[0, 0]) and rates[0, 0] == 0
            return
    pytest.fail("no luminance with a negative rounded variance found")


def test_edge_tiles_are_zero_padded_17x9():
    """At 17x9 the tiles hold 144, 9 in-image lanes; the rest read 0 and still count in the 256."""
    w, h = 17, 9
    color = np.zeros((h, w, 4), np.float32)
    color[..., :3] = 0.8
    velocity = np.full((h, w, 2), 0.3, np.float32)
    frame = frame_with_dt(w, h, 1.0)
    _, lum = vo.shading_rate(frame, settings(LUM), color, velocity, debug=True)
    _, speed = vo.shading_rate(frame, settings(SPEED), color, velocity, debug=True)
    l1 = np.float32((np.float32(0.8 + np.float32(0.8)) + np.float32(0.8)) * np.float32(1 / 3))
    assert lum.shape == (1, 2)
    np.testing.assert_allclose(lum[0], [l1 * 144 / 256, l1 * 9 / 256], rtol=1e-6)
    np.testing.assert_allclose(speed[0], [np.hypot(0.3, 0.3) * 144 / 256, np.hypot(0.3, 0.3) * 9 / 256], rtol=1e-6)
    pre, want, *_ = classify64(frame, settings(), color, velocity)
    assert np.array_equal(vo.shading_rate(frame, settings(), color, velocity), want)


def test_rejected_settings():
    frame = frame_with_dt(16, 16, 1.0)
    z4, z2 = np.zeros((16, 16, 4), np.float32), np.zeros((16, 16, 2), np.float32)
    import ctypes
    r, d = np.zeros((1, 1), np.uint8), np.zeros((1, 1), np.float32)
    fr = np.ascontiguousarray(frame)
    for st, dbg in ((settings(5), None), (settings(-1), None), (settings(0), d), (settings(1), d), (settings(0, np.inf), None),
                    (settings(0, 0.2, np.nan), None)):
        assert vo.lib().oracle_shading_rate(fr.ctypes.data, ctypes.byref(st), z4.ctypes.data, z2.ctypes.data, 16, 16, r.ctypes.data,
                                            dbg.ctypes.data if dbg is not None else None) == -1


# ---- coarse deferred lighting
def lit_cornell():
    scene, cam = rl.lit_cornell(3)
    return scene, cam, rl.crossed_shadows(scene, 0.1, 0.1)


def synthetic_inputs(w, h, seed):
    """A seeded G-buffer (sky pixels included), SSAO, indirect light, RT visibility and two seeded 8^2 cube maps."""
    rng = np.random.default_rng(seed)
    depth = (0.97 + 0.029 * rng.random((h, w))).astype(np.float32)
    depth[rng.random((h, w)) < 0.08] = 1.0
    n = rng.normal(size=(h, w, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    m = n / np.sum(np.abs(n), -1, keepdims=True)
    wrap = (1.0 - np.abs(m[..., [1, 0]])) * np.where(m[..., :2] < 0, -1.0, 1.0)
    nrg = (np.where((m[..., 2] > 0)[..., None], m[..., :2], wrap) * 0.5 + 0.5).astype(np.float32)
    albedo = rng.random((h, w, 3), dtype=np.float32)
    mr = rng.random((h, w, 2), dtype=np.float32)
    emissive = np.where(rng.random((h, w, 1)) < 0.2, rng.random((h, w, 3)) * 0.5, 0.0).astype(np.float32)
    ao = rng.integers(0, 256, (h, w), dtype=np.uint8)
    gi = rng.random((h, w, 4), dtype=np.float32)
    rt = [rng.random((h, w), dtype=np.float32) for _ in range(2)]
    maps = [rng.integers(50000, 65536, (6, 8, 8)).astype(np.uint16) for _ in range(2)]
    return (depth, nrg, albedo, mr, emissive), ao, gi, rt, maps


MODES = [(0, False, False), (1, True, True), (2, True, False)]


@pytest.mark.parametrize("w, h", [(37, 23), (1, 1), (5, 3), (48, 32)])
def test_rate_zero_equals_per_pixel_oracle(w, h):
    scene, cam, shadows = lit_cornell()
    frame = scenes.camera_frame(cam, w, h)
    g, ao, gi, rt, maps = synthetic_inputs(w, h, 11)
    zero = np.zeros(vo.tiles_of(w, h), np.uint8)
    for mode, is_ssao, is_vxgi in MODES:
        kw = dict(jitter=(0.01, -0.02), ssao=ao if is_ssao else None, indirect=gi if is_vxgi else None, rt=rt if mode == 2 else None)
        want = do.deferred_lighting(scene.lights, frame, mode, shadows, maps, g, **kw)
        got = vo.deferred_lighting_vrs(scene.lights, frame, mode, shadows, maps, g, zero, **kw)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def fragments(w, h, rates):
    """The coarse fragments NV_shading_rate_image makes: [(x0, y0, cw, ch, imgCoord, uv)] restated in numpy."""
    out = []
    for ty in range(rates.shape[0]):
        for tx in range(rates.shape[1]):
            cw, ch = capi.VRS_PALETTE[rates[ty, tx]]
            for y0 in range(ty * 16, min(ty * 16 + 16, h), ch):
                for x0 in range(tx * 16, min(tx * 16 + 16, w), cw):
                    img = (min(x0 + cw // 2, w - 1), min(y0 + ch // 2, h - 1))
                    uv = (np.float32(x0 + 0.5 * cw) / np.float32(w), np.float32(y0 + 0.5 * ch) / np.float32(h))
                    out.append((x0, y0, cw, ch, img, uv))
    return out


@pytest.mark.parametrize("w, h, seed", [(37, 23, 1), (1, 1, 2), (5, 3, 3), (50, 34, 4)])
def test_fragments_are_constant_and_equal_the_sample_at_their_centre(w, h, seed):
    scene, cam, shadows = lit_cornell()
    frame = scenes.camera_frame(cam, w, h)
    g, ao, gi, rt, maps = synthetic_inputs(w, h, seed)
    rng = np.random.default_rng(seed)
    tiles = vo.tiles_of(w, h)
    for rates in (rng.integers(0, 5, tiles).astype(np.uint8), np.full(tiles, 4, np.uint8), np.full(tiles, 3, np.uint8)):
        frags = fragments(w, h, rates)
        for mode, is_ssao, is_vxgi in MODES:
            kw = dict(jitter=(0.01, -0.02), ssao=ao if is_ssao else None, indirect=gi if is_vxgi else None, rt=rt if mode == 2 else None)
            got = vo.deferred_lighting_vrs(scene.lights, frame, mode, shadows, maps, g, rates, **kw)
            samples = vo.deferred_samples(scene.lights, frame, mode, shadows, maps, g, [f[4] for f in frags], [f[5] for f in frags], **kw)
            covered = np.zeros((h, w), int)
            for (x0, y0, cw, ch, _, _), s in zip(frags, samples):
                block = got[y0:y0 + ch, x0:x0 + cw]
                assert np.array_equal(block.reshape(-1, 4).view(np.uint32), np.broadcast_to(s, block.shape).reshape(-1, 4).view(np.uint32))
                covered[y0:y0 + ch, x0:x0 + cw] += 1
            assert np.all(covered == 1)
    # the clamp: at odd sizes some 2- or 4-wide fragment's centre lies past the last column / row
    if w % 2 or h % 2:
        assert any(x0 + cw // 2 >= w or y0 + ch // 2 >= h for x0, y0, cw, ch, _, _ in fragments(w, h, np.full(tiles, 4, np.uint8)))
