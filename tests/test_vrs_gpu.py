"""The shading-rate classifier (k_shading_rate) and coarse-shaded deferred lighting (k_vrs_scan + k_deferred_lighting_vrs) on the
GPU, bit for bit against the oracle.

float32 images are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import numpy as np
import pytest

import vrs_oracle as vo
from idkengine_b200 import capi, multigpu, scenes
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon, cone_trace_gi, deferred_settings, deferred_setup, gbuffer, rt_images


def frame_dt(cam, w, h, dt=1.0 / 60.0):
    f = scenes.camera_frame(cam, w, h).copy()
    f["DeltaRenderTime"] = dt
    return f


def classifier_inputs(w, h, seed):
    """Seeded lit image and velocity whose tiles spread over the rates: per-tile brightness (some dark), contrast and speed."""
    rng = np.random.default_rng(seed)
    ty, tx = vo.tiles_of(w, h)

    def per_tile(choices):
        return np.repeat(np.repeat(rng.choice(choices, (ty, tx)), 16, 0), 16, 1)[:h, :w]
    color = np.empty((h, w, 4), np.float32)
    color[..., :3] = per_tile([0.0005, 0.05, 0.5, 2.0])[..., None] * (1.0 + per_tile([0.0, 0.5, 1.0, 2.0])[..., None] * (rng.random((h, w, 3)) - 0.5))
    color[..., 3] = 1.0
    velocity = (per_tile([0.0, 0.02, 0.05, 0.2])[..., None] * (rng.random((h, w, 2)) - 0.5)).astype(np.float32)
    return color, velocity


def five_rate_inputs(w, h, seed):
    """Inputs that give every palette index with LumVarianceFactor 0, SpeedFactor 1 and DeltaRenderTime 1: busy bright tiles
    whose mean speed is about k / 4 (rate k), and dark tiles (rate 4)."""
    rng = np.random.default_rng(seed)
    ty, tx = vo.tiles_of(w, h)
    k = (np.arange(tx)[None, :] + 2 * np.arange(ty)[:, None]) % 6
    # the mean runs over all 256 lanes: an edge tile's in-image pixels move faster by 256 / their count
    lanes = np.minimum(16, w - 16 * np.arange(tx))[None, :] * np.minimum(16, h - 16 * np.arange(ty))[:, None]
    speed = np.repeat(np.repeat((np.minimum(k, 4) / 4.0 + 0.01) * 256.0 / lanes, 16, 0), 16, 1)[:h, :w]
    ang = rng.random((h, w)) * 2 * np.pi
    velocity = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32) * speed[..., None].astype(np.float32)
    color = np.empty((h, w, 4), np.float32)
    color[..., :3] = (0.2 + rng.random((h, w, 3))).astype(np.float32)
    dark = np.repeat(np.repeat(k == 5, 16, 0), 16, 1)[:h, :w]
    color[dark, :3] = 0.0002
    color[..., 3] = 1.0
    return color, velocity


FIVE = capi.IdkPtShadingRateSettings(0, 1.0, 0.0)
SIZES = [(1, 1), (16, 16), (17, 9), (37, 23), (1920, 1080)]


@pytest.mark.gpu
@pytest.mark.parametrize("w, h", SIZES)
def test_gpu_shading_rate_matches_oracle(w, h):
    import torch
    scene, cam, _ = deferred_setup("cornell")
    frame = frame_dt(cam, w, h)
    color, velocity = classifier_inputs(w, h, w + h)
    dcolor, dvel = torch.from_numpy(color).cuda(), torch.from_numpy(velocity).cuda()
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        for mode in range(5):
            st = capi.IdkPtShadingRateSettings(mode, 0.2, 0.04)
            debug = mode >= 2
            want = vo.shading_rate(frame, st, color, velocity, debug=debug)
            for got in (pt.ShadingRate(frame, velocity, st, color=color, debug=debug),
                        pt.ShadingRate(frame, dvel, st, color=dcolor, debug=debug)):
                if debug:
                    assert np.array_equal(got[0], want[0]) and np.array_equal(canon(got[1]), canon(want[1]))
                else:
                    assert got.shape == vo.tiles_of(w, h) and np.array_equal(got, want)
        if w * h > 256:
            assert len(np.unique(want[0] if isinstance(want, tuple) else want)) >= 2
        # DEFERRED source: the lit image of the last idkpt_deferred_lighting call
        g = gbuffer(pt, scene, frame, w, h)
        lit = pt.DeferredLighting(frame, *g, settings=deferred_settings(0, 0, 0), jitter=JITTER)
        for mode in (0, 4):
            st = capi.IdkPtShadingRateSettings(mode, 0.2, 0.04)
            want = vo.shading_rate(frame, st, lit, velocity, debug=mode >= 2)
            got_host = pt.ShadingRate(frame, velocity, st, source=capi.LIT_SOURCE_DEFERRED, debug=mode >= 2)
            got_dev = pt.ShadingRate(frame, dvel, st, source=capi.LIT_SOURCE_DEFERRED, debug=mode >= 2)
            for got in (got_host, got_dev):
                if mode >= 2:
                    assert np.array_equal(got[0], want[0]) and np.array_equal(canon(got[1]), canon(want[1]))
                else:
                    assert np.array_equal(got, want)


def run_vrs(pt, scene, frame, shadows, maps, g, st, rates, ssao=None, indirect=None, rt=None):
    got = pt.DeferredLighting(frame, *g, settings=st, jitter=JITTER, indirect=indirect if st.IsVXGI else None,
                              rt_visibility=rt if st.ShadowMode == 2 else None, vrs=True)
    want = vo.deferred_lighting_vrs(scene.lights, frame, st.ShadowMode, shadows, maps, g, rates, JITTER, ssao if st.IsSSAO else None,
                                    indirect if st.IsVXGI else None, rt if st.ShadowMode == 2 else None)
    assert got.shape == want.shape
    assert np.array_equal(canon(got), canon(want))
    return got


@pytest.mark.gpu
def test_gpu_coarse_deferred_every_mode_matches_oracle():
    """Every ShadowMode x IsSSAO x IsVXGI on the Cornell box under a rate image with all five rates and partial edge tiles."""
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 37, 23
    frame = frame_dt(cam, W, H, 1.0)
    gi = cone_trace_gi(W, H)
    color, velocity = five_rate_inputs(W, H, 1)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [64, 33])
        pt.RenderPointShadows()
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        g = gbuffer(pt, scene, frame, W, H)
        ao = pt.Ssao(frame, g[0], g[1])
        rt = rt_images(pt, scene, frame, g, shadows)
        rates = pt.ShadingRate(frame, velocity, FIVE, color=color)
        assert set(np.unique(rates)) >= {1, 2, 3, 4}
        for mode in (0, 1, 2):
            for is_ssao in (0, 1):
                for is_vxgi in (0, 1):
                    run_vrs(pt, scene, frame, shadows, maps, g, deferred_settings(mode, is_ssao, is_vxgi), rates, ssao=ao, indirect=gi, rt=rt)


@pytest.mark.gpu
@pytest.mark.parametrize("W, H", [(53, 37), (96, 64), (1, 1), (5, 3)])
def test_gpu_coarse_deferred_atrium_all_rates(W, H):
    scene, cam, shadows = deferred_setup("atrium")
    frame = frame_dt(cam, W, H, 1.0)
    color, velocity = five_rate_inputs(W, H, W)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [48, 32])
        pt.RenderPointShadows()
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        g = gbuffer(pt, scene, frame, W, H)
        ao = pt.Ssao(frame, g[0], g[1])
        rates = pt.ShadingRate(frame, velocity, FIVE, color=color)
        if W * H > 2000:
            assert set(np.unique(rates)) == {0, 1, 2, 3, 4}
        run_vrs(pt, scene, frame, shadows, maps, g, deferred_settings(1, 1, 0), rates, ssao=ao)
        for r in range(5):   # every rate over the whole image, from uniform inputs
            c = np.full((H, W, 4), 0.5, np.float32)
            c[..., :3] += np.random.default_rng(r).random((H, W, 3)).astype(np.float32) * 0.1
            v = np.full((H, W, 2), 0.0, np.float32)
            v[..., 0] = r / 4.0 + 0.01
            only = pt.ShadingRate(frame, v, FIVE, color=c)
            if W >= 16 and H >= 16:
                assert only[0, 0] == r
            run_vrs(pt, scene, frame, shadows, maps, g, deferred_settings(1, 1, 0), only, ssao=ao)


@pytest.mark.gpu
def test_gpu_vrs_at_full_rate_equals_the_per_pixel_pass():
    """A flat lit image gives cov 0 -> NaN -> rate 0 in every tile; IsVariableRateShading then returns exactly the bytes of 0."""
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 61, 35
    frame = frame_dt(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        pt.Ssao(frame, g[0], g[1])
        rates = pt.ShadingRate(frame, np.zeros((H, W, 2), np.float32), color=np.full((H, W, 4), 0.5, np.float32))
        assert not rates.any()
        for mode in (0, 1):
            st = deferred_settings(mode, 1, 0)
            full = pt.DeferredLighting(frame, *g, settings=st, jitter=JITTER)
            coarse = pt.DeferredLighting(frame, *g, settings=st, jitter=JITTER, vrs=True)
            assert np.array_equal(full.view(np.uint32), coarse.view(np.uint32))


def device_u8(p, n):
    import torch
    return torch.as_tensor(multigpu.DeviceArray(p, (n,), "|u1"), device="cuda").cpu().numpy()


@pytest.mark.gpu
def test_gpu_device_only_chain():
    """Frame N: deferred; classify its image (DEFERRED); frame N+1: deferred under the rates. CUDA tensors in, nothing
    downloaded; the device pointers equal the downloads of the same calls and the host-array chain."""
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 83, 45
    frame = frame_dt(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        vel = np.random.default_rng(4).normal(0.0, 0.004, (H, W, 2)).astype(np.float32)
        dg = [torch.from_numpy(a).cuda() for a in g]
        dvel = torch.from_numpy(vel).cuda()
        with pytest.raises(IdkPtError, match="call idkpt_shading_rate first"):
            pt.ShadingRateDevicePtr()
        # host chain
        pt.Ssao(frame, g[0], g[1])
        lit_n = pt.DeferredLighting(frame, *g, jitter=JITTER)
        rates = pt.ShadingRate(frame, vel, source=capi.LIT_SOURCE_DEFERRED)
        lit_n1 = pt.DeferredLighting(frame, *g, jitter=JITTER, vrs=True)
        assert np.array_equal(rates, vo.shading_rate(frame, capi.default_shading_rate_settings(), lit_n, vel))
        # device chain
        assert pt.Ssao(frame, dg[0], dg[1], download=False) is None
        assert pt.DeferredLighting(frame, *dg, jitter=JITTER, download=False) is None
        assert pt.ShadingRate(frame, dvel, source=capi.LIT_SOURCE_DEFERRED, download=False) is None
        p, n = pt.ShadingRateDevicePtr()
        assert n == rates.size and np.array_equal(device_u8(p, n).reshape(rates.shape), rates)
        assert pt.DeferredLighting(frame, *dg, jitter=JITTER, download=False, vrs=True) is None
        p, nbytes = pt.DeferredDevicePtr()
        dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 4,), "<f4"), device="cuda").cpu().numpy()
        assert np.array_equal(canon(dev.reshape(H, W, 4)), canon(lit_n1))
        assert pt.last_shading_rate_ms > 0 and pt.last_deferred_ms > 0


@pytest.mark.gpu
def test_gpu_shading_rate_errors_leave_the_context_working():
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 40, 24
    frame = frame_dt(cam, W, H)
    fr = np.ascontiguousarray(frame)
    lib = capi.load()
    color, velocity = classifier_inputs(W, H, 9)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [16, 16])
        pt.RenderPointShadows()
        g = gbuffer(pt, scene, frame, W, H)
        pt.Ssao(frame, g[0], g[1])
        with pytest.raises(IdkPtError, match="IsVariableRateShading needs an idkpt_shading_rate image"):
            pt.DeferredLighting(frame, *g, vrs=True)
        good = pt.ShadingRate(frame, velocity, color=color)
        good_lit = pt.DeferredLighting(frame, *g, jitter=JITTER, vrs=True)
        st0 = capi.default_shading_rate_settings()
        inputs = capi.IdkPtShadingRateInputs(W, H, 0, capi.LIT_SOURCE_ARRAY, velocity.ctypes.data, color.ctypes.data)
        out = np.zeros(vo.tiles_of(W, H), np.uint8)
        dbg = np.zeros(vo.tiles_of(W, H), np.float32)

        def rc(f=fr, s=st0, i=inputs, o=out.ctypes.data, d=None):
            return lib.idkpt_shading_rate(pt._ctx, f.ctypes.data if f is not None else None, s, i, o, d, None)

        def expect(code, msg):
            with pytest.raises(IdkPtError, match=msg):
                pt._check(code, "call")
        assert rc(f=None) == -1 and lib.idkpt_shading_rate(pt._ctx, fr.ctypes.data, None, inputs, None, None, None) == -1
        assert lib.idkpt_shading_rate(pt._ctx, fr.ctypes.data, st0, None, None, None, None) == -1
        bad = capi.IdkPtShadingRateInputs.from_buffer_copy(inputs)
        bad.VelocityRG = None
        expect(rc(i=bad), "idkpt_shading_rate: null argument")
        bad = capi.IdkPtShadingRateInputs.from_buffer_copy(inputs)
        bad.ColorRgba32f = None
        expect(rc(i=bad), "ARRAY source without a colour array")
        for w, h in ((0, H), (W, 0), (-1, H), (16385, H), (W, 16385)):
            bad = capi.IdkPtShadingRateInputs.from_buffer_copy(inputs)
            bad.Width, bad.Height = w, h
            expect(rc(i=bad), "size outside 1..16384")
        bad = capi.IdkPtShadingRateInputs.from_buffer_copy(inputs)
        bad.OnDevice = 2
        expect(rc(i=bad), "OnDevice is neither 0 nor 1")
        bad.OnDevice = 1
        expect(rc(i=bad), "not device memory on the context's device")
        for src in (capi.LIT_SOURCE_MERGED, 7, -1):
            bad = capi.IdkPtShadingRateInputs.from_buffer_copy(inputs)
            bad.Source = src
            expect(rc(i=bad), "source is neither ARRAY nor DEFERRED")
        for mode in (-1, 5):
            expect(rc(s=capi.IdkPtShadingRateSettings(mode, 0.2, 0.04)), "DebugMode outside 0..4")
        for mode in (0, 1):
            expect(rc(s=capi.IdkPtShadingRateSettings(mode, 0.2, 0.04), d=dbg.ctypes.data), "a debug image needs DebugMode 2, 3 or 4")
        for sf, lv in ((np.inf, 0.04), (np.nan, 0.04), (0.2, -np.inf), (0.2, np.nan)):
            expect(rc(s=capi.IdkPtShadingRateSettings(0, sf, lv)), "SpeedFactor or LumVarianceFactor not finite")
        with PathTracer(16, 16) as other:                                # DEFERRED needs a deferred image of the render size
            other.SetScene(scene)
            with pytest.raises(IdkPtError, match="DEFERRED source needs an idkpt_deferred_lighting image"):
                other.ShadingRate(frame, velocity, source=capi.LIT_SOURCE_DEFERRED)
        # misaligned device arrays: rejected before anything runs
        dv, dc = torch.from_numpy(velocity).cuda(), torch.from_numpy(color).cuda()
        buf = torch.zeros(velocity.size + 8, dtype=torch.float32, device="cuda")
        di = capi.IdkPtShadingRateInputs(W, H, 1, capi.LIT_SOURCE_ARRAY, buf.data_ptr() + 4, dc.data_ptr())
        expect(rc(i=di), "OnDevice VelocityRG pointer not 8-byte aligned")
        di = capi.IdkPtShadingRateInputs(W, H, 1, capi.LIT_SOURCE_ARRAY, dv.data_ptr(), dc.data_ptr() + 8)
        expect(rc(i=di), "OnDevice colour pointer not 16-byte aligned")
        dst = deferred_settings(1, 1, 0)
        dst.IsVariableRateShading = 2
        with pytest.raises(IdkPtError, match="IsVariableRateShading is neither 0 nor 1"):
            pt.DeferredLighting(frame, *g, settings=dst)
        # the rejected calls left the rate image valid
        p, n = pt.ShadingRateDevicePtr()
        assert np.array_equal(device_u8(p, n).reshape(good.shape), good)
        assert np.array_equal(canon(pt.DeferredLighting(frame, *g, jitter=JITTER, vrs=True)), canon(good_lit))
        # a rate image of another size
        pt.ShadingRate(frame, velocity[:16, :20], color=color[:16, :20])
        with pytest.raises(IdkPtError, match="IsVariableRateShading needs an idkpt_shading_rate image"):
            pt.DeferredLighting(frame, *g, vrs=True)
        pt.DeferredLighting(frame, *g, jitter=JITTER)                     # the per-pixel pass still works
        pt.ShadingRate(frame, velocity, color=color)
        assert np.array_equal(canon(pt.DeferredLighting(frame, *g, jitter=JITTER, vrs=True)), canon(good_lit))
        pt.SetScene(scene)                                                # a new scene drops the rate image
        with pytest.raises(IdkPtError, match="call idkpt_shading_rate first"):
            pt.ShadingRateDevicePtr()
        pt.Ssao(frame, g[0], g[1])
        with pytest.raises(IdkPtError, match="IsVariableRateShading needs an idkpt_shading_rate image"):
            pt.DeferredLighting(frame, *g, vrs=True)


@pytest.mark.gpu
def test_gpu_vrs_between_async_computes():
    scene, cam, shadows = deferred_setup("cornell")
    w, h = 160, 120
    frame = frame_dt(cam, w, h)
    color, velocity = classifier_inputs(w, h, 5)

    def go(with_vrs):
        with PathTracer(w, h, lanes=4) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            pt.SetFrame(frame)
            pt.SetPointShadows(shadows, [64, 64])
            pt.RenderPointShadows()
            g = gbuffer(pt, scene, frame, w, h)
            pt.Ssao(frame, g[0], g[1])
            want_rates = pt.ShadingRate(frame, velocity, color=color)
            want = pt.DeferredLighting(frame, *g, jitter=JITTER, vrs=True)
            got = []
            for k in range(6):
                pt.ComputeAsync()
                if with_vrs and k in (1, 3):
                    got.append((pt.ShadingRate(frame, velocity, color=color), pt.DeferredLighting(frame, *g, jitter=JITTER, vrs=True)))
            pt.Sync()
            return pt.Result.copy(), (want_rates, want), got

    img0, _, _ = go(False)
    img1, (want_rates, want), got = go(True)
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32))
    for r, lit in got:
        assert np.array_equal(r, want_rates) and np.array_equal(canon(lit), canon(want))
