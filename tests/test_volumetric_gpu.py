"""Volumetric lighting (k_volumetric_march, k_volumetric_upscale) on the GPU, bit for bit against the oracle as uint16.

NaN halves are compared as NaN: the device stores every NaN with one payload, the oracle keeps the sign of x86's default NaN."""
import copy
import functools

import numpy as np
import pytest

import volumetric_oracle as vo
from idkengine_b200 import capi, multigpu, scenes, vxgi
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon, crossed_shadows, lit_cornell


@functools.lru_cache(maxsize=None)
def setup(which):
    """(scene, camera, shadows): two shadows per scene, the second one's LightIndex pointing at an earlier light."""
    if which == "cornell":
        scene, cam = lit_cornell(2)
        return scene, cam, crossed_shadows(scene, 0.1, 0.2)
    if which == "multi_blas_tlas":
        scene, cam = scenes.multi_blas(threads=1)
        scene.build_tlas()
        p = (0.2, 1.9, 0.8)
    else:
        scene, cam = scenes.atrium(20000, threads=1)
        p = (0.0, 3.0, 0.5)
    scene.add_light(p, (20.0, 18.0, 15.0), 0.3)
    n = len(scene.lights)
    return scene, cam, scenes.point_shadows([(p, 0.3, 60.0, n - 1), (scene.lights[0]["Position"], 0.3, 60.0, 0)])


def settings(scale=0.6, samples=5, max_dist=50.0):
    st = capi.default_volumetric_settings()
    st.Absorbance[:] = [0.025, 0.04, 0.06]
    st.ResolutionScale, st.SampleCount, st.MaxDist = scale, samples, max_dist
    return st


def run(pt, scene, cam, shadows, maps, W, H, gw, gh, st, jitter=JITTER):
    """One GPU call and the oracle on the maps the GPU holds; asserts equality and returns the GPU image."""
    frame = scenes.camera_frame(cam, W, H)
    depth = vxgi.synth_gbuffer(pt, scene, frame, gw, gh)[0]
    got = pt.VolumetricLighting(frame, depth, W, H, st, jitter)
    want = vo.volumetric_lighting(scene.lights, frame, st, shadows, maps, depth, W, H, jitter)[0]
    assert got.shape == (H, W, 4)
    assert np.array_equal(canon(got), canon(want))
    return got, depth


CASES = {   # name: (W, H, Wg, Hg, scale, SampleCount, MaxDist)
    "scale1": (37, 23, 37, 23, 1.0, 5, 50.0),
    "scale0.6": (37, 23, 37, 23, 0.6, 5, 50.0),
    "scale0.5": (37, 23, 37, 23, 0.5, 5, 50.0),
    "render1x1": (37, 23, 37, 23, 0.05, 5, 50.0),
    "gbuffer_smaller": (160, 90, 96, 54, 0.6, 5, 50.0),
    "samples1": (37, 23, 37, 23, 0.6, 1, 50.0),
    "samples64": (37, 23, 37, 23, 0.6, 64, 50.0),
    "maxdist_clamps": (37, 23, 37, 23, 0.6, 5, 0.4),
}


# every setting on the Cornell box, three of them on the two larger scenes
RUNS = [("cornell", c) for c in CASES] + [(w, c) for w in ("multi_blas_tlas", "atrium") for c in ("scale0.6", "gbuffer_smaller", "samples64")]


@pytest.mark.gpu
@pytest.mark.parametrize("which, case", RUNS)
def test_gpu_volumetric_matches_oracle(which, case):
    scene, cam, shadows = setup(which)
    W, H, gw, gh, scale, samples, max_dist = CASES[case]
    st = settings(scale, samples, max_dist)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [64, 33])
        pt.RenderPointShadows()
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        got, depth = run(pt, scene, cam, shadows, maps, W, H, gw, gh, st)
    assert (depth == 1.0).any() or which != "cornell"                          # sky pixels
    if case == "render1x1":
        assert vo.render_size(W, H, scale) == (1, 1)
        assert np.all(got == got[0, 0])
    assert (got[..., :3] > 0).any()


@pytest.mark.gpu
def test_gpu_volumetric_maps_cleared_rendered_masked_and_none():
    scene, cam, shadows = setup("cornell")
    W, H = 64, 48
    st = settings()
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        results = []
        pt.SetPointShadows(shadows, [48, 32])                                  # freshly cleared: 65535 everywhere
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        assert all(np.all(m == 65535) for m in maps)
        results.append(run(pt, scene, cam, shadows, maps, W, H, W, H, st)[0])
        pt.RenderPointShadows(0, 2, [0b010101, 0b101010])                      # partially rendered through face masks
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        assert all(np.any(m == 65535) and np.any(m != 65535) for m in maps)
        results.append(run(pt, scene, cam, shadows, maps, W, H, W, H, st)[0])
        pt.RenderPointShadows()                                                # fully rendered
        maps = [pt.ReadPointShadow(i) for i in range(2)]
        results.append(run(pt, scene, cam, shadows, maps, W, H, W, H, st)[0])
        assert not np.array_equal(results[0], results[2]) and not np.array_equal(results[1], results[2])
        f = results[0][..., :3].astype(np.float32)
        assert np.all(results[2][..., :3].astype(np.float32) <= f + np.abs(f) * 2e-3)   # occluders only take light away
        pt.SetPointShadows(shadows[:0], [])                                    # no shadows: 0, as with shadowsUBO.Count == 0
        got = run(pt, scene, cam, shadows[:0], [], W, H, W, H, st)[0]
        assert np.all(got[..., :3] == 0) and np.all(got[..., 3] == 1)


@pytest.mark.gpu
def test_gpu_volumetric_device_ptr_matches_download():
    scene, cam, shadows = setup("cornell")
    W, H = 53, 31
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [40, 24])
        pt.RenderPointShadows()
        depth = vxgi.synth_gbuffer(pt, scene, frame, W, H)[0]
        with pytest.raises(IdkPtError, match="call idkpt_volumetric_lighting first"):
            pt.VolumetricDevicePtr()
        host = pt.VolumetricLighting(frame, depth, W, H, settings(), JITTER)
        assert pt.VolumetricLighting(frame, depth, W, H, settings(), JITTER, download=False) is None
        p, nbytes = pt.VolumetricDevicePtr()
        assert nbytes == W * H * 8
        import torch
        dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 2,), "<i2"), device="cuda").cpu().numpy().view(np.uint16)
        assert np.array_equal(dev.reshape(H, W, 4), host.view(np.uint16))
        assert pt.last_volumetric_ms > 0


@pytest.mark.gpu
def test_gpu_volumetric_errors_leave_the_context_working():
    scene, cam, shadows = setup("cornell")
    W, H = 24, 16
    frame = scenes.camera_frame(cam, W, H)
    depth = np.full((H, W), 0.5, np.float32)
    lib = capi.load()
    with PathTracer(16, 16) as pt:
        with pytest.raises(IdkPtError, match="idkpt_volumetric_lighting: no scene"):
            pt.VolumetricLighting(frame, depth, W, H)
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [16, 16])
        pt.RenderPointShadows()
        good = pt.VolumetricLighting(frame, depth, W, H)
        st = settings()
        fr = np.ascontiguousarray(frame)
        for args, msg in (((None, st, depth), "null argument"), ((fr, None, depth), "null argument"), ((fr, st, None), "null argument")):
            f, s, d = args
            rc = lib.idkpt_volumetric_lighting(pt._ctx, f.ctypes.data if f is not None else None, s, d.ctypes.data if d is not None else None,
                                               W, H, W, H, None, None, None)
            assert rc == -1                                                      # IDKPT_ERR_INVALID_ARGUMENT
        for (w, h, gw, gh) in ((0, H, W, H), (W, 16385, W, H), (W, H, 0, H), (W, H, W, 16385), (-1, H, W, H)):
            with pytest.raises(IdkPtError, match="size outside 1..16384"):
                pt._check(lib.idkpt_volumetric_lighting(pt._ctx, fr.ctypes.data, st, depth.ctypes.data, gw, gh, w, h, None, None, None),
                          "idkpt_volumetric_lighting")
        for n in (0, 1025, -5):
            with pytest.raises(IdkPtError, match="SampleCount outside 1..1024"):
                pt.VolumetricLighting(frame, depth, W, H, settings(samples=n))
        for sc in (0.0, -0.5, 1.01, np.nan):
            with pytest.raises(IdkPtError, match=r"ResolutionScale not in \(0, 1\]"):
                pt.VolumetricLighting(frame, depth, W, H, settings(scale=sc))
        with pytest.raises(IdkPtError, match="render size of 0"):
            pt.VolumetricLighting(frame, depth, W, H, settings(scale=0.05))           # (int)(16 * 0.05) == 0
        bad = shadows.copy()
        for li in (len(scene.lights), -1):
            bad[1]["LightIndex"] = li
            pt.SetPointShadows(bad, [16, 16])                                        # accepted: only the volumetric pass reads it
            with pytest.raises(IdkPtError, match="LightIndex is not below the scene's light count"):
                pt.VolumetricLighting(frame, depth, W, H)
        pt.SetPointShadows(shadows, [16, 16])
        assert np.array_equal(pt.VolumetricLighting(frame, depth, W, H).view(np.uint16), good.view(np.uint16))
        pt.SetScene(scene)                                                           # a new scene drops the image
        with pytest.raises(IdkPtError, match="call idkpt_volumetric_lighting first"):
            pt.VolumetricDevicePtr()
        lit = copy.deepcopy(scene)
        lit.lights = lit.lights[:0]
        pt.SetScene(lit)                                                             # no lights: LightIndex 0 is out of range
        pt.SetPointShadows(shadows[:1], [8])
        with pytest.raises(IdkPtError, match="LightIndex is not below"):
            pt.VolumetricLighting(frame, depth, W, H)


@pytest.mark.gpu
def test_gpu_volumetric_between_async_computes():
    scene, cam, shadows = setup("cornell")
    w, h = 160, 120
    frame = scenes.camera_frame(cam, w, h)

    def go(with_volumetric):
        with PathTracer(w, h, lanes=4) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            pt.SetFrame(frame)
            pt.SetPointShadows(shadows, [64, 64])
            pt.RenderPointShadows()
            depth = vxgi.synth_gbuffer(pt, scene, frame, w, h)[0]
            want = pt.VolumetricLighting(frame, depth, w, h, settings(), JITTER)
            got = []
            for k in range(6):
                pt.ComputeAsync()
                if with_volumetric and k in (1, 3):
                    got.append(pt.VolumetricLighting(frame, depth, w, h, settings(), JITTER))
            pt.Sync()
            return pt.Result.copy(), want, got

    img0, _, _ = go(False)
    img1, want, got = go(True)
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32))
    for g in got:
        assert np.array_equal(g.view(np.uint16), want.view(np.uint16))
