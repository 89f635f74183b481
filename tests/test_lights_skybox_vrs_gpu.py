"""The light spheres and the skybox under the shading-rate image (k_lights_skybox_vrs) on the GPU: bit for bit against the
oracle, against the per-pixel call at full rate, in the device chain, and its errors and ordering.

float32 images are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import ctypes

import numpy as np
import pytest

import lights_skybox_oracle as lo
import lights_skybox_vrs_oracle as lvo
import vrs_oracle as vo
from idkengine_b200 import capi
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon
from test_lights_skybox_gpu import cube_sky, frame_of, setup, snapshot
from test_vrs_gpu import FIVE, five_rate_inputs

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4
NO_SHADOWS = capi.IdkPtDeferredSettings(0, 0, 0, 0)


def vrs_frame(cam, w, h, turn, dt):
    f = frame_of(cam, w, h, turn).copy()
    f["DeltaRenderTime"] = dt
    return f


def rate_image(pt, kind, frame, w, h, velocity):
    """The context's rate image: "five" (every palette index, the classifier over five_rate_inputs), "frame" (the classifier
    over this frame's lit image and G-buffer velocity, the engine's settings), "1x1" (a flat image: every tile full rate) or
    "4x4" (fast motion: every tile 4x4)."""
    if kind == "five":
        color, vel = five_rate_inputs(w, h, w + h)
        return pt.ShadingRate(frame, vel, FIVE, color=color)
    if kind == "frame":
        return pt.ShadingRate(frame, velocity, source=capi.LIT_SOURCE_DEFERRED)
    v = np.zeros((h, w, 2), np.float32)
    if kind == "1x1":                # no motion and no contrast: 0 / 0 is NaN, which rounds to rate 0
        return pt.ShadingRate(frame, v, FIVE, color=np.full((h, w, 4), 0.5, np.float32))
    v[..., 0] = 1000.0               # fast enough for rate 4 even in a tile with one pixel in the image
    c = np.full((h, w, 4), 0.5, np.float32)
    c[..., :3] += np.random.default_rng(w * h).random((h, w, 3)).astype(np.float32) * 0.1
    return pt.ShadingRate(frame, v, FIVE, color=c)


def run(which, lights, w, h, rates_kind, jitter=None, sky=(0.6, 0.7, 0.9), moving=False, turn=False):
    """GBuffer -> DeferredLighting -> ShadingRate -> LightsAndSkybox(vrs=True) on the GPU, against the oracle on the same inputs."""
    scene, cam = setup(which, lights, moving)
    frame = vrs_frame(cam, w, h, turn, 1.0 if rates_kind in ("five", "4x4") else 1.0 / 60.0)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        g = pt.GBuffer(frame, w, h, jitter=jitter)
        lit = pt.DeferredLighting(frame, *g[:5], settings=NO_SHADOWS, jitter=jitter)
        rates = rate_image(pt, rates_kind, frame, w, h, g[5])
        out = pt.LightsAndSkybox(frame, jitter=jitter, vrs=True)
        assert pt.last_lights_and_skybox_ms > 0
        got_g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
        again = pt.LightsAndSkybox(frame, jitter=jitter, vrs=True)              # idempotent
        again_g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
    want_g, want_col, winner = lvo.lights_and_skybox_vrs(scene, frame, g, lit, rates, jitter=jitter, sky=sky)
    for k, (a, b) in enumerate(zip(got_g, want_g)):
        bad = canon(a) != canon(b)
        assert not bad.any(), f"plane {k}: {int(bad.sum())} values differ"
    assert np.array_equal(canon(got_g[2]), canon(g[2])) and np.array_equal(canon(got_g[3]), canon(g[3]))   # never written
    bad = canon(out) != canon(want_col)
    assert not bad.any(), f"{int(bad.sum())} lit values differ"
    assert out.tobytes() == again.tobytes() and all(a.tobytes() == b.tobytes() for a, b in zip(got_g, again_g))
    if rates_kind == "five" and w * h > 2000:
        assert set(np.unique(rates)) == {0, 1, 2, 3, 4}
    if rates_kind == "4x4":
        assert (rates == 4).all()
    return winner, rates


@pytest.mark.parametrize("which", ["rule", "cornell", "multi_blas", "multi_blas_tlas", "atrium"])
def test_matches_oracle_startup_lights(which):
    winner, _ = run(which, "startup", 96, 64, "five", jitter=JITTER, moving=True, turn=True)
    assert (winner // lo.SPHERE_TRIANGLES == 3).any()   # the light in front of the camera


@pytest.mark.parametrize("which", ["cornell", "atrium"])
def test_matches_oracle_without_lights_classified_frame(which):
    winner, rates = run(which, "none", 96, 64, "frame", jitter=JITTER, sky=cube_sky(), turn=True)
    assert not (winner >= 0).any() and (winner == lo.SKY).any()
    assert rates.max() > 0


@pytest.mark.parametrize("jitter,sky,rates", [(None, "const", "five"), (JITTER, "cube", "frame"), (JITTER, "cube", "4x4")])
def test_matches_oracle_256_lights(jitter, sky, rates):
    winner, _ = run("atrium", "many", 96, 64, rates, jitter=jitter, sky=(0.2, 0.3, 0.4) if sky == "const" else cube_sky(),
                    moving=True, turn=True)
    assert len(np.unique(winner[winner >= 0] // lo.SPHERE_TRIANGLES)) > 10


@pytest.mark.parametrize("w,h", [(97, 61), (37, 23), (1, 1)])
@pytest.mark.parametrize("rates", ["five", "4x4"])
def test_matches_oracle_odd_sizes(w, h, rates):
    run("cornell", "startup", w, h, rates, jitter=JITTER, sky=cube_sky(), moving=True, turn=True)


@pytest.mark.parametrize("which,lights", [("atrium", "startup"), ("cornell", "many")])
def test_full_rate_is_the_per_pixel_call(which, lights):
    """A rate image of all 1x1 gives exactly the bytes of idkpt_lights_and_skybox."""
    scene, cam = setup(which, lights, moving=True)
    w, h = 96, 64
    frame = vrs_frame(cam, w, h, True, 1.0)
    sky = cube_sky()
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        res = []
        for vrs in (False, True):
            pt.GBuffer(frame, w, h, jitter=JITTER, download=False)
            g = pt.GBufferDevicePtrs(tensors=True)
            pt.DeferredLighting(frame, *g[:5], settings=NO_SHADOWS, jitter=JITTER, download=False)
            if vrs:
                assert not rate_image(pt, "1x1", frame, w, h, None).any()
            out = pt.LightsAndSkybox(frame, jitter=JITTER, vrs=vrs)
            res.append([a.tobytes() for a in [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)] + [out]])
    assert res[0] == res[1]


def test_device_chain_equals_array_chain():
    """G-buffer -> coarse deferred lighting -> lights and skybox under the rates -> transparency (DEFERRED), with nothing on the
    host, gives the bytes of the chain whose lights-and-skybox step is the oracle's, fed as arrays."""
    import torch
    scene, cam = setup("rule", "startup", moving=True)
    w, h = 48, 32
    frame = vrs_frame(cam, w, h, True, 1.0)
    st = capi.IdkPtTransparencySettings(0, 0)
    sky = cube_sky()
    color, vel = five_rate_inputs(w, h, 3)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        rates = pt.ShadingRate(frame, vel, FIVE, color=color)
        g = pt.GBuffer(frame, w, h, jitter=JITTER)
        lit = pt.DeferredLighting(frame, *g[:5], settings=NO_SHADOWS, jitter=JITTER, vrs=True)
        want_lit = vo.deferred_lighting_vrs(scene.lights, frame, 0, np.zeros(0, gt.GpuPointShadow), [], g[:5], rates, JITTER)
        assert np.array_equal(canon(lit), canon(want_lit))
        g2, arr, _ = lvo.lights_and_skybox_vrs(scene, frame, g, lit, rates, jitter=JITTER, sky=sky)
        pt.Transparency(frame, g2[0], settings=st, jitter=JITTER, color=arr)

    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        assert pt.ShadingRate(frame, torch.from_numpy(vel).cuda(), FIVE, color=torch.from_numpy(color).cuda(), download=False) is None
        pt.GBuffer(frame, w, h, jitter=JITTER, download=False)
        gt_ = pt.GBufferDevicePtrs(tensors=True)
        pt.DeferredLighting(frame, *gt_[:5], settings=NO_SHADOWS, jitter=JITTER, download=False, vrs=True)
        assert pt.LightsAndSkybox(frame, jitter=JITTER, download=False, vrs=True) is None
        dev_g = [t.cpu().numpy() for t in gt_]
        dev = pt.Transparency(frame, gt_[0], settings=st, jitter=JITTER, source=capi.LIT_SOURCE_DEFERRED)
    assert all(np.array_equal(canon(a), canon(b)) for a, b in zip(dev_g, g2))
    assert np.array_equal(canon(dev), canon(arr))


def call(pt, frame, jitter=None):
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    fr = None if frame is None else np.ascontiguousarray(frame)
    ms = ctypes.c_float()
    return pt._lib.idkpt_lights_and_skybox_vrs(pt._ctx, fr.ctypes.data if fr is not None else None,
                                               jit.ctypes.data if jit is not None else None, None, ctypes.byref(ms))


def test_errors_change_nothing_and_leave_the_context_working():
    scene, cam = setup("cornell", "startup")
    w, h = 40, 24
    frame = vrs_frame(cam, w, h, True, 1.0)
    sky = (0.3, 0.4, 0.5)
    color, vel = five_rate_inputs(w, h, 7)
    with PathTracer(16, 16) as pt:
        assert call(pt, frame) == ERR_NO_SCENE
        pt.SetScene(scene)
        pt.SetSky(sky)
        assert call(pt, None) == ERR_INVALID_ARGUMENT
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # no G-buffer
        g = pt.GBuffer(frame, w, h)
        lit = pt.DeferredLighting(frame, *g[:5], settings=NO_SHADOWS)
        before = snapshot(pt)
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # no rate image
        with pytest.raises(IdkPtError, match="idkpt_lights_and_skybox_vrs: needs an idkpt_shading_rate image of the G-buffer's size"):
            pt.LightsAndSkybox(frame, vrs=True)
        pt.ShadingRate(frame, vel[:16, :20], FIVE, color=color[:16, :20])
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # a rate image of another size
        rates = pt.ShadingRate(frame, vel, FIVE, color=color)
        assert call(pt, None) == ERR_INVALID_ARGUMENT                        # a NULL frame
        assert call(pt, frame, (np.nan, 0.0)) == ERR_INVALID_ARGUMENT
        assert snapshot(pt) == before                                         # a failed call changes no byte
        assert call(pt, frame) == 0                                           # the context still works
        after = snapshot(pt)
        want_g, want_col, _ = lvo.lights_and_skybox_vrs(scene, frame, g, lit, rates, sky=sky)
        assert all(np.array_equal(canon(np.frombuffer(a, np.float32)), canon(b.ravel())) for a, b in zip(after, want_g + (want_col,)))
        pt.SetScene(scene)                                                    # a new scene drops the rate image
        g = pt.GBuffer(frame, w, h)
        pt.DeferredLighting(frame, *g[:5], settings=NO_SHADOWS)
        before = snapshot(pt)
        assert call(pt, frame) == ERR_INVALID_ARGUMENT
        assert snapshot(pt) == before
        pt.ShadingRate(frame, vel, FIVE, color=color)
        assert call(pt, frame) == 0


def test_between_asynchronous_computes():
    scene, cam = setup("cornell", "startup")
    w, h = 32, 24
    frame = vrs_frame(cam, w, h, False, 1.0)
    color, vel = five_rate_inputs(w, h, 2)
    with PathTracer(w, h) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.3, 0.4, 0.5))
        pt.SetFrame(frame)
        g = pt.GBuffer(frame, w, h, jitter=JITTER)
        lit = pt.DeferredLighting(frame, *g[:5], settings=NO_SHADOWS, jitter=JITTER)
        rates = pt.ShadingRate(frame, vel, FIVE, color=color)
        pt.ComputeAsync()
        out = pt.LightsAndSkybox(frame, jitter=JITTER, vrs=True)
        pt.ComputeAsync()
        got_g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
        pt.Sync()
    want_g, want_col, _ = lvo.lights_and_skybox_vrs(scene, frame, g, lit, rates, jitter=JITTER, sky=(0.3, 0.4, 0.5))
    assert np.array_equal(canon(out), canon(want_col))
    assert all(np.array_equal(canon(a), canon(b)) for a, b in zip(got_g, want_g))
