"""The light spheres and the skybox (k_lights_skybox) on the GPU: bit for bit against the oracle, in the device chain, and its
errors and lifetime.

float32 images are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import copy
import ctypes
import functools

import numpy as np
import pytest

import lights_skybox_oracle as lo
from idkengine_b200 import capi, scenes
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon, rule_scene

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4


def cube_sky(n=5):
    """A small cube map with distinct faces, so cube edges and corners are on screen."""
    rng = np.random.default_rng(11)
    faces = rng.random((6, n, n, 4), dtype=np.float32)
    faces[..., 0] += np.arange(6, dtype=np.float32)[:, None, None]
    return faces


@functools.lru_cache(maxsize=None)
def base(which):
    if which == "rule":
        return rule_scene()
    if which == "cornell":
        return scenes.cornell_1k(threads=1)
    if which in ("multi_blas", "multi_blas_tlas"):
        scene, cam = scenes.multi_blas(threads=1)
        if which == "multi_blas_tlas":
            scene.build_tlas()
        return scene, cam
    return scenes.atrium(20000, threads=1)


def setup(which, lights, moving=False):
    """(scene, camera) with its lights replaced: "none", "startup" (the three startup lights and a radius-0.3 light 0.5 in
    front of the camera, the engine's add-light click) or "many" (256 lights around the view, the near one first)."""
    scene, cam = base(which)
    scene = copy.deepcopy(scene)
    scene.lights = np.zeros(0, gt.GpuLight)
    eye = np.asarray(cam["position"], np.float64)
    vd = np.asarray(cam["view_dir"], np.float64)
    vd = vd / np.linalg.norm(vd)
    near = (tuple(eye + vd * 0.5), (61.0, 42.0, 55.0), 0.3)
    if lights == "startup":
        for L in scenes.STARTUP_LIGHTS + [near]:
            scene.add_light(*L)
    elif lights == "many":
        scene.add_light(*near)
        rng = np.random.default_rng(5)
        for _ in range(255):
            p = eye + vd * rng.uniform(0.5, 8.0) + rng.uniform(-2.5, 2.5, 3)
            scene.add_light(tuple(p), tuple(rng.uniform(0.5, 60.0, 3)), float(rng.uniform(0.02, 0.6)))
    if moving and len(scene.lights):
        scene.lights["PrevPosition"] = scene.lights["Position"] - np.array([0.04, -0.02, 0.07], np.float32)
    return scene, cam


def frame_of(cam, w, h, turn):
    frame = scenes.camera_frame(cam, w, h)
    if turn:   # the previous frame looked 3 degrees to the side and a little down
        vd = np.asarray(cam["view_dir"], np.float64)
        c, s = np.cos(0.05), np.sin(0.05)
        prev = scenes.make_per_frame_data(cam["position"], (c * vd[0] + s * vd[2], vd[1] - 0.03, -s * vd[0] + c * vd[2]), w, h,
                                          cam.get("fov_y_deg", 102.0))
        frame["PrevView"], frame["PrevProjView"] = prev["View"], prev["ProjView"]
    return frame


def run(which, lights, w, h, jitter=None, sky=(0.6, 0.7, 0.9), moving=False, turn=False):
    """The pass on the GPU after GBuffer and DeferredLighting, against the oracle on the same inputs."""
    scene, cam = setup(which, lights, moving)
    frame = frame_of(cam, w, h, turn)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        g = pt.GBuffer(frame, w, h, jitter=jitter)
        lit = pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), jitter=jitter)
        out = pt.LightsAndSkybox(frame, jitter=jitter)
        assert pt.last_lights_and_skybox_ms > 0
        got_g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
        again = pt.LightsAndSkybox(frame, jitter=jitter)                      # idempotent
        again_g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
    want_g, want_col, winner = lo.lights_and_skybox(scene, frame, g, lit, jitter=jitter, sky=sky)
    for k, (a, b) in enumerate(zip(got_g, want_g)):
        bad = canon(a) != canon(b)
        assert not bad.any(), f"plane {k}: {int(bad.sum())} values differ"
    assert np.array_equal(canon(got_g[2]), canon(g[2])) and np.array_equal(canon(got_g[3]), canon(g[3]))   # never written
    bad = canon(out) != canon(want_col)
    assert not bad.any(), f"{int(bad.sum())} lit values differ"
    assert out.tobytes() == again.tobytes() and all(a.tobytes() == b.tobytes() for a, b in zip(got_g, again_g))
    return winner


@pytest.mark.parametrize("which", ["rule", "cornell", "multi_blas", "multi_blas_tlas", "atrium"])
def test_matches_oracle_startup_lights(which):
    winner = run(which, "startup", 96, 64, jitter=JITTER, moving=True, turn=True)
    assert (winner // lo.SPHERE_TRIANGLES == 3).any()   # the light in front of the camera


@pytest.mark.parametrize("which", ["cornell", "atrium"])
def test_matches_oracle_without_lights(which):
    winner = run(which, "none", 96, 64, sky=cube_sky(), turn=True)
    assert not (winner >= 0).any()


@pytest.mark.parametrize("jitter,sky", [(None, "const"), (JITTER, "cube")])
def test_matches_oracle_256_lights(jitter, sky):
    winner = run("atrium", "many", 96, 64, jitter=jitter, sky=(0.2, 0.3, 0.4) if sky == "const" else cube_sky(), moving=True)
    assert len(np.unique(winner[winner >= 0] // lo.SPHERE_TRIANGLES)) > 10


@pytest.mark.parametrize("w,h", [(37, 23), (8, 8), (1, 1)])
@pytest.mark.parametrize("which", ["cornell", "multi_blas_tlas"])
def test_matches_oracle_odd_sizes(which, w, h):
    run(which, "startup", w, h, jitter=JITTER, sky=cube_sky(), moving=True, turn=True)


def test_cube_sky_edges_and_corners_with_a_turning_camera():
    scene, cam = setup("cornell", "startup", moving=True)
    cam = dict(cam, position=(0.0, 0.5, 60.0), view_dir=(0.6, 0.9, 0.5))   # away from the scene, at a cube corner
    w, h = 64, 48
    frame = frame_of(cam, w, h, True)
    sky = cube_sky(3)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        g = pt.GBuffer(frame, w, h)
        lit = pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0))
        out = pt.LightsAndSkybox(frame)
        got_v = pt.GBufferDevicePtrs(tensors=True)[5].cpu().numpy()
    want_g, want_col, winner = lo.lights_and_skybox(scene, frame, g, lit, sky=sky)
    assert (winner == lo.SKY).all()
    assert np.abs(want_g[5]).max() > 1e-3
    assert np.array_equal(canon(out), canon(want_col)) and np.array_equal(canon(got_v), canon(want_g[5]))


def test_device_chain_equals_array_chain():
    """G-buffer -> deferred lighting -> lights and skybox -> transparency (DEFERRED) -> SSR -> TAA (MERGED) on device pointers gives
    the bytes of the chain fed with the oracle's lights-and-skybox result as arrays."""
    scene, cam = setup("rule", "startup", moving=True)
    w, h = 48, 32
    frame = frame_of(cam, w, h, True)
    st = capi.IdkPtTransparencySettings(0, 0)
    ds = capi.IdkPtDeferredSettings(0, 0, 0, 0)
    sky = cube_sky()
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        g = pt.GBuffer(frame, w, h, jitter=JITTER)
        lit = pt.DeferredLighting(frame, *g[:5], settings=ds, jitter=JITTER)
        g2, arr, _ = lo.lights_and_skybox(scene, frame, g, lit, jitter=JITTER, sky=sky)
        pt.Transparency(frame, g2[0], settings=st, jitter=JITTER, color=arr)
        m_arr = pt.Ssr(frame, g2[0], g2[1], g2[2], g2[3], color=arr)[0]
        t_arr = pt.TaaResolve(g2[0], g2[5], w, h, color=m_arr)

    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        pt.GBuffer(frame, w, h, jitter=JITTER, download=False)
        gt_ = pt.GBufferDevicePtrs(tensors=True)
        pt.DeferredLighting(frame, *gt_[:5], settings=ds, jitter=JITTER, download=False)
        pt.LightsAndSkybox(frame, jitter=JITTER, download=False)
        dev = pt.Transparency(frame, gt_[0], settings=st, jitter=JITTER, source=capi.LIT_SOURCE_DEFERRED)
        m_dev = pt.Ssr(frame, *gt_[:4], source=capi.LIT_SOURCE_DEFERRED)[0]
        t_dev = pt.TaaResolve(gt_[0], gt_[5], w, h, source=capi.LIT_SOURCE_MERGED)
    assert np.array_equal(canon(dev), canon(arr))
    assert np.array_equal(canon(m_dev), canon(m_arr))
    assert np.array_equal(np.asarray(t_dev).view(np.uint16), np.asarray(t_arr).view(np.uint16))


def call(pt, frame, jitter=None):
    jit = None if jitter is None else np.ascontiguousarray(jitter, np.float32)
    fr = None if frame is None else np.ascontiguousarray(frame)
    ms = ctypes.c_float()
    return pt._lib.idkpt_lights_and_skybox(pt._ctx, fr.ctypes.data if fr is not None else None,
                                           jit.ctypes.data if jit is not None else None, None, ctypes.byref(ms))


def snapshot(pt):
    g = [t.cpu().numpy().copy() for t in pt.GBufferDevicePtrs(tensors=True)]
    p, n = pt.DeferredDevicePtr()
    out = np.zeros(n // 4, np.float32)
    import torch
    from idkengine_b200.multigpu import DeviceArray
    out[:] = torch.as_tensor(DeviceArray(p, (n // 4,)), device="cuda").cpu().numpy()
    return [a.tobytes() for a in g + [out]]


def test_errors_change_nothing_and_set_scene_drops_the_images():
    scene, cam = setup("cornell", "startup")
    w, h = 24, 16
    frame = frame_of(cam, w, h, False)
    with PathTracer(16, 16) as pt:
        assert call(pt, frame) == ERR_NO_SCENE
        pt.SetScene(scene)
        assert call(pt, None) == ERR_INVALID_ARGUMENT
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # no G-buffer
        g = pt.GBuffer(frame, w, h)
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # no deferred image
        pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0))
        before = snapshot(pt)
        assert call(pt, frame, (np.nan, 0.0)) == ERR_INVALID_ARGUMENT
        assert call(pt, frame, (0.0, np.inf)) == ERR_INVALID_ARGUMENT
        assert snapshot(pt) == before                                         # a failed call changes no byte
        pt.GBuffer(frame, w + 8, h, download=False)
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # deferred image of another size
        pt.GBuffer(frame, w, h, download=False)
        assert call(pt, frame) == 0
        pt.SetScene(scene)
        assert call(pt, frame) == ERR_INVALID_ARGUMENT                       # set_scene dropped the G-buffer
        with pytest.raises(IdkPtError):
            pt.LightsAndSkybox(frame)


def test_between_asynchronous_computes():
    scene, cam = setup("cornell", "startup")
    w, h = 32, 24
    frame = frame_of(cam, w, h, False)
    with PathTracer(w, h) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.3, 0.4, 0.5))
        pt.SetFrame(frame)
        g = pt.GBuffer(frame, w, h, jitter=JITTER)
        lit = pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), jitter=JITTER)
        pt.ComputeAsync()
        out = pt.LightsAndSkybox(frame, jitter=JITTER)
        pt.ComputeAsync()
        got_g = [t.cpu().numpy() for t in pt.GBufferDevicePtrs(tensors=True)]
        pt.Sync()
    want_g, want_col, _ = lo.lights_and_skybox(scene, frame, g, lit, jitter=JITTER, sky=(0.3, 0.4, 0.5))
    assert np.array_equal(canon(out), canon(want_col))
    assert all(np.array_equal(canon(a), canon(b)) for a, b in zip(got_g, want_g))
