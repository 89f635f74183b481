"""The G-buffer pass (k_gbuffer) on the GPU, bit for bit against the oracle, the device chain fed from its images, and its
errors and lifetime.

float32 images are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import functools

import numpy as np
import pytest

import gbuffer_oracle as go
from idkengine_b200 import capi, scenes
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, assert_bits
from test_gbuffer import small_scene

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_NO_SCENE = -1, -4   # IdkPtStatus


@functools.lru_cache(maxsize=None)
def setup(which):
    if which == "cornell":
        return scenes.cornell_1k(threads=1)
    if which in ("multi_blas", "multi_blas_tlas"):
        scene, cam = scenes.multi_blas(threads=1)
        scene.mesh_transforms["PrevModelMatrix"][1, :, 3] -= np.float32([0.2, 0.05, 0.0])
        if which == "multi_blas_tlas":
            scene.build_tlas()
        return scene, cam
    if which == "atrium":
        return scenes.atrium(20000, threads=1)
    if which == "textured_room":
        return scenes.textured_room(threads=1)
    return small_scene()


def prev_of(scene):
    """Previous positions: every vertex moved by a small seeded offset."""
    p = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float32)
    return p + np.random.default_rng(3).uniform(-0.02, 0.02, p.shape).astype(np.float32)


def assert_same(got, want):
    for a, b in zip(got, want):
        assert a.shape == b.shape
        assert_bits(a, b)


@pytest.mark.parametrize("which", ["cornell", "multi_blas", "multi_blas_tlas", "atrium", "textured_room", "small"])
@pytest.mark.parametrize("size", [(96, 64), (37, 23), (8, 8), (1, 1)])
def test_gbuffer_matches_oracle(which, size):
    scene, cam = setup(which)
    w, h = size
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h, device=0) as pt:
        pt.SetScene(scene)
        got = pt.GBuffer(frame, w, h, jitter=JITTER)
        assert pt.last_gbuffer_ms > 0
    assert_same(got, go.gbuffer(scene, frame, w, h, jitter=JITTER))
    if size == (96, 64):
        assert (got[0] < 1).any()


@pytest.mark.parametrize("jitter", [None, JITTER])
@pytest.mark.parametrize("prev", [False, True])
def test_small_scene_jitter_and_previous_positions(jitter, prev):
    scene, cam = setup("small")
    w, h = 64, 48
    frame = scenes.camera_frame(cam, w, h)
    pp = prev_of(scene) if prev else None
    with PathTracer(w, h, device=0) as pt:
        pt.SetScene(scene)
        got = pt.GBuffer(frame, w, h, jitter=jitter, prev_positions=pp)
    assert_same(got, go.gbuffer(scene, frame, w, h, jitter=jitter, prev_positions=pp))


def test_device_chain_equals_host_arrays():
    """idkpt_gbuffer -> ssao -> deferred lighting -> ssr -> taa -> shading rate on the device images gives the same bytes as the
    same calls fed the downloaded arrays."""
    import torch
    scene, cam = setup("cornell")
    w, h = 80, 56
    frame = scenes.camera_frame(cam, w, h)
    results = []
    for on_device in (False, True):
        with PathTracer(w, h, device=0) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            host = pt.GBuffer(frame, w, h, jitter=JITTER)
            if on_device:
                d, n, a, mr, e, v = pt.GBufferDevicePtrs(tensors=True)
                g, vptr = pt.GBufferDevicePtrs()
                assert g.OnDevice == 1 and g.Width == w and g.Height == h and vptr == v.data_ptr()
                assert np.array_equal(d.cpu().numpy(), host[0])
            else:
                d, n, a, mr, e, v = host
            ao = pt.Ssao(frame, d, n)
            st = capi.default_deferred_settings()
            st.ShadowMode = 0
            lit = pt.DeferredLighting(frame, d, n, a, mr, e, settings=st, jitter=JITTER)
            merged = pt.Ssr(frame, d, n, a, mr, source=capi.LIT_SOURCE_DEFERRED)
            taa = pt.TaaResolve(d, v, w, h, source=capi.LIT_SOURCE_MERGED)
            rates = pt.ShadingRate(frame, v, source=capi.LIT_SOURCE_DEFERRED)
            if on_device:
                torch.cuda.synchronize()
            results.append((ao, lit, merged, taa, rates))
    for x, y in zip(*results):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))


def test_errors_and_lifetime():
    scene, cam = setup("small")
    w, h = 32, 24
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h, device=0) as pt:
        L, ctx = pt._lib, pt._ctx
        fr = np.ascontiguousarray(frame)
        assert L.idkpt_gbuffer(ctx, fr.ctypes.data, w, h, None, None, None) == ERR_NO_SCENE
        pt.SetScene(scene)
        assert L.idkpt_gbuffer(None, fr.ctypes.data, w, h, None, None, None) == ERR_INVALID_ARGUMENT
        assert L.idkpt_gbuffer(ctx, None, w, h, None, None, None) == ERR_INVALID_ARGUMENT
        for bw, bh in ((0, h), (w, 0), (16385, h), (w, -1)):
            assert L.idkpt_gbuffer(ctx, fr.ctypes.data, bw, bh, None, None, None) == ERR_INVALID_ARGUMENT
        for bad in ((np.nan, 0.0), (0.0, np.inf)):
            jit = np.float32(bad)
            assert L.idkpt_gbuffer(ctx, fr.ctypes.data, w, h, jit.ctypes.data, None, None) == ERR_INVALID_ARGUMENT
        with pytest.raises(IdkPtError):   # nothing rendered yet
            pt.GBufferDevicePtrs()
        want = go.gbuffer(scene, frame, w, h)
        assert_same(pt.GBuffer(frame, w, h), want)        # the context still works
        g, _ = pt.GBufferDevicePtrs()
        assert g.Depth % 256 == 0 and g.NormalRG % 256 == 0 and g.AlbedoRGB % 256 == 0
        # a failed call leaves no stale pointer
        assert L.idkpt_gbuffer(ctx, fr.ctypes.data, 0, h, None, None, None) == ERR_INVALID_ARGUMENT
        assert_same(pt.GBuffer(frame, w, h), want)
        jit = np.float32((np.nan, 0.0))
        # a call that fails validation runs nothing: the images of the last call stay valid
        assert L.idkpt_gbuffer(ctx, fr.ctypes.data, w, h, jit.ctypes.data, None, None) == ERR_INVALID_ARGUMENT
        pt.GBufferDevicePtrs()
        # idkpt_set_scene drops the images
        pt.SetScene(scene)
        with pytest.raises(IdkPtError):
            pt.GBufferDevicePtrs()
        with pytest.raises(ValueError):   # the previous positions must cover every vertex position
            pt.GBuffer(frame, w, h, prev_positions=np.zeros((3, 3), np.float32))


def test_call_between_async_computes_changes_no_path_traced_image():
    scene, cam = setup("cornell")
    w, h = 64, 48
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.RayDepth = 3
    images = []
    for interleave in (False, True):
        with PathTracer(w, h, s, device=0) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            pt.SetFrame(frame)
            for _ in range(3):
                pt.ComputeAsync()
                if interleave:
                    pt.GBuffer(frame, w, h, jitter=JITTER)
            pt.Sync()
            images.append(pt.Result.copy())
    assert np.array_equal(images[0], images[1])
