"""The sky generators (k_sky_atmosphere, k_sky_equirect) on the GPU: bit for bit against the oracle, what the sky's consumers
see afterwards, and the calls' semantics (accumulation, validation, ordering, reallocation).

float32 faces are compared as bytes with every NaN canonicalised (the device and x86 produce different NaN payloads)."""
import ctypes
import functools

import numpy as np
import pytest

import oracle_lib as ol
import sky_oracle as so
from idkengine_b200 import capi, scenes
from idkengine_b200.pathtracer import PathTracer
from raster_lib import assert_bits
from test_sky import synthetic_equirect

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT = -1


def atmo(i_steps=40, j_steps=8, intensity=15.0, azimuth=0.0, elevation=0.0):
    return capi.IdkPtAtmosphereSettings(i_steps, j_steps, intensity, azimuth, elevation)


@pytest.mark.parametrize("n", [1, 2, 3, 7, 128, 512])
def test_atmosphere_defaults_match_oracle(n):
    with PathTracer(16, 16) as pt:
        ms = pt.SkyAtmosphere(capi.default_atmosphere_settings(), n)
        got = pt.read_sky()
    assert ms > 0 and got.shape == (6, n, n, 4)
    assert_bits(got, so.atmosphere(capi.default_atmosphere_settings(), n))


SWEEP = [atmo(1, 1), atmo(40, 16, 15.0, 0.7, np.pi / 4), atmo(40, 8, 30.0, 2.5, np.pi / 2), atmo(12, 3, 15.0, -1.0, 1.9),
         atmo(40, 8, 0.0, 0.3, 0.4), atmo(40, 8, -5.0, 0.3, 0.4), atmo(7, 9, 1e3, 7.0, -0.6)]


@pytest.mark.parametrize("k", range(len(SWEEP)))
@pytest.mark.parametrize("n", [3, 16])
def test_atmosphere_sweep_matches_oracle(k, n):
    with PathTracer(16, 16) as pt:
        pt.SkyAtmosphere(SWEEP[k], n)
        got = pt.read_sky()
    assert_bits(got, so.atmosphere(SWEEP[k], n))


@pytest.mark.parametrize("w,h", [(4, 1), (7, 3), (12, 6), (64, 32), (130, 65), (2048, 1024)])
def test_equirect_matches_oracle(w, h):
    img = synthetic_equirect(w, h, w * 1000 + h)
    with PathTracer(16, 16) as pt:
        ms = pt.SkyEquirectangular(img)
        got = pt.read_sky()
    assert ms > 0 and got.shape == (6, w // 4, w // 4, 4)
    assert_bits(got, so.equirect(img))


# ---- consumers: after a generator they see exactly what idkpt_set_sky with the read-back faces gives them -----------------------
@functools.lru_cache(maxsize=None)
def cornell():
    return scenes.cornell_1k(threads=1)


def consumers(pt, scene, cam, w, h):
    """(path-traced Result, lit image after idkpt_lights_and_skybox, SSR-merged image, G-buffer depth) on the context's sky."""
    frame = scenes.camera_frame(cam, w, h)
    pt.SetFrame(frame)
    pt.Compute()
    result = pt.Result
    g = pt.GBuffer(frame, w, h)
    pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0))
    lit = pt.LightsAndSkybox(frame)
    g = pt.GBuffer(frame, w, h)
    merged = pt.Ssr(frame, g[0], g[1], g[2], g[3], color=lit)[0]
    return result, lit, merged, g[0]


def sky_view():
    """Cornell box from outside its open side, so the sky is on screen in every consumer."""
    scene, cam = cornell()
    return scene, dict(cam, position=(0.0, 0.5, 6.0), view_dir=(0.3, 0.35, -1.0))


@pytest.mark.parametrize("gen", ["atmosphere", "equirect"])
def test_consumers_see_the_generated_faces(gen):
    scene, cam = sky_view()
    w, h = 48, 32
    s = capi.default_settings()
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        if gen == "atmosphere":
            pt.SkyAtmosphere(atmo(40, 8, 15.0, 0.4, 0.8), 9)
        else:
            pt.SkyEquirectangular(synthetic_equirect(36, 18, 5))
        faces = pt.read_sky()
        got = consumers(pt, scene, cam, w, h)
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        pt.SetSky(faces)
        want = consumers(pt, scene, cam, w, h)
    for a, b in zip(got, want):
        assert_bits(a, b)
    assert (got[3] == 1.0).any() and (got[3] < 1.0).any()      # sky and surfaces on screen
    o = ol.path_trace(scene, scenes.camera_frame(cam, w, h), s, w, h, sky=faces)
    assert_bits(got[0], o.result)


# ---- semantics ----------------------------------------------------------------------------------------------------------------
def test_resets_accumulation_keeps_colour_and_constant_sky_returns():
    scene, cam = sky_view()
    w, h = 32, 24
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.3, 0.4, 0.5))
        assert pt.read_sky() is None
        pt.SetFrame(frame)
        pt.Compute()
        pt.Compute()
        assert pt.AccumulatedSamples == 2
        pt.SkyAtmosphere(capi.default_atmosphere_settings(), 4)
        assert pt.AccumulatedSamples == 0
        pt.Compute()
        pt.SkyEquirectangular(synthetic_equirect(20, 10, 1))
        assert pt.AccumulatedSamples == 0 and pt.read_sky().shape == (6, 5, 5, 4)
        pt.SetSky((0.3, 0.4, 0.5))                           # FaceSize 0: back to the constant colour
        assert pt.read_sky() is None
        pt.Compute()
        img = pt.Result
    assert_bits(img, ol.path_trace(scene, frame, capi.default_settings(), w, h, sky=(0.3, 0.4, 0.5)).result)


def test_size_changes_reallocate():
    with PathTracer(16, 16) as pt:
        for n in (8, 64, 8, 3, 200):
            pt.SkyAtmosphere(atmo(10, 4, 15.0, 0.2, 0.5), n)
            assert_bits(pt.read_sky(), so.atmosphere(atmo(10, 4, 15.0, 0.2, 0.5), n))
        img = synthetic_equirect(40, 20, 2)
        pt.SkyEquirectangular(img)
        assert_bits(pt.read_sky(), so.equirect(img))


def test_failed_calls_change_no_byte():
    with PathTracer(16, 16) as pt:
        L, c = pt._lib, pt._ctx
        ms = ctypes.c_float()
        pt.SkyAtmosphere(capi.default_atmosphere_settings(), 5)
        before = pt.read_sky().tobytes()
        ok = capi.default_atmosphere_settings()
        img = np.ones((2, 8, 3), np.float32)
        bad_settings = [atmo(0, 8), atmo(1025, 8), atmo(40, 0), atmo(40, 1025), atmo(40, 8, np.nan), atmo(40, 8, np.inf),
                        atmo(40, 8, 15.0, np.inf), atmo(40, 8, 15.0, 0.0, np.nan)]
        for s in bad_settings:
            assert L.idkpt_sky_atmosphere(c, ctypes.byref(s), 5, ctypes.byref(ms)) == ERR_INVALID_ARGUMENT
        for n in (0, -1, 8193):
            assert L.idkpt_sky_atmosphere(c, ctypes.byref(ok), n, ctypes.byref(ms)) == ERR_INVALID_ARGUMENT
        assert L.idkpt_sky_atmosphere(c, None, 5, None) == ERR_INVALID_ARGUMENT
        assert L.idkpt_sky_atmosphere(None, ctypes.byref(ok), 5, None) == ERR_INVALID_ARGUMENT
        assert L.idkpt_sky_equirectangular(c, None, 8, 2, None) == ERR_INVALID_ARGUMENT
        for w, h in ((3, 2), (0, 1), (8, 0), (8, -1), (32772, 1)):
            assert L.idkpt_sky_equirectangular(c, img.ctypes.data, w, h, None) == ERR_INVALID_ARGUMENT
        assert L.idkpt_read_sky(c, None, None, 0) == ERR_INVALID_ARGUMENT
        n = ctypes.c_int32()
        small = np.zeros(6 * 5 * 5 * 4 - 1, np.float32)
        assert L.idkpt_read_sky(c, ctypes.byref(n), small.ctypes.data, small.nbytes) == ERR_INVALID_ARGUMENT
        assert pt.read_sky().tobytes() == before
        assert L.idkpt_sky_atmosphere(c, ctypes.byref(ok), 5, ctypes.byref(ms)) == 0   # the context still works
        assert pt.read_sky().tobytes() == before


def test_ordered_after_queued_samples():
    """A generator called between asynchronous computes waits for the queued samples: they keep the old sky, the next one sees
    the new faces."""
    scene, cam = sky_view()
    w, h = 32, 24
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.3, 0.4, 0.5))
        pt.SetFrame(frame)
        pt.ComputeAsync()
        pt.SkyAtmosphere(capi.default_atmosphere_settings(), 16)
        first = pt.Result                                   # the sample queued before the call, accumulated alone
        pt.ComputeAsync()
        pt.Sync()
        second = pt.Result
        faces = pt.read_sky()
    assert_bits(first, ol.path_trace(scene, frame, s, w, h, sky=(0.3, 0.4, 0.5)).result)
    assert_bits(second, ol.path_trace(scene, frame, s, w, h, sky=faces).result)   # the call reset the accumulation


def test_two_contexts_give_identical_bytes():
    img = synthetic_equirect(64, 32, 9)
    out = []
    for _ in range(2):
        with PathTracer(16, 16) as pt:
            pt.SkyAtmosphere(atmo(40, 8, 15.0, 1.0, 1.0), 32)
            a = pt.read_sky()
            pt.SkyEquirectangular(img)
            out.append((a.tobytes(), pt.read_sky().tobytes()))
    assert out[0] == out[1]
