"""Scope table 8f.3: Bloom + TonemapAndGammaCorrect present chain (Application.cs:217-223)."""
import numpy as np
import pytest

import oracle_lib as ol
import post_ref64
from idkengine_b200 import capi, scenes


def synthetic_hdr(w, h, seed=0):
    rng = np.random.default_rng(seed)
    img = rng.uniform(0.0, 1.2, (h, w, 4)).astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    blob = 30.0 * np.exp(-(((xx - w * 0.3) ** 2 + (yy - h * 0.6) ** 2) / (0.002 * w * h)))
    img[..., :3] += blob[..., None].astype(np.float32)
    img[..., 3] = 1.0
    return img


def test_oracle_tonemap_properties():
    """Oracle sanity: black stays (dithered) black, the curve is monotonic in luminance and saturates at white, the sRGB
    transfer of mid-grey lands where the closed-form AgX-less formula says when tonemapping is off."""
    st = capi.default_post_settings()
    st.IsBloom = 0
    ramp = np.zeros((8, 256, 4), np.float32)
    ramp[..., :3] = (np.arange(256, dtype=np.float32) / 32.0)[None, :, None] ** 2
    out = ol.post_process(ramp, st)
    assert out[..., 3].min() == 255
    lum = out[0, :, 0].astype(int)
    assert lum[0] <= 1 and lum[-1] >= 250
    assert (np.diff(out[0, ::8, 0].astype(int)) >= 0).all()
    st.DoTonemapAndSrgbTransform = 0
    flat = np.full((8, 8, 4), 0.5, np.float32)
    out = ol.post_process(flat, st)
    vals = np.unique(out[..., :3]).astype(int)
    assert vals.min() >= 125 and vals.max() <= 130 and len(vals) >= 3      # 0.5 * 255 = 127.5 +- Bayer dither of +-2 LSB


def test_oracle_bloom_properties_two_prefiltered_levels():
    """No bloom below the threshold; around a hot spot, bloom that falls off and peaks where the float64 chain of
    tests/post_ref64.py peaks (0.147 here: Prefilter runs on down levels 0 and 1, as the engine's Lod-0 dispatches do)."""
    st = capi.default_post_settings()
    img = np.full((96, 128, 4), 0.3, np.float32)
    _, bloom = ol.post_process(img, st, want_bloom=True)
    assert bloom.shape == (48, 64, 3) and np.abs(bloom).max() == 0.0            # nothing above the threshold: no bloom
    img[40:44, 60:64, :3] = 50.0
    out, bloom = ol.post_process(img, st, want_bloom=True)
    peak = post_ref64.bloom64(img, st.BloomThreshold, st.BloomMaxColor, st.BloomMinusLods)[1][0].max()
    assert 0.1 < peak < 0.2 and abs(bloom.max() - peak) <= 2.0 ** -10 * peak
    assert bloom[22, 31].sum() > bloom[2, 2].sum()                                # energy around the hot spot, falling off
    st.IsBloom = 0
    plain = ol.post_process(img, st)
    assert (out.astype(int) >= plain.astype(int) - 1).all() and (out.astype(int) > plain.astype(int) + 3).any()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,bloom,tonemap,minus", [(256, 144, 1, 1, 3), (250, 131, 1, 1, 1), (64, 48, 0, 1, 3), (97, 33, 1, 0, 0), (2, 2, 1, 1, 3)])
def test_post_process_bit_exact(w, h, bloom, tonemap, minus):
    from idkengine_b200.pathtracer import PathTracer
    st = capi.default_post_settings()
    st.IsBloom, st.DoTonemapAndSrgbTransform, st.BloomMinusLods = bloom, tonemap, minus
    st.Exposure = 0.3
    img = synthetic_hdr(w, h, seed=w)
    with PathTracer(w, h) as pt:
        pt.WriteResult(img)
        g, ms = pt.PostProcess(st)
        g2, _ = pt.PostProcess(st)
    o = ol.post_process(img, st)
    assert np.array_equal(g, o), int(np.abs(g.astype(int) - o.astype(int)).max())
    assert np.array_equal(g, g2) and ms > 0


@pytest.mark.gpu
def test_post_process_of_path_traced_frame(cornell):
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = cornell
    w, h = 160, 120
    with PathTracer(w, h) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(scenes.camera_frame(cam, w, h))
        for _ in range(3):
            pt.Compute()
        hdr = pt.Result.copy()
        ldr, _ = pt.PostProcess()
        assert pt.AccumulatedSamples == 3                    # presenting does not disturb the accumulation
        none, _ = pt.PostProcess(download=False)
        assert none is None
    assert np.array_equal(ldr, ol.post_process(hdr))
    assert ldr[..., :3].std() > 10


@pytest.mark.gpu
def test_post_process_errors():
    from idkengine_b200.pathtracer import PathTracer
    with PathTracer(64, 64, tile=(8, 0, 2)) as pt:
        with pytest.raises(RuntimeError):
            pt.PostProcess()                                 # a tile holds only its own rows
    with PathTracer(1, 1) as pt:
        with pytest.raises(RuntimeError):
            pt.PostProcess()                                 # bloom needs 2x2


# ------------------------------------------------------------------------------------------------ denoise hand-off (8f.3)
def noisy_scene_images(w=96, h=64, seed=3):
    """A piecewise-flat 'render' with heavy noise plus clean albedo / normal guides: two materials split by an edge."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    left = (xx < w // 2)[..., None]
    albedo = np.where(left, np.array([0.8, 0.2, 0.2], np.float32), np.array([0.2, 0.3, 0.9], np.float32)).astype(np.float32)
    normal = np.where(left, np.array([0.0, 0.0, 1.0], np.float32), np.array([1.0, 0.0, 0.0], np.float32)).astype(np.float32)
    light = (0.5 + 0.5 * yy / h)[..., None].astype(np.float32)
    clean = albedo * light
    noisy = clean * rng.uniform(0.2, 1.8, (h, w, 1)).astype(np.float32)
    pad = lambda a: np.concatenate([a, np.ones((h, w, 1), np.float32)], -1)
    return pad(noisy.astype(np.float32)), pad(albedo), pad(normal), clean


def test_oracle_denoise_reduces_noise_and_keeps_edges():
    noisy, albedo, normal, clean = noisy_scene_images()
    out = ol.denoise(noisy, albedo, normal)
    err_in = np.abs(noisy[..., :3] - clean).mean()
    err_out = np.abs(out[..., :3] - clean).mean()
    assert err_out < 0.35 * err_in                       # the noise is mostly gone
    w = noisy.shape[1]
    # ... and nothing bled across the material edge: both sides keep their own hue
    assert out[:, w // 2 - 3, 0].mean() > 2.0 * out[:, w // 2 - 3, 2].mean()
    assert out[:, w // 2 + 3, 2].mean() > 2.0 * out[:, w // 2 + 3, 0].mean()
    assert np.all(out[..., 3] == 1.0)
    st = capi.default_denoise_settings()
    st.Iterations = 0
    assert np.array_equal(ol.denoise(noisy, albedo, normal, st)[..., :3], noisy[..., :3] / np.maximum(albedo[..., :3], np.float32(0.001)) * np.maximum(albedo[..., :3], np.float32(0.001)))


@pytest.mark.gpu
@pytest.mark.parametrize("demod", [1, 0])
def test_gpu_denoise_bit_exact_and_oidn_buffers(demod):
    """idkpt_denoise on a real low-sample render with AOVs == oracle_denoise, bit for bit; the OIDN-layout device buffers
    hold the packed RGB floats Texture.Download(PixelFormat.RGB, Float) would produce; the denoised image feeds the present chain."""
    import torch
    from idkengine_b200 import multigpu
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = scenes.cornell_1k(threads=1)
    w, h = 160, 104
    s = capi.default_settings()
    s.OutputAOVs = 1
    st = capi.default_denoise_settings()
    st.Demodulate = demod
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(scenes.camera_frame(cam, w, h))
        for _ in range(4):
            pt.Compute()
        res, alb, nrm = pt.Result, pt.AlbedoTexture, pt.NormalTexture
        ms = pt.Denoise(st)
        den = pt.Denoised
        ptrs, nbytes = pt.DenoiseDevicePtrs()
        assert nbytes == w * h * 12
        packed = [torch.as_tensor(multigpu.DeviceArray(p, (h, w, 3)), device="cuda").cpu().numpy() for p in ptrs]
        ldr, _ = pt.PostProcess(source=capi.IDKPT_IMAGE_DENOISED)
        # the OIDN path: an external filter writes the output buffer, the library adopts it
        out_t = torch.as_tensor(multigpu.DeviceArray(ptrs[3], (h, w, 3)), device="cuda")
        out_t.copy_(torch.as_tensor(multigpu.DeviceArray(ptrs[0], (h, w, 3)), device="cuda") * 0.5)
        torch.cuda.synchronize()
        pt.DenoiseImportOutput()
        adopted = pt.Denoised
    want = ol.denoise(res, alb, nrm, st)
    assert ms > 0 and np.array_equal(den.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(packed[0], res[..., :3]) and np.array_equal(packed[1], alb[..., :3]) and np.array_equal(packed[2], nrm[..., :3])
    assert np.array_equal(packed[3], den[..., :3])
    assert np.array_equal(ldr, ol.post_process(want))
    assert np.array_equal(adopted[..., :3], res[..., :3] * np.float32(0.5)) and np.all(adopted[..., 3] == 1.0)
    noise_in = np.abs(np.diff(res[..., :3], axis=1)).mean()
    assert np.abs(np.diff(den[..., :3], axis=1)).mean() < 0.9 * noise_in       # real edges remain, the noise between them shrinks
