"""SSR + merge (k_ssr) and the TAA resolve (k_taa_resolve) on the GPU, bit for bit against the oracle.

float32 and float16 images are compared as bits with every NaN canonicalised (the device and x86 produce different NaN
payloads)."""

import numpy as np
import pytest

import ssr_taa_oracle as so
from idkengine_b200 import capi, multigpu, scenes
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, canon, deferred_setup, gbuffer

SKY = (0.35, 0.55, 0.9)


def sky_faces(n=8, seed=2):
    return np.random.default_rng(seed).random((6, n, n, 4), dtype=np.float32) * 2.0


def ssr_gbuffer(pt, scene, frame, w, h, seed=1):
    """raster_lib.gbuffer with seeded metallic values (a tenth of them below SSR's 0.001 threshold) and a seeded
    rgba32f lit image."""
    d, n, a, mr, e = gbuffer(pt, scene, frame, w, h, seed)
    rng = np.random.default_rng(seed + 100)
    mr = mr.copy()
    mr[..., 0] = np.where(rng.random((h, w)) < 0.1, 0.0, rng.random((h, w)) * 0.9 + 0.1)
    lit = np.concatenate([rng.random((h, w, 3), dtype=np.float32) * 4.0, np.ones((h, w, 1), np.float32)], -1)
    return (d, n, a, mr, e), lit


def check_ssr(pt, frame, g, st, sky, lit, source=None):
    """Ssr on the library (ARRAY with `lit`, or DEFERRED with lit = the deferred image) against the oracle."""
    if source == capi.LIT_SOURCE_DEFERRED:
        got = pt.Ssr(frame, g[0], g[1], g[2], g[3], st, source=source)
    else:
        got = pt.Ssr(frame, g[0], g[1], g[2], g[3], st, color=lit)
    want = so.ssr(frame, st, sky, g[0], g[1], g[2], g[3], lit)
    assert np.array_equal(canon(got[0]), canon(want[0]))
    assert np.array_equal(canon(got[1]), canon(want[1]))
    return got


SSR_CASES = {   # name: (W, H, SampleCount, BinarySearchCount, MaxDist)
    "37x23_s30_b8": (37, 23, 30, 8, 50.0),
    "37x23_s1": (37, 23, 1, 8, 50.0),
    "37x23_s64_b0": (37, 23, 64, 0, 3.0),
    "37x23_s64_b1": (37, 23, 64, 1, 3.0),
    "37x23_tiny": (37, 23, 30, 8, 1e-3),
    "37x23_huge": (37, 23, 30, 8, 1e6),
    "8x8_s30_b8": (8, 8, 30, 8, 5.0),
    "1x1_s30_b8": (1, 1, 30, 8, 5.0),
}
SSR_RUNS = [("cornell", c) for c in SSR_CASES] + [(w, c) for w in ("multi_blas_tlas", "atrium") for c in ("37x23_s30_b8", "37x23_s64_b1")]


@pytest.mark.gpu
@pytest.mark.parametrize("which, case", SSR_RUNS)
@pytest.mark.parametrize("faces", [False, True], ids=["constant_sky", "cube_sky"])
def test_gpu_ssr_matches_oracle(which, case, faces):
    scene, cam, _ = deferred_setup(which)
    W, H, samples, bsc, max_dist = SSR_CASES[case]
    st = capi.IdkPtSsrSettings(samples, bsc, max_dist)
    frame = scenes.camera_frame(cam, W, H)
    sky = capi.sky_desc(SKY, sky_faces() if faces else None)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(SKY, sky_faces() if faces else None)
        g, lit = ssr_gbuffer(pt, scene, frame, W, H)
        merged, ssr = check_ssr(pt, frame, g, st, sky, lit)
    assert np.all(merged[..., 3] == 1)
    if max_dist > 1e5:                                   # every reflection's first step already leaves the screen
        assert not np.any(ssr[..., :3])
    elif W * H > 1:
        assert np.any(ssr[..., 3] == 0) and np.any(ssr[..., :3] != 0)


@pytest.mark.gpu
def test_gpu_ssr_every_source_and_device_tensors():
    """ARRAY (host and device) and DEFERRED sources, host and device G-buffers: identical bytes, equal to the oracle."""
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 37, 23
    frame = scenes.camera_frame(cam, W, H)
    st = capi.default_ssr_settings()
    sky = capi.sky_desc(SKY, sky_faces())
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(SKY, sky_faces())
        pt.SetPointShadows(shadows, [32, 32])
        pt.RenderPointShadows()
        g, lit = ssr_gbuffer(pt, scene, frame, W, H)
        host = check_ssr(pt, frame, g, st, sky, lit)
        dg = [torch.from_numpy(a).cuda() for a in g]
        dev = pt.Ssr(frame, dg[0], dg[1], dg[2], dg[3], st, color=torch.from_numpy(lit).cuda())
        assert np.array_equal(canon(host[0]), canon(dev[0])) and np.array_equal(canon(host[1]), canon(dev[1]))
        pt.Ssao(frame, g[0], g[1])
        deferred = pt.DeferredLighting(frame, *g, jitter=JITTER)
        from_deferred = check_ssr(pt, frame, g, st, sky, deferred, source=capi.LIT_SOURCE_DEFERRED)
        pt.DeferredLighting(frame, *dg, jitter=JITTER, download=False)
        dev = pt.Ssr(frame, dg[0], dg[1], dg[2], dg[3], st, source=capi.LIT_SOURCE_DEFERRED)
        assert np.array_equal(canon(from_deferred[0]), canon(dev[0])) and np.array_equal(canon(from_deferred[1]), canon(dev[1]))
        with pytest.raises(TypeError):
            pt.Ssr(frame, dg[0], dg[1], dg[2], dg[3], st, color=lit)


def frame_sequence(cam, w, h, n):
    """n GpuPerFrameData of a camera that moves and turns a little every frame, each with the previous one's ProjView in
    PrevProjView, and a changing TAA jitter."""
    frames, jitters = [], []
    prev = None
    for k in range(n):
        c = dict(cam)
        c["position"] = tuple(np.asarray(cam["position"], np.float64) + np.array([0.02 * k, -0.01 * k, 0.015 * k]))
        c["view_dir"] = tuple(np.asarray(cam["view_dir"], np.float64) + np.array([0.01 * k, 0.0, -0.005 * k]))
        f = scenes.camera_frame(c, w, h)
        if prev is not None:
            f["PrevProjView"] = prev["ProjView"]
        prev = f
        frames.append(f)
        jitters.append(((k % 3 - 1) * 0.37 / w, ((k * 5) % 4 - 1.5) * 0.29 / h))
    return frames, jitters


def reprojected_velocity(frame, depth):
    """uv - uv in the previous frame of every pixel's depth (the G-buffer's velocity), with seeded pixels: pushed off-screen,
    and pixels made the closest of their neighbourhood (depth 0) whose history uv lands exactly on 0 or on 1."""
    h, w = depth.shape
    f = frame[0] if frame.ndim else frame
    ipv = np.asarray(f["InvProjView"], np.float64).reshape(4, 4)
    ppv = np.asarray(f["PrevProjView"], np.float64).reshape(4, 4)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    u, v = (xx + 0.5) / w, (yy + 0.5) / h
    ndc = np.stack([u * 2 - 1, v * 2 - 1, depth.astype(np.float64), np.ones_like(u)], -1)
    world = ndc @ ipv
    world /= world[..., 3:]
    prev = world @ ppv
    pu, pv = prev[..., 0] / prev[..., 3] * 0.5 + 0.5, prev[..., 1] / prev[..., 3] * 0.5 + 0.5
    vel = np.stack([u - pu, v - pv], -1).astype(np.float32)
    vel[~np.isfinite(vel)] = 0.0
    depth = depth.copy()
    vel[1, :: 5] = (2.0, 0.0)                                                  # off-screen
    vel[2, 1:: 6] = (0.0, -3.0)
    f32 = np.float32
    uf = (np.arange(w, dtype=f32) + f32(0.5)) / f32(w)
    vf = (np.arange(h, dtype=f32) + f32(0.5)) / f32(h)
    for y in range(3, h, 4):
        for x in range(0, w, 3):
            depth[y, x] = 0.0
            if uf[x] >= 0.5 and vf[y] >= 0.5:                                  # uv - (uv - 1) == 1 exactly (Sterbenz)
                vel[y, x] = (uf[x] - f32(1.0), vf[y] - f32(1.0))
            else:                                                               # uv - uv == 0
                vel[y, x] = (uf[x], vf[y])
    return depth, vel


TAA_SETTINGS = [(0, 0.25, 6), (0, 0.0, 6), (0, 1.0, 1), (0, 0.25, 1), (1, 0.25, 6), (1, 0.0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1.0, 0.6, 0.5])
@pytest.mark.parametrize("naive, prefer, samples", TAA_SETTINGS)
def test_gpu_taa_sequence_matches_oracle(scale, naive, prefer, samples):
    """Six frames of a moving camera: the deferred image of each frame (with its jitter) resolved against the history, frame by
    frame, at render = presentation size and at render scales 0.6 and 0.5."""
    scene, cam, _ = deferred_setup("cornell")
    W, H = 37, 23
    rw, rh = max(1, int(W * scale)), max(1, int(H * scale))
    st = capi.IdkPtTaaSettings(naive, prefer, samples)
    frames, jitters = frame_sequence(cam, rw, rh, 6)
    history = np.zeros((H, W, 4), np.float16)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        for k, (frame, jit) in enumerate(zip(frames, jitters)):
            g = gbuffer(pt, scene, frame, rw, rh, seed=k)
            depth, vel = reprojected_velocity(frame, g[0])
            lit = pt.DeferredLighting(frame, *g, settings=capi.IdkPtDeferredSettings(0, 0, 0), jitter=jit)
            got = pt.TaaResolve(depth, vel, W, H, st, source=capi.LIT_SOURCE_DEFERRED)
            want = so.taa_resolve(st, lit, depth, vel, history)
            assert np.array_equal(canon(got), canon(want)), k
            assert np.all(got[..., 3] == 1)
            history = want


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(8, 8), (1, 1)])
def test_gpu_taa_tiny_sizes(size):
    W, H = size
    rng = np.random.default_rng(W)
    st = capi.default_taa_settings()
    history = np.zeros((H, W, 4), np.float16)
    with PathTracer(16, 16) as pt:
        for k in range(3):
            color = rng.random((H, W, 4), dtype=np.float32)
            depth = rng.random((H, W), dtype=np.float32)
            vel = ((rng.random((H, W, 2)) - 0.5) * 0.2).astype(np.float32)
            got = pt.TaaResolve(depth, vel, W, H, st, color=color)
            want = so.taa_resolve(st, color, depth, vel, history)
            assert np.array_equal(canon(got), canon(want))
            history = want


@pytest.mark.gpu
def test_gpu_taa_restarts_from_zero_history_on_resize_and_new_scene():
    import torch
    scene, cam, _ = deferred_setup("cornell")
    rng = np.random.default_rng(9)
    st = capi.default_taa_settings()
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        with pytest.raises(IdkPtError, match="call idkpt_taa_resolve first"):
            pt.TaaDevicePtr()

        def step(W, H, rw, rh, history):
            color = rng.random((rh, rw, 4), dtype=np.float32)
            depth = rng.random((rh, rw), dtype=np.float32)
            vel = ((rng.random((rh, rw, 2)) - 0.5) * 0.05).astype(np.float32)
            got = pt.TaaResolve(depth, vel, W, H, st, color=color)
            want = so.taa_resolve(st, color, depth, vel, history if history is not None else np.zeros((H, W, 4), np.float16))
            assert np.array_equal(canon(got), canon(want))
            p, nbytes = pt.TaaDevicePtr()
            assert nbytes == W * H * 8
            dev = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 2,), "<f2"), device="cuda").cpu().numpy()
            assert np.array_equal(canon(dev.reshape(H, W, 4)), canon(got))
            return got
        h = step(20, 12, 12, 8, None)
        h = step(20, 12, 12, 8, h)
        h = step(20, 12, 20, 12, h)                 # a new render size keeps the history
        h = step(24, 12, 20, 12, None)              # a new presentation size restarts from zero
        h = step(24, 12, 20, 12, h)
        pt.SetScene(scene)                          # so does a new scene
        with pytest.raises(IdkPtError, match="call idkpt_taa_resolve first"):
            pt.TaaDevicePtr()
        step(24, 12, 20, 12, None)


@pytest.mark.gpu
def test_gpu_device_ptrs_and_the_merged_source():
    import torch
    scene, cam, _ = deferred_setup("cornell")
    W, H = 53, 31
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(SKY)
        g, lit = ssr_gbuffer(pt, scene, frame, W, H)
        with pytest.raises(IdkPtError, match="call idkpt_ssr first"):
            pt.SsrDevicePtrs()
        merged, ssr = pt.Ssr(frame, *g[:4], color=lit)
        assert pt.Ssr(frame, *g[:4], color=lit, download=False) is None
        (pm, nm), (ps, ns) = pt.SsrDevicePtrs()
        assert nm == W * H * 16 and ns == W * H * 8
        dm = torch.as_tensor(multigpu.DeviceArray(pm, (nm // 4,), "<f4"), device="cuda").cpu().numpy().reshape(H, W, 4)
        ds = torch.as_tensor(multigpu.DeviceArray(ps, (ns // 2,), "<f2"), device="cuda").cpu().numpy().reshape(H, W, 4)
        assert np.array_equal(canon(dm), canon(merged)) and np.array_equal(canon(ds), canon(ssr))
        depth, vel = g[0], np.zeros((H, W, 2), np.float32)
        a = pt.TaaResolve(depth, vel, W, H, source=capi.LIT_SOURCE_MERGED)
        with PathTracer(16, 16) as other:                                      # the same image as an ARRAY
            b = other.TaaResolve(depth, vel, W, H, color=merged)
        assert np.array_equal(canon(a), canon(b))
        assert pt.last_ssr_ms > 0 and pt.last_taa_ms > 0


@pytest.mark.gpu
def test_gpu_errors_leave_the_context_working():
    import torch
    scene, cam, _ = deferred_setup("cornell")
    W, H = 24, 16
    frame = scenes.camera_frame(cam, W, H)
    fr = np.ascontiguousarray(frame)
    lib = capi.load()

    def expect(rc, msg):
        with pytest.raises(IdkPtError, match=msg):
            pt._check(rc, "call")
    with PathTracer(16, 16) as pt:
        z = np.zeros((H, W), np.float32)
        with pytest.raises(IdkPtError, match="idkpt_ssr: no scene"):
            pt.Ssr(frame, z, np.zeros((H, W, 2), np.float32), np.zeros((H, W, 3), np.float32), np.zeros((H, W, 2), np.float32),
                   color=np.zeros((H, W, 4), np.float32))
        pt.SetScene(scene)
        g, lit = ssr_gbuffer(pt, scene, frame, W, H)
        good = pt.Ssr(frame, *g[:4], color=lit)
        gb, _, keep = PathTracer._gbuffer([g[0], g[1], g[2], g[3], None, lit], [1, 2, 3, 2, 3, 4])
        sst = capi.default_ssr_settings()

        def ssr_rc(f=fr, s=sst, gg=None, source=capi.LIT_SOURCE_ARRAY, color=lit.ctypes.data):
            return lib.idkpt_ssr(pt._ctx, f.ctypes.data if f is not None else None, s, gg if gg is not None else gb, source, color, None, None, None)
        assert ssr_rc(f=None) == -1 and lib.idkpt_ssr(pt._ctx, fr.ctypes.data, None, gb, 0, lit.ctypes.data, None, None, None) == -1
        for field in ("Depth", "NormalRG", "AlbedoRGB", "MetallicRoughness"):
            bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
            setattr(bad, field, None)
            expect(ssr_rc(gg=bad), "idkpt_ssr: null argument")
        for w, h in ((0, H), (W, 16385)):
            bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
            bad.Width, bad.Height = w, h
            expect(ssr_rc(gg=bad), "size outside 1..16384")
        for s, msg in ((capi.IdkPtSsrSettings(0, 8, 50.0), "SampleCount outside 1..1024"), (capi.IdkPtSsrSettings(1025, 8, 50.0), "SampleCount outside"),
                       (capi.IdkPtSsrSettings(30, -1, 50.0), "BinarySearchCount outside 0..64"), (capi.IdkPtSsrSettings(30, 65, 50.0), "BinarySearchCount"),
                       (capi.IdkPtSsrSettings(30, 8, float("inf")), "MaxDist not finite"), (capi.IdkPtSsrSettings(30, 8, float("nan")), "MaxDist not finite")):
            expect(ssr_rc(s=s), msg)
        expect(ssr_rc(source=capi.LIT_SOURCE_MERGED), "source is neither ARRAY nor DEFERRED")
        expect(ssr_rc(source=7), "source is neither ARRAY nor DEFERRED")
        expect(ssr_rc(color=None), "ARRAY source without a colour array")
        expect(ssr_rc(source=capi.LIT_SOURCE_DEFERRED), "DEFERRED source needs an idkpt_deferred_lighting image")
        pt.DeferredLighting(frame, *[a[:8, :8] for a in g], settings=capi.IdkPtDeferredSettings(0, 0, 0))
        expect(ssr_rc(source=capi.LIT_SOURCE_DEFERRED), "DEFERRED source needs an idkpt_deferred_lighting image of the render size")
        bad = capi.IdkPtGBuffer.from_buffer_copy(gb)
        bad.OnDevice = 1                                                         # host pointers passed as device memory
        expect(ssr_rc(gg=bad), "not device memory on the context's device")
        dg = [torch.from_numpy(a).cuda() for a in g]
        dlit = torch.from_numpy(lit).cuda()
        buf = torch.zeros(dlit.numel() + 8, dtype=torch.float32, device="cuda")
        shifted = buf[2:2 + dlit.numel()].view(dlit.shape)
        shifted.copy_(dlit)
        with pytest.raises(IdkPtError, match="OnDevice colour pointer not 16-byte aligned"):
            pt.Ssr(frame, *dg[:4], color=shifted)
        with pytest.raises(ValueError):
            pt.Ssr(frame, g[0], g[1], g[2], g[3], color=lit[:, :-1])
        # the rejected calls left the last images valid
        (pm, nm), _ = pt.SsrDevicePtrs()
        assert nm == W * H * 16
        dm = torch.as_tensor(multigpu.DeviceArray(pm, (nm // 4,), "<f4"), device="cuda").cpu().numpy().reshape(H, W, 4)
        assert np.array_equal(canon(dm), canon(good[0]))

        # TAA
        vel = np.zeros((H, W, 2), np.float32)
        pt.TaaResolve(g[0], vel, W, H, color=lit)
        inputs = capi.IdkPtTaaInputs(W, H, 0, capi.LIT_SOURCE_ARRAY, g[0].ctypes.data, vel.ctypes.data, lit.ctypes.data)
        tst = capi.default_taa_settings()

        def taa_rc(s=tst, i=None, w=W, h=H):
            return lib.idkpt_taa_resolve(pt._ctx, s, i if i is not None else inputs, w, h, None, None)
        assert lib.idkpt_taa_resolve(pt._ctx, None, inputs, W, H, None, None) == -1 and lib.idkpt_taa_resolve(pt._ctx, tst, None, W, H, None, None) == -1
        for field in ("Depth", "VelocityRG"):
            bad = capi.IdkPtTaaInputs.from_buffer_copy(inputs)
            setattr(bad, field, None)
            expect(taa_rc(i=bad), "idkpt_taa_resolve: null argument")
        for w, h in ((0, H), (W, 16385), (-1, 3)):
            expect(taa_rc(w=w, h=h), "size outside 1..16384")
            bad = capi.IdkPtTaaInputs.from_buffer_copy(inputs)
            bad.Width, bad.Height = w, h
            expect(taa_rc(i=bad), "size outside 1..16384")
        bad = capi.IdkPtTaaInputs.from_buffer_copy(inputs)
        bad.OnDevice = 2
        expect(taa_rc(i=bad), "OnDevice is neither 0 nor 1")
        bad.OnDevice = 1
        expect(taa_rc(i=bad), "not device memory on the context's device")
        for s, msg in ((capi.IdkPtTaaSettings(2, 0.25, 6), "IsNaiveTaa is neither 0 nor 1"), (capi.IdkPtTaaSettings(0, 0.25, 0), "SampleCount outside 1..1024"),
                       (capi.IdkPtTaaSettings(0, 0.25, 1025), "SampleCount outside"), (capi.IdkPtTaaSettings(0, float("nan"), 6), "PreferAliasingOverBlur not finite")):
            expect(taa_rc(s=s), msg)
        for src, msg in ((3, "source is not ARRAY, DEFERRED or MERGED"), (capi.LIT_SOURCE_DEFERRED, "DEFERRED source needs"),
                         (capi.LIT_SOURCE_MERGED, None)):
            bad = capi.IdkPtTaaInputs.from_buffer_copy(inputs)
            bad.Source = src
            if msg:
                expect(taa_rc(i=bad), msg)
            else:
                assert taa_rc(i=bad) == 0                                           # the merged image of the last Ssr, 24 x 16
                bad.Width = 12
                expect(taa_rc(i=bad), "MERGED source needs an idkpt_ssr image of the render size")
        bad = capi.IdkPtTaaInputs.from_buffer_copy(inputs)
        bad.ColorRgba32f = None
        expect(taa_rc(i=bad), "ARRAY source without a colour array")
        dvel = torch.zeros(H * W * 2 + 4, dtype=torch.float32, device="cuda")
        with pytest.raises(IdkPtError, match="OnDevice VelocityRG pointer not 8-byte aligned"):
            pt.TaaResolve(dg[0], dvel[1:1 + H * W * 2].view(H, W, 2), W, H, color=dlit)
        with pytest.raises(IdkPtError, match="OnDevice colour pointer not 16-byte aligned"):
            pt.TaaResolve(dg[0], dvel[:H * W * 2].view(H, W, 2), W, H, color=shifted)
        with pytest.raises(ValueError):
            pt.TaaResolve(g[0], vel[:, :-1], W, H, color=lit)
        with pytest.raises(ValueError):
            pt.TaaResolve(g[0], vel, W, H, color=lit, source=capi.LIT_SOURCE_DEFERRED)
        # the rejected calls left the last image valid, and the context keeps working
        p, nbytes = pt.TaaDevicePtr()
        last = torch.as_tensor(multigpu.DeviceArray(p, (nbytes // 2,), "<f2"), device="cuda").cpu().numpy().reshape(H, W, 4)
        assert np.all(last[..., 3] == 1)
        assert pt.TaaResolve(g[0], vel, W, H, color=lit).shape == (H, W, 4)


@pytest.mark.gpu
def test_gpu_ssr_taa_between_async_computes():
    scene, cam, _ = deferred_setup("cornell")
    w, h = 160, 120
    frame = scenes.camera_frame(cam, w, h)

    def go(with_passes):
        with PathTracer(w, h, lanes=4) as pt:
            pt.SetScene(scene)
            pt.SetSky(SKY)
            pt.SetFrame(frame)
            g, lit = ssr_gbuffer(pt, scene, frame, w, h)
            vel = np.zeros((h, w, 2), np.float32)
            want = pt.Ssr(frame, *g[:4], color=lit)
            want_taa = [pt.TaaResolve(g[0], vel, w, h, source=capi.LIT_SOURCE_MERGED) for _ in range(2)]
            pt.SetScene(scene)
            pt.SetSky(SKY)
            got = []
            for k in range(6):
                pt.ComputeAsync()
                if with_passes and k in (1, 3):
                    got.append((pt.Ssr(frame, *g[:4], color=lit), pt.TaaResolve(g[0], vel, w, h, source=capi.LIT_SOURCE_MERGED)))
            pt.Sync()
            return pt.Result.copy(), (want, want_taa), got

    img0, _, _ = go(False)
    img1, (want, want_taa), got = go(True)
    assert np.array_equal(img0.view(np.uint32), img1.view(np.uint32))
    for k, ((merged, ssr), taa) in enumerate(got):
        assert np.array_equal(canon(merged), canon(want[0])) and np.array_equal(canon(ssr), canon(want[1]))
        assert np.array_equal(canon(taa), canon(want_taa[k]))


@pytest.mark.gpu
def test_gpu_whole_chain_on_the_device_equals_host_arrays():
    """G-buffer -> SSAO -> deferred lighting -> SSR + merge -> TAA with every image on the device, against the same chain fed
    with host arrays and downloads in between, over three frames at render scale 0.6."""
    import torch
    scene, cam, shadows = deferred_setup("cornell")
    W, H = 61, 37
    rw, rh = int(W * 0.6), int(H * 0.6)
    frames, jitters = frame_sequence(cam, rw, rh, 3)

    def run(on_device):
        out = []
        with PathTracer(16, 16) as pt:
            pt.SetScene(scene)
            pt.SetSky(SKY, sky_faces())
            pt.SetPointShadows(shadows, [32, 32])
            pt.RenderPointShadows()
            for k, (frame, jit) in enumerate(zip(frames, jitters)):
                g, _ = ssr_gbuffer(pt, scene, frame, rw, rh, seed=k)
                depth, vel = reprojected_velocity(frame, g[0])
                if on_device:
                    dg = [torch.from_numpy(a).cuda() for a in g]
                    pt.Ssao(frame, dg[0], dg[1], download=False)
                    pt.DeferredLighting(frame, *dg, jitter=jit, download=False)
                    pt.Ssr(frame, *dg[:4], source=capi.LIT_SOURCE_DEFERRED, download=False)
                    pt.TaaResolve(torch.from_numpy(depth).cuda(), torch.from_numpy(vel).cuda(), W, H, source=capi.LIT_SOURCE_MERGED, download=False)
                    p, n = pt.TaaDevicePtr()
                    out.append(torch.as_tensor(multigpu.DeviceArray(p, (n // 2,), "<f2"), device="cuda").cpu().numpy().reshape(H, W, 4))
                else:
                    pt.Ssao(frame, g[0], g[1])
                    lit = pt.DeferredLighting(frame, *g, jitter=jit)
                    merged, _ = pt.Ssr(frame, *g[:4], color=lit)
                    out.append(pt.TaaResolve(depth, vel, W, H, color=merged))
        return out

    dev, host = run(True), run(False)
    for a, b in zip(dev, host):
        assert np.array_equal(canon(a), canon(b))


@pytest.mark.gpu
def test_gpu_full_size_atrium_1152x648_to_1080p():
    scene, cam, _ = deferred_setup("atrium")
    rw, rh, W, H = 1152, 648, 1920, 1080
    frames, jitters = frame_sequence(cam, rw, rh, 3)
    st, tst = capi.default_ssr_settings(), capi.default_taa_settings()
    sky = capi.sky_desc(SKY)
    history = np.zeros((H, W, 4), np.float16)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.SetSky(SKY)
        for k, frame in enumerate(frames):
            g, lit = ssr_gbuffer(pt, scene, frame, rw, rh, seed=k)
            merged, ssr = check_ssr(pt, frame, g, st, sky, lit)
            depth, vel = reprojected_velocity(frame, g[0])
            got = pt.TaaResolve(depth, vel, W, H, tst, source=capi.LIT_SOURCE_MERGED)
            want = so.taa_resolve(tst, merged, depth, vel, history)
            assert np.array_equal(canon(got), canon(want)), k
            history = want
