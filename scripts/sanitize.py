"""Tiny run of every kernel family for compute-sanitizer (memcheck): small sizes, torch only for the device-memory G-buffer of
the last section."""
import os, sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import numpy as np
from idkengine_b200 import capi, scenes, vxgi, gpu_types as gt
from idkengine_b200.pathtracer import PathTracer

scene, cam = scenes.textured_room(threads=1)
scene.build_tlas(use=False)
w, h = 96, 64
frame = scenes.camera_frame(cam, w, h)
s = capi.default_settings()
s.RayDepth, s.OutputAOVs, s.DoRaySorting = 6, 1, 1
s.Gpu.DoTraceLights = 1
with PathTracer(w, h, s, lanes=3) as pt:
    pt.SetScene(scene); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
    pt.CollectStats = 1
    st = pt.Compute()
    pt.CollectStats = 0
    for _ in range(5):
        pt.ComputeAsync()
    pt.Sync()
    ldr, _ = pt.PostProcess()
    rng = np.random.default_rng(1)
    rays = np.zeros(3000, gt.IdkPtRay)
    rays["Origin"] = rng.uniform(-2.5, 2.5, (3000, 3)).astype(np.float32)
    d = rng.normal(size=(3000, 3)); rays["Direction"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["TMax"] = np.float32(3.4028235e38)
    pt.TraceRays(rays, trace_lights=True); pt.TraceRaysAny(rays, trace_lights=True)
    depth = np.full((h, w), 0.97, np.float32); nrg = np.full((h, w, 2), 0.5, np.float32)
    pt.ShadowsRayTraced(frame, depth, nrg, 0, samples=2)
    pt.SetTextures(scene.textures)
    pt.ComputeAsync(); pt.Sync()
    pt.SetSize(64, 40); pt.SetFrame(scenes.camera_frame(cam, 64, 40))
    pt.ComputeAsync(); pt.ComputeAsync(); pt.Sync()
print("path tracer ok", st.Rays)

scene2, cam2 = scenes.multi_blas(threads=1)
scene2.build_tlas()
with PathTracer(64, 48) as pt:
    pt.SetScene(scene2); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(scenes.camera_frame(cam2, 64, 48))
    pt.Compute()
    dsc = scene2.blas_descs[2]
    tris = scene2.blas_triangles[dsc["TriangleOffset"]:dsc["TriangleOffset"] + dsc["TriangleCount"]]
    idx = np.concatenate([tris["X"], tris["Y"], tris["Z"]]); v0, v1 = int(idx.min()), int(idx.max()) + 1
    u = np.zeros(v1 - v0, gt.GpuUnskinnedVertex)
    u["JointWeights"][:, 0] = 1.0
    for k, c in enumerate("xyz"): u["Position"][:, k] = scene2.positions[c][v0:v1]
    u["Normal"], u["Tangent"] = scene2.vertices["Normal"][v0:v1], scene2.vertices["Tangent"][v0:v1]
    jm = np.zeros((1, 3, 4), np.float32); jm[0, 0, 0] = jm[0, 1, 1] = jm[0, 2, 2] = 1.1
    cmd = np.zeros(1, gt.IdkPtSkinningCmd); cmd["OutputVertexOffset"], cmd["VertexCount"] = v0, v1 - v0
    pt.SetSkinningData(u); pt.SkinVertices(jm, cmd); pt.BlasRefit(0, 3)
    pt.Compute()
print("dynamic ok")

# round 2 additions: TLAS walk inside k_traverse2 (async lanes), BC7 / BC5 / BC4 decode at upload, float textures, cube-map sky
# with seamless filtering, denoise hand-off, point-shadowed lights in the voxeliser
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import copy
import bcn_ref
scene3, cam3 = scenes.instance_grid(2, threads=1)
with PathTracer(80, 56, lanes=3) as pt:
    pt.SetScene(scene3); pt.SetFrame(scenes.camera_frame(cam3, 80, 56))
    rng = np.random.default_rng(3)
    pt.SetSky((0, 0, 0), rng.uniform(0, 2, (6, 8, 8, 4)).astype(np.float32))
    pt.Compute()
    for _ in range(3):
        pt.ComputeAsync()
    pt.Sync()
    pt.TlasBuild(15); pt.TlasBuild(2)
    pt.Compute()
print("tlas phase + cube sky + device tlas build ok")
comp = copy.copy(scene)
comp.textures = []
rng = np.random.default_rng(4)
for k, t in enumerate(scene.textures):
    px = t["pixels"]; hh, ww = px.shape[:2]
    nb = ((hh + 3) // 4) * ((ww + 3) // 4)
    common = dict(wrap_s=t["wrap_s"], wrap_t=t["wrap_t"])
    if k % 3 == 0:
        comp.textures.append(dict(format=capi.IDKPT_TEX_BC7_SRGB, width=ww, height=hh, data=rng.integers(0, 256, (nb, 16), dtype=np.uint8), **common))
    elif k % 3 == 1:
        comp.textures.append(dict(format=capi.IDKPT_TEX_BC5_RG_UNORM, width=ww, height=hh, data=rng.integers(0, 256, (nb, 16), dtype=np.uint8), **common))
    else:
        comp.textures.append(dict(format=capi.IDKPT_TEX_BC4_R_UNORM, width=ww, height=hh, data=rng.integers(0, 256, (nb, 8), dtype=np.uint8), flags=0, **common))
comp.textures[1] = dict(format=capi.IDKPT_TEX_RGBA32F, width=5, height=3, data=rng.uniform(0, 1, (3, 5, 4)).astype(np.float32), wrap_s=33071, wrap_t=33648, flags=1)
s2 = capi.default_settings(); s2.OutputAOVs = 1
with PathTracer(w, h, s2) as pt:
    pt.SetScene(comp); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
    pt.Compute(); pt.Compute()
    pt.Denoise()
    pt.PostProcess(source=capi.IDKPT_IMAGE_DENOISED)
    pt.DenoiseDevicePtrs(); pt.DenoiseImportOutput()
    shadowed = copy.copy(comp)
    shadowed.lights = comp.lights.copy(); shadowed.lights["PointShadowIndex"][:] = 0
    with vxgi.Voxelizer((20, 16, 24), (-3.1, -0.1, -3.1), (3.1, 4.1, 3.1)) as vx:
        vx.SetScene(shadowed); vx.SetShadowTracer(pt); vx.Render()
        vx.SetSlab(5, 17); vx.Render(); vx.LevelDevicePtr(0); vx.Mipmap(); vx.SetSlab(0, 24)
        f3 = scenes.camera_frame(cam, 40, 24)
        vx.ConeTraceRows(f3, np.full((8, 40), 0.95, np.float32), np.full((8, 40, 2), 0.5, np.float32), np.full((8, 40, 2), 0.5, np.float32), 24, 8)
print("bcn + denoise + point shadows + slabs ok")

with vxgi.Voxelizer((24, 20, 28), (-3.1, -0.1, -3.1), (3.1, 4.1, 3.1)) as vx:
    vx.SetScene(scene)
    vx.Render()
    f2 = scenes.camera_frame(cam, 48, 32)
    vx.ConeTrace(f2, np.full((32, 48), 0.95, np.float32), np.full((32, 48, 2), 0.5, np.float32), np.full((32, 48, 2), 0.5, np.float32), vxgi.default_cone_settings())
print("vxgi ok")

# G-buffer lighting: SSAO -> deferred lighting in every ShadowMode (cube maps for Pcf, idkpt_shadows_ray_traced images for
# RayTraced), host arrays and a device-memory G-buffer (OnDevice = 1), odd sizes so that the last tiles are partial
scene4, cam4 = scenes.cornell_1k(threads=1)
scene4.add_light((0.0, 1.6, 0.3), (6.0, 5.5, 5.0), 0.2)
scene4.add_light((-0.6, 0.5, 0.6), (0.5, 0.8, 3.0), 0.1)
scene4.add_light((0.5, 1.2, 0.8), (1.0, 0.4, 0.3), 0.15)
scene4.lights["PointShadowIndex"][:] = [1, 0, -1]
sh4 = scenes.point_shadows([(scene4.lights[li]["Position"], 0.1, 60.0, li) for li in (1, 0)])
gw, gh = 37, 23
f4 = scenes.camera_frame(cam4, gw, gh)
with PathTracer(16, 16) as pt:
    pt.SetScene(scene4)
    pt.SetPointShadows(sh4, [16, 9])
    pt.RenderPointShadows()
    gd, gn, gmr = vxgi.synth_gbuffer(pt, scene4, f4, gw, gh)
    rng = np.random.default_rng(5)
    gb = (gd, gn, rng.random((gh, gw, 3), dtype=np.float32), gmr, rng.random((gh, gw, 3), dtype=np.float32))
    gi = rng.random((gh, gw, 4), dtype=np.float32)
    rtv = [pt.ShadowsRayTraced(f4, gd, gn, li, samples=1)[0] for li in (1, 0)]
    pt.Ssao(f4, gd, gn, capi.IdkPtSsaoSettings(64, 0.5, 1.3, 3))
    for mode in (0, 1, 2):
        pt.DeferredLighting(f4, *gb, settings=capi.IdkPtDeferredSettings(mode, 1, 1), jitter=(0.01, -0.02), indirect=gi, rt_visibility=rtv)
    import torch
    dgb = [torch.from_numpy(a).cuda() for a in gb]
    pt.Ssao(f4, dgb[0], dgb[1], download=False)
    for mode in (1, 2):
        pt.DeferredLighting(f4, *dgb, settings=capi.IdkPtDeferredSettings(mode, 1, 1), indirect=torch.from_numpy(gi).cuda(),
                            rt_visibility=[torch.from_numpy(v).cuda() for v in rtv], download=False)
    pt.SsaoDevicePtr(); pt.DeferredDevicePtr()
print("ssao + deferred lighting ok")

# the end of the raster frame: SSR + merge (ARRAY and DEFERRED sources, constant and 6-face sky, host and device G-buffer),
# then the TAA resolve naive and clamped, upscaling from the render size, from host arrays and on the device from MERGED
with PathTracer(16, 16) as pt:
    pt.SetScene(scene4)
    rng = np.random.default_rng(6)
    gd, gn, gmr = vxgi.synth_gbuffer(pt, scene4, f4, gw, gh)
    gmr = gmr.copy()
    gmr[..., 0] = rng.random((gh, gw), dtype=np.float32)
    gb = (gd, gn, rng.random((gh, gw, 3), dtype=np.float32), gmr, rng.random((gh, gw, 3), dtype=np.float32))
    lit = rng.random((gh, gw, 4), dtype=np.float32)
    vel = ((rng.random((gh, gw, 2)) - 0.5) * 0.1).astype(np.float32)
    pt.Ssr(f4, *gb[:4], color=lit)
    pt.SetSky((0.3, 0.4, 0.5), rng.random((6, 8, 8, 4), dtype=np.float32))
    pt.DeferredLighting(f4, *gb, settings=capi.IdkPtDeferredSettings(0, 0, 0))
    pt.Ssr(f4, *gb[:4], capi.IdkPtSsrSettings(64, 1, 3.0), source=capi.LIT_SOURCE_DEFERRED)
    for naive in (0, 1):
        pt.TaaResolve(gd, vel, 61, 39, capi.IdkPtTaaSettings(naive, 0.25, 6), color=lit)
    dgb = [torch.from_numpy(a).cuda() for a in gb]
    pt.Ssr(f4, *dgb[:4], color=torch.from_numpy(lit).cuda(), download=False)
    pt.TaaResolve(dgb[0], torch.from_numpy(vel).cuda(), 61, 39, source=capi.LIT_SOURCE_MERGED, download=False)
    pt.SsrDevicePtrs(); pt.TaaDevicePtr()
print("ssr + taa resolve ok")

# variable-rate deferred lighting: the classifier in every DebugMode (ARRAY and DEFERRED, host and device inputs), then the
# coarse pass under rate images with every rate, uniform and mixed, at odd sizes (partial tiles, clamped fragment centres)
with PathTracer(16, 16) as pt:
    pt.SetScene(scene4)
    pt.SetPointShadows(sh4, [16, 9])
    pt.RenderPointShadows()
    for vw, vh in ((37, 23), (5, 3), (1, 1), (49, 33)):
        fv = scenes.camera_frame(cam4, vw, vh).copy()
        fv["DeltaRenderTime"] = 1.0
        gd, gn, gmr = vxgi.synth_gbuffer(pt, scene4, fv, vw, vh)
        rng = np.random.default_rng(vw)
        gb = (gd, gn, rng.random((vh, vw, 3), dtype=np.float32), gmr, rng.random((vh, vw, 3), dtype=np.float32))
        pt.Ssao(fv, gd, gn)
        pt.DeferredLighting(fv, *gb, jitter=(0.01, -0.02))
        col = (0.2 + rng.random((vh, vw, 4))).astype(np.float32)
        for mode in range(5):
            pt.ShadingRate(fv, ((rng.random((vh, vw, 2)) - 0.5) * 0.02).astype(np.float32), capi.IdkPtShadingRateSettings(mode, 0.2, 0.04),
                           color=col, debug=mode >= 2)
            pt.ShadingRate(fv, np.zeros((vh, vw, 2), np.float32), capi.IdkPtShadingRateSettings(mode, 0.2, 0.04),
                           source=capi.LIT_SOURCE_DEFERRED, debug=mode >= 2)
        for r in range(5):   # LumVarianceFactor 0, SpeedFactor 1: a mean speed of r / 4 gives rate r
            pt.ShadingRate(fv, np.full((vh, vw, 2), (r / 4.0 + 0.01) / np.sqrt(2), np.float32), capi.IdkPtShadingRateSettings(0, 1.0, 0.0), color=col)
            pt.DeferredLighting(fv, *gb, settings=capi.IdkPtDeferredSettings(1, 1, 0, 1), jitter=(0.01, -0.02))
        spd = np.repeat(np.repeat(rng.integers(0, 5, ((vh + 15) // 16, (vw + 15) // 16)) / 4.0 + 0.01, 16, 0), 16, 1)[:vh, :vw]
        pt.ShadingRate(fv, np.stack([spd, np.zeros_like(spd)], -1).astype(np.float32), capi.IdkPtShadingRateSettings(0, 1.0, 0.0), color=col)
        dgb = [torch.from_numpy(a).cuda() for a in gb]
        pt.DeferredLighting(fv, *dgb, settings=capi.IdkPtDeferredSettings(2, 1, 0, 1), rt_visibility=[dgb[0], dgb[0]], download=False)
        pt.ShadingRate(fv, torch.zeros((vh, vw, 2), device="cuda"), source=capi.LIT_SOURCE_DEFERRED, download=False)
        pt.ShadingRateDevicePtr()
print("shading rate + coarse deferred lighting ok")

# the G-buffer pass: the textured room (alpha cut-outs, every texture slot) through the instance loop and the TLAS walk, odd
# sizes, jitter and previous positions, then the device chain on its images
for use_tlas in (False, True):
    scene.build_tlas(use=use_tlas)
    prev = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float32) + 0.01
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        for gw, gh in ((37, 23), (1, 1), (96, 64)):
            fg = scenes.camera_frame(cam, gw, gh)
            pt.GBuffer(fg, gw, gh, jitter=(0.01, -0.02), prev_positions=prev)
            d, n, a, mr, e, v = pt.GBufferDevicePtrs(tensors=True)
            pt.Ssao(fg, d, n, download=False)
            pt.DeferredLighting(fg, d, n, a, mr, e, settings=capi.IdkPtDeferredSettings(0, 1, 0, 0), download=False)
print("g-buffer pass ok")

# transparency: the textured room's blended card through the instance loop and the TLAS walk, odd sizes, every ShadowMode,
# IsVXGI, host and device arrays and the deferred image
with vxgi.Voxelizer(16, (-3.0, -1.0, -3.0), (3.0, 3.0, 3.0)) as tvx:
    tvx.SetScene(scene); tvx.Render()
    for use_tlas in (False, True):
        scene.build_tlas(use=use_tlas)
        with PathTracer(16, 16) as pt:
            pt.SetScene(scene)
            for gw, gh in ((37, 23), (1, 1), (96, 64)):
                fg = scenes.camera_frame(cam, gw, gh)
                pt.GBuffer(fg, gw, gh, jitter=(0.01, -0.02))
                d, n, a, mr, e, v = pt.GBufferDevicePtrs(tensors=True)
                pt.DeferredLighting(fg, d, n, a, mr, e, settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), download=False)
                for mode in (0, 2):
                    pt.Transparency(fg, d, settings=capi.IdkPtTransparencySettings(mode, 0), source=capi.LIT_SOURCE_DEFERRED, download=False)
                pt.Transparency(fg, d, settings=capi.IdkPtTransparencySettings(0, 1), source=capi.LIT_SOURCE_DEFERRED, voxelizer=tvx)
                pt.Transparency(fg, d.cpu().numpy(), settings=capi.IdkPtTransparencySettings(0, 0), color=np.ones((gh, gw, 4), np.float32))
print("transparency ok")

# the light spheres and the skybox: the textured room with its lights, a light in front of the camera and a cube-map sky, odd
# sizes and jitter, in place into the G-buffer and the deferred image
lit_scene = scenes.textured_room(threads=1)[0]
eye, vd = np.asarray(cam["position"], np.float64), np.asarray(cam["view_dir"], np.float64)
lit_scene.add_light(tuple(eye + vd / np.linalg.norm(vd) * 0.5), (40.0, 50.0, 60.0), 0.3)
with PathTracer(16, 16) as pt:
    pt.SetScene(lit_scene)
    pt.SetSky(np.random.default_rng(2).random((6, 5, 5, 4), dtype=np.float32))
    for gw, gh in ((37, 23), (1, 1), (96, 64)):
        fg = scenes.camera_frame(cam, gw, gh)
        pt.GBuffer(fg, gw, gh, jitter=(0.01, -0.02), download=False)
        d, n, a, mr, e, v = pt.GBufferDevicePtrs(tensors=True)
        pt.DeferredLighting(fg, d, n, a, mr, e, settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), download=False)
        pt.LightsAndSkybox(fg, jitter=(0.01, -0.02))
print("lights and skybox ok")

# the grid visualisation: the brick masks and the march, a constant and a cube-map sky, odd sizes and grid shapes (partial
# bricks and 8x8 blocks), cone angles 0 and 0.25, from outside and inside the grid
with PathTracer(16, 16) as pt, vxgi.Voxelizer((23, 9, 14), (-3.1, -0.1, -3.1), (3.1, 4.1, 3.1)) as vx:
    vx.SetScene(scene); vx.Render()
    for sky in ((0.6, 0.7, 0.9), None):
        if sky is None:
            pt.SkyAtmosphere(face_size=5)
        else:
            pt.SetSky(sky)
        for gw, gh in ((37, 23), (1, 1)):
            for cone in (0.0, 0.25):
                vx.DebugConeAngle = cone
                vx.DebugRender(pt, scenes.camera_frame(cam, gw, gh), gw, gh)
                vx.DebugRender(pt, scenes.camera_frame(dict(position=(6.0, 5.0, -7.0), view_dir=(-0.6, -0.4, 0.7)), gw, gh), gw, gh, out=False)
    vx.DebugDevicePtr()
print("grid visualisation ok")
