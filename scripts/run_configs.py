#!/usr/bin/env python
"""Run the BASELINE.json configs other than the bench workload on one GPU and print one JSON line each
(timings from the library's CUDA events; sampled bit-exact parity against the CPU oracle where it finishes in seconds).

  python scripts/run_configs.py [config3] [config4] [config5] [sort]
"""
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import oracle_lib as ol  # noqa: E402
from idkengine_b200 import capi, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402


def pt_config(name, scene, cam, w, h, depth, sort, steps=5, band=None):
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.RayDepth, s.DoRaySorting = depth, sort
    out = {"config": name, "width": w, "height": h, "ray_depth": depth, "sort": sort, "build": scene.build_info}
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        pt.CollectStats = 1
        st = pt.Compute()
        S, T, I, R = st.NodePairFetches, st.TriangleTests, st.InstanceVisits, st.Rays
        pt.CollectStats = 0
        for _ in range(3):
            pt.Compute()
        pt.ResetAccumulation()
        ms = trav = shade = sortms = 0.0
        rays = 0
        for _ in range(steps):
            st = pt.Compute()
            ms += st.TotalMs; trav += st.TraverseMs; shade += st.ShadeMs; sortms += st.SortMs; rays += st.Rays
        out.update(mrays_per_s=rays / ms / 1e3, ms_per_frame=ms / steps, traverse_ms=trav / steps, shade_ms=shade / steps,
                   sort_ms=sortms / steps, rays_per_frame=rays / steps, S_per_ray=S / R, T_per_ray=T / R,
                   traverse_alg_gbs=(64 * S + 52 * T + 48 * I + 52 * R) / 1e9 / (trav / steps * 1e-3) * (rays / steps / R))
        # sampled parity: stand-alone traversal of every 997th primary ray vs the oracle
        r = ol.gui_test_rays(frame, w, h)[::997].copy()
        g, _ = pt.TraceRays(r)
        o = ol.trace_rays(scene, r)
        out["sampled_traversal_parity"] = bool(all(np.array_equal(g[k], o[k]) for k in ("T", "TriangleId", "BaryX", "BaryY", "NodePairFetches", "TriangleTests")))
    if band is not None:
        # full path-tracer parity on a stripe tile (same tile map on both sides)
        with PathTracer(w, h, s, tile=band) as pt:
            pt.SetScene(scene)
            pt.SetSky((0.6, 0.7, 0.9))
            pt.SetFrame(frame)
            pt.Compute()
            img = pt.Result
        ref = ol.path_trace(scene, frame, s, w, h, tile=band, want_rays=False)
        rows = ref.result[..., 3] == 1.0
        out["band_path_trace_parity"] = bool(np.array_equal(img[rows], ref.result[rows]))
        out["band_rows"] = int(rows[:, 0].sum())
    print(json.dumps(out))


def config3():
    t0 = time.time()
    scene, cam = scenes.atrium(9_000_000)
    print(f"# config3 scene built in {time.time() - t0:.1f}s", file=sys.stderr)
    pt_config("config3: Intel-Sponza-sized synthetic 9M tris 1920x1080 8 bounces, ray-sort on", scene, cam, 1920, 1080, 9, 1, band=(8, 40, 135))


def config4():
    t0 = time.time()
    scene, cam = scenes.street_canyon(3_900_000)
    print(f"# config4 scene built in {time.time() - t0:.1f}s", file=sys.stderr)
    pt_config("config4: Bistro-sized synthetic 3.9M tris (rotated) 3840x2160 8 bounces (1 GPU leg)", scene, cam, 3840, 2160, 9, 0, band=(8, 100, 270))


def sort_ab():
    scene, cam = scenes.atrium(262144)
    for sort in (0, 1):
        pt_config(f"bench workload, sort={sort}", scene, cam, 1920, 1080, 9, sort)


def config5():
    scene, cam = scenes.atrium(262144)
    for light in scenes.STARTUP_LIGHTS:
        scene.add_light(*light)
    w, h = 1920, 1080
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, mr = ol.synth_gbuffer(scene, frame, w, h)
    out = {"config": "config5: VXGI 384^3 rgba16f voxelize + mip + cone trace, 262k atrium, 3 lights, 1920x1080"}
    with vxgi.Voxelizer(384) as vx:
        vx.SetScene(scene)
        vx.Render()
        best = None
        for _ in range(5):
            s = vx.Render()
            tot = s.ClearMs + s.VoxelizeMs + s.MipmapMs
            if best is None or tot < best[0]:
                best = (tot, s.ClearMs, s.VoxelizeMs, s.MipmapMs, s.Fragments)
        out.update(voxelize_total_ms=best[0], clear_ms=best[1], voxelize_ms=best[2], mipmap_ms=best[3], fragments=int(best[4]))
        cone = None
        for _ in range(3):
            img, cs = vx.ConeTrace(frame, depth, nrg, mr)
            cone = cs.ConeTraceMs if cone is None else min(cone, cs.ConeTraceMs)
        out.update(cone_trace_ms=cone, cone_steps=int(cs.ConeSteps), cone_alg_gbs=cs.ConeSteps * 16 * 8 / 1e9 / (cone * 1e-3),
                   clear_gbs=384 ** 3 * 8 / 1e9 / (best[1] * 1e-3), mean_indirect=[float(v) for v in img[..., :3].mean(axis=(0, 1))])
    # parity at a size the oracle finishes in seconds (same scene, 96^3, 480x270)
    ci = vxgi.create_info(96)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    f2 = scenes.camera_frame(cam, 480, 270)
    d2, n2, m2 = ol.synth_gbuffer(scene, f2, 480, 270)
    ref, steps = ol.vx_cone_trace(ci, raw, f2, vxgi.default_cone_settings(), d2, n2, m2)
    with vxgi.Voxelizer(96) as vx:
        vx.SetScene(scene)
        s = vx.Render()
        ok = s.Fragments == frags and all(np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)) for l, lv in enumerate(levels))
        img, cs = vx.ConeTrace(f2, d2, n2, m2)
        out["parity_96cubed_all_levels"] = bool(ok)
        out["parity_cone_trace_480x270"] = bool(np.array_equal(img, ref) and cs.ConeSteps == steps)
    print(json.dumps(out))


if __name__ == "__main__":
    which = sys.argv[1:] or ["config5", "sort", "config3", "config4"]
    for w in which:
        {"config3": config3, "config4": config4, "config5": config5, "sort": sort_ab}[w]()
