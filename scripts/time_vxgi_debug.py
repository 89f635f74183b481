"""Cost of Voxelizer.DebugRender (idkvx_debug_render, DESIGN 8f.1k) and of its empty-space skip: bench.py's atrium with the
reference's startup lights, voxelised at 256^3 and 384^3 over the default bounds, rendered at 1920x1080 from the bench camera
(inside the grid) and from a camera outside the grid looking across it, at DebugConeAngle 0 and 0.25 and DebugStepMultiplier
0.4 and 0.05.

    python scripts/time_vxgi_debug.py [--reps 10] [--warmup 2] [--grids 256,384] [--variant-lib PATH] [--out FILE]

The library skips the fetches of level-0 samples in empty 4^3 bricks. To time the march without the skip, the script
compiles a second copy of libidkpt with -DIDKVX_DEBUG_SKIP=0 into a temporary directory (or loads --variant-lib), and the
two variants run alternately, each on its own contexts, so that drift hits both alike. Both must give the same image and
ConeSteps. Reported per case: ConeTraceMs (CUDA events around the call's kernels, median of --reps after --warmup calls),
samples per second from ConeSteps, and bytes per second at 64 B per sample (eight 8-B texels of one level; cone angle 0,
where every sample reads level 0 only) or 128 B per sample (two levels; cone angle 0.25, an upper bound: samples whose lod
is an integer read one level). The card name and power limit are read in the same run.
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile

REPO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402

from idkengine_b200 import build, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402

OUTSIDE = dict(position=(34.0, 24.0, -30.0), view_dir=(-0.7, -0.35, 0.6))   # beyond the +x, +y, -z corner, looking across


def build_variant(tmp):
    """libidkpt without the empty-space skip, compiled with the library's own flags into tmp."""
    out = os.path.join(tmp, "libidkpt_noskip.so")
    srcs = [os.path.join(build.CSRC_DIR, f) for f in sorted(os.listdir(build.CSRC_DIR)) if f.endswith(".cu")]
    subprocess.run([build.find_nvcc()] + build.NVCC_FLAGS + ["-DIDKVX_DEBUG_SKIP=0", "-I", build.INCLUDE_DIR, "-I", build.CSRC_DIR,
                                                             "-o", out] + srcs, check=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--grids", default="256,384")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--variant-lib", default=None, help="a libidkpt built with -DIDKVX_DEBUG_SKIP=0 (default: build one)")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam = scenes.atrium(a.tris)
    sc = copy.copy(scene)
    sc.lights = scene.lights.copy()
    for light in scenes.STARTUP_LIGHTS:
        sc.add_light(*light)
    w, h = a.width, a.height
    views = {"bench_camera_inside": scenes.camera_frame(cam, w, h), "outside_across": scenes.camera_frame(OUTSIDE, w, h)}
    out = dict(card=card(), triangles=int(len(sc.blas_triangles)), resolution=f"{w}x{h}", reps=a.reps, warmup=a.warmup, cases=[])
    with tempfile.TemporaryDirectory() as tmp:
        variant = a.variant_lib or build_variant(tmp)
        libs = {"skip": build.LIBIDKPT, "no_skip": variant}
        for g in (int(s) for s in a.grids.split(",")):
            ctx = {}
            try:
                for k, path in libs.items():
                    vx = vxgi.Voxelizer(g, lib_path=path)
                    pt = PathTracer(8, 8, lib_path=path)
                    pt.SkyAtmosphere(face_size=128)
                    vx.SetScene(sc)
                    vx.Render()
                    ctx[k] = (vx, pt)
                for view, frame in views.items():
                    for cone in (0.0, 0.25):
                        for step in (0.4, 0.05):
                            ms = {k: [] for k in libs}
                            res = {}
                            for i in range(a.warmup + a.reps):
                                for k, (vx, pt) in ctx.items():            # the variants alternate
                                    vx.DebugConeAngle, vx.DebugStepMultiplier = cone, step
                                    img, st = vx.DebugRender(pt, frame, w, h, out=(i == 0))
                                    if i == 0:
                                        res[k] = (img, int(st.ConeSteps))
                                    if i >= a.warmup:
                                        ms[k].append(st.ConeTraceMs)
                            assert res["skip"][1] == res["no_skip"][1] and np.array_equal(res["skip"][0].view(np.uint32), res["no_skip"][0].view(np.uint32))
                            steps = res["skip"][1]
                            bps = 64 if cone == 0.0 else 128
                            case = dict(grid=f"{g}^3", view=view, cone_angle=cone, step_multiplier=step, cone_steps=steps, bytes_per_sample=bps)
                            for k in libs:
                                med = float(np.median(ms[k]))
                                case[k] = dict(ms_median=med, ms_min=float(np.min(ms[k])), ms_max=float(np.max(ms[k])),
                                               gsamples_per_s=steps / med / 1e6, gb_per_s=steps * bps / med / 1e6)
                            case["speedup"] = case["no_skip"]["ms_median"] / case["skip"]["ms_median"]
                            out["cases"].append(case)
                            print("CASE", json.dumps(case), flush=True)
            finally:
                for vx, pt in ctx.values():
                    vx.Dispose()
                    pt.Dispose()
    print("VXGI_DEBUG", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
