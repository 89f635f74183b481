"""Timing of the point-shadow cube maps (DESIGN 8f.1b) and of the voxeliser's two point-shadow modes on the bench atrium
(262k triangles) with the reference's three startup lights (Application.cs:487-498), all shadowed, near = radius, far = 60.

    python scripts/time_point_shadows.py [--tris 262144] [--reps 10] [--out FILE]

Reports the card name and power limit read in the same run. Times are CUDA-event kernel times (median of --reps after two
warm-up calls); Grays/s = traced texels / kernel time.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, shadowed_atrium, write_out  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--grid", type=int, default=384)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam, shadows = shadowed_atrium(a.tris)

    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), lights=len(scenes.STARTUP_LIGHTS))
    med = lambda xs: float(np.median(xs))  # noqa: E731
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        for n in (512, 1024):
            pt.SetPointShadows(shadows, [n] * len(scenes.STARTUP_LIGHTS))
            for count in (1, 3):
                for label, mask, faces in (("all faces", None, 6), ("3-face mask", 0b010101, 3)):
                    masks = None if mask is None else [mask] * count
                    ms = [pt.RenderPointShadows(0, count, masks) for _ in range(a.reps + 2)][2:]
                    texels = faces * n * n * count
                    out[f"render N={n} shadows={count} {label}"] = dict(kernel_ms=med(ms), grays_per_s=texels / (med(ms) * 1e-3) / 1e9)
        # the engine's maps for the voxeliser comparison
        pt.SetPointShadows(shadows, [512] * len(scenes.STARTUP_LIGHTS))
        render_ms = med([pt.RenderPointShadows() for _ in range(a.reps + 2)][2:])
        with vxgi.Voxelizer(a.grid) as vx:
            vx.SetScene(scene)
            res = {}
            for mode in ("shadow rays", "shadow maps"):
                vx.SetShadowTracer(pt if mode == "shadow rays" else None)
                vx.SetShadowMaps(pt if mode == "shadow maps" else None)
                st = [vx.Render() for _ in range(a.reps + 2)][2:]
                res[mode] = dict(voxelize_ms=med([s.VoxelizeMs for s in st]), fragments=int(st[-1].Fragments))
            res["shadow maps"]["render_ms_3x512"] = render_ms
            out[f"voxelize {a.grid}^3"] = res
    print("POINT_SHADOWS", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
