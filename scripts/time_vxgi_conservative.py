"""Cost of Voxelizer.IsConservativeRasterization (DESIGN section 7) on bench.py's VXGI record: the bench atrium (262k
triangles) with its lights plus the reference's three startup lights (Application.cs:488-490), a 384^3 grid over the
default bounds. The two coverage rules alternate within one run on one context.

    python scripts/time_vxgi_conservative.py [--tris 262144] [--reps 15] [--warmup 3] [--out FILE]
    python scripts/time_vxgi_conservative.py --cpu-only      # the oracle's fragment counts of both rules, no GPU

Reports VoxelizeMs (CUDA events around the voxelise kernels, median of --reps after --warmup calls per rule) and Fragments
for both rules, with the card name and power limit read in the same run, and the oracle's fragment counts of both rules
(computed on the CPU, which needs no GPU), which the device counts must equal.
"""
import argparse
import copy
import json
import os
import sys

REPO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import numpy as np  # noqa: E402

from idkengine_b200 import scenes, vxgi  # noqa: E402
from timing_lib import card, write_out  # noqa: E402

RULES = {"centre": False, "conservative": True}


def bench_scene(tris):
    """bench.py's vxgi_record scene: the atrium's own lights plus the three startup lights, radius 0.3."""
    scene, _ = scenes.atrium(tris)
    sc = copy.copy(scene)
    sc.lights = scene.lights.copy()
    for light in scenes.STARTUP_LIGHTS:
        sc.add_light(*light)
    return sc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--grid", type=int, default=384)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-only", action="store_true", help="only the oracle's fragment counts")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    import oracle_lib as ol
    import vxgi_conservative_oracle as vco
    scene = bench_scene(a.tris)
    ci = vxgi.create_info(a.grid)
    out = dict(triangles=int(len(scene.blas_triangles)), lights=int(len(scene.lights)), grid=f"{a.grid}^3")
    out["oracle_fragments"] = {k: int((vco if c else ol).vx_voxelize(scene, ci)[2]) for k, c in RULES.items()}
    if not a.cpu_only:
        out["card"] = card()
        ms = {k: [] for k in RULES}
        frags = {}
        with vxgi.Voxelizer(a.grid) as vx:
            vx.SetScene(scene)
            for i in range(a.warmup + a.reps):
                for k, c in RULES.items():                     # the two rules alternate, so drift hits both alike
                    vx.IsConservativeRasterization = c
                    st = vx.Render()
                    frags[k] = int(st.Fragments)
                    if i >= a.warmup:
                        ms[k].append(st.VoxelizeMs)
        for k in RULES:
            assert frags[k] == out["oracle_fragments"][k], (k, frags[k], out["oracle_fragments"][k])
            out[k] = dict(voxelize_ms_median=float(np.median(ms[k])), voxelize_ms_min=float(np.min(ms[k])),
                          voxelize_ms_max=float(np.max(ms[k])), fragments=frags[k])
        out["ratio_ms"] = out["conservative"]["voxelize_ms_median"] / out["centre"]["voxelize_ms_median"]
    out["ratio_fragments"] = out["oracle_fragments"]["conservative"] / out["oracle_fragments"]["centre"]
    print("VXGI_CONSERVATIVE", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
