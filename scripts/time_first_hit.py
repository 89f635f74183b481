"""Bounce 0 against the rest of the sample on the bench workload (1080p atrium, RayDepth 9, 1 spp), from the library's CUDA
events (IdkPtStats of a synchronous Compute).

Bounce 0 is ray generation, the primary walk, FirstHit shading and the compaction of its survivors:
    BounceTraverseMs[0] + BounceShadeMs[0] + (OtherMs - AccumulateMs)
k_first_hit is bounce 0's traversal launch and k_compact its shade span; the last term is a separate ray-generation launch,
which only builds before k_first_hit have (0 otherwise), so the script times those the same way.
Prints one JSON line: medians over --samples synchronous samples after --warmup, and the GPU's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import bench  # noqa: E402  (the workload constants)
from idkengine_b200 import capi, scenes  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--samples", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    scene, cam = scenes.atrium(bench.WORKLOAD_TRIS)
    w, h = bench.WIDTH, bench.HEIGHT
    s = capi.default_settings()
    s.RayDepth = bench.RAY_DEPTH
    rows = {"bounce0": [], "rest": [], "total": [], "launches": []}
    with PathTracer(w, h, s, device=0) as pt:
        pt.SetScene(scene)
        pt.SetSky(bench.SKY)
        pt.SetFrame(scenes.camera_frame(cam, w, h))
        for i in range(args.warmup + args.samples):
            st = pt.Compute().as_dict()
            if i < args.warmup:
                continue
            b0 = st["BounceTraverseMs"][0] + st["BounceShadeMs"][0] + (st["OtherMs"] - st["AccumulateMs"])
            rows["bounce0"].append(b0)
            rows["rest"].append(st["TotalMs"] - b0)
            rows["total"].append(st["TotalMs"])
            rows["launches"].append(st["KernelLaunches"])
    out = {k: statistics.median(v) for k, v in rows.items()}
    out = {"bounce0_ms": out["bounce0"], "rest_of_sample_ms": out["rest"], "sample_ms": out["total"],
           "kernel_launches": int(out["launches"]), "samples": args.samples, "gpu": gpu_info()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
