"""Timing of the sky generators (DESIGN 8f.1j).

    python scripts/time_sky.py [--reps 10] [--out FILE]

k_sky_atmosphere at face sizes 128 (the engine's), 512 and 1024, each with 40 x 8 (the engine's) and 40 x 16 steps: the
kernel's CUDA-event time, median of --reps after two warm-up calls, and its rate in det_exp calls (6 n^2 ISteps (2 JSteps + 5)
per call; the kernel is arithmetic-bound). k_sky_equirect from a 2048 x 1024 and an 8192 x 4096 RGB float image: the kernel
time and the call time including the host-to-device upload of the image (host clock around the synchronous call), medians of
--reps after two warm-ups. The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, median_ms, write_out  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    result = dict(card=card(), reps=a.reps, atmosphere=[], equirect=[])
    with PathTracer(16, 16) as pt:
        for n in (128, 512, 1024):
            for i_steps, j_steps in ((40, 8), (40, 16)):
                s = capi.IdkPtAtmosphereSettings(i_steps, j_steps, 15.0, 0.0, 0.5)
                ms = median_ms(lambda: pt.SkyAtmosphere(s, n), a.reps)
                exps = 6 * n * n * i_steps * (2 * j_steps + 5)
                run = dict(face_size=n, i_steps=i_steps, j_steps=j_steps, k_sky_atmosphere_ms=round(ms, 4),
                           det_exp_per_s=float("%.4g" % (exps / (ms * 1e-3))))
                result["atmosphere"].append(run)
                print(json.dumps(run), flush=True)
        rng = np.random.default_rng(0)
        for w, h in ((2048, 1024), (8192, 4096)):
            img = rng.uniform(0.0, 4.0, (h, w, 3)).astype(np.float32)
            kernel, call = [], []
            for _ in range(a.reps + 2):
                t0 = time.perf_counter()
                kernel.append(pt.SkyEquirectangular(img))
                call.append((time.perf_counter() - t0) * 1e3)
            run = dict(width=w, height=h, face_size=w // 4, k_sky_equirect_ms=round(float(np.median(kernel[2:])), 4),
                       call_ms=round(float(np.median(call[2:])), 3), source_mb=round(img.nbytes / 1e6, 1))
            result["equirect"].append(run)
            print(json.dumps(run), flush=True)
    print(json.dumps(dict(card=result["card"])), flush=True)
    write_out(a.out, result)


if __name__ == "__main__":
    main()
