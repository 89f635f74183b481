"""Timing of SSR + merge and the TAA resolve (DESIGN 8f.1e) on the bench atrium (--tris 262144 requested, 267k BLAS triangles
built), with a G-buffer synthesised from the bench camera's first hits (seeded albedo, metallic and lit image), at the engine's
defaults: SSR SampleCount 30, BinarySearchCount 8, MaxDist 50, constant sky; TAA neighbourhood-clamped, PreferAliasingOverBlur
0.25, 6 samples.

    python scripts/time_ssr_taa.py [--tris 262144] [--reps 10] [--out FILE]

Two configurations: render = presentation = 1920x1080, and render scale 0.6 (1152x648) -> 1920x1080. All inputs are CUDA
tensors (OnDevice = 1) and the results stay on the device; TAA reads the merged image (LIT_SOURCE_MERGED). Reports the card
name and power limit read in the same run. kernel_ms is the CUDA-event time of the kernel (median of --reps after two warm-up
calls); call_ms is the host time of the whole synchronous call. algorithmic_bytes counts each buffer once; GB/s = algorithmic
bytes / kernel time, against the 3.35 TB/s HBM3 bound of the H100 SXM data sheet.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def algorithmic_bytes(pas, rw, rh, W=0, H=0):
    """Bytes each pass must move at least once. SSR: depth, normal, albedo, metallic/roughness and the lit image read (4 + 8 +
    12 + 8 + 16 B), the rgba16f SSR image and the rgba32f merged image written (8 + 16 B) per render pixel; the march's depth
    taps and the hit's colour taps fall in the same images. TAA: colour, depth and velocity read once (16 + 4 + 8 B per render
    pixel), the rgba16f history read and the result written (8 + 8 B per presentation pixel)."""
    if pas == "ssr":
        return rw * rh * 72
    return rw * rh * 28 + W * H * 16


def timed(fn, last, reps):
    kernel, call = [], []
    for _ in range(reps + 2):
        t0 = time.perf_counter()
        fn()
        call.append((time.perf_counter() - t0) * 1e3)
        kernel.append(last())
    return float(np.median(kernel[2:])), float(np.median(call[2:]))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam = scenes.atrium(a.tris)
    W, H = 1920, 1080
    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), presentation=[W, H])
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        for scale in (1.0, 0.6):
            rw, rh = int(W * scale), int(H * scale)
            frame = scenes.camera_frame(cam, rw, rh)
            depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, rw, rh)
            rng = np.random.default_rng(1)
            mr = mr.copy()
            mr[..., 0] = rng.random((rh, rw), dtype=np.float32)
            albedo = rng.random((rh, rw, 3), dtype=np.float32)
            lit = rng.random((rh, rw, 4), dtype=np.float32)
            vel = ((rng.random((rh, rw, 2)) - 0.5) * 0.01).astype(np.float32)
            dev = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (depth, nrg, albedo, mr, lit, vel)]
            k, c = timed(lambda: pt.Ssr(frame, *dev[:4], color=dev[4], download=False), lambda: pt.last_ssr_ms, a.reps)
            nb = algorithmic_bytes("ssr", rw, rh)
            out[f"ssr {rw}x{rh}"] = dict(kernel_ms=k, call_ms=c, algorithmic_bytes=nb, gb_per_s=nb / (k * 1e-3) / 1e9,
                                         share_of_hbm_bound=nb / HBM_BYTES_PER_S / (k * 1e-3))
            k, c = timed(lambda: pt.TaaResolve(dev[0], dev[5], W, H, source=capi.LIT_SOURCE_MERGED, download=False),
                         lambda: pt.last_taa_ms, a.reps)
            nb = algorithmic_bytes("taa", rw, rh, W, H)
            out[f"taa {rw}x{rh} -> {W}x{H}"] = dict(kernel_ms=k, call_ms=c, algorithmic_bytes=nb, gb_per_s=nb / (k * 1e-3) / 1e9,
                                                    share_of_hbm_bound=nb / HBM_BYTES_PER_S / (k * 1e-3))
    print("SSR_TAA", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
