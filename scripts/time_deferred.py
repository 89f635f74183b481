"""Timing of the G-buffer lighting passes (DESIGN 8f.1d) on the bench atrium (--tris 262144 requested, 267k BLAS triangles
built) with the reference's three startup lights (Application.cs:487-498), all shadowed at 512^2 (near = radius, far = 60), and a 1080p G-buffer synthesised from the
bench camera's first hits (seeded albedo and emissive).

    python scripts/time_deferred.py [--tris 262144] [--reps 10] [--out FILE]

Runs SSAO at the engine's defaults and deferred lighting in ShadowMode Pcf with IsSSAO, VXGI off and on (the indirect image is
a constant rgba32f image; the kernel reads it once per pixel whatever it holds). Reports the card name and power limit read
in the same run. kernel_ms is the CUDA-event time of the kernel (median of --reps after two warm-up calls); call_ms is the host
time of the whole synchronous call, once with host arrays (uploaded per call, result downloaded) and once with CUDA tensors
(OnDevice = 1, result kept on the device). algorithmic_bytes (algorithmic_bytes() below) counts each buffer once; GB/s =
algorithmic bytes / kernel time, against the 3.35 TB/s HBM3 bound of the H100 SXM data sheet.
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
from timing_lib import card, shadowed_atrium, write_out  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def algorithmic_bytes(pas, w, h, lights=0, shadow_sizes=(), vxgi_on=False):
    """Bytes each pass must move at least once. SSAO: depth (4 B) and normal (8 B) read, R8 result written (1 B) per pixel; its
    SampleCount depth taps per pixel hit the same depth image. Deferred: depth, normal, albedo, metallic/roughness, emissive
    (4 + 8 + 12 + 8 + 12 B), the SSAO image (1 B), the result (16 B) and with VXGI the indirect image (16 B) per pixel; the
    lights (48 B each) and the cube maps (6 N^2 2 B per shadow, an upper bound: the PCF taps read only the texels they
    fall in)."""
    n = w * h
    if pas == "ssao":
        return n * 13
    return n * (61 + (16 if vxgi_on else 0)) + 48 * lights + sum(6 * s * s * 2 for s in shadow_sizes)


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

    scene, cam, shadows = shadowed_atrium(a.tris)
    size, W, H = 512, 1920, 1080

    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), shadows=len(scenes.STARTUP_LIGHTS), shadow_map_size=size, size=[W, H])
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [size] * len(scenes.STARTUP_LIGHTS))
        pt.RenderPointShadows()
        frame = scenes.camera_frame(cam, W, H)
        depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, W, H)
        rng = np.random.default_rng(1)
        albedo = rng.random((H, W, 3), dtype=np.float32)
        emissive = np.where(rng.random((H, W, 1)) < 0.05, 1.0, 0.0).astype(np.float32) * albedo
        host = (depth, nrg, albedo, mr, emissive)
        dev = tuple(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in host)
        gi = np.full((H, W, 4), 0.1, np.float32)
        gi_dev = torch.from_numpy(gi).cuda()
        jitter = (0.0, 0.0)

        k, c_host = timed(lambda: pt.Ssao(frame, host[0], host[1]), lambda: pt.last_ssao_ms, a.reps)
        _, c_dev = timed(lambda: pt.Ssao(frame, dev[0], dev[1], download=False), lambda: pt.last_ssao_ms, a.reps)
        nb = algorithmic_bytes("ssao", W, H)
        out["ssao"] = dict(kernel_ms=k, call_ms_host_arrays=c_host, call_ms_on_device=c_dev, algorithmic_bytes=nb,
                           gb_per_s=nb / (k * 1e-3) / 1e9, share_of_hbm_bound=nb / HBM_BYTES_PER_S / (k * 1e-3))
        for vx in (0, 1):
            st = capi.IdkPtDeferredSettings(capi.SHADOW_MODE_PCF, 1, vx)
            k, c_host = timed(lambda: pt.DeferredLighting(frame, *host, settings=st, jitter=jitter, indirect=gi if vx else None),
                              lambda: pt.last_deferred_ms, a.reps)
            _, c_dev = timed(lambda: pt.DeferredLighting(frame, *dev, settings=st, jitter=jitter, indirect=gi_dev if vx else None,
                                                         download=False), lambda: pt.last_deferred_ms, a.reps)
            nb = algorithmic_bytes("deferred", W, H, len(scenes.STARTUP_LIGHTS), [size] * len(scenes.STARTUP_LIGHTS), bool(vx))
            out[f"deferred pcf vxgi={vx}"] = dict(kernel_ms=k, call_ms_host_arrays=c_host, call_ms_on_device=c_dev, algorithmic_bytes=nb,
                                                  gb_per_s=nb / (k * 1e-3) / 1e9, share_of_hbm_bound=nb / HBM_BYTES_PER_S / (k * 1e-3))
    print("DEFERRED", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
