"""Call time of the ray-traced shadows, the cone trace and the volumetric light with the G-buffer as host arrays (the host-array
entry points) against the device G-buffer of idkpt_gbuffer read in place (the *_gbuffer entry points, results kept on the
device), on the bench atrium (262k triangles) with the reference's three startup lights, all shadowed at 512^2, at 1920x1080
(DESIGN 8f.1c).

    python scripts/time_device_lighting.py [--tris 262144] [--reps 10] [--out FILE]

Reports the card name, power limit and maximum SM clock read in the same run. call_ms is the host time of the whole
synchronous call (uploads and downloads included), kernel_ms the CUDA-event time of its kernels; each the median of --reps
after two warm-up calls. Shadows: light 0, one sample (RasterPipeline.RayTracingSamples). Cone trace: the engine's 256^3 grid
and cone settings. Volumetric: the engine's settings at ResolutionScale 0.6 and 1.0.
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


def timed(call, reps):
    """(median call ms, median kernel ms) over reps runs after two warm-up runs; call() runs the call and returns its kernel ms."""
    calls, kernels = [], []
    for _ in range(reps + 2):
        t0 = time.perf_counter()
        kernels.append(call())
        calls.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(calls[2:])), float(np.median(kernels[2:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam, shadows = shadowed_atrium(a.tris)
    W, H = 1920, 1080
    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), size=[W, H])
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(64, 64) as pt, vxgi.Voxelizer(256) as vx:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [512] * len(scenes.STARTUP_LIGHTS))
        pt.RenderPointShadows()
        vx.SetScene(scene)
        vx.SetShadowMaps(pt)
        vx.Render()
        host = pt.GBuffer(frame, W, H)
        dev = pt.GBufferDevicePtrs()

        def row(host_call, dev_call):
            h_call, h_kernel = timed(host_call, a.reps)
            d_call, d_kernel = timed(dev_call, a.reps)
            return dict(host_call_ms=h_call, host_kernel_ms=h_kernel, device_call_ms=d_call, device_kernel_ms=d_kernel)

        out["shadows_ray_traced"] = row(lambda: pt.ShadowsRayTraced(frame, host[0], host[1], 0, samples=1)[1],
                                        lambda: (pt.ShadowsRayTracedGBuffer(frame, dev, 0, 0, samples=1, download=False), pt.last_shadows_ms)[1])
        out["cone_trace"] = row(lambda: vx.ConeTrace(frame, host[0], host[1], host[3])[1].ConeTraceMs,
                                lambda: vx.ConeTraceGBuffer(frame, dev, download=False)[1].ConeTraceMs)
        for scale in (0.6, 1.0):
            st = capi.default_volumetric_settings()
            st.ResolutionScale = scale
            out[f"volumetric scale={scale}"] = row(lambda: (pt.VolumetricLighting(frame, host[0], W, H, st), pt.last_volumetric_ms)[1],
                                                   lambda: (pt.VolumetricLightingGBuffer(frame, dev, W, H, st, download=False),
                                                            pt.last_volumetric_ms)[1])
    print("DEVICE_LIGHTING", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
