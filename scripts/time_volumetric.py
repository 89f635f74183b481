"""Timing of the volumetric lighting pass (DESIGN 8f.1c) on the bench atrium (262k triangles) with the reference's three startup
lights (Application.cs:487-498), all shadowed at 512^2 (near = radius, far = 60), and the G-buffer depth synthesised from the
bench camera's first hits at the presentation size.

    python scripts/time_volumetric.py [--tris 262144] [--reps 10] [--out FILE]

Reports the card name and power limit read in the same run. kernel_ms is the CUDA-event time of both kernels (median of --reps
after two warm-up calls); call_ms is the host time of the whole synchronous call, including the depth upload and the result
download. algorithmic_bytes counts each buffer once: the G-buffer depth (read by both kernels), the render-size image and
depth (written, then read), the presentation image and the cube maps; GB/s = algorithmic bytes / kernel time, against the
3.35 TB/s HBM3 bound of the H100 SXM data sheet.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam, shadows = shadowed_atrium(a.tris)
    size = 512

    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), shadows=len(scenes.STARTUP_LIGHTS), shadow_map_size=size)
    med = lambda xs: float(np.median(xs))  # noqa: E731
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [size] * len(scenes.STARTUP_LIGHTS))
        pt.RenderPointShadows()
        for W, H in ((1920, 1080), (3840, 2160)):
            frame = scenes.camera_frame(cam, W, H)
            depth = vxgi.synth_gbuffer(pt, scene, frame, W, H)[0]
            for scale in (0.6, 1.0):
                for samples in (5, 32):
                    st = capi.default_volumetric_settings()
                    st.ResolutionScale, st.SampleCount = scale, samples
                    kernel, call = [], []
                    for _ in range(a.reps + 2):
                        t0 = time.perf_counter()
                        pt.VolumetricLighting(frame, depth, W, H, st, (0.0, 0.0))
                        call.append((time.perf_counter() - t0) * 1e3)
                        kernel.append(pt.last_volumetric_ms)
                    kernel, call = kernel[2:], call[2:]
                    w, h = int(np.float32(W) * np.float32(scale)), int(np.float32(H) * np.float32(scale))
                    nbytes = 2 * W * H * 4 + 2 * w * h * 12 + W * H * 8 + len(scenes.STARTUP_LIGHTS) * 6 * size * size * 2
                    out[f"{W}x{H} scale={scale} samples={samples}"] = dict(
                        render_size=[w, h], kernel_ms=med(kernel), call_ms=med(call), algorithmic_bytes=nbytes,
                        gb_per_s=nbytes / (med(kernel) * 1e-3) / 1e9, share_of_hbm_bound=nbytes / HBM_BYTES_PER_S / (med(kernel) * 1e-3))
    print("VOLUMETRIC", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
