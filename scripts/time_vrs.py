"""Timing of variable-rate deferred lighting (DESIGN 8f.1f) on the bench atrium (--tris 262144 requested) with the reference's
three startup lights (Application.cs:487-498), all shadowed at 512^2 (near = radius, far = 60), ShadowMode Pcf with IsSSAO,
and a 1080p G-buffer synthesised from the bench camera's first hits; every input is a CUDA tensor and every output stays on
the device.

    python scripts/time_vrs.py [--tris 262144] [--reps 20] [--out FILE]

Reports the classifier's kernel time (over this frame's lit image and a seeded camera-motion velocity), and the deferred
lighting call's kernel time (CUDA events around its kernels) per pixel (k_deferred_lighting) and coarse
(k_vrs_scan + k_deferred_lighting_vrs) at all 1x1, at the classifier's image for this frame (with the share of tiles per
rate) and at all 4x4; each is the median of --reps after two warm-up calls, the per-pixel and coarse calls alternating. The
card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, shadowed_atrium, write_out  # noqa: E402


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam, shadows = shadowed_atrium(a.tris)
    size, W, H = 512, 1920, 1080

    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), shadows=len(scenes.STARTUP_LIGHTS), shadow_map_size=size, size=[W, H])
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, [size] * len(scenes.STARTUP_LIGHTS))
        pt.RenderPointShadows()
        frame = scenes.camera_frame(cam, W, H).copy()
        frame["DeltaRenderTime"] = 1.0 / 60.0
        depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, W, H)
        rng = np.random.default_rng(1)
        albedo = rng.random((H, W, 3), dtype=np.float32)
        emissive = np.where(rng.random((H, W, 1)) < 0.05, 1.0, 0.0).astype(np.float32) * albedo
        dev = tuple(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (depth, nrg, albedo, mr, emissive))
        # a camera pan: screen-space motion that grows towards the image's right edge
        xs = np.linspace(0.0, 1.0, W, dtype=np.float32)
        vel = np.zeros((H, W, 2), np.float32)
        vel[..., 0] = 0.002 * xs[None, :]
        dvel = torch.from_numpy(vel).cuda()
        st = capi.IdkPtDeferredSettings(capi.SHADOW_MODE_PCF, 1, 0, 0)
        pt.Ssao(frame, dev[0], dev[1], download=False)

        def lighting(vrs):
            pt.DeferredLighting(frame, *dev, settings=st, download=False, vrs=vrs)
            return pt.last_deferred_ms

        lighting(False)
        ks = []
        for _ in range(a.reps + 2):
            pt.ShadingRate(frame, dvel, source=capi.LIT_SOURCE_DEFERRED, download=False)
            ks.append(pt.last_shading_rate_ms)
        rates = pt.ShadingRate(frame, dvel, source=capi.LIT_SOURCE_DEFERRED)
        out["classifier"] = dict(kernel_ms=float(np.median(ks[2:])))

        flat = torch.full((H, W, 4), 0.5, device="cuda")
        cases = {"all 1x1": (dict(color=flat), capi.IdkPtShadingRateSettings(0, 0.2, 0.04), np.zeros((H, W, 2), np.float32)),
                 "classifier": None,
                 "all 4x4": (dict(color=flat * 0.0), capi.IdkPtShadingRateSettings(0, 0.2, 0.04), np.zeros((H, W, 2), np.float32))}
        for name, case in cases.items():
            # set the rate image: a flat lit image gives rate 0 everywhere (cov 0), a black one 4 (mean <= 0.001); "classifier"
            # is this frame's own classification of the per-pixel image
            lighting(False)
            if case is None:
                got = pt.ShadingRate(frame, dvel, source=capi.LIT_SOURCE_DEFERRED)
            else:
                kw, sst, v = case
                got = pt.ShadingRate(frame, torch.from_numpy(v).cuda(), sst, **kw)
            share = {f"{capi.VRS_PALETTE[r][0]}x{capi.VRS_PALETTE[r][1]}": float(np.mean(got == r)) for r in range(5)}
            frags = sum(float(np.sum(got == r)) * 256 / (capi.VRS_PALETTE[r][0] * capi.VRS_PALETTE[r][1]) for r in range(5))
            per_pixel, coarse = [], []
            for _ in range(a.reps + 2):
                per_pixel.append(lighting(False))
                coarse.append(lighting(True))
            kp, kc = float(np.median(per_pixel[2:])), float(np.median(coarse[2:]))
            out[f"deferred pcf ssao, {name}"] = dict(k_deferred_lighting_ms=kp, coarse_ms=kc, coarse_over_per_pixel=kc / kp,
                                                      tile_share=share, invocations_over_pixels=frags / (W * H))
        out["classifier rates"] = {f"{capi.VRS_PALETTE[r][0]}x{capi.VRS_PALETTE[r][1]}": float(np.mean(rates == r)) for r in range(5)}
    print("VRS", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
