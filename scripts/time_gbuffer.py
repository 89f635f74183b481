"""Timing of the G-buffer pass (DESIGN 8f.1g) on the bench atrium (--tris 262144 requested) from the bench camera, and of the
whole device raster frame on its images.

    python scripts/time_gbuffer.py [--tris 262144] [--reps 20] [--out FILE]

For 1920x1080 and 1152x648 (render scale 0.6) it reports k_gbuffer's kernel time (CUDA events, median of --reps after two
warm-up calls) and rate in Grays/s, and idkpt_trace_rays' kernel time on the same primary rays (the difference is what the
depth-test rules and the attribute work cost). Then the raster frame with every input a device pointer and nothing
downloaded: idkpt_gbuffer, idkpt_ssao, idkpt_deferred_lighting (Pcf + IsSSAO, the reference's three startup lights shadowed at
512^2), idkpt_ssr and idkpt_taa_resolve, each call's kernel time (median) and the sum. The card name and power limit are read
in the same run.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, gpu_types as gt, scenes  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import JITTER, card, median_ms, shadowed_atrium, write_out  # noqa: E402


def primary_rays(frame, w, h):
    """The rays k_gbuffer casts (rule 1, float64 here: the timing does not depend on their last bits)."""
    f = frame[0]
    ipv = np.asarray(f["InvProjView"], np.float64).reshape(4, 4).T
    eye = np.asarray(f["ViewPos"], np.float64)
    ys, xs = np.mgrid[0:h, 0:w]
    ndc = np.stack([(xs + 0.5) / w * 2 - 1 - JITTER[0], (ys + 0.5) / h * 2 - 1 - JITTER[1], np.ones((h, w)), np.ones((h, w))], -1)
    p = ndc.reshape(-1, 4) @ ipv.T
    d = p[:, :3] / p[:, 3:] - eye
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = np.zeros(w * h, gt.IdkPtRay)
    r["Origin"], r["Direction"], r["TMax"] = eye, d, 3.4028235e+38
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam, shadows = shadowed_atrium(a.tris)

    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), reps=a.reps)
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetPointShadows(shadows, [512] * len(scenes.STARTUP_LIGHTS))
        pt.RenderPointShadows()
        for W, H in ((1920, 1080), (1152, 648)):
            frame = scenes.camera_frame(cam, W, H)
            rays = primary_rays(frame, W, H)

            def gbuffer():
                pt.GBuffer(frame, W, H, jitter=JITTER, download=False)
                return pt.last_gbuffer_ms
            kg = median_ms(gbuffer, a.reps)
            kt = median_ms(lambda: pt.TraceRays(rays)[1], a.reps)
            row = dict(k_gbuffer_ms=kg, grays_per_s=W * H / (kg * 1e-3) / 1e9, trace_rays_ms=kt, gbuffer_over_trace_rays=kg / kt)

            pt.GBuffer(frame, W, H, jitter=JITTER, download=False)
            d, n, al, mr, e, v = pt.GBufferDevicePtrs(tensors=True)
            st = capi.IdkPtDeferredSettings(capi.SHADOW_MODE_PCF, 1, 0, 0)

            def ssao():
                pt.Ssao(frame, d, n, download=False)
                return pt.last_ssao_ms

            def lighting():
                pt.DeferredLighting(frame, d, n, al, mr, e, settings=st, jitter=JITTER, download=False)
                return pt.last_deferred_ms

            def ssr():
                pt.Ssr(frame, d, n, al, mr, source=capi.LIT_SOURCE_DEFERRED, download=False)
                return pt.last_ssr_ms

            def taa():
                pt.TaaResolve(d, v, W, H, source=capi.LIT_SOURCE_MERGED, download=False)
                return pt.last_taa_ms
            frame_ms = dict(idkpt_gbuffer=kg, idkpt_ssao=median_ms(ssao, a.reps), idkpt_deferred_lighting=median_ms(lighting, a.reps),
                            idkpt_ssr=median_ms(ssr, a.reps), idkpt_taa_resolve=median_ms(taa, a.reps))
            frame_ms["sum"] = float(sum(frame_ms.values()))
            row["raster_frame_kernel_ms"] = frame_ms
            out[f"{W}x{H}"] = row
    print("GBUFFER", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
