"""Timing of the transparency pass (DESIGN 8f.1h) on the bench atrium (--tris 262144 requested) from the bench camera, and of
the whole device raster frame with the pass inserted.

    python scripts/time_transparency.py [--tris 262144] [--reps 20] [--out FILE]

For 1920x1080 and 1152x648 (render scale 0.6) it reports k_transparency's kernel time (CUDA events, median of --reps after two
warm-up calls) for ShadowMode Pcf with IsVXGI off and on (a 256^3 grid voxelised once, the engine's cone settings), next to
k_gbuffer's on the same rays. Then the raster frame with every input a device pointer and nothing downloaded: idkpt_gbuffer,
idkpt_ssao, idkpt_deferred_lighting (Pcf + IsSSAO, the reference's three startup lights shadowed at 512^2),
idkpt_transparency (Pcf, DEFERRED), idkpt_ssr and idkpt_taa_resolve, each call's kernel time (median) and the sum. The
fraction of pixels with at least one layer and the mean layer count come from the CPU oracle's walk at 480x270 (the same
camera and rule; the device keeps no per-pixel count). The card name and power limit are read in the same run.
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import JITTER, card, median_ms, shadowed_atrium, write_out  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam, shadows = shadowed_atrium(a.tris)
    blended = int((scene.materials["AlphaCutoff"] == 2.0).sum())

    out = dict(card=card(), triangles=int(len(scene.blas_triangles)), blended_materials=blended, reps=a.reps)
    unshadowed = copy.deepcopy(scene)
    unshadowed.lights["PointShadowIndex"][:] = -1
    lo = np.min([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1) - 0.5
    hi = np.max([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1) + 0.5
    with PathTracer(64, 64) as pt, vxgi.Voxelizer(256, tuple(lo), tuple(hi)) as vx:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetPointShadows(shadows, [512] * len(scenes.STARTUP_LIGHTS))
        pt.RenderPointShadows()
        vx.SetScene(unshadowed)
        vx.Render()
        cone = vxgi.default_cone_settings()
        for W, H in ((1920, 1080), (1152, 648)):
            frame = scenes.camera_frame(cam, W, H)

            def gbuffer():
                pt.GBuffer(frame, W, H, jitter=JITTER, download=False)
                return pt.last_gbuffer_ms
            kg = median_ms(gbuffer, a.reps)
            d, n, al, mr, e, v = pt.GBufferDevicePtrs(tensors=True)
            st = capi.IdkPtDeferredSettings(capi.SHADOW_MODE_PCF, 1, 0, 0)
            pt.Ssao(frame, d, n, download=False)
            pt.DeferredLighting(frame, d, n, al, mr, e, settings=st, jitter=JITTER, download=False)

            def transparency(is_vxgi):
                def run():
                    pt.Transparency(frame, d, settings=capi.IdkPtTransparencySettings(capi.SHADOW_MODE_PCF, is_vxgi), jitter=JITTER,
                                    source=capi.LIT_SOURCE_DEFERRED, voxelizer=vx if is_vxgi else None, cone=cone, download=False)
                    return pt.last_transparency_ms
                return run
            kt0 = median_ms(transparency(0), a.reps)
            kt1 = median_ms(transparency(1), a.reps)
            row = dict(k_gbuffer_ms=kg, k_transparency_pcf_ms=kt0, k_transparency_pcf_vxgi_ms=kt1, transparency_over_gbuffer=kt0 / kg)

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
                            idkpt_transparency=kt0, idkpt_ssr=median_ms(ssr, a.reps), idkpt_taa_resolve=median_ms(taa, a.reps))
            frame_ms["sum"] = float(sum(frame_ms.values()))
            row["raster_frame_kernel_ms"] = frame_ms
            out[f"{W}x{H}"] = row
        # coverage: the oracle's walk at 480x270
        import transparency_oracle as to
        W, H = 480, 270
        frame = scenes.camera_frame(cam, W, H)
        depth = pt.GBuffer(frame, W, H, jitter=JITTER)[0]
        _, _, counts = to.transparency(scene, frame, depth, np.zeros((H, W, 4), np.float32), jitter=JITTER)
        out["coverage_480x270"] = dict(pixels_with_a_layer=float((counts > 0).mean()), mean_layers=float(counts.mean()),
                                       mean_layers_where_any=float(counts[counts > 0].mean()) if (counts > 0).any() else 0.0,
                                       max_layers=int(counts.max()))
    print("TRANSPARENCY", json.dumps(out))
    write_out(a.out, out)


if __name__ == "__main__":
    main()
