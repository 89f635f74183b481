"""Timing of the light spheres and the skybox per pixel against the same draws under the shading-rate image (DESIGN 8f.1i) on
the bench atrium (--tris 262144 requested) from the bench camera at 1920x1080.

    python scripts/time_lights_skybox_vrs.py [--tris 262144] [--reps 15] [--out FILE]

For the three startup lights and for 256 lights spread through the view, and for three rate images (all 1x1, all 4x4, and the
classifier's image of a frame panning 3 degrees to the side at 60 fps, with the engine's settings), it reports the kernel time
of idkpt_lights_and_skybox and of idkpt_lights_and_skybox_vrs (CUDA events). Each repetition renders the G-buffer and the
deferred image afresh, so every timed call draws the lights and the sky into an untouched frame, and the two calls alternate,
per-pixel first in even repetitions and VRS first in odd ones; the table holds the median of --reps repetitions after two
warm-ups. The card name and power limit are read in the same run.
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, scenes  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from time_lights_skybox import light_sets  # noqa: E402
from timing_lib import JITTER, card, write_out  # noqa: E402

FIVE = capi.IdkPtShadingRateSettings(0, 1.0, 0.0)   # SpeedFactor 1, LumVarianceFactor 0: the rate follows the speed alone


def panning_frame(cam, w, h):
    """The bench camera's frame whose previous view looked 3 degrees to the side, 1/60 s earlier."""
    frame = copy.deepcopy(scenes.camera_frame(cam, w, h))
    vd = np.asarray(cam["view_dir"], np.float64)
    c, s = np.cos(np.deg2rad(3.0)), np.sin(np.deg2rad(3.0))
    prev = scenes.make_per_frame_data(cam["position"], (c * vd[0] + s * vd[2], vd[1], -s * vd[0] + c * vd[2]), w, h,
                                      cam.get("fov_y_deg", 102.0))
    frame["PrevView"], frame["PrevProjView"] = prev["View"], prev["ProjView"]
    frame["DeltaRenderTime"] = 1.0 / 60.0
    return frame


def render(pt, frame, w, h):
    pt.GBuffer(frame, w, h, jitter=JITTER, download=False)
    g = pt.GBufferDevicePtrs(tensors=True)
    pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), jitter=JITTER, download=False)
    return g


def make_rates(pt, kind, frame, w, h, velocity):
    if kind == "classified":
        return pt.ShadingRate(frame, velocity, source=capi.LIT_SOURCE_DEFERRED)
    v = np.zeros((h, w, 2), np.float32)
    c = np.full((h, w, 4), 0.5, np.float32)
    if kind == "4x4":
        v[..., 0] = 1000.0
        c[..., :3] += np.random.default_rng(0).random((h, w, 3)).astype(np.float32) * 0.1
    return pt.ShadingRate(frame, v, FIVE, color=c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam = scenes.atrium(a.tris)
    sets = light_sets(scene, cam)
    w, h = 1920, 1080
    frame = panning_frame(cam, w, h)
    result = dict(card=card(), tris=int(len(scene.blas_triangles)), width=w, height=h, reps=a.reps, runs=[])
    for name in ("startup", "256"):
        s = sets[name]
        with PathTracer(16, 16) as pt:
            pt.SetScene(s)
            pt.SetSky((0.6, 0.7, 0.9))
            for kind in ("1x1", "4x4", "classified"):
                g = render(pt, frame, w, h)
                rates = make_rates(pt, kind, frame, w, h, g[5])
                times = {False: [], True: []}
                for rep in range(a.reps + 2):
                    for vrs in ((False, True) if rep % 2 == 0 else (True, False)):
                        render(pt, frame, w, h)
                        pt.LightsAndSkybox(frame, jitter=JITTER, download=False, vrs=vrs)
                        times[vrs].append(pt.last_lights_and_skybox_ms)
                per_pixel, coarse = (float(np.median(times[v][2:])) for v in (False, True))
                run = dict(lights=name, light_count=int(len(s.lights)), rates=kind,
                           rate_histogram=[int((rates == r).sum()) for r in range(5)],
                           k_lights_skybox_ms=round(per_pixel, 4), k_lights_skybox_vrs_ms=round(coarse, 4),
                           vrs_over_per_pixel=round(coarse / per_pixel, 3))
                result["runs"].append(run)
                print(json.dumps(run), flush=True)
    print(json.dumps(dict(card=result["card"])), flush=True)
    write_out(a.out, result)


if __name__ == "__main__":
    main()
