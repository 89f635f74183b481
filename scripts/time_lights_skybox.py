"""Timing of the light spheres and the skybox (DESIGN 8f.1i) on the bench atrium (--tris 262144 requested) from the bench camera.

    python scripts/time_lights_skybox.py [--tris 262144] [--reps 10] [--out FILE]

For 1920x1080 and 1152x648 (render scale 0.6) it reports k_lights_skybox's kernel time (CUDA events, median of --reps after two
warm-up calls; the call is idempotent, so every repetition does the same work) with the reference's three startup lights,
with those and a radius-0.3 light 0.5 in front of the camera (the engine's add-light click: the sphere covers much of the
screen and every covered pixel tests its 264 triangles), and with 256 lights spread through the view. k_gbuffer's kernel time
on the same frame is measured in the same run for scale, and the share of pixels each draw wrote comes from the CPU oracle at
480x270 (without the 256-light set). The card name and power limit are read in the same run.
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
from timing_lib import JITTER, card, median_ms, write_out  # noqa: E402


def light_sets(scene, cam):
    eye = np.asarray(cam["position"], np.float64)
    vd = np.asarray(cam["view_dir"], np.float64)
    vd /= np.linalg.norm(vd)
    near = (tuple(eye + vd * 0.5), (61.0, 42.0, 55.0), 0.3)
    rng = np.random.default_rng(5)
    many = [near] + [(tuple(eye + vd * rng.uniform(0.5, 12.0) + rng.uniform(-3.0, 3.0, 3)), tuple(rng.uniform(0.5, 60.0, 3)),
                      float(rng.uniform(0.02, 0.6))) for _ in range(255)]
    out = {}
    for name, lights in (("startup", scenes.STARTUP_LIGHTS), ("startup_near", scenes.STARTUP_LIGHTS + [near]), ("256", many)):
        s = copy.deepcopy(scene)
        s.lights = s.lights[:0]
        for p, c, r in lights:
            s.add_light(p, c, r)
        out[name] = s
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    scene, cam = scenes.atrium(a.tris)
    sets = light_sets(scene, cam)
    result = dict(card=card(), tris=int(len(scene.blas_triangles)), reps=a.reps, runs=[])
    for w, h in ((1920, 1080), (1152, 648)):
        frame = scenes.camera_frame(cam, w, h)
        for name, s in sets.items():
            with PathTracer(16, 16) as pt:
                pt.SetScene(s)
                pt.SetSky((0.6, 0.7, 0.9))

                def gbuffer():
                    pt.GBuffer(frame, w, h, jitter=JITTER, download=False)
                    return pt.last_gbuffer_ms
                gb_ms = median_ms(gbuffer, a.reps)
                g = pt.GBufferDevicePtrs(tensors=True)
                pt.DeferredLighting(frame, *g[:5], settings=capi.IdkPtDeferredSettings(0, 0, 0, 0), jitter=JITTER, download=False)

                def lights():
                    pt.LightsAndSkybox(frame, jitter=JITTER, download=False)
                    return pt.last_lights_and_skybox_ms
                ms = median_ms(lights, a.reps)
            run = dict(width=w, height=h, lights=name, light_count=int(len(s.lights)), k_lights_skybox_ms=round(ms, 4),
                       k_gbuffer_ms=round(gb_ms, 4))
            result["runs"].append(run)
            print(json.dumps(run), flush=True)

    # coverage at 480x270 from the oracle (the device keeps no per-pixel record of which draw wrote a pixel)
    import gbuffer_oracle as go
    import lights_skybox_oracle as lo
    w, h = 480, 270
    frame = scenes.camera_frame(cam, w, h)
    g = go.gbuffer(scene, frame, w, h, jitter=JITTER)
    cov = {}
    for name in ("startup", "startup_near"):   # 256 lights would take the brute-force oracle minutes
        s = sets[name]
        _, _, winner = lo.lights_and_skybox(s, frame, g, np.zeros((h, w, 4), np.float32), jitter=JITTER)
        cov[name] = dict(light=round(float((winner >= 0).mean()), 4), sky=round(float((winner == lo.SKY).mean()), 4))
    result["coverage_480x270"] = cov
    print(json.dumps(dict(card=result["card"], coverage_480x270=cov)), flush=True)
    write_out(a.out, result)


if __name__ == "__main__":
    main()
