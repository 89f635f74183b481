"""What the timing scripts share: the card a number was measured on, the median timer, the --out writer and the shadowed
bench atrium."""
import json
import os
import subprocess

import numpy as np

from idkengine_b200 import scenes

JITTER = (0.0003, -0.0002)


def card():
    """Name, power limit and maximum SM clock of GPU 0: a timing means nothing without them."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def median_ms(fn, reps):
    """Median of fn()'s returned milliseconds over reps calls, after two warm-up calls."""
    t = [fn() for _ in range(reps + 2)]
    return float(np.median(t[2:]))


def write_out(path, result):
    """The --out file: result as JSON at path (its directory created), nothing when path is empty."""
    if path:
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        with open(path, "w") as f:
            json.dump(result, f, indent=1)


def shadowed_atrium(tris):
    """(scene, camera, shadows): bench.py's atrium lit by the engine's startup lights only, each with a point shadow whose near
    plane is the light's radius and far plane 60."""
    scene, cam = scenes.atrium(tris)
    scene.lights = scene.lights[:0]
    for light in scenes.STARTUP_LIGHTS:
        scene.add_light(*light)
    scene.lights["PointShadowIndex"][:] = np.arange(len(scenes.STARTUP_LIGHTS))
    return scene, cam, scenes.point_shadows([(p, r, 60.0, i) for i, (p, _, r) in enumerate(scenes.STARTUP_LIGHTS)])
