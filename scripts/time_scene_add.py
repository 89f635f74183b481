"""Timing of adding models to a loaded scene (idkpt_add_models, DESIGN 8f.5 "Adding models").

    python scripts/time_scene_add.py [--reps 3] [--bases atrium,config3] [--models 1k,8k,262k,textured] [--out FILE]

Bases: the 262 k-triangle atrium and the 9 M-triangle configuration scene (scenes.atrium(9_000_000), BASELINE config 3),
both with a TLAS. Models, seeded: soups of 1 k, 8 k and 262 k triangles (pre-split), and the textured room with its eight
textures. Each round times, on a context holding the base scene:
  add      PathTracer.AddModels(model): the call's device time (kernel_ms) and the host clock around it;
  reload   what a runtime load costs without it: host.Scene.add(model) onto the base with the device batch builder
           (PathTracer.BuildBlases), then PathTracer.SetScene of the whole scene; the batch's device time and the host
           clock around both calls.
Both end with the same scene: the device arrays after each are compared byte for byte. The base is set again, untimed,
before every round. Medians over --reps rounds after one warm-up of each; the card name and power limit are read in the
same run.
"""
import argparse
import copy
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, host, scenes  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402


def soup(n, seed):
    """n triangles in small clusters inside the atrium's box, as one model."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-6.0, 6.0, (n, 1, 3)) + np.array([0.0, 3.0, 0.0])
    p = (c + rng.normal(0.0, 0.05, (n, 3, 3))).reshape(-1, 3).astype(np.float32)
    return host.Model(p, np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), name=f"soup{n}")


def textured():
    """The textured room, shrunk into the scene, with its textures as the call's own table (handles unchanged)."""
    got = []
    orig = scenes.Scene

    class Recording(host.Scene):
        def add(self, *models, **kw):
            got.extend(models)
            return super().add(*models, **kw)

    scenes.Scene = Recording
    try:
        room, _ = scenes.textured_room(threads=os.cpu_count())
    finally:
        scenes.Scene = orig
    m = copy.copy(got[0])
    m.model_matrix = host.trs_matrix(0.5, 20.0, (1.0, 0.0, 1.0))
    return m, room.textures


def base_scene(name, pt):
    """The base with its BLASes built on the device (the 9 M scene would take minutes on the host)."""
    got = []
    orig = scenes.Scene

    class Recording(host.Scene):
        def add(self, *models, **kw):
            got.extend(models)
            return self

    scenes.Scene = Recording
    try:
        scenes.atrium(target_tris=262144 if name == "atrium" else 9_000_000)
    finally:
        scenes.Scene = orig
    scene = host.Scene().add(*got, blas_batch_builder=pt.BuildBlases)
    scene.add_light((0.0, 3.0, 0.5), (30.0, 28.0, 20.0), 0.3)
    scene.build_tlas()
    return scene


def reload(pt, base, model, textures):
    s = copy.copy(base)
    s.build_info = list(base.build_info)
    s.add(with_handles(model, len(base.textures)), blas_batch_builder=pt.BuildBlases)
    s.textures = base.textures + list(textures)
    s.build_tlas()
    pt.SetScene(s)
    return s


def with_handles(model, offset):
    m = copy.copy(model)
    m.materials = model.materials.copy()
    for f in host.TEXTURE_SLOTS:
        h = m.materials[f]
        m.materials[f] = np.where(h > 0, h + np.uint64(offset), np.uint64(0))
    return m


def device_arrays(pt, scene):
    last = scene.blas_descs[-1]
    out = [pt.ReadRange(capi.IDKPT_ARRAY_BLAS_DESCS, 0, len(scene.blas_descs)),
           pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, int(last["NodeOffset"] + last["NodeCount"])),
           pt.ReadRange(capi.IDKPT_ARRAY_BLAS_TRIANGLES, 0, int(last["TriangleOffset"] + last["TriangleCount"])),
           pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * len(scene.blas_instances) - 1),
           pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))]
    return b"".join(a.tobytes() for a in out)


def med(v):
    return round(float(np.median(v)), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--bases", default="atrium,config3")
    ap.add_argument("--models", default="1k,8k,262k,textured")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    result = dict(card=card(), reps=a.reps, runs=[])
    tex_model, tex_table = textured()
    models = {"1k": (soup(1024, 1), []), "8k": (soup(8192, 2), []), "262k": (soup(262144, 3), []), "textured": (tex_model, tex_table)}
    with PathTracer(64, 48) as pt:
        for bname in a.bases.split(","):
            base = base_scene(bname, pt)
            for mname in a.models.split(","):
                model, textures = models[mname]
                want = reload(pt, base, model, textures)   # warm-up of both paths, which end with the same device arrays
                reloaded = device_arrays(pt, want)
                pt.SetScene(base)
                pt.AddModels(model, textures=textures)
                equal = device_arrays(pt, want) == reloaded
                add_ms, add_ev, old_ms, old_ev = [], [], [], []
                for _ in range(a.reps):
                    pt.SetScene(base)
                    t0 = time.perf_counter()
                    add_ev.append(pt.AddModels(model, textures=textures))
                    add_ms.append((time.perf_counter() - t0) * 1e3)
                    t0 = time.perf_counter()
                    reload(pt, base, model, textures)
                    old_ms.append((time.perf_counter() - t0) * 1e3)
                    old_ev.append(pt.last_blas_build_ms)
                run = dict(base=bname, base_triangles=int(base.source_triangle_count), model=mname,
                           model_triangles=int(len(model.indices)), textures=len(textures),
                           add_call_ms=med(add_ms), add_device_ms=med(add_ev),
                           reload_call_ms=med(old_ms), reload_build_device_ms=med(old_ev),
                           speedup=round(float(np.median(old_ms) / np.median(add_ms)), 1), same_arrays=equal)
                result["runs"].append(run)
                print(json.dumps(run), flush=True)
    print(json.dumps(result))
    write_out(a.out, result)


if __name__ == "__main__":
    main()
