"""Regenerate tests/golden/bvh_build_digests.json from the host BVH builds (python tests/golden/make_bvh_digests.py).

The device builds are checked against the host builds (tests/test_blas_build_gpu.py, tests/test_dynamic.py); these digests
check the host builds against their own past output, so a change to the builders' shared arithmetic that moves a single
bit fails on a CPU. A BLAS digest covers the node bytes, the triangle bytes, the required stack size, the fragment count and
the SAH's float64 bits; a TLAS digest covers the node bytes."""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from idkengine_b200 import host, scenes  # noqa: E402
from test_blas_build_gpu import SMALL_SCENES, mesh, recorded  # noqa: E402

OUT = os.path.join(HERE, "bvh_build_digests.json")


def blas_digest(b):
    h = hashlib.sha256()
    h.update(b["nodes"].tobytes())
    h.update(b["triangles"].tobytes())
    h.update(np.int32(b["required_stack_size"]).tobytes())
    h.update(np.int32(b["fragment_count"]).tobytes())
    h.update(np.float64(b["sah"]).tobytes())
    return h.hexdigest()


def build(positions, triangles, presplit=True, threads=1, **settings):
    s = host.default_build_settings()
    for k, v in settings.items():
        setattr(s, k, v)
    return blas_digest(host.build_blas(positions, triangles, presplit=presplit, threads=threads, settings=s))


def small_scene_cases():
    """Every BLAS of the small test scenes, built as the scene builds it and with pre-splitting the other way round."""
    out = {}
    for name in sorted(SMALL_SCENES):
        for k, (positions, triangles, presplit, _) in enumerate(recorded(SMALL_SCENES[name])):
            out[f"{name}/{k}"] = lambda p=positions, t=triangles, s=presplit: build(p, t, presplit=s)
            out[f"{name}/{k}/presplit={not presplit}"] = lambda p=positions, t=triangles, s=presplit: build(p, t, presplit=not s)
    return out


def atrium_cases():
    """atrium(40000): 1 and 4 threads (the task pool and the wide split), pre-splitting off, leaf and stop settings, and a
    stack optimisation that collapses several levels."""
    positions, triangles, _, _ = recorded(scenes.atrium, target_tris=40000)[0]
    cases = {
        "threads=1": dict(threads=1),
        "threads=4": dict(threads=4),
        "presplit=False": dict(presplit=False, threads=4),
        "MaxLeafTriangleCount=1": dict(MaxLeafTriangleCount=1),
        "MaxLeafTriangleCount=8": dict(MaxLeafTriangleCount=8),
        "StopSplittingThreshold=4": dict(StopSplittingThreshold=4),
        "StackOptThreshold=1": dict(StackOptThreshold=1, StackOptSahIncreaseAcceptance=0.05),
        "StackOptThreshold=1/presplit=False": dict(presplit=False, StackOptThreshold=1, StackOptSahIncreaseAcceptance=0.05),
    }
    return {f"atrium_40k/{k}": (lambda kw=kw: build(positions, triangles, **kw)) for k, kw in cases.items()}


def root_leaf_case():
    """A refittable BLAS whose root stays a leaf: two copies of the root, each listing all triangles."""
    pos, tris = mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0], [3, 0, 1]], [[0, 1, 2], [1, 3, 2]])
    return {"root_leaf/presplit=False": lambda: build(pos, tris, presplit=False, StopSplittingThreshold=2)}


def forest():
    """40 scaled, turned copies of a small sphere at seeded positions."""
    rng = np.random.default_rng(2)
    pos, idx = scenes.uv_sphere([0, 0, 0], 0.5, 8, 12)
    sc = host.Scene()
    for k in range(40):
        t = (rng.uniform(-6, 6), rng.uniform(0, 3), rng.uniform(-6, 6))
        sc.add(host.Model(pos, idx, model_matrix=host.trs_matrix(0.5 + 0.02 * k, 7.0 * k, t), name=f"s{k}"), threads=1)
    return sc


def tlas_cases():
    def tlas(make, radius):
        sc = make()
        sc.build_tlas(search_radius=radius)
        return hashlib.sha256(sc.tlas_nodes.tobytes()).hexdigest()
    out = {}
    for radius in (15, 2):
        out[f"tlas/multi_blas/radius={radius}"] = lambda r=radius: tlas(lambda: scenes.multi_blas(threads=1)[0], r)
        out[f"tlas/forest_40/radius={radius}"] = lambda r=radius: tlas(forest, r)
    return out


def cases():
    """name -> function returning the digest."""
    return {**small_scene_cases(), **atrium_cases(), **root_leaf_case(), **tlas_cases()}


if __name__ == "__main__":
    out = {name: f() for name, f in cases().items()}
    with open(OUT, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(f"{len(out)} digests written to {OUT}")
