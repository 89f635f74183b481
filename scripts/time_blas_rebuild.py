"""Timing of refit against rebuild for a skinned, refittable BLAS under growing articulated motion: idkpt_blas_refit against
idkpt_blas_rebuild, the global SAH of each tree (idkpt_blas_sah), and what each tree costs the path tracer.

    python scripts/time_blas_rebuild.py [--tris 4096 32768 262144] [--steps 4] [--reps 5] [--out FILE]

Each mesh is a tessellated strip of 8 segments along x, one joint per segment; joint k turns its segment by k * angle about
z around the segment's start, so the strip curls up more with every step (the skinning_setup pattern with growing angles).
Two path tracers hold the same scene: one refits the rest-pose tree every step, the other rebuilds it every step. Per size
and step it prints: the call's device time and a host clock around the synchronous call (median of --reps after two
warm-ups), the SAH after the refit and after the rebuild, and node-pair fetches per ray (CollectStats) and ms per 1080p
sample of Compute through each tree. The card's name and power limit are read in the same run.
"""
import argparse
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, host, scenes  # noqa: E402
from idkengine_b200 import gpu_types as gt  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402

SEGMENTS = 8
W, H = 1920, 1080


def strip(tris):
    """A refittable grid 8 long in x, 1 wide in z, with about `tris` triangles; its joints and unskinned vertices."""
    nv = max(1, int(np.sqrt(tris / 2 / 8)))
    nu = max(SEGMENTS, tris // (2 * nv))
    pos, idx = scenes.grid([0.0, 0.5, -0.5], [8.0, 0, 0], [0, 0, 1.0], nu, nv)
    scene = host.Scene().add(host.Model(pos, idx, refittable=True, name="strip"), threads=os.cpu_count())
    scene.add_light((4.0, 4.0, 2.0), (40.0, 38.0, 30.0), 0.3)
    scene.build_tlas()
    n = len(scene.positions)
    u = np.zeros(n, gt.GpuUnskinnedVertex)
    seg = np.clip((scene.positions["x"] / (8.0 / SEGMENTS)).astype(np.int64), 0, SEGMENTS - 1)
    u["JointIndices"][:, 0] = seg
    u["JointWeights"][:, 0] = 1.0
    for k, c in enumerate("xyz"):
        u["Position"][:, k] = scene.positions[c]
    u["Normal"] = scene.vertices["Normal"]
    u["Tangent"] = scene.vertices["Tangent"]
    cmd = np.zeros(1, gt.IdkPtSkinningCmd)
    cmd["VertexCount"] = n
    return scene, u, cmd


def joints(angle):
    """Joint k: the rotation by k * angle about z around x = k (the segment's start), chained like an arm's bones."""
    jm = np.zeros((SEGMENTS, 3, 4), np.float32)
    m = np.eye(4)
    L = 8.0 / SEGMENTS
    for k in range(SEGMENTS):
        c, s = np.cos(angle), np.sin(angle)
        rot = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])
        to, back = np.eye(4), np.eye(4)
        to[0, 3], back[0, 3] = -k * L, k * L
        m = m @ back @ rot @ to if k else back @ rot @ to
        jm[k] = m[:3].astype(np.float32)
    return jm


def call_ms(fn, reps):
    """(median device ms, median host ms) of a synchronous call over reps after two warm-ups."""
    dev, wall = [], []
    for _ in range(reps + 2):
        t0 = time.perf_counter()
        dev.append(fn())
        wall.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(dev[2:])), float(np.median(wall[2:]))


def render(pt):
    pt.ResetAccumulation()
    pt.Compute()                                   # warm-up
    fetch, ms = [], []
    for _ in range(3):
        st = pt.Compute()
        fetch.append(st.NodePairFetches / max(1, st.Rays))
        ms.append(st.TotalMs)
    return float(np.median(fetch)), float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, nargs="+", default=[4096, 32768, 262144])
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    result = dict(card=card(), sizes=[])
    print(result["card"])
    cam = dict(position=(4.0, 3.0, 9.0), view_dir=(0.0, -0.25, -1.0), fov_y_deg=60.0)
    frame = scenes.camera_frame(cam, W, H)
    s = capi.default_settings()
    s.CollectStats = 1
    for tris in a.tris:
        scene, u, cmd = strip(tris)
        size = dict(triangles=int(len(scene.blas_triangles)), steps=[])
        with PathTracer(W, H, s) as refit, PathTracer(W, H, s) as rebuild:
            for pt in (refit, rebuild):
                pt.SetScene(scene)
                pt.SetSky((0.6, 0.7, 0.9))
                pt.SetFrame(frame)
                pt.SetSkinningData(u)
            for step in range(a.steps):
                jm = joints(0.25 * step)
                row = dict(angle=0.25 * step)
                for pt in (refit, rebuild):
                    pt.SkinVertices(jm, cmd)
                row["refit_ms"], row["refit_wall_ms"] = call_ms(lambda: refit.BlasRefit(0, 1), a.reps)
                row["rebuild_ms"], row["rebuild_wall_ms"] = call_ms(lambda: rebuild.RebuildBlases(0, 1), a.reps)
                for pt in (refit, rebuild):
                    pt.TlasBuild()
                row["sah_refit"] = float(refit.BlasSah(0)[0])
                row["sah_rebuild"] = float(rebuild.BlasSah(0)[0])
                row["fetches_per_ray_refit"], row["sample_ms_refit"] = render(refit)
                row["fetches_per_ray_rebuild"], row["sample_ms_rebuild"] = render(rebuild)
                size["steps"].append(row)
                print(tris, {k: round(v, 4) for k, v in row.items()})
        result["sizes"].append(size)
    write_out(a.out, result)


if __name__ == "__main__":
    main()
