"""Timing of scene-versus-moving-sphere collision on the device (idkpt_collide_spheres and idkpt_collide_spheres_tlas,
DESIGN 8f "Collision").

    python scripts/time_collision.py [--reps 5] [--counts 1,257,65536] [--scenes atrium,instances] [--modes linear,tlas] [--out FILE]

Scenes: the 262 k-triangle atrium (one instance; its TLAS is that instance's leaf) and the 262 144-instance grid of the TLAS
timings (instance_grid(2)'s BLASes, scale 0.4, 1.25 apart) with its TLAS built on the device. Spheres, seeded: a start
anywhere in the scene's bounds, a destination up to 0.5 away, radius 0.02 .. 0.5. For each scene, mode, sphere count and
preset (the lights' 1 test step and 8 recursive steps with Plane.Reflect, the camera's 3 and 12 with Plane.Project):
  device   PathTracer.CollideSpheres: the kernel's device time (kernel_ms) and the host clock around the call (upload, kernel,
           download), median over --reps calls after two warm-ups. Mode `linear` visits every instance in index order
           (CpuUseTlas == false), mode `tlas` walks the TLAS (CpuUseTlas == true); a scene without a TLAS has no tlas rows.
Beside each scene: the bytes of the read-backs the call makes unnecessary, from the scene's shapes: the vertex positions, the
BLAS nodes and triangles (the host BVH that BVH.Intersect walks) and the mesh transforms. The card name and power limit are
read in the same run.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import gpu_types as gt, scenes  # noqa: E402
from idkengine_b200.pathtracer import CAMERA_COLLISION, LIGHT_COLLISION, PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402

PRESETS = {"lights": LIGHT_COLLISION, "camera": CAMERA_COLLISION}


def make_scene(name):
    if name == "atrium":
        sc, _ = scenes.atrium(262144, threads=os.cpu_count())
        return sc.build_tlas()
    return scenes._instanced(scenes._grid_matrices(262144))


def world_bounds(sc):
    p = np.stack([sc.positions["x"], sc.positions["y"], sc.positions["z"]], 1)
    if len(sc.blas_instances) == 1:
        m = sc.mesh_transforms["ModelMatrix"][0].astype(np.float64)
        p = p @ m[:, :3].T + m[:, 3]
        return p.min(0), p.max(0)
    t = sc.mesh_transforms["ModelMatrix"][:, :, 3]
    return t.min(0) - 1.0, t.max(0) + 1.0


def spheres(sc, n, seed):
    lo, hi = world_bounds(sc)
    rng = np.random.default_rng(seed)
    s = np.zeros(n, gt.IdkPtMovingSphere)
    s["PrevPosition"] = rng.uniform(lo, hi, (n, 3))
    s["Position"] = s["PrevPosition"] + rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32)
    s["Velocity"] = rng.uniform(-3.0, 3.0, (n, 3))
    s["Radius"] = rng.uniform(0.02, 0.5, n)
    return s


def readback_bytes(sc):
    return dict(positions=len(sc.positions) * 12, blas_nodes=len(sc.blas_nodes) * 32, blas_triangles=len(sc.blas_triangles) * 16,
                mesh_transforms=len(sc.mesh_transforms) * 144)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--counts", default="1,257,65536")
    ap.add_argument("--scenes", default="atrium,instances")
    ap.add_argument("--modes", default="linear,tlas")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['max_sm_clock']}")
    result = dict(card=dev, scenes={})
    for name in a.scenes.split(","):
        sc = make_scene(name)
        rb = readback_bytes(sc)
        print(f"\n{name}: {len(sc.blas_triangles)} BLAS triangles, {len(sc.blas_instances)} instances, TLAS {'yes' if sc.use_tlas else 'no'}")
        print("  read-backs made unnecessary: " + ", ".join(f"{k} {v / 2**20:.2f} MiB" for k, v in rb.items())
              + f"; total {sum(rb.values()) / 2**20:.2f} MiB")
        rows = []
        with PathTracer(16, 16) as pt:
            pt.SetScene(sc)
            if sc.use_tlas:
                pt.TlasBuild()
            for mode in (m for m in a.modes.split(",") if m == "linear" or sc.use_tlas):
                for n in (int(x) for x in a.counts.split(",")):
                    s = spheres(sc, n, seed=n)
                    for preset, st in PRESETS.items():
                        kernel, host = [], []
                        for _ in range(a.reps + 2):
                            t0 = time.perf_counter()
                            out, ms = pt.CollideSpheres(s, st, use_tlas=mode == "tlas")
                            host.append((time.perf_counter() - t0) * 1e3)
                            kernel.append(ms)
                        row = dict(mode=mode, spheres=n, preset=preset, kernel_ms=float(np.median(kernel[2:])),
                                   call_ms=float(np.median(host[2:])), hit_spheres=int((out["Hits"] > 0).sum()), hits=int(out["Hits"].sum()))
                        rows.append(row)
                        print(f"  {mode:6s}  {n:6d} spheres  {preset:6s}  kernel {row['kernel_ms']:9.3f} ms  call {row['call_ms']:9.3f} ms  "
                              f"({row['hit_spheres']} spheres hit, {row['hits']} hits)")
        result["scenes"][name] = dict(readback_bytes=rb, triangles=len(sc.blas_triangles), instances=len(sc.blas_instances), rows=rows)
    write_out(a.out, result)


if __name__ == "__main__":
    main()
