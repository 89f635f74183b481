"""Timing of batched BLAS builds (idkpt_blas_build_batch, idkpt_blas_rebuild over a range) (DESIGN 8f.5, "Batches").

    python scripts/time_blas_batch.py [--reps 5] [--workloads a,b,c,d] [--out FILE]

Workloads, all seeded:
  a  512 models of 1 k triangles      b  128 models of 8 k triangles
  c  a Sponza-like load: 300 models, log-uniform 12-50 k triangles, a quarter of them refittable
  d  RebuildBlases(0, 64) over 64 strips of 4 k triangles against 64 calls of RebuildBlases(k, 1)
For a-c each round times the batched call, a loop of idkpt_blas_build calls (one per model, the integration without
batches) and the host mirror with every core, one model after another; the first two are checked byte for byte against
each other. Medians over --reps rounds after one warm-up of each. Device times: the host clock around the synchronous call
and the calls' own event times (kernel_ms). The card name and power limit are read in the same run; the batch's per-stage
device times (IDKPT_BLAS_TIMING) are printed once per workload.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import gpu_types as gt  # noqa: E402
from idkengine_b200 import host  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402


def soup(n, rng):
    """n triangles scattered as small clusters: local vertex ids 0..3n-1."""
    c = rng.uniform(-10.0, 10.0, (n, 1, 3))
    p = (c + rng.normal(0.0, 0.3, (n, 3, 3))).reshape(-1, 3).astype(np.float32)
    pos = np.zeros(len(p), gt.PackedVec3)
    pos["x"], pos["y"], pos["z"] = p[:, 0], p[:, 1], p[:, 2]
    tris = np.zeros(n, gt.GpuBlasTriangle)
    idx = np.arange(3 * n).reshape(-1, 3)
    tris["X"], tris["Y"], tris["Z"] = idx[:, 0], idx[:, 1], idx[:, 2]
    return pos, tris


def workload(sizes, refittable, seed):
    """One position array, one triangle array and descs for models of the given sizes."""
    rng = np.random.default_rng(seed)
    pos, tris, v_off = [], [], 0
    descs = np.zeros(len(sizes), gt.GpuBlasDesc)
    for k, n in enumerate(sizes):
        p, t = soup(int(n), rng)
        for f in ("X", "Y", "Z"):
            t[f] += v_off
        descs[k]["TriangleOffset"], descs[k]["TriangleCount"], descs[k]["IsRefittable"] = sum(map(len, tris)), n, int(refittable[k])
        pos.append(p)
        tris.append(t)
        v_off += len(p)
    return np.concatenate(pos), np.concatenate(tris), descs


def models_of(name):
    rng = np.random.default_rng(11)
    if name == "a":
        return workload([1024] * 512, [False] * 512, 1)
    if name == "b":
        return workload([8192] * 128, [False] * 128, 2)
    sizes = np.exp(rng.uniform(np.log(12000), np.log(50000), 300)).astype(int)
    return workload(sizes, rng.uniform(size=300) < 0.25, 3)


def strips_scene(count=64, quads=2048):
    models = []
    for k in range(count):
        x = np.linspace(0.0, 4.0, quads + 1, dtype=np.float32)
        p = np.zeros((2 * (quads + 1), 3), np.float32)
        p[:quads + 1, 0] = p[quads + 1:, 0] = x - 2.0
        p[quads + 1:, 1] = 0.25 + 0.1 * np.sin(3.0 * x)
        p[:, 2] = -2.0 + 0.06 * k
        i = np.arange(quads)
        idx = np.concatenate([np.stack([i, i + 1, quads + 2 + i], 1), np.stack([i, quads + 2 + i, quads + 1 + i], 1)])
        models.append(host.Model(p, idx, refittable=(k % 4 == 3), name=f"strip{k}"))
    return host.Scene().add(*models, threads=os.cpu_count())


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def med(v):
    return round(float(np.median(v)), 2)


def build_loop(pt, positions, triangles, descs):
    out, ms = [], 0.0
    for d in descs:
        out.append(pt.BuildBlas(positions, triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]],
                                presplit=not d["IsRefittable"]))
        ms += pt.last_blas_build_ms
    return out, ms


def same(batch, loop):
    for k, b in enumerate(loop):
        d = batch["descs"][k]
        if (batch["nodes"][d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]].tobytes() != b["nodes"].tobytes()
                or batch["triangles"][d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]].tobytes() != b["triangles"].tobytes()
                or np.float64(batch["sahs"][k]).tobytes() != np.float64(b["sah"]).tobytes()):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default="a,b,c,d")
    ap.add_argument("--host-reps", type=int, default=1, help="rounds of the host mirror (slow at c)")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    threads = os.cpu_count()
    result = dict(card=card(), host_threads=threads, reps=a.reps, runs=[])
    with PathTracer(16, 16) as pt:
        for name in a.workloads.split(","):
            if name == "d":
                scene = strips_scene()
                pt.SetScene(scene)
                pt.RebuildBlases(0, 64)
                pt.RebuildBlases(0, 1)
                batch, batch_ev, loop, loop_ev = [], [], [], []
                for _ in range(a.reps):
                    ms, ev = timed(lambda: pt.RebuildBlases(0, 64))
                    batch.append(ms)
                    batch_ev.append(ev)
                    ms, ev = timed(lambda: sum(pt.RebuildBlases(k, 1) for k in range(64)))
                    loop.append(ms)
                    loop_ev.append(ev)
                run = dict(workload="d: rebuild 64 strips of 4 k", batch_call_ms=med(batch), batch_event_ms=med(batch_ev),
                           loop_call_ms=med(loop), loop_event_ms=med(loop_ev), speedup_over_loop=round(float(np.median(loop) / np.median(batch)), 1))
            else:
                positions, triangles, descs = models_of(name)
                os.environ["IDKPT_BLAS_TIMING"] = "1"
                pt.BuildBlases(positions, triangles, descs)       # warm-up, with the stage printout
                os.environ.pop("IDKPT_BLAS_TIMING")
                build_loop(pt, positions, triangles, descs)
                batch, batch_ev, loop, loop_ev, hst, equal = [], [], [], [], [], True
                for _ in range(a.reps):
                    ms, r = timed(lambda: pt.BuildBlases(positions, triangles, descs))
                    batch.append(ms)
                    batch_ev.append(pt.last_blas_build_ms)
                    ms, (lr, lev) = timed(lambda: build_loop(pt, positions, triangles, descs))
                    loop.append(ms)
                    loop_ev.append(lev)
                    equal = equal and same(r, lr)
                for _ in range(a.host_reps):
                    ms, _ = timed(lambda: [host.build_blas(positions, triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]],
                                                           presplit=not d["IsRefittable"], threads=threads) for d in descs])
                    hst.append(ms)
                run = dict(workload=name, blases=len(descs), triangles=int(descs["TriangleCount"].sum()),
                           fragments=int(r["fragment_counts"].sum()), batch_call_ms=med(batch), batch_event_ms=med(batch_ev),
                           loop_call_ms=med(loop), loop_event_ms=med(loop_ev), host_ms=med(hst),
                           speedup_over_loop=round(float(np.median(loop) / np.median(batch)), 1),
                           speedup_over_host=round(float(np.median(hst) / np.median(batch)), 1), batch_equals_loop=equal)
            result["runs"].append(run)
            print(json.dumps(run), flush=True)
    print(json.dumps(result))
    write_out(a.out, result)


if __name__ == "__main__":
    main()
