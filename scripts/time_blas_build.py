"""Timing of the BLAS build, device (idkpt_blas_build) against host (host.build_blas with every core) (DESIGN 8f.5).

    python scripts/time_blas_build.py [--reps 3] [--sizes 262144,1000000,9000000] [--out FILE]

The synthetic atrium at 262 k, 1 M and 9 M triangles (config 3), pre-split as the engine builds it. Per size, --reps rounds
that alternate a device and a host build of the same model, after one device warm-up build; each build is timed with a host
clock around the synchronous call (host arrays in and out, copies included), and the device build's own event time is kept
too. The per-stage device times of the last device build are printed (IDKPT_BLAS_TIMING). Every device build is checked
byte for byte against the host build of its round. The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

os.environ.setdefault("IDKPT_BLAS_TIMING", "1")   # libidkpt prints per-stage device times of every build to stderr
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import host, scenes  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402


def atrium_model(n):
    """Positions and source triangles of the atrium's one BLAS, without building it."""
    rec = []

    def capture(positions, triangles, presplit=True, threads=None, settings=None):
        rec.append((positions.copy(), triangles.copy()))
        raise StopIteration

    orig = host.build_blas
    host.build_blas = capture
    try:
        scenes.atrium(n)
    except StopIteration:
        pass
    finally:
        host.build_blas = orig
    return rec[0]


def same(a, b):
    return (a["nodes"].tobytes() == b["nodes"].tobytes() and a["triangles"].tobytes() == b["triangles"].tobytes()
            and a["required_stack_size"] == b["required_stack_size"] and a["fragment_count"] == b["fragment_count"]
            and np.float64(a["sah"]).tobytes() == np.float64(b["sah"]).tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="262144,1000000,9000000")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    threads = os.cpu_count()
    result = dict(card=card(), host_threads=threads, reps=a.reps, runs=[])
    with PathTracer(16, 16) as pt:
        for n in (int(s) for s in a.sizes.split(",")):
            positions, triangles = atrium_model(n)
            pt.BuildBlas(positions, triangles)      # warm-up: module load, allocator
            dev_ms, dev_kernel_ms, host_ms, equal = [], [], [], True
            for _ in range(a.reps):
                t0 = time.perf_counter()
                d = pt.BuildBlas(positions, triangles)
                dev_ms.append((time.perf_counter() - t0) * 1e3)
                dev_kernel_ms.append(pt.last_blas_build_ms)
                t0 = time.perf_counter()
                h = host.build_blas(positions, triangles, threads=threads)
                host_ms.append((time.perf_counter() - t0) * 1e3)
                equal = equal and same(d, h)
            run = dict(triangles=len(triangles), fragments=d["fragment_count"], nodes=len(d["nodes"]),
                       device_call_ms=round(float(np.median(dev_ms)), 2), device_event_ms=round(float(np.median(dev_kernel_ms)), 2),
                       host_ms=round(float(np.median(host_ms)), 2), speedup=round(float(np.median(host_ms) / np.median(dev_ms)), 2),
                       equal_to_host=equal)
            result["runs"].append(run)
            print(json.dumps(run), flush=True)
    print(json.dumps(result))
    write_out(a.out, result)


if __name__ == "__main__":
    main()
