"""Timing of the device TLAS build (idkpt_tlas_build, DESIGN 8f.2) from 3 to 1 M instances, and of both of its builds.

    python scripts/time_tlas_build.py [--reps 15] [--sizes 3,64,1024,16384,65536,262144,1048576] [--compare 3,64,1024,16384]
                                      [--variant-libs GRID.so,SINGLE.so] [--out FILE]

Scene: the nine small BLASes of scenes.instance_grid(2), instanced n times on a square 2-D grid (scale 0.4, 1.25 apart),
set with a placeholder TLAS. For every n of --sizes, on one context of the library as built:
  device   PathTracer.TlasBuild(15): the call's device time (kernel_ms, all its kernels) and the host clock around the call,
           median and min / max over --reps calls after two warm-ups; its nodes are checked byte for byte against the host
           build once. A tree deeper than the walk's 24-entry stack is refused: then only the host clock of the refusal;
  syncs    the host synchronisations of one call, counted by torch.profiler from the CUDA runtime calls that wait for the
           device (stream / device / event synchronise, and synchronous memcpy), less the profiler's own;
  recipe   what a scene above the old single-CTA limit had to do instead: read the (refitted) BLAS nodes back, build
           on the host (host.instance_boxes + idkhost_tlas_build) and upload the 2n - 1 nodes with UpdateRange; host clock.
The library picks its build from n (IDK_TLAS_SINGLE_CTA_MAX). To time both builds at the same n, every n of --compare is
also timed on two copies of the library compiled with the library's own flags into a temporary directory:
-DIDK_TLAS_SINGLE_CTA_MAX=0 (always the grid build) and -DIDK_TLAS_SINGLE_CTA_MAX=16384 (the single CTA up to 16384; its
rank sort is O(n^2), so not beyond). --variant-libs loads two such libraries instead of compiling them.
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import build, capi, host, scenes  # noqa: E402
from idkengine_b200 import gpu_types as gt  # noqa: E402
from idkengine_b200.pathtracer import IdkPtError, PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402


def grid_scene(base, n):
    k = int(np.ceil(np.sqrt(n)))
    i = np.arange(n)
    sc = base.__class__.__new__(base.__class__)
    sc.__dict__.update(base.__dict__)
    t = np.zeros(n, gt.GpuMeshTransform)
    for f in ("ModelMatrix", "PrevModelMatrix"):
        t[f][:, 0, 0] = t[f][:, 1, 1] = t[f][:, 2, 2] = 0.4
        t[f][:, 0, 3], t[f][:, 2, 3] = (i % k) * 1.25, (i // k) * 1.25
    t["InvModelMatrix"][:, 0, 0] = t["InvModelMatrix"][:, 1, 1] = t["InvModelMatrix"][:, 2, 2] = 2.5
    t["InvModelMatrix"][:, 0, 3], t["InvModelMatrix"][:, 2, 3] = -(i % k) * 1.25 * 2.5, -(i // k) * 1.25 * 2.5
    sc.mesh_transforms = t
    sc.blas_instances = np.zeros(n, gt.GpuBlasInstance)
    sc.blas_instances["BlasId"] = 1 + i % 8
    sc.blas_instances["MeshTransformId"] = i
    tl = np.zeros(2 * n - 1, gt.GpuTlasNode)        # a valid placeholder: node k's children at 2k + 1 and 2k + 2
    tl["IsLeafAndChildOrInstanceId"][:n - 1] = 2 * np.arange(n - 1) + 1
    tl["IsLeafAndChildOrInstanceId"][n - 1:] = np.uint32(0x80000000) | i.astype(np.uint32)
    sc.tlas_nodes = tl
    sc.use_tlas = 1
    return sc


def build_variants(tmp):
    """(grid, single): libidkpt with IDK_TLAS_SINGLE_CTA_MAX = 0 and = 16384, compiled in parallel into tmp."""
    srcs = [os.path.join(build.CSRC_DIR, f) for f in sorted(os.listdir(build.CSRC_DIR)) if f.endswith(".cu")]
    outs, procs = [], []
    for name, cap in (("grid", 0), ("single", 16384)):
        out = os.path.join(tmp, f"libidkpt_{name}.so")
        procs.append(subprocess.Popen([build.find_nvcc()] + build.NVCC_FLAGS + [f"-DIDK_TLAS_SINGLE_CTA_MAX={cap}", "-I", build.INCLUDE_DIR,
                                       "-I", build.CSRC_DIR, "-o", out] + srcs))
        outs.append(out)
    for p in procs:
        if p.wait():
            raise RuntimeError("compiling a libidkpt variant failed")
    return outs


SYNC_CALLS = ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy")


def host_syncs(pt):
    """Runtime calls of one TlasBuild that wait for the device, as torch.profiler records them, less those the profiler makes
    itself (counted over an empty profiled region)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    def count(work):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
            work()
        names = [e.name for e in prof.events()]
        return {c: names.count(c) for c in SYNC_CALLS}

    torch.cuda.init()
    empty = count(lambda: None)
    build = count(lambda: pt.TlasBuild(15))
    calls = {c: build[c] - empty[c] for c in SYNC_CALLS if build[c] - empty[c]}
    return dict(total=sum(calls.values()), **calls)


def time_builds(lib, sc, n, reps):
    """(kernel ms, host clock ms, nodes) of reps + 2 TlasBuild(15) calls on a fresh context of `lib`, after SetScene(sc)."""
    with PathTracer(16, 16, lib_path=lib) as pt:
        pt.SetScene(sc)
        kernel, clock = [], []
        for _ in range(reps + 2):
            t0 = time.perf_counter()
            kernel.append(pt.TlasBuild(15))
            clock.append(1e3 * (time.perf_counter() - t0))
        return kernel[2:], clock[2:], pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * n - 1)


def stats(xs):
    return dict(median=round(float(np.median(xs)), 4), min=round(float(np.min(xs)), 4), max=round(float(np.max(xs)), 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--sizes", default="3,64,1024,16384,65536,262144,1048576")
    ap.add_argument("--compare", default="3,64,1024,16384")
    ap.add_argument("--variant-libs", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    base, _ = scenes.instance_grid(2, threads=1)
    out = dict(card=card(), rows=[], compare=[])
    with tempfile.TemporaryDirectory() as tmp:
        compare = [int(s) for s in a.compare.split(",") if s]
        if compare:
            grid_lib, single_lib = a.variant_libs.split(",") if a.variant_libs else build_variants(tmp)
            for n in compare:
                sc = grid_scene(base, n)
                row = dict(n=n)
                boxes = host.instance_boxes(sc)
                want = np.zeros(2 * n - 1, gt.GpuTlasNode)
                host.lib().idkhost_tlas_build(boxes.ctypes.data, n, want.ctypes.data, 15)
                for name, lib in (("grid", grid_lib), ("single_cta", single_lib)):
                    k, c, nodes = time_builds(lib, sc, n, a.reps)
                    row[name] = dict(kernel_ms=stats(k), call_ms=stats(c), equal_to_host=nodes.tobytes() == want.tobytes())
                print(json.dumps(row), flush=True)
                out["compare"].append(row)
        time_sizes(a, base, out)
    print(json.dumps(out["card"]))
    write_out(a.out, out)


def time_sizes(a, base, out):
    for n in (int(s) for s in a.sizes.split(",")):
        sc = grid_scene(base, n)
        row = dict(n=n)
        with PathTracer(16, 16) as pt:
            pt.SetScene(sc)
            kernel, clock = [], []
            for _ in range(a.reps + 2):
                t0 = time.perf_counter()
                try:
                    kernel.append(pt.TlasBuild(15))
                except IdkPtError:                       # deeper than the walk's stack: refused, the scene is set again
                    row["refused"] = True
                clock.append(1e3 * (time.perf_counter() - t0))
                if row.get("refused"):
                    pt.SetScene(sc)
            if row.get("refused"):
                row["device_call_ms"] = stats(clock[2:])
                print(json.dumps(row), flush=True)
                out["rows"].append(row)
                continue
            got = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * n - 1)
            want = np.zeros(2 * n - 1, gt.GpuTlasNode)
            boxes = host.instance_boxes(sc)
            host.lib().idkhost_tlas_build(boxes.ctypes.data, n, want.ctypes.data, 15)
            row["equal_to_host"] = got.tobytes() == want.tobytes()
            row["device_kernel_ms"], row["device_call_ms"] = stats(kernel[2:]), stats(clock[2:])
            row["host_syncs"] = host_syncs(pt)
            recipe = []
            for _ in range(max(3, a.reps // 3)):
                t0 = time.perf_counter()
                rb = host.Scene.__new__(host.Scene)
                rb.blas_descs, rb.blas_instances = sc.blas_descs, sc.blas_instances
                rb.blas_nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, len(sc.blas_nodes))
                rb.mesh_transforms = sc.mesh_transforms      # the host sets them, so it holds them
                nodes = np.zeros(2 * n - 1, gt.GpuTlasNode)
                boxes = host.instance_boxes(rb)
                host.lib().idkhost_tlas_build(boxes.ctypes.data, n, nodes.ctypes.data, 15)
                pt.UpdateRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, nodes)
                recipe.append(1e3 * (time.perf_counter() - t0))
            row["readback_host_build_upload_ms"] = stats(recipe)
        print(json.dumps(row), flush=True)
        out["rows"].append(row)


if __name__ == "__main__":
    main()
