"""Timing of ModelManager.Update on the device (idkpt_update_models, DESIGN 8f.2) against the host recipe it replaces.

    python scripts/time_update_models.py [--frames 30] [--warmup 5] [--out FILE]

Workloads (idkengine_b200.scenes):
  crowd    262 144 instances whose transforms one node owns, under a moving parent (animated_crowd)
  nodes    10 000 root nodes, each with one instance and a translation channel of its own (animated_nodes)
  rig      a skinned cylinder of 102 464 vertices bent by 64 joints (animated_tentacle)
Per frame, on two contexts holding the same scene, alternately:
  host     the recipe idkpt_update_models replaces: the host mirror's update (idkhost_anim_update: keyframes, hierarchy,
           transforms, joint matrices), the upload of the transforms (every transform an animated node owns, when one
           moved: the whole array in these workloads), idkpt_skin_vertices with the mirror's joint matrices, idkpt_blas_refit
           of each skin's BLAS and idkpt_tlas_build, exactly when idkpt_update_models runs them;
  device   PathTracer.UpdateModels.
Both are host clocks around calls that end in a device synchronise (every call is synchronous). Median and min / max
over --frames frames (animation time advancing 1/60 s per frame) after --warmup frames. At the end both contexts' device
arrays (mesh transforms, positions, vertices, BLAS and TLAS nodes) are compared byte for byte.
kernel   k_anim_transforms' time from torch.profiler over --frames moving device frames of the crowd, and its achieved
         bytes/s: each moved transform reads and writes 144 B, and every transform's owner id (4 B) and moved bit (1 B)
         is read; against the H100 SXM data sheet's 3.35 TB/s.
The card name and power limit are read in the same run.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402

from idkengine_b200 import capi, host, scenes  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from timing_lib import card, write_out  # noqa: E402

A = capi
PEAK_BYTES_S = 3.35e12


def arrays(pt, sc):
    return [pt.ReadRange(w, 0, n).tobytes() for w, n in ((A.IDKPT_ARRAY_MESH_TRANSFORMS, len(sc.mesh_transforms)),
                                                        (A.IDKPT_ARRAY_VERTEX_POSITIONS, len(sc.positions)),
                                                        (A.IDKPT_ARRAY_VERTICES, len(sc.vertices)),
                                                        (A.IDKPT_ARRAY_BLAS_NODES, len(sc.blas_nodes)),
                                                        (A.IDKPT_ARRAY_TLAS_NODES, len(sc.tlas_nodes)))]


def stats(v):
    v = np.asarray(v)
    return dict(median_ms=float(np.median(v)), min_ms=float(v.min()), max_ms=float(v.max()))


def workload(name, sc, anim, unskinned, frames, warmup):
    mirror = host.AnimationMirror(anim, len(sc.mesh_transforms), len(sc.blas_descs))
    xf = np.ascontiguousarray(sc.mesh_transforms.copy())
    cmds = mirror.skinning_cmds()
    blases = [int(b) for b in anim.skins["BlasId"]]
    with PathTracer(16, 16) as dev, PathTracer(16, 16) as ref:
        for p in (dev, ref):
            p.SetScene(sc)
            if unskinned is not None:
                p.SetSkinningData(unskinned)
        dev.SetAnimations(anim)

        def host_frame(t):
            moved, skin = mirror.update(t, xf)
            if moved:
                ref.UpdateRange(A.IDKPT_ARRAY_MESH_TRANSFORMS, 0, xf)
            if skin and len(cmds):
                ref.SkinVertices(mirror.read(2), cmds)
            if moved & 1:
                for b in blases:
                    ref.BlasRefit(b, 1)
            if moved:
                ref.TlasBuild()
            return moved

        th, td, flags = [], [], []
        for f in range(warmup + frames):
            t = f / 60.0
            t0 = time.perf_counter()
            mh = host_frame(t)
            t1 = time.perf_counter()
            md, _ = dev.UpdateModels(t)
            t2 = time.perf_counter()
            assert mh == md, (name, f, mh, md)
            if f >= warmup:
                th.append((t1 - t0) * 1e3)
                td.append((t2 - t1) * 1e3)
                flags.append(md)
        same = arrays(dev, sc) == arrays(ref, sc)
    out = dict(workload=name, transforms=len(sc.mesh_transforms), nodes=len(anim.nodes),
               skinned_vertices=int(anim.skins["VertexCount"].sum()) if len(anim.skins) else 0,
               joints=int(anim.skins["JointCount"].sum()) if len(anim.skins) else 0,
               moving_frames=int(sum(1 for m in flags if m)), host=stats(th), device=stats(td),
               speedup=float(np.median(th) / np.median(td)), device_arrays_identical=bool(same))
    print(out, flush=True)
    return out


def transform_kernel(frames):
    import torch
    from torch.profiler import ProfilerActivity, profile
    sc, anim = scenes.animated_crowd(262144)
    n = len(sc.mesh_transforms)
    with PathTracer(16, 16) as dev:
        dev.SetScene(sc)
        dev.SetAnimations(anim)
        for f in range(3):
            dev.UpdateModels(f / 60.0)
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            moving = 0
            for f in range(3, 3 + frames):
                moving += dev.UpdateModels(f / 60.0)[0] & 2 != 0
    ev = [e for e in prof.events() if "k_anim_transforms" in e.name]
    us = [e.device_time for e in ev] if ev and hasattr(ev[0], "device_time") else [e.cuda_time for e in ev]
    ms = float(np.median(us)) / 1e3 if us else float("nan")
    moved_bytes = n * (144 + 144) + n * (4 + 1)
    return dict(kernel="k_anim_transforms", transforms=n, launches=len(us), moving_frames=int(moving), median_ms=ms,
                bytes_per_launch=moved_bytes, achieved_gb_s=moved_bytes / (ms * 1e-3) / 1e9, share_of_3_35_tb_s=moved_bytes / (ms * 1e-3) / PEAK_BYTES_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    result = dict(card=card())
    print(result["card"], flush=True)
    rows = []
    sc, anim = scenes.animated_crowd(262144)
    rows.append(workload("crowd 262144 instances under one animated node", sc, anim, None, a.frames, a.warmup))
    sc, anim = scenes.animated_nodes(10000)
    rows.append(workload("10000 animated single-instance nodes", sc, anim, None, a.frames, a.warmup))
    sc, anim, u = scenes.animated_tentacle(64)
    rows.append(workload("skinned rig, 64 joints", sc, anim, u, a.frames, a.warmup))
    result["workloads"] = rows
    result["transform_kernel"] = transform_kernel(a.frames)
    print(result["transform_kernel"], flush=True)
    write_out(a.out, result)
    assert all(r["device_arrays_identical"] for r in rows)


if __name__ == "__main__":
    main()
