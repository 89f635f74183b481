"""Timing of an animated frame's geometry work with VXGI: skin -> BLAS refit -> TLAS build -> voxelise at 256^3, with the
voxeliser bound to the path tracer's scene (idkvx_set_scene_from) against today's read-back recipe (idkpt_read_range of the
positions and vertices, then idkvx_set_scene of the whole scene), and of the G-buffer pass reading the previous positions
skinning keeps against a read-back and upload of them.

    python scripts/time_animated_frame.py [--tris 262144] [--frames 20] [--out FILE]

Scenes: the bench atrium (--tris requested) and the textured room, one BLAS skinned the way tests/raster_lib.skinning_setup
does it, every frame with other joint matrices. The two recipes run alternately, frame by frame, in one process; each frame is
timed with a host clock around calls that all end in a device synchronise. It prints the median, 10th and 90th percentile
of each, the device memory the voxeliser's own scene copy takes (free memory before and after idkvx_set_scene on a voxeliser
that has voxelised bound, so that both hold the same work queue), then
idkpt_gbuffer at 1920x1080 with prev_positions="kept" against idkpt_read_range + an upload, and the card's name and power
limit read in the same run.
"""
import argparse
import copy
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from idkengine_b200 import capi, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402
from raster_lib import TEX_GRID_MAX, TEX_GRID_MIN, skinning_setup  # noqa: E402
from timing_lib import JITTER, card, write_out  # noqa: E402

GRID = 256


def spread(ms):
    return dict(median=float(np.median(ms)), p10=float(np.percentile(ms, 10)), p90=float(np.percentile(ms, 90)), n=len(ms))


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def largest_blas(scene):
    return int(np.argmax(scene.blas_descs["TriangleCount"]))


def run_scene(name, scene, gmin, gmax, frames):
    scene.build_tlas()
    blas = largest_blas(scene)
    u, _, cmd = skinning_setup(scene, blas)
    joints = [skinning_setup(scene, blas, seed=100 + k)[1] for k in range(frames + 2)]
    read = copy.deepcopy(scene)
    npos, nvtx = len(scene.positions), len(scene.vertices)
    with PathTracer(64, 64) as pt, vxgi.Voxelizer(GRID, gmin, gmax) as bound, vxgi.Voxelizer(GRID, gmin, gmax) as owned:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        for vx in (bound, owned):
            vx.SetShadowTracer(pt)
            vx.SetSceneFrom(pt)
            vx.Render()                          # allocates the work queue both kinds of voxeliser hold
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        owned.SetScene(scene)                    # what a voxeliser with its own scene holds on top
        copy_bytes = free0 - torch.cuda.mem_get_info()[0]

        def geometry(k):
            pt.SkinVertices(joints[k], cmd)
            pt.BlasRefit(blas, 1)
            pt.TlasBuild()

        def recipe_bound(k):
            geometry(k)
            bound.Render()

        def recipe_today(k):
            geometry(k)
            read.positions[:] = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, npos)
            read.vertices[:] = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, nvtx)
            owned.SetScene(read)
            owned.Render()

        t = {"bound": [], "today": []}
        for k in range(frames + 2):              # the first two frames of each are warm-up
            order = (("bound", recipe_bound), ("today", recipe_today)) if k % 2 == 0 else (("today", recipe_today), ("bound", recipe_bound))
            for key, fn in order:
                ms = timed(lambda: fn(k))
                if k >= 2:
                    t[key].append(ms)
        same = all(np.array_equal(bound.ReadLevel(l).view(np.uint16), owned.ReadLevel(l).view(np.uint16)) for l in range(len(bound.sizes)))
    arrays = sum(a.nbytes for a in (scene.positions, scene.vertices, scene.blas_triangles, scene.blas_descs, scene.blas_instances,
                                    scene.mesh_transforms, scene.meshes, scene.materials, scene.lights))
    return dict(scene=name, triangles=int(len(scene.blas_triangles)), skinned_vertices=int(cmd["VertexCount"][0]),
                scene_array_bytes=int(arrays), owned_scene_copy_bytes=int(copy_bytes), bound_ms=spread(t["bound"]), today_ms=spread(t["today"]),
                last_grids_equal=bool(same))


def run_gbuffer(scene, cam, frames, w=1920, h=1080):
    blas = largest_blas(scene)
    u, jm, cmd = skinning_setup(scene, blas)
    frame = scenes.camera_frame(cam, w, h)
    npos = len(scene.positions)
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        t = {"kept": [], "read_back": []}
        held = {}

        def read_back():
            p = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, npos)
            held["prev"] = np.stack([p["x"], p["y"], p["z"]], 1)

        for k in range(frames + 2):              # alternately; the first two calls are warm-up
            if k % 2 == 0:
                pt.SkinVertices(jm, cmd)
                key, ms = "kept", timed(lambda: pt.GBuffer(frame, w, h, jitter=JITTER, prev_positions="kept", download=False))
            else:                                # today's recipe: read the positions back before the skin, upload them with the call
                ms = timed(read_back)
                pt.SkinVertices(jm, cmd)
                key = "read_back"
                ms += timed(lambda: pt.GBuffer(frame, w, h, jitter=JITTER, prev_positions=held["prev"], download=False))
            if k >= 2:
                t[key].append(ms)
    return dict(size=[w, h], vertex_positions=npos, kept_ms=spread(t["kept"]), read_back_and_upload_ms=spread(t["read_back"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    out = dict(card=card(), grid=GRID, frames=a.frames, scenes=[])
    atrium, cam = scenes.atrium(a.tris)
    room, _ = scenes.textured_room()
    out["scenes"].append(run_scene("atrium", copy.deepcopy(atrium), vxgi.DEFAULT_GRID_MIN, vxgi.DEFAULT_GRID_MAX, a.frames))
    out["scenes"].append(run_scene("textured_room", room, TEX_GRID_MIN, TEX_GRID_MAX, a.frames))
    out["gbuffer"] = run_gbuffer(atrium, cam, a.frames)
    for s in out["scenes"]:
        print(f"{s['scene']:14s} {s['triangles']:7d} tris, {s['skinned_vertices']} skinned vertices: bound {s['bound_ms']['median']:.2f} ms "
              f"[{s['bound_ms']['p10']:.2f}, {s['bound_ms']['p90']:.2f}], today {s['today_ms']['median']:.2f} ms "
              f"[{s['today_ms']['p10']:.2f}, {s['today_ms']['p90']:.2f}]; owned copy {s['owned_scene_copy_bytes'] / 2**20:.1f} MiB "
              f"({s['scene_array_bytes'] / 2**20:.1f} MiB of arrays); "
              f"grids equal {s['last_grids_equal']}")
    g = out["gbuffer"]
    print(f"gbuffer 1920x1080: kept {g['kept_ms']['median']:.3f} ms [{g['kept_ms']['p10']:.3f}, {g['kept_ms']['p90']:.3f}], read back + upload "
          f"{g['read_back_and_upload_ms']['median']:.3f} ms [{g['read_back_and_upload_ms']['p10']:.3f}, {g['read_back_and_upload_ms']['p90']:.3f}]")
    print(f"card: {out['card']}")
    write_out(a.out, out)


if __name__ == "__main__":
    main()
