"""host.Scene.add with a batch builder (blas_batch_builder, PathTracer.BuildBlases's signature): the slicing of one batch
result into the scene's arrays, checked with a stand-in batch builder made of host.build_blas; and the C++ wrapper's
BuildBlases, compiled and linked against the library."""
import os
import subprocess

import numpy as np

from idkengine_b200 import build, host, scenes

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def host_batch_builder(calls):
    """BuildBlases's contract over host.build_blas: BLAS s from triangles[TriangleOffset, +TriangleCount), pre-split when not
    refittable; descs with offsets into the concatenated nodes and triangles."""
    def batch(positions, triangles, descs, settings=None):
        calls.append(len(descs))
        out = descs.copy()
        nodes, tris, frags, sahs = [], [], [], []
        for k, d in enumerate(descs):
            b = host.build_blas(positions, triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]],
                                presplit=not d["IsRefittable"], threads=1, settings=settings)
            out[k]["NodeOffset"], out[k]["NodeCount"] = sum(map(len, nodes)), len(b["nodes"])
            out[k]["TriangleOffset"], out[k]["TriangleCount"] = sum(map(len, tris)), len(b["triangles"])
            out[k]["RequiredStackSize"] = b["required_stack_size"]
            nodes.append(b["nodes"])
            tris.append(b["triangles"])
            frags.append(b["fragment_count"])
            sahs.append(b["sah"])
        return dict(descs=out, nodes=np.concatenate(nodes), triangles=np.concatenate(tris),
                    fragment_counts=np.array(frags, np.int32), sahs=np.array(sahs, np.float64))
    return batch


def assert_same_scene(a, b):
    for f in ("positions", "vertices", "blas_nodes", "blas_triangles", "blas_descs", "blas_instances", "meshes", "materials",
              "mesh_transforms"):
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
    assert a.blas_stack_size == b.blas_stack_size
    assert [dict(i) for i in a.build_info] == [dict(i) for i in b.build_info]


def test_scene_add_slices_one_batch(tmp_path):
    models = scenes.multi_blas_models()
    calls = []
    a = host.Scene().add(*models, threads=1)
    b = host.Scene().add(*models, blas_batch_builder=host_batch_builder(calls))
    assert calls == [len(models)]
    assert_same_scene(a, b)
    # appended to a scene that already holds models: offsets continue behind them
    a.add(*models[:2], threads=1)
    b.add(*models[:2], blas_batch_builder=host_batch_builder(calls))
    assert calls == [len(models), 2]
    assert_same_scene(a, b)


def test_scene_add_batches_only_what_the_cache_lacks(tmp_path):
    room, ball, crate = scenes.multi_blas_models()
    host.Scene().add(ball, threads=1, cache_dir=str(tmp_path / "c"))          # the cache holds the ball
    calls = []
    a = host.Scene().add(room, ball, crate, threads=1, cache_dir=str(tmp_path / "h"))
    b = host.Scene().add(room, ball, crate, cache_dir=str(tmp_path / "c"), blas_batch_builder=host_batch_builder(calls))
    assert calls == [2]
    assert [i["from_cache"] for i in b.build_info] == [False, True, False]
    for i in b.build_info:
        i["from_cache"] = False
    assert_same_scene(a, b)
    names = sorted(os.listdir(tmp_path / "h"))
    assert names == sorted(os.listdir(tmp_path / "c"))
    for n in names:
        assert (tmp_path / "h" / n).read_bytes() == (tmp_path / "c" / n).read_bytes()
    calls.clear()
    host.Scene().add(room, ball, crate, cache_dir=str(tmp_path / "c"), blas_batch_builder=host_batch_builder(calls))
    assert calls == []                                                       # everything from the cache: no batch


def test_cpp_build_blases_compiles_and_links(tmp_path):
    exe = str(tmp_path / "hpp_blas_batch")
    libdir = os.path.dirname(build.LIBIDKPT)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-Wno-comment", "-I", os.path.join(REPO, "include"),
           os.path.join(REPO, "tests", "cpp", "hpp_blas_batch.cpp"), "-L", libdir, "-lidkpt", "-Wl,-rpath," + libdir, "-o", exe]
    subprocess.run(cmd, check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
