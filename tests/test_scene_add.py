"""ModelManager.Add on the device scene in place (idkpt_add_models, PathTracer.AddModels), the parts that need no GPU: the
shared record helper and the documented rebase reproduce host.Scene.add exactly, the ctypes struct matches the header, and
the C++ wrapper's AddModels compiles and links."""
import copy
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from idkengine_b200 import build, capi, host, scenes
from idkengine_b200 import gpu_types as gt

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENE_ARRAYS = ("positions", "vertices", "meshes", "materials", "mesh_transforms", "blas_nodes", "blas_triangles", "blas_descs",
                "blas_instances")


def append_records(scene, models, textures=()):
    """What idkpt_add_models does, on a host scene: model_records, the rebase onto the scene's counts, the arrays appended,
    one host build per desc (pre-split when not refittable) with its desc filled as BVH.cs:363-386 fills it."""
    rec = host.rebase_records(host.model_records(models), vertices=len(scene.positions), meshes=len(scene.meshes),
                              materials=len(scene.materials), textures=len(scene.textures), blases=len(scene.blas_descs),
                              transforms=len(scene.mesh_transforms))
    for f in ("positions", "vertices", "meshes", "materials", "mesh_transforms", "blas_instances"):
        setattr(scene, f, np.concatenate([getattr(scene, f), rec[f]]))
    for d in rec["blas_descs"]:
        b = host.build_blas(scene.positions, rec["triangles"][d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]],
                            presplit=not d["IsRefittable"], threads=1)
        d = d.copy()
        d["NodeOffset"], d["NodeCount"] = len(scene.blas_nodes), len(b["nodes"])
        d["TriangleOffset"], d["TriangleCount"] = len(scene.blas_triangles), len(b["triangles"])
        d["RequiredStackSize"] = b["required_stack_size"]
        scene.blas_descs = np.concatenate([scene.blas_descs, [d]])
        scene.blas_nodes = np.concatenate([scene.blas_nodes, b["nodes"]])
        scene.blas_triangles = np.concatenate([scene.blas_triangles, b["triangles"]])
    scene.textures = scene.textures + list(textures)
    scene.blas_stack_size = max(1, int(scene.blas_descs["RequiredStackSize"].max()))
    return scene


def assert_same_arrays(a, b):
    for f in SCENE_ARRAYS:
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
    assert a.blas_stack_size == b.blas_stack_size


@pytest.mark.parametrize("split", [1, 3], ids=["one_model", "several_models"])
def test_records_and_rebase_give_scene_add(split):
    room, ball, crate = scenes.multi_blas_models()
    base = host.Scene().add(room, threads=1)
    added = [ball, crate][:1] if split == 1 else [ball, crate, ball]
    want = copy.deepcopy(base).add(*added, threads=1)
    got = append_records(copy.deepcopy(base), added)
    assert_same_arrays(got, want)
    # onto an empty scene too: the call-local records themselves, with their BLASes
    assert_same_arrays(append_records(host.Scene(), added), host.Scene().add(*added, threads=1))


def test_rebase_of_texture_handles_and_ids():
    room, ball, crate = scenes.multi_blas_models()
    room = copy.copy(room)
    room.materials = room.materials.copy()
    room.materials["BaseColorTexture"] = [0, 2]
    room.materials["NormalTexture"] = [1, 0]
    rec = host.model_records([room, crate])
    out = host.rebase_records(rec, vertices=10, meshes=3, materials=4, textures=5, blases=6, transforms=7)
    assert list(out["materials"]["BaseColorTexture"][:2]) == [0, 7] and list(out["materials"]["NormalTexture"][:2]) == [6, 0]
    assert out["materials"]["BaseColorTexture"].dtype == np.uint64
    assert list(out["blas_instances"]["BlasId"]) == [6, 7] and list(out["blas_instances"]["MeshTransformId"]) == [7, 8]
    assert np.array_equal(out["triangles"]["X"], rec["triangles"]["X"] + 10)
    assert np.array_equal(out["triangles"]["MeshId"], rec["triangles"]["MeshId"] + 3)
    assert np.array_equal(out["meshes"]["MaterialId"], rec["meshes"]["MaterialId"] + 4)
    assert out["blas_descs"].tobytes() == rec["blas_descs"].tobytes()     # triangle ranges stay call-local
    assert list(rec["blas_descs"]["IsRefittable"]) == [0, 1]
    assert list(rec["blas_descs"]["TriangleOffset"]) == [0, len(room.indices)]
    assert rec["materials"]["BaseColorTexture"][1] == 2                    # the input is not changed


def test_struct_size_matches_the_header():
    hdr = open(os.path.join(REPO, "include", "idkpt.h")).read()
    size = int(re.search(r"IDK_STATIC_ASSERT\(sizeof\(IdkPtAddModelsDesc\) == (\d+)", hdr).group(1))
    assert ctypes.sizeof(capi.IdkPtAddModelsDesc) == size == gt.IdkPtAddModelsDesc.itemsize
    names = [n for n, _ in capi.IdkPtAddModelsDesc._fields_]
    assert names == list(gt.IdkPtAddModelsDesc.names)
    assert "idkpt_add_models" in capi.EXPORTS


def test_desc_borrows_the_records():
    room, ball, crate = scenes.multi_blas_models()
    rec = host.model_records([ball, crate])
    d, keep = capi.add_models_desc(rec, textures=[dict(pixels=np.zeros((2, 2, 4), np.uint8))])
    assert (d.TriangleCount, d.BlasDescCount, d.BlasInstanceCount, d.MeshTransformCount, d.VertexCount, d.TextureCount) == \
        (len(rec["triangles"]), 2, 2, 2, len(rec["positions"]), 1)
    assert d.UnskinnedVertices is None and d.UnskinnedVertexCount == 0
    assert np.frombuffer((ctypes.c_char * 16).from_address(d.Triangles), gt.GpuBlasTriangle)[0] == rec["triangles"][0]


def test_cpp_add_models_compiles_and_links(tmp_path):
    exe = str(tmp_path / "hpp_add_models")
    libdir = os.path.dirname(build.LIBIDKPT)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-Wno-comment", "-I", os.path.join(REPO, "include"),
           os.path.join(REPO, "tests", "cpp", "hpp_add_models.cpp"), "-L", libdir, "-lidkpt", "-Wl,-rpath," + libdir, "-o", exe]
    subprocess.run(cmd, check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
