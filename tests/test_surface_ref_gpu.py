"""The device's textured materials and normal mapping: the G-buffer, the path tracer's first-hit AOVs and skinning on the
scenes of tests/test_surface_ref.py, with block-compressed textures decoded by the CUDA kernels. Each result equals the CPU
oracle's bit for bit and meets the same float64 bounds, so a fault the oracle shares is still caught."""
import numpy as np
import pytest

import gbuffer_oracle as go
import oracle_lib as ol
import surface_ref64 as sr
import test_surface_ref as tsr
from idkengine_b200 import capi, scenes
from idkengine_b200 import gpu_types as gt
from idkengine_b200.host import Model, Scene, compute_vertex_normals

pytestmark = pytest.mark.gpu
W, H = tsr.W, tsr.H


@pytest.fixture(scope="module")
def scene():
    return sr.textured_scene()


def test_gbuffer_textured(scene):
    from idkengine_b200.pathtracer import PathTracer
    gpu, cpu, cam = scene
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(W, H) as pt:
        pt.SetScene(gpu)
        got = pt.GBuffer(frame, W, H)
    want = go.gbuffer(cpu, frame, W, H)
    for k, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), k
    pix, mesh, rng, counts = sr.gbuffer_ref(cpu, frame, W, H)
    assert tsr.check_gbuffer(got, pix, mesh, rng, counts, "device G-buffer") == tsr.GBUFFER_REACH


def test_first_hit_aovs(scene):
    from idkengine_b200.pathtracer import PathTracer
    gpu, cpu, cam = scene
    frame = scenes.camera_frame(cam, W, H)
    s = capi.default_settings()
    s.RayDepth, s.OutputAOVs = 1, 1
    with PathTracer(W, H, s) as pt:
        pt.SetScene(gpu)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        pt.Compute()
        alb, nrm = pt.AlbedoTexture.copy().reshape(-1, 4), pt.NormalTexture.copy().reshape(-1, 4)
    oalb, onrm = tsr.first_hit_aovs(cpu, frame)
    assert np.array_equal(alb.view(np.uint32), oalb.view(np.uint32))
    assert np.array_equal(nrm.view(np.uint32), onrm.view(np.uint32))
    pix, mesh, rng, counts = sr.first_hit_ref(cpu, frame, W, H)
    tsr.check_aovs(alb, nrm, pix, rng, "device first hit")
    assert tsr.reached(mesh, rng) == tsr.FIRST_HIT_REACH


def test_skinning_non_rigid():
    from idkengine_b200.pathtracer import PathTracer
    u, jm, cmd = tsr.skinning_case()
    p, i = scenes.cylinder((0, -0.8, 0), 0.5, 1.6, 24, 8)
    n = compute_vertex_normals(p, i)
    scene = Scene().add(Model(p, i, normals=n, refittable=True), threads=1)
    with PathTracer(32, 32) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        vtx = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(u))
        pos = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(u))
    want_pos = np.zeros(len(u), gt.PackedVec3)
    want_vtx = scene.vertices.copy()
    ol.skin_vertices(u, jm, want_pos, want_vtx, cmd[0])
    assert np.array_equal(vtx["Normal"], want_vtx["Normal"]) and np.array_equal(vtx["Tangent"], want_vtx["Tangent"])
    assert np.array_equal(pos.view(np.uint32), want_pos.view(np.uint32))
    assert tsr.check_skinned(u, jm, vtx, "device skinning") == [2, 5]
