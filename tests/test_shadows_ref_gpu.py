"""The device's ray-traced point shadows (ShadowsRayTraced on host arrays, ShadowsRayTracedGBuffer on a G-buffer) on the
scenes of tests/test_shadows_ref.py, at image shapes the other shadow tests never use: 1x1, one row, one column, 33x9,
37x19, and a 1920-wide band of more pixels than one grid of the kernel's grid-stride loop holds (at most 2048 threads on
each of the H100's 132 SMs). Each image equals the CPU oracle's bit for bit and meets the float64 bounds."""
import numpy as np
import pytest

import test_shadows_ref as tsr

pytestmark = pytest.mark.gpu
SHAPES = [(1, 1), (37, 1), (1, 29), (33, 9), (37, 19)]


def device(scene, frame, depth, nrg, li, samples, noise_index=0, jitter=(0.0, 0.0)):
    from idkengine_b200.pathtracer import PathTracer
    h, w = depth.shape
    seed = np.full(depth.shape, tsr.SEED, np.float32)
    with PathTracer(max(w, 8), max(h, 8)) as pt:
        pt.SetScene(scene)
        host, _ = pt.ShadowsRayTraced(frame, depth, nrg, li, samples=samples, noise_index=noise_index, jitter=jitter, visibility=seed)
        slot = pt.ShadowsRayTracedGBuffer(frame, (depth, nrg), li, 0, samples=samples, noise_index=noise_index, jitter=jitter)
    return host, slot


def check(scene, cam, li, w, h, tag, min_share, samples=4, gscene=None, **kw):
    frame, depth, nrg = tsr.gbuffer(gscene or scene, cam, w, h)
    host, slot = device(scene, frame, depth, nrg, li, samples, **kw)
    want = tsr.oracle(scene, frame, depth, nrg, li, samples, **kw)
    assert np.array_equal(host.view(np.uint32), want.view(np.uint32)), tag
    lit = depth < 1.0
    assert np.array_equal(slot[lit].view(np.uint32), want[lit].view(np.uint32)) and np.all(slot[~lit] == 0.0), tag
    ref = tsr.judge(host, scene, frame, depth, nrg, li, tag, min_share if lit.sum() >= 100 else 0.0, samples=samples, **kw)
    return ref


@pytest.mark.parametrize("radius", tsr.RADII)
def test_slot_independence(radius):
    for dist in tsr.DISTANCES:
        s0, s2 = tsr.slot_scenes(radius, dist)
        frame, depth, nrg = tsr.gbuffer(s0, tsr.STAGE_CAM, 37, 19)
        v0, _ = device(s0, frame, depth, nrg, 0, 16)
        v2, _ = device(s2, frame, depth, nrg, 2, 16)
        assert np.array_equal(v0.view(np.uint32), v2.view(np.uint32)), (radius, dist)
        check(s0, tsr.STAGE_CAM, 0, 64, 48, "device radius %g distance %g" % (radius, dist), 0.9, samples=16)


@pytest.mark.parametrize("w,h", SHAPES)
def test_shapes(w, h):
    scene = tsr.stage([tsr.light((0.2, 2.0, 0.1), 0.5)])
    check(scene, tsr.STAGE_CAM, 0, w, h, "device penumbra %dx%d" % (w, h), 0.9, samples=16, noise_index=7,
          jitter=(0.37 / w, -0.61 / h))


def test_band_past_one_grid():
    scene = tsr.stage([tsr.light((0.2, 2.2, 0.1), 0.3)])
    check(scene, tsr.STAGE_CAM, 0, 1920, 144, "device band 1920x144", 0.9, samples=1, noise_index=1 << 20)


def test_scenes():
    check(tsr.open_floor([tsr.light((0.1, 0.25, 0.3), 0.5)]), tsr.STAGE_CAM, 0, 37, 19, "device inside the light", 0.9)
    check(tsr.open_floor([tsr.light((0.0, 3.0, 0.0), 0.3), tsr.light((0.2, 1.2, 0.1), 0.25)]), tsr.STAGE_CAM, 0, 33, 9,
          "device another light", 0.9, samples=8)
    for count, alpha_byte, _ in tsr.PANES:
        scene, floor_only = tsr.panes_scene([0.5 + 0.1 * k for k in range(count)], alpha_byte)
        check(scene, tsr.STAGE_CAM, 0, 64, 48, "device %d panes" % count, 0.85, gscene=floor_only)
    for gap, share in ((0.0005, 0.3), (0.01, 0.9)):
        scene, floor_only = tsr.panes_scene([0.6, 0.6 + gap], 128, wall=False)
        check(scene, tsr.STAGE_CAM, 0, 64, 48, "device panes %g apart" % gap, share, samples=1, gscene=floor_only)
    check(tsr.stage([tsr.light((3.5, 0.4, 0.0), 0.1)]), tsr.STAGE_CAM, 0, 37, 19, "device facing away", 0.9)


def test_textured_and_instances():
    from idkengine_b200 import scenes
    gpu, cpu, cam = tsr.textured()
    frame, depth, nrg = tsr.gbuffer(cpu, cam, 64, 48)
    host, slot = device(gpu, frame, depth, nrg, 0, 4)
    want = tsr.oracle(cpu, frame, depth, nrg, 0, 4)
    assert np.array_equal(host.view(np.uint32), want.view(np.uint32))
    tsr.judge(host, gpu, frame, depth, nrg, 0, "device textured", 0.4, samples=4)
    for tlas in (False, True):
        scene, cam = scenes.multi_blas(threads=1)
        if tlas:
            scene.build_tlas()
        check(scene, cam, 0, 37, 19, "device instances tlas=%s" % tlas, 0.8)


def test_masked():
    specs = [dict(color=(0.8, 0.2, 0.2, 129 / 255), cutoff=0.5), dict(color=(0.2, 0.8, 0.2, 126 / 255), cutoff=0.5)]
    from idkengine_b200 import scenes
    parts = [(scenes.quad([-1.2, 0.8, -1.2], [-1.2, 0.8, 0.8], [-0.1, 0.8, 0.8], [-0.1, 0.8, -1.2]), 1),
             (scenes.quad([0.1, 0.8, -1.2], [0.1, 0.8, 0.8], [1.2, 0.8, 0.8], [1.2, 0.8, -1.2]), 2)]
    lights = [tsr.light((0.0, 2.6, -0.2), 0.05)]
    ref = check(tsr.open_floor(lights, parts, specs), tsr.STAGE_CAM, 0, 64, 48, "device masked", 0.85, gscene=tsr.open_floor(lights))
    assert ref["judged"].sum() > 100
