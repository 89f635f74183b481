"""The previous vertex positions skinning keeps (prevVertexPositionSSBO: idkpt_prev_positions_device_ptr), and the G-buffer
pass reading them in place (PathTracer.GBuffer(prev_positions="kept"))."""
import copy

import numpy as np
import pytest

import gbuffer_oracle as go
import oracle_lib as ol
from idkengine_b200 import capi, multigpu, scenes
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import JITTER, assert_bits, skinning_setup

pytestmark = pytest.mark.gpu

W, H = 96, 64


def xyz(positions):
    return np.stack([positions["x"], positions["y"], positions["z"]], 1).astype(np.float32)


def kept(pt):
    """The kept buffer, read through a zero-copy tensor."""
    import torch
    p, n = pt.PrevPositionsDevicePtr()
    assert n % 12 == 0
    return torch.as_tensor(multigpu.DeviceArray(p, (n // 12, 3)), device="cuda").cpu().numpy()


def device_positions(pt, n):
    return xyz(pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, n))


def assert_same(got, want):
    for a, b in zip(got, want):
        assert a.shape == b.shape
        assert_bits(a, b)


def skinned_scene():
    scene, cam = scenes.multi_blas(threads=1)
    u, jm, cmd = skinning_setup(scene, 2)
    return scene, cam, u, jm, cmd


def test_kept_buffer_starts_as_the_positions():
    scene, _ = scenes.multi_blas(threads=1)
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        assert np.array_equal(kept(pt), xyz(scene.positions))


def test_static_scene_kept_equals_this_frames_positions():
    scene, cam = scenes.multi_blas(threads=1)
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        want = pt.GBuffer(frame, W, H, jitter=JITTER)
        got = pt.GBuffer(frame, W, H, jitter=JITTER, prev_positions="kept")
    assert_same(got, want)


def test_after_a_skin_the_gbuffer_reads_the_positions_before_it():
    scene, cam, u, jm, cmd = skinned_scene()
    frame = scenes.camera_frame(cam, W, H)
    expect = copy.deepcopy(scene)
    ol.skin_vertices(u, jm, expect.positions, expect.vertices, cmd[0])
    ol.blas_refit(expect, 2)
    n = len(scene.positions)
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        before = device_positions(pt, n)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)                   # ModelManager.Update refits what it skinned: the pass traces the refitted records
        assert np.array_equal(kept(pt), before)
        got = pt.GBuffer(frame, W, H, jitter=JITTER, prev_positions="kept")
        uploaded = pt.GBuffer(frame, W, H, jitter=JITTER, prev_positions=before)
        still = pt.GBuffer(frame, W, H, jitter=JITTER)
    assert_same(got, uploaded)
    assert_same(got, go.gbuffer(expect, frame, W, H, jitter=JITTER, prev_positions=before))
    moved = np.any(got[5] != still[5], axis=-1)
    assert moved.any() and np.all(np.any(got[5][moved] != 0, axis=-1))


def test_second_skin_keeps_the_first_skins_output():
    scene, cam, u, jm, cmd = skinned_scene()
    jm2 = skinning_setup(scene, 2, seed=9)[1]
    n = len(scene.positions)
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        first = device_positions(pt, n)
        pt.SkinVertices(jm2, cmd)
        assert np.array_equal(kept(pt), first)
        assert not np.array_equal(device_positions(pt, n), first)


def test_overlapping_commands_follow_command_order():
    """Two commands write the same range: the kept range is what the first command left, as dispatch by dispatch in the engine."""
    scene, cam, u, jm, cmd = skinned_scene()
    jm2 = skinning_setup(scene, 2, seed=9)[1]
    joints = np.concatenate([jm, jm2])
    cmds = np.concatenate([cmd, cmd])
    cmds["JointMatricesOffset"][1] = len(jm) + 2
    after_first = copy.deepcopy(scene)
    ol.skin_vertices(u, joints, after_first.positions, after_first.vertices, cmds[0])
    after_both = copy.deepcopy(after_first)
    ol.skin_vertices(u, joints, after_both.positions, after_both.vertices, cmds[1])
    n = len(scene.positions)
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(joints, cmds)
        assert np.array_equal(kept(pt), xyz(after_first.positions))
        assert np.array_equal(device_positions(pt, n), xyz(after_both.positions))


def test_rejected_skin_leaves_the_kept_buffer():
    scene, cam, u, jm, cmd = skinned_scene()
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        k0 = kept(pt)
        bad = cmd.copy()
        bad["JointMatricesOffset"] = 100
        with pytest.raises(IdkPtError, match="joint index points past the joint matrices"):
            pt.SkinVertices(jm, np.concatenate([cmd, bad]))
        assert np.array_equal(kept(pt), k0)


def test_set_scene_resets_the_kept_buffer():
    scene, cam, u, jm, cmd = skinned_scene()
    with PathTracer(W, H) as pt:
        pt.SetScene(scene)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.SkinVertices(jm, cmd)
        assert not np.array_equal(kept(pt), xyz(scene.positions))
        pt.SetScene(scene)
        assert np.array_equal(kept(pt), xyz(scene.positions))
        with pytest.raises(ValueError):
            pt.GBuffer(scenes.camera_frame(cam, W, H), W, H, prev_positions="previous")


def test_no_scene():
    with PathTracer(W, H) as pt:
        with pytest.raises(IdkPtError, match="no scene"):
            pt.PrevPositionsDevicePtr()
