"""idkpt_update_models (ModelManager.Update on the device) against the host mirror (idkhost_anim_update) and against the
existing path fed the mirror's results (idkpt_update_range, idkpt_skin_vertices, idkpt_blas_refit, idkpt_tlas_build),
byte for byte, frame by frame."""
import copy

import numpy as np
import pytest

from idkengine_b200 import capi, host, scenes
from idkengine_b200.pathtracer import IdkPtError, PathTracer

pytestmark = pytest.mark.gpu

A = capi


def device_state(pt, sc, anim):
    n, t = len(anim.nodes), len(sc.mesh_transforms)
    out = dict(locals=pt.ReadRange(A.IDKPT_ARRAY_NODE_LOCAL_TRANSFORMS, 0, n), globals=pt.ReadRange(A.IDKPT_ARRAY_NODE_GLOBAL_TRANSFORMS, 0, n),
               xforms=pt.ReadRange(A.IDKPT_ARRAY_MESH_TRANSFORMS, 0, t))
    if len(anim.skins):
        jc = int((anim.skins["JointMatricesOffset"] + anim.skins["JointCount"]).max())
        out["joints"] = pt.ReadRange(A.IDKPT_ARRAY_JOINT_MATRICES, 0, jc)
    return out


def geometry(pt, sc):
    return dict(positions=pt.ReadRange(A.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(sc.positions)),
                vertices=pt.ReadRange(A.IDKPT_ARRAY_VERTICES, 0, len(sc.vertices)),
                blas=pt.ReadRange(A.IDKPT_ARRAY_BLAS_NODES, 0, len(sc.blas_nodes)),
                tlas=pt.ReadRange(A.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes)))


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def run_frames(sc, anim, times, unskinned=None, edits=None):
    """Every frame: UpdateModels on one context, the mirror + the existing calls on another; everything equal."""
    mirror = host.AnimationMirror(anim, len(sc.mesh_transforms), len(sc.blas_descs))
    xf = np.ascontiguousarray(copy.deepcopy(sc.mesh_transforms))
    flags = []
    with PathTracer(16, 16) as pt, PathTracer(16, 16) as ref:
        for p in (pt, ref):
            p.SetScene(sc)
            if unskinned is not None:
                p.SetSkinningData(unskinned)
        pt.SetAnimations(anim)
        for f, t in enumerate(times):
            if edits and f in edits:
                first, nodes = edits[f]
                pt.SetNodeTransforms(first, nodes)
                mirror.set_node_transforms(first, nodes)
            moved, _ = pt.UpdateModels(t)
            want = mirror.update(t, xf)
            assert want is not None and moved == want[0], (f, moved, want)
            flags.append((moved, want[1]))
            ref.UpdateRange(A.IDKPT_ARRAY_MESH_TRANSFORMS, 0, xf)
            if want[1] and len(anim.skins):
                ref.SkinVertices(mirror.read(2), mirror.skinning_cmds())
            if moved & 1:
                for b in anim.skins["BlasId"]:
                    ref.BlasRefit(int(b), 1)
            if moved:
                ref.TlasBuild()
            got = device_state(pt, sc, anim)
            exp = dict(locals=mirror.read(0), globals=mirror.read(1), xforms=xf)
            if "joints" in got:
                exp["joints"] = mirror.read(2)[:len(got["joints"])]
            assert_same(got, exp)
            assert_same(geometry(pt, sc), geometry(ref, sc))
    return flags, xf


def test_skinned_rig_frames():
    sc, anim, u = scenes.animated_skinned_rig()
    times = [0.0, 0.13, 0.37, 0.37, 0.5, 0.81, 1.25, 1.6, 2.2, 2.9, 3.4, 3.4, 3.4]
    flags, _ = run_frames(sc, anim, times, unskinned=u)
    assert flags[3] == (0, True)         # time == prev: nothing moves, skinning runs once more
    assert flags[-1] == (0, False)
    assert any(m == 3 for m, _ in flags)


def test_disabled_animation_and_host_edit():
    sc, anim, u = scenes.animated_skinned_rig()
    anim.animations["Enabled"] = 0
    nodes = copy.deepcopy(anim.nodes[1:2])
    nodes["Translation"] = (0.1, 0.2, 0.0)
    flags, _ = run_frames(sc, anim, [0.2, 0.4, 0.6, 0.8], unskinned=u, edits={2: (1, nodes)})
    assert flags == [(0, False), (0, False), (1, True), (0, True)]


def test_262144_transform_crowd():
    sc, anim = scenes.animated_crowd(262144)
    flags, _ = run_frames(sc, anim, [0.0, 0.25, 0.5, 0.5, 0.75])
    assert [m for m, _ in flags] == [0, 3, 3, 0, 3]


def test_2000_deep_chain():
    sc, anim = scenes.animated_chain(2000)
    flags, _ = run_frames(sc, anim, [0.0, 0.3, 0.6])
    assert flags[1][0] == 3


def test_singular_matrix_is_refused_and_changes_nothing():
    sc, anim, u = scenes.animated_skinned_rig()
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SetAnimations(anim)
        pt.UpdateModels(0.3)
        before = device_state(pt, sc, anim), geometry(pt, sc)
        flat = copy.deepcopy(anim.nodes[0:1])
        flat["Scale"] = (1.0, 0.0, 1.0)       # the root's, and so the skinned node's, global becomes singular
        pt.SetNodeTransforms(0, flat)
        with pytest.raises(IdkPtError, match="singular"):
            pt.UpdateModels(0.3)                      # the same time: no channel overwrites the scale
        after = device_state(pt, sc, anim), geometry(pt, sc)
        assert_same(before[1], after[1])
        for k in ("globals", "xforms", "joints"):
            assert before[0][k].tobytes() == after[0][k].tobytes(), k


def test_set_time_refusals_keep_the_set():
    sc, anim, u = scenes.animated_skinned_rig()
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        with pytest.raises(IdkPtError):
            pt.UpdateModels(0.0)                          # no set
        pt.SetSkinningData(u)
        pt.SetAnimations(anim)
        bad = copy.deepcopy(anim)
        bad.skins["BlasId"][0] = len(sc.blas_descs)
        with pytest.raises(IdkPtError):
            pt.SetAnimations(bad)
        pt.UpdateModels(0.2)                              # the old set is kept


def test_set_scene_drops_the_set_and_accumulation_resets_only_on_motion():
    sc, anim, u = scenes.animated_skinned_rig()
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SetAnimations(anim)
        assert pt.UpdateModels(0.2)[0] == 3
        pt._lib.idkpt_set_accumulated_samples(pt._ctx, 5)
        assert pt.UpdateModels(0.2)[0] == 0
        assert pt._lib.idkpt_accumulated_samples(pt._ctx) == 5
        assert pt.UpdateModels(0.4)[0] == 3
        assert pt._lib.idkpt_accumulated_samples(pt._ctx) == 0
        pt.SetScene(sc)
        with pytest.raises(IdkPtError):
            pt.UpdateModels(0.6)


def test_10000_animated_nodes():
    sc, anim = scenes.animated_nodes(10000)
    flags, _ = run_frames(sc, anim, [0.0, 0.2, 0.4, 0.4, 0.4])
    assert [m for m, _ in flags] == [0, 3, 3, 0, 0]


def test_tentacle_64_joints():
    sc, anim, u = scenes.animated_tentacle(64, seg=16, rings=200, threads=1)
    flags, _ = run_frames(sc, anim, [0.0, 0.3, 0.7, 0.7, 0.7], unskinned=u)
    assert flags == [(0, False), (1, True), (1, True), (0, True), (0, False)]


@pytest.mark.parametrize("bad", ["parent", "overlap", "keys", "data", "type", "mode", "transforms", "joint"])
def test_device_refusals_change_nothing(bad):
    sc, anim, u = scenes.animated_skinned_rig()
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SetAnimations(anim)
        pt.UpdateModels(0.4)
        before = device_state(pt, sc, anim), geometry(pt, sc)
        b = copy.deepcopy(anim)
        if bad == "parent":
            b.nodes["Parent"][2] = 2
        elif bad == "overlap":
            b.nodes["MeshTransformsStart"][1], b.nodes["MeshTransformsCount"][1] = 0, 1
        elif bad == "keys":
            b.channels["KeyFrameCount"][1] = 1
        elif bad == "data":
            b.channels["DataOffset"][2] = len(b.data)
        elif bad == "type":
            b.channels["Type"][0] = 7
        elif bad == "mode":
            b.channels["Mode"][0] = 2
        elif bad == "transforms":
            b.nodes["MeshTransformsCount"][0] = len(sc.mesh_transforms) + 1
        else:
            b.joint_nodes[0] = len(b.nodes)
        with pytest.raises(IdkPtError) as e:
            pt.SetAnimations(b)
        assert "(-1)" in str(e.value)
        after = device_state(pt, sc, anim), geometry(pt, sc)
        assert_same(before[0], after[0])
        assert_same(before[1], after[1])
        assert pt.UpdateModels(0.4)[0] == 0          # the old set, its time and state, are kept


def test_add_models_keeps_the_set():
    sc, anim, u = scenes.animated_skinned_rig()
    mirror = host.AnimationMirror(anim, len(sc.mesh_transforms), len(sc.blas_descs))
    xf = np.ascontiguousarray(copy.deepcopy(sc.mesh_transforms))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        pt.SetSkinningData(u)
        pt.SetAnimations(anim)
        assert pt.UpdateModels(0.2)[0] == mirror.update(0.2, xf)[0]
        pt.AddModels(*scenes.multi_blas_models()[:1])
        n = len(sc.mesh_transforms)
        added = pt.ReadRange(A.IDKPT_ARRAY_MESH_TRANSFORMS, n, 1)
        assert pt.UpdateModels(0.6)[0] == mirror.update(0.6, xf)[0] == 3
        assert pt.ReadRange(A.IDKPT_ARRAY_MESH_TRANSFORMS, 0, n).tobytes() == xf.tobytes()
        assert pt.ReadRange(A.IDKPT_ARRAY_MESH_TRANSFORMS, n, 1).tobytes() == added.tobytes()   # not the set's: untouched
        assert pt.ReadRange(A.IDKPT_ARRAY_NODE_GLOBAL_TRANSFORMS, 0, len(anim.nodes)).tobytes() == mirror.read(1).tobytes()


W, H = 96, 64


def animated_expectation(frames):
    """The skinned rig after `frames` UpdateModels on a device context, and the same state built by the oracle from the
    mirror: its transforms, the skin of its last joint matrices (oracle skin_vertices), the refit, the host TLAS build."""
    import oracle_lib as ol
    from test_tlas_build_gpu import host_tlas
    sc, anim, u = scenes.animated_skinned_rig()
    mirror = host.AnimationMirror(anim, len(sc.mesh_transforms), len(sc.blas_descs))
    expect = copy.deepcopy(sc)
    xf = np.ascontiguousarray(expect.mesh_transforms)
    cmd = mirror.skinning_cmds()[0]
    prev = None
    pt = PathTracer(W, H)
    pt.SetScene(sc)
    pt.SetSkinningData(u)
    pt.SetAnimations(anim)
    for t in frames:
        pt.UpdateModels(t)
        moved, skin = mirror.update(t, xf)
        if skin:
            prev = expect.positions.copy()
            ol.skin_vertices(u, mirror.read(2), expect.positions, expect.vertices, cmd)
    expect.mesh_transforms = xf
    ol.blas_refit(expect, 2)
    expect.tlas_nodes = host_tlas(expect, 15)
    return pt, expect, prev


def test_path_traced_image_after_the_sequence_equals_the_oracle():
    import oracle_lib as ol
    pt, expect, _ = animated_expectation([0.0, 0.3, 0.9, 1.4])
    _, cam = scenes.multi_blas(threads=1)
    frame = scenes.camera_frame(cam, W, H)
    s = capi.default_settings()
    with pt:
        assert pt.ReadRange(A.IDKPT_ARRAY_TLAS_NODES, 0, len(expect.tlas_nodes)).tobytes() == expect.tlas_nodes.tobytes()
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        pt.ResetAccumulation()
        pt.Compute()
        res = np.zeros((H, W, 4), np.float32)
        ol.path_trace(expect, frame, s, W, H, sky=(0.6, 0.7, 0.9), result=res)
        assert np.array_equal(pt.Result.view(np.uint32), res.view(np.uint32))


def test_gbuffer_velocity_after_the_sequence_equals_the_oracle():
    """idkpt_gbuffer reads the PrevModelMatrix idkpt_update_models kept and the previous positions its skinning kept."""
    import gbuffer_oracle as go
    from raster_lib import JITTER
    pt, expect, prev = animated_expectation([0.0, 0.3, 0.9, 1.4])
    assert prev is not None
    _, cam = scenes.multi_blas(threads=1)
    frame = scenes.camera_frame(cam, W, H)
    with pt:
        got = pt.GBuffer(frame, W, H, jitter=JITTER, prev_positions="kept")
    want = go.gbuffer(expect, frame, W, H, jitter=JITTER, prev_positions=np.stack([prev[c] for c in "xyz"], 1))
    for g, w in zip(got, want):
        assert np.asarray(g).tobytes() == np.asarray(w).tobytes()
    assert np.any(got[5] != 0)


def test_voxeliser_bound_to_the_animated_scene():
    """A voxeliser bound with idkvx_set_scene_from voxelises the scene idkpt_update_models animated exactly as one given the
    oracle's arrays of the same state, and as the voxeliser oracle."""
    import oracle_lib as ol
    from idkengine_b200 import vxgi
    lo, hi = (-3.2, -1.2, -3.2), (3.2, 4.2, 3.2)
    pt, expect, _ = animated_expectation([0.0, 0.3, 0.9])
    with pt, vxgi.Voxelizer(64, lo, hi) as bound, vxgi.Voxelizer(64, lo, hi) as owned:
        bound.SetSceneFrom(pt)
        owned.SetScene(expect)
        sb, so = bound.Render(), owned.Render()
        assert sb.Fragments == so.Fragments > 0
        got = [bound.ReadLevel(l).view(np.uint16) for l in range(len(bound.sizes))]
        want = [owned.ReadLevel(l).view(np.uint16) for l in range(len(owned.sizes))]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    ref = ol.vx_voxelize(expect, vxgi.create_info(64, lo, hi))[0]
    assert all(np.array_equal(np.asarray(a).view(np.uint16), np.asarray(b).view(np.uint16)) for a, b in zip(got, ref))
