"""The host mirror of idkpt_update_models (idkhost_anim_*): its sin / acos / Slerp / SortedLowerBound, the set-time checks,
and frame sequences against a float64 restatement of ModelManager.Update."""
import copy
import ctypes

import numpy as np
import pytest

from idkengine_b200 import capi, host
from idkengine_b200 import scenes
from idkengine_b200.scenes import quat
from idkengine_b200 import gpu_types as gt

A = capi


def _f(name, x):
    x = np.ascontiguousarray(x, np.float32)
    y = np.zeros_like(x)
    getattr(host.lib(), name)(x.ctypes.data, y.ctypes.data, len(x))
    return y


def _ulps(a, b):
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_sin_and_acos_within_one_ulp():
    x = np.linspace(0.0, np.pi / 2, 2_000_001).astype(np.float32)
    assert _ulps(_f("idkhost_anim_sin", x), np.sin(x.astype(np.float64)).astype(np.float32)).max() <= 1
    c = np.linspace(-1.0, 1.0, 2_000_001).astype(np.float32)
    assert _ulps(_f("idkhost_anim_acos", c), np.arccos(c.astype(np.float64)).astype(np.float32)).max() <= 1


def sorted_lower_bound(arr, value):
    """Algorithms.SortedLowerBound, transcribed literally."""
    lo, hi = 0, len(arr) - 1
    while lo < hi:
        mid = lo + (hi - lo) // 2
        if arr[mid] < value:
            lo = mid + 1
        else:
            hi = mid - 1
    if arr[lo] < value:
        lo += 1
    return lo


def test_sorted_lower_bound():
    rng = np.random.default_rng(5)
    for n in range(1, 40):
        for keys in (np.sort(rng.uniform(0, 4, n)), np.sort(rng.integers(0, 5, n)).astype(np.float64)):
            keys = np.ascontiguousarray(keys, np.float32)
            for v in np.concatenate([keys, rng.uniform(-1, 5, 20)]).astype(np.float32):
                assert host.lib().idkhost_anim_lower_bound(keys.ctypes.data, n, float(v)) == sorted_lower_bound(keys, v)


def slerp64(q1, q2, blend):
    q1, q2 = np.asarray(q1, np.float64), np.asarray(q2, np.float64).copy()
    c = q1 @ q2
    if c >= 1 or c <= -1:
        return q1
    if c < 0:
        q2, c = -q2, -c
    if c < 0.99:
        h = np.arccos(c)
        a, b = np.sin(h * (1 - blend)) / np.sin(h), np.sin(h * blend) / np.sin(h)
    else:
        a, b = 1 - blend, blend
    r = a * q1 + b * q2
    return r / np.linalg.norm(r)


@pytest.mark.parametrize("case", ["cos>=0.99", "cos<0.99", "negative dot", "dot +1", "dot -1"])
def test_slerp_branches(case):
    q1 = quat((0, 1, 0), 10.0)
    q2 = {"cos>=0.99": quat((0.3, 1, 0), 15.0), "cos<0.99": quat((0.3, 1, 0), 70.0), "negative dot": -quat((0, 1, 0), 180.0),
          "dot +1": q1.copy(), "dot -1": -q1}[case]
    c = float(q1.astype(np.float64) @ q2.astype(np.float64))
    assert {"cos>=0.99": c >= 0.99, "cos<0.99": 0 < c < 0.99, "negative dot": c < 0, "dot +1": c >= 1 - 1e-7, "dot -1": c <= -1 + 1e-7}[case]
    for blend in (0.0, 0.25, 0.5, 1.0):
        out = np.zeros(4, np.float32)
        host.lib().idkhost_anim_slerp(q1.ctypes.data, q2.ctypes.data, blend, out.ctypes.data)
        assert np.allclose(out, slerp64(q1, q2, blend), atol=2e-6)


def ref_update(state, anim, time, xf):
    """float64 restatement of ModelManager.Update's host half (ModelManager.cs:236-592) over `state`."""
    loc, glob, bits = state["locals"], state["globals"], state["bits"]
    dirty = np.zeros(len(anim.nodes), bool)
    if time != state["prev"]:
        state["prev"] = time
        for a in anim.animations:
            if not a["Enabled"]:
                continue
            t = np.fmod(np.float32(time), np.float32(a["TMax"] - a["TMin"]))
            for c in anim.channels[a["FirstChannel"]:a["FirstChannel"] + a["ChannelCount"]]:
                keys = anim.times[c["KeyFrameOffset"]:c["KeyFrameOffset"] + c["KeyFrameCount"]]
                if not (keys[0] <= t <= keys[-1]):
                    continue
                i = max(sorted_lower_bound(keys, t), 1)
                al = 0.0 if c["Mode"] == A.IDKPT_ANIM_STEP else (t - keys[i - 1]) / (keys[i] - keys[i - 1])
                w = 4 if c["Type"] == A.IDKPT_ANIM_ROTATION else 3
                d = anim.data[c["DataOffset"]:c["DataOffset"] + w * len(keys)].reshape(-1, w).astype(np.float64)
                v = slerp64(d[i - 1], d[i], al) if w == 4 else d[i - 1] + al * (d[i] - d[i - 1])
                field = {A.IDKPT_ANIM_ROTATION: "Rotation", A.IDKPT_ANIM_SCALE: "Scale", A.IDKPT_ANIM_TRANSLATION: "Translation"}[int(c["Type"])]
                if not np.array_equal(loc[c["TargetNode"]][field], v):
                    loc[c["TargetNode"]][field] = v
                    dirty[c["TargetNode"]] = True
    in_set = np.zeros(len(anim.nodes), bool)
    diffs = {}
    for i, n in enumerate(anim.nodes):
        p = n["Parent"]
        in_set[i] = dirty[i] or (p >= 0 and in_set[p])
        if in_set[i]:
            before = glob[i]
            g = host.AnimationMirror.node_matrix(loc[i])
            glob[i] = g if p < 0 else g @ glob[p]
            if n["MeshTransformsCount"]:
                diffs[i] = glob[i] @ np.linalg.inv(before)
    any_inst = False
    for i, n in enumerate(anim.nodes):
        for t in range(n["MeshTransformsStart"], n["MeshTransformsStart"] + n["MeshTransformsCount"]):
            if not in_set[i] and not bits[t]:
                continue
            old = xf[t]["Model"].copy()
            if in_set[i]:
                m4 = np.eye(4)
                m4[:, :3] = old.T
                xf[t]["Model"] = (diffs[i] @ m4)[:, :3].T
            xf[t]["Prev"] = old
            bits[t] = not np.array_equal(old, xf[t]["Model"])
            any_inst |= bits[t]
    if in_set.any():
        for s in anim.skins:
            inv_node = np.linalg.inv(glob[s["SkinnedNode"]])
            for j in range(s["JointCount"]):
                jj = s["FirstJoint"] + j
                m4 = anim.inverse_joints[jj].astype(np.float64) @ glob[anim.joint_nodes[jj]] @ inv_node
                state["joints"][s["JointMatricesOffset"] + j] = m4[:, :3].T          # Matrix4x4ToTranposed3x4
    return int(in_set.any()) | (2 if any_inst else 0)


def small_rig():
    an = host.Animations()
    r = an.add_node(transforms=(0, 2))
    c = an.add_node(parent=r, translation=(0.5, 0, 0), transforms=(2, 1))
    an.add_node(parent=c, translation=(0.0, 0.5, 0), transforms=(3, 2))
    an.add_node(transforms=(5, 1))                    # a second model's root, never animated
    an.init_globals()
    an.add_channel(r, A.IDKPT_ANIM_TRANSLATION, A.IDKPT_ANIM_LINEAR, [0, 1, 2], [[0, 0, 0], [1, 0, 0], [1, 1, 0]])
    an.add_channel(c, A.IDKPT_ANIM_ROTATION, A.IDKPT_ANIM_LINEAR, [0.5, 1.5], [quat((0, 0, 1), 0), quat((0, 0, 1), 70)])
    an.add_channel(c, A.IDKPT_ANIM_SCALE, A.IDKPT_ANIM_STEP, [0.0, 1.0, 2.0], [[1, 1, 1], [1.5, 2, 1], [1, 1, 1]])
    an.add_animation(0, 3, 0.0, 2.0)
    xf = np.zeros(6, gt.GpuMeshTransform)
    rng = np.random.default_rng(1)
    for i in range(6):
        xf[i] = host.mesh_transform(np.vstack([np.hstack([np.eye(3) * rng.uniform(0.5, 2), rng.uniform(-1, 1, (3, 1))]), [0, 0, 0, 1]]))
    return an, xf


def run_against_float64(an, xf, times):
    """Frames of the mirror against ref_update: flags exactly; the locals' matrices, the globals, every mesh transform (Model,
    Prev, and InvModel against the float64 inverse of the new Model) and the joint matrices to float32 accuracy."""
    m = host.AnimationMirror(an, len(xf), max(1, int(an.skins["BlasId"].max()) + 1) if len(an.skins) else 1)
    jc = int((an.skins["JointMatricesOffset"] + an.skins["JointCount"]).max()) if len(an.skins) else 0
    state = dict(locals=[{k: n[k].astype(np.float64) for k in ("Translation", "Rotation", "Scale")} for n in an.nodes],
                 globals=[n["GlobalTransform"].astype(np.float64) for n in an.nodes], bits=np.zeros(len(xf), bool), prev=-np.inf,
                 joints=np.zeros((jc, 3, 4)))
    ref = [{"Model": x["ModelMatrix"].astype(np.float64), "Prev": x["PrevModelMatrix"].astype(np.float64)} for x in xf]
    flags = []
    for t in times:
        got = m.update(t, xf)
        want = ref_update(state, an, t, ref)
        assert got[0] == want, (t, got, want)
        flags.append(got)
        for i in range(len(xf)):
            assert np.allclose(xf[i]["ModelMatrix"], ref[i]["Model"], atol=2e-5)
            assert np.allclose(xf[i]["PrevModelMatrix"], ref[i]["Prev"], atol=2e-5)
            full = np.vstack([ref[i]["Model"], [0, 0, 0, 1]])
            assert np.allclose(xf[i]["InvModelMatrix"], np.linalg.inv(full)[:3], rtol=1e-5, atol=2e-5), (t, i)
        assert np.allclose(m.read(1), np.array(state["globals"]), atol=2e-5)
        for k, loc in enumerate(m.read(0)):
            for f in ("Translation", "Rotation", "Scale"):
                assert np.allclose(loc[f], state["locals"][k][f], atol=2e-6), (t, k, f)
        if jc:
            assert np.allclose(m.read(2), state["joints"], atol=5e-5), t
    return flags


def test_mirror_against_float64_restatement():
    an, xf = small_rig()
    times = [0.0, 0.0, 0.25, 0.5, 1.0, 1.0, 1.7, 2.0, 2.5, 3.9, 3.9, 3.9]     # on keys, the % wrap, time == prev
    flags = run_against_float64(an, xf, times)
    assert flags[1] == (0, False) and flags[2][0] == 3
    assert flags[-2] == (0, True) and flags[-1] == (0, False)                  # the one extra skinning call
    assert np.array_equal(xf[5]["ModelMatrix"], xf[5]["PrevModelMatrix"])       # the untouched model keeps its matrices


def test_skinned_rig_against_float64_restatement():
    """The rig of the GPU tests: slerp in both branches, a negative dot, equal keys (dot 1), STEP, two channels on one
    property (the later animation wins), joint matrices at offset 2."""
    sc, an, _ = scenes.animated_skinned_rig()
    xf = np.ascontiguousarray(sc.mesh_transforms.copy())
    flags = run_against_float64(an, xf, [0.0, 0.13, 0.37, 0.37, 0.5, 0.81, 1.25, 1.6, 2.2, 2.9, 3.4, 3.4, 3.4])
    assert any(f[0] == 3 for f in flags) and flags[-1] == (0, False)


def test_writing_the_current_value_does_not_dirty():
    an, xf = small_rig()
    m = host.AnimationMirror(an, len(xf), 1)
    m.update(0.5, xf)
    nodes = copy.deepcopy(an.nodes)
    for k in ("Translation", "Rotation", "Scale"):
        nodes[k] = m.read(0)[k]
    assert nodes["Translation"][0][1] == 0.0 and not np.signbit(nodes["Translation"][0][1])
    nodes["Translation"][0][1] = -0.0                 # +0 written as -0: float.Equals says equal, so no node is dirty
    m.set_node_transforms(0, nodes)
    assert m.update(0.5, xf)[0] == 0
    assert not np.signbit(m.read(0)["Translation"][0][1])   # and the setter kept the +0 it had
    nodes["Scale"][3] = np.nan
    m.set_node_transforms(0, nodes)
    assert m.update(0.5, xf)[0] == 3
    m.set_node_transforms(0, nodes)                   # NaN == NaN under float.Equals
    assert m.update(0.5, xf)[0] == 0


def test_disabled_animation_moves_nothing():
    an, xf = small_rig()
    an.animations["Enabled"] = 0
    m = host.AnimationMirror(an, len(xf), 1)
    assert [m.update(t, xf)[0] for t in (0.3, 0.6)] == [0, 0]
    m.enable(0, [1])
    assert m.update(0.9, xf)[0] == 3


def _refused(an, transforms=6, blases=1):
    with pytest.raises(ValueError):
        host.AnimationMirror(an, transforms, blases)


def test_set_time_refusals():
    an, _ = small_rig()
    host.AnimationMirror(an, 6, 1)
    for change in (lambda a: a.nodes["Parent"].__setitem__(1, 1),
                   lambda a: a.nodes["Parent"].__setitem__(1, -2),
                   lambda a: a.nodes["MeshTransformsCount"].__setitem__(2, 5),
                   lambda a: a.nodes["MeshTransformsStart"].__setitem__(1, 1),
                   lambda a: a.channels["TargetNode"].__setitem__(0, 9),
                   lambda a: a.channels["Type"].__setitem__(0, 3),
                   lambda a: a.channels["Mode"].__setitem__(0, 2),
                   lambda a: a.channels["KeyFrameCount"].__setitem__(1, 1),
                   lambda a: a.channels["KeyFrameOffset"].__setitem__(2, 7),
                   lambda a: a.channels["DataOffset"].__setitem__(1, 20),
                   lambda a: a.animations["ChannelCount"].__setitem__(0, 4)):
        bad = copy.deepcopy(an)
        change(bad)
        _refused(bad)
    _refused(an, transforms=5)
    sk = copy.deepcopy(an)
    sk.joint_nodes = np.array([1, 2], np.uint32)
    sk.inverse_joints = np.tile(np.eye(4, dtype=np.float32), (2, 1, 1))
    sk.skins = np.zeros(1, gt.IdkPtSkin)
    sk.skins["SkinnedNode"], sk.skins["JointCount"] = 0, 2
    host.AnimationMirror(sk, 6, 1)
    for f, v in (("BlasId", 1), ("SkinnedNode", 4), ("FirstJoint", 1), ("JointMatricesOffset", 2 ** 31 - 1)):
        bad = copy.deepcopy(sk)
        bad.skins[f] = v
        _refused(bad)
    bad = copy.deepcopy(sk)
    bad.joint_nodes[1] = 4
    _refused(bad)


def test_struct_sizes():
    assert ctypes.sizeof(capi.IdkPtAnimationDesc) == 120
    for name, size in (("IdkPtNodeLocal", 40), ("IdkPtNode", 116), ("IdkPtNodeAnimation", 24), ("IdkPtModelAnimation", 20), ("IdkPtSkin", 32)):
        assert getattr(gt, name).itemsize == size
