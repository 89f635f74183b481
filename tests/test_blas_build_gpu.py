"""idkpt_blas_build (PathTracer.BuildBlas): the device SweepSAH build with pre-splitting against the host build
(host.build_blas). Every comparison is exact: node and triangle bytes, required stack size, fragment count, SAH bits."""
import ctypes
import os

import numpy as np
import pytest

from idkengine_b200 import capi, host, scenes
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import IdkPtError, PathTracer

pytestmark = pytest.mark.gpu

IDKPT_ERR_INVALID_ARGUMENT, IDKPT_ERR_UNSUPPORTED = -1, -6


@pytest.fixture(scope="module")
def pt():
    with PathTracer(64, 48, device=0) as p:
        yield p


def assert_same(dev, ref):
    assert len(dev["nodes"]) == len(ref["nodes"])
    assert dev["nodes"].tobytes() == ref["nodes"].tobytes()
    assert len(dev["triangles"]) == len(ref["triangles"])
    assert dev["triangles"].tobytes() == ref["triangles"].tobytes()
    assert dev["required_stack_size"] == ref["required_stack_size"]
    assert dev["fragment_count"] == ref["fragment_count"]
    assert np.float64(dev["sah"]).tobytes() == np.float64(ref["sah"]).tobytes(), (dev["sah"], ref["sah"])


def host_settings(**kw):
    s = host.default_build_settings()
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def root_leaf_without_presplit(pt, positions, triangles, **settings):
    """A refittable BLAS whose root stays a leaf: the root is duplicated into nodes 2 and 3, each listing all n triangles.
    The host build's unindexing then writes 2n triangles into its n-element array (a heap overflow), so it is not run;
    what it returns is known: the first copy's n triangles, and the offset n for the second copy."""
    dev = pt.BuildBlas(positions, triangles, presplit=False, settings=host_settings(**settings))
    n = len(triangles)
    nodes = dev["nodes"]
    if not (len(nodes) == 4 and nodes[2]["TriCount"] == n and nodes[3]["TriCount"] == n):
        return None
    assert nodes[2]["TriStartOrChild"] == 0 and nodes[3]["TriStartOrChild"] == n and nodes[1]["TriStartOrChild"] == 2
    assert nodes[2]["Min"].tobytes() == nodes[1]["Min"].tobytes() == nodes[3]["Min"].tobytes()
    assert len(dev["triangles"]) == n
    assert sorted(dev["triangles"].tobytes()[16 * i:16 * i + 16] for i in range(n)) == \
        sorted(triangles.tobytes()[16 * i:16 * i + 16] for i in range(n))
    return dev


def compare(pt, positions, triangles, presplit=True, **settings):
    if not presplit:
        dev = root_leaf_without_presplit(pt, positions, triangles, **settings)
        if dev is not None:
            return dev
    ref = host.build_blas(positions, triangles, presplit=presplit, threads=os.cpu_count(), settings=host_settings(**settings))
    dev = pt.BuildBlas(positions, triangles, presplit=presplit, settings=host_settings(**settings))
    assert_same(dev, ref)
    return dev


def recorded(make, **kw):
    """Runs a scene constructor, recording every BLAS build it makes as (positions, triangles, presplit, host result)."""
    calls = []
    orig = host.build_blas

    def rec(positions, triangles, presplit=True, threads=None, settings=None):
        b = orig(positions, triangles, presplit=presplit, threads=os.cpu_count(), settings=settings)
        calls.append((positions.copy(), triangles.copy(), presplit, b))
        return b

    host.build_blas = rec
    try:
        make(**kw)
    finally:
        host.build_blas = orig
    return calls


def soup(n, seed=0, scale=1.0, size=0.05):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-scale, scale, (n, 1, 3))
    p = (c + rng.normal(0.0, size * scale, (n, 3, 3))).reshape(-1, 3).astype(np.float32)
    return mesh(p, np.arange(3 * n).reshape(-1, 3))


def mesh(p, idx):
    p = np.asarray(p, np.float32).reshape(-1, 3)
    pos = np.zeros(len(p), gt.PackedVec3)
    pos["x"], pos["y"], pos["z"] = p[:, 0], p[:, 1], p[:, 2]
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    tris = np.zeros(len(idx), gt.GpuBlasTriangle)
    tris["X"], tris["Y"], tris["Z"] = idx[:, 0], idx[:, 1], idx[:, 2]
    tris["MeshId"] = np.arange(len(idx)) % 7
    return pos, tris


# ---------------------------------------------------------------------------------------------------- scenes
SMALL_SCENES = {"cornell_1k": scenes.cornell_1k, "multi_blas": scenes.multi_blas, "closed_box": lambda: scenes.closed_box(subdiv=8),
                "open_floor": scenes.open_floor, "instance_grid": scenes.instance_grid, "textured_room": scenes.textured_room}


@pytest.mark.parametrize("name", sorted(SMALL_SCENES))
def test_every_model_of_the_test_scenes(pt, name):
    calls = recorded(SMALL_SCENES[name])
    assert calls
    for positions, triangles, presplit, ref in calls:
        assert_same(pt.BuildBlas(positions, triangles, presplit=presplit), ref)
        compare(pt, positions, triangles, presplit=not presplit)


@pytest.mark.parametrize("make", [lambda: scenes.atrium(262144), lambda: scenes.atrium(1_000_000), lambda: scenes.street_canyon(),
                                  lambda: scenes.atrium(9_000_000)], ids=["atrium_262k", "atrium_1m", "street_canyon_3.9m", "atrium_9m"])
def test_large_scenes(pt, make):
    calls = recorded(make)
    for positions, triangles, presplit, ref in calls:
        assert_same(pt.BuildBlas(positions, triangles, presplit=presplit), ref)


# ---------------------------------------------------------------------------------------------------- settings
@pytest.fixture(scope="module")
def atrium_model():
    calls = recorded(scenes.atrium, target_tris=40000)
    positions, triangles, _, _ = calls[0]
    return positions, triangles


@pytest.mark.parametrize("presplit", [True, False])
@pytest.mark.parametrize("setting", [dict(MaxLeafTriangleCount=1), dict(MaxLeafTriangleCount=8), dict(StopSplittingThreshold=4),
                                     dict(TriangleCost=0.5), dict(TriangleCost=3.0), dict(StackOptThreshold=1),
                                     dict(StackOptThreshold=1000), dict(StackOptSahIncreaseAcceptance=0.0),
                                     dict(StackOptSahIncreaseAcceptance=0.05), dict(SplitFactor=0.0), dict(SplitFactor=1.5)],
                         ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_settings(pt, atrium_model, setting, presplit):
    compare(pt, *atrium_model, presplit=presplit, **setting)


def test_stack_optimisation_collapses(pt, atrium_model):
    """StackOptThreshold 1 with a generous acceptance runs several collapse passes."""
    default = compare(pt, *atrium_model)
    collapsed = compare(pt, *atrium_model, StackOptThreshold=1, StackOptSahIncreaseAcceptance=0.05)
    assert collapsed["required_stack_size"] < default["required_stack_size"]


# ---------------------------------------------------------------------------------------------------- edge inputs
def _sliver_mesh():
    pos, tris = soup(2000, seed=3)
    p = np.stack([pos["x"], pos["y"], pos["z"]], 1)
    slivers = np.array([[-40, 0, 0], [40, 0.001, 0], [40, 0, 0.002], [0, -30, 5], [0.001, 30, 5], [0, 30, 5.001]], np.float32)
    p = np.concatenate([p, slivers])
    idx = np.concatenate([np.arange(len(p) - 6).reshape(-1, 3), np.arange(len(p) - 6, len(p)).reshape(-1, 3)])
    return mesh(p, idx)


def _sheet():
    g = np.stack(np.meshgrid(np.arange(40, dtype=np.float32), np.arange(30, dtype=np.float32)), -1).reshape(-1, 2)
    p = np.zeros((len(g), 3), np.float32)
    p[:, 0], p[:, 2] = g[:, 0] * 0.25, g[:, 1] * 0.25
    i = np.arange(40 * 30).reshape(30, 40)
    a, b, c, d = i[:-1, :-1].ravel(), i[:-1, 1:].ravel(), i[1:, :-1].ravel(), i[1:, 1:].ravel()
    return mesh(p, np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)]))


EDGES = {
    "one_triangle": lambda: mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 1, 2]]),
    "two_triangles": lambda: mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0], [3, 0, 1]], [[0, 1, 2], [1, 3, 2]]),
    "zero_area": lambda: mesh(np.repeat(np.random.default_rng(1).uniform(-1, 1, (300, 1, 3)), 3, 1) * np.array([1, 1, 1], np.float32)
                              + np.array([[0, 0, 0], [0.1, 0.1, 0.1], [0.3, 0.3, 0.3]], np.float32), np.arange(900).reshape(-1, 3)),
    "coincident_3000": lambda: mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.tile([0, 1, 2], (3000, 1))),
    "flat_sheet": _sheet,
    "slivers": _sliver_mesh,
    "huge_coordinates": lambda: soup(3000, seed=5, scale=1e30, size=0.2),
    "random_soup": lambda: soup(20000, seed=7, size=0.2),
}


@pytest.mark.parametrize("presplit", [True, False])
@pytest.mark.parametrize("name", sorted(EDGES))
def test_edge_inputs(pt, name, presplit):
    compare(pt, *EDGES[name](), presplit=presplit)


def test_huge_coordinates_have_infinite_areas(pt):
    pos, tris = EDGES["huge_coordinates"]()
    b = compare(pt, pos, tris)
    n = b["nodes"][1]
    s = (n["Max"] - n["Min"]).astype(np.float32)
    assert not np.isfinite(np.float32(s[0] * s[1]))


# ---------------------------------------------------------------------------------------------------- rejections
def _raw_build(pt, pos, tris, n_pos, n_tris, settings):
    h = ctypes.c_void_p()
    rc = pt._lib.idkpt_blas_build(pt._ctx, pos, n_pos, tris, n_tris, settings, ctypes.byref(h), None)
    if rc == 0:
        pt._lib.idkpt_blas_build_free(h)
    return rc, h


def test_rejections_leave_the_context_usable(pt):
    pos, tris = soup(500, seed=11)
    P, T = pos.ctypes.data, tris.ctypes.data
    d = capi.default_blas_build_settings
    cases = [
        ((None, T, len(pos), len(tris), None), IDKPT_ERR_INVALID_ARGUMENT),
        ((P, None, len(pos), len(tris), None), IDKPT_ERR_INVALID_ARGUMENT),
        ((P, T, len(pos), 0, None), IDKPT_ERR_INVALID_ARGUMENT),
        ((P, T, len(pos) - 1, len(tris), None), IDKPT_ERR_INVALID_ARGUMENT),   # the last vertex id is out of range
    ]
    for field, value in [("TriangleCost", np.inf), ("TriangleCost", np.nan), ("StackOptSahIncreaseAcceptance", np.nan),
                         ("SplitFactor", -np.inf), ("StopSplittingThreshold", 0)]:
        s = d()
        setattr(s, field, value)
        cases.append(((P, T, len(pos), len(tris), ctypes.byref(s)), IDKPT_ERR_INVALID_ARGUMENT))
    s = d()
    s.SplitFactor = 1e9      # far more than 2^24 fragments
    cases.append(((P, T, len(pos), len(tris), ctypes.byref(s)), IDKPT_ERR_UNSUPPORTED))
    for (p_, t_, np_, nt_, s_), want in cases:
        rc, h = _raw_build(pt, p_, t_, np_, nt_, s_)
        assert rc == want, (rc, want)
        assert not h.value
    h = ctypes.c_void_p()
    assert pt._lib.idkpt_blas_build(pt._ctx, P, len(pos), T, len(tris), None, None, None) == IDKPT_ERR_INVALID_ARGUMENT
    bad = tris.copy()
    bad["Y"][17] = -1
    with pytest.raises(IdkPtError):
        pt.BuildBlas(pos, bad)
    compare(pt, pos, tris)
    compare(pt, pos, tris, presplit=False)


# ---------------------------------------------------------------------------------------------------- context behaviour
def test_builds_between_queued_samples_change_nothing():
    scene, cam = scenes.cornell_1k(threads=1)
    model = recorded(scenes.cornell_1k)[0]
    w, h = 96, 64
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.RayDepth = 4
    images, builds = [], []
    for with_builds in (False, True):
        with PathTracer(w, h, s, device=0) as p:
            p.SetScene(scene)
            p.SetSky((0.6, 0.7, 0.9))
            p.SetFrame(frame)
            for _ in range(3):
                p.ComputeAsync()
            if with_builds:
                builds.append(p.BuildBlas(model[0], model[1]))      # queued samples: ordered after them
            p.Sync()
            if with_builds:
                builds.append(p.BuildBlas(model[0], model[1], presplit=False))
            p.ComputeAsync()
            p.Sync()
            assert p.AccumulatedSamples == 4
            images.append(p.Result.copy())
    assert np.array_equal(images[0], images[1])
    assert_same(builds[0], model[3])
    assert_same(builds[1], host.build_blas(model[0], model[1], presplit=False))


def test_scene_add_with_the_device_builder(pt, tmp_path):
    a = host.Scene().add(*scenes.multi_blas_models(), cache_dir=str(tmp_path / "host"))
    b = host.Scene().add(*scenes.multi_blas_models(), cache_dir=str(tmp_path / "device"), blas_builder=pt.BuildBlas)
    for f in ("positions", "blas_nodes", "blas_triangles", "blas_descs", "blas_instances", "meshes"):
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
    assert a.blas_stack_size == b.blas_stack_size
    assert [dict(i) for i in a.build_info] == [dict(i) for i in b.build_info]
    names = sorted(os.listdir(tmp_path / "host"))
    assert names and names == sorted(os.listdir(tmp_path / "device"))
    for n in names:
        assert (tmp_path / "host" / n).read_bytes() == (tmp_path / "device" / n).read_bytes()
