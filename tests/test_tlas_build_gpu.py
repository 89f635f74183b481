"""idkpt_tlas_build and the TLAS step of idkpt_add_models at any instance count: the device PLOC build over the grid against
the host mirror's TLAS.Build (idkhost_tlas_build) of the same world-space boxes, node for node. A build whose tree the TLAS
walk's 24-entry stack cannot hold is refused, exactly when the host tree is deeper than 24."""
import copy
import time

import numpy as np
import pytest

import oracle_lib as ol
from idkengine_b200 import capi, host, scenes
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import IdkPtError, PathTracer
from raster_lib import skinning_setup
from test_blas_rebuild_gpu import assert_image, opened, settings
from test_scene_add_gpu import ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, check, mirror, raw_add

pytestmark = pytest.mark.gpu

STACK = 24


def matrices(n, layout, seed=1):
    """n model matrices (n x 3 x 4, float64): `uniform` in a cube, a 2-D `grid`, or 64 gaussian `clusters`; each instance
    scaled and turned about y."""
    rng = np.random.default_rng(seed)
    side = max(1.0, n ** (1.0 / 3.0)) * 1.5
    if layout == "uniform":
        pos = rng.uniform(-side, side, (n, 3))
    elif layout == "grid":
        k = int(np.ceil(np.sqrt(n)))
        i = np.arange(n)
        pos = np.stack([(i % k) * 1.25, np.zeros(n), (i // k) * 1.25], 1)
    else:
        centres = rng.uniform(-4 * side, 4 * side, (64, 3))
        pos = centres[rng.integers(0, 64, n)] + rng.normal(0.0, 0.25 * side, (n, 3))
    scale = rng.uniform(0.2, 0.6, n)
    a = rng.uniform(0.0, 2 * np.pi, n)
    m = np.zeros((n, 3, 4))
    m[:, 0, 0], m[:, 0, 2], m[:, 2, 0], m[:, 2, 2] = np.cos(a) * scale, np.sin(a) * scale, -np.sin(a) * scale, np.cos(a) * scale
    m[:, 1, 1] = scale
    m[:, :, 3] = pos
    return m


def transforms(m):
    out = np.zeros(len(m), gt.GpuMeshTransform)
    m32 = m.astype(np.float32)
    full = np.zeros((len(m), 4, 4))
    full[:, :3, :] = m32
    full[:, 3, 3] = 1.0
    out["ModelMatrix"] = m32
    singular = np.linalg.det(full) == 0.0                  # a zero-scale instance: its inverse is never used by a hit
    full[singular] = np.eye(4)
    out["InvModelMatrix"] = np.linalg.inv(full)[:, :3, :].astype(np.float32)
    out["PrevModelMatrix"] = m32
    return out


def heap_tlas(n):
    """A valid TLAS of n instances and height ceil(log2 n): node k's children at 2k + 1 and 2k + 2, leaves behind the inner
    nodes. It lets a scene whose radius-15 tree is deep be set before the device build replaces it."""
    t = np.zeros(2 * n - 1, gt.GpuTlasNode)
    t["IsLeafAndChildOrInstanceId"][:n - 1] = 2 * np.arange(n - 1) + 1
    t["IsLeafAndChildOrInstanceId"][n - 1:] = np.uint32(0x80000000) | np.arange(n, dtype=np.uint32)
    return t


def height(t):
    """Stack entries the TLAS walk needs: the tree's height."""
    w = t["IsLeafAndChildOrInstanceId"].astype(np.int64)
    inner = np.nonzero(w < 0x80000000)[0]
    c = w[inner]
    h = np.zeros(len(t), np.int64)
    while True:
        nh = h.copy()
        nh[inner] = 1 + np.maximum(h[c], h[c + 1])
        if np.array_equal(nh, h):
            return int(h[0])
        h = nh


_BASE = None


def base():
    """Nine small BLASes (a floor, spheres, boxes, cylinders) and a light, without instances."""
    global _BASE
    if _BASE is None:
        _BASE, _ = scenes.instance_grid(2, threads=1)
    return copy.deepcopy(_BASE)


def instanced(m, blas_ids=None):
    """base() with one instance per model matrix; instance i uses BLAS 1 + i % 8 (not the floor) unless given."""
    sc = base()
    n = len(m)
    sc.mesh_transforms = transforms(m)
    sc.blas_instances = np.zeros(n, gt.GpuBlasInstance)
    sc.blas_instances["BlasId"] = 1 + np.arange(n) % 8 if blas_ids is None else blas_ids
    sc.blas_instances["MeshTransformId"] = np.arange(n)
    sc.tlas_nodes = heap_tlas(n)
    sc.use_tlas = 1
    return sc


def host_tlas(sc, radius):
    n = len(sc.blas_instances)
    boxes = host.instance_boxes(sc)
    out = np.zeros(2 * n - 1, gt.GpuTlasNode)
    host.lib().idkhost_tlas_build(boxes.ctypes.data, n, out.ctypes.data, radius)
    return out


def assert_device_build(pt, sc, radius):
    """TlasBuild(radius) equals the host build when that fits the stack, else is refused and invalidates the scene."""
    want = host_tlas(sc, radius)
    n = len(sc.blas_instances)
    if height(want) <= STACK:
        pt.TlasBuild(radius)
        got = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * n - 1)
        assert got.tobytes() == want.tobytes()
        return True
    with pytest.raises(IdkPtError):
        pt.TlasBuild(radius)
    with pytest.raises(IdkPtError):                       # "set it again"
        pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 1)
    return False


# ---------------------------------------------------------------------------------------------------- node for node
@pytest.mark.parametrize("layout", ["uniform", "grid", "clusters"])
def test_instance_counts(layout):
    fits = 0
    with PathTracer(16, 16) as pt:
        for n in (1, 2, 3, 31, 16384, 16385, 65536):
            sc = instanced(matrices(n, layout, seed=n))
            pt.SetScene(sc)
            fits += assert_device_build(pt, sc, 15)
    assert fits >= 6


def test_262144_instance_grid():
    m = matrices(262144, "grid")
    m[:, :, :3] = np.eye(3) * 0.4
    sc = instanced(m)
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        assert assert_device_build(pt, sc, 15)


@pytest.mark.parametrize("radius", [1, 2, 15, 1024])
def test_search_radius(radius):
    with PathTracer(16, 16) as pt:
        for n, layout in ((700, "uniform"), (5000, "clusters"), (20000, "grid")):
            sc = instanced(matrices(n, layout, seed=radius))
            pt.SetScene(sc)
            assert assert_device_build(pt, sc, radius)


def test_ties():
    cases = []
    # equal keys: pairs of boxes of different sizes whose centres fall into one Morton cell
    m = matrices(3000, "grid")
    m[1::2, :, 3] = m[0::2, :, 3] + 1e-3
    cases.append(m)
    # equal areas: identical boxes, few enough that the chain fits the stack
    m = np.zeros((STACK, 3, 4))
    m[:, 0, 0] = m[:, 1, 1] = m[:, 2, 2] = 1.0
    cases.append(m)
    # zero-size boxes (scale 0) at grid points, several per point, among ordinary ones
    m = matrices(5000, "grid")
    m[::3, :, :3] = 0.0
    m[1::7, :, 3] = m[0::7, :, 3][:len(m[1::7])]
    cases.append(m)
    # equal areas among neighbours: unit boxes on a line at equal spacing
    m = np.zeros((4000, 3, 4))
    m[:, 0, 0] = m[:, 1, 1] = m[:, 2, 2] = 1.0
    m[:, 0, 3] = np.arange(4000) * 2.0
    cases.append(m)
    with PathTracer(16, 16) as pt:
        for m in cases:
            sc = instanced(m, blas_ids=np.full(len(m), 2) if len(m) == STACK else None)
            pt.SetScene(sc)
            assert assert_device_build(pt, sc, 15)


def test_too_deep_is_refused_fast():
    """1 + 16384 instances, all but one identical: the host tree is a chain of height 16384. The device build stops at the
    first parent deeper than the stack, refuses the tree and invalidates the scene."""
    m = np.zeros((16385, 3, 4))
    m[:, 0, 0] = m[:, 1, 1] = m[:, 2, 2] = 1.0
    m[0, :, 3] = (5.0, 0.0, 0.0)
    sc = instanced(m, blas_ids=np.full(16385, 2))
    pt, _ = opened(sc)
    with pt:
        pt.Compute()
        t0 = time.perf_counter()
        with pytest.raises(IdkPtError) as e:
            pt.TlasBuild()
        assert time.perf_counter() - t0 < 1.0
        assert "deeper" in str(e.value)
        with pytest.raises(IdkPtError):
            pt.Compute()
        pt.SetScene(instanced(matrices(100, "grid")))     # set it again
        pt.Compute()


def test_after_transform_update():
    sc = instanced(matrices(20000, "uniform"))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        assert assert_device_build(pt, sc, 15)
        moved = sc.mesh_transforms.copy()
        m = moved["ModelMatrix"].astype(np.float64)
        m[::3, :, 3] += np.array([3.0, -1.5, 2.0])
        moved = transforms(m)
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 0, moved)
        sc.mesh_transforms = moved
        assert assert_device_build(pt, sc, 15)


def test_skinned_instanced_blas():
    """Skin, refit and TlasBuild of a BLAS that 20000 instances share."""
    scene, _ = scenes.multi_blas(threads=1)
    m = matrices(20000, "grid")
    scene.mesh_transforms = transforms(m)
    scene.blas_instances = np.zeros(len(m), gt.GpuBlasInstance)
    scene.blas_instances["BlasId"] = np.arange(len(m)) % len(scene.blas_descs)
    scene.blas_instances["MeshTransformId"] = np.arange(len(m))
    scene.tlas_nodes = heap_tlas(len(m))
    scene.use_tlas = 1
    expect = copy.deepcopy(scene)
    u, jm, cmd = skinning_setup(scene, 2)
    ol.skin_vertices(u, jm, expect.positions, expect.vertices, cmd[0])
    ol.blas_refit(expect, 2)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        pt.TlasBuild()
        before = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * len(m) - 1)
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.BlasRefit(2, 1)
        pt.TlasBuild()
        got = pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, 2 * len(m) - 1)
    want = host_tlas(expect, 15)
    assert got.tobytes() == want.tobytes() and got.tobytes() != before.tobytes()


def crowd(n):
    """A lit floor and n small instances standing on it in a 2-D grid, seen from above."""
    k = int(np.ceil(np.sqrt(n)))
    m = matrices(n, "grid")
    m[:, :, 3] = np.stack([(np.arange(n) % k) * 0.1 - 0.05 * k, np.full(n, 0.5), (np.arange(n) // k) * 0.1 - 0.05 * k], 1)
    m[:, :, :3] *= 0.1
    floor = np.eye(4)[None, :3]
    return instanced(np.concatenate([floor, m]), blas_ids=np.concatenate([[0], 1 + np.arange(n) % 8]))


def test_path_traced_image_over_16384_instances():
    sc = crowd(20000)
    s = settings()
    pt, frame = opened(sc, s)
    with pt:
        pt.TlasBuild()
        want = copy.deepcopy(sc)
        want.tlas_nodes = host_tlas(sc, 15)
        assert pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(want.tlas_nodes)).tobytes() == want.tlas_nodes.tobytes()
        assert_image(pt, want, frame, s)


def test_add_models_across_16384_instances():
    """AddModels onto a 16300-instance TLAS scene: 120 models take it past 16384; equal to host.Scene.add + build_tlas."""
    sc = crowd(16299)
    sc.tlas_nodes = host_tlas(sc, 15)
    _, ball, crate = scenes.multi_blas_models()
    models = []
    for i in range(120):
        t = host.trs_matrix(0.05, 7.0 * i, (-1.5 + 0.025 * i, 0.8 + 0.01 * (i % 5), 0.3 * np.sin(i)))
        mdl = copy.copy(crate if i % 2 else ball)
        mdl.model_matrix = t
        models.append(mdl)
    s = settings()
    pt, frame = opened(sc, s)
    with pt:
        pt.AddModels(*models)
        want = mirror(sc, models)
        assert len(want.blas_instances) == 16300 + 120 and want.use_tlas
        check(pt, frame, want, s)


def test_add_models_too_deep_changes_nothing():
    sc = crowd(100)
    sc.tlas_nodes = host_tlas(sc, 15)
    _, ball, _ = scenes.multi_blas_models()
    rec = host.model_records([ball])
    rec["blas_instances"] = np.zeros(20000, gt.GpuBlasInstance)      # 20000 identical boxes: a chain
    s = settings()
    pt, frame = opened(sc, s)
    with pt:
        pt.Compute()
        image = pt.Result.copy()
        assert raw_add(pt, rec) == ERR_UNSUPPORTED
        assert pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes)).tobytes() == sc.tlas_nodes.tobytes()
        with pytest.raises(IdkPtError):
            pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes) + 1)
        assert np.array_equal(pt.Result.view(np.uint32), image.view(np.uint32))


# ---------------------------------------------------------------------------------------------------- the two builds' seam
@pytest.mark.parametrize("radius", [2, 15])
def test_single_cta_and_grid_sizes(radius):
    """Both sides of IDK_TLAS_SINGLE_CTA_MAX (64), and the grid build on one block (65..256) and on two (257)."""
    with PathTracer(16, 16) as pt:
        for n in (63, 64, 65, 100, 256, 257, 600):
            sc = instanced(matrices(n, "uniform", seed=n + radius))
            pt.SetScene(sc)
            assert assert_device_build(pt, sc, radius)


@pytest.mark.parametrize("groups", [16, 40])
def test_identical_boxes_in_the_grid_build(groups):
    """Groups of 12 identical boxes, far apart: inside a group every area ties, so the first smallest decides."""
    k = np.repeat(np.arange(groups), 12)
    m = np.zeros((len(k), 3, 4))
    m[:, 0, 0] = m[:, 1, 1] = m[:, 2, 2] = 1.0
    m[:, 0, 3], m[:, 2, 3] = (k % 8) * 10.0, (k // 8) * 10.0
    sc = instanced(m, blas_ids=np.full(len(m), 2))
    with PathTracer(16, 16) as pt:
        pt.SetScene(sc)
        assert assert_device_build(pt, sc, 15)


# ---------------------------------------------------------------------------------------------------- non-finite boxes
@pytest.mark.parametrize("n", [3, 1000])
def test_non_finite_box_is_refused(n):
    """A NaN model matrix gives a box no area test accepts, so that node never merges. Both builds stop at the iteration that
    merges nothing, refuse the tree and invalidate the scene."""
    sc = instanced(matrices(n, "uniform"))
    pt, _ = opened(sc)
    with pt:
        moved = sc.mesh_transforms.copy()
        moved["ModelMatrix"][n // 2][0, 0] = np.nan
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 0, moved)
        with pytest.raises(IdkPtError) as e:
            pt.TlasBuild()
        assert "not finite" in str(e.value)
        with pytest.raises(IdkPtError):
            pt.Compute()
        pt.SetScene(sc)                                   # set it again
        assert assert_device_build(pt, sc, 15)


def test_add_models_non_finite_box_changes_nothing():
    sc = crowd(100)
    sc.tlas_nodes = host_tlas(sc, 15)
    _, ball, crate = scenes.multi_blas_models()
    rec = host.model_records([ball, crate])
    rec["mesh_transforms"]["ModelMatrix"][1][1, 3] = np.inf
    pt, _ = opened(sc, settings())
    with pt:
        pt.Compute()
        image = pt.Result.copy()
        assert raw_add(pt, rec) == ERR_INVALID_ARGUMENT
        assert pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes)).tobytes() == sc.tlas_nodes.tobytes()
        with pytest.raises(IdkPtError):
            pt.ReadRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, len(sc.tlas_nodes) + 1)
        assert np.array_equal(pt.Result.view(np.uint32), image.view(np.uint32))
