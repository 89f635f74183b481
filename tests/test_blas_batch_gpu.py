"""idkpt_blas_build_batch (PathTracer.BuildBlases): many BLASes built in one device call, each against its host build
(host.build_blas) or its single device build (idkpt_blas_build); and idkpt_blas_rebuild, which builds its range as one batch,
against host.Scene.rebuild_blases. Every comparison is exact: node and triangle bytes, descs, fragment counts, SAH bits."""
import copy
import ctypes
import os

import numpy as np
import pytest

from idkengine_b200 import capi, host, scenes
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import PathTracer
from raster_lib import skinning_setup
from test_blas_build_gpu import EDGES, SMALL_SCENES, assert_same, host_settings, mesh, recorded, root_leaf_without_presplit, soup
from test_blas_rebuild_gpu import assert_image, assert_scene, mirror, opened, read_scene

pytestmark = pytest.mark.gpu

IDKPT_ERR_INVALID_ARGUMENT, IDKPT_ERR_UNSUPPORTED = -1, -6


@pytest.fixture(scope="module")
def pt():
    with PathTracer(64, 48, device=0) as p:
        yield p


def batch_inputs(models):
    """models: (positions, triangles, presplit) with model-local vertex ids -> one position array, one triangle array, descs."""
    pos, tris, descs, v_off, t_off = [], [], np.zeros(len(models), gt.GpuBlasDesc), 0, 0
    for k, (p, t, presplit) in enumerate(models):
        t = t.copy()
        for f in ("X", "Y", "Z"):
            t[f] += v_off
        pos.append(p)
        tris.append(t)
        descs[k]["TriangleOffset"], descs[k]["TriangleCount"], descs[k]["IsRefittable"] = t_off, len(t), 0 if presplit else 1
        descs[k]["LeafIndicesOffset"], descs[k]["ParentIndicesCount"] = 7 * k, 3 * k + 1   # copied through untouched
        v_off += len(p)
        t_off += len(t)
    return np.concatenate(pos), np.concatenate(tris), descs


def blas_of(r, k):
    d = r["descs"][k]
    return dict(nodes=r["nodes"][d["NodeOffset"]:d["NodeOffset"] + d["NodeCount"]],
                triangles=r["triangles"][d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]],
                required_stack_size=int(d["RequiredStackSize"]), fragment_count=int(r["fragment_counts"][k]), sah=float(r["sahs"][k]))


def check_batch(pt, positions, triangles, descs, refs, settings=None):
    """Builds the batch and checks every BLAS against refs[k] (a build_blas-style result) and the descs' packing."""
    r = pt.BuildBlases(positions, triangles, descs, settings=settings)
    assert len(r["descs"]) == len(descs)
    n_off = t_off = 0
    for k, ref in enumerate(refs):
        d = r["descs"][k]
        assert (d["NodeOffset"], d["TriangleOffset"]) == (n_off, t_off)
        for f in ("IsRefittable", "LeafIndicesOffset", "LeafIndicesCount", "ParentIndicesOffset", "ParentIndicesCount"):
            assert d[f] == descs[k][f], f
        assert_same(blas_of(r, k), ref)
        n_off += int(d["NodeCount"])
        t_off += int(d["TriangleCount"])
    assert (n_off, t_off) == (len(r["nodes"]), len(r["triangles"]))
    return r


def host_ref(positions, triangles, presplit, settings=None):
    return host.build_blas(positions, triangles, presplit=presplit, threads=os.cpu_count(), settings=settings)


def info(pt, positions, triangles, descs):
    h = ctypes.c_void_p()
    assert pt._lib.idkpt_blas_build_batch(pt._ctx, positions.ctypes.data, len(positions), triangles.ctypes.data, len(triangles),
                                          descs.ctypes.data, len(descs), None, ctypes.byref(h), None) == 0
    try:
        nn, nt, st, fr, sah = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_double()
        assert pt._lib.idkpt_blas_build_info(h, ctypes.byref(nn), ctypes.byref(nt), ctypes.byref(st), ctypes.byref(fr), ctypes.byref(sah)) == 0
        return nn.value, nt.value, st.value, fr.value, sah.value
    finally:
        pt._lib.idkpt_blas_build_free(h)


# ---------------------------------------------------------------------------------------------------- whole scenes
@pytest.fixture(scope="module")
def scene_models():
    """Every model of the small test scenes, in one list: (positions, triangles, presplit, host result)."""
    return [c for name in sorted(SMALL_SCENES) for c in recorded(SMALL_SCENES[name])]


@pytest.mark.parametrize("invert", [False, True], ids=["own_flags", "inverted_flags"])
def test_every_model_of_the_test_scenes_in_one_batch(pt, scene_models, invert):
    models = [(positions, triangles, presplit != invert) for positions, triangles, presplit, _ in scene_models]
    assert len(models) >= 10
    positions, triangles, descs = batch_inputs(models)
    check_batch(pt, positions, triangles, descs, refs_for(pt, positions, triangles, descs))


def refs_for(pt, positions, triangles, descs, **setting):
    """The host build of every BLAS of a batch; for a refittable BLAS whose root stays a leaf, which the host build cannot
    make (see root_leaf_without_presplit), the single device build."""
    refs = []
    for d in descs:
        src = triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]]
        dev = root_leaf_without_presplit(pt, positions, src, **setting) if d["IsRefittable"] else None
        refs.append(dev if dev is not None else host_ref(positions, src, not d["IsRefittable"], settings=host_settings(**setting)))
    return refs


# ---------------------------------------------------------------------------------------------------- many BLASes
def random_models(count, seed, lo=1, hi=20000, refittable_share=0.25):
    rng = np.random.default_rng(seed)
    sizes = np.exp(rng.uniform(np.log(lo), np.log(hi), count)).astype(int)
    out = []
    for k, n in enumerate(sizes):
        p, t = soup(int(max(1, n)), seed=seed * 1000 + k, scale=float(rng.uniform(0.5, 20.0)), size=float(rng.uniform(0.01, 0.3)))
        out.append((p, t, bool(rng.uniform() >= refittable_share)))
    return out


def atrium_model(n):
    calls = recorded(scenes.atrium, target_tris=n)
    return calls[0][0], calls[0][1], calls[0][2]


def test_many_blases_of_mixed_size(pt):
    models = random_models(400, seed=21)
    models.insert(200, atrium_model(262144))
    positions, triangles, descs = batch_inputs(models)
    refs = refs_for(pt, positions, triangles, descs)
    r = check_batch(pt, positions, triangles, descs, refs)
    nn, nt, stack, frags, sah = info(pt, positions, triangles, descs)
    total = np.float64(0.0)
    for ref in refs:
        total = np.float64(total + np.float64(ref["sah"]))
    assert np.float64(sah).tobytes() == total.tobytes()
    assert (nn, nt) == (len(r["nodes"]), len(r["triangles"]))
    assert stack == max(ref["required_stack_size"] for ref in refs)
    assert frags == sum(ref["fragment_count"] for ref in refs)


def test_a_blas_does_not_depend_on_its_batch(pt):
    models = random_models(40, seed=5, hi=5000)
    probe = (*atrium_model(30000)[:2], True)
    alone = pt.BuildBlas(probe[0], probe[1], presplit=True)
    for order in ([probe] + models, models + [probe], [probe] + models[::-1], (models + [probe])[::-1]):
        positions, triangles, descs = batch_inputs(order)
        k = next(i for i, m in enumerate(order) if m is probe)
        r = pt.BuildBlases(positions, triangles, descs)
        got = blas_of(r, k)
        d = descs[k]
        got["triangles"] = got["triangles"].copy()
        shift = int(triangles[d["TriangleOffset"]]["X"]) - int(probe[1][0]["X"])
        for f in ("X", "Y", "Z"):
            got["triangles"][f] -= shift
        assert_same(got, alone)


def test_ranges_anywhere_in_the_array(pt):
    """Descs may overlap, repeat and come in any order; each BLAS is built from its own range."""
    p, t = soup(3000, seed=9)
    descs = np.zeros(4, gt.GpuBlasDesc)
    for k, (o, n, refit) in enumerate([(1000, 500, 0), (0, 3000, 1), (1000, 500, 0), (2999, 1, 0)]):
        descs[k]["TriangleOffset"], descs[k]["TriangleCount"], descs[k]["IsRefittable"] = o, n, refit
    check_batch(pt, p, t, descs, refs_for(pt, p, t, descs))


# ---------------------------------------------------------------------------------------------------- edge inputs
def test_edge_blases_beside_ordinary_ones(pt):
    models, refs = [], []
    ordinary = random_models(6, seed=33, hi=3000)
    for k, name in enumerate(sorted(EDGES)):
        p, t = EDGES[name]()
        for presplit in (True, False):
            models += [ordinary[(2 * k + presplit) % len(ordinary)], (p, t, presplit)]
    # a refittable BLAS whose root stays a leaf: two coincident triangles with a large leaf limit
    leaf_root = mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.tile([0, 1, 2], (2, 1)))
    models.append((*leaf_root, False))
    models.append(ordinary[0])
    positions, triangles, descs = batch_inputs(models)
    refs = refs_for(pt, positions, triangles, descs)
    d = descs[-2]
    leaf = blas_of(pt.BuildBlases(positions, triangles, descs), len(descs) - 2)["nodes"]
    assert len(leaf) == 4 and leaf[2]["TriCount"] == leaf[3]["TriCount"] == 2 and d["IsRefittable"]
    check_batch(pt, positions, triangles, descs, refs)


# ---------------------------------------------------------------------------------------------------- settings
@pytest.mark.parametrize("setting", [dict(MaxLeafTriangleCount=1), dict(MaxLeafTriangleCount=8), dict(StopSplittingThreshold=4),
                                     dict(TriangleCost=0.5), dict(TriangleCost=3.0), dict(StackOptThreshold=1),
                                     dict(StackOptThreshold=1000), dict(StackOptSahIncreaseAcceptance=0.0),
                                     dict(StackOptSahIncreaseAcceptance=0.05), dict(SplitFactor=0.0), dict(SplitFactor=1.5),
                                     dict(StackOptThreshold=1, StackOptSahIncreaseAcceptance=0.05)],
                         ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_settings_on_a_mixed_batch(pt, setting):
    models = random_models(24, seed=77, hi=8000)
    models.insert(5, (*atrium_model(40000)[:2], True))
    models.insert(15, (*atrium_model(40000)[:2], False))
    positions, triangles, descs = batch_inputs(models)
    s = host_settings(**setting)
    refs = refs_for(pt, positions, triangles, descs, **setting)
    check_batch(pt, positions, triangles, descs, refs, settings=s)
    if setting == dict(StackOptThreshold=1):        # the BLASes leave the collapse rounds after different passes
        default = [host_ref(positions, triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]], not d["IsRefittable"],
                            settings=host_settings(StackOptThreshold=1000)) for d in descs]
        passes = {default[k]["required_stack_size"] - refs[k]["required_stack_size"] for k in range(len(refs))}
        assert len(passes) > 1


# ---------------------------------------------------------------------------------------------------- rejections
def _raw_batch(pt, pos, n_pos, tris, n_tris, descs, n_descs, settings, out=True):
    h = ctypes.c_void_p()
    rc = pt._lib.idkpt_blas_build_batch(pt._ctx, pos, n_pos, tris, n_tris, descs, n_descs, settings, ctypes.byref(h) if out else None, None)
    if rc == 0:
        pt._lib.idkpt_blas_build_free(h)
    return rc, h


def test_rejections_leave_the_context_usable(pt):
    models = random_models(5, seed=3, hi=2000)
    pos, tris, descs = batch_inputs(models)
    P, T, D = pos.ctypes.data, tris.ctypes.data, descs.ctypes.data
    d = capi.default_blas_build_settings

    def with_desc(k, **kw):
        x = descs.copy()
        for f, v in kw.items():
            x[k][f] = v
        return x

    keep = []
    cases = [((None, len(pos), T, len(tris), D, len(descs), None), IDKPT_ERR_INVALID_ARGUMENT),
             ((P, len(pos), None, len(tris), D, len(descs), None), IDKPT_ERR_INVALID_ARGUMENT),
             ((P, len(pos), T, len(tris), None, len(descs), None), IDKPT_ERR_INVALID_ARGUMENT),
             ((P, len(pos), T, len(tris), D, 0, None), IDKPT_ERR_INVALID_ARGUMENT)]
    for kw in (dict(TriangleCount=0), dict(TriangleCount=-3), dict(TriangleOffset=-1),
               dict(TriangleOffset=int(len(tris) - descs[4]["TriangleCount"] + 1))):
        x = with_desc(4 if "TriangleOffset" in kw else 2, **kw)
        keep.append(x)
        cases.append(((P, len(pos), T, len(tris), x.ctypes.data, len(x), None), IDKPT_ERR_INVALID_ARGUMENT))
    cases.append(((P, len(pos), T, len(tris) - 1, D, len(descs), None), IDKPT_ERR_INVALID_ARGUMENT))   # the last range ends past it
    cases.append(((P, int(tris[-1]["X"]), T, len(tris), D, len(descs), None), IDKPT_ERR_INVALID_ARGUMENT))  # a vertex id too large
    for field, value in [("TriangleCost", np.inf), ("TriangleCost", np.nan), ("StackOptSahIncreaseAcceptance", np.nan),
                         ("SplitFactor", -np.inf), ("StopSplittingThreshold", 0)]:
        s = d()
        setattr(s, field, value)
        keep.append(s)
        cases.append(((P, len(pos), T, len(tris), D, len(descs), ctypes.byref(s)), IDKPT_ERR_INVALID_ARGUMENT))
    s = d()
    s.SplitFactor = 1e9      # one pre-split BLAS of far more than 2^24 fragments
    cases.append(((P, len(pos), T, len(tris), D, len(descs), ctypes.byref(s)), IDKPT_ERR_UNSUPPORTED))
    for args, want in cases:
        rc, h = _raw_batch(pt, *args)
        assert rc == want, (rc, want)
        assert not h.value
    assert _raw_batch(pt, P, len(pos), T, len(tris), D, len(descs), None, out=False)[0] == IDKPT_ERR_INVALID_ARGUMENT
    # a refittable batch is not pre-split, so the same settings build it
    refit = descs.copy()
    refit["IsRefittable"] = 1
    assert _raw_batch(pt, P, len(pos), T, len(tris), refit.ctypes.data, len(refit), ctypes.byref(s))[0] == 0
    check_batch(pt, pos, tris, descs, refs_for(pt, pos, tris, descs))


def test_batch_copy_takes_null_outputs(pt):
    pos, tris, descs = batch_inputs(random_models(3, seed=4, hi=500))
    h = ctypes.c_void_p()
    assert pt._lib.idkpt_blas_build_batch(pt._ctx, pos.ctypes.data, len(pos), tris.ctypes.data, len(tris), descs.ctypes.data,
                                          len(descs), None, ctypes.byref(h), None) == 0
    try:
        assert pt._lib.idkpt_blas_build_batch_copy(h, None, None, None, None, None) == 0
        sahs = np.zeros(3, np.float64)
        assert pt._lib.idkpt_blas_build_batch_copy(h, None, None, None, None, sahs.ctypes.data) == 0
        assert (sahs > 0).all()
    finally:
        pt._lib.idkpt_blas_build_free(h)
    assert pt._lib.idkpt_blas_build_batch_copy(None, None, None, None, None, None) == IDKPT_ERR_INVALID_ARGUMENT


# ---------------------------------------------------------------------------------------------------- context behaviour
def test_batch_between_queued_samples_changes_nothing():
    scene, cam = scenes.cornell_1k(threads=1)
    pos, tris, descs = batch_inputs(random_models(30, seed=8, hi=3000))
    w, h = 96, 64
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.RayDepth = 4
    images = []
    for with_builds in (False, True):
        with PathTracer(w, h, s, device=0) as p:
            p.SetScene(scene)
            p.SetSky((0.6, 0.7, 0.9))
            p.SetFrame(frame)
            for _ in range(3):
                p.ComputeAsync()
            if with_builds:
                check_batch(p, pos, tris, descs, refs_for(p, pos, tris, descs))      # queued samples: ordered after them
            p.Sync()
            p.ComputeAsync()
            p.Sync()
            assert p.AccumulatedSamples == 4
            images.append(p.Result.copy())
    assert np.array_equal(images[0], images[1])


# ---------------------------------------------------------------------------------------------------- rebuild
def strips_scene(count=63, quads=2048):
    """A pre-split hall of large quads, which splits again on every rebuild, then `count` strips of 2 * quads triangles
    each, every fourth one refittable."""
    room = scenes.multi_blas_models()[0]
    a = scenes._Assembler()
    a.add(scenes.quad([-3, 0, -3], [-3, 0, 3], [3, 0, 3], [3, 0, -3]), 0)
    a.add(scenes.quad([-3, 0, -3], [3, 0, -3], [3, 4, -3], [-3, 4, -3]), 0)
    a.add(scenes.uv_sphere([0, 1, 0], 0.5, 12, 16), 0)
    models = [a.model(room.meshes[:1], room.materials[:1], name="hall")]
    for k in range(count):
        x = np.linspace(0.0, 4.0, quads + 1, dtype=np.float32)
        p = np.zeros((2 * (quads + 1), 3), np.float32)
        p[: quads + 1, 0] = p[quads + 1:, 0] = x - 2.0
        p[quads + 1:, 1] = 0.25
        p[:, 2] = -2.0 + 0.06 * k
        p[:, 1] += 0.01 * k
        i = np.arange(quads)
        idx = np.concatenate([np.stack([i, i + 1, quads + 2 + i], 1), np.stack([i, quads + 2 + i, quads + 1 + i], 1)])
        models.append(host.Model(p, idx, meshes=room.meshes[:1], materials=room.materials[:1], refittable=(k % 4 == 3), name=f"strip{k}"))
    scene = host.Scene().add(*models, threads=os.cpu_count())
    scene.add_light((-1.0, 2.5, 1.0), (30.0, 28.0, 20.0), 0.3)
    return scene


def bend(pt, scene, first, count, amount):
    """Moves the vertices of BLASes [first, first + count) on the device: a bend about x."""
    pos = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
    for b in range(first, first + count):
        d = scene.blas_descs[b]
        t = scene.blas_triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]]
        v = np.unique(np.concatenate([t["X"], t["Y"], t["Z"]]))
        x = pos["x"][v].astype(np.float64)
        pos["y"][v] = (pos["y"][v] + amount * (1 + b % 5) * np.sin(x * 1.7)).astype(np.float32)
        pos["z"][v] = (pos["z"][v] + 0.5 * amount * np.cos(x * 0.9 + b)).astype(np.float32)
    return pos


def test_rebuild_of_many_moved_blases():
    scene = strips_scene()
    scene.build_tlas()
    s = capi.default_settings()
    s.Gpu.DoTraceLights = 1
    pt, frame = opened(scene, s)
    with pt:
        moved = copy.deepcopy(scene)
        moved.positions = bend(pt, scene, 0, 64, 0.05)
        pt.SetScene(moved)
        pt.RebuildBlases(0, 64)
        pt.TlasBuild()
        want = mirror(pt, moved, 0, 64)
        got = assert_scene(pt, want)
        assert want.blas_descs[0]["TriangleCount"] > scene.blas_descs[0]["TriangleCount"]   # pre-split again: it grew
        assert got.blas_stack_size == want.blas_stack_size
        assert_image(pt, want, frame, s)

        # a failed rebuild (one BLAS of the range over 2^24 fragments) changes nothing
        before = read_scene(pt, want)
        pt.Compute()
        image = pt.Result.copy()
        bad = host.default_build_settings()
        bad.SplitFactor = 1e9
        with pytest.raises(Exception, match=f"failed \\({IDKPT_ERR_UNSUPPORTED}\\)"):
            pt.RebuildBlases(0, 64, settings=bad)
        after = read_scene(pt, want)
        for f in ("blas_descs", "blas_nodes", "blas_triangles", "tlas_nodes"):
            assert getattr(after, f).tobytes() == getattr(before, f).tobytes(), f
        assert np.array_equal(pt.Result.view(np.uint32), image.view(np.uint32))


def test_rebuild_of_skinned_blases():
    from test_blas_rebuild import room_crate_ball
    scene = room_crate_ball()
    scene.build_tlas()
    u, jm, cmd = skinning_setup(scene, 1)
    s = capi.default_settings()
    s.Gpu.DoTraceLights = 1
    pt, frame = opened(scene, s)
    with pt:
        pt.SetSkinningData(u)
        pt.SkinVertices(jm, cmd)
        pt.RebuildBlases(0, len(scene.blas_descs))
        pt.TlasBuild()
        want = mirror(pt, scene, 0, len(scene.blas_descs))
        assert_scene(pt, want)
        assert_image(pt, want, frame, s)


# ---------------------------------------------------------------------------------------------------- Scene.add
@pytest.mark.parametrize("cached", [False, True], ids=["no_cache", "cache"])
def test_scene_add_with_the_batch_builder(pt, tmp_path, cached):
    kw = lambda sub: dict(cache_dir=str(tmp_path / sub)) if cached else {}
    a = host.Scene().add(*scenes.multi_blas_models(), **kw("host"))
    b = host.Scene().add(*scenes.multi_blas_models(), blas_batch_builder=pt.BuildBlases, **kw("device"))
    for f in ("positions", "vertices", "blas_nodes", "blas_triangles", "blas_descs", "blas_instances", "meshes", "mesh_transforms"):
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
    assert a.blas_stack_size == b.blas_stack_size
    assert [dict(i) for i in a.build_info] == [dict(i) for i in b.build_info]
    if cached:
        names = sorted(os.listdir(tmp_path / "host"))
        assert names and names == sorted(os.listdir(tmp_path / "device"))
        for n in names:
            assert (tmp_path / "host" / n).read_bytes() == (tmp_path / "device" / n).read_bytes()
        c = host.Scene().add(*scenes.multi_blas_models(), blas_batch_builder=pt.BuildBlases, **kw("device"))   # all from the cache
        assert c.blas_nodes.tobytes() == a.blas_nodes.tobytes() and all(i["from_cache"] for i in c.build_info)
