"""Traversal and the wavefront pipeline at their edges, on the GPU, against the CPU oracle (bit-exact) and the float64
reference of tests/edge_lib.py:

  A  TraceRays / TraceRaysAny on the edge battery (lights on and off), batch sizes 0, 1, 31, 32, 33 and large counts that
     are not multiples of 32, the slab-test artefact class (0 * inf = NaN), and the leak rate of a closed box.
  B  wavefront counts: no alive ray after the first hit, a count that falls to zero mid-path, RayDepth 1 and 64, frame
     sizes around the 8x8 groups and the 20-column swizzle, alive counts around the 2048-entry tiles, a tile with no rows,
     a partial last stripe.
  C  full-frame ray sorting above the grid-stride threshold of the sort kernels (4 * SMs * 2048 alive rays).

Every test also asserts that it reached its edge."""
import ctypes
import os

import numpy as np
import pytest

import edge_lib as el
import oracle_lib as ol
from idkengine_b200 import capi, scenes
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import PathTracer

from test_gpu_parity import assert_same, feq, run_both

pytestmark = pytest.mark.gpu

SKY = (0.6, 0.7, 0.9)
THREADS = os.cpu_count() or 1
HIT_FIELDS = ("T", "TriangleId", "MeshTransformId", "NodePairFetches", "TriangleTests")


def assert_bits_equal(g, o):
    for k in HIT_FIELDS:
        assert np.array_equal(g[k].view(np.uint32), o[k].view(np.uint32)), (k, int((g[k].view(np.uint32) != o[k].view(np.uint32)).sum()))
    for k in ("BaryX", "BaryY"):
        assert np.array_equal(g[k].view(np.uint32), o[k].view(np.uint32)), k


@pytest.fixture(scope="module")
def multi_blas_tlas():
    scene, cam = scenes.multi_blas(threads=1)
    scene.build_tlas()
    return scene, cam


# ------------------------------------------------------------------------------------------------ A: traversal edges
@pytest.mark.parametrize("name", ["cornell", "multi_blas", "multi_blas_tlas", "atrium_small"])
def test_edge_battery_gpu_equals_oracle_and_float64(name, request):
    scene, _ = request.getfixturevalue(name)
    tris = el.world_triangles(scene)
    rays = np.concatenate([el.edge_rays(scene, 7, tris=tris), el.random_rays(20000, scene, 8, tris=tris)])
    art = el.artefact_class(scene, rays)
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        for lights in (False, True):
            if lights is False or len(scene.lights):
                ref = el.ref64_closest(scene, rays, trace_lights=lights, tris=tris)
            for any_hit in (False, True):
                g, _ = (pt.TraceRaysAny if any_hit else pt.TraceRays)(rays, trace_lights=lights)
                o = (ol.trace_rays_any if any_hit else ol.trace_rays)(scene, rays, trace_lights=lights)
                if any_hit:      # the any-hit query reports no work counters
                    g["TriangleTests"] = o["TriangleTests"] = 0
                assert_bits_equal(g, o)
                cg, co = el.classify(scene, rays, g, ref, any_hit), el.classify(scene, rays, o, ref, any_hit)
                print(f"{name} lights={lights} any={any_hit}: robust hits {len(cg['robust_hit'])}, robust misses "
                      f"{len(cg['robust_miss'])}, artefact class {len(cg['artefact'])}, culled {len(cg['culled'])}")
                assert len(cg["bad"]) == 0, cg["bad"][:10]
                assert np.array_equal(cg["culled"], co["culled"])     # the GPU culls exactly the rays the oracle culls
    assert art.sum() >= 50


@pytest.mark.parametrize("count", [0, 1, 31, 32, 33, 4097, 100_003, 262_147])
def test_trace_batch_sizes(cornell, count):
    """Partial warps in the ticket loop and the persistent-grid tail: any count equals the oracle. Count 0 returns OK and
    writes nothing."""
    scene, _ = cornell
    rays = el.random_rays(max(count, 1), scene, 1000 + count)[:count]
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        if count == 0:
            hits = np.frombuffer(np.full(gt.IdkPtHit.itemsize * 2, 0xAB, np.uint8).tobytes(), gt.IdkPtHit).copy()
            before = hits.tobytes()
            ms = ctypes.c_float(-1.0)
            one = el.random_rays(1, scene, 5)
            for fn in (pt._lib.idkpt_trace_rays, pt._lib.idkpt_trace_rays_any):
                assert fn(pt._ctx, one.ctypes.data, 0, 0, hits.ctypes.data, ctypes.byref(ms)) == 0
            assert hits.tobytes() == before
            return
        for any_hit in (False, True):
            g, _ = (pt.TraceRaysAny if any_hit else pt.TraceRays)(rays)
            o = (ol.trace_rays_any if any_hit else ol.trace_rays)(scene, rays)
            if any_hit:
                g["TriangleTests"] = o["TriangleTests"] = 0
            assert_bits_equal(g, o)


def test_closed_box_leak_rate():
    """Rays from inside a closed box at its 12 edges and 8 corners all hit in exact arithmetic. The intersector is not
    watertight (a ray through a shared edge can fail both triangles' barycentric tests), so some slip through: the GPU
    leaks exactly the rays the oracle leaks, and the rate stays pinned."""
    rates = []
    for sub in (1, 4):
        scene, _ = scenes.closed_box(sub, threads=1)
        rays = el.box_leak_rays((-1, 0, -1), (1, 2, 1))
        with PathTracer(64, 64) as pt:
            pt.SetScene(scene)
            g, _ = pt.TraceRays(rays)
        o = ol.trace_rays(scene, rays)
        assert_bits_equal(g, o)
        leaks = int((g["TriangleId"] == el.MISS).sum())
        rates.append(leaks / len(rays))
        print(f"closed_box({sub}): {leaks} of {len(rays)} edge / corner rays leak")
    assert rates[0] == 38 / 696 and rates[1] == 54 / 696, rates


# ------------------------------------------------------------------------------------------------ B: wavefront counts
def box_settings(depth=9, sorting=0, aovs=0, spp=1):
    s = capi.default_settings()
    s.RayDepth, s.DoRaySorting, s.OutputAOVs, s.SamplesPerPixel = depth, sorting, aovs, spp
    s.Gpu.DoRussianRoulette = 0
    return s


@pytest.fixture(scope="module")
def box12():
    return scenes.closed_box(1, threads=1)


@pytest.mark.parametrize("sky", ["constant", "cubemap"])
def test_no_alive_rays_after_the_first_hit(cornell, sky):
    """Camera outside the Cornell box, looking away: every primary ray misses, so compaction, the sort and the traversal
    of bounces 1.. all run on zero rays."""
    scene, cam = cornell
    away = scenes.camera_away(cam)
    faces = np.random.RandomState(3).uniform(0.0, 2.0, (6, 8, 8, 4)).astype(np.float32) if sky == "cubemap" else SKY
    for s in (box_settings(6, sorting=1, aovs=1), box_settings(6, sorting=0, spp=2)):
        g, o = run_both(scene, away, 96, 64, s, calls=2, sky=faces)
        assert_same(g, o, aovs=True)
        for st in g["stats"]:
            b = list(st.BounceRays)
            assert b[0] == 96 * 64 * s.SamplesPerPixel and not any(b[1:]), b
        assert st.Hits == 0
        if sky == "constant":
            assert np.all(g["result"][..., :3] == np.array(SKY, np.float32))
    frame = scenes.camera_frame(away, 96, 64)
    s = box_settings(6, sorting=1)
    with PathTracer(96, 64, s, lanes=3) as pt:
        pt.SetScene(scene); pt.SetSky(faces); pt.SetFrame(frame)
        for _ in range(4):
            pt.ComputeAsync()
        pt.Sync()
        img = pt.Result
    acc, res = 0, np.zeros((64, 96, 4), np.float32)
    for _ in range(4):
        acc = ol.path_trace(scene, frame, s, 96, 64, sky=faces, accumulated=acc, result=res).accumulated
    assert feq(img, res)


def test_alive_count_falls_to_zero_mid_path():
    scene, cam = scenes.open_floor(threads=1)
    for sorting in (0, 1):
        g, o = run_both(scene, cam, 80, 48, box_settings(9, sorting=sorting, aovs=1))
        assert_same(g, o, aovs=True)
        b = list(g["stats"][0].BounceRays)[:9]
        assert b[0] == b[1] == 80 * 48 and b[2] == 0 and not any(b[2:]), b


@pytest.mark.parametrize("depth", [1, capi.IDKPT_MAX_RAY_DEPTH])
def test_ray_depth_extremes_in_the_closed_box(box12, depth):
    scene, cam = box12
    for sorting in (0, 1):
        g, o = run_both(scene, cam, 48, 40, box_settings(depth, sorting=sorting, aovs=1))
        assert_same(g, o, aovs=True)
        b = list(g["stats"][0].BounceRays)
        assert b[0] == 48 * 40 and not any(b[depth:]), b
        assert b[depth - 1] > 0.99 * 48 * 40     # the deepest counts / tickets slot is in use


@pytest.mark.parametrize("w,h", [(1, 1), (1, 9), (9, 1), (7, 7), (8, 8), (152, 8), (160, 8), (168, 16), (8, 200)])
def test_frame_sizes_around_groups_and_swizzle(box12, w, h):
    """k_raygen's ReorderInvocations(20): no full 20-group column (width < 160), exactly 20 columns, a last column one group
    wide; partial 8x8 groups."""
    scene, cam = box12
    g, o = run_both(scene, cam, w, h, box_settings(4, sorting=1, aovs=1), calls=2)
    assert_same(g, o, aovs=True)
    assert list(g["stats"][0].BounceRays)[0] == w * h


@pytest.mark.parametrize("w,h", [(89, 23), (64, 32), (683, 3), (45, 91), (241, 17)])
def test_alive_counts_around_the_2048_tiles(box12, w, h):
    """n = 2047, 2048, 2049, 4095, 4097 alive rays: the k_compact and k_sort_* tile boundaries."""
    scene, cam = box12
    n = w * h
    for sorting in (0, 1):
        g, o = run_both(scene, cam, w, h, box_settings(6, sorting=sorting))
        assert_same(g, o)
        b = list(g["stats"][0].BounceRays)[:6]
        assert b[0] == n and all(x >= 0.999 * n for x in b), b


@pytest.mark.parametrize("h", [8, 16])
def test_tile_that_owns_no_rows(cornell, h):
    """tile (8, 2, 3) of an 8- or 16-row image owns no stripe: Compute / ComputeAsync only count the sample, the image is
    untouched, TileRows() is empty, PresentAsync copies nothing."""
    import torch
    scene, cam = cornell
    w = 64
    s = capi.default_settings()
    with PathTracer(w, h, s, tile=(8, 2, 3), lanes=2) as pt:
        assert len(pt.TileRows()) == 0
        pt.SetScene(scene); pt.SetSky(SKY); pt.SetFrame(scenes.camera_frame(cam, w, h))
        pt.CollectStats = 1
        st = pt.Compute()
        assert st.Rays == 0 and not any(st.BounceRays) and pt.AccumulatedSamples == 1
        pt.CollectStats = 0
        pt.ComputeAsync(); pt.ComputeAsync()
        pt.Sync()
        assert pt.AccumulatedSamples == 3
        assert not pt.Result.any()
        buf = torch.full((h, w, 4), 7.0, dtype=torch.float32).pin_memory()
        pt.PresentAsync(buf.data_ptr(), buf.numel() * 4)
        pt.PresentWait()
        assert bool((buf == 7.0).all())
    o = ol.path_trace(scene, scenes.camera_frame(cam, w, h), s, w, h, sky=SKY, tile=(8, 2, 3))
    assert o.stats.Rays == 0 and not o.result.any()


def test_partial_last_stripe_tiles_stitch_to_the_untiled_first_bounce(box12):
    """Height 20 with 8-row stripes: the last stripe has 4 rows. Each of three tiles equals the oracle with the same tile
    map, and their first bounces stitch to the untiled image's."""
    scene, cam = box12
    w, h = 40, 20
    s = box_settings(1, aovs=1)
    full, _ = run_both(scene, cam, w, h, s)
    img = np.zeros((h, w, 4), np.float32)
    for t in range(3):
        g, o = run_both(scene, cam, w, h, s, tile=(8, t, 3))
        assert_same(g, o, aovs=True)
        rows = g["result"][..., 3] == 1.0
        img[rows] = g["result"][rows]
    assert feq(img, full["result"])


# ------------------------------------------------------------------------------------------------ C: full-frame sorting
def sort_threshold():
    import torch
    return 4 * torch.cuda.get_device_properties(0).multi_processor_count * 2048


def full_frame_sorted(scene, cam, s, w=1920, h=1080):
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene); pt.SetSky(SKY); pt.SetFrame(frame)
        pt.CollectStats = 1
        st = pt.Compute()
        img = pt.Result
    with PathTracer(w, h, s, lanes=2) as pt:
        pt.SetScene(scene); pt.SetSky(SKY); pt.SetFrame(frame)
        pt.ComputeAsync()
        pt.Sync()
        img_async = pt.Result
    res = np.zeros((h, w, 4), np.float32)
    o = ol.path_trace(scene, frame, s, w, h, sky=SKY, result=res, want_rays=False, threads=THREADS)
    assert list(st.BounceRays) == list(o.stats.BounceRays) and st.Rays == o.stats.Rays
    assert (st.NodePairFetches, st.TriangleTests, st.InstanceVisits, st.Hits) == \
           (o.stats.NodePairFetches, o.stats.TriangleTests, o.stats.InstanceVisits, o.stats.Hits)
    assert feq(img, res), int((img != res).sum())
    assert feq(img_async, res)
    sorted_counts = list(st.BounceRays)[2:s.RayDepth]
    print(f"sorted bounce counts {sorted_counts}, grid-stride threshold {sort_threshold()}")
    assert max(sorted_counts) > sort_threshold()
    return st


def test_full_frame_sort_few_distinct_keys(box12):
    """12 triangles: ~2.07 M rays per sorted bounce over 12 keys -- long equal-key runs across ~1013 tiles (stability)."""
    scene, cam = box12
    full_frame_sorted(scene, cam, box_settings(9, sorting=1))


def test_full_frame_sort_keys_above_2_pow_21():
    """A closed box of 2.1 M triangles: triangle ids wrap under `key & 0x1FFFFF` and all three 7-bit digits vary."""
    scene, cam = scenes.closed_box(419)
    assert len(scene.blas_triangles) > 1 << 21
    full_frame_sorted(scene, cam, box_settings(9, sorting=1))


def test_full_frame_sort_bench_atrium():
    """atrium-262k (the bench.py scene) with ray sorting and Russian roulette on. At 1920x1080 the first sorted bounce keeps
    only ~843 k rays, below the threshold, so the frame is 2560x1440 (~1.5 M rays in that bounce)."""
    scene, cam = scenes.atrium(262144)
    s = capi.default_settings()
    s.RayDepth, s.DoRaySorting = 9, 1
    full_frame_sorted(scene, cam, s, 2560, 1440)
