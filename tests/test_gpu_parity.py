"""GPU parity: libidkpt (through the C ABI) vs the CPU oracle on the same seeded inputs -- bit-exact hit indices,
distances, barycentrics, per-ray work counters, images, AOVs and wavefront state."""
import numpy as np
import pytest

import oracle_lib as ol
from idkengine_b200 import capi, scenes
from idkengine_b200.pathtracer import PathTracer, IdkPtError

pytestmark = pytest.mark.gpu


def feq(a, b):
    """float equality with -0 == +0 (values, not bit patterns)"""
    return np.array_equal(np.asarray(a), np.asarray(b))


def assert_hits_equal(g, o):
    for k in ("T", "BaryX", "BaryY", "TriangleId", "MeshTransformId", "NodePairFetches", "TriangleTests"):
        assert feq(g[k], o[k]), (k, int((g[k] != o[k]).sum()))


def random_rays(n, lo, hi, seed):
    rng = np.random.RandomState(seed)
    o = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return ol.make_rays(o, d)


@pytest.mark.parametrize("name", ["cornell", "multi_blas", "atrium_small"])
def test_trace_rays_bit_exact(name, request):
    scene, cam = request.getfixturevalue(name)
    frame = scenes.camera_frame(cam, 160, 90)
    rays = np.concatenate([ol.gui_test_rays(frame, 160, 90), random_rays(20000, -2.5, 2.5, 11)])
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        g, ms = pt.TraceRays(rays, trace_lights=False)
    assert_hits_equal(g, ol.trace_rays(scene, rays))
    assert (g["TriangleId"] != 0xFFFFFFFF).mean() > 0.3


def test_trace_rays_lights_and_tmax(multi_blas):
    scene, cam = multi_blas
    rays = random_rays(8000, -2.0, 2.0, 5)
    rays["Origin"][:, 1] = np.abs(rays["Origin"][:, 1]) + 0.3
    rays["TMax"][::3] = 1.5
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        g, _ = pt.TraceRays(rays, trace_lights=True)
    o = ol.trace_rays(scene, rays, trace_lights=True)
    assert_hits_equal(g, o)
    assert ((g["TriangleId"] == 0xFFFFFFFF) & (g["T"] < rays["TMax"])).sum() > 0   # some rays hit the light sphere


def run_both(scene, cam, w, h, settings, calls=1, tile=(8, 0, 1), sky=(0.6, 0.7, 0.9)):
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h, settings, tile=tile) as pt:
        pt.SetScene(scene)
        pt.SetSky(sky)
        pt.SetFrame(frame)
        pt.CollectStats = 1
        pt.EnableWavefrontExport(True)
        gstats = [pt.Compute() for _ in range(calls)]
        g = dict(result=pt.Result, albedo=pt.AlbedoTexture, normal=pt.NormalTexture, rays=pt.ReadWavefrontRays(),
                 acc=pt.AccumulatedSamples, stats=gstats)
    res = np.zeros((h, w, 4), np.float32)
    alb, nrm = np.zeros_like(res), np.zeros_like(res)
    acc, ostats, o = 0, [], None
    for _ in range(calls):
        o = ol.path_trace(scene, frame, settings, w, h, sky=sky, tile=tile, accumulated=acc, result=res, albedo=alb, normal=nrm)
        acc = o.accumulated
        ostats.append(o.stats)
    return g, dict(result=res, albedo=alb, normal=nrm, rays=o.rays, acc=acc, stats=ostats)


def assert_same(g, o, aovs=False):
    assert g["acc"] == o["acc"]
    for gs, os_ in zip(g["stats"], o["stats"]):
        assert gs.Rays == os_.Rays
        assert list(gs.BounceRays) == list(os_.BounceRays)
        assert gs.NodePairFetches == os_.NodePairFetches and gs.TriangleTests == os_.TriangleTests
        assert gs.InstanceVisits == os_.InstanceVisits and gs.Hits == os_.Hits
    for k in ("Origin", "PreviousIOROrTraverseCost", "Throughput", "PackedDirectionX", "Radiance", "PackedDirectionY"):
        assert feq(g["rays"][k], o["rays"][k]), (k, int((g["rays"][k] != o["rays"][k]).sum()))
    assert feq(g["result"], o["result"])
    if aovs:
        assert feq(g["albedo"], o["albedo"]) and feq(g["normal"], o["normal"])


def test_path_trace_cornell_config1(cornell):
    """BASELINE.json configs[0] geometry (1k-tri Cornell box, 256x256, 1 spp) through the GPU path."""
    scene, cam = cornell
    s = capi.default_settings()
    g, o = run_both(scene, cam, 256, 256, s)
    assert_same(g, o)
    assert g["stats"][0].Rays > 65536 * 2


def test_path_trace_accumulation_aovs_three_calls(cornell):
    scene, cam = cornell
    s = capi.default_settings()
    s.OutputAOVs = 1
    s.SamplesPerPixel = 2
    g, o = run_both(scene, cam, 200, 120, s, calls=3)
    assert g["acc"] == 6
    assert_same(g, o, aovs=True)


def test_path_trace_no_russian_roulette_depth_9(cornell):
    scene, cam = cornell
    s = capi.default_settings()
    s.Gpu.DoRussianRoulette = 0
    s.RayDepth = 9
    assert_same(*run_both(scene, cam, 128, 128, s))


def test_path_trace_ray_sorting(cornell):
    scene, cam = cornell
    s = capi.default_settings()
    s.DoRaySorting = 1
    s.RayDepth = 6
    s.OutputAOVs = 1
    assert_same(*run_both(scene, cam, 192, 160, s, calls=2), aovs=True)


def test_path_trace_lights_multi_blas_thin_lens(multi_blas):
    scene, cam = multi_blas
    s = capi.default_settings()
    s.Gpu.DoTraceLights = 1
    s.Gpu.LenseRadius = 0.05
    s.Gpu.FocalLength = 4.0
    s.OutputAOVs = 1
    assert_same(*run_both(scene, cam, 160, 96, s, calls=2), aovs=True)


def test_path_trace_cubemap_sky(cornell):
    """SkyBoxManager's samplerCube on ray miss (FirstHit:227, NHit:208): six rgba32f faces instead of a constant."""
    scene, cam = cornell
    rng = np.random.RandomState(9)
    faces = rng.uniform(0.0, 2.0, (6, 16, 16, 4)).astype(np.float32)
    faces[2] *= 3.0          # bright +Y
    s = capi.default_settings()
    s.OutputAOVs = 1
    g, o = run_both(scene, cam, 160, 120, s, calls=2, sky=faces)
    assert_same(g, o, aovs=True)
    g2, _ = run_both(scene, cam, 160, 120, s, calls=2, sky=(0.0, 0.0, 0.0))
    assert not np.array_equal(g["result"], g2["result"])


def test_tlas_traversal(multi_blas):
    """USE_TLAS path (BVHIntersect.glsl:205-272): PLOC TLAS over the three BLAS instances, strict `<` child test, no
    BLAS root test. Closest hits equal the no-TLAS instance loop except for exact-distance ties."""
    scene, cam = scenes.multi_blas(threads=1)
    scene.build_tlas()
    assert len(scene.tlas_nodes) == 5 and scene.use_tlas == 1
    rays = random_rays(12000, -2.5, 2.5, 21)
    rays["Origin"][:, 1] = np.abs(rays["Origin"][:, 1]) + 0.2
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        g, _ = pt.TraceRays(rays, trace_lights=True)
    o = ol.trace_rays(scene, rays, trace_lights=True)
    assert_hits_equal(g, o)
    flat = ol.trace_rays(multi_blas[0], rays, trace_lights=True)
    assert feq(g["T"], flat["T"])
    s = capi.default_settings()
    s.Gpu.DoTraceLights = 1
    assert_same(*run_both(scene, cam, 128, 96, s, calls=2))


def test_tlas_walk_in_the_production_kernel():
    """28 instances -> 55 TLAS nodes. The phase-scheduled kernel (TLAS = 4th phase, default) and the one-ray-per-lane kernel
    (IDKPT_TRAVERSE_VARIANT=1) both equal the oracle: images, wavefront state and S/T/I counters; so do 4 samples in flight."""
    import os
    scene, cam = scenes.instance_grid(3, threads=1)
    assert scene.use_tlas == 1 and len(scene.tlas_nodes) == 2 * len(scene.blas_instances) - 1 == 55
    s = capi.default_settings()
    s.RayDepth = 6
    s.Gpu.DoTraceLights = 1
    w, h = 256, 160
    g, o = run_both(scene, cam, w, h, s, calls=2)
    assert_same(g, o)
    assert g["stats"][0].InstanceVisits > g["stats"][0].Rays // 2    # the walk reaches BLASes for most rays (28 instances, culled by the TLAS)
    os.environ["IDKPT_TRAVERSE_VARIANT"] = "1"
    try:
        g1, _ = run_both(scene, cam, w, h, s, calls=2)
    finally:
        del os.environ["IDKPT_TRAVERSE_VARIANT"]
    assert_same(g1, o)
    frame = scenes.camera_frame(cam, w, h)
    with PathTracer(w, h, s, lanes=4) as pt:
        pt.SetScene(scene); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
        pt.ComputeAsync(); pt.ComputeAsync()
        pt.Sync()
        assert feq(pt.Result, o["result"])


def test_tlas_deeper_than_the_walk_stack_is_rejected():
    """The TLAS walk has a fixed 24-entry stack (BVHIntersect.glsl:4). A host TLAS that needs more (here a 27-deep chain over 28
    instances) is an error at hand-over, not a device fault later."""
    from idkengine_b200 import gpu_types as gt
    scene, cam = scenes.instance_grid(3, threads=1)
    n = len(scene.blas_instances)
    good = scene.tlas_nodes
    chain = np.zeros(2 * n - 1, gt.GpuTlasNode)
    lo, hi = good["Min"][0], good["Max"][0]
    for k in range(n - 1):                      # node 2k: internal with children (2k+1 = leaf k, 2k+2 = rest of the chain)
        chain["Min"][2 * k], chain["Max"][2 * k] = lo, hi
        chain["IsLeafAndChildOrInstanceId"][2 * k] = 2 * k + 1
        chain["Min"][2 * k + 1], chain["Max"][2 * k + 1] = lo, hi
        chain["IsLeafAndChildOrInstanceId"][2 * k + 1] = 0x80000000 | k
    chain["Min"][2 * n - 2], chain["Max"][2 * n - 2] = lo, hi
    chain["IsLeafAndChildOrInstanceId"][2 * n - 2] = 0x80000000 | (n - 1)
    with PathTracer(32, 32) as pt:
        pt.SetScene(scene)                       # the PLOC tree is fine
        with pytest.raises(IdkPtError, match="deeper"):
            pt.UpdateRange(capi.IDKPT_ARRAY_TLAS_NODES, 0, chain)
        scene.tlas_nodes = chain
        with pytest.raises(IdkPtError, match="deeper"):
            pt.SetScene(scene)


def test_compaction_epoch_wraps_without_hanging(cornell):
    """The decoupled look-back's status words carry a 30-bit epoch; a long-running renderer wraps it (advisor finding,
    round 1: the kernel used to spin forever). IDKPT_DEBUG_EPOCH_START puts a fresh context 6 compactions before the wrap."""
    import os
    scene, cam = cornell
    s = capi.default_settings()
    s.RayDepth = 6
    os.environ["IDKPT_DEBUG_EPOCH_START"] = str(0x3FFFFFFF - 6)
    try:
        g, o = run_both(scene, cam, 160, 120, s, calls=4)      # 20 compactions on lane 0: crosses the wrap
        assert_same(g, o)
        frame = scenes.camera_frame(cam, 160, 120)
        with PathTracer(160, 120, s, lanes=3) as pt:            # every lane wraps on its own stream
            pt.SetScene(scene); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
            for _ in range(4):
                pt.ComputeAsync()
            pt.Sync()
            assert feq(pt.Result, o["result"])
    finally:
        del os.environ["IDKPT_DEBUG_EPOCH_START"]


def test_path_trace_debug_traversal(cornell):
    scene, cam = cornell
    s = capi.default_settings()
    s.Gpu.DoDebugBVHTraversal = 1
    g, o = run_both(scene, cam, 128, 96, s)
    assert_same(g, o)
    assert g["result"][..., :3].max() > 0.2


def test_path_trace_atrium_transform_masks_glass(atrium_small):
    scene, cam = atrium_small
    s = capi.default_settings()
    s.RayDepth = 8
    assert_same(*run_both(scene, cam, 240, 136, s, calls=2))


def test_path_trace_odd_size_and_tiles(cornell):
    scene, cam = cornell
    s = capi.default_settings()
    s.RayDepth = 5
    w, h = 203, 117     # not multiples of 8: partial work groups + a partial last swizzle column
    assert_same(*run_both(scene, cam, w, h, s))
    img_g = np.zeros((h, w, 4), np.float32)
    for t in range(3):
        g, o = run_both(scene, cam, w, h, s, tile=(8, t, 3))
        assert_same(g, o)
        rows = g["result"][..., 3] == 1.0
        img_g[rows] = g["result"][rows]
    assert np.all(img_g[..., 3] == 1.0)


def test_large_config_properties():
    """BASELINE.json configs[1] scale (262k triangles, 1920x1080): size-independent properties + sampled parity."""
    scene, cam = scenes.atrium(262144)
    w, h = 1920, 1080
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.RayDepth = 5
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        pt.CollectStats = 1
        st = pt.Compute()
        img1 = pt.Result
        pt.ResetAccumulation()
        st2 = pt.Compute()
        img2 = pt.Result
        # determinism: identical image and counters on a re-run
        assert np.array_equal(img1, img2) and st.NodePairFetches == st2.NodePairFetches
        b = list(st.BounceRays)[:5]
        assert b[0] == w * h and all(b[i] >= b[i + 1] for i in range(4)) and st.Rays == sum(b)
        assert np.isfinite(img1).all() and np.all(img1[..., 3] == 1.0)
        # sampled bit-exact parity of the traversal at full scale
        rays = ol.gui_test_rays(frame, w, h)[::199].copy()
        g, _ = pt.TraceRays(rays)
        assert_hits_equal(g, ol.trace_rays(scene, rays))
        # re-tracing from the hit point backwards along the ray finds the same triangle (closest-hit consistency)
        hit = g["TriangleId"] != 0xFFFFFFFF
        back = rays[hit].copy()
        back["TMax"] = g["T"][hit] * np.float32(1.0001) + np.float32(1e-4)
        g2, _ = pt.TraceRays(back)
        assert feq(g2["T"], g["T"][hit])
        ta, tb = scene.blas_triangles[g2["TriangleId"]], scene.blas_triangles[g["TriangleId"][hit]]
        # same triangle up to presplit duplicates / exact-distance ties (a shorter TMax changes which duplicate is met first)
        assert ((ta["X"] != tb["X"]) | (ta["Y"] != tb["Y"]) | (ta["Z"] != tb["Z"])).mean() < 0.01
    # sampled parity of the full path tracer: a 1920-wide, 16-row band traced as its own tile on both sides
    band = (8, 33, 67)   # stripe 8, tile 33 of 67 -> rows 264..271, 800..807 (2 stripes)
    g, o = run_both(scene, cam, w, h, s, tile=band)
    assert_same(g, o)


def test_treelet_and_kernel_variants_agree(atrium_small):
    """Developer knobs select other code paths (plain loop everywhere, phase-scheduled everywhere, TMA-staged treelet with
    the BFS-first node re-layout): every one of them must reproduce the oracle bit for bit."""
    import os
    scene, cam = atrium_small
    s = capi.default_settings()
    s.RayDepth = 5
    rays = random_rays(6000, -6.0, 6.0, 31)
    ref = ol.trace_rays(scene, rays)
    for env in ({"IDKPT_TRAVERSE_VARIANT": "1"}, {"IDKPT_TRAVERSE_VARIANT": "2"},
                {"IDKPT_TRAVERSE_VARIANT": "2", "IDKPT_TREELET_PAIRS": "192"}, {"IDKPT_TREELET_PAIRS": "5"},
                {"IDKPT_TRAVERSE_VARIANT": "2", "IDKPT_TREELET_PAIRS": "100000"}):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            assert_same(*run_both(scene, cam, 160, 96, s))
            with PathTracer(32, 32) as pt:
                pt.SetScene(scene)
                g, _ = pt.TraceRays(rays)
            assert_hits_equal(g, ref)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v


def test_errors(cornell):
    scene, cam = cornell
    with PathTracer(32, 32) as pt:
        pt.SetFrame(scenes.camera_frame(cam, 32, 32))
        with pytest.raises(IdkPtError, match="idkpt_set_scene has not been called"):
            pt.Compute()
        pt.SetScene(scene)
        pt.RayDepth = 0
        with pytest.raises(IdkPtError, match="RayDepth"):
            pt.Compute()
        pt.RayDepth = 3
        pt.Compute()
        assert pt.AccumulatedSamples == 1
        pt.FocalLength = 5.0                      # setters reset the accumulation (PathTracer.cs:39-48)
        assert pt.AccumulatedSamples == 0
        bad = scenes.cornell_1k(threads=1)[0]
        bad.blas_descs["NodeCount"][0] += 1000
        with pytest.raises(IdkPtError, match="GpuBlasDesc range"):
            pt.SetScene(bad)
        bad = scenes.cornell_1k(threads=1)[0]
        interior = [i for i in range(10, len(bad.blas_nodes)) if bad.blas_nodes["TriCount"][i] == 0][0]
        bad.blas_nodes["TriStartOrChild"][interior] = 4        # points back up the tree: a cycle
        with pytest.raises(IdkPtError, match="DFS order|child index"):
            pt.SetScene(bad)
        bad = scenes.cornell_1k(threads=1)[0]
        bad.blas_stack_size = 3                                # smaller than the tree needs
        bad.blas_descs["RequiredStackSize"][0] = 3
        with pytest.raises(IdkPtError, match="traversal stack"):
            pt.SetScene(bad)
    with pytest.raises(IdkPtError, match="device ordinal"):
        PathTracer(32, 32, device=99)


def test_update_range_materials_meshes_transforms(multi_blas):
    """Dirty-range edits (ModelManager.cs:236-261): material / mesh / transform changes reach the kernels."""
    scene, cam = scenes.multi_blas(threads=1)
    s = capi.default_settings()
    s.RayDepth = 4
    frame = scenes.camera_frame(cam, 96, 64)
    with PathTracer(96, 64, s) as pt:
        pt.SetScene(scene)
        pt.SetFrame(frame)
        pt.Compute()
        scene.materials["BaseColorFactor"][2] = 0xFF2040F0
        scene.materials["MetallicFactor"][2] = 0.9
        pt.UpdateRange(capi.IDKPT_ARRAY_MATERIALS, 2, scene.materials[2:3])
        scene.meshes["EmissiveBias"][0] = 0.7
        scene.meshes["RoughnessBias"][2] = -0.4
        pt.UpdateRange(capi.IDKPT_ARRAY_MESHES, 0, scene.meshes)
        from idkengine_b200.host import mesh_transform, trs_matrix
        scene.mesh_transforms[1] = mesh_transform(trs_matrix(0.9, 30.0, (-1.0, 0.9, 0.2)))[0]
        pt.UpdateRange(capi.IDKPT_ARRAY_MESH_TRANSFORMS, 1, scene.mesh_transforms[1:2])
        assert pt.AccumulatedSamples == 0
        pt.Compute()
        img = pt.Result
    o = ol.path_trace(scene, frame, s, 96, 64, sky=(0, 0, 0))
    assert feq(img, o.result)


def test_present_async_matches_read_result(cornell):
    import torch
    scene, cam = cornell
    w, h = 160, 96
    bufs = [torch.zeros((h, w, 4), dtype=torch.float32).pin_memory() for _ in range(2)]
    with PathTracer(w, h) as pt:
        pt.SetScene(scene)
        pt.SetFrame(scenes.camera_frame(cam, w, h))
        imgs = []
        for k in range(4):
            pt.Compute()
            pt.PresentAsync(bufs[k & 1].data_ptr(), bufs[k & 1].numel() * 4)
            if k >= 1:
                pass
            imgs.append(pt.Result)            # synchronous read of the same frame
            pt.PresentWait()
            assert np.array_equal(bufs[k & 1].numpy(), imgs[-1])
        # pipelined use: present k overlaps compute k+1
        pt.ResetAccumulation()
        for k in range(4):
            pt.Compute()
            pt.PresentAsync(bufs[k & 1].data_ptr(), bufs[k & 1].numel() * 4)
        pt.PresentWait()
        assert np.array_equal(bufs[1].numpy(), imgs[3])


def test_resize_and_snapshot_restore(cornell):
    scene, cam = cornell
    s = capi.default_settings()
    with PathTracer(64, 64, s) as pt:
        pt.SetScene(scene)
        pt.SetFrame(scenes.camera_frame(cam, 64, 64))
        pt.Compute(); pt.Compute()
        snap, n = pt.Result, pt.AccumulatedSamples
        pt.Compute()
        third = pt.Result
        pt.WriteResult(snap, accumulated=n)       # checkpoint / resume of the accumulation (SURVEY.md section 5)
        pt.Compute()
        assert np.array_equal(pt.Result, third)
        pt.SetSize(96, 48)
        assert pt.AccumulatedSamples == 0
        pt.SetFrame(scenes.camera_frame(cam, 96, 48))
        pt.Compute()
        o = ol.path_trace(scene, scenes.camera_frame(cam, 96, 48), s, 96, 48, sky=(0, 0, 0))
        assert feq(pt.Result, o.result)


def test_multi_gpu_peer_gather():
    """Fused FinalDraw + NVLink peer-memory gather vs NCCL all-gather vs per-tile oracle (needs >= 2 GPUs; skipped
    on a single-GPU machine)."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                          "--master-port", "29541", os.path.join(repo, "scripts", "check_peer_gather.py")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "PEER_GATHER_OK" in out.stdout, out.stdout[-1000:] + out.stderr[-2000:]


@pytest.mark.parametrize("world,epoch_start", [(2, None), (3, None), (2, "0xFFFFFFF8")])
def test_global_slots_tiles_equal_one_gpu_image(world, epoch_start):
    """SURVEY 8e option (ii), strict multi-GPU parity: `world` tile contexts with IDKPT_CREATE_GLOBAL_SLOTS, wired to each other
    in one process by idkpt_gather_connect (so this runs on a single-GPU box, through the same peer-memory scatter / arrival
    wait / per-bounce slot exchange kernels the multi-process path uses), reproduce the untiled image bit for bit -- in their
    own rows and in every context's gathered frame -- while the default tile-local numbering does not."""
    import json
    import os
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32", IDKPT_GATHER_TIMEOUT_MS="3000")   # fresh process: enough hardware queues for all streams
    if epoch_start:      # the 32-bit exchange epoch wraps inside the run (successor of 0xFFFFFFFF is 2: parity keeps alternating, 0 stays "unpublished")
        env["IDKPT_DEBUG_SLOT_EPOCH_START"] = epoch_start
    out = subprocess.run([sys.executable, os.path.join(repo, "scripts", "check_global_slots.py"), "--world", str(world)],
                         capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stdout[-1500:] + out.stderr[-2500:]
    rec = json.loads(out.stdout.strip().splitlines()[-1])
    assert rec["ok"] and rec["tiles_eq_one_gpu"] and all(rec["gathered_eq_one_gpu"]) and rec["control_local_slots_differ"], rec


# ---- scope table 8f.1: any-hit traversal and ray-traced shadows ---------------------------------------------------

@pytest.mark.parametrize("name", ["cornell", "multi_blas", "atrium_small"])
def test_trace_rays_any_bit_exact(name, request):
    scene, cam = request.getfixturevalue(name)
    frame = scenes.camera_frame(cam, 160, 90)
    rays = np.concatenate([ol.gui_test_rays(frame, 160, 90), random_rays(20000, -2.5, 2.5, 13)])
    rays["TMax"][::4] = 2.0
    for lights in (False, True):
        with PathTracer(64, 64) as pt:
            pt.SetScene(scene)
            g, _ = pt.TraceRaysAny(rays, trace_lights=lights)
            closest, _ = pt.TraceRays(rays, trace_lights=lights)
        o = ol.trace_rays_any(scene, rays, trace_lights=lights)
        for f in ("T", "TriangleId", "MeshTransformId", "NodePairFetches"):
            assert np.array_equal(g[f], o[f]), f
        for f in ("BaryX", "BaryY"):
            assert np.array_equal(g[f].view(np.uint32), o[f].view(np.uint32)), f
        # occluded exactly when the closest-hit query finds something in range
        assert np.array_equal(g["NodePairFetches"] == 1, closest["T"] != rays["TMax"])
        assert 0.2 < (g["NodePairFetches"] == 1).mean() < 1.0


def test_trace_rays_any_tlas():
    scene, cam = scenes.multi_blas(threads=1)
    scene.build_tlas()
    rays = random_rays(20000, -2.5, 2.5, 17)
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        g, _ = pt.TraceRaysAny(rays)
    o = ol.trace_rays_any(scene, rays)
    for f in ("T", "TriangleId", "MeshTransformId", "NodePairFetches"):
        assert np.array_equal(g[f], o[f]), f


@pytest.mark.parametrize("name,samples", [("cornell", 1), ("multi_blas", 4)])
def test_shadows_ray_traced_bit_exact(name, samples):
    scene, cam = scenes.cornell_1k(threads=1) if name == "cornell" else scenes.multi_blas(threads=1)
    if len(scene.lights) == 0:
        scene.add_light((0.0, 1.6, 0.0), (20.0, 20.0, 20.0), 0.15)
    w, h = 192, 128
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, _ = ol.synth_gbuffer(scene, frame, w, h)
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        g, ms = pt.ShadowsRayTraced(frame, depth, nrg, 0, samples=samples, noise_index=3 * samples)
    o = ol.shadows_ray_traced(scene, frame, depth, nrg, 0, samples=samples, noise_index=3 * samples)
    assert np.array_equal(g.view(np.uint32), o.view(np.uint32))
    lit = g[depth < 1.0]
    assert (lit == 0.0).any() and (lit == 1.0).any()      # both shadowed and lit pixels exist


def test_shadows_errors(cornell):
    scene, cam = cornell
    frame = scenes.camera_frame(cam, 32, 32)
    with PathTracer(32, 32) as pt:
        pt.SetScene(scene)
        with pytest.raises(RuntimeError):
            pt.ShadowsRayTraced(frame, np.ones((32, 32), np.float32), np.zeros((32, 32, 2), np.float32), 99)
