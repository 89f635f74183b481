"""VXGI passes (BASELINE.json configs[4]): CPU oracle sanity (not gpu) and CUDA vs oracle parity (gpu)."""
import numpy as np
import pytest

import oracle_lib as ol
from idkengine_b200 import scenes, vxgi

GRID_MIN, GRID_MAX = (-1.2, -0.2, -1.2), (1.2, 2.2, 1.2)


def lit_cornell():
    scene, cam = scenes.cornell_1k(threads=1)
    scene.add_light((0.0, 1.6, 0.3), (6.0, 5.5, 5.0), 0.2)
    scene.add_light((-0.6, 0.5, 0.6), (0.5, 0.8, 3.0), 0.1)
    return scene, cam


def test_half_conversion_and_log2():
    L = ol.lib()
    x = np.concatenate([np.linspace(0, 70000, 20001), 10.0 ** np.linspace(-9, 5, 3001), [65504, 65519.9, 65520, 1e-8, 6e-8, 5.96e-8, 2.98e-8]]).astype(np.float32)
    h, back = np.zeros(len(x), np.uint16), np.zeros(len(x), np.float32)
    L.oracle_half_roundtrip(x.ctypes.data, len(x), h.ctypes.data, back.ctypes.data)
    with np.errstate(over="ignore"):
        ref = x.astype(np.float16)
    assert np.array_equal(h, ref.view(np.uint16))
    assert np.array_equal(back, ref.astype(np.float32))
    v = np.linspace(1.0, 600.0, 50001).astype(np.float32)
    y = np.zeros_like(v)
    L.oracle_det_log2(v.ctypes.data, len(v), y.ctypes.data)
    assert np.abs(y - np.log2(v.astype(np.float64))).max() < 2e-6


def test_oracle_voxelize_and_mip_properties():
    scene, cam = lit_cornell()
    ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    assert [l.shape[0] for l in levels] == [48, 24, 12, 6, 3, 1]
    l0 = levels[0].astype(np.float32)
    occ = l0[..., 3] == 1.0
    assert frags >= occ.sum() > 48 * 48          # at least the walls
    assert np.all(l0[~occ] == 0) and np.all(l0[occ][:, :3] >= 0)
    # floor (y ~ 0) and back wall (z ~ -1) are solid slabs of voxels
    y0 = int((0.0 - GRID_MIN[1]) / (GRID_MAX[1] - GRID_MIN[1]) * 48)
    assert occ[8:40, y0 - 1:y0 + 1, 8:40].any(axis=1).mean() > 0.95   # the plane sits on a voxel boundary
    # the emitter voxels are the brightest
    assert l0[..., :3].max() > 10.0
    # every mip level = Mipmap/compute.glsl in float64 of the level below, to 1 ulp (tests/test_vxgi_ref.py has the odd shapes)
    import vxgi_ref64
    for l in range(1, len(levels)):
        want = vxgi_ref64.mip64(levels[l - 1], vxgi_ref64.level_sizes((48, 48, 48))[l])
        assert vxgi_ref64.half_ulp_distance(want, levels[l]).max() <= 1.0, f"level {l}"
    assert levels[1].astype(np.float32)[..., 3].max() <= 1.0
    assert 0 < levels[-1].astype(np.float32)[0, 0, 0, 3] < 1


@pytest.mark.parametrize("which", ["cornell", "atrium"])
def test_oracle_raster_rule_is_close_to_gl_top_left_rule(which):
    """The product's coverage rule (fp32 edge functions, inclusive boundaries) against a model of the GL rasteriser the reference
    runs on (1/256-pixel snapping, exact integer edges, top-left fill rule): the merge is a per-voxel max, so a sample that both
    neighbours of a shared edge cover is harmless; what remains are samples within 1/512 pixel of a silhouette edge.
    Measured (DESIGN section 7): 384^3 bench atrium 114 of 321,400 occupied voxels differ in occupancy, 7 in value."""
    if which == "cornell":
        scene, cam = lit_cornell()
        ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    else:
        scene, cam = scenes.atrium(20000)
        scene.lights = scene.lights[:0]
        scene.add_light((0.0, 6.0, 0.0), (40.0, 38.0, 30.0), 0.3)
        ci = vxgi.create_info(128)
    ours, _, frags_ours = ol.vx_voxelize(scene, ci, raster_rule=0)
    gl, _, frags_gl = ol.vx_voxelize(scene, ci, raster_rule=1)
    a, b = ours[0].view(np.uint16), gl[0].view(np.uint16)
    occ_a, occ_b = a[..., 3] != 0, b[..., 3] != 0
    both = occ_a & occ_b
    occupancy_diff = int((occ_a ^ occ_b).sum())
    value_diff = int((a[both] != b[both]).any(axis=1).sum())
    assert occupancy_diff <= 1e-3 * occ_a.sum() and value_diff <= 1e-3 * occ_a.sum(), (occupancy_diff, value_diff, int(occ_a.sum()))
    assert abs(frags_ours - frags_gl) <= 0.03 * frags_ours      # samples exactly on shared edges are rasterised twice by the inclusive rule
    again, _, _ = ol.vx_voxelize(scene, ci)                       # the rule switch does not leak into later calls
    assert np.array_equal(again[0].view(np.uint16), a)


def test_oracle_cone_trace_plausible():
    scene, cam = lit_cornell()
    ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    levels, raw, _ = ol.vx_voxelize(scene, ci)
    w, h = 64, 48
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, mr = ol.synth_gbuffer(scene, frame, w, h)
    out, steps = ol.vx_cone_trace(ci, raw, frame, vxgi.default_cone_settings(), depth, nrg, mr)
    assert np.isfinite(out).all() and steps > w * h
    assert np.all(out[depth < 1.0][:, 3] == 1.0) and np.all(out[depth == 1.0] == 0)
    assert out[..., :3].mean() > 0.01


@pytest.mark.gpu
@pytest.mark.parametrize("size", [48, (40, 56, 32)])
def test_gpu_voxelize_mip_cone_match_oracle(size):
    scene, cam = lit_cornell()
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    w, h = 96, 64
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, mr = ol.synth_gbuffer(scene, frame, w, h)
    st = vxgi.default_cone_settings()
    st.NoiseIndex = 3
    ref, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as vx:
        vx.SetScene(scene)
        s = vx.Render()
        assert s.Fragments == frags
        for l, lv in enumerate(levels):
            g = vx.ReadLevel(l)
            assert np.array_equal(g.view(np.uint16), lv.view(np.uint16)), f"level {l}"
        out, cs = vx.ConeTrace(frame, depth, nrg, mr, st)
        assert cs.ConeSteps == steps
        assert np.array_equal(out, ref)
        s2 = vx.Render()        # re-voxelising clears first: same grid
        assert np.array_equal(vx.ReadLevel(0).view(np.uint16), levels[0].view(np.uint16)) and s2.Fragments == frags


@pytest.mark.gpu
def test_gpu_vxgi_atrium_transformed_scene(atrium_small):
    scene, cam = atrium_small
    scene.lights = scene.lights[:0]
    scene.add_light((0.0, 6.0, 0.0), (40.0, 38.0, 30.0), 0.3)
    ci = vxgi.create_info(64)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    with vxgi.Voxelizer(64) as vx:
        vx.SetScene(scene)
        s = vx.Render()
        assert s.Fragments == frags
        for l, lv in enumerate(levels):
            assert np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"level {l}"


@pytest.mark.gpu
def test_gpu_vxgi_errors():
    scene, cam = lit_cornell()
    with vxgi.Voxelizer(16, GRID_MIN, GRID_MAX) as vx:
        with pytest.raises(vxgi.IdkVxError, match="idkvx_set_scene has not been called"):
            vx.Render()
        scene.lights["PointShadowIndex"][0] = 0
        vx.SetScene(scene)                                     # accepted ...
        with pytest.raises(vxgi.IdkVxError, match="point-shadowed"):
            vx.Render()                                        # ... but needs a shadow tracer to evaluate Visibility()


def test_oracle_point_shadowed_light_darkens_occluded_voxels():
    """fragment.glsl:55-58: a light with PointShadowIndex >= 0 is multiplied by Visibility(). With the shadow-ray substitute the
    voxels behind the tall box (seen from the light) lose that light's contribution; lit voxels keep it exactly."""
    scene, cam = lit_cornell()
    ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    plain = ol.vx_voxelize(scene, ci)[0][0].astype(np.float32)
    scene.lights["PointShadowIndex"][:] = [0, 1]
    shadowed = ol.vx_voxelize(scene, ci)[0][0].astype(np.float32)
    assert np.array_equal(plain[..., 3], shadowed[..., 3])                    # same coverage
    assert (shadowed[..., :3] <= plain[..., :3]).all()
    darker = (shadowed[..., :3] < plain[..., :3]).any(-1)
    occ = plain[..., 3] == 1.0
    assert 0.02 < darker.sum() / occ.sum() < 0.9                              # some voxels are in shadow, many are not
    same = occ & ~darker
    assert np.array_equal(shadowed[same], plain[same])


@pytest.mark.gpu
def test_gpu_point_shadowed_lights_match_oracle():
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = lit_cornell()
    scene.lights["PointShadowIndex"][:] = [0, 1]
    ci = vxgi.create_info((48, 40, 44), GRID_MIN, GRID_MAX)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    with PathTracer(32, 32) as pt, vxgi.Voxelizer((48, 40, 44), GRID_MIN, GRID_MAX) as vx:
        pt.SetScene(scene)
        vx.SetScene(scene)
        vx.SetShadowTracer(pt)
        s = vx.Render()
        assert s.Fragments == frags
        for l, lv in enumerate(levels):
            assert np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"level {l}"
        vx.SetShadowTracer(None)
        with pytest.raises(vxgi.IdkVxError, match="point-shadowed"):
            vx.Render()


# ---- material textures in the voxeliser (BaseColor / Emissive slots, base level, same sampler rules as the path tracer)
TEX_GRID_MIN, TEX_GRID_MAX = (-3.1, -0.1, -3.1), (3.1, 4.1, 3.1)


def test_oracle_voxelize_textured_differs_from_factor_only():
    import copy
    scene, cam = scenes.textured_room(threads=1)
    ci = vxgi.create_info(40, TEX_GRID_MIN, TEX_GRID_MAX)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    plain = copy.deepcopy(scene)
    for f in ("BaseColorTexture", "MetallicRoughnessTexture", "NormalTexture", "EmissiveTexture", "TransmissionTexture"):
        plain.materials[f] = 0
    levels_p, _, frags_p = ol.vx_voxelize(plain, ci)
    assert frags == frags_p                                   # same coverage
    a, b = levels[0].astype(np.float32), levels_p[0].astype(np.float32)
    assert np.array_equal(a[..., 3], b[..., 3])               # same written voxels
    assert not np.array_equal(a[..., :3], b[..., :3])         # different colours
    assert (a[..., :3] <= b[..., :3] + 1e-3).all()            # textures only darken the factor-only albedo / emission here


@pytest.mark.gpu
def test_gpu_voxelize_textured_matches_oracle():
    scene, cam = scenes.textured_room(threads=1)
    ci = vxgi.create_info((48, 40, 56), TEX_GRID_MIN, TEX_GRID_MAX)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    with vxgi.Voxelizer((48, 40, 56), TEX_GRID_MIN, TEX_GRID_MAX) as vx:
        vx.SetScene(scene)
        s = vx.Render()
        assert s.Fragments == frags
        for l, lv in enumerate(levels):
            assert np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"level {l}"
        bad = scenes.textured_room(threads=1)[0]
        bad.materials["EmissiveTexture"][0] = 77
        with pytest.raises(vxgi.IdkVxError, match="texture"):
            vx.SetScene(bad)


@pytest.mark.gpu
def test_gpu_vxgi_slabs_and_row_tiles_equal_single_pass():
    """The multi-GPU decomposition (SURVEY 8e) on one device: two contexts voxelise the two z-slabs, the second slab is copied
    into the first context's grid exactly where the all-gather would put it, the mip chain is built there -- every level equals
    the single-pass grid (and the oracle's); cone-tracing the image in two row tiles equals the single call."""
    import torch
    from idkengine_b200 import multigpu
    scene, cam = lit_cornell()
    size = (40, 56, 30)
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    levels, raw, frags = ol.vx_voxelize(scene, ci)
    w, h = 96, 64
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, mr = ol.synth_gbuffer(scene, frame, w, h)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as a, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as b:
        a.SetScene(scene); b.SetScene(scene)
        d = size[2]
        za, zb = multigpu.slab_range(d, 0, 2), multigpu.slab_range(d, 1, 2)
        assert za == (0, 15) and zb == (15, 30) and multigpu.slab_range(31, 2, 4) == (16, 24)
        a.SetSlab(*za); b.SetSlab(*zb)
        sa, sb = a.Render(), b.Render()
        assert sa.Fragments + sb.Fragments == frags                    # every fragment lands in exactly one slab
        pa, _ = a.LevelDevicePtr(0)
        pb, nbytes = b.LevelDevicePtr(0)
        ta = torch.as_tensor(multigpu.DeviceArray(pa, (d, size[1] * size[0] * 2), "<i4"), device="cuda")
        tb = torch.as_tensor(multigpu.DeviceArray(pb, (d, size[1] * size[0] * 2), "<i4"), device="cuda")
        assert not ta[zb[0]:].any() and not tb[:zb[0]].any()            # nothing written outside the own slab
        ta[zb[0]:zb[1]].copy_(tb[zb[0]:zb[1]])                          # = the all-gather
        torch.cuda.synchronize()
        a.Mipmap()
        for l, lv in enumerate(levels):
            assert np.array_equal(a.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"level {l}"
        a.SetSlab(0, d)
        full, cs = a.ConeTrace(frame, depth, nrg, mr)
        top, c0 = a.ConeTraceRows(frame, depth[:24], nrg[:24], mr[:24], h, 0)
        bot, c1 = a.ConeTraceRows(frame, depth[24:], nrg[24:], mr[24:], h, 24)
        assert np.array_equal(np.concatenate([top, bot]), full) and c0.ConeSteps + c1.ConeSteps == cs.ConeSteps
        with pytest.raises(vxgi.IdkVxError):
            a.SetSlab(5, 5)
