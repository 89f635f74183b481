"""The VXGI oracle (oracle/oracle_vxgi.inc) against the float64 restatement of the engine's shaders (tests/vxgi_ref64.py):
level sizes, the mip chain on synthetic level-0 grids at odd shapes and extreme halves, the cone trace on synthetic chains
and on the voxelised Cornell box, and voxelisation. The kernels are pinned to the oracle bit for bit (tests/test_vxgi.py),
so these tests check what the kernels compute against an independent reading of the reference.

Measured bounds (Cornell box with two lights, grid (-1.2, -0.2, -1.2)..(1.2, 2.2, 1.2)):
- mip chain: every texel within 1 float16 ulp of mip64 of the oracle's own level below; of the 37,968 texels of levels 1..5
  of (40, 56, 30), 2 (random), 33 (sparse), 10 (subnormal), 7 (near 65504) and 3 (inf) differ; (7, 3, 129): 4 (sparse) and
  1 (subnormal) of 1,020; the other shapes and fills none.
- cone trace: rgb within 2.6e-4 relative on the pixels whose decision margin is >= 1e-6; 95 % of the covered pixels are
  compared with 64 cones per pixel, more with fewer.
- voxelisation at (40, 56, 30): occupancy equal on every unambiguous voxel, rgb within 1 ulp; 201 of 7,111 occupied voxels
  are touched by an ambiguous sample; at 48^3 the walls lie exactly on voxel planes, which makes their voxels ambiguous."""
import numpy as np
import pytest

import oracle_lib as ol
import vxgi_ref64 as r
from idkengine_b200 import gpu_types as gt, host, scenes, vxgi
from raster_lib import FILLS, GRID_MAX, GRID_MIN, check_voxelized, level0_fill, lit_cornell, synthetic_chain

SKY = (0.6, 0.7, 0.9)

SHAPES = [(1, 1, 1), (1, 1, 2), (3, 1, 7), (5, 33, 2), (40, 56, 30), (384, 384, 384), (2048, 1, 1)]
MIP_SHAPES = [s for s in SHAPES if s != (384, 384, 384)] + [(7, 3, 129), (1, 64, 3)]
def check_chain(levels, shape):
    """Every level of an oracle (or kernel) chain against mip64 of the chain's own level below: within 1 ulp, and at most
    0.1 % of the texels differing at all (at least 4: fp32 rounding moves a texel by one ulp where the exact value lies next
    to a float16 rounding boundary, 4 of the 1,020 texels of the sparse (7, 3, 129) chain). Returns (worst ulp, differing
    texels, texels)."""
    sizes = r.level_sizes(shape)
    assert [lv.shape for lv in levels] == [(d, h, w, 4) for (w, h, d) in sizes]
    worst, ndiff, n = 0.0, 0, 0
    for l in range(1, len(levels)):
        u = r.half_ulp_distance(r.mip64(levels[l - 1], sizes[l]), levels[l])
        worst, ndiff, n = max(worst, float(u.max())), ndiff + int((u > 0).sum()), n + u.size
    assert worst <= 1.0 and ndiff <= max(4, 1e-3 * n), (shape, worst, ndiff, n)
    return worst, ndiff, n


# ---------------------------------------------------------------------------------------------------------- level sizes
@pytest.mark.parametrize("shape", SHAPES)
def test_level_sizes(shape):
    """Texture.GetMaxMipmapLevel = ILogB(max extent) + 1 and GetMipmapLevelSize = max(1, extent >> level), against the
    host's level table and the oracle's level count (the oracle sizes each level by the same rule; test_mip_chain_* checks
    it through the level shapes the chain has)."""
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    sizes = r.level_sizes(shape)
    assert vxgi.level_sizes(ci) == sizes
    assert sizes[-1] == tuple(max(1, s >> (len(sizes) - 1)) for s in shape) and max(sizes[-1]) == 1
    if shape != (384, 384, 384):             # 453 MB of level 0
        levels, _ = ol.vx_mipmap(ci, np.zeros((shape[2], shape[1], shape[0], 4), np.float16))
        assert [lv.shape[:3][::-1] for lv in levels] == sizes
    expected = {(1, 1, 1): 1, (1, 1, 2): 2, (3, 1, 7): 3, (5, 33, 2): 6, (40, 56, 30): 6, (384, 384, 384): 9, (2048, 1, 1): 12}
    assert len(sizes) == expected[shape]


# ---------------------------------------------------------------------------------------------------------- mip chain
@pytest.mark.parametrize("fill", FILLS)
@pytest.mark.parametrize("shape", MIP_SHAPES)
def test_mip_chain_matches_float64(shape, fill):
    """The oracle's k_vx_mipmap rule against Mipmap/compute.glsl in float64, each level from the oracle's own level below.
    inf texels make NaN where a filter weight is exactly 0 (0 * inf) on both sides; NaN == NaN counts as agreement."""
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    levels, _ = ol.vx_mipmap(ci, level0_fill(shape, fill))
    check_chain(levels, shape)
    if fill == "zeros":
        assert all(not lv.view(np.uint16).any() for lv in levels)
    if fill == "inf" and len(levels) > 1:
        # 0 * inf in a filter weight: the oracle stores the canonical NaN 0x7FFF that the device's __float2half_rn writes
        # (it once stored x86's negative default NaN, 0xFE00, and the device chain differed from it bit for bit)
        nan = np.concatenate([lv[np.isnan(lv)] for lv in levels[1:]])
        assert len(nan) and np.all(nan.view(np.uint16) == 0x7FFF)


@pytest.mark.parametrize("value", [0.5, 0.1, 65504.0, 6.0e-8, 3.1e-5])
@pytest.mark.parametrize("shape", [(5, 33, 2), (7, 3, 129), (3, 1, 7)])
def test_mip_chain_of_a_constant_is_that_constant(shape, value):
    """Seven taps of a constant average to it: every level equals a half-representable constant bit for bit."""
    c = np.float16(value)
    w, h, d = shape
    levels, _ = ol.vx_mipmap(vxgi.create_info(shape, GRID_MIN, GRID_MAX), np.full((d, h, w, 4), c, np.float16))
    for lv in levels:
        assert np.array_equal(lv.view(np.uint16), np.full(lv.shape, c, np.float16).view(np.uint16))


@pytest.mark.parametrize("shape,axis", [((64, 6, 5), 0), ((129, 7, 3), 0), ((5, 61, 9), 1), ((6, 3, 67), 2), ((1, 1, 40), 2)])
def test_mip_level1_reproduces_a_ramp(shape, axis):
    """A ramp value = texel index along one axis is linear, so every unclamped tap reads it at its exact position and the
    +-1 taps cancel: level 1's texel x equals the source position of its centre, p = (x + 0.5) * S / s - 0.5, within 1 ulp,
    wherever the taps p - 1 .. p + 2 stay inside the source."""
    w, h, d = shape
    idx = np.meshgrid(np.arange(d), np.arange(h), np.arange(w), indexing="ij")[2 - axis]
    level0 = np.repeat(idx[..., None], 4, -1).astype(np.float16)
    levels, _ = ol.vx_mipmap(vxgi.create_info(shape, GRID_MIN, GRID_MAX), level0)
    S, s = shape[axis], levels[1].shape[2 - axis]
    x = np.arange(s)
    p = (x + 0.5) * S / s - 0.5
    interior = (p - 1 >= 0) & (p + 2 <= S - 1)
    got = np.moveaxis(levels[1][..., 0], 2 - axis, -1)
    want = np.broadcast_to(p.astype(np.float16), got.shape)
    assert interior.sum() >= 2
    u = r.half_ulp_distance(got[..., interior], want[..., interior])
    assert u.max() <= 1.0, (shape, axis, u.max())


def test_oracle_voxelized_chain_matches_float64():
    """The chain of the voxelised Cornell box at the odd grid (40, 56, 30), each level from the oracle's level below."""
    scene, cam = lit_cornell()
    ci = vxgi.create_info((40, 56, 30), GRID_MIN, GRID_MAX)
    levels, _, _ = ol.vx_voxelize(scene, ci)
    check_chain(levels, (40, 56, 30))


# ---------------------------------------------------------------------------------------------------------- cone trace
def cornell_gbuffer(w, h, metal_rough=None, seed=0):
    scene, cam = lit_cornell()
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, mr = ol.synth_gbuffer(scene, frame, w, h)
    rng = np.random.default_rng(seed)
    if metal_rough == "zero":
        mr = np.zeros_like(mr)
    elif metal_rough == "one":
        mr = np.ones_like(mr)
    elif metal_rough == "mirror":
        mr = np.stack([np.ones_like(depth), np.zeros_like(depth)], -1)
    elif metal_rough == "mixed":
        mr = rng.random(mr.shape).astype(np.float32)
        mr[rng.random(depth.shape) < 0.2] = 0.0
        mr[rng.random(depth.shape) < 0.2] = 1.0
    return scene, frame, depth, nrg, mr


def cone_settings(max_samples=4, step_multiplier=0.16, normal_ray_offset=1.0, noise_index=0, gi_boost=1.3, sky_boost=1.0 / 1.3):
    return vxgi.IdkVxConeSettings(max_samples, step_multiplier, gi_boost, sky_boost, normal_ray_offset, noise_index)


def compare_cone_trace(ci, levels, raw, frame, st, depth, nrg, mr, eps=1e-6, rtol=1e-3, min_fraction=0.9):
    """Oracle against indirect_light64: rgb within rtol on the pixels whose decision margin is >= eps, at least min_fraction
    of the covered pixels compared, step totals equal when no pixel is excluded. Returns (oracle image, oracle steps)."""
    out, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr, sky=SKY)
    ref, ref_steps, margin = r.indirect_light64(levels, list(ci.GridMin), list(ci.GridMax), frame, st, depth, nrg, mr, SKY)
    covered = depth != 1.0
    assert np.array_equal(out[~covered], np.zeros_like(out[~covered])) and np.all(out[covered][:, 3] == 1.0)
    ok = covered & (margin >= eps)
    assert ok.sum() >= min_fraction * covered.sum(), (int(ok.sum()), int(covered.sum()))
    np.testing.assert_allclose(out[ok][:, :3], ref[ok][:, :3], rtol=rtol, atol=1e-6)
    if ok.sum() == covered.sum():
        assert steps == ref_steps.sum()
    return out, steps


CONE_CASES = {
    # name: (image w, h, grid shape, chain, metal/rough, MaxSamples, StepMultiplier, NormalRayOffset, NoiseIndex)
    "cornell48_scene_materials": (64, 48, 48, "voxelized", None, 4, 0.16, 1.0, 3),
    "cornell_odd_grid_diffuse_64": (37, 19, (40, 56, 30), "voxelized", "zero", 64, 0.16, 0.0, 5),
    "sparse_odd_grid_mirror": (37, 19, (40, 56, 30), "sparse", "mirror", 4, 0.5, 1.0, 1),
    "sparse_rough_metal_1": (64, 48, (40, 56, 30), "sparse", "one", 1, 0.16, 1.0, 2),
    "dense_mixed_64": (37, 19, (33, 20, 47), "dense", "mixed", 64, 0.5, 0.0, 9),
    "dense_mixed_4": (64, 48, (24, 24, 24), "dense", "mixed", 4, 0.16, 1.0, 11),
}


@pytest.mark.parametrize("case", sorted(CONE_CASES))
def test_cone_trace_matches_float64(case):
    """The grids of (40, 56, 30) and (33, 20, 47) over the same bounds have voxel edges that differ by axis, so
    voxelMinLength != voxelMaxLength."""
    w, h, shape, chain, mrk, ms, sm, nro, noise = CONE_CASES[case]
    scene, frame, depth, nrg, mr = cornell_gbuffer(w, h, mrk)
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    if chain == "voxelized":
        levels, raw, _ = ol.vx_voxelize(scene, ci)
    else:
        levels, raw = synthetic_chain(ci, chain)
    compare_cone_trace(ci, levels, raw, frame, cone_settings(ms, sm, nro, noise), depth, nrg, mr)


EXACT = dict(sky=(0.5, 0.75, 1.0), sky_boost=0.5, gi_boost=1.5)   # products and sums of these are exact in float32


def _uniform_chain(ci, rgb, alpha):
    w, h, d = ci.Width, ci.Height, ci.Depth
    level0 = np.empty((d, h, w, 4), np.float16)
    level0[..., :3], level0[..., 3] = rgb, alpha
    return ol.vx_mipmap(ci, level0)


@pytest.mark.parametrize("max_samples", [1, 4])
def test_cone_trace_empty_grid_returns_the_sky(max_samples):
    """An empty grid accumulates nothing: every covered pixel is sky * GISkyBoxBoost * GIBoost exactly, and the cones march
    until they leave the grid (step totals against indirect_light64)."""
    scene, frame, depth, nrg, mr = cornell_gbuffer(37, 19, "zero")
    ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    levels, raw = _uniform_chain(ci, 0.0, 0.0)
    st = cone_settings(max_samples, gi_boost=EXACT["gi_boost"], sky_boost=EXACT["sky_boost"], noise_index=4)
    out, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr, sky=EXACT["sky"])
    want = np.array(EXACT["sky"]) * EXACT["sky_boost"] * EXACT["gi_boost"]
    covered = depth != 1.0
    assert np.array_equal(out[covered][:, :3], np.broadcast_to(want.astype(np.float32), (int(covered.sum()), 3)))
    _, ref_steps, margin = r.indirect_light64(levels, GRID_MIN, GRID_MAX, frame, st, depth, nrg, mr, EXACT["sky"])
    # with nothing to accumulate, the only decision is where a cone leaves the grid; one that passes a face within the
    # margin may take one step more or less
    near = int((covered & (margin < 1e-6)).sum())
    assert ref_steps.sum() > 0 and abs(steps - ref_steps.sum()) <= near * max_samples, (steps, int(ref_steps.sum()), near)


@pytest.mark.parametrize("alpha,n", [(0.5, 7), (0.75, 4)])
@pytest.mark.parametrize("max_samples", [1, 4])
def test_cone_trace_uniform_grid_closed_form(alpha, n, max_samples):
    """A uniform grid of colour c and alpha a: every level and every filter tap is (c, a), so after k steps acc.a =
    1 - (1 - a)^k and acc.rgb = c (1 - (1 - a)^k) / a; the loop stops at the smallest n with 1 - (1 - a)^n >= 0.99 (a = 0.5:
    7, a = 0.75: 4). The cones start at most one voxel inside the Cornell walls, which are four voxels from the grid's faces,
    and n steps of at most 0.16 voxelMinLength cannot leave it: every cone takes exactly n steps."""
    scene, frame, depth, nrg, mr = cornell_gbuffer(37, 19, "zero")
    ci = vxgi.create_info(48, GRID_MIN, GRID_MAX)
    c = 0.25
    levels, raw = _uniform_chain(ci, c, alpha)
    assert 1 - (1 - alpha) ** n >= 0.99 > 1 - (1 - alpha) ** (n - 1)
    st = cone_settings(max_samples, gi_boost=EXACT["gi_boost"], sky_boost=EXACT["sky_boost"])
    out, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr, sky=EXACT["sky"])
    covered = depth != 1.0
    assert steps == n * max_samples * covered.sum()
    keep = (1 - alpha) ** n
    want = (c * (1 - keep) / alpha + keep * np.array(EXACT["sky"]) * EXACT["sky_boost"]) * EXACT["gi_boost"]
    np.testing.assert_allclose(out[covered][:, :3], np.broadcast_to(want, (int(covered.sum()), 3)), rtol=1e-6)


def test_cone_trace_origin_outside_grid_returns_the_sky():
    """Every cone of a G-buffer outside the grid leaves it before its first sample: sky only, no steps."""
    scene, frame, depth, nrg, mr = cornell_gbuffer(37, 19, "mixed")
    ci = vxgi.create_info((12, 8, 16), (5.0, 5.0, 5.0), (6.0, 7.0, 6.5))
    levels, raw = synthetic_chain(ci, "dense")
    st = cone_settings(4, gi_boost=EXACT["gi_boost"], sky_boost=EXACT["sky_boost"])
    out, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr, sky=EXACT["sky"])
    covered = depth != 1.0
    want = (np.array(EXACT["sky"]) * EXACT["sky_boost"] * EXACT["gi_boost"]).astype(np.float32)
    assert steps == 0 and np.array_equal(out[covered][:, :3], np.broadcast_to(want, (int(covered.sum()), 3)))


def probe_gbuffer(frag_pos):
    """A 1x1 G-buffer whose one cone is a mirror cone (metallic 1, roughness 0: one sample, cone angle 0) along +x from
    frag_pos: InvProjView is a translation, the view position sits one unit in +x, the normal is +x. All of it is dyadic, so
    every sample position is exact in fp32."""
    frame = np.zeros(1, gt.GpuPerFrameData)
    m = np.eye(4, dtype=np.float32)
    m[3, :3] = np.asarray(frag_pos, np.float32) - np.float32([0.0, 0.0, 0.5])   # world = [ndc, 1] @ m; the pixel's ndc is (0, 0, 0.5)
    frame["InvProjView"][0] = m.reshape(-1)
    frame["ViewPos"][0] = np.asarray(frag_pos, np.float32) + np.float32([1.0, 0.0, 0.0])
    depth = np.full((1, 1), 0.5, np.float32)
    nrg = np.array([[[1.0, 0.5]]], np.float32)                                 # EncodeUnitVec(+x)
    mr = np.array([[[1.0, 0.0]]], np.float32)
    return frame, depth, nrg, mr


PROBES = {
    # an empty 16^3 grid over [0, 4]^3 and a cone along +x from x = 1 stepping 0.125: its 23rd sample lands exactly on
    # u = 1, which `uvw >= 1` rejects: 22 steps
    "sample_on_the_far_face": ((16, 16, 16), (0.0, 0.0, 0.0), (4.0, 4.0, 4.0), (1.0, 2.0625, 2.0625), 0.0, 22),
    # a 1x1x1 grid of alpha 0.5: maxLevel 0, and a cone of angle 0 samples at lod log2(voxelMin / voxelMin) = 0 exactly, which
    # `sampleLod > maxLevel` accepts; from x = -1 the samples at x = 3 and 3.5 are inside: 2 steps
    "lod_equal_to_max_level": ((1, 1, 1), (0.0, 1.5, 1.5), (4.0, 2.5, 2.5), (-1.0, 2.0625, 2.0625), 0.5, 2),
}


def probe_case(name):
    shape, gmin, gmax, frag_pos, alpha, n = PROBES[name]
    ci = vxgi.create_info(shape, gmin, gmax)
    levels, raw = _uniform_chain(ci, 0.25 if alpha else 0.0, alpha)
    frame, depth, nrg, mr = probe_gbuffer(frag_pos)
    st = cone_settings(4, 0.5, 0.0, gi_boost=EXACT["gi_boost"], sky_boost=EXACT["sky_boost"])
    keep = (1 - alpha) ** n
    want = ((0.25 * (1 - keep) / alpha if alpha else 0.0) + keep * np.array(EXACT["sky"]) * EXACT["sky_boost"]) * EXACT["gi_boost"]
    return ci, levels, raw, frame, st, depth, nrg, mr, n, want


@pytest.mark.parametrize("name", sorted(PROBES))
def test_cone_trace_exact_decisions(name):
    """Two cones whose decisions land exactly on their thresholds, with closed-form step counts and results (a uniform grid
    of colour 0.25 and alpha a: acc.a = 1 - (1 - a)^n stays below 0.99 for these n)."""
    ci, levels, raw, frame, st, depth, nrg, mr, n, want = probe_case(name)
    out, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr, sky=EXACT["sky"])
    assert steps == n
    np.testing.assert_allclose(out[0, 0, :3], want, rtol=1e-6)
    _, ref_steps, _ = r.indirect_light64(levels, list(ci.GridMin), list(ci.GridMax), frame, st, depth, nrg, mr, EXACT["sky"])
    assert ref_steps.sum() == n


# ---------------------------------------------------------------------------------------------------------- voxelisation
def compare_voxelize(scene, ci, max_ambiguous_fraction):
    levels, _, frags = ol.vx_voxelize(scene, ci)
    v = r.voxelize64(scene, ci)
    check_voxelized(levels[0], frags, v, max_ambiguous_fraction)
    return levels, v


def test_voxelize_cornell_odd_grid_matches_float64():
    scene, _ = lit_cornell()
    compare_voxelize(scene, vxgi.create_info((40, 56, 30), GRID_MIN, GRID_MAX), 0.03)


def test_voxelize_cornell_48_matches_float64():
    """At 48^3 every Cornell wall lies exactly on a voxel plane (x, z = +-1 and y = 0, 2 map to voxel coordinates 4 and 44),
    where the fp32 FragPos decides between the two neighbouring voxels: most occupied voxels are ambiguous, and the check is
    that every voxel the oracle writes is either written by voxelize64 or one of those candidates."""
    scene, _ = lit_cornell()
    levels, v = compare_voxelize(scene, vxgi.create_info(48, GRID_MIN, GRID_MAX), 0.9)
    occ = levels[0][..., 3] != 0
    assert not (occ & ~v["written"] & ~v["ambiguous"]).any()
    assert (v["written"] & ~v["ambiguous"]).sum() > 1000


def hand_scene(lights=True, emissive_bias=0.5):
    """45-degree triangles (dominant-axis ties), triangles smaller than a voxel, triangles crossing the grid's faces, and a
    wall exactly on a voxel plane, in a (32, 24, 40) grid over (0, 0, 0)..(3.2, 2.4, 4.0) (0.1 voxels)."""
    specs = [dict(color=(0.8, 0.6, 0.4)), dict(color=(0.2, 0.5, 0.9), emissive=(1.5, 0.25, 0.0), emissive_bias=emissive_bias),
             dict(color=(0.9, 0.9, 0.9, 0.5))]
    meshes, mats = scenes._materials(specs)
    a = scenes._Assembler()
    a.add(scenes.quad([0.35, 0.45, 0.5], [2.85, 0.45, 0.5], [2.85, 1.95, 3.0], [0.35, 1.95, 3.0]), 0)    # 45 deg about x: y/z tie
    a.add(scenes.quad([0.5, 0.25, 3.5], [2.5, 0.25, 3.5], [2.5, 1.85, 3.5], [0.5, 1.85, 3.5]), 1)        # z = 3.5: a voxel plane
    a.add(scenes.quad([-0.5, 2.13, -0.5], [3.7, 2.13, -0.5], [3.7, 2.13, 4.5], [-0.5, 2.13, 4.5]), 2)    # crosses every face
    rng = np.random.default_rng(5)
    for k in range(60):                                                                                   # smaller than a voxel
        c = rng.uniform([0.2, 0.2, 0.2], [3.0, 2.2, 3.8])
        p = c + rng.uniform(-0.04, 0.04, (3, 3))
        a.add((p.astype(np.float32), np.array([[0, 1, 2]], np.uint32)), k % 2)
    scene = host.Scene().add(a.model(meshes, mats, name="hand"), threads=1)
    if lights:
        scene.add_light((1.6, 2.0, 1.5), (4.0, 3.0, 2.0), 0.3)
    return scene


HAND_MIN, HAND_MAX, HAND_SIZE = (0.0, 0.0, 0.0), (3.2, 2.4, 4.0), (32, 24, 40)


def test_voxelize_hand_made_scene_matches_float64():
    scene = hand_scene()
    compare_voxelize(scene, vxgi.create_info(HAND_SIZE, HAND_MIN, HAND_MAX), 0.5)


def test_voxelize_unlit_quad_known_answer():
    """No lights: an axis-aligned quad writes half(Albedo * 0.02 + Emissive + EmissiveBias * Albedo) (times Alpha = 1) into
    exactly the voxels whose pixel centres it covers."""
    specs = [dict(color=(0.2, 0.5, 0.9), emissive=(1.5, 0.25, 0.0), emissive_bias=0.75)]
    meshes, mats = scenes._materials(specs)
    a = scenes._Assembler()
    a.add(scenes.quad([0.52, 0.33, 1.27], [2.61, 0.33, 1.27], [2.61, 1.88, 1.27], [0.52, 1.88, 1.27]), 0)
    scene = host.Scene().add(a.model(meshes, mats, name="quad"), threads=1)
    ci = vxgi.create_info(HAND_SIZE, HAND_MIN, HAND_MAX)
    levels, _, frags = ol.vx_voxelize(scene, ci)
    albedo = (gt.pack_unorm4x8(np.array([0.2, 0.5, 0.9, 1.0])) >> np.array([0, 8, 16])) & 255
    albedo = albedo / 255.0
    want = (albedo * float(np.float32(0.02)) + np.array([1.5, 0.25, 0.0]) + 0.75 * albedo).astype(np.float16)
    occ = levels[0][..., 3] != 0
    zs, ys, xs = np.nonzero(occ)
    assert set(zs) == {12} and (xs.min(), xs.max(), ys.min(), ys.max()) == (5, 25, 3, 18) and occ.sum() == 21 * 16 == frags
    assert np.array_equal(levels[0][occ][:, :3].view(np.uint16), np.broadcast_to(want, (int(occ.sum()), 3)).view(np.uint16))
