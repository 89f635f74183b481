"""The VXGI kernels on grids written by hand through idkvx_level_device_ptr, at the shapes the voxelised scenes of
tests/test_vxgi.py never produce: bit for bit against the oracle, and within the float64 bounds of tests/test_vxgi_ref.py
against tests/vxgi_ref64.py."""
import numpy as np
import pytest

import oracle_lib as ol
import vxgi_ref64 as r
from idkengine_b200 import vxgi
from raster_lib import GRID_MAX, GRID_MIN, check_voxelized, level0_fill, lit_cornell, synthetic_chain, write_level
from test_vxgi_ref import EXACT, MIP_SHAPES, PROBES, SKY, check_chain, compare_cone_trace, cone_settings, cornell_gbuffer, probe_case

pytestmark = pytest.mark.gpu


def gpu_chain(vx, level0):
    write_level(vx, 0, level0)
    vx.Mipmap()
    return [vx.ReadLevel(l) for l in range(len(vx.sizes))]


MIP_CASES = [(s, "random") for s in MIP_SHAPES] + [(s, f) for s in [(40, 56, 30), (7, 3, 129), (1, 64, 3), (3, 1, 7)]
                                                   for f in ("sparse", "subnormal", "near_max", "inf")]
MIP_CASES.append(((256, 256, 80), "sparse"))   # level 1 has 655,360 texels, more than one pass of the grid-stride loop


@pytest.mark.parametrize("shape,fill", MIP_CASES)
def test_gpu_mipmap_of_hand_made_grid(shape, fill):
    """k_vx_mipmap on a synthetic level 0: every level equals the oracle's bit for bit (subnormal, 65504 and inf halves
    check __float2half_rn against the oracle's and numpy's rounding) and is within 1 ulp of mip64 of the level below."""
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    level0 = level0_fill(shape, fill)
    ref, _ = ol.vx_mipmap(ci, level0)
    with vxgi.Voxelizer(shape, GRID_MIN, GRID_MAX) as vx:
        got = gpu_chain(vx, level0)
    for l, (g, o) in enumerate(zip(got, ref)):
        assert np.array_equal(g.view(np.uint16), o.view(np.uint16)), f"level {l}"
    check_chain(got, shape)


@pytest.mark.parametrize("size", [(1, 1), (7, 5), (37, 19), (64, 48)])
def test_gpu_cone_trace_of_hand_written_chain(size):
    """k_vx_cone_trace on a chain written level by level: image and step count equal the oracle's, the image is within
    the float64 bound, and two row tiles split at row 13 (inside an 8-row block) equal the single call."""
    w, h = size
    scene, frame, depth, nrg, mr = cornell_gbuffer(w, h, "mixed", seed=w)
    shape = (40, 56, 30)
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    levels, raw = synthetic_chain(ci, "sparse", seed=3)
    st = cone_settings(16, 0.16, 1.0, noise_index=6)
    ref, steps = compare_cone_trace(ci, levels, raw, frame, st, depth, nrg, mr, min_fraction=0.9 if w * h > 1 else 1.0)
    with vxgi.Voxelizer(shape, GRID_MIN, GRID_MAX) as vx:
        for l, lv in enumerate(levels):
            write_level(vx, l, lv)
        out, cs = vx.ConeTrace(frame, depth, nrg, mr, st, sky=SKY)
        assert np.array_equal(out, ref) and cs.ConeSteps == steps
        if h > 13:
            top, c0 = vx.ConeTraceRows(frame, depth[:13], nrg[:13], mr[:13], h, 0, st, sky=SKY)
            bot, c1 = vx.ConeTraceRows(frame, depth[13:], nrg[13:], mr[13:], h, 13, st, sky=SKY)
            assert np.array_equal(np.concatenate([top, bot]), out) and c0.ConeSteps + c1.ConeSteps == steps


@pytest.mark.parametrize("name", sorted(PROBES))
def test_gpu_cone_trace_exact_decisions(name):
    """The cones of test_cone_trace_exact_decisions (a sample exactly on u = 1, a lod exactly equal to maxLevel) on the device:
    the closed-form step count and the oracle's image."""
    ci, levels, raw, frame, st, depth, nrg, mr, n, want = probe_case(name)
    ref, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr, sky=EXACT["sky"])
    w, h, d = levels[0].shape[2], levels[0].shape[1], levels[0].shape[0]
    with vxgi.Voxelizer((w, h, d), list(ci.GridMin), list(ci.GridMax)) as vx:
        for l, lv in enumerate(levels):
            write_level(vx, l, lv)
        out, cs = vx.ConeTrace(frame, depth, nrg, mr, st, sky=EXACT["sky"])
    assert cs.ConeSteps == steps == n and np.array_equal(out, ref)
    np.testing.assert_allclose(out[0, 0, :3], want, rtol=1e-6)


def test_gpu_voxelize_odd_grid_and_uneven_slabs_match_float64():
    """The voxeliser kernels at (40, 56, 30) against voxelize64, whole and as two z-slabs of 11 and 19 layers split at z = 11:
    the gathered slabs and their mip chain equal the single pass and the oracle bit for bit."""
    import torch
    from idkengine_b200 import multigpu
    scene, _ = lit_cornell()
    size = (40, 56, 30)
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    levels, _, frags = ol.vx_voxelize(scene, ci)
    v = r.voxelize64(scene, ci)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as a, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as b:
        a.SetScene(scene)
        b.SetScene(scene)
        s = a.Render()
        whole = [a.ReadLevel(l) for l in range(len(levels))]
        assert s.Fragments == frags
        check_voxelized(whole[0], s.Fragments, v, 0.03)
        a.SetSlab(0, 11)
        b.SetSlab(11, 30)
        sa, sb = a.Render(), b.Render()
        assert sa.Fragments + sb.Fragments == frags
        pa, _ = a.LevelDevicePtr(0)
        pb, _ = b.LevelDevicePtr(0)
        ta = torch.as_tensor(multigpu.DeviceArray(pa, (size[2], size[1] * size[0] * 2), "<i4"), device="cuda")
        tb = torch.as_tensor(multigpu.DeviceArray(pb, (size[2], size[1] * size[0] * 2), "<i4"), device="cuda")
        assert not ta[11:].any() and not tb[:11].any()
        ta[11:].copy_(tb[11:])
        torch.cuda.synchronize()
        a.Mipmap()
        for l, lv in enumerate(levels):
            g = a.ReadLevel(l)
            assert np.array_equal(g.view(np.uint16), lv.view(np.uint16)) and np.array_equal(g.view(np.uint16), whole[l].view(np.uint16)), f"level {l}"
