"""Voxelizer.IsConservativeRasterization on the device (idkvx_set_conservative_rasterization, k_vx_voxelize_*<true>): every
mip level and the fragment count equal the conservative oracle bit for bit, with point shadows in both modes, over uneven
z-slabs and under the cone trace; toggling the setting and the argument checks."""
import numpy as np
import pytest

import oracle_lib as ol
import point_shadow_oracle as pso
import vxgi_conservative_oracle as vco
from idkengine_b200 import multigpu, scenes, vxgi
from idkengine_b200.pathtracer import PathTracer
from raster_lib import GRID_MAX, GRID_MIN, TEX_GRID_MAX, TEX_GRID_MIN, lit_cornell, lit_cornell_shadowed
from test_vxgi_conservative import THIN_MAX, THIN_MIN, THIN_SIZE, atrium_lit, thin_scene

pytestmark = pytest.mark.gpu

IDKPT_ERR_INVALID_ARGUMENT = -1


def same_chain(vx, levels, what=""):
    for l, lv in enumerate(levels):
        assert np.array_equal(vx.ReadLevel(l).view(np.uint16), lv.view(np.uint16)), f"{what} level {l}"


def textured():
    return scenes.textured_room(threads=1)[0]


CASES = {
    # name: (scene, grid size, grid min, grid max)
    "cornell48": (lambda: lit_cornell()[0], 48, GRID_MIN, GRID_MAX),
    "cornell_odd": (lambda: lit_cornell()[0], (40, 56, 32), GRID_MIN, GRID_MAX),
    "cornell_tiles": (lambda: lit_cornell()[0], 200, GRID_MIN, GRID_MAX),     # walls of ~170 pixels: 3 x 3 tiles of 64
    "atrium": (atrium_lit, 128, vxgi.DEFAULT_GRID_MIN, vxgi.DEFAULT_GRID_MAX),
    "thin": (thin_scene, THIN_SIZE, THIN_MIN, THIN_MAX),
    "textured": (textured, (48, 40, 56), TEX_GRID_MIN, TEX_GRID_MAX),        # extrapolated texcoords through all wrap modes
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_gpu_conservative_matches_oracle(case):
    make, size, gmin, gmax = CASES[case]
    scene = make()
    ci = vxgi.create_info(size, gmin, gmax)
    levels, _, frags = vco.vx_voxelize(scene, ci)
    _, _, centre_frags = ol.vx_voxelize(scene, ci)
    assert frags > centre_frags
    with vxgi.Voxelizer(size, gmin, gmax) as vx:
        vx.SetScene(scene)
        vx.IsConservativeRasterization = True
        s = vx.Render()
        assert s.Fragments == frags
        same_chain(vx, levels)


def test_gpu_conservative_point_shadows_both_modes():
    """Shadow maps (the PCF lookup) and the shadow tracer (any-hit rays), each against its oracle under the conservative rule."""
    scene, shadows = lit_cornell_shadowed()
    sizes, dims = [96, 128], (48, 40, 44)
    ci = vxgi.create_info(dims, GRID_MIN, GRID_MAX)
    maps = [pso.point_shadow_render(scene, shadows[i], sizes[i]) for i in range(2)]
    pcf_levels, _, pcf_frags = vco.vx_voxelize_shadow_maps(scene, ci, shadows, maps)
    ray_levels, _, ray_frags = vco.vx_voxelize(scene, ci)
    assert not np.array_equal(pcf_levels[0].view(np.uint16), ray_levels[0].view(np.uint16))
    with PathTracer(16, 16) as pt, vxgi.Voxelizer(dims, GRID_MIN, GRID_MAX) as vx:
        pt.SetScene(scene)
        pt.SetPointShadows(shadows, sizes)
        pt.RenderPointShadows()
        vx.SetScene(scene)
        vx.IsConservativeRasterization = True
        vx.SetShadowTracer(pt)
        s = vx.Render()
        assert s.Fragments == ray_frags
        same_chain(vx, ray_levels, "shadow tracer")
        vx.SetShadowMaps(pt)
        s = vx.Render()
        assert s.Fragments == pcf_frags
        same_chain(vx, pcf_levels, "shadow maps")


def test_gpu_conservative_uneven_slabs_equal_single_pass():
    """Two contexts voxelise z-slabs of 13 and 19 layers: the gathered grid and its mip chain equal the single pass and the
    oracle, and the slabs' fragments add up to the single pass's."""
    import torch
    scene, _ = lit_cornell()
    size = (40, 56, 32)
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    levels, _, frags = vco.vx_voxelize(scene, ci)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as a, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as b:
        a.IsConservativeRasterization = True
        b.IsConservativeRasterization = True
        a.SetScene(scene)
        b.SetScene(scene)
        a.SetSlab(0, 13)
        b.SetSlab(13, 32)
        sa, sb = a.Render(), b.Render()
        assert sa.Fragments + sb.Fragments == frags
        pa, _ = a.LevelDevicePtr(0)
        pb, _ = b.LevelDevicePtr(0)
        ta = torch.as_tensor(multigpu.DeviceArray(pa, (size[2], size[1] * size[0] * 2), "<i4"), device="cuda")
        tb = torch.as_tensor(multigpu.DeviceArray(pb, (size[2], size[1] * size[0] * 2), "<i4"), device="cuda")
        assert not ta[13:].any() and not tb[:13].any()
        ta[13:].copy_(tb[13:])
        torch.cuda.synchronize()
        a.Mipmap()
        same_chain(a, levels, "gathered")
        a.SetSlab(0, 32)
        s = a.Render()
        assert s.Fragments == frags
        same_chain(a, levels, "single pass")


def test_gpu_cone_trace_on_conservative_grid_matches_oracle():
    scene, cam = lit_cornell()
    size = (40, 56, 32)
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    levels, raw, _ = vco.vx_voxelize(scene, ci)
    _, centre_raw, _ = ol.vx_voxelize(scene, ci)
    w, h = 96, 64
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, mr = ol.synth_gbuffer(scene, frame, w, h)
    st = vxgi.default_cone_settings()
    st.NoiseIndex = 5
    ref, steps = ol.vx_cone_trace(ci, raw, frame, st, depth, nrg, mr)
    centre_ref, _ = ol.vx_cone_trace(ci, centre_raw, frame, st, depth, nrg, mr)
    assert not np.array_equal(ref, centre_ref)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as vx:
        vx.SetScene(scene)
        vx.IsConservativeRasterization = True
        vx.Render()
        out, cs = vx.ConeTrace(frame, depth, nrg, mr, st)
        assert cs.ConeSteps == steps and np.array_equal(out, ref)


def test_gpu_conservative_toggle():
    """On, voxelise, off, voxelise: the default grid of a fresh context and of the oracle. The setting survives SetScene,
    SetGrid and SetSlab, and toggling alone leaves the current grid's bytes unchanged."""
    scene, _ = lit_cornell()
    size = 48
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    centre, _, centre_frags = ol.vx_voxelize(scene, ci)
    cons, _, cons_frags = vco.vx_voxelize(scene, ci)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as vx, vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as fresh:
        assert not vx.IsConservativeRasterization
        vx.SetScene(scene)
        vx.IsConservativeRasterization = True
        assert vx.Render().Fragments == cons_frags
        same_chain(vx, cons, "on")
        vx.IsConservativeRasterization = False                     # toggling alone does not touch the grid
        same_chain(vx, cons, "after toggling off")
        assert vx.Render().Fragments == centre_frags
        same_chain(vx, centre, "off")
        fresh.SetScene(scene)
        assert fresh.Render().Fragments == centre_frags
        same_chain(fresh, centre, "fresh context")
        vx.IsConservativeRasterization = True
        same_chain(vx, centre, "after toggling on")
        vx.SetScene(scene)                                          # survives SetScene, SetGrid and SetSlab
        vx.SetGrid(GRID_MIN, GRID_MAX)
        vx.SetSlab(0, 20)
        vx.SetSlab(0, size)
        assert vx.Render().Fragments == cons_frags
        same_chain(vx, cons, "on after SetScene / SetGrid / SetSlab")


def test_gpu_conservative_argument_errors():
    """A null context, enable = 2 and enable = -1 are refused with IDKPT_ERR_INVALID_ARGUMENT; the next voxelisation keeps the
    previous mode."""
    scene, _ = lit_cornell()
    size = (40, 56, 32)
    ci = vxgi.create_info(size, GRID_MIN, GRID_MAX)
    centre, _, centre_frags = ol.vx_voxelize(scene, ci)
    cons, _, cons_frags = vco.vx_voxelize(scene, ci)
    with vxgi.Voxelizer(size, GRID_MIN, GRID_MAX) as vx:
        L = vx._lib
        assert L.idkvx_set_conservative_rasterization(None, 1) == IDKPT_ERR_INVALID_ARGUMENT
        vx.SetScene(scene)
        for bad in (2, -1):
            assert L.idkvx_set_conservative_rasterization(vx._ctx, bad) == IDKPT_ERR_INVALID_ARGUMENT
            assert b"enable must be 0 or 1" in L.idkvx_last_error(vx._ctx)
        assert vx.Render().Fragments == centre_frags               # still the default
        same_chain(vx, centre, "default after refusals")
        vx.IsConservativeRasterization = True
        for bad in (2, -1):
            assert L.idkvx_set_conservative_rasterization(vx._ctx, bad) == IDKPT_ERR_INVALID_ARGUMENT
        assert vx.Render().Fragments == cons_frags                 # still conservative
        same_chain(vx, cons, "conservative after refusals")
        with pytest.raises(TypeError):
            vx.IsConservativeRasterization = 2
