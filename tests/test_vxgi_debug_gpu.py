"""k_vx_debug_render (idkvx_debug_render, Voxelizer.DebugRender) against the grid-visualisation oracle bit for bit: the image
and ConeSteps, over views that enter the grid through every face, graze its edges, start inside it or face away from it; image
sizes that leave partial 8x8 blocks; cone angles and step multipliers across the GUI's range; a constant sky and cube maps of
face size 128 and 5; voxelised and hand-written grids, mostly empty so that the empty-space skip takes most samples, one with
+-inf texels; and the full-size atrium. Then the call's semantics: the device pointer, repeat calls and every rejected
argument, which must leave the previous image as it was."""
import functools

import numpy as np
import pytest

import oracle_lib as ol
import vxgi_debug_oracle as vdo
from idkengine_b200 import capi, scenes, vxgi
from idkengine_b200.pathtracer import PathTracer
from raster_lib import GRID_MAX, GRID_MIN, lit_cornell, synthetic_chain, write_level
from test_vxgi_debug import hand_frame

pytestmark = pytest.mark.gpu

SHAPE = (40, 56, 30)
CENTRE = tuple((a + b) / 2 for a, b in zip(GRID_MIN, GRID_MAX))
VIEWS = {
    # name: (ViewPos, forward, half-extent of mat2(InvProjection))
    "outside_low_corner": ((-2.9, -1.6, -3.1), np.subtract(CENTRE, (-2.9, -1.6, -3.1)), (0.55, 0.45)),     # enters by -x, -y, -z
    "outside_high_corner": ((2.7, 3.9, 3.3), np.subtract(CENTRE, (2.7, 3.9, 3.3)), (0.55, 0.45)),         # enters by +x, +y, +z
    "grazing_edge": ((GRID_MIN[0], GRID_MIN[1], GRID_MIN[2] - 2.0), (0.0, 0.0, 1.0), (0.3, 0.3)),          # centre ray on the edge
    "grazing_face": ((0.1, GRID_MAX[1], GRID_MIN[2] - 2.0), (0.0, 0.0, 1.0), (0.4, 0.3)),                  # a row in the +y plane
    "inside": ((0.2, 1.1, -0.3), (0.4, -0.2, 1.0), (1.1, 0.8)),
    "behind_facing_away": ((0.0, 1.0, GRID_MAX[2] + 0.5), (0.1, 0.0, 1.0), (0.9, 0.7)),
}
SIZES = [(1, 1), (7, 5), (37, 19), (64, 48)]
INVALID_ARGUMENT = -1                            # IDKPT_ERR_INVALID_ARGUMENT


def same(a, b):
    """Bit for bit, except that NaN payloads differ between the device and the host: a NaN matches a NaN."""
    an, bn = np.isnan(a), np.isnan(b)
    return np.array_equal(an, bn) and np.array_equal(np.where(an, np.float32(0), a).view(np.uint32), np.where(bn, np.float32(0), b).view(np.uint32))


@functools.lru_cache(None)
def sky_case(kind):
    """(the PathTracer context's sky setter, the oracle's IdkPtSkyDesc) of one sky: constant, or the atmosphere at face
    size 128 (the engine's) or 5 (texels at every cube corner), generated on the device and read back for the oracle."""
    if kind == "constant":
        return (lambda pt: pt.SetSky((0.6, 0.7, 0.9))), capi.sky_desc((0.6, 0.7, 0.9))
    n = int(kind[len("atmosphere"):])
    with PathTracer(8, 8) as pt:
        pt.SkyAtmosphere(face_size=n)
        faces = pt.read_sky()
    return (lambda pt: pt.SetSky((0.0, 0.0, 0.0), faces)), capi.sky_desc((0.0, 0.0, 0.0), faces)


def mostly_empty(shape, seed):
    """synthetic_chain's sparse level 0 kept only inside a few boxes: empty bricks, occupied bricks and their borders."""
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    levels, _ = synthetic_chain(ci, "sparse", seed=seed)
    level0 = np.zeros_like(levels[0])
    rng = np.random.default_rng(seed)
    d, h, w = level0.shape[:3]
    for _ in range(4):
        lo = [int(rng.integers(0, n)) for n in (d, h, w)]
        hi = [min(n, l + int(rng.integers(1, max(2, n // 3)))) for l, n in zip(lo, (d, h, w))]
        level0[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = levels[0][lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    return ol.vx_mipmap(ci, level0)[0]


def infinite_texels(shape):
    """A mostly empty level 0 with blocks of +inf colour, of -inf alpha and of opaque texels, and its mip chain."""
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    level0 = np.zeros(shape[::-1] + (4,), np.float16)
    d, h, w = level0.shape[:3]
    level0[d // 4:d // 4 + 3, h // 3:h // 3 + 4, w // 3:w // 3 + 5] = (np.inf, 1.0, 0.5, 1.0)
    level0[d // 2:d // 2 + 4, h // 2:h // 2 + 3, w // 2:w // 2 + 4] = (0.5, 2.0, 1.0, -np.inf)
    level0[(3 * d) // 4:(3 * d) // 4 + 2, :, (2 * w) // 3:(2 * w) // 3 + 2] = (0.1, 0.2, 0.3, 1.0)
    return ol.vx_mipmap(ci, level0)[0]


@functools.lru_cache(None)
def grid_levels(kind):
    """The levels (float16 [d, h, w, 4] each) of one grid at (40, 56, 30) or (7, 3, 129) over the test bounds."""
    if kind == "cornell":
        scene, _ = lit_cornell()
        with vxgi.Voxelizer(SHAPE, GRID_MIN, GRID_MAX) as vx:      # the voxeliser's chain is pinned to the oracle by test_vxgi*.py
            vx.SetScene(scene)
            vx.Render()
            return tuple(vx.ReadLevel(l) for l in range(len(vx.sizes)))
    if kind == "empty_blocks_40":
        return tuple(mostly_empty(SHAPE, 5))
    if kind == "empty_blocks_7_3_129":
        return tuple(mostly_empty((7, 3, 129), 6))
    if kind == "inf":
        return tuple(infinite_texels(SHAPE))
    raise ValueError(kind)


def grid_shape(levels):
    d, h, w = levels[0].shape[:3]
    return (w, h, d)


def run_case(grid, sky, frame, w, h, cone, step):
    """The device image and stats next to the oracle's image and step count."""
    levels = grid_levels(grid)
    shape = grid_shape(levels)
    set_sky, sky_desc = sky_case(sky)
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    raw = np.concatenate([np.ascontiguousarray(lv).reshape(-1).view(np.uint16) for lv in levels])
    ref, steps = vdo.debug_render(ci, raw, frame, step, cone, w, h, sky=sky_desc)
    with vxgi.Voxelizer(shape, GRID_MIN, GRID_MAX) as vx, PathTracer(8, 8) as pt:
        set_sky(pt)
        for l, lv in enumerate(levels):
            write_level(vx, l, lv)
        vx.DebugConeAngle, vx.DebugStepMultiplier = cone, step
        img, st = vx.DebugRender(pt, frame, w, h)
    return img, st, ref, steps


def view_frame(name):
    pos, fwd, half = VIEWS[name]
    return hand_frame(pos, fwd, half=half)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("view", sorted(VIEWS))
def test_gpu_debug_render_views(view, size):
    w, h = size
    img, st, ref, steps = run_case("empty_blocks_40", "atmosphere128", view_frame(view), w, h, 0.0, 0.4)
    assert st.ConeSteps == steps and same(img, ref)
    if view == "behind_facing_away":
        assert steps == 0


@pytest.mark.parametrize("step", [0.05, 0.4, 1.0])
@pytest.mark.parametrize("cone", [0.0, 0.25, 0.5])
def test_gpu_debug_render_cone_and_step(cone, step):
    img, st, ref, steps = run_case("cornell", "atmosphere5", view_frame("outside_low_corner"), 37, 19, cone, step)
    assert st.ConeSteps == steps > 0 and same(img, ref)


@pytest.mark.parametrize("sky", ["constant", "atmosphere128", "atmosphere5"])
@pytest.mark.parametrize("grid", ["cornell", "empty_blocks_40", "empty_blocks_7_3_129", "inf"])
def test_gpu_debug_render_grids_and_skies(grid, sky):
    """Each grid from outside and from inside, with cone angles 0 (level 0 only: the skip) and 0.25 (every level)."""
    for view in ("outside_high_corner", "inside"):
        for cone in (0.0, 0.25):
            img, st, ref, steps = run_case(grid, sky, view_frame(view), 64, 48, cone, 0.4)
            assert st.ConeSteps == steps > 0 and same(img, ref), (view, cone)


def test_gpu_debug_render_inf_texels_hit():
    """The -inf alpha block is crossed: a march whose alpha became -inf takes its later (empty) samples as 0 * inf = NaN,
    on the device as in the oracle."""
    levels = grid_levels("inf")
    w, h, d = grid_shape(levels)
    sx = (GRID_MAX[0] - GRID_MIN[0]) / w
    sy = (GRID_MAX[1] - GRID_MIN[1]) / h
    target = (GRID_MIN[0] + (w // 2 + 2) * sx, GRID_MIN[1] + (h // 2 + 1.5) * sy)
    frame = hand_frame((target[0], target[1], GRID_MIN[2] - 1.0), (0.0, 0.0, 1.0))
    img, st, ref, steps = run_case("inf", "constant", frame, 1, 1, 0.0, 0.4)
    assert st.ConeSteps == steps and same(img, ref)
    assert np.isnan(img[0, 0]).any()


def test_gpu_debug_render_atrium_full_size():
    """bench.py's atrium with the reference's startup lights, voxelised at 256^3 over the default bounds and rendered at
    1920x1080 with the engine's defaults (cone angle 0, step multiplier 0.4) from the bench camera, inside the grid, and
    from outside it looking across."""
    import copy
    scene, cam = scenes.atrium(262144)
    sc = copy.copy(scene)
    sc.lights = scene.lights.copy()
    for light in scenes.STARTUP_LIGHTS:
        sc.add_light(*light)
    w, h = 1920, 1080
    set_sky, sky_desc = sky_case("atmosphere128")
    frames = [scenes.camera_frame(cam, w, h), scenes.camera_frame(dict(position=(34.0, 24.0, -30.0), view_dir=(-0.7, -0.35, 0.6)), w, h)]
    with vxgi.Voxelizer(256) as vx, PathTracer(8, 8) as pt:
        set_sky(pt)
        vx.SetScene(sc)
        vx.Render()
        raw = np.concatenate([vx.ReadLevel(l).reshape(-1).view(np.uint16) for l in range(len(vx.sizes))])
        for frame in frames:
            img, st = vx.DebugRender(pt, frame, w, h)
            ref, steps = vdo.debug_render(vx.ci, raw, frame, 0.4, 0.0, w, h, sky=sky_desc)
            assert st.ConeSteps == steps > 0 and same(img, ref)


def test_gpu_debug_device_ptr_and_repeat():
    """A fresh context's cleared grid renders as the oracle's empty grid (the sky, test_vxgi_debug.py); out = NULL leaves the
    image on the device, where idkvx_debug_device_ptr finds it equal to the downloaded one; two calls give identical images
    and step counts."""
    import torch
    from idkengine_b200 import multigpu
    levels = grid_levels("empty_blocks_40")
    set_sky, sky_desc = sky_case("atmosphere5")
    frame = view_frame("outside_low_corner")
    ci = vxgi.create_info(SHAPE, GRID_MIN, GRID_MAX)
    zeros = np.zeros(sum(x * y * z for x, y, z in vxgi.level_sizes(ci)) * 4, np.uint16)
    empty_ref, empty_steps = vdo.debug_render(ci, zeros, frame, 0.4, 0.0, 37, 19, sky=sky_desc)
    with vxgi.Voxelizer(SHAPE, GRID_MIN, GRID_MAX) as vx, PathTracer(8, 8) as pt:
        set_sky(pt)
        assert vx.DebugDevicePtr() == (None, 0)
        blank, bst = vx.DebugRender(pt, frame, 37, 19)
        assert np.array_equal(blank, empty_ref) and bst.ConeSteps == empty_steps > 0
        for l, lv in enumerate(levels):
            write_level(vx, l, lv)
        a, sa = vx.DebugRender(pt, frame, 37, 19)
        b, sb = vx.DebugRender(pt, frame, 37, 19)
        assert np.array_equal(a, b) and sa.ConeSteps == sb.ConeSteps and sa.KernelLaunches == sb.KernelLaunches
        none, sn = vx.DebugRender(pt, frame, 37, 19, out=False)
        assert none is None and sn.ConeSteps == sa.ConeSteps
        ptr, nbytes = vx.DebugDevicePtr()
        assert nbytes == 37 * 19 * 16
        dev = torch.as_tensor(multigpu.DeviceArray(ptr, (19, 37, 4), "<f4"), device="cuda").cpu().numpy()
        assert np.array_equal(dev, a)


def step_bound(shape, grid_min, grid_max):
    """The step multiplier at which (|GridMax - GridMin| + voxelMaxLength) / (voxelMinLength * m) = 65536, from the float32
    extents and voxel edges as the call computes them."""
    e = [np.float32(np.float32(b) - np.float32(a)) for a, b in zip(grid_min, grid_max)]
    vs = [float(np.float32(x / np.float32(n))) for x, n in zip(e, shape)]
    diag = float(np.sqrt(sum(float(x) * float(x) for x in e)))
    return (diag + max(vs)) / (min(vs) * 65536.0)


def test_gpu_debug_render_rejects_invalid_arguments():
    """Every rejected call returns IDKPT_ERR_INVALID_ARGUMENT before launching anything: the previous image keeps every byte.
    A step multiplier just under the 65536-step bound fails and one just over it passes (a grid of 512 x 512 x 2 over a flat
    box makes the bound reachable)."""
    import torch
    from idkengine_b200 import multigpu
    shape, gmin, gmax = (512, 512, 2), (-10.0, -10.0, -0.05), (10.0, 10.0, 0.05)
    m_star = step_bound(shape, gmin, gmax)
    frame = hand_frame((0.0, 0.0, -3.0), (0.0, 0.0, 1.0), half=(2.0, 2.0))
    with vxgi.Voxelizer(shape, gmin, gmax) as vx, PathTracer(8, 8) as pt:
        pt.SetSky((0.6, 0.7, 0.9))
        L, ctx = vx._lib, vx._ctx
        first, _ = vx.DebugRender(pt, frame, 7, 5)
        ptr, nbytes = vx.DebugDevicePtr()

        def device_image():
            return torch.as_tensor(multigpu.DeviceArray(ptr, (5, 7, 4), "<f4"), device="cuda").cpu().numpy()
        fr = np.ascontiguousarray(frame)
        out = np.full((5, 7, 4), -7.0, np.float32)

        def call(sky=pt._ctx, frame_ptr=fr.ctypes.data, m=0.4, cone=0.0, w=7, h=5, ctx_=ctx):
            return L.idkvx_debug_render(ctx_, sky, frame_ptr, m, cone, w, h, out.ctypes.data, None)
        bad = [dict(ctx_=None), dict(sky=None), dict(frame_ptr=None), dict(w=0), dict(h=0), dict(w=16385), dict(h=16385),
               dict(cone=float("nan")), dict(cone=float("inf")), dict(cone=-1e-6), dict(cone=1.5000001), dict(m=0.0),
               dict(m=-0.4), dict(m=float("nan")), dict(m=float("inf")), dict(m=float(np.float32(m_star) * np.float32(0.9999)))]
        for kw in bad:
            assert call(**kw) == INVALID_ARGUMENT, kw
            assert np.all(out == -7.0) and np.array_equal(device_image(), first), kw
        ok = float(np.float32(m_star) * np.float32(1.0001))
        assert call(m=ok) == 0 and np.array_equal(out, device_image())
        assert call(cone=1.5, m=0.4) == 0
