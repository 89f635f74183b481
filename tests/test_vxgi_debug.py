"""The grid-visualisation oracle (oracle/oracle_vxgi_debug.cpp, Voxelizer.DebugRender) against facts that do not come from
it: rays that miss the grid or have it behind them store the sky, an empty grid renders as the sky, an axis-parallel march
through an empty grid takes the closed-form number of steps, a march from inside the grid starts at ViewPos, and a ray in
the plane of a face follows the fminf / fmaxf rule of DESIGN.md 8f.1k."""
import math

import numpy as np
import pytest

import oracle_lib as ol
import vxgi_debug_oracle as vdo
from idkengine_b200 import capi, gpu_types as gt, vxgi

GRID_MIN, GRID_MAX = (-1.2, -0.2, -1.2), (1.2, 2.2, 1.2)
SHAPE = (12, 10, 8)                   # voxel edges 0.2, 0.24, 0.3


def hand_frame(pos, fwd, up=(0.0, 1.0, 0.0), half=(0.8, 0.6)):
    """A GpuPerFrameData whose centre pixel looks along fwd from pos: InvView's columns are (right, up, -fwd, pos) and
    mat2(InvProjection) = diag(half)."""
    f = np.zeros(1, gt.GpuPerFrameData)
    fw = np.asarray(fwd, np.float64) / np.linalg.norm(fwd)
    r = np.cross(fw, up)
    r /= np.linalg.norm(r)
    u = np.cross(r, fw)
    iv = np.zeros(16, np.float32)
    iv[0:3], iv[4:7], iv[8:11], iv[12:15], iv[15] = r, u, -fw, pos, 1.0
    ip = np.zeros(16, np.float32)
    ip[0], ip[5], ip[10], ip[15] = half[0], half[1], 1.0, 1.0
    f["InvView"], f["InvProjection"], f["ViewPos"] = iv, ip, pos
    return f


def directions(frame, w, h):
    """The pixel directions of DebugVisualization/compute.glsl in float32, in the kernel's operation order."""
    f32 = np.float32
    iv = frame["InvView"][0].astype(f32)
    ip = frame["InvProjection"][0].astype(f32)
    nx = ((np.arange(w, dtype=f32) + f32(0.5)) / f32(w) * f32(2.0) - f32(1.0))[None, :]
    ny = ((np.arange(h, dtype=f32) + f32(0.5)) / f32(h) * f32(2.0) - f32(1.0))[:, None]
    rvx, rvy = ip[0] * nx + ip[4] * ny, ip[1] * nx + ip[5] * ny
    d = np.stack([((iv[c] * rvx + iv[4 + c] * rvy) + iv[8 + c] * f32(-1.0)) + iv[12 + c] * f32(0.0) for c in range(3)], -1)
    inv = f32(1.0) / np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    return (d * inv[..., None]).astype(f32)


def chain(shape=SHAPE, level0=None):
    ci = vxgi.create_info(shape, GRID_MIN, GRID_MAX)
    total = sum(a * b * c for a, b, c in vxgi.level_sizes(ci))
    raw = np.zeros(total * 4, np.uint16)
    if level0 is not None:
        raw[:level0.size] = np.ascontiguousarray(level0, np.float16).reshape(-1).view(np.uint16)
    return ci, raw


def cube_faces(n, seed=0):
    rng = np.random.default_rng(seed)
    f = rng.uniform(0.0, 4.0, (6, n, n, 4)).astype(np.float32)
    f[..., 3] = 1.0
    return f


SKIES = {"constant": lambda: (capi.sky_desc((0.6, 0.7, 0.9)), None), "cube5": lambda: (capi.sky_desc((0, 0, 0), cube_faces(5)), cube_faces(5))}


def expected_sky(sky_kind, dirs):
    sky, faces = SKIES[sky_kind]()
    flat = dirs.reshape(-1, 3)
    rgb = np.tile(np.array(sky.Color[:], np.float32), (len(flat), 1)) if faces is None else ol.sample_sky(faces, flat)
    return np.concatenate([rgb, np.ones((len(flat), 1), np.float32)], 1).reshape(dirs.shape[:-1] + (4,))


def render(ci, raw, frame, w, h, sky_kind="constant", step=0.4, cone=0.0):
    sky, _ = SKIES[sky_kind]()
    return vdo.debug_render(ci, raw, frame, step, cone, w, h, sky=sky)


MISS_VIEWS = {
    # name: (ViewPos, forward): the grid beside, behind, or wholly behind the camera
    "beside": ((3.0, 1.0, 0.0), (1.0, 0.2, 0.3)),
    "behind": ((0.0, 1.0, 1.2 + 1.0), (0.0, 0.0, 1.0)),
    "above_looking_up": ((0.0, 4.0, 0.0), (0.1, 1.0, 0.0)),
    "far_face_t2_zero": ((0.0, 1.0, 1.2), (0.0, 0.0, 1.0)),        # on the +z face looking out: t1 = t2 = 0
}


@pytest.mark.parametrize("sky_kind", sorted(SKIES))
@pytest.mark.parametrize("view", sorted(MISS_VIEWS))
def test_rays_that_miss_store_the_sky(view, sky_kind):
    """Every ray of these views either misses the box or has it behind the camera (t2 <= 0, including t2 == 0 with the
    camera on the far face): each pixel is texture(sky, dir) with alpha 1, and no cone sample is taken. The grid is full of
    opaque texels, so a ray that entered it would show."""
    pos, fwd = MISS_VIEWS[view]
    w, h = (1, 1) if view == "far_face_t2_zero" else (9, 7)
    frame = hand_frame(pos, fwd, half=(0.05, 0.05) if view == "far_face_t2_zero" else (0.3, 0.3))
    full = np.zeros(SHAPE[::-1] + (4,), np.float16)
    full[...] = (1.0, 0.5, 0.25, 1.0)
    ci, raw = chain(level0=full)
    img, steps = render(ci, raw, frame, w, h, sky_kind)
    want = expected_sky(sky_kind, directions(frame, w, h))
    assert steps == 0
    assert np.array_equal(img, want)


@pytest.mark.parametrize("sky_kind", sorted(SKIES))
@pytest.mark.parametrize("cone", [0.0, 0.25])
def test_empty_grid_renders_the_sky(sky_kind, cone):
    """A cleared grid (all levels zero) accumulates (0, 0, 0, 0): every pixel, inside or outside the box, is exactly the sky
    with alpha 1, while the rays that cross the grid still take their steps."""
    ci, raw = chain()
    for pos, fwd in [((0.0, 1.0, -3.0), (0.1, 0.05, 1.0)), ((0.3, 1.1, 0.2), (1.0, -0.3, 0.4))]:
        frame = hand_frame(pos, fwd, half=(1.2, 0.9))
        img, steps = render(ci, raw, frame, 13, 11, sky_kind, step=0.4, cone=cone)
        assert steps > 0
        assert np.array_equal(img, expected_sky(sky_kind, directions(frame, 13, 11)))


def axis_steps(extent, vmax, delta):
    """Samples of an empty march along one axis from the entry face: distances vmax + k * delta below the extent."""
    return max(0, math.ceil((extent - vmax) / delta))


@pytest.mark.parametrize("step", [0.05, 0.4, 1.0])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_axis_parallel_march_closed_form(axis, step):
    """A 1x1 image whose ray runs along an axis through an empty grid from outside: the march takes the samples at
    vmax + k * vmin * step inside the grid's extent along that axis, in float64 within one step."""
    ci, raw = chain()
    ext = [GRID_MAX[i] - GRID_MIN[i] for i in range(3)]
    vs = [ext[i] / SHAPE[i] for i in range(3)]
    pos = [GRID_MIN[i] + 0.37 * ext[i] for i in range(3)]
    pos[axis] = GRID_MIN[axis] - 0.75
    fwd = [0.0, 0.0, 0.0]
    fwd[axis] = 1.0
    frame = hand_frame(pos, fwd, up=(1.0, 0.0, 0.0) if axis == 1 else (0.0, 1.0, 0.0))
    img, steps = render(ci, raw, frame, 1, 1, step=step)
    want = axis_steps(ext[axis], max(vs), min(vs) * step)
    assert abs(steps - want) <= 1, (steps, want)
    assert np.array_equal(img[0, 0], np.array([0.6, 0.7, 0.9, 1.0], np.float32))


def test_march_from_inside_starts_at_view_pos():
    """With the camera inside the grid t1 = 0, so the march starts at ViewPos: the closed-form count from ViewPos to the
    exit face, far fewer than from the entry face behind the camera. A single opaque voxel at ViewPos ends the march at its
    first sample."""
    ci, raw = chain()
    ext = [GRID_MAX[i] - GRID_MIN[i] for i in range(3)]
    vs = [ext[i] / SHAPE[i] for i in range(3)]
    pos = (0.5, 1.0, 0.3)
    frame = hand_frame(pos, (0.0, 0.0, 1.0))
    _, steps = render(ci, raw, frame, 1, 1, step=0.4)
    want = axis_steps(GRID_MAX[2] - pos[2], max(vs), min(vs) * 0.4)
    assert abs(steps - want) <= 1 and want < axis_steps(ext[2], max(vs), min(vs) * 0.4) - 3, (steps, want)
    first = [pos[0], pos[1], pos[2] + max(vs)]              # the first sample, voxelMaxLength along the ray
    ix = [int((first[i] - GRID_MIN[i]) / vs[i]) for i in range(3)]
    level0 = np.zeros(SHAPE[::-1] + (4,), np.float16)
    level0[ix[2] - 1:ix[2] + 2, ix[1] - 1:ix[1] + 2, ix[0] - 1:ix[0] + 2] = (2.0, 3.0, 4.0, 2.0)   # alpha 2: one sample ends it
    ci, raw = chain(level0=level0)
    img, steps = render(ci, raw, frame, 1, 1, step=0.4)
    assert steps == 1
    np.testing.assert_allclose(img[0, 0], [2.0 - 0.6, 3.0 - 0.7, 4.0 - 0.9, 1.0], rtol=1e-6)   # c + (1 - 2) * (sky, 1)


def ray_box_rule(o, d, bmin, bmax):
    """DESIGN.md 8f.1k's RayBoxIntersect in float32: fminf / fmaxf ignore a NaN operand. Returns (t1, t2)."""
    f32 = np.float32
    with np.errstate(all="ignore"):
        inv = f32(1.0) / np.asarray(d, f32)
        t0 = (np.asarray(bmin, f32) - np.asarray(o, f32)) * inv
        t1s = (np.asarray(bmax, f32) - np.asarray(o, f32)) * inv
    small, big = np.fmin(t0, t1s), np.fmax(t0, t1s)
    return np.fmax(small[0], np.fmax(small[1], np.fmax(small[2], f32(0.0)))), np.fmin(big[0], np.fmin(big[1], big[2]))


@pytest.mark.parametrize("face", ["min_x", "max_x", "min_y", "max_y"])
def test_ray_in_a_face_plane(face):
    """A ray that runs inside the plane of a face: 1 / 0 = inf, and (plane - origin) * inf = 0 * inf = NaN on that face.
    fminf / fmaxf drop the NaN, so that axis's slab becomes (+-inf, +-inf) and the ray misses: the pixel is the sky and
    no sample is taken, as the float32 rule computes."""
    ci, raw = chain(level0=np.full(SHAPE[::-1] + (4,), 1.0, np.float16))
    axis = 0 if face.endswith("x") else 1
    pos = [0.1, 1.0, GRID_MIN[2] - 1.0]
    pos[axis] = (GRID_MIN if face.startswith("min") else GRID_MAX)[axis]
    frame = hand_frame(pos, (0.0, 0.0, 1.0))
    d = directions(frame, 1, 1)[0, 0]
    t1, t2 = ray_box_rule(np.float32(pos), d, np.float32(GRID_MIN), np.float32(GRID_MAX))
    assert not (t1 <= t2 and t2 > 0)
    img, steps = render(ci, raw, frame, 1, 1, "cube5")
    assert steps == 0
    assert np.array_equal(img, expected_sky("cube5", d[None, None]))
