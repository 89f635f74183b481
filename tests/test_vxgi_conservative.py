"""Voxelizer.IsConservativeRasterization in the oracle (oracle/oracle_vxgi_conservative.cpp, DESIGN section 7): a triangle covers every
pixel whose closed square it touches, with attributes extrapolated to the pixel centre. Checked against the float64
restatement (tests/vxgi_conservative_ref64.py voxelize64_conservative), which decides coverage by vertex-in-square, corner-in-triangle
and edge crossing instead of the edge offsets, against the centre rule (a superset of it), on thin geometry (no gaps) and
on known answers. The kernels are pinned to the oracle bit for bit in tests/test_vxgi_conservative_gpu.py.

Measured (ambiguous = touched by a sample within the float64 margins of voxelize64):
- lit Cornell box, (40, 56, 30): 268 of 7,508 occupied voxels ambiguous, no ill-conditioned sample; 48^3: most voxels
  ambiguous because the walls lie on voxel planes (as for the centre rule).
- atrium(20000) at 128^3: 8,380 of 37,485 (walls on voxel planes), no ill-conditioned sample.
- thin-geometry scene: 49 of 791, 1 ill-conditioned sample of 2,174 fragments."""
import numpy as np
import pytest

import oracle_lib as ol
import vxgi_conservative_oracle as vco
import vxgi_conservative_ref64 as r64c
from idkengine_b200 import host, scenes, vxgi
from raster_lib import GRID_MAX, GRID_MIN, check_voxelized, lit_cornell

# a 32^3 grid over [0, 4]^3: window coordinates are 8 * world, so dyadic world coordinates are exact in fp32
KNOWN_MIN, KNOWN_MAX, KNOWN_SIZE = (0.0, 0.0, 0.0), (4.0, 4.0, 4.0), 32
KNOWN_Z = 2.0625                      # voxel 16.5: the triangles of the known answers lie in the middle of voxel layer 16

THIN_MIN, THIN_MAX, THIN_SIZE = (0.0, 0.0, 0.0), (3.2, 2.4, 4.0), (32, 24, 40)   # 0.1 voxels
THIN_WIDTHS = (0.05, 0.1, 0.2, 0.5)   # voxels
THIN_ANGLES = (3.0, 17.0, 31.0, 45.0, 62.0, 84.0)   # degrees from the x axis, in the z = const plane


def _scene(tris, mesh_ids=None, lights=True, specs=None):
    specs = specs or [dict(color=(0.8, 0.6, 0.4)), dict(color=(0.2, 0.5, 0.9), emissive=(0.5, 0.25, 0.0), emissive_bias=0.25)]
    meshes, mats = scenes._materials(specs)
    a = scenes._Assembler()
    for k, t in enumerate(tris):
        p = np.asarray(t, np.float32).reshape(-1, 3)
        idx = np.arange(len(p), dtype=np.uint32).reshape(-1, 3)
        a.add((p, idx), 0 if mesh_ids is None else mesh_ids[k])
    scene = host.Scene().add(a.model(meshes, mats, name="conservative"), threads=1)
    if lights:
        scene.add_light((1.6, 2.0, 1.5), (4.0, 3.0, 2.0), 0.3)
    return scene


def strip(z, centre, angle_deg, length, width):
    """A flat strip (two triangles) in the plane z = const, `width` world units wide."""
    d = np.array([np.cos(np.radians(angle_deg)), np.sin(np.radians(angle_deg)), 0.0])
    n = np.array([-d[1], d[0], 0.0])
    c = np.array([centre[0], centre[1], z])
    p0, p1 = c - d * length / 2 - n * width / 2, c + d * length / 2 - n * width / 2
    p2, p3 = c + d * length / 2 + n * width / 2, c - d * length / 2 + n * width / 2
    return [np.array([p0, p1, p2]), np.array([p0, p2, p3])]


def rod(a, b, width):
    """A rod of square cross-section `width` from a to b: four long quads (eight triangles)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    d = (b - a) / np.linalg.norm(b - a)
    u = np.cross(d, [0.0, 0.0, 1.0] if abs(d[2]) < 0.9 else [1.0, 0.0, 0.0])
    u /= np.linalg.norm(u)
    v = np.cross(d, u)
    h = width / 2
    ring = [u * h + v * h, -u * h + v * h, -u * h - v * h, u * h - v * h]
    out = []
    for k in range(4):
        q0, q1 = ring[k], ring[(k + 1) % 4]
        out += [np.array([a + q0, b + q0, b + q1]), np.array([a + q0, b + q1, a + q1])]
    return out


def thin_scene(seed=7):
    """Strips 0.05 - 0.5 voxel wide at several angles, rods, slivers, and triangles smaller than a pixel, inside one pixel and
    straddling pixel corners, in the THIN grid (0.1 voxels)."""
    rng = np.random.default_rng(seed)
    tris = []
    for k, w in enumerate(THIN_WIDTHS):
        for m, ang in enumerate(THIN_ANGLES):
            z = 0.4 + 0.1 * (k * len(THIN_ANGLES) + m) * 0.13 + 0.0371
            tris += strip(z, (1.6 + 0.05 * m, 1.2 - 0.03 * k), ang, 2.0, 0.1 * w)
    tris += rod((0.3, 0.3, 3.3), (2.9, 2.1, 3.7), 0.02)
    tris += rod((0.4, 2.0, 0.3), (2.8, 0.35, 0.45), 0.035)
    for k in range(12):                                       # slivers: long and thin, altitude 0.02 - 0.2 voxel
        c = rng.uniform([0.5, 0.5, 0.5], [2.7, 1.9, 3.5])
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        n = np.cross(d, rng.normal(size=3))
        n /= np.linalg.norm(n)
        tris.append(np.array([c - d * 0.3, c + d * 0.3, c + n * rng.uniform(0.002, 0.02)]))
    for k in range(40):                                       # smaller than a pixel
        c = rng.uniform([0.2, 0.2, 0.2], [3.0, 2.2, 3.8])
        if k % 2:
            c = np.round(c / 0.1) * 0.1 + rng.uniform(-0.004, 0.004, 3)   # near a pixel corner of every projection
        tris.append(c + rng.uniform(-0.02, 0.02, (3, 3)))
    return _scene(tris, mesh_ids=[k % 2 for k in range(len(tris))])


def thin_ci():
    return vxgi.create_info(THIN_SIZE, THIN_MIN, THIN_MAX)


def known_ci():
    return vxgi.create_info(KNOWN_SIZE, KNOWN_MIN, KNOWN_MAX)


def window_triangle(q, z=KNOWN_Z):
    """A triangle given in window coordinates (pixels) of the KNOWN grid's z projection."""
    q = np.asarray(q, np.float64)
    return np.concatenate([q / 8.0, np.full((3, 1), z)], 1)


def occupied(levels):
    return levels[0][..., 3] != 0


def compare_conservative(scene, ci, max_ambiguous_fraction):
    levels, _, frags = vco.vx_voxelize(scene, ci)
    v = r64c.voxelize64_conservative(scene, ci)
    check_voxelized(levels[0], frags, v, max_ambiguous_fraction)
    return levels, frags, v


# ------------------------------------------------------------------------------------------------ against float64
def test_conservative_cornell_odd_grid_matches_float64():
    scene, _ = lit_cornell()
    _, _, v = compare_conservative(scene, vxgi.create_info((40, 56, 30), GRID_MIN, GRID_MAX), 0.05)
    assert v["ill_conditioned_samples"] == 0


def test_conservative_cornell_48_matches_float64():
    """The walls lie on voxel planes at 48^3 (test_voxelize_cornell_48_matches_float64): most voxels are ambiguous, every
    voxel the oracle writes is written by voxelize64 or one of its candidates."""
    scene, _ = lit_cornell()
    levels, _, v = compare_conservative(scene, vxgi.create_info(48, GRID_MIN, GRID_MAX), 0.95)
    occ = occupied(levels)
    assert not (occ & ~v["written"] & ~v["ambiguous"]).any()
    assert (v["written"] & ~v["ambiguous"]).sum() > 1000


def atrium_lit():
    scene, cam = scenes.atrium(20000)
    scene.lights = scene.lights[:0]
    scene.add_light((0.0, 6.0, 0.0), (40.0, 38.0, 30.0), 0.3)
    return scene


def test_conservative_atrium_matches_float64():
    scene = atrium_lit()
    _, frags, v = compare_conservative(scene, vxgi.create_info(128), 0.25)
    assert v["ill_conditioned_samples"] <= 1e-3 * frags, (v["ill_conditioned_samples"], frags)


def test_conservative_thin_geometry_matches_float64():
    scene = thin_scene()
    _, frags, v = compare_conservative(scene, thin_ci(), 0.1)
    assert v["ill_conditioned_samples"] <= 0.02 * frags, (v["ill_conditioned_samples"], frags)


# ------------------------------------------------------------------------------------------------ superset of the centre rule
@pytest.mark.parametrize("which", ["cornell48", "cornell_odd", "thin", "atrium"])
def test_conservative_is_a_superset_of_the_centre_rule(which):
    """Every pixel centre the centre rule covers lies in its pixel's square, and both rules evaluate the attributes at that
    centre with the same fp32 operations: the conservative grid holds every voxel of the centre grid with every channel >=
    (non-negative halves order like unsigned shorts), and it has at least as many fragments."""
    if which.startswith("cornell"):
        scene, _ = lit_cornell()
        ci = vxgi.create_info(48 if which == "cornell48" else (40, 56, 30), GRID_MIN, GRID_MAX)
    elif which == "thin":
        scene, ci = thin_scene(), thin_ci()
    else:
        scene, ci = atrium_lit(), vxgi.create_info(128)
    centre, _, fc = ol.vx_voxelize(scene, ci)
    cons, _, fk = vco.vx_voxelize(scene, ci)
    oc = occupied(centre)
    assert not (oc & ~occupied(cons)).any()
    assert (cons[0].view(np.uint16)[oc] >= centre[0].view(np.uint16)[oc]).all()
    assert fk >= fc and occupied(cons).sum() >= oc.sum()


# ------------------------------------------------------------------------------------------------ thin geometry
@pytest.mark.parametrize("width", THIN_WIDTHS)
@pytest.mark.parametrize("angle", THIN_ANGLES)
def test_thin_strip_is_continuous(angle, width):
    """A strip narrower than a voxel: the conservative grid contains every voxel of the float64 answer, and its projection
    covers every pixel column along the strip's length; the centre rule leaves gaps on the same strip."""
    z = 2.0 + 0.0437
    scene = _scene(strip(z, (1.6, 1.2), angle, 2.0, 0.1 * width))
    ci = thin_ci()
    cons, _, frags = vco.vx_voxelize(scene, ci)
    centre, _, _ = ol.vx_voxelize(scene, ci)
    v = r64c.voxelize64_conservative(scene, ci)
    occ = occupied(cons)
    assert v["written"].sum() > 10 and not (v["written"] & ~occ).any()
    check_voxelized(cons[0], frags, v, 0.5)
    # the strip lies in one voxel layer; along its major axis every column between its ends is occupied
    zs = np.nonzero(occ.any((1, 2)))[0]
    assert len(zs) == 1
    layer_c, layer_o = occ[zs[0]], occupied(centre)[zs[0]]
    axis = 1 if abs(np.cos(np.radians(angle))) >= abs(np.sin(np.radians(angle))) else 0     # occ[y, x]: x columns = axis 1
    cols = np.nonzero(layer_c.any(1 - axis))[0]
    assert np.array_equal(cols, np.arange(cols[0], cols[-1] + 1)) and len(cols) >= 12
    got_o = set(np.nonzero(layer_o.any(1 - axis))[0])
    assert len(got_o) < len(cols), "the centre rule covers every column of a strip narrower than a voxel"


# ------------------------------------------------------------------------------------------------ known answers
def _known(tris, conservative):
    scene = _scene([window_triangle(t) for t in tris], lights=False)
    levels, _, frags = (vco if conservative else ol).vx_voxelize(scene, known_ci())
    zs, ys, xs = np.nonzero(occupied(levels))
    return frags, sorted(zip(xs.tolist(), ys.tolist(), zs.tolist()))


SUB_PIXEL = [(5.125, 7.125), (5.5, 7.125), (5.125, 7.5)]                      # inside pixel (5, 7), away from its centre
ACROSS_CORNER = [(5.875, 7.875), (6.25, 7.875), (5.875, 8.25)]               # the same triangle across the corner (6, 8)


def test_sub_pixel_triangle_inside_one_square_gives_one_fragment():
    assert _known([SUB_PIXEL], True) == (1, [(5, 7, 16)])
    assert _known([SUB_PIXEL], False) == (0, [])


def test_sub_pixel_triangle_across_a_pixel_corner_gives_four_fragments():
    assert _known([ACROSS_CORNER], True) == (4, [(5, 7, 16), (5, 8, 16), (6, 7, 16), (6, 8, 16)])
    assert _known([ACROSS_CORNER], False)[0] == 0
    assert _known([ACROSS_CORNER[::-1]], True) == _known([ACROSS_CORNER], True)      # either winding


@pytest.mark.parametrize("tri,want", [
    ([(4.25, 2.25), (5.0, 2.25), (5.0, 2.75)], [(4, 2, 16), (5, 2, 16)]),        # bounding box ends on the pixel edge x = 5
    ([(5.0, 2.25), (5.75, 2.25), (5.0, 2.75)], [(4, 2, 16), (5, 2, 16)]),        # ... starts on it
    ([(2.25, 6.25), (2.75, 6.25), (2.5, 7.0)], [(2, 6, 16), (2, 7, 16)]),        # a vertex on the pixel edge y = 7
    ([(9.25, 3.0), (9.75, 3.0), (9.5, 3.5)], [(9, 2, 16), (9, 3, 16)]),          # an edge on the pixel edge y = 3
])
def test_bounding_box_on_a_pixel_edge_is_inclusive(tri, want):
    """Boundaries are inclusive: a pixel whose square only touches the triangle on its edge is covered."""
    assert _known([tri], True) == (len(want), want)


@pytest.mark.parametrize("conservative", [False, True])
def test_zero_area_triangle_gives_nothing(conservative):
    assert _known([[(3.25, 3.25), (4.25, 4.25), (5.75, 5.75)]], conservative) == (0, [])
    assert _known([[(3.25, 3.25), (3.25, 3.25), (3.25, 3.25)]], conservative) == (0, [])


def test_known_answers_against_float64():
    """The known-answer triangles through voxelize64_conservative: same voxels, no ambiguous sample."""
    scene = _scene([window_triangle(t) for t in (SUB_PIXEL, ACROSS_CORNER)], lights=False)
    levels, _, frags = vco.vx_voxelize(scene, known_ci())
    v = r64c.voxelize64_conservative(scene, known_ci())
    assert frags == v["fragments"] == 5 and v["ambiguous_samples"] == 0
    assert np.array_equal(occupied(levels), v["written"])
