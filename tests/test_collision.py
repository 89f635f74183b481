"""The C#-semantics scene-versus-moving-sphere oracle (oracle_collide_spheres, the checker of idkpt_collide_spheres) against
closed forms and a float64 brute force, and the collision records' layout."""
import numpy as np
import pytest

import collision_oracle as co
import oracle_lib as ol
from edge_lib import world_triangles
from idkengine_b200 import capi, gpu_types as gt, scenes
from idkengine_b200.pathtracer import CAMERA_COLLISION, LIGHT_COLLISION

EPS = 0.001
SLIDE, REFLECT = capi.IDKPT_COLLISION_SLIDE, capi.IDKPT_COLLISION_REFLECT


def spheres(prev, dest, radius, vel=None):
    s = np.zeros(len(prev), gt.IdkPtMovingSphere)
    s["PrevPosition"], s["Position"], s["Radius"] = prev, dest, radius
    s["Velocity"] = 0.0 if vel is None else vel
    return s


def test_record_layouts():
    assert gt.IdkPtCollisionSettings.itemsize == 16 and gt.IdkPtMovingSphere.itemsize == 48 and gt.IdkPtSphereCollision.itemsize == 32
    assert [gt.IdkPtCollisionSettings.fields[f][1] for f in ("TestSteps", "RecursiveSteps", "EpsilonNormalOffset", "Response")] == [0, 4, 8, 12]
    assert [gt.IdkPtMovingSphere.fields[f][1] for f in ("PrevPosition", "Radius", "Position", "Velocity")] == [0, 12, 16, 32]
    assert [gt.IdkPtSphereCollision.fields[f][1] for f in ("Position", "Hits", "Velocity")] == [0, 12, 16]
    assert LIGHT_COLLISION == (1, 8, EPS, REFLECT) and CAMERA_COLLISION == (3, 12, EPS, SLIDE)


def test_sphere_dropped_on_the_floor_rests_at_radius_plus_epsilon():
    sc, _ = scenes.open_floor(threads=1)
    r = np.array([0.25, 0.1, 0.5], np.float32)
    s = spheres([[0.3, 1.0, 0.2], [-1.0, 0.5, 2.0], [1.5, 1.2, -0.7]], [[0.3, 0.1, 0.2], [-1.0, 0.05, 2.0], [1.5, 0.3, -0.7]], r)
    out, first, _ = co.collide_spheres(sc, s, CAMERA_COLLISION, threads=1)
    assert (out["Hits"] == 1).all() and (first[:, 0] >= 0).all()
    np.testing.assert_allclose(out["Position"][:, 1], r + EPS, rtol=0, atol=2e-6)
    np.testing.assert_allclose(out["Position"][:, [0, 2]], s["PrevPosition"][:, [0, 2]], rtol=0, atol=1e-5)


@pytest.mark.parametrize("settings", [LIGHT_COLLISION, CAMERA_COLLISION], ids=["lights", "camera"])
def test_reflect_flips_and_slide_zeroes_the_normal_velocity(settings):
    sc, _ = scenes.open_floor(threads=1)
    vel = np.array([[1.0, -3.0, 0.5], [-0.2, -1.0, 0.0]], np.float32)
    s = spheres([[0.3, 0.5, 0.2], [1.0, 0.4, -1.0]], [[0.5, -0.2, 0.3], [0.9, 0.1, -1.0]], 0.25, vel)
    out, _, _ = co.collide_spheres(sc, s, settings, threads=1)
    assert (out["Hits"] == 1).all()
    want = vel.copy()
    want[:, 1] = -vel[:, 1] if settings[3] == REFLECT else 0.0
    # the normal is (c - q) / d of a float32 closest point q: off the axis by about ulp(|q|) / d
    np.testing.assert_allclose(out["Velocity"], want, rtol=0, atol=1e-4)


def test_untouched_sphere_is_bit_unchanged():
    sc, _ = scenes.closed_box(threads=1)
    vel = np.array([[0.3, -0.1, 7.0], [0.0, 0.0, 0.0], [1e-30, -2.5, 3.0]], np.float32)
    s = spheres([[0.0, 1.0, 0.0], [0.1, 0.9, -0.2], [0.2, 1.1, 0.3]], [[0.2, 1.2, 0.1], [0.1, 0.9, -0.2], [-0.3, 0.8, 0.3]], 0.3, vel)
    for st in (LIGHT_COLLISION, CAMERA_COLLISION, (5, 0, EPS, SLIDE)):
        out, first, _ = co.collide_spheres(sc, s, st, threads=1)
        assert (out["Hits"] == 0).all() and (first == -1).all()
        assert out["Position"].tobytes() == s["Position"].tobytes() and out["Velocity"].tobytes() == s["Velocity"].tobytes()


@pytest.mark.parametrize("settings", [LIGHT_COLLISION, CAMERA_COLLISION], ids=["lights", "camera"])
def test_sphere_driven_into_a_corner_takes_several_steps(settings):
    sc, _ = scenes.closed_box(subdiv=3, threads=1)
    r = 0.2
    s = spheres([[0.7, 0.3, 0.7]], [[0.86, 0.17, 0.84]], r, [[1.0, -1.0, 1.0]])
    out, _, _ = co.collide_spheres(sc, s, settings, threads=1)
    assert out["Hits"][0] >= 3, out["Hits"]
    if settings[3] == SLIDE:   # the slide comes to rest in the corner, a radius plus the offset off the two walls and the floor
        np.testing.assert_allclose(out["Position"][0], [1.0 - r - EPS, r + EPS, 1.0 - r - EPS], rtol=0, atol=1e-5)
        np.testing.assert_allclose(out["Velocity"][0], 0.0, rtol=0, atol=1e-5)
    else:                      # each wall and the floor reflected the velocity once
        assert (np.sign(out["Velocity"][0]) == [-1, -1, -1]).all() and out["Hits"][0] == 4


def _closest64(p0, e1, e2, c):
    """Float64 closest point of c on every triangle (Ericson's regions), vectorised."""
    a, b, cc = p0, p0 + e1, p0 + e2
    ab, ac, ap = e1, e2, c - a
    d1, d2 = (ab * ap).sum(1), (ac * ap).sum(1)
    bp = c - b
    d3, d4 = (ab * bp).sum(1), (ac * bp).sum(1)
    cp = c - cc
    d5, d6 = (ab * cp).sum(1), (ac * cp).sum(1)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    with np.errstate(divide="ignore", invalid="ignore"):
        den = va + vb + vc
        q = a + ab * (vb / den)[:, None] + ac * (vc / den)[:, None]
        m = (va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0)
        q[m] = (b + (cc - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[:, None])[m]
        m = (vb <= 0) & (d2 >= 0) & (d6 <= 0)
        q[m] = (a + ac * (d2 / (d2 - d6))[:, None])[m]
        m = (d6 >= 0) & (d5 <= d6)
        q[m] = cc[m]
        m = (vc <= 0) & (d1 >= 0) & (d3 <= 0)
        q[m] = (a + ab * (d1 / (d1 - d3))[:, None])[m]
        m = (d3 >= 0) & (d4 <= d3)
        q[m] = b[m]
        m = (d1 <= 0) & (d2 <= 0)
        q[m] = a[m]
    return q


def test_chosen_triangle_and_distance_match_a_float64_brute_force():
    """Stationary spheres (one test step at PrevPosition) near random atrium triangles: where the float64 nearest source
    triangle is clear of the runner-up, the oracle picks it and its distance agrees with float64."""
    sc, _ = scenes.atrium(target_tris=20000, threads=ol.default_threads())
    wt = world_triangles(sc)
    rng = np.random.default_rng(5)
    n = 96
    k = rng.integers(0, len(wt["p0"]), n)
    u, v = rng.uniform(0, 1, n), rng.uniform(0, 1, n)
    flip = u + v > 1
    u[flip], v[flip] = 1 - u[flip], 1 - v[flip]
    nrm = wt["n"][k] / np.linalg.norm(wt["n"][k], axis=1, keepdims=True)
    radius = rng.uniform(0.05, 0.3, n).astype(np.float32)
    off = rng.uniform(0.1, 0.9, n) * radius * np.where(rng.uniform(0, 1, n) < 0.5, -1, 1)
    centers = (wt["p0"][k] + u[:, None] * wt["e1"][k] + v[:, None] * wt["e2"][k] + off[:, None] * nrm).astype(np.float32)
    out, first, dist = co.collide_spheres(sc, spheres(centers, centers, radius), (1, 1, EPS, REFLECT))
    checked = 0
    for i in range(n):
        c = centers[i].astype(np.float64)
        d = np.linalg.norm(_closest64(wt["p0"], wt["e1"], wt["e2"], c) - c, axis=1)
        order = np.argsort(d)
        best, second = d[order[0]], d[order[1]]
        assert best < radius[i] and first[i, 0] >= 0 and out["Hits"][i] == 1
        if second - best < 1e-4 * max(1.0, best):
            continue                                   # a tie (shared edge or vertex): the visit order decides
        assert wt["frag2src"][first[i, 0]] == order[0], i
        assert abs(float(dist[i]) - best) <= 1e-5 * max(1.0, float(np.abs(c).max())), (i, dist[i], best)
        checked += 1
    assert checked >= n // 2, checked
