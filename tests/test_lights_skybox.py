"""The light spheres and the skybox (DESIGN.md 8f.1i) on the CPU: the oracle against an independent float64 restatement.

The light draw only reads the scene's lights, so most tests feed the oracle a hand-made G-buffer (constant depth) over the
Cornell box's scene record and place their own lights and cameras."""
import copy

import numpy as np
import pytest

import lights_skybox_oracle as lo
from idkengine_b200 import gpu_types as gt
from idkengine_b200 import host, scenes

W, H = 48, 32
T = lo.SPHERE_TRIANGLES


@pytest.fixture(scope="module")
def base_scene():
    scene, _ = scenes.cornell_1k(threads=1)
    return scene


def with_lights(scene, lights):
    """A copy of scene whose lights are [(position, color, radius[, prev_position])]."""
    s = copy.deepcopy(scene)
    s.lights = np.zeros(0, gt.GpuLight)
    for L in lights:
        s.add_light(L[0], L[1], L[2])
        if len(L) > 3:
            s.lights[-1]["PrevPosition"] = L[3]
    return s


def frame_at(eye=(0.0, 0.0, 0.0), view_dir=(0.0, 0.0, -1.0), w=W, h=H, fov=60.0):
    return host.make_per_frame_data(eye, view_dir, w, h, fov)


def blank_gbuffer(h=H, w=W, depth=1.0):
    return (np.full((h, w), depth, np.float32), np.zeros((h, w, 2), np.float32), np.full((h, w, 3), 0.25, np.float32),
            np.full((h, w, 2), 0.5, np.float32), np.zeros((h, w, 3), np.float32), np.zeros((h, w, 2), np.float32))


def run(scene, frame, depth=1.0, jitter=None, sky=(0.6, 0.7, 0.9), gbuffer=None):
    """The oracle over a W x H G-buffer (constant depth, or gbuffer) and a constant lit image."""
    g = gbuffer if gbuffer is not None else blank_gbuffer(H, W, depth)
    color = np.full((H, W, 4), 0.125, np.float32)
    return lo.lights_and_skybox(scene, frame, g, color, jitter=jitter, sky=sky, threads=4)


def mat(frame, name):
    """A GpuPerFrameData matrix as the float64 column-vector matrix GLSL sees."""
    return np.asarray(frame[name][0], np.float64).reshape(4, 4).T


def pixel_rays(frame, w, h, jitter=(0.0, 0.0)):
    """float64 eye and unit directions [h, w, 3] through the (jittered) pixel centres."""
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    ndc = np.stack([(x + 0.5) / w * 2 - 1 - jitter[0], (y + 0.5) / h * 2 - 1 - jitter[1], np.ones_like(x, np.float64),
                    np.ones_like(x, np.float64)], -1)
    p = ndc @ mat(frame, "InvProjView").T
    p = p[..., :3] / p[..., 3:]
    eye = np.asarray(frame["ViewPos"][0], np.float64)
    d = p - eye
    return eye, d / np.linalg.norm(d, axis=-1, keepdims=True)


def world_triangles(light, mesh, position=None):
    v, idx = mesh
    pos = np.asarray(light["Position"] if position is None else position, np.float64)
    wv = float(light["Radius"]) * v.astype(np.float64) + pos
    return wv[idx[:, 0]], wv[idx[:, 1]], wv[idx[:, 2]]


def window_area(frame, a, b, c, w, h):
    """Signed window-space area (lower-left origin) of triangles a, b, c [n, 3]; all vertices must be in front of the eye."""
    pv = mat(frame, "ProjView")

    def win(p):
        q = np.concatenate([p, np.ones((len(p), 1))], 1) @ pv.T
        return np.stack([(q[:, 0] / q[:, 3] * 0.5 + 0.5) * w, (q[:, 1] / q[:, 3] * 0.5 + 0.5) * h], 1)
    A, B, C = win(a), win(b), win(c)
    return (B[:, 0] - A[:, 0]) * (C[:, 1] - A[:, 1]) - (B[:, 1] - A[:, 1]) * (C[:, 0] - A[:, 0])


def brute_force(scene, frame, w, h, gdepth, mesh):
    """float64 Moller-Trumbore over every triangle of every light, front faces by window-space winding, LESS against gdepth:
    (winner [h, w] (-1: none), min barycentric margin [h, w], depth gap to the runner-up [h, w])."""
    eye, d = pixel_rays(frame, w, h)
    d = d.reshape(-1, 3)
    best = np.full(len(d), np.inf)
    second = np.full(len(d), np.inf)
    winner = np.full(len(d), -1)
    margin = np.full(len(d), np.inf)
    pv = mat(frame, "ProjView")
    for li, L in enumerate(scene.lights):
        a, b, c = world_triangles(L, mesh)
        e1, e2 = b - a, c - a
        front = window_area(frame, a, b, c, w, h) > 0
        for t in range(len(a)):
            if not front[t]:
                continue
            pvec = np.cross(d, e2[t])
            det = pvec @ e1[t]
            tvec = eye - a[t]
            u = (pvec @ tvec) / det
            qvec = np.cross(tvec, e1[t])
            v = (d @ qvec) / det
            tt = (e2[t] @ qvec) / det
            hit = (u >= 0) & (v >= 0) & (u + v <= 1) & (tt >= 0)
            X = eye + d * tt[:, None]
            q = np.concatenate([X, np.ones((len(X), 1))], 1) @ pv.T
            depth = q[:, 2] / q[:, 3]
            ok = hit & (depth >= 0) & (depth <= 1) & (depth < gdepth.reshape(-1))
            m = np.minimum(np.minimum(u, v), 1 - u - v)
            closer = ok & (depth < best)
            second = np.where(closer, best, np.where(ok, np.minimum(second, depth), second))
            best = np.where(closer, depth, best)
            winner = np.where(closer, li * T + t, winner)
            margin = np.where(closer, m, margin)
            near_edge = hit & (np.abs(m) < 1e-4) & ~closer
            margin = np.where(near_edge, np.minimum(margin, np.abs(m)), margin)
    with np.errstate(invalid="ignore"):   # inf - inf where nothing was hit: no tie
        gap = np.nan_to_num(second - best, nan=np.inf)
    return winner.reshape(h, w), margin.reshape(h, w), gap.reshape(h, w)


# ---- the mesh table ---------------------------------------------------------------------------------------------------------
def test_mesh_table_is_the_float64_formula_rounded_once():
    v, idx = lo.sphere_mesh()
    assert v.shape == (169, 3) and idx.shape == (264, 3)
    f = np.float32
    d_lat, d_lon = f(np.pi) / f(12), f(2) * f(np.pi) / f(12)
    want = []
    for i in range(13):
        lat = f(np.pi) / f(2) - f(i) * d_lat
        xy, z = f(np.cos(np.float64(lat))), f(np.sin(np.float64(lat)))
        for j in range(13):
            lon = f(j) * d_lon
            want.append((xy * f(np.cos(np.float64(lon))), xy * f(np.sin(np.float64(lon))), z))
    assert np.array_equal(v, np.array(want, np.float32))
    # on the unit sphere within 4 ulp of 1 (each vertex is two rounded factors and one rounded product)
    r = np.linalg.norm(v.astype(np.float64), axis=1)
    assert np.abs(r - 1).max() <= 4 * np.spacing(np.float32(1))


def test_mesh_has_264_outward_triangles():
    v, idx = lo.sphere_mesh()
    assert set(np.unique(idx)) == set(range(1, 168))   # the first north-pole and the last south-pole vertex are never referenced
    a, b, c = (v[idx[:, k]].astype(np.float64) for k in range(3))
    n = np.cross(b - a, c - a)
    assert (np.einsum("ij,ij->i", n, a + b + c) > 0).all()
    assert (np.linalg.norm(n, axis=1) > 0).all()


# ---- the front-face rule ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("radius", [0.7, -0.7])
def test_front_face_rule_matches_window_winding(radius):
    mesh = lo.sphere_mesh()
    frame = frame_at()
    light = np.zeros(1, gt.GpuLight)[0]
    light["Radius"] = radius
    rng = np.random.default_rng(3)
    checked = 0
    for _ in range(6):
        light["Position"] = (rng.uniform(-1.5, 1.5), rng.uniform(-1.0, 1.0), rng.uniform(-6.0, -3.0))
        a, b, c = world_triangles(light, mesh)
        area = window_area(frame, a, b, c, W, H)
        eye = np.asarray(frame["ViewPos"][0], np.float64)
        # the kernel's rule: dot(e1 x e2, d) < 0 for a ray d from the eye to any point of the triangle's plane
        rule = np.einsum("ij,ij->i", np.cross(b - a, c - a), (a + b + c) / 3 - eye) < 0
        keep = np.abs(area) > 1e-9
        assert np.array_equal(rule[keep], area[keep] > 0)
        checked += keep.sum()
    assert checked > 6 * 200


def test_drawn_fragments_are_counter_clockwise(base_scene):
    mesh = lo.sphere_mesh()
    frame = frame_at()
    scene = with_lights(base_scene, [((0.3, 0.1, -4.0), (2.0, 1.0, 0.5), 0.8), ((-0.8, -0.2, -3.0), (0.2, 3.0, 0.4), -0.6)])
    _, _, winner = run(scene, frame)
    drawn = np.unique(winner[winner >= 0])
    assert len(drawn) > 50 and ((drawn // T) == 1).any()
    for wi in drawn:
        a, b, c = world_triangles(scene.lights[wi // T], mesh)
        t = wi % T
        assert window_area(frame, a[t:t + 1], b[t:t + 1], c[t:t + 1], W, H)[0] > 0


# ---- coverage -----------------------------------------------------------------------------------------------------------------
def test_coverage_matches_float64_brute_force(base_scene):
    mesh = lo.sphere_mesh()
    frame = frame_at(view_dir=(0.1, 0.05, -1.0))
    scene = with_lights(base_scene, [((0.4, 0.2, -4.0), (5.0, 4.5, 4.0), 0.9), ((-1.2, -0.3, -5.0), (1.0, 0.5, 0.3), 1.3),
                                     ((0.0, 0.8, -2.5), (0.3, 0.3, 3.0), 0.25), ((0.2, 0.0, -3.5), (2.0, 2.0, 2.0), 0.6)])
    gdepth = np.ones((H, W))
    gdepth[:, : W // 3] = 0.985   # a wall in front of some of the spheres on the left
    gb = blank_gbuffer()
    gb[0][...] = gdepth
    g, _, winner = run(scene, frame, gbuffer=gb)
    want, margin, gap = brute_force(scene, frame, W, H, gdepth, mesh)
    excluded = (margin < 1e-4) | (gap < 1e-6)
    assert excluded.sum() <= 0.05 * W * H, excluded.sum()   # pixels on a triangle edge or at a depth tie are not compared
    got = np.where(winner >= 0, winner, -1)
    assert np.array_equal(got[~excluded], want[~excluded])
    assert (want >= 0).sum() > 0.15 * W * H and (got // T == 3).any() and (got // T == 1).any()
    assert (g[0][winner >= 0] < gdepth[winner >= 0]).all()


def test_depth_test_against_the_gbuffer(base_scene):
    frame = frame_at()
    scene = with_lights(base_scene, [((0.0, 0.0, -4.0), (1.0, 2.0, 3.0), 1.0)])
    g_far, _, w_far = run(scene, frame, depth=1.0)
    drawn = w_far >= 0
    assert drawn.sum() > 100
    near = float(g_far[0][drawn].min())
    _, _, w_front = run(scene, frame, depth=near * 0.5)              # a surface in front of the whole sphere hides it
    assert (w_front == lo.UNTOUCHED).all()
    mid = float(np.median(g_far[0][drawn]))
    g_mid, _, w_mid = run(scene, frame, depth=mid)                   # a surface through the sphere: only what is in front
    assert np.array_equal(w_mid >= 0, drawn & (g_far[0] < mid))
    assert np.array_equal(g_mid[0][w_mid >= 0], g_far[0][w_mid >= 0])


def test_overlapping_spheres_resolve_by_depth_then_draw_order(base_scene):
    frame = frame_at()
    a = ((0.0, 0.0, -4.0), (1.0, 0.0, 0.0), 1.0)
    b = ((0.0, 0.0, -4.0), (0.0, 1.0, 0.0), 1.0)
    c = ((0.3, 0.0, -3.0), (0.0, 0.0, 1.0), 0.5)
    _, col, win = run(with_lights(base_scene, [a, b]), frame)
    assert (win >= 0).sum() > 100 and ((win[win >= 0] // T) == 0).all()                       # a tie keeps the first light
    assert np.array_equal(col[win >= 0][:, :3], np.tile([1.0, 0.0, 0.0], ((win >= 0).sum(), 1)))
    _, col, win = run(with_lights(base_scene, [a, c]), frame)
    assert ((win // T) == 1).sum() > 10 and ((win // T) == 0).sum() > 10                       # the nearer sphere in front
    _, col2, win2 = run(with_lights(base_scene, [c, a]), frame)
    assert np.array_equal(np.where(win >= 0, 1 - win // T, -1), np.where(win2 >= 0, win2 // T, -1))


def test_sphere_straddling_the_near_plane_is_clipped(base_scene):
    frame = frame_at()
    near = float(frame["NearPlane"][0])
    g, _, win = run(with_lights(base_scene, [((0.0, 0.0, -near - 0.05), (1.0, 1.0, 1.0), 0.3)]), frame)
    drawn = win >= 0
    assert not drawn.all()
    assert (g[0][drawn] >= 0).all() and (g[0][drawn] <= 1).all()
    _, _, win_whole = run(with_lights(base_scene, [((0.0, 0.0, -near - 0.5), (1.0, 1.0, 1.0), 0.3)]), frame)
    assert (win_whole >= 0).sum() > 0


def test_camera_inside_a_sphere_draws_nothing(base_scene):
    frame = frame_at()
    _, col, win = run(with_lights(base_scene, [((0.1, 0.0, -0.2), (1.0, 1.0, 1.0), 2.0)]), frame)
    assert (win == lo.SKY).all()
    assert np.allclose(col[..., :3], np.array([0.6, 0.7, 0.9], np.float32))


# ---- the skybox -------------------------------------------------------------------------------------------------------------
def cube_sky(n=16):
    faces = np.zeros((6, n, n, 4), np.float32)
    for f in range(6):
        faces[f, ..., 0] = f + 1
        faces[f, ..., 1] = np.arange(n)[None, :] / n
        faces[f, ..., 2] = np.arange(n)[:, None] / n
        faces[f, ..., 3] = 1
    return faces


def sky_dirs64(frame, w, h):
    x, y = np.meshgrid(np.arange(w), np.arange(h))
    ndc = np.stack([(x + 0.5) / w * 2 - 1, (y + 0.5) / h * 2 - 1, np.ones_like(x, np.float64), np.ones_like(x, np.float64)], -1)
    v = ndc @ mat(frame, "InvProjection").T
    v = v[..., :3] / v[..., 3:]
    return v @ mat(frame, "InvView")[:3, :3].T


@pytest.mark.parametrize("view_dir", [(0.0, 0.0, -1.0), (1.0, 0.9, -1.05), (-0.7, -1.0, 0.4)])
def test_sky_face_is_where_the_view_ray_leaves_the_cube(base_scene, view_dir):
    frame = frame_at(view_dir=view_dir, fov=100.0)
    faces = cube_sky()
    _, col, win = run(with_lights(base_scene, []), frame, sky=faces)
    assert (win == lo.SKY).all()
    d = sky_dirs64(frame, W, H)
    a = np.abs(d)
    face = np.argmax(a, -1) * 2 + (np.take_along_axis(d, np.argmax(a, -1)[..., None], -1)[..., 0] < 0)
    s = np.sort(a, -1)
    clear = s[..., 1] < 0.9 * s[..., 2]   # more than a texel from the cube's edges, where seamless filtering mixes faces
    got_face = np.rint(col[..., 0]).astype(int) - 1
    assert clear.sum() > 0.5 * W * H
    assert np.array_equal(got_face[clear], face[clear])


def test_sky_velocity_static_camera_is_zero(base_scene):
    frame = frame_at(view_dir=(0.3, 0.2, -1.0))
    g, _, _ = run(with_lights(base_scene, []), frame)
    assert np.abs(g[5]).max() < 1e-5


def test_sky_velocity_of_a_yaw_matches_float64_reprojection(base_scene):
    frame = frame_at(view_dir=(0.0, 0.0, -1.0))
    prev = frame_at(view_dir=(np.sin(0.08), 0.0, -np.cos(0.08)))
    frame["PrevView"] = prev["View"]
    g, _, _ = run(with_lights(base_scene, []), frame)
    d = sky_dirs64(frame, W, H)
    pv = d @ mat(frame, "PrevView")[:3, :3].T
    q = np.concatenate([pv, np.ones(pv.shape[:2] + (1,))], -1) @ mat(frame, "Projection").T
    x, y = np.meshgrid(np.arange(W), np.arange(H))
    ndc = np.stack([(x + 0.5) / W * 2 - 1, (y + 0.5) / H * 2 - 1], -1)
    want = (ndc - q[..., :2] / q[..., 3:]) * 0.5
    assert np.abs(want).max() > 0.02
    assert np.abs(g[5] - want).max() < 2e-4


# ---- light velocity -----------------------------------------------------------------------------------------------------------
def test_moved_light_velocity_is_the_projected_difference(base_scene):
    mesh = lo.sphere_mesh()
    frame = frame_at()
    delta = np.array([0.12, -0.05, 0.3])
    pos = np.array([0.2, 0.1, -4.0])
    scene = with_lights(base_scene, [(pos, (1.0, 1.0, 1.0), 1.0, pos - delta)])
    g, _, win = run(scene, frame)
    drawn = win >= 0
    assert drawn.sum() > 100
    eye, d = pixel_rays(frame, W, H)
    a, b, c = world_triangles(scene.lights[0], mesh)
    pvm, ppv = mat(frame, "ProjView"), mat(frame, "PrevProjView")
    errs = []
    for (y, x) in zip(*np.nonzero(drawn)):
        t = win[y, x] % T
        n = np.cross(b[t] - a[t], c[t] - a[t])
        X = eye + d[y, x] * (n @ (a[t] - eye)) / (n @ d[y, x])
        q, qp = pvm @ np.append(X, 1), ppv @ np.append(X - delta, 1)
        want = (q[:2] / q[3] - qp[:2] / qp[3]) * 0.5
        errs.append(np.abs(g[5][y, x] - want).max())
    assert max(errs) < 5e-4


# ---- idempotence ------------------------------------------------------------------------------------------------------------
def test_a_second_call_changes_nothing(base_scene):
    frame = frame_at(view_dir=(0.2, 0.1, -1.0))
    scene = with_lights(base_scene, [((0.0, 0.0, -4.0), (1.0, 2.0, 3.0), 1.0), ((0.5, 0.2, -3.0), (3.0, 2.0, 1.0), 0.4, (0.6, 0.2, -3.0))])
    g1, c1, _ = run(scene, frame, jitter=(0.01, -0.02), sky=cube_sky())
    g2, c2, _ = lo.lights_and_skybox(scene, frame, g1, c1, jitter=(0.01, -0.02), sky=cube_sky(), threads=4)
    for a, b in zip(g1 + (c1,), g2 + (c2,)):
        assert a.tobytes() == b.tobytes()
