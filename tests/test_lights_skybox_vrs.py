"""The light spheres and the skybox under the shading-rate image (DESIGN.md 8f.1i, VRS) on the CPU: the oracle against the
per-pixel oracle and an independent float64 restatement of the fragment-centre rules.

As in tests/test_lights_skybox.py the oracle reads a hand-made G-buffer over the Cornell box's scene record, with its own lights
and cameras; the rate images come from the classifier oracle (five rates) or are written directly."""
import copy

import numpy as np
import pytest

import lights_skybox_oracle as lo
import lights_skybox_vrs_oracle as lvo
import vrs_oracle as vo
from idkengine_b200 import gpu_types as gt
from idkengine_b200 import host, scenes
from test_vrs_gpu import FIVE, five_rate_inputs
from vxgi_ref64 import decode_unit_vec64

T = lo.SPHERE_TRIANGLES
JIT = (0.0123, -0.0311)
SIZES = [(80, 48), (97, 61)]   # 97 x 61: coarse fragments cross the right and bottom edges


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


LIGHTS = [((0.3, 0.1, -4.0), (2.0, 1.0, 0.5), 0.9, (0.2, 0.15, -4.1)), ((-0.9, -0.3, -3.0), (0.2, 3.0, 0.4), 0.6),
          ((0.6, 0.5, -2.5), (0.3, 0.3, 3.0), 0.25, (0.65, 0.5, -2.5)), ((-0.2, 0.6, -5.0), (4.0, 4.0, 4.0), 0.7)]


def frame_at(w, h, view_dir=(0.0, 0.0, -1.0), fov=60.0, yaw=0.06):
    """A camera at the origin whose previous view looked yaw radians to the side (the sky moves)."""
    f = host.make_per_frame_data((0.0, 0.0, 0.0), view_dir, w, h, fov)
    c, s = np.cos(yaw), np.sin(yaw)
    vd = np.asarray(view_dir, np.float64)
    prev = host.make_per_frame_data((0.0, 0.0, 0.0), (c * vd[0] + s * vd[2], vd[1], -s * vd[0] + c * vd[2]), w, h, fov)
    f["PrevView"], f["PrevProjView"] = prev["View"], prev["ProjView"]
    f["DeltaRenderTime"] = 1.0
    return f


def cube_sky(n=16):
    """Face f has red f + 1 and a gradient in green and blue, so a sky colour names its face."""
    faces = np.zeros((6, n, n, 4), np.float32)
    for f in range(6):
        faces[f, ..., 0] = f + 1
        faces[f, ..., 1] = np.arange(n)[None, :] / n
        faces[f, ..., 2] = np.arange(n)[:, None] / n
        faces[f, ..., 3] = 1
    return faces


def gbuffer(w, h):
    """Depth 1 with a wall at 0.985 over the left third; the other planes constant."""
    depth = np.ones((h, w), np.float32)
    depth[:, : w // 3] = 0.985
    return (depth, np.zeros((h, w, 2), np.float32), np.full((h, w, 3), 0.25, np.float32), np.full((h, w, 2), 0.5, np.float32),
            np.zeros((h, w, 3), np.float32), np.zeros((h, w, 2), np.float32))


def five_rates(w, h, seed=1):
    """The classifier oracle's image of inputs that give every palette index (test_vrs_gpu.five_rate_inputs)."""
    color, velocity = five_rate_inputs(w, h, seed)
    return vo.shading_rate(frame_at(w, h), FIVE, color, velocity)


def rate_image(kind, w, h):
    if kind == "five":
        return five_rates(w, h)
    return np.full(lvo.tiles_of(w, h), {"1x1": 0, "4x4": 4}[kind], np.uint8)


def run_both(scene, frame, rates, w, h, jitter=JIT, sky=None):
    """(per-pixel oracle, VRS oracle) over the same G-buffer and lit image; each is (gbuffer planes, colour, winner)."""
    g = gbuffer(w, h)
    color = np.full((h, w, 4), 0.125, np.float32)
    sky = cube_sky() if sky is None else sky
    per_pixel = lo.lights_and_skybox(scene, frame, g, color, jitter=jitter, sky=sky, threads=4)
    coarse = lvo.lights_and_skybox_vrs(scene, frame, g, color, rates, jitter=jitter, sky=sky, threads=4)
    return per_pixel, coarse


def mat(frame, name):
    return np.asarray(frame[name][0], np.float64).reshape(4, 4).T


def centres(rates, w, h):
    """float64 fragment centres (xc, yc) [h, w] and the fragment table of lvo.fragment_of."""
    fr = lvo.fragment_of(rates, w, h)
    return fr[..., 0] + 0.5 * fr[..., 2], fr[..., 1] + 0.5 * fr[..., 3], fr


def rays64(frame, px, py, w, h, jitter):
    """float64 eye and unit directions through window points (px, py) [h, w] (rule 2's construction)."""
    ndc = np.stack([px / w * 2 - 1 - jitter[0], py / h * 2 - 1 - jitter[1], np.ones_like(px), np.ones_like(px)], -1)
    p = ndc @ mat(frame, "InvProjView").T
    p = p[..., :3] / p[..., 3:]
    eye = np.asarray(frame["ViewPos"][0], np.float64)
    d = p - eye
    return eye, d / np.linalg.norm(d, axis=-1, keepdims=True)


def sky_dirs64(frame, px, py, w, h):
    ndc = np.stack([px / w * 2 - 1, py / h * 2 - 1, np.ones_like(px), np.ones_like(px)], -1)
    v = ndc @ mat(frame, "InvProjection").T
    v = v[..., :3] / v[..., 3:]
    return v @ mat(frame, "InvView")[:3, :3].T


# ---- full rate and coverage -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("jitter", [None, JIT])
def test_all_full_rate_is_the_per_pixel_oracle(base_scene, w, h, jitter):
    scene = with_lights(base_scene, LIGHTS)
    frame = frame_at(w, h, view_dir=(0.1, 0.05, -1.0))
    (pg, pc, pw), (cg, cc, cw) = run_both(scene, frame, rate_image("1x1", w, h), w, h, jitter=jitter)
    assert (pw >= 0).sum() > 0.1 * w * h and (pw == lo.SKY).sum() > 0.1 * w * h
    for a, b in zip(pg + (pc, pw), cg + (cc, cw)):
        assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("kind", ["five", "4x4"])
def test_coarse_rates_keep_coverage_depth_and_emissive(base_scene, w, h, kind):
    scene = with_lights(base_scene, LIGHTS)
    frame = frame_at(w, h, view_dir=(0.1, 0.05, -1.0))
    rates = rate_image(kind, w, h)
    if kind == "five":
        assert set(np.unique(rates)) == {0, 1, 2, 3, 4}
    (pg, pc, pw), (cg, cc, cw) = run_both(scene, frame, rates, w, h)
    assert np.array_equal(pw, cw)                                          # light / sky / untouched and the winning triangle
    for k in (0, 2, 3, 4):                                                 # depth, emissive; albedo and metallic never written
        assert pg[k].tobytes() == cg[k].tobytes()
    assert np.array_equal(cc[pw >= 0], pc[pw >= 0])                        # the light's colour
    # the centre moved the values: normals and velocities differ from the per-pixel call somewhere
    assert (cg[1] != pg[1]).any() and (cg[5] != pg[5]).any()


# ---- one value per (triangle, coarse fragment) --------------------------------------------------------------------------------
def own_face(frame, w, h):
    """The face axis of each pixel's own float64 sky direction and whether it is clear of a cube edge by 1e-6."""
    x, y = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    a = np.abs(sky_dirs64(frame, x, y, w, h))
    s = np.sort(a, -1)
    return np.argmax(a, -1), s[..., 1] < s[..., 2] * (1 - 1e-6)


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("kind", ["five", "4x4"])
def test_pixels_of_a_fragment_share_the_shaded_values(base_scene, w, h, kind):
    scene = with_lights(base_scene, LIGHTS)
    frame = frame_at(w, h, view_dir=(0.7, 0.55, -0.8), fov=90.0)   # cube edges on screen
    rates = rate_image(kind, w, h)
    _, (g, col, win) = run_both(scene, frame, rates, w, h)
    fr = lvo.fragment_of(rates, w, h)
    face, clear = own_face(frame, w, h)
    key = np.where(win >= 0, win, np.where(win == lo.SKY, -10 - face, -1))
    fid = fr[..., 1] * w + fr[..., 0]
    vals = np.concatenate([g[1], g[5], col], -1).reshape(h * w, -1)
    groups, shared = {}, 0
    for p in range(h * w):
        y, x = divmod(p, w)
        if key[y, x] == -1 or (win[y, x] == lo.SKY and not clear[y, x]):
            continue
        k = (fid[y, x], key[y, x])
        if k in groups:
            assert vals[p].tobytes() == vals[groups[k]].tobytes(), (x, y, k)
            shared += 1
        else:
            groups[k] = p
    assert shared > 0.3 * w * h
    assert sum(1 for (_, k) in groups if k >= 0) > 20 and sum(1 for (_, k) in groups if k <= -10) > 20


# ---- the centre values against float64 ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("kind", ["five", "4x4"])
def test_light_normal_and_velocity_are_the_winning_plane_at_the_centre_ray(base_scene, w, h, kind):
    scene = with_lights(base_scene, LIGHTS)
    frame = frame_at(w, h, view_dir=(0.1, 0.05, -1.0))
    rates = rate_image(kind, w, h)
    _, (g, _, win) = run_both(scene, frame, rates, w, h)
    xc, yc, _ = centres(rates, w, h)
    eye, dc = rays64(frame, xc, yc, w, h, JIT)
    _, dp = rays64(frame, *np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5), w, h, JIT)
    v, idx = lo.sphere_mesh()
    pvm, ppv = mat(frame, "ProjView"), mat(frame, "PrevProjView")
    lit = np.argwhere(win >= 0)
    assert len(lit) > 0.1 * w * h
    n_err, v_err, moved = [], [], 0
    for y, x in lit:
        L = scene.lights[win[y, x] // T]
        tri = idx[win[y, x] % T]
        pos, prev, r = (np.asarray(L[k], np.float64) for k in ("Position", "PrevPosition", "Radius"))
        a, b, c = (float(r) * v[i].astype(np.float64) + pos for i in tri)
        n = np.cross(b - a, c - a)
        X = eye + dc[y, x] * (n @ (a - eye)) / (n @ dc[y, x])          # the plane at the centre ray, t < 0 included
        Xp = eye + dp[y, x] * (n @ (a - eye)) / (n @ dp[y, x])         # ... and at the pixel's own ray
        want_n, pix_n = (X - pos) / r, (Xp - pos) / r
        got_n = decode_unit_vec64(g[1][y, x])
        n_err.append(np.arccos(np.clip(got_n @ want_n / np.linalg.norm(want_n), -1, 1)))
        moved += np.arccos(np.clip(want_n @ pix_n / np.linalg.norm(want_n) / np.linalg.norm(pix_n), -1, 1)) > 0.05
        qp = ppv @ np.append(X - pos + prev, 1)
        ndc = np.array([xc[y, x] / w * 2 - 1 - JIT[0], yc[y, x] / h * 2 - 1 - JIT[1]])
        v_err.append(np.abs(g[5][y, x] - (ndc - qp[:2] / qp[3]) * 0.5).max())
    assert max(n_err) < 0.02, max(n_err)         # R8 octahedral quantisation
    assert max(v_err) < 5e-4, max(v_err)
    assert moved > 10                            # pixels whose own normal is more than 0.05 rad from the centre's


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("view_dir", [(0.7, 0.55, -0.8), (-0.7, -1.0, 0.4)])
def test_sky_face_and_reprojection_are_the_centre_direction(base_scene, w, h, view_dir):
    frame = frame_at(w, h, view_dir=view_dir, fov=100.0)
    rates = five_rates(w, h)
    _, (g, col, win) = run_both(with_lights(base_scene, []), frame, rates, w, h)
    sky = win == lo.SKY                            # all but the wall over the left third
    assert sky.sum() > 0.6 * w * h and not (win >= 0).any()
    xc, yc, _ = centres(rates, w, h)
    d = sky_dirs64(frame, xc, yc, w, h)
    a = np.abs(d)
    face = np.argmax(a, -1) * 2 + (np.take_along_axis(d, np.argmax(a, -1)[..., None], -1)[..., 0] < 0)
    s = np.sort(a, -1)
    clear = sky & (s[..., 1] < 0.9 * s[..., 2])  # more than a texel from the cube's edges, where seamless filtering mixes faces
    assert clear.sum() > 0.4 * w * h
    assert np.array_equal(np.rint(col[..., 0]).astype(int)[clear] - 1, face[clear])
    pv = d @ mat(frame, "PrevView")[:3, :3].T
    q = np.concatenate([pv, np.ones(pv.shape[:2] + (1,))], -1) @ mat(frame, "Projection").T
    ndc = np.stack([xc / w * 2 - 1, yc / h * 2 - 1], -1)
    want = (ndc - q[..., :2] / q[..., 3:]) * 0.5
    assert np.abs(want[sky]).max() > 0.02
    assert np.abs(g[5] - want)[sky].max() < 2e-4
    # the centre's values are not the pixel's: the per-pixel reprojection is farther off in coarse fragments
    x, y = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dp = sky_dirs64(frame, x, y, w, h) @ mat(frame, "PrevView")[:3, :3].T
    qp = np.concatenate([dp, np.ones(dp.shape[:2] + (1,))], -1) @ mat(frame, "Projection").T
    per_pixel = (np.stack([x / w * 2 - 1, y / h * 2 - 1], -1) - qp[..., :2] / qp[..., 3:]) * 0.5
    assert (np.abs(g[5] - per_pixel).max(-1)[sky] > 1e-3).sum() > 0.05 * w * h


# ---- idempotence --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", SIZES)
def test_a_second_call_changes_nothing(base_scene, w, h):
    scene = with_lights(base_scene, LIGHTS)
    frame = frame_at(w, h, view_dir=(0.2, 0.1, -1.0))
    rates = five_rates(w, h)
    _, (g1, c1, _) = run_both(scene, frame, rates, w, h)
    g2, c2, _ = lvo.lights_and_skybox_vrs(scene, frame, g1, c1, rates, jitter=JIT, sky=cube_sky(), threads=4)
    for a, b in zip(g1 + (c1,), g2 + (c2,)):
        assert a.tobytes() == b.tobytes()
