"""The SSR / merge / TAA resolve oracle (oracle/oracle_ssr_taa.cpp) against a float64 restatement of the shaders and against
exact properties. CPU only."""
import numpy as np
import pytest

import ssr_taa_oracle as so
from idkengine_b200 import capi, scenes, vxgi

W, H = 23, 17


def frame_and_camera(w=W, h=H):
    _, cam = scenes.cornell_1k(threads=1)
    return scenes.camera_frame(cam, w, h)


def mat(frame, name):
    """GpuPerFrameData matrix as M with GLSL's M * v == v @ M."""
    f = frame[0] if frame.ndim else frame
    return np.asarray(f[name], np.float64).reshape(4, 4)


def decode_unit_vec(e):
    f = np.asarray(e, np.float64) * 2.0 - 1.0
    n = np.array([f[0], f[1], 1.0 - abs(f[0]) - abs(f[1])])
    t = max(-n[2], 0.0)
    n[0] += -t if n[0] >= 0 else t
    n[1] += -t if n[1] >= 0 else t
    return n / np.linalg.norm(n)


def synthetic_gbuffer(seed, w=W, h=H):
    """A smooth depth field in front of the camera, seeded normals, albedo, metallic (some below 0.001) and source colours;
    one sky pixel."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    depth = (0.93 + 0.03 * np.sin(xx * 0.4) * np.cos(yy * 0.3)).astype(np.float32)
    depth[0, 0] = 1.0
    n = rng.normal(size=(h, w, 3))
    n[..., 2] = np.abs(n[..., 2]) + 0.5
    nrg = vxgi.encode_unit_vec(n / np.linalg.norm(n, axis=-1, keepdims=True))
    albedo = rng.random((h, w, 3), dtype=np.float32)
    mr = rng.random((h, w, 2), dtype=np.float32)
    mr[rng.random((h, w)) < 0.15, 0] = 0.0005
    src = np.concatenate([rng.random((h, w, 3), dtype=np.float32) * 2.0, np.ones((h, w, 1), np.float32)], -1)
    return depth, nrg, albedo, mr, src


def bilinear64(img, u, v):
    h, w = img.shape[:2]
    px, py = u * w - 0.5, v * h - 0.5
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = px - x0, py - y0
    x0, y0 = int(x0), int(y0)
    cx = lambda x: min(max(x, 0), w - 1)
    cy = lambda y: min(max(y, 0), h - 1)
    a = img[cy(y0), cx(x0)] * (1 - fx) + img[cy(y0), cx(x0 + 1)] * fx
    b = img[cy(y0 + 1), cx(x0)] * (1 - fx) + img[cy(y0 + 1), cx(x0 + 1)] * fx
    return a * (1 - fy) + b * fy


def nearest64(img, u, v):
    h, w = img.shape[:2]
    return img[min(max(int(np.floor(v * h)), 0), h - 1), min(max(int(np.floor(u * w)), 0), w - 1)]


def ssr64(frame, st, sky_color, depth, nrg, albedo, mr, src):
    """SSR/compute.glsl in float64 (constant sky) -> rgba float64 [H, W, 4] before the half store."""
    P, IP, IV = mat(frame, "Projection"), mat(frame, "InvProjection"), mat(frame, "InvView")
    h, w = depth.shape
    out = np.zeros((h, w, 4))

    def project(p):
        q = np.append(p, 1.0) @ P
        q = q[:3] / q[3]
        return np.array([q[0] * 0.5 + 0.5, q[1] * 0.5 + 0.5, q[2]])

    for y in range(h):
        for x in range(w):
            if mr[y, x, 0] < 0.001 or depth[y, x] == 1.0:
                continue
            u, v = (x + 0.5) / w, (y + 0.5) / h
            q = np.array([u * 2 - 1, v * 2 - 1, depth[y, x], 1.0]) @ IP
            frag = q[:3] / q[3]
            normal = IV[:3, :3] @ decode_unit_vec(nrg[y, x])
            i = frag / np.linalg.norm(frag)
            r = i - 2.0 * np.dot(normal, i) * normal
            step = r * st.MaxDist / st.SampleCount
            p = frag.copy()
            color = None
            for _ in range(st.SampleCount):
                p = p + step
                ps = project(p)
                if ps[0] >= 1 or ps[1] >= 1 or ps[0] < 0 or ps[1] < 0 or ps[2] > 1:
                    color = np.zeros(3)
                    break
                if ps[2] > nearest64(depth, ps[0], ps[1]):
                    d = step * 0.5
                    p = p - d * 0.5
                    for _ in range(1, st.BinarySearchCount):
                        ps = project(p)
                        dd = nearest64(depth, ps[0], ps[1])
                        d = d * 0.5
                        p = p - d if ps[2] > dd else p + d
                    color = bilinear64(src[..., :3].astype(np.float64), ps[0], ps[1])
                    break
            if color is None:
                color = np.asarray(sky_color, np.float64)
            out[y, x, :3] = color * mr[y, x, 0] * albedo[y, x]
            out[y, x, 3] = 1.0
    return out


def catmull_rom64(img, u, v):
    h, w = img.shape[:2]

    def axis(t, n):
        ts = 1.0 / n
        sp = t / ts
        t1 = np.floor(sp - 0.5) + 0.5
        f = sp - t1
        w0 = f * (-0.5 + f * (1.0 - 0.5 * f))
        w1 = 1.0 + f * f * (-2.5 + 1.5 * f)
        w2 = f * (0.5 + f * (2.0 - 1.5 * f))
        w3 = f * f * (-0.5 + 0.5 * f)
        return (w0, w1 + w2, w3), ((t1 - 1) * ts, (t1 + w2 / (w1 + w2)) * ts, (t1 + 2) * ts)
    (wx, px), (wy, py) = axis(u, w), axis(v, h)
    return sum(bilinear64(img, px[i], py[j]) * wx[i] * wy[j] for j in range(3) for i in range(3))


def taa64(st, color, depth, velocity, history):
    """TAAResolve/compute.glsl in float64 -> rgb [H, W, 3] before the half store."""
    H_, W_ = history.shape[:2]
    c = color[..., :3].astype(np.float64)
    hist = history[..., :3].astype(np.float64)
    out = np.zeros((H_, W_, 3))
    for y in range(H_):
        for x in range(W_):
            u, v = (x + 0.5) / W_, (y + 0.5) / H_
            if st.IsNaiveTaa:
                vel = nearest64(velocity, u, v)
                b = 1.0 / st.SampleCount
                out[y, x] = bilinear64(hist, u - vel[0], v - vel[1]) * (1 - b) + bilinear64(c, u, v) * b
                continue
            lo, hi, best, md = np.full(3, np.inf), np.full(3, -np.inf), (u, v), np.inf
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    nu, nv = (x + dx + 0.5) / W_, (y + dy + 0.5) / H_
                    t = bilinear64(c, nu, nv)
                    lo, hi = np.minimum(lo, t), np.maximum(hi, t)
                    d = nearest64(depth, nu, nv)
                    if d < md:
                        md, best = d, (nu, nv)
            cur = bilinear64(c, u, v)
            vel = nearest64(velocity, *best)
            hu, hv = u - vel[0], v - vel[1]
            if hu >= 1 or hv >= 1 or hu < 0 or hv < 0:
                out[y, x] = cur
                continue
            hc = np.minimum(np.maximum(catmull_rom64(hist, hu, hv), lo), hi)
            dist = abs(0.5 - (hu * W_ - np.floor(hu * W_))) + abs(0.5 - (hv * H_ - np.floor(hv * H_)))
            b = 1.0 / st.SampleCount
            b = b + (1.0 - b) * dist * st.PreferAliasingOverBlur
            out[y, x] = hc * (1 - b) + cur * b
    return out


def test_ssr_matches_float64():
    frame = frame_and_camera()
    sky = (0.3, 0.5, 0.9)
    for seed, st in ((1, capi.IdkPtSsrSettings(30, 8, 5.0)), (2, capi.IdkPtSsrSettings(12, 0, 2.0)), (3, capi.IdkPtSsrSettings(64, 1, 0.5))):
        d, n, a, mr, src = synthetic_gbuffer(seed)
        merged, ssr = so.ssr(frame, st, capi.sky_desc(sky), d, n, a, mr, src)
        want = ssr64(frame, st, sky, d, n, a, mr, src)
        got = ssr.astype(np.float64)
        close = np.all(np.abs(got - want) <= 2e-3 * np.abs(want) + 1e-3, -1)
        assert close.mean() > 0.95, (seed, close.mean())
        hit = (want[..., 3] == 1) & np.any(np.abs(want[..., :3] - np.asarray(sky) * mr[..., :1] * a) > 1e-3, -1) & np.any(want[..., :3] != 0, -1)
        assert hit.any()                                   # some rays hit the depth field
        # the merge: the source plus the SSR value as its half holds it, alpha 1
        assert np.array_equal(merged[..., :3], src[..., :3] + ssr[..., :3].astype(np.float32)) and np.all(merged[..., 3] == 1)


def test_ssr_early_out_is_zero_with_alpha_zero():
    frame = frame_and_camera()
    d, n, a, mr, src = synthetic_gbuffer(4)
    _, ssr = so.ssr(frame, capi.default_ssr_settings(), capi.sky_desc((1.0, 1.0, 1.0)), d, n, a, mr, src)
    off = (mr[..., 0] < 0.001) | (d == 1.0)
    assert off.any() and (~off).any()
    assert np.all(ssr[off].view(np.uint16) == 0)
    assert np.all(ssr[~off][:, 3] == 1)


def mirror_gbuffer(frame, r_view, metallic=0.75, w=W, h=H):
    """One mirror pixel at the image centre (depth 0.95) whose normal reflects the view ray into r_view (view space); every other
    pixel is sky (depth 1)."""
    IP, IV = mat(frame, "InvProjection"), mat(frame, "InvView")
    x, y = w // 2, h // 2
    depth = np.ones((h, w), np.float32)
    depth[y, x] = 0.95
    q = np.array([((x + 0.5) / w) * 2 - 1, ((y + 0.5) / h) * 2 - 1, 0.95, 1.0]) @ IP
    i = q[:3] / q[3]
    i /= np.linalg.norm(i)
    r = np.asarray(r_view, np.float64) - 0.3 * i                         # and towards the camera: the depth falls along the ray
    r /= np.linalg.norm(r)
    nv = (r - i) / np.linalg.norm(r - i)
    nw = np.linalg.solve(IV[:3, :3], nv)
    nrg = np.zeros((h, w, 2), np.float32)
    nrg[y, x] = vxgi.encode_unit_vec(nw / np.linalg.norm(nw))
    albedo = np.full((h, w, 3), 0.5, np.float32)
    albedo[y, x] = (0.9, 0.6, 0.3)
    mr = np.zeros((h, w, 2), np.float32)
    mr[y, x, 0] = metallic
    src = np.ones((h, w, 4), np.float32)
    return (depth, nrg, albedo, mr, src), (y, x)


def test_ssr_reflection_leaving_the_screen_is_zero_and_a_short_one_sees_the_sky():
    frame = frame_and_camera()
    sky = np.array([0.3, 0.5, 0.9], np.float32)
    g, (y, x) = mirror_gbuffer(frame, (1.0, 0.0, 0.0))
    _, ssr = so.ssr(frame, capi.IdkPtSsrSettings(30, 8, 50.0), capi.sky_desc(tuple(sky)), *g)
    assert np.all(ssr[y, x] == np.array([0, 0, 0, 1], np.float16))
    _, ssr = so.ssr(frame, capi.IdkPtSsrSettings(30, 8, 1e-3), capi.sky_desc(tuple(sky)), *g)
    want = ((sky * np.float32(0.75)) * g[2][y, x]).astype(np.float16)
    assert np.array_equal(ssr[y, x, :3].view(np.uint16), want.view(np.uint16)) and ssr[y, x, 3] == 1


def test_binary_search_count_0_and_1_read_the_hit_step():
    frame = frame_and_camera()
    d, n, a, mr, src = synthetic_gbuffer(5)
    sky = capi.sky_desc((0.0, 0.0, 0.0))
    r0 = so.ssr(frame, capi.IdkPtSsrSettings(30, 0, 5.0), sky, d, n, a, mr, src)[1]
    r1 = so.ssr(frame, capi.IdkPtSsrSettings(30, 1, 5.0), sky, d, n, a, mr, src)[1]
    r8 = so.ssr(frame, capi.IdkPtSsrSettings(30, 8, 5.0), sky, d, n, a, mr, src)[1]
    assert np.array_equal(r0.view(np.uint16), r1.view(np.uint16))
    assert not np.array_equal(r0.view(np.uint16), r8.view(np.uint16))


def taa_inputs(seed, rw, rh):
    rng = np.random.default_rng(seed)
    color = np.concatenate([rng.random((rh, rw, 3), dtype=np.float32) * 3.0 + 0.05, np.ones((rh, rw, 1), np.float32)], -1)
    depth = rng.random((rh, rw), dtype=np.float32)
    velocity = ((rng.random((rh, rw, 2)) - 0.5) * 0.08).astype(np.float32)
    return color, depth, velocity


@pytest.mark.parametrize("scale", [1.0, 0.6, 0.5])
@pytest.mark.parametrize("naive, prefer, samples", [(0, 0.25, 6), (0, 1.0, 1), (1, 0.25, 6), (0, 0.0, 6)])
def test_taa_matches_float64_over_frames(scale, naive, prefer, samples):
    rw, rh = max(1, int(W * scale)), max(1, int(H * scale))
    st = capi.IdkPtTaaSettings(naive, prefer, samples)
    history = np.zeros((H, W, 4), np.float16)
    for frame in range(3):
        color, depth, velocity = taa_inputs(10 + frame, rw, rh)
        want = taa64(st, color, depth, velocity, history.astype(np.float64))
        history = so.taa_resolve(st, color, depth, velocity, history)
        got = history[..., :3].astype(np.float64)
        assert np.all(history[..., 3] == 1)
        assert np.allclose(got, want, rtol=2e-3, atol=1e-3), np.abs(got - want).max()


def test_taa_off_screen_history_uv_returns_the_current_tap():
    color, depth, _ = taa_inputs(3, W, H)
    velocity = np.full((H, W, 2), 2.0, np.float32)
    velocity[::2, :, 0] = -1.5
    out = so.taa_resolve(capi.default_taa_settings(), color, depth, velocity, np.full((H, W, 4), 7.0, np.float16))
    assert np.array_equal(out[..., :3], color[..., :3].astype(np.float16)) and np.all(out[..., 3] == 1)


def test_naive_taa_with_one_sample_returns_the_current_tap():
    color, depth, velocity = taa_inputs(4, W, H)
    out = so.taa_resolve(capi.IdkPtTaaSettings(1, 0.25, 1), color, depth, velocity, np.full((H, W, 4), 5.0, np.float16))
    assert np.array_equal(out[..., :3], color[..., :3].astype(np.float16)) and np.all(out[..., 3] == 1)


def test_zero_history_is_fully_clamped_on_the_first_frame():
    color, depth, _ = taa_inputs(5, W, H)
    velocity = np.zeros((H, W, 2), np.float32)
    out = so.taa_resolve(capi.IdkPtTaaSettings(0, 0.0, 6), color, depth, velocity, np.zeros((H, W, 4), np.float16))
    c = color[..., :3]
    f32 = np.float32

    def tap(dx, dy):   # the fp32 bilinear rule at the neighbour's uv, vectorised
        yy, xx = np.mgrid[0:H, 0:W]
        px = ((xx + dx).astype(f32) + f32(0.5)) / f32(W) * f32(W) - f32(0.5)
        py = ((yy + dy).astype(f32) + f32(0.5)) / f32(H) * f32(H) - f32(0.5)
        x0, y0 = np.floor(px), np.floor(py)
        fx, fy = (px - x0)[..., None], (py - y0)[..., None]
        x0, y0 = x0.astype(int), y0.astype(int)
        t = lambda y, x: c[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)]
        a = t(y0, x0) * (f32(1) - fx) + t(y0, x0 + 1) * fx
        b = t(y0 + 1, x0) * (f32(1) - fx) + t(y0 + 1, x0 + 1) * fx
        return a * (f32(1) - fy) + b * fy
    lo = np.min(np.stack([tap(dx, dy) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]), 0)
    b = f32(1.0) / f32(6.0)
    want = (lo * (f32(1.0) - b) + tap(0, 0) * b).astype(np.float16)
    assert np.array_equal(out[..., :3].view(np.uint16), want.view(np.uint16))
