"""An independent float64 restatement of the sky generators (DESIGN.md 8f.1j) in numpy, vectorised over texels: the texel
directions, AtmosphericScattering/compute.glsl and UnprojectEquirectangular/compute.glsl with the exact functions (np.exp,
np.arctan2, np.arcsin, **) in place of the library's polynomials. tests/test_sky.py holds the fp32 oracle to it within
tolerances derived from fp32 rounding.

Besides the colours, the atmosphere returns per texel what the tolerance needs: the largest optical depth of any attenuation
term, and masks of the texels where fp32 cannot follow float64 (a ray-sphere discriminant within 1e-3 of zero, where the two
may take different branches of Rsi; an exp argument beyond fp32's range)."""
import numpy as np

# GetWorldSpaceDirection(ndc, face), Math.glsl:17-39: each component as a function of (x, y) = ndc
_FACES = [lambda x, y, o: (o, -y, -x), lambda x, y, o: (-o, -y, x), lambda x, y, o: (x, o, y),
          lambda x, y, o: (x, -o, -y), lambda x, y, o: (x, -y, o), lambda x, y, o: (-x, -y, -o)]


def directions(n):
    """Normalised texel directions, float64 [6, n, n, 3] (face, row y, column x)."""
    c = (np.arange(n, dtype=np.float64) + 0.5) / n * 2.0 - 1.0
    x, y = np.meshgrid(c, c)                  # x varies along columns, y along rows
    one = np.ones_like(x)
    d = np.stack([np.stack(f(x, y, one), -1) for f in _FACES])
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def _rsi(r0, rd, sr):
    a = np.sum(rd * rd, -1)
    b = 2.0 * np.sum(rd * r0, -1)
    c = np.sum(r0 * r0, -1) - sr * sr
    d = b * b - 4.0 * a * c
    fragile = np.abs(d) <= 1e-3 * (b * b + np.abs(4.0 * a * c))
    sq = np.sqrt(np.maximum(d, 0.0))
    miss = d < 0.0
    return np.where(miss, 1e5, (-b - sq) / (2.0 * a)), np.where(miss, -1e5, (-b + sq) / (2.0 * a)), fragile


def atmosphere(n, i_steps=40, j_steps=8, intensity=15.0, azimuth=0.0, elevation=0.0):
    """-> (rgb float64 [6, n, n, 3], max optical depth [6, n, n], fragile mask, overflow mask)."""
    r = directions(n).reshape(-1, 3)
    sun = np.array([np.sin(elevation) * np.cos(azimuth), np.cos(elevation), np.sin(elevation) * np.sin(azimuth)])
    sun = sun / np.linalg.norm(sun)
    i_sun = max(intensity, 0.0)
    r0 = np.array([0.0, 6376e3, 0.0])
    r_planet, r_atmos = 6371e3, 6471e3
    k_rlh = np.array([5.5e-6, 13.0e-6, 22.4e-6])
    k_mie, sh_rlh, sh_mie, g = 21e-6, 8e3, 1.2e3, 0.758
    m = len(r)
    px, py, fragile = _rsi(r0[None], r, r_atmos)
    outside = px > py
    qx, _, f2 = _rsi(r0[None], r, r_planet)
    fragile |= f2
    py = np.minimum(py, qx)
    step = (py - px) / i_steps
    mu = r @ sun
    gg = g * g
    p_rlh = 3.0 / (16.0 * np.pi) * (1.0 + mu * mu)
    p_mie = 3.0 / (8.0 * np.pi) * ((1.0 - gg) * (mu * mu + 1.0)) / ((1.0 + gg - 2.0 * mu * g) ** 1.5 * (2.0 + gg))
    tot_rlh, tot_mie = np.zeros((m, 3)), np.zeros((m, 3))
    od_rlh, od_mie = np.zeros(m), np.zeros(m)
    tau = np.zeros(m)
    overflow = np.zeros(m, bool)
    t = np.zeros(m)
    for _ in range(i_steps):
        pos = r0[None] + r * (t + step * 0.5)[:, None]
        h = np.linalg.norm(pos, axis=-1) - r_planet
        overflow |= -h / sh_mie > 87.0
        step_rlh = np.exp(-h / sh_rlh) * step
        step_mie = np.exp(-h / sh_mie) * step
        od_rlh += step_rlh
        od_mie += step_mie
        _, sy, f3 = _rsi(pos, np.broadcast_to(sun, pos.shape), r_atmos)
        fragile |= f3
        j_step = sy / j_steps
        j_rlh, j_mie, jt = np.zeros(m), np.zeros(m), np.zeros(m)
        for _ in range(j_steps):
            jp = pos + sun[None] * (jt + j_step * 0.5)[:, None]
            jh = np.linalg.norm(jp, axis=-1) - r_planet
            overflow |= -jh / sh_mie > 87.0
            j_rlh += np.exp(-jh / sh_rlh) * j_step
            j_mie += np.exp(-jh / sh_mie) * j_step
            jt += j_step
        od = k_mie * (od_mie + j_mie)[:, None] + k_rlh[None] * (od_rlh + j_rlh)[:, None]
        tau = np.maximum(tau, np.abs(od).max(-1))
        attn = np.exp(-od)
        tot_rlh += step_rlh[:, None] * attn
        tot_mie += step_mie[:, None] * attn
        t += step
    rgb = i_sun * (p_rlh[:, None] * k_rlh[None] * tot_rlh + (p_mie * k_mie)[:, None] * tot_mie)
    rgb[outside] = 0.0
    shape = (6, n, n)
    return rgb.reshape(shape + (3,)), tau.reshape(shape), fragile.reshape(shape), overflow.reshape(shape)


def srgb_to_linear(s):
    return np.where(s < 0.04045, s / 12.92, ((s + 0.055) / 1.055) ** 2.4)


def equirect_uv(d):
    """SampleSphericalMap with its rounded constants, float64: (u, v) of directions [..., 3]."""
    return np.arctan2(d[..., 2], d[..., 0]) * 0.1591 + 0.5, np.arcsin(np.clip(d[..., 1], -1.0, 1.0)) * 0.3183 + 0.5


def equirect(rgb, round_source=True):
    """-> (faces rgb float64 [6, n, n, 3] before the half rounding of the face format, the filter's pixel coordinates
    (px, py) per texel). The source is rounded to half as the RGB16F upload does (round_source=False: it is not)."""
    src = np.asarray(rgb, np.float32)
    src = (src.astype(np.float16) if round_source else src).astype(np.float64)
    h, w = src.shape[:2]
    n = w // 4
    u, v = equirect_uv(directions(n))
    px, py = u * w - 0.5, v * h - 0.5
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = (px - x0)[..., None], (py - y0)[..., None]
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    xa, xb, ya, yb = x0 % w, (x0 + 1) % w, y0 % h, (y0 + 1) % h
    c = (src[ya, xa] * (1 - fx) + src[ya, xb] * fx) * (1 - fy) + (src[yb, xa] * (1 - fx) + src[yb, xb] * fx) * fy
    return srgb_to_linear(c), (px, py)
