"""The sky generators' rules on the CPU (DESIGN.md 8f.1j): the texel layout against GL cube-map face selection, det_atan2 and
det_asin against float64, and the fp32 oracle of both kernels against the independent float64 restatement in sky_ref64."""
import numpy as np
import pytest

import sky_oracle as so
import sky_ref64 as sr
from idkengine_b200 import capi

PI32_ULP = float(np.spacing(np.float32(np.pi)))   # 2.4e-7


def gl_face_st(d):
    """GL 4.6 table 8.19: (face, s, t) of float64 directions [..., 3]."""
    ax, ay, az = np.abs(d[..., 0]), np.abs(d[..., 1]), np.abs(d[..., 2])
    face = np.where((ax >= ay) & (ax >= az), np.where(d[..., 0] >= 0, 0, 1),
                    np.where(ay >= az, np.where(d[..., 1] >= 0, 2, 3), np.where(d[..., 2] >= 0, 4, 5)))
    sc = np.choose(face, [-d[..., 2], d[..., 2], d[..., 0], d[..., 0], d[..., 0], -d[..., 0]])
    tc = np.choose(face, [-d[..., 1], -d[..., 1], d[..., 2], -d[..., 2], -d[..., 1], -d[..., 1]])
    ma = np.choose(face, [ax, ax, ay, ay, az, az])
    return face, (sc / ma + 1) / 2, (tc / ma + 1) / 2


@pytest.mark.parametrize("n", [1, 2, 3, 8, 128])
def test_every_texel_direction_selects_its_own_face_and_texel(n):
    f, y, x = np.meshgrid(np.arange(6), np.arange(n), np.arange(n), indexing="ij")
    for d in (so.directions(n).astype(np.float64), sr.directions(n)):
        face, s, t = gl_face_st(d)
        assert np.array_equal(face, f)
        assert np.array_equal(np.floor(s * n), x) and np.array_equal(np.floor(t * n), y)
    d = so.directions(n)
    assert np.abs(np.linalg.norm(d.astype(np.float64), axis=-1) - 1).max() < 3e-7
    if n % 2:   # the centre texel of each face is the exact axis direction
        c = d[:, n // 2, n // 2]
        assert np.array_equal(np.abs(c), np.eye(3, dtype=np.float32)[[0, 0, 1, 1, 2, 2]])


def test_det_atan2_within_1p5_ulp_of_pi():
    rng = np.random.default_rng(1)
    y = np.concatenate([rng.uniform(-1, 1, 1_000_000), rng.uniform(-1e4, 1e4, 200_000), rng.normal(0, 1e-20, 50_000)]).astype(np.float32)
    x = np.concatenate([rng.uniform(-1, 1, 1_000_000), rng.uniform(-1e4, 1e4, 200_000), rng.normal(0, 1e-20, 50_000)]).astype(np.float32)
    ang = np.linspace(-np.pi, np.pi, 400_001)
    y = np.concatenate([y, np.sin(ang).astype(np.float32)])
    x = np.concatenate([x, np.cos(ang).astype(np.float32)])
    err = np.abs(so.det_atan2(y, x).astype(np.float64) - np.arctan2(y.astype(np.float64), x.astype(np.float64)))
    assert err.max() <= 1.5 * PI32_ULP, err.max()
    # the special cases, C's atan2 on the signed zeros included (atan(0, 0) at the poles of odd face sizes)
    ys = np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0, 1.0, -1.0, 0.0, -0.0, 1.0, 1e-30, -1e-30, 1.0, 1.0, np.nan, 0.0], np.float32)
    xs = np.array([0.0, 0.0, -0.0, -0.0, 0.0, 0.0, -0.0, -0.0, 1.0, -1.0, 1.0, 1.0, -1.0, 1e-30, -1e-30, 0.0, np.nan], np.float32)
    got = so.det_atan2(ys, xs)
    want = np.arctan2(ys.astype(np.float64), xs.astype(np.float64))
    assert np.array_equal(np.signbit(got[:15]), np.signbit(want[:15]))
    assert np.abs(got[:15] - want[:15]).max() <= 1.5 * PI32_ULP
    assert got[0] == 0.0 and not np.signbit(got[0]) and got[1] == 0.0 and np.signbit(got[1])
    assert got[11] == np.float32(1e-30)                                  # tiny angles keep their digits
    assert np.isnan(got[15:]).all()


def test_det_asin_within_2e_minus_7():
    x = np.concatenate([np.linspace(-1, 1, 2_000_001), np.geomspace(1e-30, 1, 100_000), -np.geomspace(1e-30, 1, 100_000)]).astype(np.float32)
    x64 = x.astype(np.float64)
    want = np.arcsin(x64)
    err = np.abs(so.det_asin(x).astype(np.float64) - want)
    assert err.max() <= 2e-7, err.max()
    assert (err <= 4e-7 * np.abs(want) + 1e-45).all()                 # relative, so tiny arguments keep their digits
    sp = np.array([0.0, -0.0, 1.0, -1.0, 0.5, -0.5, 1e-5, 1.0000001, -2.0, np.nan], np.float32)
    got = so.det_asin(sp)
    assert got[0] == 0.0 and not np.signbit(got[0]) and np.signbit(got[1])
    assert got[2] == np.float32(np.pi / 2) and got[3] == -np.float32(np.pi / 2)
    assert got[6] == np.float32(1e-5)
    assert np.isnan(got[7:]).all()


# fp32 loses about 0.5 m in length(iPos) - rPlanet (ulp(6.4e6) = 0.5); against the 1.2 km Mie scale height that is a relative
# error of 0.5 / 1200 = 4.2e-4 in each exp(-h / H), which the optical-depth sums and the scattering sum average rather than
# add. The tolerance is twice that. Largest error observed (n = 8, every case below): 2.5e-4.
ATMOSPHERE_RTOL = 2 * 0.5 / 1200


@pytest.mark.parametrize("steps", [(1, 1), (40, 8)])
@pytest.mark.parametrize("sun", [(0.0, 0.0), (0.7, np.pi / 4), (0.3, np.pi / 2), (1.1, 1.9)], ids=["zenith", "45deg", "horizon", "below"])
@pytest.mark.parametrize("intensity", [15.0, 0.0])
def test_atmosphere_oracle_against_float64(steps, sun, intensity):
    n = 8
    s = capi.IdkPtAtmosphereSettings(steps[0], steps[1], intensity, sun[0], sun[1])
    got = so.atmosphere(s, n)
    assert (got[..., 3] == 1.0).all()
    ref, _, fragile, overflow = sr.atmosphere(n, steps[0], steps[1], intensity, sun[0], sun[1])
    got = got[..., :3].astype(np.float64)
    finite = np.isfinite(got).all(-1)
    assert (finite | overflow).all()               # fp32 overflows only where float64 leaves fp32's exp range
    ok = finite & ~fragile
    assert ok.mean() > 0.9
    err = np.abs(got - ref)
    assert (err[ok] <= ATMOSPHERE_RTOL * np.abs(ref[ok]) + 1e-30).all(), (err / np.maximum(np.abs(ref), 1e-30))[ok].max()
    if intensity == 0.0:
        assert (got[finite] == 0.0).all()
    elif sun[1] < 1.6:
        assert (ref[ok] > 0).any()


def synthetic_equirect(w, h, seed):
    """Values on both sides of the sRGB cutoff, HDR values above 1, and fp32 values that the RGB16F upload rounds."""
    rng = np.random.default_rng(seed)
    img = rng.uniform(0.0, 0.12, (h, w, 3)).astype(np.float32)
    img[rng.random((h, w)) < 0.2] *= 30.0                      # HDR
    img[:, 0] = (0.9, 0.04, 0.2)                               # column 0 against column w - 1: the u = 0 / 1 seam
    img[:, w - 1] = (0.01, 0.5, 0.045)
    return img


def equirect_tolerance(ref, src_max, w):
    """The oracle rounds to half (half an ulp, 2^-11 relative); its fp32 pixel coordinate is off by about 2 ulp of w
    (det_atan2 / det_asin within 1.5 ulp of pi, times 0.1591 w) plus the fp32 products, which moves the bilinear weights
    by that much times the texel difference (at most 2 src_max), and pow(., 2.4) scales relative errors by 2.4."""
    return np.abs(ref) * 2.0 ** -11 * 1.001 + 2.4 * 2 * src_max * (4 * np.spacing(np.float32(w))) + 1e-7


@pytest.mark.parametrize("w,h", [(4, 1), (7, 3), (64, 32), (130, 65)])
def test_equirect_oracle_against_float64(w, h):
    img = synthetic_equirect(w, h, w * 1000 + h)
    got = so.equirect(img)
    n = w // 4
    assert got.shape == (6, n, n, 4) and (got[..., 3] == 1.0).all()
    assert np.array_equal(got[..., :3], got[..., :3].astype(np.float16).astype(np.float32))   # RGBA16F values
    ref, (px, py) = sr.equirect(img)
    src_max = float(np.abs(img.astype(np.float16).astype(np.float64)).max())
    err = np.abs(got[..., :3] - ref)
    tol = equirect_tolerance(ref, src_max, w)
    assert (err <= tol).all(), (err - tol).max()
    # what the shapes cover: on the small shapes, texels that filter across the u = 0 / 1 seam and rows that wrap past a pole
    # (0.1591 < 1 / 2pi keeps u inside [0.00017, 0.99983], so at even face sizes below w = 2941 no texel centre is close enough
    # to the seam); the pole texels themselves (the face centres of odd face sizes, atan(0, 0)); results on both sides of the
    # sRGB cutoff
    if w < 64:
        assert ((px < 0) | (px >= w - 1)).any() and ((py < 0) | (py >= h - 1)).any()
    if n % 2:
        assert (np.abs(sr.directions(n)[2:4, n // 2, n // 2, 1]) == 1).all()
    if w >= 64:
        assert (ref < 0.04045 / 12.92).any() and (ref > 0.04045 / 12.92).any()


@pytest.mark.parametrize("w,h", [(12, 6), (4, 1)])
def test_equirect_seam_mixes_first_and_last_columns(w, h):
    """At odd face sizes the texels with z = 0 and x < 0 look at u = 0.99983: their footprint is column w - 1 and, wrapped,
    column 0."""
    img = np.zeros((h, w, 3), np.float32)
    img[:, 0, 0] = 1.0          # red only in column 0, green only in column w - 1
    img[:, w - 1, 1] = 1.0
    got = so.equirect(img)
    _, (px, _) = sr.equirect(img)
    seam = (px > w - 1) & (px < w - 0.1)
    assert seam.sum() >= 1
    assert (got[..., 0][seam] > 0).all() and (got[..., 1][seam] > 0).all()


def test_equirect_rounds_the_source_to_half():
    """Inputs chosen between two halves: the RNE rounding of the upload is visible in the faces, and a float source would
    miss the oracle's values by more than its tolerance."""
    w, h = 64, 32
    rng = np.random.default_rng(3)
    base = rng.uniform(0.2, 0.9, (h, w, 3)).astype(np.float16)
    img = (base.astype(np.float32) + np.float32(2.0 ** -12) * 0.97).astype(np.float32)  # just below the midpoint to the next half
    assert not np.array_equal(img, img.astype(np.float16).astype(np.float32))
    got = so.equirect(img)
    ref, _ = sr.equirect(img)
    src_max = float(np.abs(img).max())
    assert (np.abs(got[..., :3] - ref) <= equirect_tolerance(ref, src_max, w)).all()
    ref_unrounded, _ = sr.equirect(img, round_source=False)
    assert (np.abs(got[..., :3] - ref_unrounded) > equirect_tolerance(ref_unrounded, src_max, w)).any()
