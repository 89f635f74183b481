"""The present chain's oracle (oracle/oracle_post.inc) against tests/post_ref64.py, a float64 restatement written from the
engine's shaders and C#: Bloom.Result texel by texel at odd, tiny and one-texel-thin shapes, the closed forms of a constant
image and of Prefilter's knee, and the AgX tonemap, dither and RGBA8 store byte by byte over a sweep of the settings."""
import numpy as np
import pytest

import oracle_lib as ol
import post_ref64 as r
from idkengine_b200 import capi
from test_post import synthetic_hdr

# Bloom.Result may differ from the float64 chain by float32 arithmetic and the half roundings it moves. The oracle and the
# kernels place each bilinear sample at u * size - 0.5 evaluated in float32; where a level's size is not a power of two
# that moves a sample by up to ~1e-5 texel, and a flip by one half ulp in a 1-texel level spreads over the whole image on
# the way up. Measured over test_oracle_bloom_chain: every component within 2 half ulps and 1 ulp of the level's peak,
# >= 99.47 % within 1 half ulp, >= 88.7 % bit-equal (250x131, MinusLods 1, high threshold; a float64 chain sampled at the
# float32 positions equals the oracle in 99.99 % of the components there). A half store that truncates instead of
# rounding to nearest even moves about half of the components.
BLOOM_REL = 2.0 ** -10      # of the largest value of the level
BLOOM_ULPS = 2              # half ulps of the float64 value, every component
BLOOM_ONE_ULP = 0.99        # fraction of the components within one half ulp
BLOOM_EXACT = 0.85          # fraction of the components equal bit for bit
# A byte is the rounding of 255 * v64 computed in float32: within half an LSB plus this much of 255 * v64.
EPS = 0.01
# How far, in texels per texel of image size, a sample meant for a pixel centre may land from it: u = (x + 0.5) / size
# and the texel coordinate u * size - 0.5 are float32 roundings, 2^-25 * size + 2 * 2^-23 * size at most.
POSITION = 2.0 ** -21

BLOOM_SHAPES = [(2, 2), (3, 2), (2, 3), (5, 3), (97, 33), (250, 131), (256, 144), (4096, 2), (2, 1500)]
BLOOM_SETTINGS = {"default": (1.5, 3.8), "low": (0.25, 0.9), "high": (6.0, 40.0)}    # (Threshold, MaxColor)

POST_SETTINGS = {
    "default": {},
    "exposure_-4": dict(Exposure=-4.0),
    "exposure_0": dict(Exposure=0.0),
    "exposure_3": dict(Exposure=3.0),
    "compression_0": dict(Compression=0.0),
    "compression_0.5": dict(Compression=0.5),
    "compression_0.9": dict(Compression=0.9),
    "saturation_0": dict(Saturation=0.0),
    "saturation_2": dict(Saturation=2.0),
    "shoulder_at_1": dict(Linear=0.5, Peak=2.0),            # Linear * Peak = 1 lies inside the inputs' range
    "shoulder_at_0.06": dict(Linear=0.1, Peak=0.6),
    "no_tonemap": dict(DoTonemapAndSrgbTransform=0),
    "no_bloom": dict(IsBloom=0),
    "bloom_low": dict(BloomThreshold=0.25, BloomMaxColor=0.9),
    "bloom_high": dict(BloomThreshold=6.0, BloomMaxColor=40.0, BloomMinusLods=0),
}


def post_settings(**kw):
    st = capi.default_post_settings()
    st.Exposure = 0.3
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def out_of_gamut_hdr(w, h):
    """Fully saturated hues (one turn of the hue circle down the rows) at intensities from 0.01 to 60 across: after the
    compression matrix, the curve and the inverse matrix they leave the sRGB gamut, so LinearToSrgb sees negative
    components. Neighbouring texels differ by a few per cent only: uv is a float32 quotient, so a sample meant for a
    pixel centre lands up to ~1e-5 texel off it, at a position that differs between float32 and float64 evaluation; next
    to a 1:600 edge at Exposure 3 that alone moves 255 * v by 0.05."""
    hue = (np.arange(h) / h * 6.0)[:, None]
    rgb = np.stack([np.clip(np.abs(hue - 3.0) - 1.0, 0, 1), np.clip(2.0 - np.abs(hue - 2.0), 0, 1), np.clip(2.0 - np.abs(hue - 4.0), 0, 1)], -1)
    img = np.ones((h, w, 4), np.float32)
    img[..., :3] = rgb * np.geomspace(0.01, 60.0, w)[None, :, None]
    return img


def check_bloom(got, want, what=""):
    """Bloom.Result of the oracle or the kernels against post_ref64's, texel by texel."""
    assert got.shape == want.shape, what
    peak = np.abs(want).max()
    err = np.abs(got.astype(np.float64) - want)
    assert err.max() <= BLOOM_REL * peak, f"{what}: max error {err.max():.3g} of a peak of {peak:.3g}"
    ulps = err / np.spacing(np.abs(want).astype(np.float16)).astype(np.float64)
    assert ulps.max() <= BLOOM_ULPS, f"{what}: a component is {ulps.max():.1f} half ulps away"
    one = (ulps <= 1).mean()
    assert one >= BLOOM_ONE_ULP, f"{what}: only {one:.4f} of the components are within one half ulp"
    exact = (err == 0).mean()
    assert exact >= BLOOM_EXACT, f"{what}: only {exact:.4f} of the components are equal after half rounding"


def check_bytes(ldr, v64, envelope=None, what=""):
    """Every byte within 0.5 + EPS of 255 * v64, and the rounding of 255 * v64 wherever that is not within EPS of a tie.
    envelope = (lo, hi) widens v64 to the values over the positions a sample may take (check_tonemap). Returns the
    largest |byte - 255 * v64| and the largest distance from a byte to 255 * [lo, hi]."""
    got = ldr[..., :3].astype(np.float64)
    lo, hi = envelope if envelope is not None else (v64, v64)
    lo, hi = 255.0 * np.minimum(lo, v64), 255.0 * np.maximum(hi, v64)
    dev = np.maximum(np.maximum(lo - got, got - hi), 0.0)
    assert dev.max() <= 0.5 + EPS, f"{what}: |byte - 255 v64| reaches {dev.max():.4f}"
    # the byte is the rounding of a value in [lo, hi] unless one of the ends is within EPS of a tie
    tie = lambda x: np.abs(x - np.floor(x) - 0.5) <= EPS
    bad = ~tie(lo) & ~tie(hi) & ((got < np.floor(lo + 0.5)) | (got > np.floor(hi + 0.5)))
    assert not bad.any(), f"{what}: {int(bad.sum())} bytes are not the rounding of 255 v64 away from a tie"
    assert (ldr[..., 3] == 255).all()
    return float(np.abs(got - 255.0 * v64).max()), float(dev.max())


def check_tonemap(ldr, img, bloom, st, what=""):
    """The LDR frame of img (with the given Bloom.Result when st.IsBloom) against post_ref64's tonemap and store, each
    sample taken at the shader's float32 uv and, for the envelope, within POSITION * size texel of the pixel centre."""
    h, w = img.shape[:2]
    bloom = bloom if st.IsBloom else None
    v64 = r.tonemap64(img, bloom, st)[0]
    d = POSITION * np.array([w, h])
    # bilinear filtering is linear in each quadrant around a texel centre, so the extremes lie on this 3 x 3 grid
    vs = [r.tonemap64(img, bloom, st, shift=(sx * d[0], sy * d[1]))[0] for sx in (-1, 0, 1) for sy in (-1, 0, 1)]
    return check_bytes(ldr, v64, (np.min(vs, 0), np.max(vs, 0)), what)


# ------------------------------------------------------------------------------------------------------------ the chain
def test_chain_geometry():
    """SetSize's integer halving and level count, and GetMipmapLevelSize, at the shapes the chain tests use."""
    assert r.level_sizes(2, 2, 3) == [(1, 1), (1, 1)]
    assert r.level_sizes(3, 2, 0) == [(1, 1), (1, 1)]                     # 3 / 2 = 1: Ceiling of an int does nothing
    assert r.level_sizes(64, 48, 3) == [(32, 24), (16, 12), (8, 6)]
    assert r.level_sizes(4096, 2, 3) == [(2048 >> l, 1) for l in range(9)]
    assert r.level_sizes(2, 1500, 3) == [(1, 750 >> l) for l in range(7)]
    assert r.level_count(250, 131, 0) == 7 and r.level_count(250, 131, 30) == 2
    assert r.level_count(1920, 1080, 3) == 7


@pytest.mark.parametrize("setting", list(BLOOM_SETTINGS))
@pytest.mark.parametrize("minus", [0, 1, 3, 30])
@pytest.mark.parametrize("w,h", BLOOM_SHAPES)
def test_oracle_bloom_chain(w, h, minus, setting):
    """Bloom.Result of the oracle against the float64 chain, every texel, at the given MinusLods and Threshold/MaxColor."""
    st = post_settings(BloomMinusLods=minus)
    st.BloomThreshold, st.BloomMaxColor = BLOOM_SETTINGS[setting]
    img = synthetic_hdr(w, h, seed=w + h)
    _, bloom = ol.post_process(img, st, want_bloom=True)
    _, up = r.bloom64(img, st.BloomThreshold, st.BloomMaxColor, minus)
    check_bloom(bloom, up[0], f"{w}x{h} MinusLods {minus} {setting}")


# -------------------------------------------------------------------------------------------------------- closed forms
@pytest.mark.parametrize("b", [3.0, 0.5, 1.3])
def test_constant_image_bloom(b):
    """A constant image of brightness b: every downsample of a constant is the constant, Prefilter runs on levels 0 and 1,
    and the up chain adds down levels 1 .. levels - 1 plus the last one once more, so Bloom.Result = levels * P(P(b)).
    b = 3 gives 3 * P(1.5) = 0.15 at 64x48 (levels 0 and 1 prefiltered; prefiltering level 0 alone would give 4.5);
    b = 0.5 and b = 1.3 (the float32 just below Threshold - Knee) give exactly 0."""
    st = post_settings()
    img = np.full((48, 64, 4), b, np.float32)
    _, bloom = ol.post_process(img, st, want_bloom=True)
    levels = r.level_count(64, 48, st.BloomMinusLods)
    p = lambda c: r.prefilter64(np.full(3, c), st.BloomMaxColor, st.BloomThreshold)[0]
    want = levels * p(p(b))
    _, up = r.bloom64(img, st.BloomThreshold, st.BloomMaxColor, st.BloomMinusLods)
    if b == 3.0:
        assert levels == 3 and p(3.0) == 1.5 and abs(p(1.5) - 0.05) < 1e-7 and abs(want - 0.15) < 1e-6
    if b <= 1.3 + 1e-6:
        assert want == 0.0 and np.all(bloom == 0.0) and np.all(up[0] == 0.0)
    ulp = np.spacing(np.float16(want)).astype(np.float64) if want else 0.0
    assert np.abs(bloom - want).max() <= 4 * ulp, (float(bloom.max()), want)
    assert np.abs(up[0] - want).max() <= 4 * ulp


def test_prefilter_knee():
    """Prefilter at its knee points: brightness Threshold - Knee gives 0, Threshold + Knee is where the quadratic knee
    (rq) and the linear part (brightness - Threshold) meet, and components above MaxColor are clamped first."""
    thr, maxc = 1.5, 3.8
    k = r.KNEE
    assert np.all(r.prefilter64([thr - k, 0.1, 0.0], maxc, thr) == 0.0)
    c = np.array([thr + k, 0.3, 0.1])
    rq = (2 * k) ** 2 * (0.25 / k)
    assert abs(rq - k) < 1e-12                                             # both branches equal at Threshold + Knee
    np.testing.assert_allclose(r.prefilter64(c, maxc, thr), c * (k / (thr + k)), rtol=1e-12)
    big = r.prefilter64([100.0, 50.0, 1.0], maxc, thr)
    m = r.f32(maxc)
    np.testing.assert_allclose(big, np.array([m, m, 1.0]) * ((m - r.f32(thr)) / m), rtol=1e-12)
    # the oracle through a whole chain: a constant MaxColor + 1 image blooms like a constant MaxColor image
    st = post_settings()
    a = ol.post_process(np.full((16, 24, 4), 4.8, np.float32), st, want_bloom=True)[1]
    b = ol.post_process(np.full((16, 24, 4), m, np.float32), st, want_bloom=True)[1]
    assert np.array_equal(a, b) and a.max() > 0


# ------------------------------------------------------------------------------------------------ tonemap and store
@pytest.mark.parametrize("name", list(POST_SETTINGS))
@pytest.mark.parametrize("image", ["synthetic", "out_of_gamut"])
def test_oracle_tonemap_and_store(image, name):
    """Every LDR byte of the oracle against the float64 tonemap of the same HDR plus the oracle's own Bloom.Result."""
    st = post_settings(**POST_SETTINGS[name])
    w, h = 97, 33
    img = synthetic_hdr(w, h, seed=5) if image == "synthetic" else out_of_gamut_hdr(w, h)
    ldr, bloom = ol.post_process(img, st, want_bloom=True)
    check_tonemap(ldr, img, bloom, st, f"{image} {name}")


def test_out_of_gamut_inputs_reach_the_linear_branch():
    """The inverse compression matrix turns saturated inputs negative before LinearToSrgb; that is the case the select
    (not a blend) of the shader's mix keeps finite."""
    st = post_settings(Exposure=3.0, IsBloom=0)
    img = out_of_gamut_hdr(97, 33)
    lin = r.agx_ds64(img[..., :3].astype(np.float64), st.Exposure, st.Saturation, st.Linear, st.Peak, st.Compression)
    assert (lin < 0).sum() > 50
    assert np.isfinite(r.tonemap64(img, None, st)[0]).all()
    check_tonemap(ol.post_process(img, st), img, None, st, "out of gamut, Exposure 3")


@pytest.mark.parametrize("w,h", [(256, 144), (250, 131), (97, 33)])
def test_oracle_present_chain_bytes(w, h):
    """The whole chain at the default settings with Exposure 0.3: the oracle's bytes within the float64 bound."""
    st = post_settings()
    img = synthetic_hdr(w, h, seed=w)
    ldr, bloom = ol.post_process(img, st, want_bloom=True)
    check_tonemap(ldr, img, bloom, st, f"{w}x{h}")
    # the float64 chain's own bloom lands on the same bytes but where a byte sits near a tie
    _, _, want = r.present64(img, st)
    assert np.abs(ldr.astype(int) - want.astype(int)).max() <= 1


# ------------------------------------------------------------------------------------------------------- known answers
def test_compression_0_is_the_srgb_transfer():
    """Compression 0 makes sRGB_to_adjusted the identity; with Saturation 1 and inputs below Peak * Linear every byte is
    the sRGB transfer of 2^Exposure * x plus the dither."""
    to_adj, from_adj = r.agx_matrices(0.0)
    np.testing.assert_allclose(to_adj, np.eye(3), atol=1e-14)
    st = post_settings(Compression=0.0, Saturation=1.0, IsBloom=0, Exposure=0.45)
    w, h = 37, 21
    S = r.f32(st.Peak) * r.f32(st.Linear)
    rng = np.random.default_rng(9)
    img = np.ones((h, w, 4), np.float32)
    img[..., :3] = rng.uniform(0.0, 0.999 * S / 2.0 ** r.f32(st.Exposure), (h, w, 3)).astype(np.float32)
    # the pixel-centre sample: uv is a float32 quotient, so it lands up to ~1e-5 texel off the centre
    x = r.bilinear64(img[..., :3].astype(np.float64), *r.uv_grid(w, h))
    assert np.abs(x - img[..., :3]).max() < 1e-5
    x = x * 2.0 ** r.f32(st.Exposure)
    f = r.f32                                                               # the shader's float literals
    srgb = np.where(x < f(0.0031308), f(12.92) * x, f(1.055) * x ** f(1 / np.float32(2.4)) - f(0.055))
    closed = np.clip(srgb + r.dither_values(w, h)[..., None], 0, 1)
    v64, _ = r.tonemap64(img, None, st)
    np.testing.assert_allclose(v64, closed, rtol=0, atol=1e-12)
    check_bytes(ol.post_process(img, st), closed, what="compression 0")


def test_flat_image_dither_bytes():
    """A flat 0.5 image with the tonemap off is 0.5 + the dither: the Bayer table indexed [x % 8][y % 8]. At (1, 0) the
    engine's entry is 33 / 65 and the byte 128; a transposed table would give 49 / 65 and 129."""
    st = post_settings(DoTonemapAndSrgbTransform=0, IsBloom=0)
    w, h = 13, 9
    img = np.full((h, w, 4), 0.5, np.float32)
    m = r.bayer()
    assert sorted(m.ravel()) == list(range(64))
    assert r.BAYER_TABLE[1, 0] == np.float32(33) / np.float32(65) and r.BAYER_TABLE[0, 1] == np.float32(49) / np.float32(65)
    y, x = np.mgrid[0:h, 0:w]
    want = np.floor(255.0 * (0.5 + ((m[y % 8, x % 8] + 1) / 65.0 - 0.5) / 64.0) + 0.5)
    ldr = ol.post_process(img, st)
    assert np.array_equal(ldr[..., :3], np.repeat(want[..., None], 3, -1).astype(np.uint8))
    assert ldr[0, 1, 0] == 128 and ldr[1, 0, 0] == 129
    _, mine = r.tonemap64(img, None, st)
    assert np.array_equal(mine, ldr)
