"""Float64 restatement of the present chain of the path-traced frame, Bloom and the AgX tonemap, written from the engine's
shaders and C# (not from oracle/oracle_post.inc or csrc/idk_post.cuh), so that the oracle and the kernels are checked
against an independent reading of the reference.

Paths are relative to the reference's IDKEngine (SHD = Resource/Shaders, BBG = the BBG project next to it):
  Source/Application.cs:217-223                    Bloom.Compute(Result) if IsBloom, then TonemapAndGamma.Compute(Result,
                                                   IsBloom ? Bloom.Result : null)
  Source/Render/PathTracer.cs:299-305              Result: R32G32B32A32Float, Linear filter, clamp to edge
  Source/Render/Bloom.cs:10-18                     Threshold 1.5, MaxColor 3.8
  Source/Render/Bloom.cs:129-147                   SetSize: size / 2 in C# integer division (MathF.Ceiling of an int changes
                                                   nothing), levels = max(GetMaxMipmapLevel - MinusLods, 2), rgba16f,
                                                   LinearMipmapNearest, clamp to edge; the upsample texture has levels - 1
  BBG/Source/Objects/Texture.cs:400-409            GetMaxMipmapLevel = ILogB(max extent) + 1, GetMipmapLevelSize = max(1, s >> l)
  Source/Render/Bloom.cs:61-78                     first downsample: unit 0 = the source, Lod = 0, writes down level 0
  Source/Render/Bloom.cs:80-92                     downsample writing level L >= 1: unit 0 = the down chain, Lod = L - 1
  Source/Render/Bloom.cs:96-111                    first upsample, writing level levels - 2: unit 1 = the DOWN chain, Lod = L + 1
  Source/Render/Bloom.cs:113-125                   upsample writing level L: unit 1 = the up chain, Lod = L + 1
  SHD/Bloom/compute.glsl:26-54                     uv = (imgCoord + 0.5) / imageSize; Downsample, then Prefilter when
                                                   Lod == 0; Upsample(SamplerUpsample) + textureLod(SamplerDownsample, uv, Lod)
  SHD/Bloom/compute.glsl:56-90                     Downsample: 13 taps
  SHD/Bloom/compute.glsl:92-107                    Upsample: 3x3 tent
  SHD/Bloom/compute.glsl:109-122                   Prefilter
  Source/Render/TonemapAndGammaCorrecter.cs:10-22  Exposure 0.45, Saturation 1.06, Linear 0.18, Peak 1, Compression 0.1
  Source/Render/TonemapAndGammaCorrecter.cs:37-61  bindings (an unbound sampler adds nothing), R8G8B8A8Unorm result
  SHD/TonemapAndGammaCorrect/compute.glsl:24-57    sum of the bound inputs, AgX_DS and LinearToSrgb (or a clamp), Dither, store
  SHD/TonemapAndGammaCorrect/compute.glsl:59-66    LinearToSrgb
  SHD/TonemapAndGammaCorrect/compute.glsl:70-108   xyYToXYZ, Unproject, PrimariesToMatrix, ComputeCompressionMatrix
  SHD/TonemapAndGammaCorrect/compute.glsl:110-156  DualSection, AgX_DS
  SHD/TonemapAndGammaCorrect/compute.glsl:158-181  Dither

The Lod uniform is 0 for the dispatch that writes down level 0 AND for the one that writes down level 1 (Bloom.cs:71 uploads
currentWriteLod = 0, Bloom.cs:85 uploads currentWriteLod - 1 = 0), so Prefilter runs on both.

A compute shader's texture() has no derivatives, so it samples level 0 (GLSL 4.60 section 8.9); textureLod with
LinearMipmapNearest samples the level named by the integer lod. GL's texture unit filters with fixed-point weights; here
the weights are exact, with the integer texel offset added before clamp-to-edge (GL 4.6 section 8.14.2).

Everything is float64 except where a value is *defined* by a float32 evaluation, stated where it happens: shader constants
and the settings uniforms are the float32 values of their literals, uv is a float32 division, and every rgba16f store rounds
to half (numpy float16, round to nearest even)."""
import math

import numpy as np

F = np.float32


def f32(x):
    """A GLSL float literal or float uniform: its float32 value."""
    return float(F(x))


KNEE = f32(0.2)                     # Prefilter's `const float Knee = 0.2`
MIN_BRIGHTNESS = f32(0.0001)        # max(brightness, 0.0001)


# ------------------------------------------------------------------------------------------------------ chain geometry
def bloom_size(w, h):
    """Bloom.SetSize: the bloom textures are half the image, C# integer division (Ceiling of an int is the int)."""
    return w // 2, h // 2


def level_count(w, h, minus_lods):
    """max(GetMaxMipmapLevel(w / 2, h / 2) - MinusLods, 2); ILogB(n) + 1 is frexp's exponent."""
    w2, h2 = bloom_size(w, h)
    return max(math.frexp(max(w2, h2))[1] - minus_lods, 2)


def level_sizes(w, h, minus_lods):
    """(width, height) of each down level; the up chain uses the first levels - 1 of them."""
    w2, h2 = bloom_size(w, h)
    return [(max(1, w2 >> l), max(1, h2 >> l)) for l in range(level_count(w, h, minus_lods))]


def half(a):
    """imageStore into rgba16f: round to nearest even half, read back exactly."""
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


# ----------------------------------------------------------------------------------------------------------- sampling
def uv_grid(w, h, shift=None):
    """uv = (imgCoord + 0.5) / size: the shader divides in float32, which fixes where each sample lands.

    shift = (sx, sy) texels instead gives the float64 quotient (imgCoord + 0.5 + shift) / size. The float32 roundings
    of uv and of a float32 texel coordinate u * size - 0.5 move a sample meant for a pixel centre by up to ~size * 2^-22
    texel; with exact weights it then takes that much of a neighbour. Next to a much brighter neighbour, where the sRGB
    curve is steep, that alone moves 255 * v by a third of an LSB at 1920 texels, so the tonemap checks take the
    values over that range of positions (test_post_ref.check_tonemap)."""
    y, x = np.mgrid[0:h, 0:w]
    if shift is not None:
        return (x + 0.5 + shift[0]) / w, (y + 0.5 + shift[1]) / h
    u = (x.astype(F) + F(0.5)) / F(w)
    v = (y.astype(F) + F(0.5)) / F(h)
    return u.astype(np.float64), v.astype(np.float64)


def bilinear64(level, u, v, ox=0, oy=0):
    """textureLodOffset(level, uv, lod, ivec2(ox, oy)).rgb on one level [h, w, 3] (float64), exact weights."""
    h, w = level.shape[:2]
    px, py = u * w - 0.5, v * h - 0.5
    fx0, fy0 = np.floor(px), np.floor(py)
    tx, ty = (px - fx0)[..., None], (py - fy0)[..., None]
    ix, iy = fx0.astype(np.int64) + ox, fy0.astype(np.int64) + oy
    x0, x1 = np.clip(ix, 0, w - 1), np.clip(ix + 1, 0, w - 1)
    y0, y1 = np.clip(iy, 0, h - 1), np.clip(iy + 1, 0, h - 1)
    return ((level[y0, x0] * (1 - tx) + level[y0, x1] * tx) * (1 - ty)
            + (level[y1, x0] * (1 - tx) + level[y1, x1] * tx) * ty)


# --------------------------------------------------------------------------------------------------------------- bloom
def downsample64(src, w, h):
    """Downsample (compute.glsl:56-90) at every texel of a w x h level, sampling src."""
    u, v = uv_grid(w, h)
    t = lambda ox, oy: bilinear64(src, u, v, ox, oy)
    center = t(0, 0)
    yellow = t(-2, 2) + t(0, 2) + center + t(-2, 0)
    green = t(0, 2) + t(2, 2) + t(2, 0) + center
    blue = center + t(2, 0) + t(2, -2) + t(0, -2)
    lila = t(-2, 0) + center + t(0, -2) + t(-2, -2)
    red = t(-1, 1) + t(1, 1) + t(1, -1) + t(-1, -1)
    return (red * 0.5 + (yellow + green + blue + lila) * 0.125) * 0.25


def upsample64(src, w, h):
    """Upsample (compute.glsl:92-107): 3x3 tent of src at every texel of a w x h level."""
    u, v = uv_grid(w, h)
    t = lambda ox, oy: bilinear64(src, u, v, ox, oy)
    return (t(-1, 1) + 2 * t(0, 1) + t(1, 1) + 2 * t(-1, 0) + 4 * t(0, 0) + 2 * t(1, 0)
            + t(-1, -1) + 2 * t(0, -1) + t(1, -1)) / 16.0


def prefilter64(color, max_color, threshold):
    """Prefilter (compute.glsl:109-122) of colours [..., 3]; Knee, 0.0001 and the uniforms are float32 values."""
    max_color, threshold = f32(max_color), f32(threshold)
    c = np.minimum(max_color, np.asarray(color, np.float64))
    brightness = c.max(-1)
    rq = np.clip(brightness - (threshold - KNEE), 0.0, KNEE * 2.0)
    rq = (rq * rq) * (0.25 / KNEE)
    return c * (np.maximum(rq, brightness - threshold) / np.maximum(brightness, MIN_BRIGHTNESS))[..., None]


def bloom64(hdr, threshold=1.5, max_color=3.8, minus_lods=3):
    """Bloom.Compute of an image [h, w, >= 3]. Returns (down, up): the levels as stored (float64 values of halves);
    Bloom.Result is up[0]."""
    h, w = hdr.shape[:2]
    if w < 2 or h < 2:
        raise ValueError("the bloom chain of an image below 2x2 has a 0-sized level")
    sizes = level_sizes(w, h, minus_lods)
    levels = len(sizes)
    down = []
    for l, (lw, lh) in enumerate(sizes):
        r = downsample64(hdr[..., :3].astype(np.float64) if l == 0 else down[l - 1], lw, lh)
        lod = 0 if l == 0 else l - 1                  # the Lod uniform of this dispatch (Bloom.cs:71, :85)
        if lod == 0:
            r = prefilter64(r, max_color, threshold)
        down.append(half(r))
    up = [None] * (levels - 1)
    for l in range(levels - 2, -1, -1):
        lw, lh = sizes[l]
        src = down[l + 1] if l == levels - 2 else up[l + 1]    # unit 1 holds the down chain for the first upsample only
        u, v = uv_grid(lw, lh)
        up[l] = half(upsample64(src, lw, lh) + bilinear64(down[l + 1], u, v))
    return down, up


# ------------------------------------------------------------------------------------------------------------- tonemap
def xyY_to_XYZ(x, y, Y=1.0):
    return np.array([(x * Y) / y, Y, ((1.0 - x - y) * Y) / y])


def primaries_to_matrix(xy_red, xy_green, xy_blue, xy_white):
    """PrimariesToMatrix: columns are the primaries' XYZ scaled so that rgb (1, 1, 1) maps to the white point."""
    R, G, B, W = (xyY_to_XYZ(*xy) for xy in (xy_red, xy_green, xy_blue, xy_white))
    temp = np.array([[R[0], G[0], B[0]], [1.0, 1.0, 1.0], [R[2], G[2], B[2]]])    # mat3(R.x, 1, R.z, G.x, ...) by columns
    scale = np.linalg.inv(temp) @ W
    return np.stack([R * scale[0], G * scale[1], B * scale[2]], axis=1)


SRGB_PRIMARIES = ((f32(0.64), f32(0.33)), (f32(0.3), f32(0.6)), (f32(0.15), f32(0.06)))
D65 = (f32(0.3127), f32(0.3290))


def compression_matrix(compression):
    """ComputeCompressionMatrix: primaries moved away from the white point by 1 / (1 - compression)."""
    sf = 1.0 / (1.0 - f32(compression))
    mix = lambda a, b: (a[0] * (1 - sf) + b[0] * sf, a[1] * (1 - sf) + b[1] * sf)
    return primaries_to_matrix(*(mix(D65, p) for p in SRGB_PRIMARIES), D65)


def agx_matrices(compression):
    """(sRGB_to_adjusted, its inverse) in the shader's product order sRGB_to_XYZ * XYZ_to_adjusted (compute.glsl:143)."""
    srgb_to_xyz = primaries_to_matrix(*SRGB_PRIMARIES, D65)
    srgb_to_adjusted = srgb_to_xyz @ np.linalg.inv(compression_matrix(compression))
    return srgb_to_adjusted, np.linalg.inv(srgb_to_adjusted)


def dual_section64(x, linear, peak):
    """DualSection: identity below S = peak * linear, an exponential shoulder towards peak above."""
    S = peak * linear
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        C = peak / (peak - S)
        shoulder = peak - (peak - S) * np.exp((-C * (x - S)) / peak)
    return np.where(x < S, x, shoulder)


def linear_to_srgb64(x):
    """LinearToSrgb: mix(higher, lower, cutoff) with a bvec is a select, so a negative component takes the linear branch."""
    lower = x * f32(12.92)
    with np.errstate(invalid="ignore"):
        higher = f32(1.055) * np.power(np.maximum(x, 0.0), f32(1.0 / F(2.4))) - f32(0.055)
    return np.where(x < f32(0.0031308), lower, higher)


LUMINANCE = np.array([f32(0.2126729), f32(0.7151522), f32(0.0721750)])


def agx_ds64(hdr, exposure, saturation, linear, peak, compression):
    """AgX_DS (compute.glsl:130-156) of colours [..., 3]."""
    to_adj, from_adj = agx_matrices(compression)
    wc = np.maximum(hdr, 0.0) * 2.0 ** f32(exposure)
    wc = wc @ to_adj.T
    wc = np.clip(dual_section64(wc, f32(linear), f32(peak)), 0.0, 1.0)
    desat = (wc @ LUMINANCE)[..., None]
    s = f32(saturation)
    wc = np.clip(desat * (1 - s) + wc * s, 0.0, 1.0)
    return wc @ from_adj.T


def bayer(n=8):
    """The recursive Bayer matrix M_2n = [[4M, 4M + 2], [4M + 3, 4M + 1]], M_1 = [[0]]; row index = y."""
    m = np.zeros((1, 1), np.int64)
    while m.shape[0] < n:
        m = np.block([[4 * m, 4 * m + 2], [4 * m + 3, 4 * m + 1]])
    return m


# Dither's BayerMatrix8 is the transpose of bayer() plus one, indexed [x % 8][y % 8]: entry (x, y) is bayer()[y % 8, x % 8] + 1.
# Each entry is the GLSL constant E / 65.0, a float32 division.
BAYER_TABLE = (bayer().T + 1).astype(F) / F(65.0)


def dither_values(w, h):
    """(BayerMatrix8[x % 8][y % 8] - 0.5) / 64 per pixel [h, w]."""
    y, x = np.mgrid[0:h, 0:w]
    return (BAYER_TABLE[x % 8, y % 8].astype(np.float64) - 0.5) / 64.0


def tonemap64(hdr, bloom, settings, shift=None):
    """TonemapAndGamma.Compute(hdr, bloom) on an image [h, w, >= 3] plus an optional Bloom.Result [h', w', 3] (None: not
    bound). settings has the fields of capi.IdkPtPostSettings; shift as in uv_grid. Returns (v64, rgba8 bytes): v64
    [h, w, 3] is the value handed to the R8G8B8A8Unorm store after the dither and the clamp to [0, 1]; the byte is
    round(255 * v64)."""
    h, w = hdr.shape[:2]
    u, v = uv_grid(w, h, shift)
    c = bilinear64(hdr[..., :3].astype(np.float64), u, v)
    if bloom is not None:
        c = c + bilinear64(np.asarray(bloom, np.float64)[..., :3], u, v)
    if settings.DoTonemapAndSrgbTransform:
        c = linear_to_srgb64(agx_ds64(c, settings.Exposure, settings.Saturation, settings.Linear, settings.Peak, settings.Compression))
    else:
        c = np.clip(c, 0.0, 1.0)
    v64 = np.clip(c + dither_values(w, h)[..., None], 0.0, 1.0)
    out = np.full((h, w, 4), 255, np.uint8)
    out[..., :3] = np.floor(v64 * 255.0 + 0.5).astype(np.uint8)
    return v64, out


def present64(hdr, settings):
    """Application.cs:217-223 for the path tracer: (Bloom.Result or None, v64, rgba8)."""
    bloom = None
    if settings.IsBloom:
        bloom = bloom64(hdr, settings.BloomThreshold, settings.BloomMaxColor, settings.BloomMinusLods)[1][0]
    v64, out = tonemap64(hdr, bloom, settings)
    return bloom, v64, out
