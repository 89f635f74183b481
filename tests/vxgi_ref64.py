"""Float64 restatement of the VXGI passes, written from the engine's shaders and C# (not from oracle/oracle_vxgi.inc or
csrc/idk_vxgi.cuh), so that the oracle and the kernels are checked against an independent reading of the reference.

Paths are relative to the reference's IDKEngine (SHD = Resource/Shaders, BBG = the BBG project next to it):
  BBG/Source/Objects/Texture.cs:400-409                 GetMaxMipmapLevel, GetMipmapLevelSize
  SHD/VXGI/Voxelize/Mipmap/compute.glsl:10-30           7-tap downsample
  SHD/include/TraceCone.glsl:5-39                       TraceCone
  SHD/VXGI/ConeTraceGI/include/Impl.glsl:26-75          IndirectLight
  SHD/VXGI/ConeTraceGI/compute.glsl:20-46               the per-pixel entry
  SHD/include/Random.glsl:35-41                         InterleavedGradientNoise
  SHD/include/Sampling.glsl:59-68,86-89                 SampleSphere, CosineSampleHemisphere
  SHD/include/Surface.glsl:106-111                      GetSurfaceVariance
  SHD/include/Compression.glsl:11-37,63-73              DecompressSR11G11B10, DecompressUR8G8B8A8, DecodeUnitVec
  SHD/include/Math.glsl:75-102                          PerspectiveTransformUvDepth, MapToZeroOne
  SHD/VXGI/Voxelize/Voxelize/{vertex,geometry,fragment}.glsl, SHD/include/Pbr.glsl:9-17   voxelisation
  Source/Render/VXGI/Voxelizer/Voxelizer.cs:210-258     mip loop, sampler state (LinearMipmapLinear, clamp to edge)

GL's texture unit filters with fixed-point weights; here, like in the product (DESIGN section 7), the filter weights are
exact. Everything is float64 except where a value is *defined* by a float32 evaluation (stated where it happens); shader
constants are the float32 values of their literals."""
import math

import numpy as np

F = np.float32


def level_count(size):
    """Texture.GetMaxMipmapLevel: ILogB(max extent) + 1 (frexp's exponent is ILogB + 1)."""
    return math.frexp(max(size))[1]


def level_sizes(size):
    """Texture.GetMipmapLevelSize per level: each extent divided by 2^level (integer division), at least 1."""
    return [tuple(max(1, s // (1 << l)) for s in size) for l in range(level_count(size))]


# ------------------------------------------------------------------------------------------------------------ filtering
def trilinear64(level, uvw, offset=(0, 0, 0)):
    """textureLodOffset on one level ([d, h, w, 4] float64) at uvw [..., 3]: texel centres at (i + 0.5) / size, the integer
    offset added to the texel index BEFORE clamp-to-edge (GL 4.6 section 8.14.2), exact weights."""
    size = np.array([level.shape[2], level.shape[1], level.shape[0]])
    p = uvw * size - 0.5
    f0 = np.floor(p)
    t = p - f0
    i0 = f0.astype(np.int64) + np.asarray(offset)
    lo, hi = np.clip(i0, 0, size - 1), np.clip(i0 + 1, 0, size - 1)
    out = 0.0
    for cz in (0, 1):
        for cy in (0, 1):
            for cx in (0, 1):
                wgt = ((t[..., 0] if cx else 1 - t[..., 0]) * (t[..., 1] if cy else 1 - t[..., 1]) * (t[..., 2] if cz else 1 - t[..., 2]))
                ix, iy, iz = (hi if cx else lo)[..., 0], (hi if cy else lo)[..., 1], (hi if cz else lo)[..., 2]
                out = out + wgt[..., None] * level[iz, iy, ix]
    return out


def texture_lod64(levels, uvw, lod):
    """textureLod with LinearMipmapLinear: lod clamped to [0, maxLevel], trilinear in floor(lod) and floor(lod) + 1, linear
    in between (GL 4.6 section 8.14.3); at lod >= maxLevel only the last level."""
    max_level = len(levels) - 1
    lod = np.clip(lod, 0.0, max_level)
    l0 = np.floor(lod).astype(np.int64)
    fl = lod - l0
    out = np.zeros(uvw.shape[:-1] + (4,))
    for l in np.unique(l0):
        m = l0 == l
        a = trilinear64(levels[l], uvw[m])
        if l < max_level:
            a = a * (1 - fl[m])[:, None] + trilinear64(levels[l + 1], uvw[m]) * fl[m][:, None]
        out[m] = a
    return out


def mip64(below, size):
    """Mipmap/compute.glsl on one level: the 7 taps (centre, +-1 texel per axis) of the level below (float16) at the
    destination texel centre, / 7, computed in float64 and rounded once to float16 (numpy's float64 -> float16 conversion
    rounds to nearest even)."""
    w, h, d = size
    z, y, x = np.meshgrid(np.arange(d), np.arange(h), np.arange(w), indexing="ij")
    uvw = (np.stack([x, y, z], -1) + 0.5) / np.array([w, h, d])
    src = below.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        r = trilinear64(src, uvw)
        for off in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)):
            r = r + trilinear64(src, uvw, off)
        return (r / 7.0).astype(np.float16)


def half_ulp_distance(a, b):
    """Distance in float16 ulps between two float16 arrays (NaN == NaN counts as 0, NaN against a number as infinity)."""
    def key(x):
        u = x.view(np.uint16).astype(np.int64)
        return np.where(u & 0x8000, -(u & 0x7FFF), u)
    na, nb = np.isnan(a), np.isnan(b)
    d = np.abs(key(a) - key(b)).astype(np.float64)
    return np.where(na | nb, np.where(na & nb, 0.0, np.inf), d)


# ------------------------------------------------------------------------------------------------------------ cone trace
def interleaved_gradient_noise(x, y, index):
    """Random.glsl:35-41. This hash is defined by its float32 evaluation (fract of a large product amplifies every rounding),
    so it is evaluated in float32, one rounding per operation and no fused multiply-add, like the GLSL; everything downstream
    of it is float64."""
    x = F(x) + F(index) * F(5.588238)
    y = F(y) + F(index) * F(5.588238)
    a = F(0.06711056) * x + F(0.00583715) * y
    a = a - np.floor(a)
    b = F(52.9829189) * a
    return (b - np.floor(b)).astype(np.float64)


def decode_unit_vec64(rg):
    """Compression.glsl:63-73."""
    f = rg.astype(np.float64) * 2.0 - 1.0
    n = np.stack([f[..., 0], f[..., 1], 1.0 - np.abs(f[..., 0]) - np.abs(f[..., 1])], -1)
    t = np.maximum(-n[..., 2], 0.0)
    n[..., 0] += np.where(n[..., 0] >= 0.0, -t, t)
    n[..., 1] += np.where(n[..., 1] >= 0.0, -t, t)
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


def _normalize(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def trace_cone64(levels, grid_min, grid_max, origin, direction, normal, cone_angle, step_multiplier, normal_ray_offset,
                 alpha_threshold=float(F(0.99))):
    """TraceCone.glsl:5-39 for N cones at once. Returns (acc [N, 4], steps [N], margin [N]): margin is the smallest distance,
    over all steps, of a discontinuous decision from its threshold -- uvw against 0 and 1, sampleLod against maxLevel (a tenth
    of it), acc.a against alphaThreshold."""
    gmin, gmax = np.asarray(grid_min, np.float64), np.asarray(grid_max, np.float64)
    size = np.array([levels[0].shape[2], levels[0].shape[1], levels[0].shape[0]], np.float64)
    voxel = (gmax - gmin) / size
    vmax, vmin = voxel.max(), voxel.min()
    max_level = len(levels) - 1
    n = len(origin)
    acc = np.zeros((n, 4))
    steps = np.zeros(n, np.int64)
    margin = np.full(n, np.inf)
    origin = origin + normal * vmax * normal_ray_offset
    dist = np.full(n, vmax)
    tan_a = np.tan(cone_angle) * np.ones(n)
    live = np.arange(n)
    while len(live):
        margin[live] = np.minimum(margin[live], np.abs(acc[live, 3] - alpha_threshold))
        live = live[acc[live, 3] < alpha_threshold]
        if not len(live):
            break
        d = dist[live]
        sample_d = np.maximum(vmin, 2.0 * tan_a[live] * d)
        lod = np.log2(sample_d / vmin)
        uvw = (origin[live] + direction[live] * d[:, None] - gmin) / (gmax - gmin)
        margin[live] = np.minimum(margin[live], np.minimum(np.abs(uvw), np.abs(uvw - 1.0)).min(-1))
        margin[live] = np.minimum(margin[live], np.abs(lod - max_level) * 0.1)   # the kernels' log2 is a polynomial good to 2e-6
        out = (uvw < 0.0).any(-1) | (uvw >= 1.0).any(-1) | (lod > max_level)
        live, uvw, lod, sample_d = live[~out], uvw[~out], lod[~out], sample_d[~out]
        if not len(live):
            break
        s = texture_lod64(levels, uvw, lod)
        acc[live] += (1.0 - acc[live, 3])[:, None] * s
        dist[live] += sample_d * step_multiplier
        steps[live] += 1
    return acc, steps, margin


def indirect_light64(levels, grid_min, grid_max, frame, settings, depth, normal_rg, metal_rough, sky, row_first=0, full_height=None):
    """ConeTraceGI/compute.glsl + Impl.glsl IndirectLight for every pixel of a G-buffer (rows [row_first, row_first + h) of a
    full_height-row image). `levels` are the float16 mip levels [d, h, w, 4]. Returns (rgba [h, w, 4], steps [h, w],
    margin [h, w]): margin is the smallest distance of any discontinuous decision from its threshold over the pixel's cones
    (trace_cone64's, metallic against rnd2, and the fractional part of mix(1, MaxSamples, variance) before uint() truncates
    it, divided by MaxSamples because its fp32 error grows with it; an exact integer there counts as a clean decision, which
    it is for the metallic / roughness values 0 and 1 that make it one). The sky texture is the constant colour `sky`."""
    h, w = depth.shape
    full_height = full_height or h
    lv = [l.astype(np.float64) for l in levels]
    ys, xs = np.meshgrid(np.arange(row_first, row_first + h), np.arange(w), indexing="ij")
    f = frame[0] if frame.ndim else frame
    ipv = np.asarray(f["InvProjView"], np.float64).reshape(4, 4)        # OpenTK rows: world = [ndc, 1] @ m
    view_pos = np.asarray(f["ViewPos"], np.float64).reshape(-1)[:3]
    out = np.zeros((h, w, 4))
    steps = np.zeros((h, w), np.int64)
    margin = np.full((h, w), np.inf)
    px = depth != 1.0
    x, y = xs[px], ys[px]
    d = depth[px].astype(np.float64)
    ndc = np.stack([(x + 0.5) / w * 2 - 1, (y + 0.5) / full_height * 2 - 1, d, np.ones_like(d)], -1)
    wp = ndc @ ipv
    frag = wp[:, :3] / wp[:, 3:4]
    normal = decode_unit_vec64(normal_rg[px])
    metallic = metal_rough[px][:, 0].astype(np.float64)
    rough = metal_rough[px][:, 1].astype(np.float64) ** 2
    incoming = frag - view_pos
    variance = (1.0 - metallic - 0.0) + metallic * rough + 0.0 * rough
    mixed = 1.0 * (1.0 - variance) + float(settings.MaxSamples) * variance
    frac = mixed - np.floor(mixed)
    pm = np.where(frac == 0.0, np.inf, np.minimum(frac, 1.0 - frac) / settings.MaxSamples)
    samples = mixed.astype(np.int64)
    refl = incoming - 2.0 * np.sum(normal * incoming, -1, keepdims=True) * normal
    sky_b = np.asarray(sky, np.float32).astype(np.float64) * float(F(settings.GISkyBoxBoost))
    irr = np.zeros((len(x), 3))
    st = np.zeros(len(x), np.int64)
    for i in range(int(samples.max()) if len(x) else 0):
        live = np.nonzero(samples > i)[0]
        k = settings.NoiseIndex + i
        rnd0 = interleaved_gradient_noise(x[live], y[live], k)
        rnd1 = interleaved_gradient_noise(x[live], y[live], k + 1)
        rnd2 = interleaved_gradient_noise(x[live], y[live], k + 2)
        cos_t = rnd0 * 2.0 - 1.0
        phi = rnd1 * 2.0 * np.pi
        sin_t = np.sqrt(1.0 - cos_t * cos_t)
        diffuse = _normalize(normal[live] + np.stack([sin_t * np.cos(phi), sin_t * np.sin(phi), cos_t], -1))
        spec = metallic[live] > rnd2
        r2 = rough[live][:, None]
        direction = np.where(spec[:, None], _normalize(refl[live] * (1 - r2) + diffuse * r2), diffuse)
        max_angle = float(F(0.32))
        angle = np.where(spec, 0.0 * (1 - rough[live]) + max_angle * rough[live], max_angle)
        acc, s, m = trace_cone64(lv, grid_min, grid_max, frag[live], direction, normal[live], angle, float(F(settings.StepMultiplier)),
                                 float(F(settings.NormalRayOffset)))
        irr[live] += acc[:, :3] + (1.0 - acc[:, 3:4]) * sky_b
        st[live] += s
        pm[live] = np.minimum(pm[live], np.minimum(m, np.abs(metallic[live] - rnd2)))
    rgb = irr / samples[:, None] * float(F(settings.GIBoost))
    out[px] = np.concatenate([rgb, np.ones((len(x), 1))], -1)
    steps[px] = st
    margin[px] = pm
    return out, steps, margin


# ------------------------------------------------------------------------------------------------------------ voxelisation
def _rows(a):
    return np.asarray(a, np.float64).reshape(3, 4)


def voxelize64(scene, ci, eps=1e-5):
    """Voxelize/{vertex,geometry,fragment}.glsl + the merge, for factor-only materials and lights without point shadows.

    Each triangle is projected along the dominant axis of its NDC-space normal (geometry.glsl:25-34) and sampled at the
    pixel centres of its bounding box, edges inclusive; the fragment's world position and normal are interpolated with float64
    barycentrics; its voxel is ivec3(MapToZeroOne(FragPos) * size) (fragment.glsl:119-124); its value is
    EvaluateDiffuseLighting over the lights + 0.02 * Albedo + Emissive + EmissiveBias * Albedo, times Alpha
    (fragment.glsl:39-98); voxels keep the per-channel max, alpha 1 where written. The projection plane has as many pixel
    centres along each axis as the grid has voxels; this is the product's rule (DESIGN section 7): the reference's three
    viewports are all Width x Height (Voxelizer.cs:150-162), which differs on non-cubic grids only.

    A sample is *ambiguous* when a decision it takes lies within eps (relative) of its threshold: an edge function, an
    integer voxel coordinate (both neighbouring voxels are flagged), or a dominant-axis tie (the triangle is rasterised along
    every tied axis and all those samples are ambiguous). Returns dict(levels0 = float16 [d, h, w, 4], written, ambiguous
    = bool [d, h, w], fragments = count of unambiguous covered samples (presplit BLAS triangles counted as often as the BLAS
    holds them), ambiguous_samples)."""
    import edge_lib
    size = np.array([ci.Width, ci.Height, ci.Depth])
    gmin = np.array(list(ci.GridMin), np.float64)
    gmax = np.array(list(ci.GridMax), np.float64)
    ext = gmax - gmin
    wt = edge_lib.world_triangles(scene)
    P = np.stack([wt["p0"], wt["p0"] + wt["e1"], wt["p0"] + wt["e2"]], 1)
    nsrc = len(P)
    first = np.full(nsrc, -1, np.int64)
    for k in range(len(wt["frag2src"]) - 1, -1, -1):
        first[wt["frag2src"][k]] = k
    mult = np.bincount(wt["frag2src"], minlength=nsrc)
    tris = scene.blas_triangles[first]
    vid = np.stack([tris["X"], tris["Y"], tris["Z"]], 1).astype(np.int64)
    packed = scene.vertices["Normal"][vid].astype(np.int64)
    nloc = np.stack([(packed & 2047) / 2047.0, ((packed >> 11) & 2047) / 2047.0, ((packed >> 22) & 1023) / 1023.0], -1) * 2.0 - 1.0
    inv = np.stack([_rows(scene.mesh_transforms["InvModelMatrix"][m]) for m in wt["mtid"]])[:, :, :3]
    N = _normalize(np.einsum("tji,tcj->tci", inv, nloc))                  # transpose(invModel) * normal (vertex.glsl:40-41)
    mesh = scene.meshes[tris["MeshId"]]
    mat = scene.materials[mesh["MaterialId"]]
    assert not any((mat[t] != 0).any() for t in ("BaseColorTexture", "EmissiveTexture")), "factor-only materials"
    assert (scene.lights["PointShadowIndex"] < 0).all(), "no point shadows"
    c = mat["BaseColorFactor"].astype(np.int64)
    rgba = np.stack([(c >> s) & 255 for s in (0, 8, 16, 24)], -1) / 255.0
    albedo, alpha = rgba[:, :3], rgba[:, 3]
    emissive = mat["EmissiveFactor"].astype(np.float64) + mesh["EmissiveBias"].astype(np.float64)[:, None] * albedo
    L = scene.lights
    lpos, lcol = L["Position"].astype(np.float64), L["Color"].astype(np.float64)
    lrad = np.maximum(L["Radius"].astype(np.float64), float(F(0.0001)))

    best = np.zeros((int(size[2]), int(size[1]), int(size[0]), 3))
    written = np.zeros(best.shape[:3], bool)
    amb = np.zeros(best.shape[:3], bool)
    frags, amb_samples = 0, 0
    uvw_all = (P - gmin) / ext
    ndc = uvw_all * 2.0 - 1.0
    nw = np.abs(np.cross(ndc[:, 1] - ndc[:, 0], ndc[:, 2] - ndc[:, 0]))
    for t in range(nsrc):
        wts = nw[t]
        dom = 1 if wts[1] > wts[0] else 0
        dom = 2 if wts[2] > wts[dom] else dom
        tied = [a for a in range(3) if a != dom and abs(wts[a] - wts[dom]) <= eps * wts[dom]]
        for axis in [dom] + tied:
            a, b = (axis + 1) % 3, (axis + 2) % 3
            qa, qb = uvw_all[t, :, a] * size[a], uvw_all[t, :, b] * size[b]
            area = (qa[1] - qa[0]) * (qb[2] - qb[0]) - (qb[1] - qb[0]) * (qa[2] - qa[0])
            scale = (max(np.abs(qa).max(), np.abs(qb).max()) + 1.0) ** 2
            if abs(area) <= eps * scale:
                continue                                                   # degenerate in this projection
            i = np.arange(max(0, math.ceil(qa.min() - 0.5 - eps)), min(size[a] - 1, math.floor(qa.max() - 0.5 + eps)) + 1)
            j = np.arange(max(0, math.ceil(qb.min() - 0.5 - eps)), min(size[b] - 1, math.floor(qb.max() - 0.5 + eps)) + 1)
            if not len(i) or not len(j):
                continue
            cx, cy = np.meshgrid(i + 0.5, j + 0.5)
            cx, cy = cx.reshape(-1), cy.reshape(-1)
            wk = []
            for p, q in ((1, 2), (2, 0), (0, 1)):
                wk.append((qa[q] - qa[p]) * (cy - qb[p]) - (qb[q] - qb[p]) * (cx - qa[p]))
            wk = np.stack(wk, -1) / area                                  # barycentrics
            near_edge = (np.abs(wk) * abs(area) <= eps * scale).any(-1)
            inside = (wk >= 0).all(-1) & ~near_edge
            cand = inside | near_edge
            bary = wk[cand]
            frag = bary @ P[t]
            u = (frag - gmin) / ext * size
            delta = eps * np.maximum(1.0, np.abs(u))
            near_int = (np.abs(u - np.round(u)) <= delta).any(-1)
            is_amb = near_edge[cand] | near_int | bool(tied)
            vox_lo, vox_hi = np.floor(u - delta).astype(np.int64), np.floor(u + delta).astype(np.int64)
            ok = lambda v: (v >= 0).all(-1) & (v < size).all(-1)          # noqa: E731
            for v in (vox_lo, vox_hi):
                m = is_amb & ok(v)
                amb[v[m, 2], v[m, 1], v[m, 0]] = True
            amb_samples += int(is_amb.sum()) * int(mult[t])
            keep = ~is_amb & ok(vox_lo)
            if not keep.any():
                continue
            frags += int(keep.sum()) * int(mult[t])
            fp, nn, vox = frag[keep], _normalize(bary[keep] @ N[t]), vox_lo[keep]
            direct = np.zeros((len(fp), 3))
            for li in range(len(L)):
                stl = lpos[li] - fp
                dist = np.linalg.norm(stl, axis=-1)
                cos = np.sum(nn * stl / dist[:, None], -1)
                att = lrad[li] ** 2 / np.maximum(dist * dist, float(F(0.0001)))
                direct += np.where(cos > 0, cos * att, 0.0)[:, None] * lcol[li] * albedo[t]
            val = (direct + albedo[t] * float(F(0.02)) + emissive[t]) * alpha[t]
            np.maximum.at(best, (vox[:, 2], vox[:, 1], vox[:, 0]), val)
            written[vox[:, 2], vox[:, 1], vox[:, 0]] = True
    lv0 = np.zeros(best.shape[:3] + (4,), np.float16)
    lv0[..., :3] = np.where(written[..., None], best, 0.0).astype(np.float16)
    lv0[..., 3] = written.astype(np.float16)
    return dict(level0=lv0, written=written, ambiguous=amb, fragments=frags, ambiguous_samples=amb_samples)
