"""Float64 restatement of the material surface and of the shading frame a normal map is applied in, written from the
engine's shaders and C# (not from oracle/ or csrc/), for every pass that shades a hit with real textures.

Paths are relative to the reference's IDKEngine (SHD = Resource/Shaders):
  SHD/include/Surface.glsl:49-77           GetSurface: five texture() reads at uv, base colour * unpackUnorm4x8(factor),
                                           ReconstructPackedNormal(normal.rg), emissive.rgb * factor, metallic = mr.r,
                                           roughness = mr.g, transmission = tr.r
  SHD/include/Surface.glsl:85-96           SurfaceApplyModificatons: mesh biases, clamps, IOR >= 1
  SHD/include/Surface.glsl:106-111         GetSurfaceVariance (the AOV weight)
  SHD/include/Compression.glsl:1-32        CompressUR11G11B10 (round), DecompressSR11G11B10
  SHD/include/Compression.glsl:78-84       ReconstructPackedNormal: xy = v * 2 - 1, z = sqrt(max(1 - dot(v, v), 0)) of the RAW
                                           [0, 1] sample v
  SHD/include/Math.glsl:49-57              Interpolate(p0, p1, p2, bary) = p0 b.x + p1 b.y + p2 b.z
  SHD/include/Math.glsl:129-137            GetTBN(T, N): N, T normalized, the Gram-Schmidt line commented out,
                                           B = normalize(cross(N, T)), mat3(T, B, N)
  SHD/PathTracing/FirstHit/compute.glsl:125-157  interpolate the decoded model-space normal / tangent, normalize, then
                                           mat3(transpose(InvModelMatrix)), normalize; GetTBN; normalize(mix(worldNormal, tbn * n,
                                           NormalMapStrength)); geometric normal from the positions; flipped towards the ray
                                           (compute.glsl:181-186)
  SHD/GBuffer/VertexPath/vertex.glsl:26-36 per vertex: normalize(mat3(transpose(InvModelMatrix)) * n) (and t)
  SHD/GBuffer/fragment.glsl:36-47          normalize the interpolated pair, GetTBN, mix, negate when !gl_FrontFacing
  SHD/Skinning/compute.glsl:25-44          skinMatrix = sum of weight * joint matrix, normalize(mat3(skinMatrix) * v), then
                                           CompressSR11G11B10
  Source/Utils/ModelLoader.cs:879-884      a slot without an image samples the white fallback (handle 0 here)
  Source/Utils/ModelLoader.cs:989-994      SetSwizzleR(B) on the metallic-roughness texture (IDKPT_TEX_FLAG_R_FROM_B)
  Source/Utils/ModelLoader.cs:1166-1196    glTF sampler: wrap modes, MagFilter (NEAREST = IDKPT_TEX_FLAG_MAG_NEAREST)

texture() in a compute or ray-cast stage has no derivatives, so it reads level 0 (GLSL 4.60 section 8.9). At level 0 the
magnification filter applies: LINEAR = bilinear over the texels around u w - 1/2, v h - 1/2 with exact weights, NEAREST = the
texel that contains (u w, v h), the integer texel index wrapped by REPEAT / CLAMP_TO_EDGE / MIRRORED_REPEAT (GL 4.6 section
8.14.2). An sRGB texel's rgb is decoded by the exact formula of GL 4.6 equation 8.17 before filtering. A two-channel texel
reads (R, G, 0, 1), a one-channel texel (R, 0, 0, 1) (GL 4.6 table 15.1). BC7 / BC5 / BC4 texels come from tests/bcn_ref.py.

Float32 enters only as data: the uploaded vertex records, matrices and factors, and the float32 uv a hit carries. Where float32
evaluation does not pin the sample position, the tests take the envelope of the float64 values over the positions the float32
evaluation allows (`envelope`), as tests/post_ref64.py does for Bloom."""
import numpy as np

import bcn_ref
from edge_lib import K, U32
from idkengine_b200 import capi
from pt_ref64 import decompress_normal as decompress_sr11g11b10   # DecompressSR11G11B10 (Compression.glsl:11-32)
from test_gbuffer import encode_unit_vec, ufloat64                 # noqa: F401  (EncodeUnitVec, the R11G11B10F store)

REPEAT, CLAMP, MIRROR = 10497, 33071, 33648
SLOTS = ("BaseColorTexture", "MetallicRoughnessTexture", "NormalTexture", "EmissiveTexture", "TransmissionTexture")


# --------------------------------------------------------------------------------------------- level-0 sampling
def srgb_to_linear(c):
    """GL 4.6 equation 8.17."""
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def texels(tex):
    """A texture dict (host.Scene.textures) -> float64 [h, w, 4] of what texelFetch at level 0 returns: RGBA8 (sRGB decoded),
    BC7 (sRGB or unorm), BC5 -> (R, G, 0, 1), BC4 / R32F -> (R, 0, 0, 1), RG32F, RGBA32F; the R <- B swizzle applied."""
    fmt = tex.get("format")
    if fmt is None or fmt in (capi.IDKPT_TEX_BC7_UNORM, capi.IDKPT_TEX_BC7_SRGB):
        px = tex["pixels"] if fmt is None else bcn_ref.decode_texture("bc7", tex["data"], tex["width"], tex["height"])
        out = px.astype(np.float64) / 255.0
        if (tex.get("srgb") if fmt is None else fmt == capi.IDKPT_TEX_BC7_SRGB):
            out[..., :3] = srgb_to_linear(out[..., :3])
    else:
        w, h = tex["width"], tex["height"]
        if fmt == capi.IDKPT_TEX_BC5_RG_UNORM:
            c = bcn_ref.decode_texture("bc5", tex["data"], w, h)
        elif fmt == capi.IDKPT_TEX_BC4_R_UNORM:
            c = bcn_ref.decode_texture("bc4", tex["data"], w, h)
        else:
            n = {capi.IDKPT_TEX_RG32F: 2, capi.IDKPT_TEX_R32F: 1, capi.IDKPT_TEX_RGBA32F: 4}[fmt]
            c = np.asarray(tex["data"], np.float32).reshape(h, w, n)
        out = np.zeros((h, w, 4))
        out[..., 3] = 1.0
        out[..., :c.shape[-1]] = c
    if tex.get("flags", 0) & capi.IDKPT_TEX_FLAG_R_FROM_B:
        out[..., 0] = out[..., 2]
    return out


def wrap(i, n, mode):
    if mode == CLAMP:
        return np.clip(i, 0, n - 1)
    if mode == MIRROR:
        m = np.mod(i, 2 * n)
        return np.where(m < n, m, 2 * n - 1 - m)
    return np.mod(i, n)


def _at(tx, x, y, nearest, ws, wt):
    """The filtered value at continuous texel coordinates: (x, y) = (u w, v h) for NEAREST, (u w - 1/2, v h - 1/2) for LINEAR."""
    h, w = tx.shape[:2]
    x0, y0 = np.floor(x), np.floor(y)
    xa, ya = wrap(x0.astype(np.int64), w, ws), wrap(y0.astype(np.int64), h, wt)
    if nearest:
        return tx[ya, xa]
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    xb, yb = wrap(x0.astype(np.int64) + 1, w, ws), wrap(y0.astype(np.int64) + 1, h, wt)
    top = tx[ya, xa] * (1 - fx) + tx[ya, xb] * fx
    bot = tx[yb, xa] * (1 - fx) + tx[yb, xb] * fx
    return top * (1 - fy) + bot * fy


def sample(tex, uv, tx=None, spread=True):
    """texture(sampler2D, uv) at level 0 for float32 uv [N, 2] -> (lo, hi) float64 [N, 4]: the range of the float64 values
    over the texel positions within the float32 rounding of fract(u) (REPEAT) and u * w (- 0.5); lo == hi with spread=False.
    Bilinear values are piecewise bilinear, so the range comes from the two ends and any texel line crossed in between."""
    tx = texels(tex) if tx is None else tx
    h, w = tx.shape[:2]
    ws, wt = tex.get("wrap_s", REPEAT), tex.get("wrap_t", REPEAT)
    nearest = bool(tex.get("flags", 0) & capi.IDKPT_TEX_FLAG_MAG_NEAREST)
    u, v = (np.asarray(uv, np.float32).astype(np.float64)[:, k] for k in (0, 1))
    if ws == REPEAT:
        u = u - np.floor(u)
    if wt == REPEAT:
        v = v - np.floor(v)
    x, y = u * w - (0.0 if nearest else 0.5), v * h - (0.0 if nearest else 0.5)
    if not spread:
        c = _at(tx, x, y, nearest, ws, wt)
        return c, c
    # fract (when |u| < 1 it rounds) and the product each round once in float32, the - 0.5 once more
    dx, dy = 4 * U32 * (np.abs(x) + w), 4 * U32 * (np.abs(y) + h)

    def pts(c, d):
        k = np.floor(c + d)
        return [c - d, c + d, np.where(k > c - d, k, c)]
    vals = [_at(tx, a, b, nearest, ws, wt) for a in pts(x, dx) for b in pts(y, dy)]
    return np.min(vals, 0), np.max(vals, 0)


# --------------------------------------------------------------------------------------------- GetSurface
def unorm8x4(c):
    c = np.asarray(c, np.uint64)
    return np.stack([(c >> np.uint64(s)) & np.uint64(255) for s in (0, 8, 16, 24)], -1).astype(np.float64) / 255.0


def reconstruct_packed_normal(v):
    """ReconstructPackedNormal (Compression.glsl:78-84): z from the raw [0, 1] sample."""
    v = np.asarray(v, np.float64)
    return np.concatenate([v * 2.0 - 1.0, np.sqrt(np.maximum(1.0 - np.sum(v * v, -1, keepdims=True), 0.0))], -1)


def surface(scene, mesh_ids, uv, textures=None, spread=True):
    """GetSurface(material, uv) + SurfaceApplyModificatons(mesh) for hits on meshes `mesh_ids` at float32 uv [N, 2].
    Returns a dict of (lo, hi) float64 ranges: albedo, alpha, normal (tangent space), emissive, metallic, roughness,
    transmission, and the exact ior / cutoff. textures: texels() of scene.textures, computed once by the caller."""
    textures = [texels(t) for t in scene.textures] if textures is None else textures
    mesh = scene.meshes[mesh_ids]
    mat = scene.materials[mesh["MaterialId"]]
    n = len(mesh_ids)
    raw = {}
    for slot in SLOTS:
        lo, hi = np.ones((n, 4)), np.ones((n, 4))        # handle 0: the white fallback
        for hnd in np.unique(mat[slot]):
            if hnd == 0:
                continue
            sel = mat[slot] == hnd
            lo[sel], hi[sel] = sample(scene.textures[int(hnd) - 1], uv[sel], textures[int(hnd) - 1], spread)
        raw[slot] = (lo, hi)
    f = unorm8x4(mat["BaseColorFactor"])
    out = {}
    b = raw["BaseColorTexture"]
    out["albedo"] = tuple(r[:, :3] * f[:, :3] for r in b)
    out["alpha"] = tuple(r[:, 3] * f[:, 3] for r in b)
    # every Surface field below is monotonic in each texel channel, except the tangent-space normal (checked per point)
    out["normal_rg"] = tuple(r[:, :2] for r in raw["NormalTexture"])
    bias = mesh["EmissiveBias"].astype(np.float64)[:, None]
    ef = mat["EmissiveFactor"].astype(np.float64)
    out["emissive"] = tuple(e[:, :3] * ef + bias * a for e, a in zip(raw["EmissiveTexture"], out["albedo"]))
    clamp = lambda x: np.clip(x, 0.0, 1.0)
    m = raw["MetallicRoughnessTexture"]
    out["metallic"] = tuple(clamp(r[:, 0] * mat["MetallicFactor"] + mesh["SpecularBias"]) for r in m)
    out["roughness"] = tuple(clamp(r[:, 1] * mat["RoughnessFactor"] + mesh["RoughnessBias"]) for r in m)
    out["transmission"] = tuple(clamp(r[:, 0] * mat["TransmissionFactor"] + mesh["TransmissionBias"]) for r in raw["TransmissionTexture"])
    out["cutoff"] = (mat["AlphaCutoff"].astype(np.float64),) * 2
    out["strength"] = (mesh["NormalMapStrength"].astype(np.float64),) * 2
    return out


def surface_variance(metallic, transmission, roughness):
    """GetSurfaceVariance (Surface.glsl:106-111), the AOV weight."""
    return (1.0 - metallic - transmission) + metallic * roughness + transmission * roughness


# --------------------------------------------------------------------------------------------- the shading frame
def unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def to_world(inv_model, v):
    """mat3(transpose(InvModelMatrix)) * v for GpuMeshTransform.InvModelMatrix rows [N, 3, 4]."""
    return np.einsum("nji,nj->ni", np.asarray(inv_model, np.float64)[:, :, :3], v)


def apply_normal_map(T, N, n_ts, strength):
    """GetTBN(T, N) as written (Math.glsl:129-137), then normalize(mix(N, tbn * n, strength)) (mix extrapolates above 1)."""
    N, T = unit(N), unit(T)
    B = unit(np.cross(N, T))
    mapped = T * n_ts[:, :1] + B * n_ts[:, 1:2] + N * n_ts[:, 2:]
    s = np.asarray(strength, np.float64)[:, None]
    return unit(N * (1.0 - s) + mapped * s)


def first_hit_frame(vn, vt, bary, inv_model):
    """FirstHit / NHit: interpolate the decoded model-space vectors, normalize, transform, normalize -> (N, T) world."""
    n = unit(np.einsum("nk,nkc->nc", bary, vn))
    t = unit(np.einsum("nk,nkc->nc", bary, vt))
    return unit(to_world(inv_model, n)), unit(to_world(inv_model, t))


def vertex_stage_frame(vn, vt, bary, inv_model):
    """GBuffer vertex.glsl + fragment.glsl (and RecordTransparent): transform and normalize per vertex, interpolate, normalize."""
    wn = unit(np.stack([to_world(inv_model, vn[:, k]) for k in range(3)], 1))
    wt = unit(np.stack([to_world(inv_model, vt[:, k]) for k in range(3)], 1))
    return unit(np.einsum("nk,nkc->nc", bary, wn)), unit(np.einsum("nk,nkc->nc", bary, wt))


# --------------------------------------------------------------------------------------------- skinning
def skin(unskinned, joints, joint_offset=0):
    """Skinning/compute.glsl for GpuUnskinnedVertex records and joint matrices [J, 3, 4] -> float64 (position, normal,
    tangent) [N, 3]: mat3 of the weighted joint sum, NOT its inverse-transpose."""
    jm = np.asarray(joints, np.float64)
    S = np.einsum("nk,nkrc->nrc", unskinned["JointWeights"].astype(np.float64),
                  jm[joint_offset + unskinned["JointIndices"].astype(np.int64)])
    p = np.einsum("nrc,nc->nr", S[:, :, :3], unskinned["Position"].astype(np.float64)) + S[:, :, 3]
    nrm = unit(np.einsum("nrc,nc->nr", S[:, :, :3], decompress_sr11g11b10(unskinned["Normal"])))
    tan = unit(np.einsum("nrc,nc->nr", S[:, :, :3], decompress_sr11g11b10(unskinned["Tangent"])))
    return p, nrm, tan


def compress_sr11g11b10(v, slack):
    """CompressSR11G11B10 of float64 unit vectors [N, 3] whose float32 evaluation may differ by `slack` per component ->
    (codes [N, 3] of the float64 values, ambiguous [N, 3]): GLSL leaves round()'s half-way case to the implementation, and a
    value within the slack of a half-way point may round either way, so such channels are flagged, not pinned."""
    scale = np.array([2047.0, 2047.0, 1023.0])
    x = (np.asarray(v, np.float64) * 0.5 + 0.5) * scale
    code = np.floor(x + 0.5)
    ambiguous = np.abs(x - np.floor(x) - 0.5) <= slack * 0.5 * scale
    return code.astype(np.int64), ambiguous


def unpack_sr11g11b10_codes(packed):
    p = np.asarray(packed, np.uint64)
    return np.stack([p & np.uint64(2047), (p >> np.uint64(11)) & np.uint64(2047), (p >> np.uint64(22)) & np.uint64(1023)], -1).astype(np.int64)


# --------------------------------------------------------------------------------------------- hits
class WorldTriangles:
    """Every BLAS triangle of a scene in world space (float64 products of the float32 ModelMatrix and positions), with what
    the shading needs: vertex records, texcoords, mesh and transform ids, world-space winding as seen from a point."""

    def __init__(self, scene):
        P = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float64)
        idx, xf = [], []
        for inst in scene.blas_instances:
            d = scene.blas_descs[inst["BlasId"]]
            t = scene.blas_triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]]
            idx.append(np.stack([t["X"], t["Y"], t["Z"], t["MeshId"]], 1).astype(np.int64))
            xf.append(np.full(len(t), inst["MeshTransformId"], np.int64))
        idx, xf = np.concatenate(idx), np.concatenate(xf)
        key = np.unique(np.c_[idx, xf], axis=0)          # pre-split fragments reference the same source triangle
        self.vid, self.mesh, self.xf = key[:, :3], key[:, 3], key[:, 4]
        M = scene.mesh_transforms["ModelMatrix"].astype(np.float64)[self.xf]
        self.p = np.einsum("nrc,nkc->nkr", M[:, :, :3], P[self.vid]) + M[:, None, :, 3]
        self.e1, self.e2 = self.p[:, 1] - self.p[:, 0], self.p[:, 2] - self.p[:, 0]
        self.n = np.cross(self.e1, self.e2)
        self.inv = scene.mesh_transforms["InvModelMatrix"][self.xf]
        self.vn = decompress_sr11g11b10(scene.vertices["Normal"][self.vid])
        self.vt = decompress_sr11g11b10(scene.vertices["Tangent"][self.vid])
        self.uv = scene.vertices["TexCoord"][self.vid].astype(np.float64)

    def subset(self, keep):
        s = object.__new__(WorldTriangles)
        for k, v in self.__dict__.items():
            s.__dict__[k] = v[keep]
        return s

    def front(self, eye):
        """gl_FrontFacing for a view from `eye`: counter-clockwise in window space = the world-space winding faces the eye."""
        return np.einsum("nk,nk->n", self.n, eye - self.p[:, 0]) > 0.0

    def bary_error(self, tri, O, D, t):
        """A bound on the float32 ray-triangle test's barycentric error (edge_lib's margin without its absolute floor)."""
        e1, e2, n = self.e1[tri], self.e2[tri], self.n[tri]
        l1, l2 = np.linalg.norm(e1, axis=1), np.linalg.norm(e2, axis=1)
        kappa = l1 * l2 / np.abs(np.einsum("nk,nk->n", D, n))
        S = np.linalg.norm(O - self.p[tri, 0], axis=1) + np.linalg.norm(O, axis=1) + np.linalg.norm(self.p[tri, 0], axis=1) + np.abs(t)
        return K * U32 * kappa * (1.0 + S / np.minimum(l1, l2))


def envelope(fn, bary, db):
    """An approximate range of fn(barycentrics) (a dict of (lo, hi) arrays) over the barycentrics within db [N] of `bary`: the
    union of fn's ranges at the point and at the four moves of +-db along two edges. It is not a bound: a bilinear sample
    along a diagonal, or a texel line crossed between the points, can have an extremum inside, and the tests widen it by a
    measured slack."""
    moves = [np.zeros(3), np.array([1.0, -1.0, 0.0]), np.array([-1.0, 1.0, 0.0]), np.array([1.0, 0.0, -1.0]), np.array([-1.0, 0.0, 1.0])]
    acc = None
    for mv in moves:
        r = fn(bary + db[:, None] * mv)
        if acc is None:
            acc = {k: [np.array(v[0], np.float64), np.array(v[1], np.float64)] for k, v in r.items()}
        else:
            for k, v in r.items():
                acc[k][0] = np.minimum(acc[k][0], v[0])
                acc[k][1] = np.maximum(acc[k][1], v[1])
    return acc


def shade_point(scene, wt, tri, bary, D, textures, order, spread=True):
    """The surface and shading normal at barycentrics `bary` of world triangles `tri`, seen along D. order: "first_hit"
    (flipped towards the ray, FirstHit) or "vertex" (negated on a back face, GBuffer / RecordTransparent).
    Returns a dict of (lo, hi) ranges; the normal's range is taken over the four corners of the sampled (r, g) box, which is
    approximate: the mapped, normalised normal is not monotonic in r and g."""
    uv = np.einsum("nk,nkc->nc", bary, wt.uv[tri]).astype(np.float32)
    s = surface(scene, wt.mesh[tri], uv, textures, spread)
    s["uv"] = (uv.astype(np.float64),) * 2
    frame = first_hit_frame if order == "first_hit" else vertex_stage_frame
    N, T = frame(wt.vn[tri], wt.vt[tri], bary, wt.inv[tri])
    lo, hi = s["normal_rg"]
    normals, flipped = [], np.zeros(len(tri), bool)
    for cx in (lo[:, 0], hi[:, 0]):
        for cy in (lo[:, 1], hi[:, 1]):
            n = apply_normal_map(T, N, reconstruct_packed_normal(np.stack([cx, cy], 1)), s["strength"][0])
            flipped |= np.einsum("nk,nk->n", n, N) < 0.0
            if order == "first_hit":
                n = np.where((np.einsum("nk,nk->n", -D, n) < 0.0)[:, None], -n, n)
            else:
                front = np.einsum("nk,nk->n", wt.n[tri], -D) > 0.0
                n = np.where(front[:, None], n, -n)
            normals.append(n)
    s["normal"] = (np.min(normals, 0), np.max(normals, 0))
    s["normal_oct"] = (np.min([encode_unit_vec(n) for n in normals], 0), np.max([encode_unit_vec(n) for n in normals], 0))
    # w = 1 - m (1 - r) - t (1 - r) falls with m and t and grows with r
    s["weight"] = (surface_variance(s["metallic"][1], s["transmission"][1], s["roughness"][0]),
                   surface_variance(s["metallic"][0], s["transmission"][0], s["roughness"][1]))
    s["flipped"] = (flipped, flipped)         # the mapped normal left N's hemisphere (mix extrapolating past strength 1)
    return s


def closest_hits(wt, O, D, keep=None):
    """Float64 closest hit through pt_ref64.closest's strict / lenient margins over the triangles `keep` (a mask) ->
    (kind, triangle index into wt, t, barycentrics)."""
    import pt_ref64
    idx = np.arange(len(wt.mesh)) if keep is None else np.nonzero(keep)[0]
    sub = wt.subset(idx)
    out = [pt_ref64.closest(sub, O[k:k + 128], D[k:k + 128]) for k in range(0, len(O), 128)]
    kind, best, t, _, bary = (np.concatenate([o[i] for o in out]) for i in range(5))
    return kind, idx[best], t, bary


# --------------------------------------------------------------------------------------------- the scene
def _tangents(normals, rng):
    """Caller-supplied tangents that are neither orthogonal to the normals nor of unit length (components within [-1, 1])."""
    from idkengine_b200.host import default_tangents
    t = default_tangents(normals).astype(np.float64) + 0.55 * normals + rng.uniform(-0.1, 0.1, normals.shape)
    return (0.62 * t / np.abs(t).max(1, keepdims=True)).astype(np.float32)


def _sphere_uv(p, c, su, sv, ou, ov):
    d = unit(p - np.asarray(c))
    return np.stack([np.arctan2(d[:, 2], d[:, 0]) / (2 * np.pi) * su + ou, np.arccos(np.clip(d[:, 1], -1, 1)) / np.pi * sv + ov], 1)


def textured_scene():
    """(scene for the device, the same scene with its block-compressed textures decoded for the CPU oracle, camera).

    Textures: 1 BC5 normal map 24x40 (REPEAT, MIRRORED_REPEAT); 2 BC7 sRGB base colour 32x20 with an alpha checker
    (CLAMP_TO_EDGE, REPEAT); 3 BC7 unorm metallic-roughness 16x12 read R <- B (MIRRORED_REPEAT both); 4 BC4 transmission
    20x28 (CLAMP_TO_EDGE both); 5 RGBA8 sRGB emissive 12x9 with NEAREST magnification (REPEAT, MIRRORED_REPEAT).
    Meshes (one instance each): 0 a sphere under a non-uniform scale, strength 0.8, base colour + metallic-roughness;
    1 a cylinder under a shear, strength 4, emissive + transmission; 2 a sphere under a mirroring transform (negative
    determinant), strength 1, base colour with an alpha cut-out; 3 a double-sided quad seen from behind, strength 1,
    texcoords far outside [0, 1] and negative; 4 a cylinder with strength 1 and no normal texture (the white fallback
    (1, 1, 0) in tangent space); 5 a back wall with a normal texture at strength 0."""
    from idkengine_b200 import scenes
    from idkengine_b200.host import Model, Scene, compute_vertex_normals, trs_matrix
    rng = np.random.default_rng(41)
    yy, xx = np.mgrid[0:40, 0:24]
    nrm = np.stack([128 + 110 * np.sin(xx * 0.9 + yy * 0.35), 128 + 110 * np.cos(yy * 0.7 - xx * 0.2)], -1)
    nrm = np.clip(nrm + rng.uniform(-10, 10, nrm.shape), 0, 255).astype(np.uint8)
    base = np.concatenate([rng.integers(30, 256, (20, 32, 3)), np.where(((np.mgrid[0:20, 0:32][0] // 4 + np.mgrid[0:20, 0:32][1] // 4) % 2)[..., None] == 0, 250, 15)], -1).astype(np.uint8)
    mr = rng.integers(0, 256, (12, 16, 4)).astype(np.uint8)
    tr = rng.integers(0, 256, (28, 20, 1)).astype(np.uint8)
    em = np.concatenate([rng.integers(0, 256, (9, 12, 3)), np.full((9, 12, 1), 255)], -1).astype(np.uint8)
    gpu_tex = [dict(format=capi.IDKPT_TEX_BC5_RG_UNORM, width=24, height=40, data=bcn_ref.encode_texture("bc5", nrm), wrap_s=REPEAT, wrap_t=MIRROR),
               dict(format=capi.IDKPT_TEX_BC7_SRGB, width=32, height=20, data=bcn_ref.encode_texture("bc7", base), wrap_s=CLAMP, wrap_t=REPEAT),
               dict(format=capi.IDKPT_TEX_BC7_UNORM, width=16, height=12, data=bcn_ref.encode_texture("bc7", mr), wrap_s=MIRROR, wrap_t=MIRROR,
                    flags=capi.IDKPT_TEX_FLAG_R_FROM_B),
               dict(format=capi.IDKPT_TEX_BC4_R_UNORM, width=20, height=28, data=bcn_ref.encode_texture("bc4", tr), wrap_s=CLAMP, wrap_t=CLAMP),
               dict(pixels=em, srgb=True, wrap_s=REPEAT, wrap_t=MIRROR, flags=capi.IDKPT_TEX_FLAG_MAG_NEAREST)]
    specs = [dict(color=(0.9, 0.85, 0.8), metallic=0.9, roughness=0.7),
             dict(color=(0.7, 0.8, 0.9), emissive=(0.8, 0.5, 0.3), transmission=0.6, roughness=0.5),
             dict(color=(1.0, 0.95, 0.9), cutoff=0.5, roughness=0.4),
             dict(color=(0.6, 0.9, 0.5), roughness=0.3, metallic=0.2),
             dict(color=(0.8, 0.4, 0.3), roughness=0.9),
             dict(color=(0.5, 0.5, 0.55), roughness=0.6)]
    meshes, mats = scenes._materials(specs)
    for k, slots in {0: dict(NormalTexture=1, BaseColorTexture=2, MetallicRoughnessTexture=3), 1: dict(NormalTexture=1, EmissiveTexture=5,
                     TransmissionTexture=4), 2: dict(NormalTexture=1, BaseColorTexture=2), 3: dict(NormalTexture=1, EmissiveTexture=5,
                     MetallicRoughnessTexture=3), 5: dict(NormalTexture=1, BaseColorTexture=2)}.items():
        for f, hnd in slots.items():
            mats[f][k] = hnd
    mats["IsDoubleSided"][3] = 1
    meshes["NormalMapStrength"] = [0.8, 4.0, 1.0, 1.0, 1.0, 0.0]
    meshes["EmissiveBias"][3] = 0.25
    meshes["RoughnessBias"][0] = -0.2
    shear = np.array([[1.0, 0.45, 0.0, 0.2], [0.0, 1.0, 0.0, -0.4], [0.3, 0.0, 1.0, 0.0], [0, 0, 0, 1.0]])
    mirror = trs_matrix((-0.8, 1.15, 0.9), 30.0, (1.7, 0.3, 0.0))

    def model(pi, k, matrix, uv):
        p, i = pi
        n = compute_vertex_normals(p, i)
        m, t = meshes[k:k + 1].copy(), mats[k:k + 1].copy()
        m["MaterialId"] = 0
        return Model(p, i, normals=n, tangents=_tangents(n.astype(np.float64), rng), texcoords=uv.astype(np.float32),
                     meshes=m, materials=t, model_matrix=matrix)
    sph = scenes.uv_sphere((0, 0, 0), 0.8, 12, 20)
    cyl = scenes.cylinder((0, -0.8, 0), 0.5, 1.6, 20, 6)
    cyl_uv = lambda p, s, o: np.stack([np.arctan2(p[:, 2], p[:, 0]) / (2 * np.pi) * s + o, p[:, 1] * 1.3], 1)
    quad = scenes.quad([-0.7, -0.6, 0], [-0.7, 0.6, 0], [0.7, 0.6, 0], [0.7, -0.6, 0])      # faces -z: seen from behind
    wall = scenes.quad([-4, -2.5, -2.5], [4, -2.5, -2.5], [4, 3, -2.5], [-4, 3, -2.5])
    models = [model(sph, 0, trs_matrix((1.4, 0.75, 1.0), 25.0, (-1.9, 0.7, 0.0)), _sphere_uv(sph[0], (0, 0, 0), 2.0, 1.5, -0.3, 0.1)),
              model(cyl, 1, shear @ trs_matrix(1.0, 0.0, (0.0, 0.6, 0.3)), cyl_uv(cyl[0], 3.0, -1.1)),
              model(sph, 2, mirror, _sphere_uv(sph[0], (0, 0, 0), 1.0, 1.0, 0.0, 0.0)),
              model(quad, 3, trs_matrix(1.0, 15.0, (-0.3, -1.2, 1.2)), np.array([[-7.3, -3.1], [-7.3, 4.6], [5.2, 4.6], [5.2, -3.1]])),
              model(cyl, 4, trs_matrix((0.6, 0.7, 0.6), 0.0, (2.0, -1.3, 1.0)), cyl_uv(cyl[0], 2.0, 0.25)),
              model(wall, 5, None, np.array([[-2.2, -1.0], [2.7, -1.0], [2.7, 2.2], [-2.2, 2.2]]))]
    gpu = Scene().add(*models, threads=1)
    gpu.textures = gpu_tex
    cpu = Scene().add(*models, threads=1)
    cpu.textures = [oracle_texture(t) for t in gpu_tex]
    cam = dict(position=(0.0, 0.2, 5.5), view_dir=(0.0, -0.05, -1.0), fov_y_deg=55.0)
    return gpu, cpu, cam


def oracle_texture(t):
    """The CPU oracle samples uncompressed texels only: a block-compressed texture decoded by tests/bcn_ref.py."""
    fmt = t.get("format")
    common = dict(wrap_s=t["wrap_s"], wrap_t=t["wrap_t"], flags=t.get("flags", 0))
    if fmt in (capi.IDKPT_TEX_BC7_UNORM, capi.IDKPT_TEX_BC7_SRGB):
        return dict(pixels=bcn_ref.decode_texture("bc7", t["data"], t["width"], t["height"]), srgb=fmt == capi.IDKPT_TEX_BC7_SRGB, **common)
    if fmt == capi.IDKPT_TEX_BC5_RG_UNORM:
        return dict(format=capi.IDKPT_TEX_RG32F, width=t["width"], height=t["height"],
                    data=bcn_ref.decode_texture("bc5", t["data"], t["width"], t["height"]), **common)
    if fmt == capi.IDKPT_TEX_BC4_R_UNORM:
        return dict(format=capi.IDKPT_TEX_R32F, width=t["width"], height=t["height"],
                    data=bcn_ref.decode_texture("bc4", t["data"], t["width"], t["height"]), **common)
    return t


# --------------------------------------------------------------------------------------------- the passes, per pixel
def pcg_rnd01(seed):
    """Random.glsl:16-33 on uint32 seeds -> (float32 value, next seed)."""
    seed = (seed.astype(np.uint64) * np.uint64(747796405) + np.uint64(2891336453)) & np.uint64(0xFFFFFFFF)
    word = (((seed >> ((seed >> np.uint64(28)) + np.uint64(4))) ^ seed) * np.uint64(277803737)) & np.uint64(0xFFFFFFFF)
    word = ((word >> np.uint64(22)) ^ word) & np.uint64(0xFFFFFFFF)
    return word.astype(np.float32) / np.float32(4294967296.0), seed


def _judge(scene, wt, textures, O, D, keep, order, cutout_retry):
    """Closest hits of rays (O, D) over triangles `keep`, alpha-tested: a hit whose alpha range lies below its cutoff is
    discarded and, with cutout_retry, the ray is traced again without that mesh (the cut-out meshes here are convex and
    single-sided, so nothing else of them lies behind). Returns (pix, tri, bary, shaded ranges, counts)."""
    kind, tri, t, bary = closest_hits(wt, O, D, keep)
    counts = dict(edge=int((kind == -1).sum()), alpha_ambiguous=0, discarded=0)
    pix = np.nonzero(kind == 1)[0]
    for attempt in range(2):
        db = wt.bary_error(tri[pix], O[pix], D[pix], t[pix])
        rng = envelope(lambda b: shade_point(scene, wt, tri[pix], b, D[pix], textures, order), bary[pix], db)
        cut = rng["cutoff"][0]
        below, above = rng["alpha"][1] < cut, rng["alpha"][0] >= cut
        counts["alpha_ambiguous"] += int((~below & ~above).sum())
        counts["discarded"] += int(below.sum())
        again = pix[below]
        if attempt == 1 or not cutout_retry or len(again) == 0:
            break
        # trace the discarded rays again without the meshes they passed through
        gone = np.isin(wt.mesh, np.unique(wt.mesh[tri[again]]))
        k2, tr2, t2, b2 = closest_hits(wt, O[again], D[again], keep & ~gone)
        counts["edge"] += int((k2 == -1).sum())
        ok = k2 == 1
        tri[again[ok]], t[again[ok]], bary[again[ok]] = tr2[ok], t2[ok], b2[ok]
        pix = np.concatenate([pix[above], again[ok]])
    sel = above
    rng = {k: (v[0][sel], v[1][sel]) for k, v in rng.items()}
    counts["judged"] = int(sel.sum())
    return pix[sel], tri[pix[sel]], bary[pix[sel]], rng, counts


def gbuffer_ref(scene, frame, w, h, textures=None):
    """The G-buffer pass at pixel centres (unjittered): the ranges of every attachment before its store, per judged pixel."""
    textures = [texels(t) for t in scene.textures] if textures is None else textures
    f = frame[0]
    ipv = np.asarray(f["InvProjView"], np.float64).reshape(4, 4).T
    eye = np.asarray(f["ViewPos"], np.float64)
    ys, xs = np.mgrid[0:h, 0:w]
    ndc = np.stack([(xs.ravel() + 0.5) / w * 2 - 1, (ys.ravel() + 0.5) / h * 2 - 1, np.ones(w * h), np.ones(w * h)])
    q = ipv @ ndc
    D = unit((q[:3] / q[3]).T - eye)
    O = np.broadcast_to(eye, D.shape).copy()
    wt = WorldTriangles(scene)
    mat = scene.materials[scene.meshes["MaterialId"][wt.mesh]]
    keep = (mat["AlphaCutoff"] != 2.0) & ((mat["IsDoubleSided"] != 0) | wt.front(eye))
    pix, tri, bary, rng, counts = _judge(scene, wt, textures, O, D, keep, "vertex", True)
    counts["back_face"] = int((~wt.front(eye)[tri]).sum())
    return pix, wt.mesh[tri], rng, counts


def first_hit_ref(scene, frame, w, h, textures=None):
    """FirstHit at RayDepth 1 through each pixel's jittered sample (lens radius 0): the ranges of the surface and the
    shading normal per judged pixel. Rays that pass through a cut-out are not judged (the path goes on to a later bounce)."""
    import pt_ref64
    textures = [texels(t) for t in scene.textures] if textures is None else textures
    ys, xs = np.mgrid[0:h, 0:w]
    seed = (ys.ravel() * 4096 + xs.ravel()).astype(np.uint64)
    sx, seed = pcg_rnd01(seed)
    sy, _ = pcg_rnd01(seed)
    D = pt_ref64.camera_dirs(frame, xs.ravel() + sx.astype(np.float64), ys.ravel() + sy.astype(np.float64), w, h)
    O = np.broadcast_to(pt_ref64.camera(frame)[0], D.shape).copy()
    wt = WorldTriangles(scene)
    pix, tri, bary, rng, counts = _judge(scene, wt, textures, O, D, np.ones(len(wt.mesh), bool), "first_hit", False)
    return pix, wt.mesh[tri], rng, counts


def product_range(a, b):
    """[lo, hi] of x * y over x in a, y in b (interval arithmetic)."""
    c = [a[i] * b[j] for i in (0, 1) for j in (0, 1)]
    return np.min(c, 0), np.max(c, 0)


def outside(got, lo, hi):
    """How far float32 values lie outside [lo, hi] (0 inside)."""
    g = np.asarray(got, np.float64)
    return np.maximum(np.maximum(lo - g, g - hi), 0.0)
