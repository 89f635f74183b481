"""Float64 rules for the path tracer's shading, judged bounce by bounce on the exported path states (no oracle calls).

The tests (tests/test_pt_shading_ref*.py) render tiny scenes at RayDepth = 1, 2, ... D in fresh contexts and read every
pixel's GpuWavefrontRay after the last bounce. The first k bounces do not depend on RayDepth, so run d and run d + 1 agree on
every ray that was dead before bounce d, and the rays they disagree on are exactly the ones bounce d shaded
(depth_states checks this before anything rests on it). That gives each pixel's state before and after each bounce.

Each transition S_k -> S_k+1 is then judged without re-deriving a single random number: the incoming ray is intersected
with the scene in float64 (only rays with an unambiguous closest hit or a clear miss, with edge_lib's margins), the
material is unpacked from the mesh as uploaded (unorm8 base colour, mesh biases and clamps of Surface.glsl), and the
outgoing state must satisfy rules that hold whatever branch the random numbers chose:

  miss      radiance += sky(dir) * throughput (2 ulp), the path ends
  hit       radiance += emissive * throughput (2 ulp; throughput after Beer-Lambert when leaving a volumetric mesh)
  origin    P + 0.001 n_g', n_g' the geometric normal turned to the incoming side (away from it on the transmission branch)
  throughput  float32(thr * f) exactly, f the branch's BSDF (pdf == 1); with Russian roulette (k >= 1) q / max(q)
  direction (roughness 0) mirror = reflect, volumetric transmission = Snell or reflect on TIR, thin transmission = the
            incoming direction, diffuse = the shading-normal hemisphere
  prevIor   kept by diffuse / mirror / TIR, the mesh IOR on entering a volumetric mesh, 1 on leaving it or on thin transmission

Statistics with closed-form expectations (branch counts against the Schlick Fresnel, cosine sampling, a furnace, the
irradiance of a per-face cube sky) complete the picture. Every output is deterministic, so none of them can flake.
"""
import numpy as np

from edge_lib import EPS, GRAZE_KAPPA, K, U32
from idkengine_b200 import scenes
from idkengine_b200.host import Scene

F32 = np.float32
OFFSET = 0.001
SKY_FACE = 64
# per-face constant sky (+X, -X, +Y, -Y, +Z, -Z) and a sentinel colour that no furnace path may see
SKY_COLORS = np.array([[0.9, 0.25, 0.1], [0.1, 0.8, 0.3], [0.35, 0.45, 1.0], [0.05, 0.07, 0.02], [0.7, 0.65, 0.2],
                       [0.2, 0.55, 0.9]], np.float32)
SENTINEL = 1.0e4


# --------------------------------------------------------------------------------------------- small float64 helpers
def unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def dot(a, b):
    return np.einsum("...k,...k->...", a, b)


def reflect(d, n):
    return d - 2.0 * dot(n, d)[..., None] * n


def decode_dir(px, py):
    """DecodeUnitVec (Compression.glsl) in float64: octahedral [0, 1]^2 -> unit vector."""
    fx = np.asarray(px, np.float64) * 2.0 - 1.0
    fy = np.asarray(py, np.float64) * 2.0 - 1.0
    nz = 1.0 - np.abs(fx) - np.abs(fy)
    t = np.maximum(-nz, 0.0)
    nx = fx + np.where(fx >= 0.0, -t, t)
    ny = fy + np.where(fy >= 0.0, -t, t)
    return unit(np.stack([nx, ny, nz], -1))


def decompress_normal(packed):
    """DecompressSR11G11B10 in float64."""
    p = np.asarray(packed, np.uint64)
    return np.stack([(p & 2047) / 2047.0 * 2.0 - 1.0, ((p >> 11) & 2047) / 2047.0 * 2.0 - 1.0,
                     ((p >> 22) & 1023) / 1023.0 * 2.0 - 1.0], -1)


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, F32))).astype(np.float64)


# --------------------------------------------------------------------------------------------- the cube sky
def cube_sky(face_size=SKY_FACE):
    """Faces [6, n, n, 4] float32, each face one constant colour (SKY_COLORS)."""
    faces = np.zeros((6, face_size, face_size, 4), np.float32)
    faces[..., :3] = SKY_COLORS[:, None, None, :]
    faces[..., 3] = 1.0
    return faces


def sky_lookup(d, face_size=SKY_FACE):
    """(colour [N, 3] float64, face [N], clear [N]): the face a direction selects (GL table 8.19, ties x >= y >= z) and
    whether it lies more than one texel from every face edge, where the seamless bilinear filter cannot reach another face."""
    d = np.asarray(d, np.float64)
    a = np.abs(d)
    xm = (a[:, 0] >= a[:, 1]) & (a[:, 0] >= a[:, 2])
    ym = ~xm & (a[:, 1] >= a[:, 2])
    axis = np.where(xm, 0, np.where(ym, 1, 2))
    ma = a[np.arange(len(d)), axis]
    face = 2 * axis + (d[np.arange(len(d)), axis] < 0)
    other = np.where(axis[:, None] == 0, a[:, [1, 2]], np.where(axis[:, None] == 1, a[:, [0, 2]], a[:, [0, 1]]))
    edge = np.max(other, 1) / ma                      # 1 on a face edge; texels are 2 / n wide in these units
    clear = edge < 1.0 - 2.0 / face_size
    return SKY_COLORS[face].astype(np.float64), face, clear


def face_normal(d):
    """CubemapFaceNormal (Math.glsl): minus the sign of the major component(s)."""
    a = np.abs(d)
    m = a >= np.maximum(a[:, [1, 2, 0]], a[:, [2, 0, 1]])
    return m * -np.sign(d)


def cosine_weighted_sky(n, samples=1 << 22, seed=5):
    """(mean, band): the cosine-weighted hemisphere mean of the face colours about unit normal n (stratified float64
    quadrature of the nearest-face sky), and the cosine-weighted share of directions within one texel of a face edge."""
    rng = np.random.RandomState(seed)
    m = int(np.sqrt(samples))
    u = (np.arange(m)[:, None] + rng.uniform(size=(m, m))) / m
    v = (np.arange(m)[None, :] + rng.uniform(size=(m, m))) / m
    r, phi = np.sqrt(u).reshape(-1), (2.0 * np.pi * v).reshape(-1)          # Malley: cosine-distributed directions
    local = np.stack([r * np.cos(phi), r * np.sin(phi), np.sqrt(np.maximum(1.0 - r * r, 0.0))], 1)
    n = unit(n)
    t = unit(np.cross(n, [0.0, 0.0, 1.0] if abs(n[2]) < 0.9 else [1.0, 0.0, 0.0]))
    b = np.cross(n, t)
    d = local[:, :1] * t + local[:, 1:2] * b + local[:, 2:] * n
    col, _, clear = sky_lookup(d)
    return col.mean(0), 1.0 - clear.mean()


# --------------------------------------------------------------------------------------------- scenes
def _unshared(pi):
    """A mesh whose triangles have their own vertices, so every vertex normal is its face's normal."""
    p, i = pi
    return p[i.reshape(-1)], np.arange(3 * len(i), dtype=np.uint32).reshape(-1, 3)


def build(parts, specs, biases=None, lights=()):
    """parts: list of ((positions, indices), mesh index); specs: scenes._materials specs; biases: {mesh: {field: value}}.
    One model, identity transform, no shared vertices between faces."""
    meshes, mats = scenes._materials(specs)
    for k, fields in (biases or {}).items():
        for name, value in fields.items():
            meshes[name][k] = value
    a = scenes._Assembler()
    for pi, k in parts:
        a.add(_unshared(pi), k)
    scene = Scene().add(a.model(meshes, mats, name="pt_ref64"), threads=1)
    for pos, color, radius in lights:
        scene.add_light(pos, color, radius)
    return scene


def floor(size=60.0, y=0.0):
    s = float(size)
    return scenes.quad([-s, y, -s], [-s, y, s], [s, y, s], [s, y, -s])


def box_faces(mn, mx):
    """An axis-aligned box as six quads wound outwards (each face its own vertices)."""
    p, i = scenes.box(mn, mx)
    c = p.astype(np.float64).mean(0)
    tri = p[i].astype(np.float64)
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    out = np.einsum("ij,ij->i", n, tri.mean(1) - c) > 0
    i = np.where(out[:, None], i, i[:, [0, 2, 1]])
    return p, i.astype(np.uint32)


# --------------------------------------------------------------------------------------------- scene tables
class Tables:
    """Source triangles (float64 world positions; every scene here has one instance with the identity transform), their
    vertex normals as uploaded, and every mesh's surface (Surface.glsl GetSurface with 1x1 white textures +
    SurfaceApplyModificatons)."""

    def __init__(self, scene):
        assert len(scene.blas_instances) == 1
        mt = scene.mesh_transforms[0]["ModelMatrix"].astype(np.float64)
        assert np.array_equal(mt, np.eye(4)[:3]), "identity transform expected"
        tri = scene.blas_triangles
        key = np.stack([tri["X"], tri["Y"], tri["Z"], tri["MeshId"]], 1).astype(np.int64)
        key = np.unique(key, axis=0)
        P = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float64)
        self.p = np.stack([P[key[:, 0]], P[key[:, 1]], P[key[:, 2]]], 1)          # [M, 3, 3]
        self.vn = decompress_normal(scene.vertices["Normal"][key[:, :3]])         # [M, 3, 3]
        self.mesh = key[:, 3]
        e1, e2 = self.p[:, 1] - self.p[:, 0], self.p[:, 2] - self.p[:, 0]
        self.e1, self.e2, self.n = e1, e2, np.cross(e1, e2)
        self.ng = unit(self.n)
        me, ma = scene.meshes, scene.materials[scene.meshes["MaterialId"]]
        c = ma["BaseColorFactor"].astype(np.uint64)
        self.albedo32 = (np.stack([c & 255, (c >> 8) & 255, (c >> 16) & 255], 1).astype(F32) / F32(255))   # unorm8, as uploaded
        self.albedo = self.albedo32.astype(np.float64)
        self.emissive = ma["EmissiveFactor"].astype(np.float64) + me["EmissiveBias"][:, None].astype(np.float64) * self.albedo
        self.absorbance = np.maximum(ma["Absorbance"].astype(np.float64) + me["AbsorbanceBias"].astype(np.float64), 0.0)
        self.metallic = np.clip(ma["MetallicFactor"].astype(np.float64) + me["SpecularBias"], 0.0, 1.0)
        self.roughness = np.clip(ma["RoughnessFactor"].astype(np.float64) + me["RoughnessBias"], 0.0, 1.0)
        self.transmission = np.clip(ma["TransmissionFactor"].astype(np.float64) + me["TransmissionBias"], 0.0, 1.0)
        self.ior32 = np.maximum(ma["IOR"].astype(F32) + me["IORBias"].astype(F32), F32(1.0))
        self.ior = self.ior32.astype(np.float64)
        self.volumetric = ma["IsVolumetric"] != 0
        self.tint = me["TintOnTransmissive"] != 0
        self.lights = scene.lights


def closest(tb, O, D, tmax=None, spread=None, want_strict=False):
    """Float64 closest hit of rays (O, D) against every source triangle, with edge_lib's strict / lenient margins.
    Returns (kind, tri, t, eps_t, barycentrics) with kind 1 = unambiguous hit (the nearest strict triangle, every other lenient candidate
    clearly farther), 0 = clear miss (no lenient candidate), -1 = not judged.
    tmax: per-ray (limit, its uncertainty) [N]: only hits with t < limit count, and a hit within the uncertainty of it is not
    judged. spread: per-ray (a, b) [N]: the float32 ray may start up to a away from O and point up to b radians away from D,
    which widens every margin by the displacement a + b t on the triangle's plane. want_strict: also return whether any
    triangle is in the strict set (an any-hit verdict that holds whichever of them is the closest)."""
    O, D = np.asarray(O, np.float64), np.asarray(D, np.float64)
    N = len(O)
    p0, e1, e2, n = tb.p[:, 0], tb.e1, tb.e2, tb.n
    l1, l2 = np.linalg.norm(e1, axis=1), np.linalg.norm(e2, axis=1)
    lmin, area2 = np.minimum(l1, l2), l1 * l2
    rop0 = O[:, None, :] - p0[None]
    det = D @ n.T
    q = np.cross(rop0, D[:, None, :])
    with np.errstate(all="ignore"):
        inv = 1.0 / det
        b1 = -np.einsum("rmk,mk->rm", q, e2) * inv
        b2 = np.einsum("rmk,mk->rm", q, e1) * inv
        b0 = 1.0 - b1 - b2
        t = -np.einsum("mk,rmk->rm", n, rop0) * inv
        kappa = np.linalg.norm(D, axis=1)[:, None] * area2[None] / np.abs(det)
        S = np.linalg.norm(rop0, axis=2) + np.linalg.norm(O, axis=1)[:, None] + np.linalg.norm(p0, axis=1)[None]
        eb = EPS + K * U32 * kappa * (1.0 + S / lmin[None])
        et = EPS * np.abs(t) + K * U32 * area2[None] * S / np.abs(det)
        dpos = 0.0
        if spread is not None:
            # a displacement d of the ray moves its hit on the plane by d / cos, a barycentric by that over the lowest height
            dpos = np.asarray(spread[0], np.float64)[:, None] + np.asarray(spread[1], np.float64)[:, None] * np.abs(t)
            lmax = np.maximum(np.maximum(l1, l2), np.linalg.norm(tb.p[:, 2] - tb.p[:, 1], axis=1))
            dn = np.linalg.norm(D, axis=1)[:, None] / np.abs(det)
            eb = eb + dpos * lmax[None] * dn
            et = et + dpos * np.linalg.norm(n, axis=1)[None] * dn
        bmin = np.minimum(np.minimum(b0, b1), b2)
        graze = ~(kappa <= GRAZE_KAPPA)
        strict = ~graze & (bmin >= eb) & (t >= et)
        dist = np.abs(np.einsum("mk,rmk->rm", n, rop0)) / np.linalg.norm(n, axis=1)[None]
        lenient = (~graze & (bmin >= -eb) & (t >= -et)) | (graze & (dist <= EPS * lmin[None] + K * U32 * S + dpos))
        if tmax is not None:
            lim, elim = (np.asarray(v, np.float64)[:, None] for v in tmax)
            strict &= t + et < lim - elim
            lenient &= graze | (t - et < lim + elim)
    ts = np.where(strict, t, np.inf)
    best = np.argmin(ts, 1)
    r = np.arange(N)
    tb_, eb_ = t[r, best], et[r, best]
    others = lenient.copy()
    others[r, best] = False
    clear = ~np.any(others & ~(t - et > tb_[:, None] + eb_[:, None]), 1)
    hit = np.isfinite(ts[r, best]) & clear
    miss = ~lenient.any(1)
    kind = np.where(hit, 1, np.where(miss, 0, -1))
    bary = np.stack([b0[r, best], b1[r, best], b2[r, best]], 1)
    if want_strict:
        return kind, best, tb_, eb_, bary, np.isfinite(ts[r, best])
    return kind, best, tb_, eb_, bary


def closest_light(tb, O, D):
    """Float64 nearest light-sphere hit: (index or -1, t)."""
    best, tbest = np.full(len(O), -1), np.full(len(O), np.inf)
    for i, lt in enumerate(tb.lights):
        oc = O - lt["Position"].astype(np.float64)
        b = dot(D, oc)
        disc = b * b - (dot(oc, oc) - float(lt["Radius"]) ** 2)
        t1 = -b - np.sqrt(np.maximum(disc, 0.0))
        ok = (disc > 0) & (t1 > 0) & (t1 < tbest)
        best, tbest = np.where(ok, i, best), np.where(ok, t1, tbest)
    return best, tbest


# --------------------------------------------------------------------------------------------- the depth runs
def state_bits(rays):
    return np.ascontiguousarray(rays).view(np.uint32).reshape(len(rays), -1)


def depth_states(run, max_depth):
    """run(depth) -> (rays [W*H] GpuWavefrontRay, bounce_rays [depth]) of a fresh context. Runs depth 1 .. max_depth + 1 and
    checks the prefix property: the rays whose state run d + 1 changes against run d are exactly as many as bounce d
    shaded (its alive count), and every deeper run shaded that many at bounce d. Returns (states, alive): states[k] = every ray after bounces 0..k, alive[k] = rays that
    bounce k left alive (so bounce k + 1 shaded them)."""
    runs = [run(d) for d in range(1, max_depth + 2)]
    states = [r[0] for r in runs]
    alive = []
    for d in range(1, max_depth + 1):
        changed = np.any(state_bits(states[d - 1]) != state_bits(states[d]), 1)
        shaded = int(runs[d][1][d])
        # a ray with zero throughput that misses (radiance += 0) leaves its state as it was
        zero = np.all(states[d - 1]["Throughput"] == 0, 1)
        assert int(changed.sum()) <= shaded <= int((changed | zero).sum()), (d, int(changed.sum()), shaded)
        # bounce d's alive list is the prefix of the deeper runs': their first d bounces agree bit for bit
        for e in range(d + 1, len(runs)):
            assert int(runs[e][1][d]) == shaded, (d, e)
        alive.append(changed)
    return states, alive


# --------------------------------------------------------------------------------------------- one bounce, judged
class Judged:
    """Counters of what a transition check reached (the tests assert each case was met)."""

    def __init__(self):
        self.c = {}

    def add(self, name, n):
        self.c[name] = self.c.get(name, 0) + int(n)

    def __getitem__(self, name):
        return self.c.get(name, 0)


def _fail(mask, what, idx=None, **cols):
    if np.any(mask):
        k = np.nonzero(mask)[0][:5]
        info = {name: np.asarray(v)[k] for name, v in cols.items()}
        raise AssertionError("%s: %d rays violate the rule, e.g. rays %s %s" % (what, int(mask.sum()),
                                                                                 (idx[k] if idx is not None else k), info))


def judge_bounce(tb, O, D, thr, rad, ior, out, ended, first, rr, trace_lights=False, judged=None, idx=None):
    """Check one bounce of N paths. O, D: float64 incoming origins and unit directions; thr, rad (float32 [N, 3]), ior
    (float32 [N]) the incoming state; out: the GpuWavefrontRay after the bounce; ended: the path did not survive it.
    first: bounce 0 (FirstHit: prevIor from the surface); rr: Russian roulette on (applies at k >= 1 only).
    Returns (Judged, per-ray dict of what was decided)."""
    J = judged or Judged()
    N = len(O)
    idx = np.arange(N) if idx is None else idx
    kind, tri, t, et, bary = closest(tb, O, D)
    lt_i, lt_t = closest_light(tb, O, D) if trace_lights else (np.full(N, -1), np.full(N, np.inf))
    # a light sphere in front of (or ambiguously near) the triangle hit makes the triangle rules moot
    light_first = lt_i >= 0
    kind = np.where(light_first & (kind == 1) & (lt_t < t + et + 1e-4), -1, kind)
    kind = np.where(light_first & (kind == 0), -1, kind)
    ro, rt, rr_ = out["Origin"].astype(np.float64), out["Throughput"], out["Radiance"]
    dout = decode_dir(out["PackedDirectionX"], out["PackedDirectionY"])
    thr64, rad64 = thr.astype(np.float64), rad.astype(np.float64)

    # ---- 1. miss: the sky, and the path ends with origin, throughput and direction untouched
    miss = kind == 0
    col, _, clear = sky_lookup(D)
    mm = miss & clear
    want = rad64 + col * thr64
    bad = np.any(np.abs(rr_ - want) > 2 * ulp(want) + 1e-30, 1)
    _fail(mm & bad, "miss radiance != radiance + sky(dir) * throughput", idx, got=rr_, want=want)
    _fail(miss & ~ended, "a missing path survived", idx)
    _fail(miss & np.any(rt != thr, 1), "a miss changed the throughput", idx)
    J.add("miss", mm.sum())

    # ---- surfaces of the judged hits
    hit = kind == 1
    m = tb.mesh[tri]
    P = O + D * t[:, None]
    ng = tb.ng[tri]
    from_inside = dot(-D, ng) < 0.0
    n_in = np.where(from_inside[:, None], -ng, ng)                 # the geometric normal on the incoming side
    ns = unit(np.einsum("rk,rkc->rc", bary, tb.vn[tri]))           # interpolated vertex normal (no normal map)
    ns = np.where((dot(-D, ns) < 0.0)[:, None], -ns, ns)
    prev = np.where(first, np.where(from_inside, tb.ior32[m], F32(1.0)), ior).astype(F32)
    vol = tb.volumetric[m]
    absorb = from_inside & vol
    att = np.where(absorb[:, None], np.exp(-tb.absorbance[m] * np.where(absorb, t, 0.0)[:, None]), 1.0)
    thr_a = thr64 * att

    # ---- 2. emission
    want = rad64 + tb.emissive[m] * thr_a
    tol = 2 * ulp(np.maximum(np.abs(want), np.abs(rad64))) + 1e-30
    tol = np.where(absorb[:, None], tol + 8 * U32 * np.abs(tb.emissive[m] * thr_a), tol)
    bad = np.any(np.abs(rr_ - want) > tol, 1)
    _fail(hit & bad, "hit radiance != radiance + emissive * throughput", idx, got=rr_, want=want)
    J.add("hit", hit.sum())

    # ---- 3. origin: P + 0.001 n_g' (away from the incoming side on the transmission branch); RR leaves it at P
    off = dot(ro - P, n_in)
    trans = hit & ~ended & (off < 0.0)
    sgn = np.where(trans, -1.0, 1.0)
    tolp = et + 8 * U32 * (np.linalg.norm(O, axis=1) + np.abs(t) + 1.0)
    want_o = np.where(ended[:, None], P, P + (OFFSET * sgn)[:, None] * n_in)
    bad = np.linalg.norm(ro - want_o, axis=1) > tolp
    _fail(hit & bad, "origin != P + 0.001 n_g'", idx, got=ro, want=want_o, tol=tolp)

    # ---- 4./5. throughput: one rounding of thr * f, and q / max(q) under Russian roulette
    t_ = tb.transmission[m]
    f_trans = np.where(((vol | ~from_inside) & tb.tint[m])[:, None], tb.albedo32[m], F32(1.0))
    f = np.where(trans[:, None], f_trans, tb.albedo32[m]).astype(F32)
    _fail(trans & (t_ == 0.0), "transmission branch on a material without transmission", idx)
    q = (thr * f).astype(F32)
    if not rr or first:
        exact = hit & ~absorb
        _fail(exact & np.any(rt != q, 1), "throughput != float32(thr * f)", idx, got=rt, want=q)
        qa = thr_a * f
        # det_exp is good to a few ulp; its argument -a t carries the float32 rounding of a * t and the hit distance's error
        arg = tb.absorbance[m] * t[:, None]
        rel = 8 * U32 + 4 * U32 * arg + tb.absorbance[m] * et[:, None]
        _fail(hit & absorb & np.any(np.abs(rt - qa) > rel * qa + 1e-37, 1), "throughput != thr * exp(-a t) * f", idx,
              got=rt, want=qa)
        _fail(hit & ended & ~absorb, "a hit path ended without Russian roulette", idx)
        J.add("throughput_exact", exact.sum())
        J.add("absorbed", (hit & absorb).sum())
        J.add("absorbed_to_zero", (hit & absorb & np.all(rt == 0, 1) & np.any(thr != 0, 1)).sum())
    else:
        assert not np.any(hit & absorb), "the roulette checks run on opaque scenes"
        p = q.max(1)
        qp = (q / p[:, None]).astype(F32)
        _fail(hit & ~ended & np.any(rt != qp, 1), "throughput != q / max(q) after Russian roulette", idx, got=rt, want=qp)
        _fail(hit & ended & np.any(rt != q, 1), "a terminated path's throughput != thr * f", idx, got=rt, want=q)
        J.add("rr_survived", (hit & ~ended).sum())
        J.add("rr_terminated", (hit & ended).sum())

    # ---- 6./7. direction and prevIor
    iout = out["PreviousIOROrTraverseCost"]
    live = hit & ~ended
    c = dot(ns, D)                                                   # GLSL refract's dot(N, I)
    new_ior = np.where(from_inside, F32(1.0), tb.ior32[m]).astype(F32)
    eta = prev.astype(np.float64) / new_ior.astype(np.float64)
    k = 1.0 - eta * eta * (1.0 - c * c)
    near_critical = vol & (np.abs(k) < 1e-4)
    tir = vol & (k < 0.0)
    refr = eta[:, None] * D - (eta * c + np.sqrt(np.maximum(k, 0.0)))[:, None] * ns
    R = reflect(D, ns)
    r0 = tb.roughness[m] == 0.0
    mirror = live & ~trans & (np.linalg.norm(dout - R, axis=1) < 1e-5)
    diffuse = live & ~trans & ~mirror
    _fail(diffuse & (dot(dout, ns) < -1e-6), "a diffuse / mirror direction below the shading-normal hemisphere", idx)
    thin = trans & ~vol
    vt = trans & vol & ~near_critical
    want_t = np.where(thin[:, None], D, np.where(tir[:, None], R, refr))
    # near the critical angle Snell amplifies the float32 error of the incoming direction by ~ 1 / sqrt(k)
    tol_t = 1e-5 + np.where(vt & ~tir, 1e-6 / np.sqrt(np.maximum(np.abs(k), 1e-12)), 0.0)
    _fail(r0 & (thin | vt) & (np.linalg.norm(dout - want_t, axis=1) > tol_t), "transmission direction", idx, got=dout,
          want=want_t)
    want_i = np.where(trans, np.where(thin, F32(1.0), np.where(tir, prev, new_ior)), prev).astype(F32)
    _fail((live & ~near_critical) & (iout != want_i), "prevIor", idx, got=iout, want=want_i)
    J.add("mirror", (mirror & r0).sum())
    J.add("diffuse", diffuse.sum())
    J.add("thin", thin.sum())
    J.add("refract_in", (vt & ~tir & ~from_inside).sum())
    J.add("refract_out", (vt & ~tir & from_inside).sum())
    J.add("tir", (vt & tir).sum())
    J.add("from_inside", (hit & from_inside).sum())
    dec = dict(kind=kind, mesh=m, ns=ns, ng=n_in, P=P, D=D, prev=prev, mirror=mirror, trans=trans, diffuse=diffuse, live=live)
    return J, dec


# --------------------------------------------------------------------------------------------- bounce 0: the camera
def camera(frame):
    """(origin float64 [3], inv_proj [16], inv_view [16]) of GpuPerFrameData as the kernels read it (column-major)."""
    iv = frame["InvView"][0].astype(np.float64)
    return iv[12:15].copy(), frame["InvProjection"][0].astype(np.float64), iv


def camera_dirs(frame, sx, sy, width, height):
    """Float64 camera directions through image points (sx, sy) in pixels (lens radius 0)."""
    _, ip, iv = camera(frame)
    nx = np.asarray(sx, np.float64) / width * 2.0 - 1.0
    ny = np.asarray(sy, np.float64) / height * 2.0 - 1.0
    rx, ry = ip[0] * nx + ip[4] * ny, ip[1] * nx + ip[5] * ny
    d = np.stack([iv[0] * rx + iv[4] * ry - iv[8], iv[1] * rx + iv[5] * ry - iv[9], iv[2] * rx + iv[6] * ry - iv[10]], -1)
    return unit(d)


def first_hits(tb, frame, out, width, height):
    """Bounce 0 seen from its output: the hit point is the exported origin moved back onto the triangle plane it was
    offset from (0.001 along its normal, either side), the incoming direction runs from the camera to it. Returns
    (pixels, P, D): only pixels whose reconstructed ray hits that very triangle unambiguously at P, and whose P lies in
    the pixel's footprint (the float64 rays through its corners), are kept."""
    C = camera(frame)[0]
    O = out["Origin"].astype(np.float64)
    best_p = np.full((len(O), 3), np.nan)
    best_tri = np.full(len(O), -1)
    planes = np.zeros(len(O), np.int64)
    tol = 16 * U32 * (np.linalg.norm(O, axis=1) + 1.0)
    for j in range(len(tb.mesh)):
        dist = dot(O - tb.p[j, 0], tb.ng[j])
        on = np.abs(np.abs(dist) - OFFSET) < tol
        Pj = O - dist[:, None] * tb.ng[j]
        new_plane = on & ~((best_tri >= 0) & (np.abs(dot(tb.p[np.maximum(best_tri, 0), 0] - tb.p[j, 0], tb.ng[j])) < 1e-9)
                           & (np.abs(dot(tb.ng[np.maximum(best_tri, 0)], tb.ng[j])) > 1 - 1e-12))
        planes += new_plane
        take = on & (best_tri < 0)
        best_p[take], best_tri[take] = Pj[take], j
    pix = np.nonzero((best_tri >= 0) & (planes == 1))[0]      # an origin 0.001 from two planes (near an edge) is not judged
    P = best_p[pix]
    D = unit(P - C)
    kind, tri, t, et, _ = closest(tb, np.broadcast_to(C, P.shape), D)
    same_plane = (kind == 1) & (np.abs(dot(tb.p[tri, 0] - P, tb.ng[tri])) < 2e-5) & (np.abs(t - np.linalg.norm(P - C, axis=1)) < 1e-4)
    keep = same_plane
    return pix[keep], P[keep], D[keep]


def footprint_ok(tb, frame, pix, P, width, height, plane_y=0.0):
    """Rule 9: every P lies in the float64 footprint of its pixel on the plane y = plane_y (the rays through its corners)."""
    C = camera(frame)[0]
    x, y = pix % width, pix // width
    corners = []
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        d = camera_dirs(frame, x + dx, y + dy, width, height)
        tt = (plane_y - C[1]) / d[:, 1]
        corners.append(C + d * tt[:, None])
    corners = np.stack(corners, 1)
    lo, hi = corners.min(1) - 1e-5, corners.max(1) + 1e-5
    inside = np.all((P[:, [0, 2]] >= lo[:, [0, 2]]) & (P[:, [0, 2]] <= hi[:, [0, 2]]), 1)
    return inside


# --------------------------------------------------------------------------------------------- branch statistics
def branch_probabilities(tb, dec, sel):
    """Float64 P(mirror), P(transmission) of each selected judged hit at its own cos(theta) (Shading.glsl SampleMaterial:
    Schlick with pow 5, metallic -> mix(metallic, 1, F), transmission renormalised). The selection draws one rnd in
    [0, 1): mirror when M > rnd, transmission when M + T > rnd, so with metallic + transmission > 1 (a negative diffuse
    chance) M + T exceeds 1 and P(transmission) is 1 - M, not T."""
    m = dec["mesh"][sel]
    cos = dot(-dec["D"][sel], dec["ns"][sel])
    prev = dec["prev"][sel].astype(np.float64)
    ior = tb.ior[m]
    f0 = ((prev - ior) / (prev + ior)) ** 2
    F = f0 + (1.0 - f0) * (1.0 - cos) ** 5
    met, tr = tb.metallic[m], tb.transmission[m]
    dc = 1.0 - met - tr
    M = met + (1.0 - met) * F
    T = np.maximum(1.0 - dc - M, 0.0)
    pm = np.minimum(M, 1.0)
    pt = np.minimum(M + T, 1.0) - pm
    return pm, pt


def z_score(count, p):
    p = np.asarray(p, np.float64)
    var = np.sum(p * (1.0 - p))
    return (count - p.sum()) / np.sqrt(max(var, 1e-300)), p.sum(), np.sqrt(var)


# --------------------------------------------------------------------------------------------- the scenarios
# Every scenario takes make_run(scene, frame, width, height, sky, rr=, lights=, aovs=) -> run(depth) -> dict(rays,
# bounce, result, albedo, normal): the oracle on the CPU, PathTracer on the GPU. Each returns what it reached.
def judge_paths(tb, frame, states, alive, width, height, rr, trace_lights=False):
    """Every judged transition of the depth runs: bounce 0 from the camera (first_hits), bounce k >= 1 from S_k."""
    J = Judged()
    def known(sel, k):
        # a path left with zero throughput that then misses keeps its state bit for bit, so "not shaded by bounce k + 1"
        # does not tell whether it ended: such paths are not judged
        return sel[alive[k][sel] | np.any(states[k][sel]["Throughput"] != 0, 1)]
    pix, P, D = first_hits(tb, frame, states[0], width, height)
    keep = np.isin(pix, known(pix, 0))
    pix, P, D = pix[keep], P[keep], D[keep]
    C = camera(frame)[0]
    one = np.ones((len(pix), 3), F32)
    J, dec0 = judge_bounce(tb, np.broadcast_to(C, D.shape), D, one, np.zeros_like(one), np.ones(len(pix), F32), states[0][pix],
                           ~alive[0][pix], True, rr, trace_lights, J, pix)
    J.add("bounce0", (dec0["kind"] == 1).sum())
    for k in range(1, len(alive)):
        sel = known(np.nonzero(alive[k - 1])[0], k)
        s = states[k - 1][sel]
        O = s["Origin"].astype(np.float64)
        Dk = decode_dir(s["PackedDirectionX"], s["PackedDirectionY"])
        J, _ = judge_bounce(tb, O, Dk, s["Throughput"], s["Radiance"], s["PreviousIOROrTraverseCost"], states[k][sel],
                            ~alive[k][sel], False, rr, trace_lights, J, sel)
    return J, (pix, P, D, dec0)


def _frame(pos, view, w, h, fov):
    return scenes.camera_frame(dict(position=pos, view_dir=view, fov_y_deg=fov), w, h)


def glass_scene():
    """A diffuse floor, a clear volumetric glass cube above it, a dark one that absorbs everything (its Beer-Lambert
    factor flushes to 0), a thin untinted pane and a tinted thin pane; roughness 0 on every transmitting surface."""
    specs = [dict(color=(0.75, 0.7, 0.6), roughness=1.0),
             dict(color=(0.9, 0.95, 1.0), transmission=1.0, roughness=0.0, ior=1.5, volumetric=True, absorbance=(0.3, 0.1, 0.05)),
             dict(color=(0.8, 0.9, 0.7), transmission=1.0, roughness=0.0, ior=1.33, volumetric=True, absorbance=(250.0, 200.0, 300.0)),
             dict(color=(0.6, 0.8, 0.9), transmission=0.7, metallic=0.1, roughness=0.0, tint=False),
             dict(color=(0.9, 0.5, 0.4), transmission=0.6, roughness=0.0, emissive=(0.5, 0.25, 0.1))]
    parts = [(floor(), 0), (box_faces([-0.9, 0.4, -2.4], [0.3, 1.6, -1.2]), 1), (box_faces([0.6, 0.3, -2.2], [1.4, 1.1, -1.4]), 2),
             (scenes.quad([-1.6, 0.0, -0.6], [-0.6, 0.0, -0.6], [-0.6, 1.2, -0.9], [-1.6, 1.2, -0.9]), 3),
             (scenes.quad([1.4, 0.0, -0.4], [2.2, 0.0, -0.4], [2.2, 1.0, -0.7], [1.4, 1.0, -0.7]), 4)]
    return build(parts, specs), ((0.2, 1.5, 1.2), (-0.05, -0.45, -1.0), 60.0)


def check_glass(make_run, w, h, depth=5):
    scene, cam = glass_scene()
    tb = Tables(scene)
    frame = _frame(*cam[:2], w, h, cam[2])
    run = make_run(scene, frame, w, h, cube_sky(), rr=False)
    states, alive = depth_states(lambda d: _rays(run(d)), depth)
    J, _ = judge_paths(tb, frame, states, alive, w, h, rr=False)
    print("glass:", J.c)
    return J


def _rays(r):
    return r["rays"], r["bounce"]


def check_inside_glass(make_run, w, h):
    """The camera inside a glass cube: FirstHit starts from the surface's IOR, leaves through Snell with eta = IOR / 1
    (prevIor 1) or stays inside by TIR / reflection (prevIor = IOR), with Beer-Lambert over the first segment."""
    specs = [dict(color=(0.95, 0.9, 0.85), transmission=1.0, roughness=0.0, ior=1.5, volumetric=True, absorbance=(0.4, 0.2, 0.1))]
    scene = build([(box_faces([-1.0, -0.8, -1.3], [1.1, 0.9, 0.7]), 0)], specs)
    tb = Tables(scene)
    frame = _frame((0.05, 0.02, -0.1), (0.3, -0.2, -1.0), w, h, 100.0)
    run = make_run(scene, frame, w, h, cube_sky(), rr=False)
    states, alive = depth_states(lambda d: _rays(run(d)), 2)
    J, _ = judge_paths(tb, frame, states, alive, w, h, rr=False)
    print("inside glass:", J.c)
    return J


def box_scene(albedo=(0.8, 0.6, 0.4), emissive=(0.0, 0.0, 0.0), metallic=0.0, roughness=1.0, lamp=True):
    specs = [dict(color=albedo, emissive=emissive, metallic=metallic, roughness=roughness),
             dict(color=(1.0, 1.0, 1.0), emissive=(4.0, 3.5, 3.0), roughness=1.0)]
    parts = [(box_faces([-1.0, 0.0, -1.0], [1.0, 2.0, 1.0]), 0)]
    if lamp:
        parts.append((scenes.quad([-0.4, 1.99, -0.4], [0.4, 1.99, -0.4], [0.4, 1.99, 0.4], [-0.4, 1.99, 0.4]), 1))
    return build(parts, specs)


def check_roulette(make_run, w, h, depth=4):
    """Russian roulette (k >= 1): a path either ends with throughput thr * f or goes on with q / max(q)."""
    scene = box_scene()
    tb = Tables(scene)
    frame = _frame((0.1, 0.9, 0.7), (0.15, -0.1, -1.0), w, h, 80.0)
    run = make_run(scene, frame, w, h, (SENTINEL, SENTINEL, SENTINEL), rr=True)
    states, alive = depth_states(lambda d: _rays(run(d)), depth)
    J, _ = judge_paths(tb, frame, states, alive, w, h, rr=True)
    print("roulette:", J.c)
    return J


FLOOR_CAM = ((0.0, 1.0, 0.0), (0.0, -0.45, -1.0), 90.0)


def floor_run(make_run, spec, w, h, depth=1, biases=None, sky=None, cam=FLOOR_CAM, **opts):
    scene = build([(floor(), 0)], [spec], biases)
    tb = Tables(scene)
    frame = _frame(*cam[:2], w, h, cam[2])
    run = make_run(scene, frame, w, h, cube_sky() if sky is None else sky, **opts)
    runs = {}

    def cached(d):
        if d not in runs:
            runs[d] = run(d)
        return runs[d]
    states, alive = depth_states(lambda d: _rays(cached(d)), depth)
    return tb, frame, states, alive, runs


BRANCH_SPECS = [
    ("dielectric 1.5", dict(color=(0.8, 0.8, 0.8), roughness=0.0), None),
    ("dielectric 1.0", dict(color=(0.7, 0.75, 0.8), roughness=0.0), {0: dict(IORBias=-0.5)}),
    ("metal 0.4", dict(color=(0.9, 0.6, 0.3), metallic=0.4, roughness=0.0), None),
    ("m+t>1 tinted", dict(color=(0.6, 0.9, 0.5), metallic=0.5, transmission=0.8, roughness=0.0), None),
    ("thin untinted", dict(color=(0.5, 0.6, 0.9), metallic=0.2, transmission=0.5, roughness=0.0, tint=False), None),
    ("biased", dict(color=(0.9, 0.9, 0.9), metallic=0.9, transmission=0.1, roughness=0.5, ior=1.2),
     {0: dict(SpecularBias=-0.6, TransmissionBias=0.2, RoughnessBias=-0.5, IORBias=0.3)}),
]


def check_branches(make_run, w, h):
    """Branch counts on roughness-0 floors against the float64 Schlick Fresnel at each ray's own cos(theta)."""
    out = {}
    for name, spec, biases in BRANCH_SPECS:
        tb, frame, states, alive, _ = floor_run(make_run, spec, w, h, biases=biases, rr=False)
        J, (pix, P, D, dec) = judge_paths(tb, frame, states, alive, w, h, rr=False)
        sel = dec["kind"] == 1
        pm, pt = branch_probabilities(tb, dec, sel)
        zm, em, sm = z_score(dec["mirror"][sel].sum(), pm)
        zt, et_, st_ = z_score(dec["trans"][sel].sum(), pt)
        print("%-15s judged %6d  mirror %6d (exp %.1f +- %.1f, z %+.2f)  transmission %6d (exp %.1f +- %.1f, z %+.2f)" % (
            name, sel.sum(), dec["mirror"][sel].sum(), em, sm, zm, dec["trans"][sel].sum(), et_, st_, zt))
        inside = footprint_ok(tb, frame, pix[sel], P[sel], w, h)
        assert inside.all(), "%s: %d first hits outside their pixel's footprint" % (name, (~inside).sum())
        out[name] = dict(J=J, judged=int(sel.sum()), mirror=int(dec["mirror"][sel].sum()), trans=int(dec["trans"][sel].sum()),
                         zm=zm, zt=zt, em=em, et=et_, frame=frame, states=states, dec=dec)
    return out


def check_cosine(make_run, w, h):
    """A roughness-1 diffuse floor: the mirror lobe collapses onto the diffuse one, so every bounce-0 direction is a
    cosine sample about the shading normal: cos^2(theta) ~ U(0, 1) and the azimuth ~ U(0, 2 pi)."""
    from scipy import stats
    tb, frame, states, alive, _ = floor_run(make_run, dict(color=(0.6, 0.6, 0.6), roughness=1.0), w, h, rr=False)
    J, (pix, P, D, dec) = judge_paths(tb, frame, states, alive, w, h, rr=False)
    sel = dec["kind"] == 1
    s = states[0][pix[sel]]
    d = decode_dir(s["PackedDirectionX"], s["PackedDirectionY"])
    n = dec["ns"][sel]
    cos = dot(d, n)
    t = unit(np.cross(n, [0.0, 0.0, 1.0]))
    b = np.cross(n, t)
    phi = np.mod(np.arctan2(dot(d, b), dot(d, t)), 2.0 * np.pi)
    ks_c = stats.kstest(np.clip(cos, 0, 1) ** 2, "uniform")
    ks_p = stats.kstest(phi / (2.0 * np.pi), "uniform")
    print("cosine sampling: %d directions, cos^2 KS D=%.5f p=%.3g, azimuth KS D=%.5f p=%.3g" % (
        len(cos), ks_c.statistic, ks_c.pvalue, ks_p.statistic, ks_p.pvalue))
    footprint = footprint_ok(tb, frame, pix[sel], P[sel], w, h)
    return dict(n=len(cos), ks_c=ks_c, ks_p=ks_p, footprint=footprint, J=J)


def check_aovs(make_run, w, h):
    """First-hit AOVs: albedo * w and N_s * w with w = (1 - m - t) + m r + t r of the surface before the roughness remap;
    on a sky miss, the face colour and the face normal."""
    spec = dict(color=(0.8, 0.5, 0.3), metallic=0.3, roughness=0.6, transmission=0.2)
    tb, frame, states, alive, runs = floor_run(make_run, spec, w, h, rr=False, aovs=True)
    r = runs[1]
    pix, P, D = first_hits(tb, frame, states[0], w, h)
    _, dec = judge_bounce(tb, np.broadcast_to(camera(frame)[0], D.shape), D, np.ones((len(pix), 3), F32),
                          np.zeros((len(pix), 3), F32), np.ones(len(pix), F32), states[0][pix], ~alive[0][pix], True, False)
    sel = dec["kind"] == 1
    px = pix[sel]
    m = dec["mesh"][sel]
    wgt = (1.0 - tb.metallic[m] - tb.transmission[m]) + tb.metallic[m] * tb.roughness[m] + tb.transmission[m] * tb.roughness[m]
    alb = r["albedo"].reshape(-1, 4)
    nrm = r["normal"].reshape(-1, 4)
    want_a = tb.albedo[m] * wgt[:, None]
    want_n = dec["ns"][sel] * wgt[:, None]
    err_a = np.abs(alb[px, :3] - want_a).max()
    err_n = np.abs(nrm[px, :3] - want_n).max()
    # sky pixels: all four corner rays select the same face, clear of its edges
    rest = np.setdiff1d(np.arange(w * h), pix)
    x, y = rest % w, rest // w
    faces, clear = [], np.ones(len(rest), bool)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        d = camera_dirs(frame, x + dx, y + dy, w, h)
        _, f, c = sky_lookup(d)
        faces.append(f)
        clear &= c & (d[:, 1] > 0.05)
    faces = np.stack(faces, 1)
    sky = rest[clear & np.all(faces == faces[:, :1], 1)]
    f0 = faces[clear & np.all(faces == faces[:, :1], 1), 0]
    fn = face_normal(camera_dirs(frame, sky % w + 0.5, sky // w + 0.5, w, h))
    err_sa = np.abs(alb[sky, :3] - SKY_COLORS[f0]).max() if len(sky) else 0.0
    err_sn = np.abs(nrm[sky, :3] - fn).max() if len(sky) else 0.0
    print("AOVs: %d surface pixels (|err| albedo %.3g normal %.3g), %d sky pixels (|err| %.3g %.3g)" % (
        len(px), err_a, err_n, len(sky), err_sa, err_sn))
    return dict(n=len(px), n_sky=len(sky), err_a=err_a, err_n=err_n, err_sa=err_sa, err_sn=err_sn,
                alpha=np.concatenate([alb[:, 3], nrm[:, 3]]))


def check_lights(make_run, w, h):
    """DoTraceLights: a camera ray that hits a light sphere ends its first bounce with radiance = throughput = Color and
    its origin 0.001 outside the float64 sphere along the sphere normal."""
    color, radius, centre = (5.0, 4.0, 3.0), 0.35, (0.1, 0.7, -2.0)
    scene = build([(floor(), 0)], [dict(color=(0.5, 0.5, 0.5))], lights=[(centre, color, radius)])
    tb = Tables(scene)
    frame = _frame((0.0, 1.0, 0.0), (0.0, -0.3, -1.0), w, h, 70.0)
    run = make_run(scene, frame, w, h, cube_sky(), rr=False, lights=True)
    rays = run(1)["rays"]
    lt = tb.lights[0]
    c, R, col = lt["Position"].astype(np.float64), float(lt["Radius"]), lt["Color"]
    O = rays["Origin"].astype(np.float64)
    near = np.linalg.norm(O - c, axis=1) < R + 0.01
    lit = np.all(rays["Radiance"] == col, 1)
    P = c + (O - c) / (1.0 + OFFSET / R)
    C = camera(frame)[0]
    d = unit(P - C)
    li, lt_t = closest_light(tb, np.broadcast_to(C, P.shape), d)
    on_sphere = np.abs(np.linalg.norm(P - c, axis=1) - R) < 2e-5
    facing = dot(P - c, C - P) > 0
    first = (li == 0) & (np.abs(lt_t - np.linalg.norm(P - C, axis=1)) < 1e-4)
    ok = lit & np.all(rays["Throughput"] == col, 1) & on_sphere & facing & first
    print("light sphere: %d pixels near it, %d lit, %d satisfy every rule" % (near.sum(), lit.sum(), ok.sum()))
    return dict(near=near, lit=lit, ok=ok)


def furnace(make_run, w, h, depth, rr, metallic=0.0, roughness=1.0):
    """A closed box whose walls share emissive E and albedo a under a sentinel sky: a path that stays inside gathers
    E * sum_{k < D} a^k with Russian roulette off, and that in expectation with it on."""
    albedo, E = (0.7, 0.7, 0.7), (0.5, 0.4, 0.3)
    scene = box_scene(albedo=albedo, emissive=E, metallic=metallic, roughness=roughness, lamp=False)
    tb = Tables(scene)
    frame = _frame((0.1, 0.8, 0.5), (0.2, -0.1, -1.0), w, h, 90.0)
    r = make_run(scene, frame, w, h, (SENTINEL, SENTINEL, SENTINEL), rr=rr)(depth)
    a = tb.albedo[0]
    want = tb.emissive[0] * sum(a ** k for k in range(depth))
    res = r["result"][..., :3].reshape(-1, 3).astype(np.float64)
    leak = np.any(res > SENTINEL / 10.0, 1)
    return res, leak, want
