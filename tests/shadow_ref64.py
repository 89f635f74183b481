"""Float64 restatement of the ray-traced point-shadow pass, written from the engine's shaders (not from oracle/ or csrc/).

Paths are relative to the reference's IDKEngine (SHD = Resource/Shaders):
  SHD/ShadowsRayTraced/compute.glsl     depth == 1 returns (the image keeps its value); cosTheta = dot(normal,
                                        normalize(light - fragPos)) <= 0 stores 0; per sample: biased = fragPos + 0.01 normal,
                                        rnd0, rnd1 = InterleavedGradientNoise(imgCoord, noiseIndex + 0 / + 1), noiseIndex++,
                                        SampleSphere, then TraceRay(ray, hit, true, distanceToLight - 0.001) in a loop:
                                        another light's sphere -> 0, the light's own sphere -> break with the visibility kept;
                                        a triangle: blended (AlphaCutoff == 2) -> visibility *= 1 - alpha, else alpha > cutoff
                                        -> 0; visibility < 0.01 -> break (the product is kept); else the origin moves on by
                                        hit.T + 0.001 and distanceToLight drops by as much. visibility /= RayTracingSamples
  SHD/include/Sampling.glsl:21-52       SampleCone (ConstructBasis, Math.glsl:112-130) and SampleSphere. distanceToSphere =
                                        length(toSphere) cosTheta - sqrt(radius^2 - distance^2 sinTheta^2): in float32 the sqrt's
                                        argument cancels when the light is small and far, and can round below zero, where the
                                        engine's distance is NaN. This project clamps the argument at 0 (the distance to the
                                        sphere's tangent point); the float64 argument is never negative for a direction in the cone.
  SHD/include/Math.glsl:75-79           PerspectiveTransform(vec3(ndc.xy - Jitter, depth), InvProjView)
  SHD/include/Compression.glsl:63-73    DecodeUnitVec (pt_ref64.decode_dir)
  SHD/include/Random.glsl:35-41         InterleavedGradientNoise
  SHD/include/BVHIntersect.glsl:183-297 TraceRay: T = maxDist; every light in order: RaySphereIntersect (IntersectionRoutines.glsl:
                                        48-69, t1 <= t2 && t2 > 0) and tMin < T -> T = tMin < 0 ? tMax : tMin; then the triangles
                                        with a strict t < T (t >= 0, barycentrics >= 0); returns T != maxDist
  SHD/include/Surface.glsl:49-104       alpha = texture(BaseColor, uv).a * unpackUnorm4x8(BaseColorFactor).a (surface_ref64)

Float32 enters as data (depth, normal RG, the matrices, light and vertex records) and through the noise: the engine defines
InterleavedGradientNoise in float32 and the fract of a product with 52.98 magnifies any rounding, so `ign` evaluates it in
numpy float32 in the shader's order without FMA. Everything after the noise is float64.

Every sample is judged against margins that bound what float32 evaluation can move: the world position (the 4x4 product
and the divide), the sampled direction (the cone's sinTheta, det_sincos, the normalisations) times the distance travelled,
the sphere distance (the cancelling sqrt), each light sphere's silhouette and its tMin / tMax comparisons, triangle edges
(pt_ref64.closest's margins widened by the ray's displacement), hits near maxDist or the origin, the 0.001 step between
blended layers, an alpha near its cutoff (surface_ref64.envelope for textures), a visibility product near 0.01, and
|cosTheta|. A pixel is judged when all its samples are. With opaque occluders only, its value is float32(k) / float32(n)
exactly; with blended layers it lies within LAYER_ULP float32 ulps per layer of the float64 value."""
import numpy as np

import pt_ref64
import surface_ref64 as sr
from edge_lib import EPS, K, U32

F32 = np.float32
BIAS, STEP, STOP = 0.01, 0.001, 0.01
SAFETY = 2.0          # on the float32 error bounds of the sampled direction and distance
LAYER_ULP = 4         # float32 ulps a blended layer's 1 - alpha and product may add
MAX_STEPS = 32
REASONS = ("cos", "basis", "light", "edge", "alpha", "stop", "loop")


def ign(x, y, index):
    """InterleavedGradientNoise (Random.glsl:35-41) in float32, the shader's order, no FMA."""
    s = np.asarray(index, np.uint32).astype(F32) * F32(5.588238)
    x = np.asarray(x, F32) + s
    y = np.asarray(y, F32) + s
    a = F32(0.06711056) * x + F32(0.00583715) * y
    b = F32(52.9829189) * (a - np.floor(a))
    return b - np.floor(b)


def frag_positions(frame, depth, jitter):
    """PerspectiveTransform of every pixel centre -> (P [N, 3] float64, bound on the float32 evaluation's error [N])."""
    h, w = depth.shape
    m = np.asarray(frame["InvProjView"], np.float64).reshape(4, 4).T        # column-major -> rows
    ys, xs = np.mgrid[0:h, 0:w]
    jx, jy = (float(v) for v in np.asarray(jitter, F32))
    v = np.stack([(xs.ravel() + 0.5) / w * 2.0 - 1.0 - jx, (ys.ravel() + 0.5) / h * 2.0 - 1.0 - jy,
                  depth.ravel().astype(np.float64), np.ones(w * h)])
    q = m @ v
    enx, eny = 4 * U32 * (2.0 + abs(jx)), 4 * U32 * (2.0 + abs(jy))
    eq = 4 * U32 * (np.abs(m) @ np.abs(v)) + np.abs(m[:, :1]) * enx + np.abs(m[:, 1:2]) * eny
    with np.errstate(all="ignore"):
        P = (q[:3] / q[3]).T
        dP = (np.linalg.norm(eq[:3], axis=0) + np.linalg.norm(P, axis=1) * eq[3]) / np.abs(q[3]) + 2 * U32 * np.linalg.norm(P, axis=1)
    return P, dP


def sample_sphere(ts, radius, rnd0, rnd1, dO):
    """SampleSphere in float64 -> (direction, distanceToSphere, direction bound [rad], distance bound, basis flag).
    dO bounds the float32 origin's error, which tilts toSphere."""
    r2 = radius * radius
    d2 = np.einsum("nk,nk->n", ts, ts)
    d = np.sqrt(d2)
    cmax = np.sqrt(np.maximum(1.0 - r2 / d2, 0.0))
    a = np.maximum(rnd1, 0.001)
    cos = cmax * (1.0 - a) + a
    sin = np.sqrt(np.maximum(1.0 - cos * cos, 0.0))
    arg = r2 - d2 * sin * sin
    dist = d * cos - np.sqrt(np.maximum(arg, 0.0))
    N = ts / d[:, None]
    near_pole = np.abs(N[:, 2]) < 0.999
    up = np.where(near_pole[:, None], [0.0, 0.0, 1.0], [1.0, 0.0, 0.0])
    cr = np.cross(up, N)
    lcr = np.linalg.norm(cr, axis=1)
    T = cr / lcr[:, None]
    B = np.cross(N, T)
    phi = 2.0 * np.pi * rnd0
    D = T * (np.cos(phi) * sin)[:, None] + N * cos[:, None] + B * (np.sin(phi) * sin)[:, None]
    # float32: cosThetaMax and the mix round to a few ulp of 1; sinTheta = sqrt(1 - cos^2) turns that into e_s
    e_c = 8 * U32
    e2 = 2 * e_c + 4 * U32
    e_s = e2 / (sin + np.sqrt(e2))
    tilt = 2.0 * dO / d
    dD = SAFETY * (e_s + e_c + 16 * U32 * np.pi * sin + 16 * U32 / lcr + 8 * U32) + tilt
    e_arg = 8 * U32 * (r2 + d2 * sin * sin) + 2 * d2 * sin * e_s + d2 * e_s * e_s + 4 * d * dO * (sin + e_s) ** 2
    e_sqrt = e_arg / (np.sqrt(np.maximum(arg, 0.0)) + np.sqrt(e_arg))
    dM = SAFETY * (e_sqrt + d * e_c + 8 * U32 * d + 32 * U32 * d / lcr) + dO
    basis = np.abs(np.abs(N[:, 2]) - 0.999) <= 8 * U32 + tilt
    return D, dist, dD, dM, basis


def _closest(wt, O, D, T, eT, dO, dD, chunk=256):
    """pt_ref64.closest over wt in chunks -> (kind, tri, t, eps_t, barycentrics, any strict hit)."""
    n = len(O)
    if n == 0 or len(wt.mesh) == 0:
        return np.zeros(n, int), np.zeros(n, int), np.full(n, np.inf), np.zeros(n), np.zeros((n, 3)), np.zeros(n, bool)
    out = [pt_ref64.closest(wt, O[k:k + chunk], D[k:k + chunk], (T[k:k + chunk], eT[k:k + chunk]), (dO[k:k + chunk], dD[k:k + chunk]),
                            want_strict=True) for k in range(0, n, chunk)]
    return tuple(np.concatenate([o[i] for o in out]) for i in range(6))


class Scene64:
    """What the walk needs of a scene, computed once: world triangles, materials per triangle, light records, texels."""

    def __init__(self, scene):
        self.scene = scene
        self.wt = sr.WorldTriangles(scene)
        mat = scene.materials[scene.meshes["MaterialId"][self.wt.mesh]]
        self.cutoff = mat["AlphaCutoff"].astype(np.float64)
        self.textured = mat["BaseColorTexture"] != 0
        self.factor_alpha = sr.unorm8x4(mat["BaseColorFactor"])[:, 3]
        self.lights = scene.lights
        self.textures = [sr.texels(t) for t in scene.textures] if self.textured.any() else None
        # opaque: any hit on it gives 0, so which of two such triangles near a shared edge is the closest does not matter
        blend = self.cutoff == 2.0
        self.opaque = ~blend & ~self.textured & (self.factor_alpha - 4 * U32 > self.cutoff)
        self.layer_ids = np.nonzero(~self.opaque)[0]
        self.wt_opaque, self.wt_layers = self.wt.subset(self.opaque), self.wt.subset(~self.opaque)

    def hits(self, o, d, T, eT, do, dd):
        """The closest triangle before T -> (kind: 1 a hit on a non-opaque triangle, 2 an opaque hit, 0 none, -1 not
        judged; triangle index into wt, t, eps_t, barycentrics)."""
        kA, tA, tt, et, bary, _ = _closest(self.wt_layers, o, d, T, eT, do, dd)
        lim = np.where(kA == 1, tt, T)
        elim = np.where(kA == 1, et, eT)
        kB, _, tB, etB, _, sB = _closest(self.wt_opaque, o, d, lim, elim, do, dd)
        kind = np.where(kA == -1, -1, np.where(sB, 2, np.where(kB == 0, np.where(kA == 1, 1, 0), -1)))
        return kind, self.layer_ids[np.where(kA == 1, tA, 0)] if len(self.layer_ids) else np.zeros(len(o), int), tt, et, bary

    def alpha(self, tri, bary, O, D, t, dO, dD):
        """(lo, hi) of the alpha at the hits: the factor's, or surface_ref64's envelope over the barycentric error."""
        lo, hi = self.factor_alpha[tri].copy(), self.factor_alpha[tri].copy()
        tx = self.textured[tri]
        if tx.any():
            k = np.nonzero(tx)[0]
            wt = self.wt
            n = wt.n[tri[k]]
            lmax = np.max(np.linalg.norm(np.stack([wt.e1[tri[k]], wt.e2[tri[k]], wt.p[tri[k], 2] - wt.p[tri[k], 1]], 1), axis=2), 1)
            db = wt.bary_error(tri[k], O[k], D[k], t[k]) + (dO[k] + dD[k] * t[k]) * lmax / np.abs(np.einsum("nk,nk->n", D[k], n))

            def fn(b):
                uv = np.einsum("nk,nkc->nc", b, wt.uv[tri[k]]).astype(F32)
                return {"alpha": sr.surface(self.scene, wt.mesh[tri[k]], uv, self.textures)["alpha"]}
            rng = sr.envelope(fn, bary[k], db)["alpha"]
            lo[k], hi[k] = rng
        return lo, hi


def trace(s64, light_index, O, D, dl, dO, dD, dM):
    """The per-sample loop of compute.glsl for rays (O, D) with distanceToLight dl -> (visibility, blended layers, reason
    index or -1). dO, dD, dM: the float32 bounds on origin, direction and maxDist."""
    n = len(O)
    O, dl, dO, dM = O.copy(), dl.copy(), dO.copy(), dM.copy()
    vis = np.ones(n)
    layers = np.zeros(n, np.int64)
    reason = np.full(n, -1)
    active = np.ones(n, bool)
    for _ in range(MAX_STEPS):
        idx = np.nonzero(active)[0]
        if len(idx) == 0:
            break
        o, d, do, dd = O[idx], D[idx], dO[idx], dD[idx]
        maxd = dl[idx] - STEP
        T, eT = maxd.copy(), dM[idx].copy()
        which = np.full(len(idx), -1)
        unsure_light = np.zeros(len(idx), bool)
        for i, lt in enumerate(s64.lights):
            oc = o - lt["Position"].astype(np.float64)
            r = float(lt["Radius"])
            b = np.einsum("nk,nk->n", d, oc)
            oc2 = np.einsum("nk,nk->n", oc, oc)
            disc = b * b - (oc2 - r * r)
            dp = do + np.abs(b) * dd
            p = np.sqrt(np.maximum(oc2 - b * b, 0.0))
            e_disc = 16 * U32 * (b * b + oc2 + r * r) + 2 * (p + dp) * dp
            sq = np.sqrt(np.maximum(disc, 0.0))
            e_sq = e_disc / (sq + np.sqrt(e_disc))
            t1, t2 = -b - sq, -b + sq
            e_t = e_sq + 8 * U32 * (np.abs(b) + np.sqrt(oc2)) + dp
            hit = (disc >= 0.0) & (t2 > 0.0)
            acc = hit & (t1 < T)
            Tn = np.where(t1 < 0.0, t2, t1)
            unsure = (np.abs(disc) <= e_disc) | (np.abs(t2) <= e_t) | (np.abs(t1 - T) <= e_t + eT) | (np.abs(t1) <= e_t)
            unsure &= disc >= -e_disc
            if i == light_index:
                # the light's own sphere ends the walk with the visibility kept, as a miss does: an unsure test only widens
                # the limit the triangles are held to
                lo = np.where(unsure, np.minimum(T - eT, Tn - e_t), np.where(acc, Tn - e_t, T - eT))
                hi = np.where(unsure, np.maximum(T + eT, Tn + e_t), np.where(acc, Tn + e_t, T + eT))
                T, eT = (lo + hi) / 2, (hi - lo) / 2
                which = np.where(acc | unsure, i, which)
            else:
                unsure_light |= unsure
                T, eT = np.where(acc, Tn, T), np.where(acc, e_t, eT)
                which = np.where(acc, i, which)
        kind, tri, t, et, bary = s64.hits(o, d, T, eT, do, dd)
        rs = np.full(len(idx), -1)
        rs[kind == -1] = REASONS.index("edge")
        rs[unsure_light] = REASONS.index("light")
        done = rs >= 0
        vis[idx[(kind == 2) & ~done]] = 0.0
        done |= kind == 2
        miss = (kind == 0) & ~done
        vis[idx[miss & (which >= 0) & (which != light_index)]] = 0.0
        done |= miss
        hit = (kind == 1) & ~done
        k = np.nonzero(hit)[0]
        if len(k):
            tk = tri[k]
            alo, ahi = s64.alpha(tk, bary[k], o[k], d[k], t[k], do[k], dd[k])
            cut = s64.cutoff[tk]
            blend = cut == 2.0
            m = 4 * U32 * np.maximum(np.abs(cut), ahi)
            occl, clear = alo - m > cut, ahi + m <= cut
            ra = np.where((~blend & ~occl & ~clear) | (blend & (ahi - alo > 4 * U32)), REASONS.index("alpha"), -1)
            g = idx[k]
            vis[g[~blend & occl]] = 0.0
            vis[g[blend]] *= 1.0 - (alo[blend] + ahi[blend]) / 2
            layers[g[blend]] += 1
            v = vis[g]
            rs_stop = np.abs(v - STOP) <= 2 * LAYER_ULP * U32 * np.maximum(layers[g], 1) * v
            ra = np.where((ra < 0) & blend & rs_stop, REASONS.index("stop"), ra)
            rs[k] = np.where(ra >= 0, ra, rs[k])
            stop = (v < STOP) | (~blend & occl)
            done[k] |= (ra >= 0) | stop
            go = k[(ra < 0) & ~stop]
            if len(go):
                dist = t[go] + STEP
                gg = idx[go]
                O[gg] = O[gg] + D[gg] * dist[:, None]
                dl[gg] -= dist
                # dD and the old dO already move the hit point; the float32 t adds edge_lib's own error (et without the spread)
                et0 = EPS * dist + K * U32 * (np.linalg.norm(O[gg], axis=1) + dist)
                dO[gg] += dist * dD[gg] + et0
                dM[gg] += et0 + 4 * U32 * (np.abs(dl[gg]) + dist)
        reason[idx[rs >= 0]] = rs[rs >= 0]
        active[idx[done]] = False
    reason[active] = REASONS.index("loop")
    return vis, layers, reason


def shadows_ref(s64, frame, depth, normal_rg, light_index, samples=1, noise_index=0, jitter=(0.0, 0.0)):
    """The pass over one G-buffer -> dict(want float64 [H, W], tol [H, W] (0: the float32 value must equal float32(k) /
    float32(n)), judged [H, W], lit [H, W] (depth != 1), blended [H, W], counts {reason: unjudged pixels})."""
    h, w = depth.shape
    lit = depth.ravel() != 1.0
    pix = np.nonzero(lit)[0]
    lt = s64.lights[light_index]
    L, r = lt["Position"].astype(np.float64), float(lt["Radius"])
    P, dP = frag_positions(frame, depth, jitter)
    P, dP = P[pix], dP[pix]
    nrg = np.asarray(normal_rg, F32).reshape(-1, 2)[pix]
    nrm = pt_ref64.decode_dir(nrg[:, 0], nrg[:, 1])
    toL = L - P
    lL = np.linalg.norm(toL, axis=1)
    cos = np.einsum("nk,nk->n", nrm, toL) / lL
    cos_unsure = np.abs(cos) <= 16 * U32 + 2 * dP / lL
    facing = (cos > 0.0) & ~cos_unsure
    fp = np.nonzero(facing)[0]
    biased = P[fp] + BIAS * nrm[fp]
    dO0 = dP[fp] + 4 * U32 * (np.linalg.norm(P[fp], axis=1) + BIAS)
    S = samples
    xs, ys = (pix[fp] % w).astype(F32), (pix[fp] // w).astype(F32)
    rep = lambda a: np.repeat(a, S, axis=0)
    k = np.tile(np.arange(S, dtype=np.uint64), len(fp))
    base = (np.uint64(noise_index) + k) & np.uint64(0xFFFFFFFF)
    rnd0 = ign(rep(xs), rep(ys), base).astype(np.float64)
    rnd1 = ign(rep(xs), rep(ys), (base + np.uint64(1)) & np.uint64(0xFFFFFFFF)).astype(np.float64)
    O, dO = rep(biased), rep(dO0)
    D, dist, dD, dM, basis = sample_sphere(L - O, r, rnd0, rnd1, dO)
    vis, layers, reason = trace(s64, light_index, O, D, dist, dO, dD, dM)
    reason = np.where(basis, REASONS.index("basis"), reason)
    vis, layers, reason = (a.reshape(len(fp), S) for a in (vis, layers, reason))
    # each unjudged pixel counted once, under its first reason
    pr = np.full(len(pix), -1)
    pr[cos_unsure] = REASONS.index("cos")
    bad = np.where(reason >= 0, reason, len(REASONS))
    pr[fp] = np.where(bad.min(1) < len(REASONS), bad.min(1), -1)
    want = np.zeros(len(pix))
    tol = np.zeros(len(pix))
    blended = np.zeros(len(pix), bool)
    want[fp] = vis.sum(1) / S
    blended[fp] = layers.max(1) > 0
    opaque = ~blended
    want[opaque] = (np.round(want[opaque] * S).astype(F32) / F32(S)).astype(np.float64)     # float32(k) / float32(n)
    tol[fp] = (np.sum(vis * (LAYER_ULP * U32 * layers + S * U32), 1) / S + U32 * want[fp]) * blended[fp]
    out = dict(want=np.zeros(h * w), tol=np.zeros(h * w), judged=np.zeros(h * w, bool), lit=lit.reshape(h, w),
               blended=np.zeros(h * w, bool))
    out["want"][pix], out["tol"][pix], out["blended"][pix] = want, tol, blended
    out["judged"][pix] = pr < 0
    for key in ("want", "tol", "judged", "blended"):
        out[key] = out[key].reshape(h, w)
    out["counts"] = {name: int((pr == i).sum()) for i, name in enumerate(REASONS) if (pr == i).any()}
    out["facing_away"] = int(((cos <= 0.0) & ~cos_unsure).sum())
    return out


def check(got, ref, tag, min_share):
    """got (the oracle's or the device's float32 image) against ref at the judged pixels; asserts the judged share of the lit
    pixels is at least min_share. Returns (judged, lit)."""
    g = np.asarray(got, F32)
    j = ref["judged"]
    exact = j & ~ref["blended"]
    want32 = ref["want"].astype(F32)
    bad = exact & (g.view(np.uint32) != want32.view(np.uint32))
    assert not bad.any(), (tag, "opaque", int(bad.sum()), np.argwhere(bad)[:5].tolist(), g[bad][:5], ref["want"][bad][:5])
    lay = j & ref["blended"]
    dev = np.abs(g.astype(np.float64) - ref["want"])
    bad = lay & (dev > ref["tol"])
    assert not bad.any(), (tag, "blended", int(bad.sum()), np.argwhere(bad)[:5].tolist(), g[bad][:5], ref["want"][bad][:5])
    n_lit, n_j = int(ref["lit"].sum()), int(j.sum())
    print("%s: judged %d of %d lit pixels (%.1f%%), %d blended, %d facing away; unjudged by reason %s" % (
        tag, n_j, n_lit, 100.0 * n_j / max(n_lit, 1), int(lay.sum()), ref["facing_away"], ref["counts"]))
    assert n_j >= min_share * n_lit, (tag, n_j, n_lit)
    return n_j, n_lit
