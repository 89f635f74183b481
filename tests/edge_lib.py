"""Edge-case rays and an independent float64 closest-hit reference for the traversal tests (tests/test_edges*.py).

edge_rays(scene, seed)      deterministic battery of legal edge inputs built from the scene's own data: axis-parallel and
                            in-plane rays (+0.0 and -0.0), origins on BLAS / TLAS node planes, rays aimed at vertices and
                            edge midpoints, rays in a wall's plane, origins on a surface, boundary TMax values, denormal
                            direction components, unnormalised directions and far origins. No NaN inputs.
ref64_closest(scene, rays)  the same query in numpy float64 from the definitions (world-space source triangles, every
                            triangle tested), as a strict and a lenient hit set per ray.
classify(...)               applies the float64 rules to a closest-hit or any-hit result (oracle or GPU).

Tolerances. A triangle is in a ray's *strict* set when every barycentric is >= +eps_b and eps_t <= t, t + eps_t < TMax; in
its *lenient* set when every barycentric is >= -eps_b, t >= -eps_t and t - eps_t < TMax. Both follow a forward error bound
of the float32 intersector (ray transform, rop0 = o - p0, q = cross(rop0, d), two dot products and a divide, each rounding
by at most u = 2^-24):

    eps_b = 1e-5 + K u kappa (1 + S / min(|e1|, |e2|)),   kappa = |d| |e1| |e2| / |dot(d, n)|
    eps_t = 1e-5 |t| + K u |e1| |e2| S / |dot(d, n)|,     S = |o - p0| + |o| + |p0|,  K = 64

1e-5 (about 170 float32 ulps of a unit barycentric) is a floor that float32 rounding cannot cross for a well-conditioned
hit; the K u terms widen it for grazing rays (kappa) and for origins far from the triangle (S). A ray parallel to a
triangle (kappa > 1e6) never enters the strict set; it is lenient when its origin lies in the triangle's plane.
The closest-hit distance may deviate from the exact one by the same eps_t (the 'delta' of the rules).
"""
import numpy as np

import oracle_lib as ol
from idkengine_b200 import gpu_types as gt

MISS = 0xFFFFFFFF
U32 = 2.0 ** -24
K = 64.0
EPS = 1e-5
GRAZE_KAPPA = 1e6
F32 = np.float32


# --------------------------------------------------------------------------------------------- scene geometry
def _rows(mt):
    return np.asarray(mt, np.float32).reshape(3, 4)


def world_triangles(scene):
    """Source triangles of every instance in world space (float64), presplit fragments folded back onto their source.
    Returns dict(p0, e1, e2, n, frag2src [len(blas_triangles)], inst [M], mtid [M], pos32 [M,3,3] float32 world vertices)."""
    P = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float64)
    blas_ids = scene.blas_instances["BlasId"]
    assert len(np.unique(blas_ids)) == len(blas_ids), "one instance per BLAS expected"
    frag2src = np.full(len(scene.blas_triangles), -1, np.int64)
    p0s, p1s, p2s, inst, mtid = [], [], [], [], []
    base = 0
    for i, ins in enumerate(scene.blas_instances):
        d = scene.blas_descs[ins["BlasId"]]
        a, b = int(d["TriangleOffset"]), int(d["TriangleOffset"] + d["TriangleCount"])
        tri = scene.blas_triangles[a:b]
        xyz = np.stack([tri["X"], tri["Y"], tri["Z"]], 1).astype(np.int64)
        uniq, inv = np.unique(xyz, axis=0, return_inverse=True)
        frag2src[a:b] = base + inv.reshape(-1)
        m = _rows(scene.mesh_transforms[ins["MeshTransformId"]]["ModelMatrix"]).astype(np.float64)
        for k, lst in enumerate((p0s, p1s, p2s)):
            lst.append(P[uniq[:, k]] @ m[:, :3].T + m[:, 3])
        inst.append(np.full(len(uniq), i))
        mtid.append(np.full(len(uniq), ins["MeshTransformId"]))
        base += len(uniq)
    p0, p1, p2 = (np.concatenate(x) for x in (p0s, p1s, p2s))
    e1, e2 = p1 - p0, p2 - p0
    return dict(p0=p0, e1=e1, e2=e2, n=np.cross(e1, e2), frag2src=frag2src, inst=np.concatenate(inst),
                mtid=np.concatenate(mtid), pos32=np.stack([p0, p1, p2], 1).astype(np.float32))


def _node_planes(scene):
    """Per instance: the float32 Min/Max values of all its BLAS nodes, per axis (the slab planes of the local-space test)."""
    out = []
    for ins in scene.blas_instances:
        d = scene.blas_descs[ins["BlasId"]]
        nodes = scene.blas_nodes[int(d["NodeOffset"]):int(d["NodeOffset"] + d["NodeCount"])]
        out.append([np.unique(np.concatenate([nodes["Min"][:, a], nodes["Max"][:, a]]).astype(np.float32)) for a in range(3)])
    return out


def local_rays32(scene, rays, inst_index):
    """RayTransform of the oracle / xform_point and xform_vector of the kernels, in the same float32 order."""
    ins = scene.blas_instances[inst_index]
    r = _rows(scene.mesh_transforms[ins["MeshTransformId"]]["InvModelMatrix"])
    o, d = rays["Origin"].astype(F32), rays["Direction"].astype(F32)
    with np.errstate(all="ignore"):
        lo = np.stack([((r[k, 0] * o[:, 0] + r[k, 1] * o[:, 1]) + r[k, 2] * o[:, 2]) + r[k, 3] for k in range(3)], 1)
        ld = np.stack([(r[k, 0] * d[:, 0] + r[k, 1] * d[:, 1]) + r[k, 2] * d[:, 2] for k in range(3)], 1)
    return lo.astype(F32), ld.astype(F32)


def artefact_class(scene, rays):
    """Rays with an exactly-zero direction component whose origin lies on a node plane on that axis: in a BLAS walk (local
    space, float32 transform) or in the TLAS walk (world space). Their slab test evaluates 0 * inf = NaN."""
    flag = np.zeros(len(rays), bool)
    for i, planes in enumerate(_node_planes(scene)):
        lo, ld = local_rays32(scene, rays, i)
        for a in range(3):
            flag |= (ld[:, a] == 0) & np.isin(lo[:, a], planes[a])
    if scene.use_tlas and len(scene.tlas_nodes):
        o, d = rays["Origin"].astype(F32), rays["Direction"].astype(F32)
        for a in range(3):
            planes = np.unique(np.concatenate([scene.tlas_nodes["Min"][:, a], scene.tlas_nodes["Max"][:, a]]).astype(F32))
            flag |= (d[:, a] == 0) & np.isin(o[:, a], planes)
    return flag


# --------------------------------------------------------------------------------------------- float64 reference
class Ref64:
    """Per ray: strict / lenient membership (as flat (ray, element) pairs), nearest strict t, nearest lenient t, and rays that
    the rules cannot judge (origin in or on a light sphere, light test with a non-unit direction). Element ids 0..M-1 are
    source triangles, M + i is light sphere i."""


def ref64_closest(scene, rays, trace_lights=False, chunk=96, tris=None):
    W = tris or world_triangles(scene)
    p0, e1, e2, n = W["p0"], W["e1"], W["e2"], W["n"]
    M = len(p0)
    l1, l2 = np.linalg.norm(e1, axis=1), np.linalg.norm(e2, axis=1)
    lmin, area2 = np.minimum(l1, l2), l1 * l2
    np0 = np.linalg.norm(p0, axis=1)
    O = rays["Origin"].astype(np.float64)
    D = rays["Direction"].astype(np.float64)
    TM = rays["TMax"].astype(np.float64)
    N = len(rays)
    dn = np.linalg.norm(D, axis=1)
    on = np.linalg.norm(O, axis=1)
    strict_t = np.full(N, np.inf)
    lenient_t = np.full(N, np.inf)
    pairs_l, pairs_s = [], []
    valid = area2 > 0
    for a in range(0, N, chunk):
        b = min(N, a + chunk)
        o, d, tm = O[a:b, None, :], D[a:b, None, :], TM[a:b, None]
        rop0 = o - p0[None]
        det = np.einsum("rk,mk->rm", D[a:b], n)
        q = np.cross(rop0, d)
        with np.errstate(all="ignore"):
            inv = 1.0 / det
            b1 = -np.einsum("rmk,mk->rm", q, e2) * inv
            b2 = np.einsum("rmk,mk->rm", q, e1) * inv
            b0 = 1.0 - b1 - b2
            t = -np.einsum("mk,rmk->rm", n, rop0) * inv
            kappa = dn[a:b, None] * area2[None] / np.abs(det)
            S = np.linalg.norm(rop0, axis=2) + on[a:b, None] + np0[None]
            eb = EPS + K * U32 * kappa * (1.0 + S / lmin[None])
            et = EPS * np.abs(t) + K * U32 * area2[None] * S / np.abs(det)
            bmin = np.minimum(np.minimum(b0, b1), b2)
            graze = ~(kappa <= GRAZE_KAPPA)
            strict = ~graze & (bmin >= eb) & (t >= et) & (t + et < tm) & valid[None]
            dist = np.abs(np.einsum("mk,rmk->rm", n, rop0)) / np.linalg.norm(n, axis=1)[None]
            in_plane = graze & (dist <= EPS * lmin[None] + K * U32 * S) & valid[None]
            lenient = (~graze & (bmin >= -eb) & (t >= -et) & (t - et < tm) & valid[None]) | in_plane
            strict_t[a:b] = np.min(np.where(strict, t + et, np.inf), axis=1)
            # a parallel triangle in the ray's plane has no defined t: it lifts the lower bound
            lenient_t[a:b] = np.min(np.where(in_plane, -np.inf, np.where(lenient, t - et, np.inf)), axis=1)
        r, m = np.nonzero(lenient)
        pairs_l.append((r + a) * (M + 64) + m)
        r, m = np.nonzero(strict)
        pairs_s.append((r + a) * (M + 64) + m)
    unjudged = np.zeros(N, bool)
    if trace_lights and len(scene.lights):
        assert len(scene.lights) < 64
        for i, lt in enumerate(scene.lights):
            c, rad = lt["Position"].astype(np.float64), float(lt["Radius"])
            oc = O - c
            bb = np.einsum("rk,rk->r", D, oc)
            cc = np.einsum("rk,rk->r", oc, oc) - rad * rad
            disc = bb * bb - cc
            tol = K * U32 * (np.einsum("rk,rk->r", oc, oc) + rad * rad + 1.0)
            unjudged |= (cc <= tol) | (np.abs(dn - 1.0) > 1e-6)
            sq = np.sqrt(np.maximum(disc, 0.0))
            t1, t2 = -bb - sq, -bb + sq
            et = EPS * np.abs(t1) + K * U32 * (np.sqrt(np.abs(cc)) + rad + 1.0) + np.sqrt(np.maximum(tol, 0.0))
            strict = (disc > tol) & (t1 >= et) & (t1 + et < TM)
            lenient = (disc >= -tol) & (t1 - et < TM) & (t2 + et > 0)
            strict_t = np.where(strict, np.minimum(strict_t, t1 + et), strict_t)
            lenient_t = np.where(lenient, np.minimum(lenient_t, t1 - et), lenient_t)
            pairs_l.append(np.nonzero(lenient)[0] * (M + 64) + M + i)
            pairs_s.append(np.nonzero(strict)[0] * (M + 64) + M + i)
    ref = Ref64()
    ref.M, ref.stride, ref.tris = M, M + 64, W
    ref.lenient_pairs = np.unique(np.concatenate(pairs_l))
    strict_pairs = np.unique(np.concatenate(pairs_s))
    ref.strict_any = np.zeros(N, bool)
    ref.strict_any[strict_pairs // ref.stride] = True
    ref.lenient_any = np.zeros(N, bool)
    ref.lenient_any[ref.lenient_pairs // ref.stride] = True
    ref.strict_t, ref.lenient_t, ref.unjudged = strict_t, lenient_t, unjudged
    return ref


def classify(scene, rays, hits, ref, any_hit=False):
    """The float64 rules for one result (oracle or GPU). Returns dict with the index arrays robust_hit, robust_miss,
    artefact, bad (robust disagreements outside the artefact class) and culled (artefact-class robust hits reported as misses
    or farther than the nearest strict hit)."""
    N = len(rays)
    tid = hits["TriangleId"].astype(np.int64)
    T = hits["T"].astype(np.float64)
    tmax = rays["TMax"].astype(np.float64)
    tri_hit = tid != MISS
    light_hit = ~tri_hit & (hits["T"] != rays["TMax"])
    elem = np.full(N, -1, np.int64)
    elem[tri_hit] = ref.tris["frag2src"][tid[tri_hit]]
    elem[light_hit] = ref.M + hits["MeshTransformId"][light_hit].astype(np.int64)
    in_lenient = np.isin(np.arange(N) * ref.stride + elem, ref.lenient_pairs) & (elem >= 0)
    reported = hits["NodePairFetches"] == 1 if any_hit else (tri_hit | light_hit)
    art = artefact_class(scene, rays)
    judged = ~ref.unjudged
    rh = ref.strict_any & judged
    rm = ~ref.lenient_any & judged
    if any_hit:
        ok_hit = reported & in_lenient & (T >= ref.lenient_t) & (T < tmax)
    else:
        ok_hit = reported & in_lenient & (T >= ref.lenient_t) & (T <= ref.strict_t)
    ok_miss = ~reported & ~tri_hit & (hits["T"] == rays["TMax"])
    bad = (rh & ~ok_hit) | (rm & ~ok_miss)
    return dict(robust_hit=np.nonzero(rh)[0], robust_miss=np.nonzero(rm)[0], artefact=np.nonzero(art)[0],
                bad=np.nonzero(bad & ~art)[0], culled=np.nonzero(art & rh & ~ok_hit)[0])


# --------------------------------------------------------------------------------------------- the battery
def _unit(v):
    v = np.asarray(v, np.float64)
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(F32)


def _fix_local_plane(scene, inst_index, o32, axis, value):
    """Nudge world component `axis` of each origin by a few ulps until the float32 local transform lands exactly on `value`
    (possible when the inverse transform keeps that axis separate, e.g. scale + translation)."""
    out = o32.copy()
    for k in range(len(out)):
        best = out[k, axis]
        for step in range(-3, 4):
            cand = out[k].copy()
            cand[axis] = best
            for _ in range(abs(step)):
                cand[axis] = np.nextafter(cand[axis], F32(np.inf) if step > 0 else F32(-np.inf))
            r = np.zeros(1, gt.IdkPtRay)
            r["Origin"], r["Direction"] = cand, (1, 1, 1)
            lo, _ = local_rays32(scene, r, inst_index)
            if lo[0, axis] == value[k]:
                out[k] = cand
                break
    return out


def edge_rays(scene, seed, tris=None):
    """Deterministic edge battery for `scene` (IdkPtRay array, TMax = FLT_MAX unless the kind sets it)."""
    rng = np.random.RandomState(seed)
    W = tris or world_triangles(scene)
    pos = W["pos32"]
    lo_b, hi_b = pos.reshape(-1, 3).min(0).astype(np.float64), pos.reshape(-1, 3).max(0).astype(np.float64)
    ctr, ext = (lo_b + hi_b) * 0.5, (hi_b - lo_b) * 0.5
    area = np.linalg.norm(W["n"], axis=1)
    big = np.argsort(-area, kind="stable")[:24]                     # walls, floors, quads: the shared edges and diagonals
    pick = np.concatenate([big, rng.choice(len(pos), min(len(pos), 40), replace=False)])
    O, D, TM = [], [], []

    def add(o, d, tmax=np.float32(3.4028235e38)):
        o, d = np.asarray(o, F32).reshape(-1, 3), np.asarray(d, F32).reshape(-1, 3)
        m = max(len(o), len(d))
        O.append(np.broadcast_to(o, (m, 3)))
        D.append(np.broadcast_to(d, (m, 3)))
        TM.append(np.broadcast_to(np.asarray(tmax, F32).reshape(-1), (m,)))

    inner = (ctr + ext * rng.uniform(-0.9, 0.9, (40, 3))).astype(F32)
    # 1. axis-parallel, with +0.0 and -0.0 in the zero components
    for s in (1.0, -1.0):
        for a in range(3):
            for zs in (0.0, -0.0):
                d = np.full(3, zs, F32)
                d[a] = s
                add(inner, d)
    # 2. exactly one zero component (either sign)
    for a in range(3):
        d = rng.normal(size=(60, 3)).astype(F32)
        d[:, a] = np.where(rng.rand(60) < 0.5, F32(0.0), F32(-0.0))
        add(inner[rng.randint(0, len(inner), 60)], _unit(d))
    # 3. origins on BLAS node planes (local space, made exact where the transform allows) and on TLAS node planes
    for i, ins in enumerate(scene.blas_instances):
        d_ = scene.blas_descs[ins["BlasId"]]
        nodes = scene.blas_nodes[int(d_["NodeOffset"]) + 1:int(d_["NodeOffset"] + d_["NodeCount"])]
        m = _rows(scene.mesh_transforms[ins["MeshTransformId"]]["ModelMatrix"]).astype(np.float64)
        sel = nodes[rng.choice(len(nodes), min(len(nodes), 40), replace=False)]
        for a in range(3):
            for side in ("Min", "Max"):
                pl = sel[side][:, a].astype(F32)
                loc = (sel["Min"] + (sel["Max"] - sel["Min"]) * rng.uniform(0.2, 0.8, (len(sel), 3))).astype(np.float64)
                loc[:, a] = pl
                w = (loc @ m[:, :3].T + m[:, 3]).astype(F32)
                w = _fix_local_plane(scene, i, w, a, pl)
                dl = rng.normal(size=(len(sel), 3))
                dl[:, a] = 0.0
                dw = _unit(dl @ m[:, :3].T)
                dw[:, a] = np.where(rng.rand(len(sel)) < 0.5, F32(0.0), F32(-0.0))
                add(w, dw)
                dw2 = _unit(rng.normal(size=(len(sel), 3)))        # crossing the plane
                add(w, dw2)
    if scene.use_tlas and len(scene.tlas_nodes):
        tn = scene.tlas_nodes
        for a in range(3):
            for side in ("Min", "Max"):
                loc = (tn["Min"] + (tn["Max"] - tn["Min"]) * rng.uniform(0.1, 0.9, (len(tn), 3))).astype(F32)
                loc[:, a] = tn[side][:, a]
                dl = rng.normal(size=(len(tn), 3)).astype(F32)
                dl[:, a] = F32(-0.0) if side == "Min" else F32(0.0)
                add(loc, _unit(dl))
    # 4. aimed exactly at vertices and edge midpoints (float32 positions)
    tgt = [pos[pick, k] for k in range(3)] + [((pos[pick, k].astype(np.float64) + pos[pick, (k + 1) % 3]) * 0.5).astype(F32) for k in range(3)]
    tgt = np.concatenate(tgt)
    src = (ctr + ext * rng.uniform(-0.8, 0.8, (len(tgt), 3))).astype(F32)
    add(src, (tgt.astype(np.float64) - src).astype(F32))                    # unnormalised: t = 1 at the target
    add(src, _unit(tgt.astype(np.float64) - src))
    # 5. in the plane of a wall: dot(d, n) == 0 for the axis-aligned walls
    for k in big[:12]:
        p0, p1, p2 = pos[k].astype(np.float64)
        o = (p0 + rng.uniform(-0.3, 1.3, (8, 1)) * (p1 - p0) + rng.uniform(-0.3, 1.3, (8, 1)) * (p2 - p0)).astype(F32)
        add(o, (p1 - p0).astype(F32))
        add(o, (p2 - p1).astype(F32))
        add(o, _unit((p2 - p0) + 0.5 * (p1 - p0)))
    # 6. origins exactly on a surface (t == 0 possible), both away from and into it
    for k in big[:12]:
        p0, p1, p2 = pos[k].astype(np.float64)
        o = (p0 + 0.3 * (p1 - p0) + 0.25 * (p2 - p0)).astype(F32)
        nn = np.cross(p1 - p0, p2 - p0)
        for s in (1.0, -1.0):
            add(o, _unit(s * nn + rng.normal(size=3) * 0.3 * np.linalg.norm(nn)))
        add(pos[k], _unit(ctr - pos[k].astype(np.float64)))
    # 7. boundary TMax: 0, smallest denormal, the float32 hit distance and its neighbours, FLT_MAX, +inf
    base = _unit(rng.normal(size=(50, 3)))
    o7 = inner[rng.randint(0, len(inner), 50)]
    probe = ol.make_rays(o7, base)
    th = ol.trace_rays(scene, probe)["T"]
    hit = th < F32(3.4028235e38)
    o7, d7, th = o7[hit], base[hit], th[hit]
    for tm in (F32(0.0), np.nextafter(F32(0), F32(1)), th, np.nextafter(th, F32(0)), np.nextafter(th, F32(np.inf)),
               F32(3.4028235e38), F32(np.inf)):
        add(o7, d7, np.broadcast_to(np.asarray(tm, F32), (len(o7),)))
    # 8. denormal direction components (1/d overflows), unnormalised lengths 1e-3..1e3, origins 1e4..1e6 away
    d8 = _unit(rng.normal(size=(60, 3)))
    den = np.array([1e-45, -1e-40, 3e-39, -1.1754942e-38], F32)
    for a in range(3):
        dd = d8.copy()
        dd[:, a] = den[rng.randint(0, len(den), 60)]
        add(inner[rng.randint(0, len(inner), 60)], dd)
    scale = (10.0 ** rng.uniform(-3, 3, (60, 1))).astype(F32)
    add(inner[rng.randint(0, len(inner), 60)], d8 * scale)
    aim = (ctr + ext * rng.uniform(-0.5, 0.5, (60, 3)))
    far = aim - d8.astype(np.float64) * (10.0 ** rng.uniform(4, 6, (60, 1)))
    add(far.astype(F32), d8)
    add(far.astype(F32), (d8 * scale).astype(F32))

    r = np.zeros(sum(len(x) for x in O), gt.IdkPtRay)
    r["Origin"], r["Direction"], r["TMax"] = np.concatenate(O), np.concatenate(D), np.concatenate(TM)
    assert np.isfinite(r["Origin"]).all() and np.isfinite(r["Direction"]).all() and not np.isnan(r["TMax"]).any()
    assert (np.abs(r["Direction"]).max(1) > 0).all()
    return r


def random_rays(n, scene, seed, tris=None):
    """Unit-direction rays from random points of the scene's bounds."""
    rng = np.random.RandomState(seed)
    W = tris or world_triangles(scene)
    pos = W["pos32"].reshape(-1, 3).astype(np.float64)
    lo, hi = pos.min(0), pos.max(0)
    o = (lo + (hi - lo) * rng.uniform(0.02, 0.98, (n, 3))).astype(F32)
    return ol.make_rays(o, _unit(rng.normal(size=(n, 3))))


def box_leak_rays(box_min, box_max, per_edge=9, origins=6, seed=3):
    """Rays from inside an axis-aligned box at points of its 12 edges and at its 8 corners (float32 targets)."""
    rng = np.random.RandomState(seed)
    lo, hi = np.asarray(box_min, np.float64), np.asarray(box_max, np.float64)
    c = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
    tgt = [c]
    s = np.linspace(0, 1, per_edge + 2)[1:-1, None]
    for i in range(8):
        for j in range(i + 1, 8):
            if np.count_nonzero(c[i] != c[j]) == 1:
                tgt.append(c[i] + s * (c[j] - c[i]))
    tgt = np.concatenate(tgt).astype(F32)
    org = (lo + (hi - lo) * rng.uniform(0.2, 0.8, (origins, 3))).astype(F32)
    o = np.repeat(org, len(tgt), 0)
    t = np.tile(tgt, (origins, 1))
    return ol.make_rays(o, _unit(t.astype(np.float64) - o))
