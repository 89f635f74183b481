"""Float64 restatement of the voxeliser under Voxelizer.IsConservativeRasterization (Voxelizer.cs:41-56,142, which enables
GL_NV_conservative_raster for the voxelise draw), written from the engine's shaders and GL's definition of conservative
rasterisation, not from oracle/oracle_vxgi_conservative.cpp or csrc/idk_vxgi.cuh. Everything but coverage is
tests/vxgi_ref64.py's voxelize64: projection along the dominant axis of the NDC-space normal, the fragment stage for
factor-only materials and lights without point shadows, the per-channel max merge.

Coverage: a pixel is covered when its closed square meets the projected triangle. This is decided without edge-function
offsets: a triangle vertex lies in the square, a square corner lies in the triangle, or a triangle edge crosses a square edge
properly (square_meets_triangle). Attributes are evaluated at the pixel centre with float64 barycentrics, which are negative
outside the triangle (GL extrapolates non-centroid inputs, and the reference's InOutData has no `centroid`)."""
import math

import numpy as np

from vxgi_ref64 import F, _normalize, _rows

EPS32 = 2.0 ** -24            # unit roundoff of float32
ILL_CONDITIONED = 0.5         # voxels: a sample whose FragPos error bound exceeds this is ill-conditioned


def _orient(ax, ay, bx, by, cx, cy):
    return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)


def square_meets_triangle(x0, y0, x1, y1, qa, qb):
    """Do the closed squares [x0, x1] x [y0, y1] (arrays) meet the closed triangle (qa, qb)? Two convex polygons meet exactly
    when a vertex of one lies in the other or their boundaries cross properly (a touching contact puts a vertex of one on
    the other)."""
    hit = np.zeros(np.broadcast(x0, y0).shape, bool)
    for k in range(3):
        hit |= (qa[k] >= x0) & (qa[k] <= x1) & (qb[k] >= y0) & (qb[k] <= y1)
    sgn = 1.0 if _orient(qa[0], qb[0], qa[1], qb[1], qa[2], qb[2]) > 0 else -1.0
    corners = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
    for cx, cy in corners:
        hit |= np.all([sgn * _orient(qa[p], qb[p], qa[q], qb[q], cx, cy) >= 0 for p, q in ((1, 2), (2, 0), (0, 1))], 0)
    for p, q in ((1, 2), (2, 0), (0, 1)):
        for c in range(4):
            (ux, uy), (vx, vy) = corners[c], corners[(c + 1) % 4]
            o1 = _orient(qa[p], qb[p], qa[q], qb[q], ux, uy)
            o2 = _orient(qa[p], qb[p], qa[q], qb[q], vx, vy)
            o3 = _orient(ux, uy, vx, vy, qa[p], qb[p])
            o4 = _orient(ux, uy, vx, vy, qa[q], qb[q])
            hit |= (o1 * o2 < 0) & (o3 * o4 < 0)
    return hit


def voxelize64_conservative(scene, ci, eps=1e-5):
    """Voxelisation under the conservative rule. Returns dict(level0 = float16 [d, h, w, 4], written, ambiguous = bool
    [d, h, w], fragments = count of unambiguous covered samples (presplit BLAS triangles counted as often as the BLAS holds
    them), ambiguous_samples, ill_conditioned_samples).

    A sample is *ambiguous* when
    - the square-to-triangle distance is within delta = eps * (max |q| + 1) pixels of 0: the square grown by delta meets
      the triangle and the square shrunk by delta does not;
    - its FragPos lies within eps (relative) plus the FragPos error bound below of an integer voxel coordinate (the voxels on
      both sides, and every voxel within a margin wider than one voxel, are flagged);
    - its triangle's dominant axis is tied (within eps) with another (rasterised along every tied axis, all samples flagged);
    - its extrapolation is ill-conditioned: the fp32 FragPos is only as good as its conditioning, with an error bound of
      err = 4 eps32 sum_k (|b_k| + |db_k|) |P_k| (world units per axis), db_k = (c_k + |b_k| c_area) / |area| the fp32 error
      bound of w_k / area, c_k the magnitude of the terms of edge function k (including the rounding of the window
      coordinates); a sample with err above ILL_CONDITIONED voxels (sum_k |b_k| is then in the thousands) counts in
      ill_conditioned_samples.
    Near-degenerate projections (|area| <= eps * scale) are sampled too, as long as the area is not exactly 0: their samples
    come out ill-conditioned."""
    import edge_lib
    size = np.array([ci.Width, ci.Height, ci.Depth])
    gmin = np.array(list(ci.GridMin), np.float64)
    gmax = np.array(list(ci.GridMax), np.float64)
    ext = gmax - gmin
    voxel = ext / size
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
    frags, amb_samples, ill_samples = 0, 0, 0
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
            if area == 0.0:
                continue
            dpx = eps * (max(np.abs(qa).max(), np.abs(qb).max()) + 1.0)
            i = np.arange(max(0, math.ceil(qa.min() - 1.0 - dpx)), min(size[a] - 1, math.floor(qa.max() + dpx)) + 1)
            j = np.arange(max(0, math.ceil(qb.min() - 1.0 - dpx)), min(size[b] - 1, math.floor(qb.max() + dpx)) + 1)
            if not len(i) or not len(j):
                continue
            cx, cy = np.meshgrid(i + 0.5, j + 0.5)
            cx, cy = cx.reshape(-1), cy.reshape(-1)
            grown = square_meets_triangle(cx - 0.5 - dpx, cy - 0.5 - dpx, cx + 0.5 + dpx, cy + 0.5 + dpx, qa, qb)
            shrunk = square_meets_triangle(cx - 0.5 + dpx, cy - 0.5 + dpx, cx + 0.5 - dpx, cy + 0.5 - dpx, qa, qb)
            near_edge = grown & ~shrunk
            cx, cy, near_edge = cx[grown], cy[grown], near_edge[grown]
            wk, ck = [], []
            for p, q in ((1, 2), (2, 0), (0, 1)):
                wk.append((qa[q] - qa[p]) * (cy - qb[p]) - (qb[q] - qb[p]) * (cx - qa[p]))
                ck.append(np.abs(qa[q] - qa[p]) * (np.abs(cy - qb[p]) + abs(qb[p])) + np.abs(qb[q] - qb[p]) * (np.abs(cx - qa[p]) + abs(qa[p])))
            bary = np.stack(wk, -1) / area                                # extrapolated barycentrics
            c_area = abs(qa[1] - qa[0]) * (abs(qb[2] - qb[0]) + abs(qb[0])) + abs(qb[1] - qb[0]) * (abs(qa[2] - qa[0]) + abs(qa[0]))
            db = (np.stack(ck, -1) + np.abs(bary) * c_area) / abs(area)
            err = ((4.0 * EPS32 * ((np.abs(bary) + db) @ np.abs(P[t]))) / voxel).max(-1)   # FragPos error bound, voxels
            frag = bary @ P[t]
            u = (frag - gmin) / ext * size
            delta = eps * np.maximum(1.0, np.abs(u)) + err[:, None]
            near_int = (np.abs(u - np.round(u)) <= delta).any(-1)
            ill = err > ILL_CONDITIONED
            is_amb = near_edge | near_int | bool(tied) | ill
            with np.errstate(invalid="ignore"):
                vox_lo, vox_hi = np.floor(u - delta).astype(np.int64), np.floor(u + delta).astype(np.int64)
            ok = lambda v: (v >= 0).all(-1) & (v < size).all(-1)          # noqa: E731
            for v in (vox_lo, vox_hi):
                m = is_amb & ok(v)
                amb[v[m, 2], v[m, 1], v[m, 0]] = True
            for k in np.nonzero(is_amb & ((vox_hi - vox_lo) > 1).any(-1))[0]:   # a margin wider than a voxel: every voxel in it
                lo, hi = np.clip(vox_lo[k], 0, size), np.clip(vox_hi[k] + 1, 0, size)
                amb[lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]] = True
            ill_samples += int(ill.sum()) * int(mult[t])
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
    return dict(level0=lv0, written=written, ambiguous=amb, fragments=frags, ambiguous_samples=amb_samples,
                ill_conditioned_samples=ill_samples)
