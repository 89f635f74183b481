"""The G-buffer pass oracle (oracle/oracle_gbuffer.cpp) on the CPU: the attachment conversions at their edges, the front-face
rule against window-space winding, the whole pass against an independent float64 brute-force restatement, and velocity known
answers (DESIGN.md 8f.1g)."""
import numpy as np
import pytest

import gbuffer_oracle as go
import oracle_lib as ol
from idkengine_b200 import scenes
from idkengine_b200.host import Model, Scene, trs_matrix

W, H = 48, 32
CAM = dict(position=(0.0, 1.0, 3.0), view_dir=(0.0, 0.0, -1.0), fov_y_deg=60.0)


def small_scene():
    """Every rule of the pass in view: an opaque back wall; a single-sided quad seen from behind (culled) and a double-sided
    one (kept, normal flipped); a blended quad in front of an opaque one; an alpha cut-out; a mirrored instance (front-facing
    only because the mirror flips its winding); a double-sided quad that crosses the near plane; and the double-sided quad's
    instance moved since the previous frame (PrevModelMatrix != ModelMatrix)."""
    specs = [dict(color=(0.7, 0.7, 0.7), roughness=0.6),                      # 0 back wall
             dict(color=(0.9, 0.1, 0.1)),                                     # 1 single-sided, seen from behind
             dict(color=(0.1, 0.9, 0.1), metallic=0.5, emissive=(0.5, 0.25, 0.0)),  # 2 double-sided, seen from behind
             dict(color=(0.2, 0.3, 0.9), roughness=0.3),                      # 3 opaque behind the blended quad
             dict(color=(0.9, 0.9, 0.2, 0.5), cutoff=2.0),                    # 4 blended
             dict(color=(1.0, 1.0, 1.0), cutoff=0.5),                         # 5 alpha cut-out (checker alpha)
             dict(color=(0.6, 0.3, 0.8), roughness=0.2),                      # 6 mirrored instance
             dict(color=(0.3, 0.8, 0.8))]                                     # 7 crosses the near plane
    scene = Scene()
    t_cut = scene.add_texture(scenes._checker(32, 4, (30, 160, 60), (30, 160, 60), alpha_a=255, alpha_b=20, seed=3), srgb=True)
    meshes, mats = scenes._materials(specs)
    mats["IsDoubleSided"][2] = mats["IsDoubleSided"][7] = 1
    mats["BaseColorTexture"][5] = t_cut

    def model(quads, mesh, matrix=None, uv=None):
        a = scenes._Assembler()
        for q in quads:
            a.add(scenes.quad(*q), 0)
        m, t = meshes[mesh:mesh + 1].copy(), mats[mesh:mesh + 1].copy()
        m["MaterialId"] = 0
        return Model(np.concatenate(a.pos), np.concatenate(a.idx), np.concatenate(a.mesh), texcoords=uv, meshes=m, materials=t,
                     model_matrix=matrix)
    ccw = lambda x0, x1, y0, y1, z: ([x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z])   # front-facing from +z
    cw = lambda x0, x1, y0, y1, z: ([x0, y0, z], [x0, y1, z], [x1, y1, z], [x1, y0, z])    # back-facing from +z
    uv = np.array([[0, 0], [2, 0], [2, 2], [0, 2]], np.float32)
    scene.add(model([ccw(-3, 3, -1, 3, -2)], 0),
              model([cw(-1.4, -0.6, 0.2, 0.9, -1)], 1),
              model([cw(0.6, 1.4, 0.2, 0.9, -1)], 2),
              model([ccw(-0.4, 0.4, 1.2, 1.8, -1.5)], 3),
              model([ccw(-0.5, 0.5, 1.1, 1.9, -0.5)], 4),
              model([ccw(-1.4, -0.6, 1.2, 1.8, -1.2)], 5, uv=uv),
              model([cw(0.6, 1.4, -0.7, -0.1, -1)], 6, matrix=np.diag([-1.0, 1.0, 1.0, 1.0])),
              model([([0.05, 0.85, 2.95], [0.35, 0.85, 2.4], [0.35, 1.15, 2.4], [0.05, 1.15, 2.95])], 7), threads=1)
    scene.mesh_transforms["PrevModelMatrix"][2] = trs_matrix(1.0, 0.0, (0.1, -0.05, 0.0)).astype(np.float32)[:3, :]
    return scene, CAM


# ---- conversions ---------------------------------------------------------------------------------------------------------------
def ufloat64(v, mbits, max_finite):
    """GL's unsigned small float, restated in float64: the nearest representable value (ties to the even mantissa)."""
    v = np.asarray(v, np.float64)
    out = np.empty_like(v)
    for i, x in np.ndenumerate(v):
        if np.isnan(x):
            out[i] = np.nan
        elif not x > 0:
            out[i] = 0.0
        elif np.isinf(x):
            out[i] = np.inf
        else:
            e = max(int(np.floor(np.log2(x))), -14)
            q = 2.0 ** (e - mbits)
            k = x / q
            r = np.floor(k)
            if k - r > 0.5 or (k - r == 0.5 and int(r) % 2 == 1):
                r += 1
            out[i] = min(r * q, max_finite)
    return out


@pytest.mark.parametrize("kind,mbits,max_finite", [(go.STORE_R11G11, 6, 65024.0), (go.STORE_B10, 5, 64512.0)])
def test_unsigned_float_store_at_its_edges(kind, mbits, max_finite):
    one_ulp = 2.0 ** -mbits
    halfway = [1 + one_ulp * (k + 0.5) for k in range(4)]                       # ties: even mantissa wins
    near_half = [np.nextafter(np.float32(h), np.float32(0)) for h in halfway] + [np.nextafter(np.float32(h), np.float32(9)) for h in halfway]
    denormals = [2.0 ** -14 * k / 2 ** mbits for k in range(0, 5)] + [2.0 ** -14 * (k + 0.5) / 2 ** mbits for k in range(4)] + [1e-30, 1e-45]
    big = [max_finite, max_finite + 1, 65535.0, 65536.0, 1e30, 3.4e38]
    special = [-0.0, -1.0, -1e-30, -np.inf, np.inf, np.nan]
    v = np.array(halfway + near_half + denormals + big + special + list(np.random.default_rng(1).random(200) * 8), np.float32)
    got = go.store(kind, v)
    want = ufloat64(v, mbits, max_finite).astype(np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok], want[ok]), np.stack([v[ok], got[ok], want[ok]], 1)[got[ok] != want[ok]]
    assert go.store(kind, np.float32([1 + one_ulp * 0.5]))[0] == 1.0 and go.store(kind, np.float32([1 + one_ulp * 1.5]))[0] == 1 + 2 * one_ulp
    assert got[v == np.float32(np.inf)][0] == np.inf and got[v == np.float32(3.4e38)][0] == max_finite


def test_rg8_and_rg16f_stores():
    k = np.arange(256, dtype=np.float64)
    eps = 1e-4
    v = np.concatenate([(k + 0.5 - eps) / 255, (k + 0.5 + eps) / 255, k / 255, [-1.0, 2.0, np.nan, np.inf, -np.inf]]).astype(np.float32)
    want = np.floor(np.clip(np.nan_to_num(v.astype(np.float64), nan=0.0), 0, 1) * 255 + 0.5) / 255
    assert np.array_equal(go.store(go.STORE_RG8, v), want.astype(np.float32))
    h = np.concatenate([np.random.default_rng(2).standard_normal(500) * 3, [65504.0, 65519.0, 1e-8, -2.0 ** -25]]).astype(np.float32)
    assert np.array_equal(go.store(go.STORE_RG16F, h), h.astype(np.float16).astype(np.float32))


# ---- the front-face rule ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["identity", "rotated", "scaled", "mirrored"])
def test_front_face_rule_matches_window_space_winding(model):
    """Rule 2's det(Model) * dot(n_local, d_local) < 0 is the sign of the projected window-space area (CCW front, lower-left
    origin) wherever that area is not within rounding of 0."""
    m = {"identity": np.eye(4), "rotated": trs_matrix(1.0, 37.0, (0.2, 0.1, -0.3)), "scaled": trs_matrix((2.0, 0.5, 1.3), -20.0),
         "mirrored": trs_matrix((-1.0, 1.2, 0.9), 25.0, (0.1, 0.0, 0.2))}[model]
    if model == "mirrored":
        assert np.linalg.det(m[:3, :3]) < 0
    f = scenes.camera_frame(CAM, W, H)[0]
    pv = np.asarray(f["ProjView"], np.float64).reshape(4, 4).T
    eye = np.asarray(f["ViewPos"], np.float64)
    rng = np.random.default_rng(7)
    inv = np.linalg.inv(m)
    checked = 0
    for _ in range(400):
        centre = eye + np.array([0, 0, -3.0]) + rng.uniform(-1, 1, 3)
        local = (inv @ np.append(centre, 1))[:3] + rng.uniform(-0.5, 0.5, (3, 3))
        world = (m @ np.c_[local, np.ones(3)].T).T[:, :3]
        clip = (pv @ np.c_[world, np.ones(3)].T).T
        ndc = clip[:, :2] / clip[:, 3:]
        e1, e2 = ndc[1] - ndc[0], ndc[2] - ndc[0]
        area = e1[0] * e2[1] - e1[1] * e2[0]
        if abs(area) < 1e-6 or (clip[:, 3] <= 0).any():
            continue
        n_local = np.cross(local[1] - local[0], local[2] - local[0])
        d_local = inv[:3, :3] @ (world.mean(0) - eye)
        det = np.linalg.det(m[:3, :3])
        assert (area > 0) == (det * np.dot(n_local, d_local) < 0)
        checked += 1
    assert checked > 300


# ---- the whole pass against float64 ----------------------------------------------------------------------------------------------
def encode_unit_vec(n):
    m = n / np.sum(np.abs(n), -1, keepdims=True)
    wrap = (1.0 - np.abs(m[..., [1, 0]])) * np.where(m[..., :2] < 0, -1.0, 1.0)
    return np.where((m[..., 2] > 0)[..., None], m[..., :2], wrap) * 0.5 + 0.5


def float64_gbuffer(scene, frame, w, h, jitter=(0.0, 0.0)):
    """Brute force over every world-space triangle in float64: the closest hit that is not blended, not a back face of a
    single-sided material (world-space winding), not clipped and not alpha-discarded. Returns (depth, normal_rg before RG8,
    albedo, metallic_roughness, emissive, velocity before RG16F, mesh id, edge distance) per pixel."""
    f = frame[0]
    pv = np.asarray(f["ProjView"], np.float64).reshape(4, 4).T
    ppv = np.asarray(f["PrevProjView"], np.float64).reshape(4, 4).T
    ipv = np.asarray(f["InvProjView"], np.float64).reshape(4, 4).T
    eye = np.asarray(f["ViewPos"], np.float64)
    P = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float64)
    tris = []
    for inst in scene.blas_instances:
        desc = scene.blas_descs[inst["BlasId"]]
        mt = scene.mesh_transforms[inst["MeshTransformId"]]
        M = np.vstack([np.asarray(mt["ModelMatrix"], np.float64), [0, 0, 0, 1]])
        Mp = np.vstack([np.asarray(mt["PrevModelMatrix"], np.float64), [0, 0, 0, 1]])
        for k in range(desc["TriangleOffset"], desc["TriangleOffset"] + desc["TriangleCount"]):
            t = scene.blas_triangles[k]
            ids = [t["X"], t["Y"], t["Z"]]
            tris.append((ids, (M @ np.c_[P[ids], np.ones(3)].T).T[:, :3], (Mp @ np.c_[P[ids], np.ones(3)].T).T[:, :3], int(t["MeshId"])))
    out = dict(depth=np.ones((h, w)), normal=np.zeros((h, w, 2)), albedo=np.zeros((h, w, 3)), mr=np.zeros((h, w, 2)),
               emissive=np.zeros((h, w, 3)), velocity=np.zeros((h, w, 2)), mesh=np.full((h, w), -1), edge=np.full((h, w), np.inf))
    for y in range(h):
        for x in range(w):
            ndc = np.array([(x + 0.5) / w * 2 - 1 - jitter[0], (y + 0.5) / h * 2 - 1 - jitter[1], 1.0, 1.0])
            q = ipv @ ndc
            d = q[:3] / q[3] - eye
            d /= np.linalg.norm(d)
            best = None
            for ids, wp, pp, mesh_id in tris:
                e1, e2 = wp[1] - wp[0], wp[2] - wp[0]
                n = np.cross(e1, e2)
                det = -np.dot(d, n)
                if abs(det) < 1e-12:
                    continue
                ao = eye - wp[0]
                dao = np.cross(ao, d)
                t = np.dot(ao, n) / det
                u = np.dot(e2, dao) / det
                v = -np.dot(e1, dao) / det
                b = np.array([1 - u - v, u, v])
                out["edge"][y, x] = min(out["edge"][y, x], abs(b).min() if t > 0 else np.inf)
                if t <= 0 or b.min() < 0 or (best is not None and t >= best[0]):
                    continue
                mesh = scene.meshes[mesh_id]
                mat = scene.materials[mesh["MaterialId"]]
                if mat["AlphaCutoff"] == 2.0 or (not mat["IsDoubleSided"] and np.dot(n, d) >= 0):
                    continue
                clip = (pv @ np.c_[wp, np.ones(3)].T).T
                depth = (b @ clip[:, 2]) / (b @ clip[:, 3])
                if not 0 <= depth <= 1:
                    continue
                c = int(mat["BaseColorFactor"])
                alpha = ((c >> 24) & 255) / 255.0
                if mat["BaseColorTexture"]:
                    tc = b @ scene.vertices["TexCoord"][ids].astype(np.float64)
                    tex = scene.textures[int(mat["BaseColorTexture"]) - 1]
                    alpha *= ol.tex_sample(tex["pixels"], tc.astype(np.float32)[None], srgb=tex["srgb"])[0, 3]
                if alpha < mat["AlphaCutoff"]:
                    continue
                best = (t, b, wp, pp, n, mesh_id, depth)
            if best is None:
                continue
            t, b, wp, pp, n, mesh_id, depth = best
            mesh = scene.meshes[mesh_id]
            mat = scene.materials[mesh["MaterialId"]]
            c = int(mat["BaseColorFactor"])
            albedo = np.array([(c >> s) & 255 for s in (0, 8, 16)]) / 255.0
            nrm = n / np.linalg.norm(n) * (1.0 if np.dot(n, d) < 0 else -1.0)    # flat quads: the vertex normals are the face's
            clip_prev = (ppv @ np.c_[pp, np.ones(3)].T).T
            pc = b @ clip_prev
            out["depth"][y, x] = depth
            out["normal"][y, x] = encode_unit_vec(nrm)
            out["albedo"][y, x] = albedo
            out["mr"][y, x] = [np.clip(mat["MetallicFactor"] + mesh["SpecularBias"], 0, 1), np.clip(mat["RoughnessFactor"] + mesh["RoughnessBias"], 0, 1)]
            out["emissive"][y, x] = np.asarray(mat["EmissiveFactor"], np.float64) + mesh["EmissiveBias"] * albedo
            out["velocity"][y, x] = (ndc[:2] - pc[:2] / pc[3]) * 0.5
            out["mesh"][y, x] = mesh_id
    return out


def rg8(v):
    return np.floor(np.clip(v, 0, 1) * 255 + 0.5) / 255


@pytest.mark.parametrize("jitter", [None, (0.0123, -0.0311)])
def test_oracle_matches_float64_brute_force(jitter):
    scene, cam = small_scene()
    frame = scenes.camera_frame(cam, W, H)
    g = go.gbuffer(scene, frame, W, H, jitter=jitter, threads=1)
    ref = float64_gbuffer(scene, frame, W, H, (0.0, 0.0) if jitter is None else jitter)
    # every rule is in view: the culled quad, the blended quad and the cut-out holes leave what is behind them visible
    seen = set(np.unique(ref["mesh"]))
    assert {0, 2, 3, 5, 6, 7} <= seen and 1 not in seen and 4 not in seen
    # away from triangle edges (the fp32 and float64 walks may pick different triangles there) and, for the RG8 normal, from
    # its rounding boundaries
    far = ref["edge"] > 1e-4
    excluded = int((~far).sum())
    assert excluded == 0, excluded          # pinned: at this size no pixel centre lies that close to an edge
    hit = ref["mesh"] >= 0
    assert np.array_equal(g[0] < 1.0, hit | ~far) or np.array_equal((g[0] < 1.0)[far], hit[far])
    m = far & hit
    assert np.allclose(g[0][m], ref["depth"][m], rtol=0, atol=2e-6)
    assert np.array_equal(g[0][far & ~hit], np.ones((far & ~hit).sum(), np.float32))
    untextured = m & (ref["mesh"] != 5)    # the cut-out's colour is its texture's (the GPU tests compare it with the oracle)
    for k, want in ((2, ref["albedo"]), (4, ref["emissive"])):
        q = np.stack([ufloat64(want[..., c], 6 if c < 2 else 5, 65024.0 if c < 2 else 64512.0) for c in range(3)], -1)
        assert np.array_equal(g[k][untextured], q[untextured].astype(np.float32))
    assert np.array_equal(g[3][m], rg8(ref["mr"])[m].astype(np.float32))
    boundary = np.abs(ref["normal"] * 255 - np.floor(ref["normal"] * 255) - 0.5) < 1e-3
    nm = m[..., None] & ~boundary
    assert np.array_equal(g[1][nm], rg8(ref["normal"])[nm].astype(np.float32))
    assert np.allclose(g[5][m], ref["velocity"][m], rtol=2 ** -10, atol=2e-6)   # fp32 NDC differences, then RG16F
    # the moved instance has velocity; the static ones have none
    moved = m & (ref["mesh"] == 2)
    assert moved.any() and (np.abs(g[5][moved]).max() > 1e-3)
    static = m & (ref["mesh"] == 0)
    assert np.abs(g[5][static]).max() < 2e-6


def test_velocity_known_answers():
    scene, cam = scenes.cornell_1k(threads=1)
    frame = scenes.camera_frame(cam, W, H)
    g = go.gbuffer(scene, frame, W, H, threads=1)
    assert np.abs(g[5]).max() < 1e-6                                   # static camera and scene
    # the camera moved by dx since the previous frame: a point at view depth z moves by the projected difference
    moved = dict(cam, position=(cam["position"][0] + 0.05, cam["position"][1], cam["position"][2]))
    prev = scenes.camera_frame(moved, W, H)
    frame2 = frame.copy()
    frame2["PrevProjView"] = prev["ProjView"]
    g2 = go.gbuffer(scene, frame2, W, H, threads=1)
    hit = g2[0] < 1
    pv = np.asarray(frame2[0]["ProjView"], np.float64).reshape(4, 4).T
    ppv = np.asarray(prev[0]["ProjView"], np.float64).reshape(4, 4).T
    ys, xs = np.nonzero(hit)
    ndc = np.stack([(xs + 0.5) / W * 2 - 1, (ys + 0.5) / H * 2 - 1, g2[0][hit].astype(np.float64), np.ones(len(xs))])
    wp = np.linalg.inv(pv) @ ndc
    pc = ppv @ (wp / wp[3])
    want = (ndc[:2] - pc[:2] / pc[3]) * 0.5
    assert np.allclose(g2[5][hit].T, want, atol=2e-3)
    # an instance moved by a translation: every pixel it covers moves by the projection of that translation
    scene3, cam3 = scenes.multi_blas(threads=1)
    f3 = scenes.camera_frame(cam3, W, H)
    ball = 1
    scene3.mesh_transforms["PrevModelMatrix"][ball, :, 3] -= np.float32([0.2, 0.0, 0.0])
    g3 = go.gbuffer(scene3, f3, W, H, threads=1)
    g0 = go.gbuffer(scene3, f3, W, H, threads=1, prev_positions=None)
    assert np.array_equal(g3[0], g0[0])
    pv3 = np.asarray(f3[0]["ProjView"], np.float64).reshape(4, 4).T
    hit3 = g3[0] < 1
    ys, xs = np.nonzero(hit3)
    ndc = np.stack([(xs + 0.5) / W * 2 - 1, (ys + 0.5) / H * 2 - 1, g3[0][hit3].astype(np.float64), np.ones(len(xs))])
    wp = np.linalg.inv(pv3) @ ndc
    wp = wp / wp[3]
    moving = np.abs(g3[5][hit3]).max(-1) > 1e-3
    assert moving.sum() > 20
    pc = pv3 @ (wp[:, moving] - np.array([[0.2], [0], [0], [0]]))
    want = (ndc[:2, moving] - pc[:2] / pc[3]) * 0.5
    assert np.allclose(g3[5][hit3][moving].T, want, atol=2e-3)
