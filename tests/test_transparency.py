"""Transparency (the record and resolve passes) on the CPU: the oracle against an independent float64 brute force over every
world-space triangle, the walk's bound against the unbounded walk, and the resolve against a numpy restatement of
ResolveTransparent/compute.glsl."""
import copy

import numpy as np
import pytest

import transparency_oracle as to
from idkengine_b200 import scenes
from raster_lib import rule_scene


def opaque_inputs(scene, frame, w, h):
    """The G-buffer oracle's depth and a seeded lit image."""
    import gbuffer_oracle as go
    depth = go.gbuffer(scene, frame, w, h)[0]
    rng = np.random.default_rng(11)
    color = np.concatenate([rng.random((h, w, 3), dtype=np.float32) * 2.0, np.ones((h, w, 1), np.float32)], -1)
    return depth, color


def _srgb(c):
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def _tex_alpha_rgb(tex, u, v):
    """Bilinear, repeat-wrapped level-0 sample of an RGBA8 texture in float64 (texel centres at half integers): (rgb, alpha)."""
    px = tex["pixels"].astype(np.float64) / 255.0
    if tex["srgb"]:
        px[..., :3] = _srgb(px[..., :3])
    h, w = px.shape[:2]
    x, y = (u - np.floor(u)) * w - 0.5, (v - np.floor(v)) * h - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = x - x0, y - y0
    X0, X1, Y0, Y1 = int(x0) % w, int(x0 + 1) % w, int(y0) % h, int(y0 + 1) % h
    c = (px[Y0, X0] * (1 - fx) + px[Y0, X1] * fx) * (1 - fy) + (px[Y1, X0] * (1 - fx) + px[Y1, X1] * fx) * fy
    return c[:3], c[3]


def _surface(scene, mesh, mat, uv):
    """GetSurface + SurfaceApplyModificatons in float64 for materials without normal, emissive or metal/roughness textures."""
    f = int(mat["BaseColorFactor"])
    factor = np.array([(f >> s) & 255 for s in (0, 8, 16, 24)], np.float64) / 255.0
    albedo, alpha = factor[:3].copy(), factor[3]
    if mat["BaseColorTexture"]:
        rgb, a = _tex_alpha_rgb(scene.textures[int(mat["BaseColorTexture"]) - 1], uv[0], uv[1])
        albedo, alpha = rgb * factor[:3], a * factor[3]
    emissive = np.asarray(mat["EmissiveFactor"], np.float64) + float(mesh["EmissiveBias"]) * albedo
    metallic = min(max(float(mat["MetallicFactor"]) + float(mesh["SpecularBias"]), 0.0), 1.0)
    roughness = min(max(float(mat["RoughnessFactor"]) + float(mesh["RoughnessBias"]), 0.0), 1.0)
    ior = max(float(mat["IOR"]) + float(mesh["IORBias"]), 1.0)
    return albedo, alpha, emissive, metallic, roughness, ior


def _light(scene, P, N, eye, albedo, metallic, roughness, ior):
    """EvaluateLighting summed over the scene's lights, unshadowed, in float64: GGX (DistributionGGX, SmithGGXCorrelated,
    FresnelSchlick) with f0 = mix(((1 - IOR) / (1 + IOR))^2, albedo, metallic), no ambient occlusion."""
    r = roughness * roughness
    r0 = ((1.0 - ior) / (1.0 + ior)) ** 2
    f0 = r0 * (1 - metallic) + albedo * metallic
    V = (eye - P) / np.linalg.norm(eye - P)
    out = np.zeros(3)
    for l in scene.lights:
        toL = np.asarray(l["Position"], np.float64) - P
        L = toL / np.linalg.norm(toL)
        H = (V + L) / np.linalg.norm(V + L)
        NoV, NoL = abs(N @ V), min(max(N @ L, 0.0), 1.0)
        NoH, LoH = min(max(N @ H, 0.0), 1.0), min(max(L @ H, 0.0), 1.0)
        rD, rG = max(r, 0.005), max(r, 0.0001)
        D = (rD / ((1.0 - NoH * NoH) + (NoH * rD) ** 2)) ** 2 / np.pi
        G = 0.5 / (NoL * np.sqrt((-NoV * rG + NoV) * NoV + rG) + NoV * np.sqrt((-NoL * rG + NoL) * NoL + rG))
        F = f0 + (1.0 - f0) * (1.0 - LoH) ** 5
        lr = max(float(l["Radius"]), 0.0001)
        att = lr * lr / max(toL @ toL, 0.0001)
        out += (F * (D * G) + albedo * (1.0 - F) * (1.0 - metallic)) * att * NoL * np.asarray(l["Color"], np.float64)
    return out


def brute_force(scene, frame, depth, color, w, h, negate_back_faces=True):
    """The record and resolve passes restated in float64 over every world-space triangle of every instance at every pixel
    centre, sharing no code with the oracle: Moller-Trumbore intersection, the record pass's tests (blended, front-facing in
    window space or double-sided, clip depth in [0, 1] and below the opaque depth, alpha != 0 with the base texture sampled
    bilinearly at level 0), the ten closest kept by (depth, triangle, transform), each lit by the lights (unshadowed, ambient
    0.015 * albedo, emissive) with the face normal (negated on a back face), premultiplied, rounded to half, and blended front to
    back over the opaque colour. Returns ({(y, x): [(depth, tri, xf)]}, composited float64 [h, w, 4], min barycentric distance
    to a triangle edge of the kept layers [h, w]). negate_back_faces=False keeps a back face's normal (the rule's negative)."""
    f = frame[0] if frame.ndim else frame
    pv = np.asarray(f["ProjView"], np.float64).reshape(4, 4)
    ipv = np.asarray(f["InvProjView"], np.float64).reshape(4, 4)
    eye = np.asarray(f["ViewPos"], np.float64)
    pos = np.stack([scene.positions["x"], scene.positions["y"], scene.positions["z"]], 1).astype(np.float64)
    uvs = np.asarray(scene.vertices["TexCoord"], np.float64)
    cands = {}
    for inst in scene.blas_instances:
        desc = scene.blas_descs[inst["BlasId"]]
        xf = int(inst["MeshTransformId"])
        M = np.eye(4)
        M[:3, :] = np.asarray(scene.mesh_transforms["ModelMatrix"][xf], np.float64)
        for k in range(int(desc["TriangleOffset"]), int(desc["TriangleOffset"]) + int(desc["TriangleCount"])):
            t = tris = scene.blas_triangles[k]
            mesh = scene.meshes[t["MeshId"]]
            mat = scene.materials[mesh["MaterialId"]]
            if mat["AlphaCutoff"] != 2.0:
                continue
            ids = [int(t[c]) for c in ("X", "Y", "Z")]
            P = [(M @ np.append(pos[i], 1.0))[:3] for i in ids]
            n = np.cross(P[1] - P[0], P[2] - P[0])
            e1, e2 = P[1] - P[0], P[2] - P[0]
            for y in range(h):
                for x in range(w):
                    q4 = np.array([(x + 0.5) / w * 2 - 1, (y + 0.5) / h * 2 - 1, 1.0, 1.0]) @ ipv
                    d = q4[:3] / q4[3] - eye
                    d /= np.linalg.norm(d)
                    pvec = np.cross(d, e2)
                    a = e1 @ pvec
                    if abs(a) < 1e-12:
                        continue
                    sv = eye - P[0]
                    u = (sv @ pvec) / a
                    qv = np.cross(sv, e1)
                    v = (d @ qv) / a
                    tt = (e2 @ qv) / a
                    if u < 0 or v < 0 or u + v > 1 or tt <= 0:
                        continue
                    front = n @ d < 0
                    if not mat["IsDoubleSided"] and not front:
                        continue
                    hp = eye + d * tt
                    clip = np.append(hp, 1.0) @ pv
                    z = clip[2] / clip[3]
                    if not (0.0 <= z <= 1.0 and z < depth[y, x]):
                        continue
                    b = np.array([1 - u - v, u, v])
                    albedo, alpha, emissive, metallic, roughness, ior = _surface(scene, mesh, mat, b @ uvs[ids])
                    if alpha == 0.0:
                        continue
                    N = n / np.linalg.norm(n) * (1.0 if front or not negate_back_faces else -1.0)
                    c = (_light(scene, hp, N, eye, albedo, metallic, roughness, ior) + 0.015 * albedo + emissive) * alpha
                    layer = np.append(c, alpha).astype(np.float16).astype(np.float64)
                    cands.setdefault((y, x), []).append((z, k, xf, layer, b.min()))
    kept = {p: sorted(v, key=lambda c: c[:3])[:to.LAYERS] for p, v in cands.items()}
    out = np.asarray(color, np.float64).copy()
    edge = np.full((h, w), np.inf)
    for (y, x), ls in kept.items():
        acc = np.zeros(4)
        for _, _, _, layer, _ in ls:
            acc = acc + (1.0 - acc[3]) * layer
        out[y, x, :3] = acc[:3] + (1.0 - acc[3]) * out[y, x, :3]
        out[y, x, 3] = 1.0
        edge[y, x] = min(c[4] for c in ls)
    return {p: [c[:3] for c in v] for p, v in kept.items()}, out, edge


@pytest.fixture(scope="module")
def rule_run():
    scene, cam = rule_scene()
    w, h = 48, 32
    frame = scenes.camera_frame(cam, w, h)
    depth, color = opaque_inputs(scene, frame, w, h)
    return scene, frame, depth, color, w, h


@pytest.fixture(scope="module")
def rule_brute(rule_run):
    scene, frame, depth, color, w, h = rule_run
    return brute_force(scene, frame, depth, color, w, h)


EDGE = 1e-4      # pixels whose kept layers come within this barycentric distance of an edge are left out (coverage there is fp32's)
TOLERANCE = 4e-3  # |oracle - float64| <= TOLERANCE * max(1, |float64|) per channel: rgba16f layers, SR11G11B10 vertex normals


def test_brute_force_agrees_with_oracle(rule_run, rule_brute):
    """The kept layers, their order and the composited colour agree with the float64 restatement (within TOLERANCE) at every
    pixel away from triangle edges, the textured card's alpha-0 texels included; every rule's surface contributes somewhere."""
    scene, frame, depth, color, w, h = rule_run
    want, want_color, edge = rule_brute
    out, layers, counts = to.transparency(scene, frame, depth, color)
    checked = 0
    for y in range(h):
        for x in range(w):
            if edge[y, x] < EDGE:
                continue
            got = [(float(l["depth"]), int(l["tri"]), int(l["xf"])) for l in layers[y, x][:counts[y, x]]]
            ref = want.get((y, x), [])
            assert [(k, f) for _, k, f in got] == [(k, f) for _, k, f in ref], (x, y)
            for (dg, _, _), (dr, _, _) in zip(got, ref):
                assert abs(dg - dr) < 1e-5
            err = np.abs(out[y, x] - want_color[y, x]) / np.maximum(1.0, np.abs(want_color[y, x]))
            assert err.max() <= TOLERANCE, (x, y, out[y, x], want_color[y, x])
            checked += 1
    assert checked > 0.9 * w * h
    assert counts.max() == to.LAYERS                                   # the 13-pane stack hits the cap
    meshes_seen = {int(scene.blas_triangles[k]["MeshId"]) for k in np.unique(layers["tri"][layers["tri"] != 0xFFFFFFFF])}
    assert {3, 4, 5, 6, 7, 8, 9, 10} <= meshes_seen and not ({1, 2} & meshes_seen)
    untouched = counts == 0
    assert np.array_equal(out[untouched].view(np.uint32), color[untouched].view(np.uint32))


def test_card_alpha_zero_texels_are_discarded(rule_run, rule_brute):
    """Inside the card's outline, pixels whose sampled alpha is 0 have no card layer, in the float64 restatement and in the
    oracle alike, and both kinds of pixel occur."""
    scene, frame, depth, color, w, h = rule_run
    want, _, edge = rule_brute
    _, layers, counts = to.transparency(scene, frame, depth, color)
    card_tris = {k for k in range(len(scene.blas_triangles)) if scene.blas_triangles[k]["MeshId"] == 4}
    with_card = {p for p, v in want.items() if any(k in card_tris for _, k, _ in v)}
    got_card = {(y, x) for y in range(h) for x in range(w) if any(int(l["tri"]) in card_tris for l in layers[y, x][:counts[y, x]])}
    assert with_card == {p for p in got_card if edge[p] >= EDGE} | {p for p in with_card if edge[p] < EDGE}
    # the card's screen box: some of its pixels are discarded (alpha-0 texels), some kept
    ys, xs = zip(*with_card)
    box = [(y, x) for y in range(min(ys), max(ys) + 1) for x in range(min(xs), max(xs) + 1)]
    assert any(p not in with_card for p in box)


def test_back_face_normal_is_negated(rule_run, rule_brute):
    """The double-sided quad seen from behind is lit with its normal negated: the oracle agrees with the float64 restatement
    within 1 % of the pixel's colour, and the restatement without the negation is farther off than that."""
    scene, frame, depth, color, w, h = rule_run
    want_layers, want, edge = rule_brute
    _, unflipped, _ = brute_force(scene, frame, depth, color, w, h, negate_back_faces=False)
    out = to.transparency(scene, frame, depth, color)[0]
    back = np.zeros((h, w), bool)
    for (y, x), v in want_layers.items():
        back[y, x] = edge[y, x] >= EDGE and any(scene.blas_triangles[k]["MeshId"] == 3 for _, k, _ in v)
    assert back.any()
    rel = np.abs(out - want)[..., :3] / np.abs(want)[..., :3]
    rel_unflipped = np.abs(out - unflipped)[..., :3] / np.abs(unflipped)[..., :3]
    assert rel[back].max() <= 0.001
    assert rel_unflipped[back].max() > 0.002


def test_coplanar_tie_is_ordered_by_triangle(rule_run):
    scene, frame, depth, color, w, h = rule_run
    _, layers, counts = to.transparency(scene, frame, depth, color)
    ties = 0
    for y in range(h):
        for x in range(w):
            l = layers[y, x][:counts[y, x]]
            for a, b in zip(l[:-1], l[1:]):
                assert (a["depth"], a["tri"], a["xf"]) < (b["depth"], b["tri"], b["xf"])
                ties += a["depth"] == b["depth"]
    assert ties > 0


@pytest.mark.parametrize("which", ["rule", "cornell", "multi_blas", "multi_blas_tlas", "atrium", "textured_room"])
def test_bound_never_drops_a_layer(which):
    if which == "rule":
        scene, cam = rule_scene()
    elif which == "cornell":
        scene, cam = scenes.cornell_1k(threads=1)
    elif which.startswith("multi_blas"):
        scene, cam = scenes.multi_blas(threads=1)
        if which == "multi_blas_tlas":
            scene.build_tlas()
    elif which == "atrium":
        scene, cam = scenes.atrium(20000, threads=1)
    else:
        scene, cam = scenes.textured_room(threads=1)
    if which in ("cornell", "multi_blas", "multi_blas_tlas", "atrium", "textured_room"):   # as the GPU tests blend them
        scene.materials["AlphaCutoff"][::3] = 2.0
        scene.materials["BaseColorFactor"][::3] = (scene.materials["BaseColorFactor"][::3] & 0x00FFFFFF) | (0x80 << 24)
    w, h = 40, 28
    frame = scenes.camera_frame(cam, w, h)
    depth, color = opaque_inputs(scene, frame, w, h)
    a = to.transparency(scene, frame, depth, color, bound=True)
    b = to.transparency(scene, frame, depth, color, bound=False)
    assert a[2].any()
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and np.array_equal(a[2], b[2])
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def resolve_glsl(colors, depths, opaque):
    """ResolveTransparent/compute.glsl for one pixel, in float32: the insertion sort of the records in record order (a new item
    goes before the first strictly greater depth, so equal depths keep their record order), front-to-back blending
    acc += (1 - acc.a) * colour, then acc += (1 - acc.a) * vec4(opaque.rgb, 1)."""
    frags = []
    for c, d in zip(colors, depths):
        for i, (_, fd) in enumerate(frags):
            if d < fd:
                frags.insert(i, (c, d))
                break
        else:
            frags.append((c, d))
    acc = np.zeros(4, np.float32)
    for c, _ in frags:
        acc = acc + np.float32(1.0 - acc[3]) * np.asarray(c, np.float32)
    acc = acc + np.float32(1.0 - acc[3]) * np.array([*opaque[:3], 1.0], np.float32)
    return acc


def test_resolve_matches_glsl_restatement(rule_run):
    """The oracle's composite equals the numpy restatement of ResolveTransparent/compute.glsl fed with the oracle's own layer
    records (its ImgRecordedColors / ImgRecordedDepths): in the kept order, and in a shuffled record order whenever no two
    depths tie, where the stable insertion sort restores the same order; a pixel with no layer keeps its bytes."""
    scene, frame, depth, color, w, h = rule_run
    out, layers, counts, lc = to.transparency(scene, frame, depth, color, layer_colors=True)
    rng = np.random.default_rng(5)
    shuffled = 0
    for y in range(h):
        for x in range(w):
            n = counts[y, x]
            if n == 0:
                assert np.array_equal(out[y, x].view(np.uint32), color[y, x].view(np.uint32))
                continue
            cols, deps = list(lc[y, x, :n]), list(layers["depth"][y, x, :n])
            want = resolve_glsl(cols, deps, color[y, x])
            assert np.array_equal(out[y, x, :3], want[:3]) and out[y, x, 3] == 1.0, (x, y)
            if n > 1 and len(set(deps)) == n:
                order = rng.permutation(n)
                assert np.array_equal(resolve_glsl([cols[i] for i in order], [deps[i] for i in order], color[y, x])[:3], want[:3])
                shuffled += 1
    assert shuffled > 0 and (counts > 1).any()


def test_glass_layer_gets_ior_reflectance():
    """A glass pane (IOR 1.5) is lit with f0 = ((1 - IOR) / (1 + IOR))^2 = 0.04, not the deferred pass's 0: with a dark, opaque
    pane over a black background and the light in its mirror direction (the highlight is mostly specular), the float64
    restatement with the real IOR agrees with the oracle within 3 %, and the same restatement at IOR 1 is off by more than half."""
    scene, cam = rule_scene()
    w, h = 48, 32
    frame = scenes.camera_frame(cam, w, h)
    glass = 6
    scene.materials["BaseColorFactor"][glass] = 0xFF0A0A0A
    scene.materials["RoughnessFactor"][glass] = 0.3
    scene.lights = scene.lights[:0]
    scene.add_light((2.6, 2.4, 3.0), (40.0, 40.0, 40.0), 0.2)
    depth = np.ones((h, w), np.float32)
    black = np.zeros((h, w, 4), np.float32)
    air_scene = copy.deepcopy(scene)
    air_scene.materials["IOR"][glass] = 1.0
    out, layers, counts = to.transparency(scene, frame, depth, black)
    want_layers, want, edge = brute_force(scene, frame, depth, black, w, h)
    _, want_air, _ = brute_force(air_scene, frame, depth, black, w, h)
    pane = np.zeros((h, w), bool)
    for (y, x), v in want_layers.items():
        pane[y, x] = len(v) == 1 and scene.blas_triangles[v[0][1]]["MeshId"] == glass and edge[y, x] >= EDGE
    assert pane.any()
    # relative to the (dim) colour itself: the highlight is sensitive to the SR11G11B10 vertex normals, hence 3 %
    rel = np.abs(out - want)[..., :3] / np.abs(want)[..., :3]
    rel_air = np.abs(out - want_air)[..., :3] / np.abs(want_air)[..., :3]
    assert rel[pane].max() <= 0.03
    assert rel_air[pane].max() > 0.5


def test_integration_doc_cone_settings_match_idkvx_header():
    """INTEGRATION.md's C# twin of IdkVxConeSettings, which idkpt_transparency's stub takes, is byte-compatible with the header."""
    import os
    import test_host_cpu as th
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    doc = open(os.path.join(repo, "INTEGRATION.md")).read()
    hdr = open(os.path.join(repo, "include", "idkvx.h")).read()
    cl, csize = th._layout(th._c_struct_fields(hdr, "IdkVxConeSettings"))
    sl, ssize = th._layout(th._cs_struct_fields(doc, "VxConeSettings"))
    assert cl == sl and csize == ssize
    assert "VxConeSettings* cone" in doc
