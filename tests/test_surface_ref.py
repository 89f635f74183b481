"""Textured materials and normal mapping on the CPU oracle against the float64 restatement of tests/surface_ref64.py: the
level-0 sampler for every texel kind, flag and wrap mode; the G-buffer's attachments and the path tracer's first-hit AOVs on
a scene that reaches every rule of GetSurface, GetTBN and the two normal paths; and skinning under non-rigid joint matrices.
tests/test_surface_ref_gpu.py holds the device to the same bounds."""
import numpy as np
import pytest

import gbuffer_oracle as go
import oracle_lib as ol
import surface_ref64 as sr
from idkengine_b200 import capi, scenes
from idkengine_b200 import gpu_types as gt

W, H = 96, 64
# Bounds on how far the float32 evaluation may lie beyond the float64 range over the sample positions it allows. Measured on
# the oracle: sampler 9.6e-8 (relative), first-hit AOVs 7.3e-8 (albedo) and 6.0e-8 (normal); each bound keeps a margin.
# The G-buffer stores are compared as codes: a code must lie between the stores of the range's ends widened by NORMAL_SLACK.
SAMPLER_SLACK = 4e-7
AOV_SLACK = 1e-6
NORMAL_SLACK = 2e-6


@pytest.fixture(scope="module")
def scene():
    return sr.textured_scene()


# --------------------------------------------------------------------------------------------- the sampler
def sampler_cases():
    rng = np.random.default_rng(12)
    rgba8 = rng.integers(0, 256, (7, 13, 4)).astype(np.uint8)
    f4 = rng.uniform(-2.0, 3.0, (9, 5, 4)).astype(np.float32)
    cases = []
    for ws in (sr.REPEAT, sr.CLAMP, sr.MIRROR):
        for wt_ in (sr.REPEAT, sr.CLAMP, sr.MIRROR):
            for flags in (0, capi.IDKPT_TEX_FLAG_R_FROM_B, capi.IDKPT_TEX_FLAG_MAG_NEAREST):
                cases.append(("rgba8_srgb", dict(pixels=rgba8, srgb=True, wrap_s=ws, wrap_t=wt_, flags=flags)))
                cases.append(("rgba32f", dict(format=capi.IDKPT_TEX_RGBA32F, width=5, height=9, data=f4, wrap_s=ws, wrap_t=wt_, flags=flags)))
    return cases


def test_sampler_every_kind_flag_and_wrap(scene):
    """Dense uv sweeps, far outside [0, 1] and negative, through every texture of the scene (BC5, BC7 sRGB, BC7 + R <- B, BC4,
    RGBA8 + NEAREST) and RGBA8 sRGB / RGBA32F textures under all nine wrap pairs with each flag."""
    gpu, cpu, _ = scene
    rng = np.random.default_rng(3)
    uv = np.concatenate([rng.uniform(-9.5, 7.25, (3000, 2)),
                         np.stack(np.meshgrid(np.linspace(-2.01, 2.01, 61), np.linspace(-1.5, 1.5, 41)), -1).reshape(-1, 2)]).astype(np.float32)
    cases = [("scene%d" % k, g, c) for k, (g, c) in enumerate(zip(gpu.textures, cpu.textures))]
    cases += [(name, t, t) for name, t in sampler_cases()]
    worst, nearest_straddled, n = 0.0, 0, 0
    for name, g, c in cases:
        w, h = (c["pixels"].shape[1], c["pixels"].shape[0]) if "pixels" in c else (c["width"], c["height"])
        # texel boundaries and texel centres
        edges = np.stack(np.meshgrid(np.arange(-w, 2 * w + 1) / w, np.arange(-h, 2 * h + 1, 3) / h), -1).reshape(-1, 2)
        u = np.concatenate([uv, edges.astype(np.float32), (edges + 0.5 / np.array([w, h])).astype(np.float32)])
        got = ol.tex_sample(c, u)
        lo, hi = sr.sample(g, u)
        dev = sr.outside(got, lo, hi)
        scale = np.maximum(np.abs(lo), np.abs(hi))
        assert np.all(dev <= SAMPLER_SLACK * np.maximum(scale, 1.0)), (name, float(dev.max()))
        worst = max(worst, float((dev / np.maximum(scale, 1.0)).max()))
        if c.get("flags", 0) & capi.IDKPT_TEX_FLAG_MAG_NEAREST:
            straddled = np.any(lo != hi, 1)
            nearest_straddled += int(straddled.sum())
            # NEAREST reads a texel: away from texel boundaries the value is exactly that texel's, rounded to float32
            exact = sr.sample(g, u, spread=False)[0]
            assert np.all(np.abs(got - exact)[~straddled] <= np.spacing(np.abs(exact[~straddled]).astype(np.float32))), name
        n += len(u)
    print("sampler: %d samples over %d textures, largest relative deviation beyond the float64 range %.3g, %d NEAREST samples "
          "within rounding of a texel boundary" % (n, len(cases), worst, nearest_straddled))
    assert nearest_straddled == 4893                 # pinned: samples within rounding of a NEAREST texel boundary


def test_sampler_channel_rules(scene):
    """The kinds differ where they should: BC5 reads (R, G, 0, 1), BC4 (R, 0, 0, 1), R <- B copies blue into red."""
    gpu, cpu, _ = scene
    uv = np.random.default_rng(5).uniform(-3, 3, (500, 2)).astype(np.float32)
    bc5 = ol.tex_sample(cpu.textures[0], uv)
    assert np.all(bc5[:, 2] == 0) and np.all(bc5[:, 3] == 1) and bc5[:, :2].std() > 0.05
    bc4 = ol.tex_sample(cpu.textures[3], uv)
    assert np.all(bc4[:, 1:3] == 0) and np.all(bc4[:, 3] == 1)
    mr = ol.tex_sample(cpu.textures[2], uv)
    assert np.array_equal(mr[:, 0], mr[:, 2])
    plain = dict(cpu.textures[2], flags=0)
    assert not np.array_equal(ol.tex_sample(plain, uv)[:, 0], mr[:, 0])


# --------------------------------------------------------------------------------------------- the passes
# Pinned: (G-buffer pixels whose normal code the float64 range does not fix, edges reached) and the first hit's edges. The
# unfixed codes come from the width of the barycentric error bound the range is taken over, not from the octahedral fold alone.
GBUFFER_REACH = (654, dict(nearest=573, nearest_boundary=2, outside_unit=2541, seam=1))
FIRST_HIT_REACH = dict(nearest=586, nearest_boundary=0, outside_unit=2368, seam=1)


def reached(mesh, rng):
    """Edges the judged pixels reach: NEAREST-filtered emissive texels (meshes 1 and 3) and those whose range crosses a texel
    boundary, texcoords outside [0, 1] (wrapped), and texcoord ranges that cross an integer (a wrap seam)."""
    near = np.isin(mesh, (1, 3))
    (elo, ehi), (ulo, uhi) = rng["emissive"], rng["uv"]
    return dict(nearest=int(near.sum()), nearest_boundary=int((near & ((ehi - elo).max(1) > 1e-3)).sum()),
                outside_unit=int(((ulo < 0) | (uhi > 1)).any(1).sum()), seam=int((np.floor(ulo) != np.floor(uhi)).any(1).sum()))


def rg8(v):
    return np.floor(np.clip(v, 0, 1) * 255 + 0.5) / 255


def r11(v, c):
    return sr.ufloat64(v, 6 if c < 2 else 5, 65024.0 if c < 2 else 64512.0)


def check_gbuffer(g, pix, mesh, rng, counts, tag):
    """Every attachment of the judged pixels within the store of the float64 range (widened by the measured slack)."""
    depth, nrg, alb, mr, em, _ = (a.reshape(W * H, -1) for a in g)
    assert np.all(depth[pix, 0] < 1.0)
    lo, hi = rng["normal_oct"]
    nlo, nhi = rg8(lo - NORMAL_SLACK), rg8(hi + NORMAL_SLACK)
    bad = (nrg[pix] < nlo - 1e-7) | (nrg[pix] > nhi + 1e-7)
    assert not bad.any(), (tag, "normal", int(bad.any(1).sum()), pix[bad.any(1)][:5])
    for name, img in (("albedo", alb), ("emissive", em)):
        lo, hi = rng[name]
        for c in range(3):
            qlo, qhi = r11(lo[:, c] * (1 - 1e-6), c), r11(hi[:, c] * (1 + 1e-6), c)
            bad = (img[pix, c] < qlo) | (img[pix, c] > qhi)
            assert not bad.any(), (tag, name, c, int(bad.sum()), pix[bad][:5], img[pix, c][bad][:5], lo[bad, c][:5], hi[bad, c][:5])
    for c, name in enumerate(("metallic", "roughness")):
        lo, hi = rng[name]
        bad = (mr[pix, c] < rg8(lo - 1e-6) - 1e-7) | (mr[pix, c] > rg8(hi + 1e-6) + 1e-7)
        assert not bad.any(), (tag, name, int(bad.sum()))
    # how many stored values the float64 range does not pin (it straddles a store boundary)
    loose = int(np.any(rg8(rng["normal_oct"][0] - NORMAL_SLACK) != rg8(rng["normal_oct"][1] + NORMAL_SLACK), 1).sum())
    print("%s: %d pixels judged per mesh %s, %s, %d with a normal code the range does not pin, %d mapped normals that left "
          "N's hemisphere" % (tag, len(pix), np.bincount(mesh, minlength=6).tolist(), counts, loose, int(rng["flipped"][0].sum())))
    return loose, reached(mesh, rng)


def test_gbuffer_textured_against_float64(scene):
    gpu, cpu, cam = scene
    frame = scenes.camera_frame(cam, W, H)
    g = go.gbuffer(cpu, frame, W, H, threads=1)
    pix, mesh, rng, counts = sr.gbuffer_ref(cpu, frame, W, H)
    loose, reach = check_gbuffer(g, pix, mesh, rng, counts, "G-buffer")
    assert (loose, reach) == GBUFFER_REACH
    # every rule is reached (pinned counts)
    assert np.bincount(mesh, minlength=6).tolist() == [291, 256, 123, 317, 141, 1735]
    assert counts == dict(edge=3, alpha_ambiguous=0, discarded=115, judged=2863, back_face=317)
    # strength 4 extrapolates past the surface; the skewed tangents tilt a few strength-1 normals over as well
    assert int(rng["flipped"][0][mesh == 1].sum()) == 188 and int(rng["flipped"][0].sum()) == 199


# --------------------------------------------------------------------------------------------- the path tracer's first hit
def first_hit_aovs(cpu, frame):
    s = capi.default_settings()
    s.RayDepth, s.OutputAOVs = 1, 1
    r = ol.path_trace(cpu, frame, s, W, H)
    return r.albedo.reshape(-1, 4), r.normal.reshape(-1, 4)


def check_aovs(alb, nrm, pix, rng, tag):
    wgt = rng["weight"]
    a = product_range(rng["albedo"], wgt)
    n = product_range(rng["normal"], wgt)
    da, dn = sr.outside(alb[pix, :3], *a), sr.outside(nrm[pix, :3], *n)
    print("%s: %d pixels, largest deviation beyond the float64 range: albedo %.3g, normal %.3g" % (tag, len(pix), da.max(), dn.max()))
    assert da.max() <= AOV_SLACK and dn.max() <= AOV_SLACK, (tag, da.max(), dn.max(), pix[np.argmax(dn.max(1))])


def product_range(a, b):
    return sr.product_range(a, (b[0][:, None], b[1][:, None]))


def test_first_hit_aovs_against_float64(scene):
    gpu, cpu, cam = scene
    frame = scenes.camera_frame(cam, W, H)
    alb, nrm = first_hit_aovs(cpu, frame)
    pix, mesh, rng, counts = sr.first_hit_ref(cpu, frame, W, H)
    check_aovs(alb, nrm, pix, rng, "first hit")
    assert reached(mesh, rng) == FIRST_HIT_REACH
    print("first hit:", np.bincount(mesh, minlength=6).tolist(), counts, int(rng["flipped"][0].sum()))
    assert np.bincount(mesh, minlength=6).tolist() == [295, 260, 122, 326, 151, 1606]
    assert counts == dict(edge=3, alpha_ambiguous=0, discarded=120, judged=2760)
    assert int(rng["flipped"][0][mesh == 1].sum()) == 185 and int(rng["flipped"][0].sum()) == 196


# --------------------------------------------------------------------------------------------- skinning
def skinning_case(seed=8):
    """A cylinder's vertices (smooth normals, skewed non-unit tangents) under four joints that scale non-uniformly and shear."""
    rng = np.random.default_rng(seed)
    p, i = scenes.cylinder((0, -0.8, 0), 0.5, 1.6, 24, 8)
    from idkengine_b200.host import compute_vertex_normals
    n = compute_vertex_normals(p, i)
    t = sr._tangents(n.astype(np.float64), rng)
    u = np.zeros(len(p), gt.GpuUnskinnedVertex)
    u["JointIndices"] = rng.integers(0, 4, (len(p), 4))
    wgt = rng.uniform(0.0, 1.0, (len(p), 4)).astype(np.float32)
    u["JointWeights"] = wgt / wgt.sum(1, keepdims=True)
    u["Position"] = p
    u["Normal"] = gt.compress_sr11g11b10(n)
    u["Tangent"] = gt.compress_sr11g11b10(t)
    jm = np.zeros((6, 3, 4), np.float32)
    for j in range(4):
        a = np.diag(rng.uniform(0.4, 1.9, 3)) @ (np.eye(3) + np.triu(rng.uniform(-0.7, 0.7, (3, 3)), 1))
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        jm[2 + j, :, :3] = q @ a
        jm[2 + j, :, 3] = rng.uniform(-0.3, 0.3, 3)
    cmd = np.zeros(1, gt.IdkPtSkinningCmd)
    cmd["InputVertexOffset"], cmd["OutputVertexOffset"], cmd["JointMatricesOffset"], cmd["VertexCount"] = 0, 0, 2, len(p)
    return u, jm, cmd


def check_skinned(u, jm, vertices, tag):
    _, n64, t64 = sr.skin(u, jm, 2)
    res = []
    for name, v in (("Normal", n64), ("Tangent", t64)):
        want, amb = sr.compress_sr11g11b10(v, 4e-6)
        got = sr.unpack_sr11g11b10_codes(vertices[name])
        bad = (got != want) & ~(amb & (np.abs(got - want) <= 1))
        assert not bad.any(), (tag, name, int(bad.any(1).sum()), np.nonzero(bad.any(1))[0][:5])
        res.append(int(amb.sum()))
    print("%s: %d vertices, channels flagged half-way-ambiguous: normal %d, tangent %d" % (tag, len(u), *res))
    return res


def test_skinning_non_rigid_against_float64():
    u, jm, cmd = skinning_case()
    pos = np.zeros(len(u), gt.PackedVec3)
    vtx = np.zeros(len(u), gt.GpuVertex)
    ol.skin_vertices(u, jm, pos, vtx, cmd[0])
    amb = check_skinned(u, jm, vtx, "skinning")
    assert amb == [2, 5]                              # pinned: channels within the float32 slack of a half-way code
    # the joints are not rigid: mat3(skin) and its inverse-transpose give different normals on most vertices
    S = np.einsum("nk,nkrc->nrc", u["JointWeights"].astype(np.float64), jm[2 + u["JointIndices"]].astype(np.float64))[:, :, :3]
    n0 = sr.decompress_sr11g11b10(u["Normal"])
    a = sr.unit(np.einsum("nrc,nc->nr", S, n0))
    b = sr.unit(np.einsum("nrc,nc->nr", np.linalg.inv(S).transpose(0, 2, 1), n0))
    assert (np.linalg.norm(a - b, axis=1) > 0.05).mean() > 0.9
