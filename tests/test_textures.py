"""Material textures (the constant-texture restriction of round 1 lifted): Surface.glsl:49-77 with real samplers."""
import copy

import numpy as np
import pytest

import oracle_lib as ol
import surface_ref64
from idkengine_b200 import capi, scenes


@pytest.fixture(scope="module")
def textured():
    return scenes.textured_room(threads=1)


def ref_sample(px, uv, srgb, wrap_s, wrap_t):
    """float64 GL bilinear sampling at lod 0 with the three wrap modes (tests/surface_ref64.py)."""
    return surface_ref64.sample(dict(pixels=px, srgb=srgb, wrap_s=wrap_s, wrap_t=wrap_t), uv, spread=False)[0]


@pytest.mark.parametrize("srgb", [False, True])
@pytest.mark.parametrize("wrap_s,wrap_t", [(10497, 10497), (33071, 33648), (33648, 33071)])
def test_oracle_sampling_matches_gl_rules(srgb, wrap_s, wrap_t):
    rng = np.random.default_rng(2)
    px = rng.integers(0, 256, (7, 12, 4)).astype(np.uint8)
    uv = rng.uniform(-2.5, 3.5, (4000, 2)).astype(np.float32)
    got = ol.tex_sample(px, uv, srgb, wrap_s, wrap_t)
    want = ref_sample(px, uv, srgb, wrap_s, wrap_t)
    assert np.abs(got - want).max() < 2e-5      # texel-boundary rounding of u*w in fp32 moves a sample by at most ~1e-6 texel
    centre = np.array([[(3 + 0.5) / 12, (2 + 0.5) / 7]], np.float32)   # texel centre: exactly that texel
    c = ol.tex_sample(px, centre, False, wrap_s, wrap_t)[0]
    assert np.allclose(c, px[2, 3] / 255.0, atol=1e-6)


@pytest.mark.parametrize("wrap_s,wrap_t", [(10497, 33071), (33648, 10497)])
def test_oracle_nearest_magnification(wrap_s, wrap_t):
    """IDKPT_TEX_FLAG_MAG_NEAREST (glTF magFilter 9728): at lod 0 the sample is the texel that contains (u, v) after wrapping."""
    rng = np.random.default_rng(6)
    px = rng.integers(0, 256, (5, 9, 4)).astype(np.uint8)
    uv = rng.uniform(-2.5, 3.5, (3000, 2)).astype(np.float32)
    got = ol.tex_sample(px, uv, False, wrap_s, wrap_t, flags=capi.IDKPT_TEX_FLAG_MAG_NEAREST)

    def wrap(i, n, mode):
        if mode == 33071:
            return np.clip(i, 0, n - 1)
        if mode == 33648:
            m = np.mod(i, 2 * n)
            return np.where(m < n, m, 2 * n - 1 - m)
        return np.mod(i, n)
    u, v = uv[:, 0].astype(np.float64), uv[:, 1].astype(np.float64)
    if wrap_s == 10497:
        u = (uv[:, 0] - np.floor(uv[:, 0])).astype(np.float64)
    if wrap_t == 10497:
        v = (uv[:, 1] - np.floor(uv[:, 1])).astype(np.float64)
    x = wrap(np.floor(u.astype(np.float32) * np.float32(9)).astype(int), 9, wrap_s)
    y = wrap(np.floor(v.astype(np.float32) * np.float32(5)).astype(int), 5, wrap_t)
    assert np.array_equal(got, (px[y, x].astype(np.float32) / np.float32(255.0)))
    assert len(np.unique(got.round(6), axis=0)) <= 45          # only texel values, nothing in between


def test_oracle_textures_change_the_image(textured):
    scene, cam = textured
    w, h = 80, 60
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.OutputAOVs = 1
    a = ol.path_trace(scene, frame, s, w, h)
    plain = copy.deepcopy(scene)
    for f in ("BaseColorTexture", "MetallicRoughnessTexture", "NormalTexture", "EmissiveTexture", "TransmissionTexture"):
        plain.materials[f] = 0
    b = ol.path_trace(plain, frame, s, w, h)
    assert not np.array_equal(a.albedo, b.albedo) and not np.array_equal(a.normal, b.normal)
    # an all-white texture is the reference's fallback: same image as handle 0
    white = copy.deepcopy(plain)
    hnd = white.add_texture(np.full((4, 4, 4), 255, np.uint8), srgb=True)
    white.materials["BaseColorTexture"][0] = hnd
    white.materials["EmissiveTexture"][4] = hnd
    c = ol.path_trace(white, frame, s, w, h)
    assert np.allclose(c.result, b.result, rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("sorting,lights", [(0, 1), (1, 0)])
def test_textured_path_trace_bit_exact(textured, sorting, lights):
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = textured
    w, h = 160, 120
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.OutputAOVs, s.DoRaySorting, s.CollectStats = 1, sorting, 1
    s.Gpu.DoTraceLights = lights
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(frame)
        st = [pt.Compute() for _ in range(2)]
        g = dict(result=pt.Result.copy(), albedo=pt.AlbedoTexture.copy(), normal=pt.NormalTexture.copy())
    res = np.zeros((h, w, 4), np.float32)
    alb, nrm = np.zeros_like(res), np.zeros_like(res)
    o = ol.path_trace(scene, frame, s, w, h, result=res, albedo=alb, normal=nrm)
    o = ol.path_trace(scene, frame, s, w, h, accumulated=o.accumulated, result=res, albedo=alb, normal=nrm)
    for name, img in (("result", res), ("albedo", alb), ("normal", nrm)):
        assert np.array_equal(g[name].view(np.uint32), img.view(np.uint32)), name
    assert st[-1].Rays == o.stats.Rays and st[-1].NodePairFetches == o.stats.NodePairFetches


@pytest.mark.gpu
def test_textured_shadows_bit_exact(textured):
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = textured
    w, h = 160, 120
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, _ = ol.synth_gbuffer(scene, frame, w, h)
    with PathTracer(64, 64) as pt:
        pt.SetScene(scene)
        g, _ = pt.ShadowsRayTraced(frame, depth, nrg, 0, samples=2)
    o = ol.shadows_ray_traced(scene, frame, depth, nrg, 0, samples=2)
    assert np.array_equal(g.view(np.uint32), o.view(np.uint32))
    partial = g[(g > 0.01) & (g < 0.99)]
    assert partial.size > 0                          # alpha-blended / cut-out cards give fractional visibility


@pytest.mark.gpu
def test_texture_handle_validation(textured):
    from idkengine_b200.pathtracer import PathTracer
    scene = copy.deepcopy(textured[0])
    scene.materials["NormalTexture"][0] = len(scene.textures) + 1
    with PathTracer(32, 32) as pt:
        with pytest.raises(RuntimeError, match="texture"):
            pt.SetScene(scene)
        good = textured[0]
        pt.SetScene(good)
        bad = good.materials[:1].copy()
        bad["EmissiveTexture"] = 99
        with pytest.raises(RuntimeError, match="texture"):
            pt.UpdateRange(capi.IDKPT_ARRAY_MATERIALS, 0, bad)
        ok = good.materials[:1].copy()
        ok["BaseColorTexture"] = 2
        pt.UpdateRange(capi.IDKPT_ARRAY_MATERIALS, 0, ok)


@pytest.mark.gpu
def test_set_textures_replaces_the_table(textured):
    from idkengine_b200.pathtracer import PathTracer
    scene = copy.deepcopy(textured[0])
    cam = textured[1]
    w, h = 128, 96
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    swapped = copy.deepcopy(scene)
    for t in swapped.textures:
        t["pixels"] = np.ascontiguousarray(255 - t["pixels"][::-1, :, :])
        t["pixels"][..., 3] = 255
    with PathTracer(w, h, s) as pt:
        pt.SetScene(scene); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
        pt.Compute()
        before = pt.Result.copy()
        pt.SetTextures(swapped.textures)
        assert pt.AccumulatedSamples == 0
        pt.Compute()
        after = pt.Result.copy()
        with pytest.raises(RuntimeError, match="beyond the new table"):
            pt.SetTextures(swapped.textures[:3])
    o = ol.path_trace(swapped, frame, s, w, h)
    assert np.array_equal(after.view(np.uint32), o.result.view(np.uint32))
    assert not np.array_equal(before, after)


# ------------------------------------------------------------------------------------------------ block-compressed textures (SURVEY 8f.4)
import os  # noqa: E402

import bcn_ref  # noqa: E402


def test_bcn_reference_decoders_match_pillow_golden_vectors():
    """tests/bcn_ref.py (written from the BPTC / RGTC format definitions) against tests/golden/bcn_blocks.npz, decoded by an
    independent implementation (Pillow's C decoder; generator: tests/golden/make_bcn_golden.py): every BC7 mode texel-exact;
    BC5 / BC4 (decoded to float per the RGTC formulas) within half an 8-bit step of Pillow's integer results."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bcn_blocks.npz"))
    blocks, texels = g["bc7_blocks"], g["bc7_texels"]
    seen = set()
    for blk, want in zip(blocks, texels):
        mode = 0
        while mode < 8 and not (int(blk[0]) >> mode) & 1:
            mode += 1
        got = bcn_ref.decode_bc7_block(blk)
        if mode == 8:
            assert not got.any()          # reserved mode: (0,0,0,0) by the specification (Pillow writes opaque black)
            continue
        seen.add(mode)
        assert np.array_equal(got, want), mode
    assert seen == set(range(8))
    for blk, want in zip(g["bc5_blocks"], g["bc5_texels"]):
        r, gg = bcn_ref.decode_bc4_block(blk[:8]), bcn_ref.decode_bc4_block(blk[8:])
        assert np.abs(r * 255.0 - want[..., 0]).max() < 0.87 and np.abs(gg * 255.0 - want[..., 1]).max() < 0.87
    for blk, want in zip(g["bc4_blocks"], g["bc4_texels"]):
        d = bcn_ref.decode_bc4_block(blk)
        assert np.abs(d * 255.0 - want[..., 0]).max() < 0.87
        pal_idx = [(int.from_bytes(bytes(blk[2:8]), "little") >> (3 * i)) & 7 for i in range(16)]
        for i, k in enumerate(pal_idx):      # the two stored endpoints are exact
            if k < 2:
                assert d.reshape(16)[i] == np.float32(int(blk[k])) / np.float32(255.0)


def compressed_variants(scene):
    """(scene whose textures are BC7 / BC5 / BC4 block streams as the engine's KTX2 loader provides them,
        the same scene with the textures decoded by tests/bcn_ref.py for the CPU oracle)."""
    gpu, cpu = copy.copy(scene), copy.copy(scene)
    gpu.textures, cpu.textures = [], []
    rng = np.random.default_rng(77)
    for k, t in enumerate(scene.textures):
        px = t["pixels"]
        h, w = px.shape[:2]
        common = dict(wrap_s=t["wrap_s"], wrap_t=t["wrap_t"])
        if k == 2:          # normal map -> BC5 (IDK_BC5_normal_metallicRoughness)
            blocks = bcn_ref.encode_texture("bc5", px[..., :2])
            gpu.textures.append(dict(format=capi.IDKPT_TEX_BC5_RG_UNORM, width=w, height=h, data=blocks, **common))
            cpu.textures.append(dict(format=capi.IDKPT_TEX_RG32F, width=w, height=h, data=bcn_ref.decode_texture("bc5", blocks, w, h), **common))
        elif k == 3:        # metallic-roughness -> BC7 unorm with the loader's R <- B swizzle; random blocks: every BC7 mode occurs
            blocks = rng.integers(0, 256, (((h + 3) // 4) * ((w + 3) // 4), 16), dtype=np.uint8)
            gpu.textures.append(dict(format=capi.IDKPT_TEX_BC7_UNORM, width=w, height=h, data=blocks, flags=capi.IDKPT_TEX_FLAG_R_FROM_B, **common))
            cpu.textures.append(dict(pixels=bcn_ref.decode_texture("bc7", blocks, w, h), srgb=False, flags=capi.IDKPT_TEX_FLAG_R_FROM_B, **common))
        elif k == 7:        # transmission -> BC4
            blocks = bcn_ref.encode_texture("bc4", px[..., :1])
            gpu.textures.append(dict(format=capi.IDKPT_TEX_BC4_R_UNORM, width=w, height=h, data=blocks, **common))
            cpu.textures.append(dict(format=capi.IDKPT_TEX_R32F, width=w, height=h, data=bcn_ref.decode_texture("bc4", blocks, w, h), **common))
        else:               # base colour / emissive -> BC7 sRGB; the floor's sampler asks for NEAREST magnification
            blocks = bcn_ref.encode_texture("bc7", px)
            fl = capi.IDKPT_TEX_FLAG_MAG_NEAREST if k == 0 else 0
            gpu.textures.append(dict(format=capi.IDKPT_TEX_BC7_SRGB if t["srgb"] else capi.IDKPT_TEX_BC7_UNORM, width=w, height=h, data=blocks, flags=fl, **common))
            cpu.textures.append(dict(pixels=bcn_ref.decode_texture("bc7", blocks, w, h), srgb=t["srgb"], flags=fl, **common))
    return gpu, cpu


def test_oracle_accepts_float_textures_and_swizzle(textured):
    scene, cam = textured
    gpu, cpu = compressed_variants(scene)
    w, h = 64, 48
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    a = ol.path_trace(scene, frame, s, w, h).result
    b = ol.path_trace(cpu, frame, s, w, h).result
    assert np.isfinite(b).all() and not np.array_equal(a, b)       # lossy compression + a noise metallic-roughness map change the image
    assert np.abs(a[..., :3].mean() - b[..., :3].mean()) < 0.2      # ... but it is still the same room


@pytest.mark.gpu
@pytest.mark.parametrize("sorting", [0, 1])
def test_gpu_block_compressed_textures_bit_exact(textured, sorting):
    """BC7 (sRGB and unorm + R<-B swizzle, all 8 modes through a random-block image), BC5 and BC4 textures decoded by the CUDA
    kernels at upload == the same textures decoded by the independent Python decoders and fed to the oracle uncompressed:
    images, counters, AOVs, two accumulated samples."""
    from idkengine_b200.pathtracer import PathTracer
    scene, cam = textured
    gpu, cpu = compressed_variants(scene)
    w, h = 200, 120
    frame = scenes.camera_frame(cam, w, h)
    s = capi.default_settings()
    s.RayDepth, s.DoRaySorting, s.OutputAOVs = 6, sorting, 1
    with PathTracer(w, h, s) as pt:
        pt.SetScene(gpu); pt.SetSky((0.6, 0.7, 0.9)); pt.SetFrame(frame)
        pt.CollectStats = 1
        st = [pt.Compute(), pt.Compute()]
        img, alb, nrm = pt.Result, pt.AlbedoTexture, pt.NormalTexture
    res = np.zeros((h, w, 4), np.float32)
    ralb, rnrm = np.zeros_like(res), np.zeros_like(res)
    o = ol.path_trace(cpu, frame, s, w, h, result=res, albedo=ralb, normal=rnrm)
    o2 = ol.path_trace(cpu, frame, s, w, h, accumulated=o.accumulated, result=res, albedo=ralb, normal=rnrm)
    assert st[0].Rays == o.stats.Rays and st[1].Rays == o2.stats.Rays and st[1].NodePairFetches == o2.stats.NodePairFetches
    assert np.array_equal(img, res) and np.array_equal(alb, ralb) and np.array_equal(nrm, rnrm)


@pytest.mark.gpu
def test_gpu_rejects_malformed_texture_descs(textured):
    from idkengine_b200.pathtracer import PathTracer, IdkPtError
    scene, cam = textured
    bad = copy.copy(scene)
    bad.textures = [dict(t) for t in scene.textures]
    bad.textures[0] = dict(format=42, width=8, height=8, data=np.zeros(256, np.uint8), wrap_s=10497, wrap_t=10497)
    with PathTracer(32, 32) as pt:
        with pytest.raises(IdkPtError):
            pt.SetScene(bad)
        bad.textures[0] = dict(format=capi.IDKPT_TEX_BC7_SRGB, width=8, height=8, data=np.zeros(64, np.uint8), wrap_s=10497, wrap_t=10497, flags=64)      # unknown flag bit
        with pytest.raises(IdkPtError):
            pt.SetScene(bad)
