"""Inputs and checks the raster-pass tests share: bitwise image comparison, the lit Cornell box and its point shadows, the
deferred-lighting scenes with their seeded G-buffer, the transparency rule scene and the VXGI grids written by hand."""
import copy
import functools

import numpy as np

import oracle_lib as ol
import vxgi_ref64 as r
from idkengine_b200 import capi, gpu_types as gt, scenes, vxgi
from idkengine_b200.host import Model, Scene
from idkengine_b200.pathtracer import PathTracer

JITTER = (0.0123, -0.0311)
GRID_MIN, GRID_MAX = (-1.2, -0.2, -1.2), (1.2, 2.2, 1.2)          # the Cornell box's VXGI grid
TEX_GRID_MIN, TEX_GRID_MAX = (-3.1, -0.1, -3.1), (3.1, 4.1, 3.1)  # the textured room's
CORNELL_LIGHTS = [((0.0, 1.6, 0.3), (6.0, 5.5, 5.0), 0.2), ((-0.6, 0.5, 0.6), (0.5, 0.8, 3.0), 0.1),
                  ((0.5, 1.2, 0.8), (1.0, 0.4, 0.3), 0.15)]


# ------------------------------------------------------------------------------------------------ bitwise comparison
def canon(a):
    """The bits of a float32 or float16 array (float16 also as its uint16 bits) with every NaN set to one payload: the device
    and x86 produce different NaN payloads."""
    a = np.ascontiguousarray(a)
    if a.dtype.itemsize == 2:
        u = a.view(np.uint16).copy()
        u[((u & 0x7C00) == 0x7C00) & ((u & 0x03FF) != 0)] = 0x7E00
        return u
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).copy()
    u[((u & 0x7F800000) == 0x7F800000) & ((u & 0x007FFFFF) != 0)] = 0x7FC00000
    return u


def assert_bits(got, want):
    """got equals want bit for bit up to NaN payloads."""
    bad = canon(got) != canon(want)
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} values differ"


# ------------------------------------------------------------------------------------------------ lit scenes
def lit_cornell(lights=2):
    """(scene, camera): the Cornell box with the first `lights` of CORNELL_LIGHTS."""
    scene, cam = scenes.cornell_1k(threads=1)
    for light in CORNELL_LIGHTS[:lights]:
        scene.add_light(*light)
    return scene, cam


def crossed_shadows(scene, near0, near1):
    """Shadows for lights 0 and 1 with crossed indices (light 0 uses shadow 1 and the other way round; a third light has none):
    shadow 0 at light 1 with near plane near0, shadow 1 at light 0 with near1, both with far plane 60."""
    scene.lights["PointShadowIndex"][:] = [1, 0, -1][:len(scene.lights)]
    return scenes.point_shadows([(scene.lights[1]["Position"], near0, 60.0, 1), (scene.lights[0]["Position"], near1, 60.0, 0)])


def lit_cornell_shadowed():
    """(scene, shadows) for the voxeliser's PCF lookup: crossed indices, both records with LightIndex 0."""
    scene, _ = lit_cornell(2)
    scene.lights["PointShadowIndex"][:] = [1, 0]
    return scene, scenes.point_shadows([(scene.lights[1]["Position"], 0.1, 60.0, 0), (scene.lights[0]["Position"], 0.2, 60.0, 0)])


@functools.lru_cache(maxsize=None)
def deferred_setup(which):
    """(scene, camera, shadows) the deferred-lighting passes light: two shadowed lights (the second shadow belongs to an earlier
    light) and one without a shadow."""
    if which == "cornell":
        scene, cam = lit_cornell(3)
        return scene, cam, crossed_shadows(scene, 0.1, 0.2)
    if which == "multi_blas_tlas":
        scene, cam = scenes.multi_blas(threads=1)
        scene.build_tlas()
        p = (0.2, 1.9, 0.8)
    else:
        scene, cam = scenes.atrium(20000, threads=1)
        p = (0.0, 3.0, 0.5)
    if len(scene.lights) == 0:
        scene.add_light((1.0, 2.0, -0.5), (3.0, 3.0, 3.0), 0.2)
    scene.add_light(p, (20.0, 18.0, 15.0), 0.3)
    scene.add_light((-0.5, 1.0, 1.0), (2.0, 1.0, 0.5), 0.1)
    n = len(scene.lights)
    scene.lights["PointShadowIndex"][:] = -1
    scene.lights["PointShadowIndex"][n - 2] = 0
    scene.lights["PointShadowIndex"][0] = 1
    return scene, cam, scenes.point_shadows([(p, 0.3, 60.0, n - 2), (scene.lights[0]["Position"], 0.3, 60.0, 0)])


RULE_CAM = dict(position=(0.0, 1.0, 3.0), view_dir=(0.0, 0.0, -1.0), fov_y_deg=60.0)


def rule_scene():
    """Every rule in view: an opaque back wall with a blended pane behind it (fails depth); a single-sided blended quad seen from
    behind (culled) and a double-sided one (kept, normal flipped); a textured blended card with alpha-0 and partial-alpha texels;
    a blended quad crossing the near plane; blended panes over the background; a mirrored blended instance; two coplanar
    duplicated quads with different materials (an exact depth tie); and a stack of 13 panes (the 10-layer cap)."""
    specs = [dict(color=(0.7, 0.7, 0.7), roughness=0.6),                               # 0 opaque back wall
             dict(color=(0.9, 0.2, 0.2, 0.5), cutoff=2.0),                             # 1 blended, behind the wall
             dict(color=(0.9, 0.1, 0.1, 0.6), cutoff=2.0),                             # 2 single-sided, seen from behind
             dict(color=(0.1, 0.9, 0.1, 0.4), cutoff=2.0, metallic=0.5, emissive=(0.5, 0.25, 0.0)),  # 3 double-sided, from behind
             dict(color=(1.0, 1.0, 1.0, 1.0), cutoff=2.0),                             # 4 textured card (alpha 0 / partial texels)
             dict(color=(0.3, 0.8, 0.8, 0.5), cutoff=2.0),                             # 5 crosses the near plane
             dict(color=(0.2, 0.4, 0.9, 0.3), cutoff=2.0, ior=1.5, roughness=0.1),     # 6 glass over the background
             dict(color=(0.6, 0.3, 0.8, 0.5), cutoff=2.0),                             # 7 mirrored instance
             dict(color=(0.9, 0.9, 0.1, 0.5), cutoff=2.0),                             # 8 coplanar tie, material A
             dict(color=(0.1, 0.9, 0.9, 0.5), cutoff=2.0),                             # 9 coplanar tie, material B
             dict(color=(0.8, 0.5, 0.2, 0.2), cutoff=2.0, ior=1.33)]                   # 10 the 13-pane stack
    scene = Scene()
    t_card = scene.add_texture(scenes._checker(32, 2, (200, 120, 60), (60, 120, 200), alpha_a=0, alpha_b=128, seed=5), srgb=True)
    meshes, mats = scenes._materials(specs)
    mats["IsDoubleSided"][3] = mats["IsDoubleSided"][5] = 1
    mats["BaseColorTexture"][4] = t_card

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
    scene.add(model([ccw(-1.5, 0.5, -1, 1.6, -2)], 0),
              model([ccw(-1.2, 0.0, 0.0, 1.0, -2.5)], 1),
              model([cw(-1.4, -0.6, 0.2, 0.9, -1)], 2),
              model([cw(0.6, 1.4, 0.2, 0.9, -1)], 3),
              model([ccw(-1.4, -0.6, 1.2, 1.8, -1.2)], 4, uv=uv),
              model([([0.05, 0.85, 2.95], [0.35, 0.85, 2.4], [0.35, 1.15, 2.4], [0.05, 1.15, 2.95])], 5),
              model([ccw(0.7, 1.9, 1.2, 2.2, -3.0)], 6),
              model([cw(0.6, 1.4, -0.7, -0.1, -1)], 7, matrix=np.diag([-1.0, 1.0, 1.0, 1.0])),
              model([ccw(-0.4, 0.4, 1.9, 2.3, -0.8)], 8),
              model([ccw(-0.4, 0.4, 1.9, 2.3, -0.8)], 9),
              model([ccw(-0.3, 0.3, 0.3, 0.9, -0.3 - 0.1 * k) for k in range(13)], 10), threads=1)
    scene.add_light((0.5, 2.0, 0.5), (4.0, 3.5, 3.0), 0.2)
    return scene, RULE_CAM


# ------------------------------------------------------------------------------------------------ G-buffer and deferred inputs
def gbuffer(pt, scene, frame, w, h, seed=1):
    """(depth, normal, albedo, metallic/roughness, emissive) from the first hit, seeded albedo / emissive, and hand-made pixels
    in row 0: sky (depth 1), roughness 0, metallic 0, metallic 1, a normal facing away from every light."""
    depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, w, h)
    rng = np.random.default_rng(seed)
    albedo = rng.random((h, w, 3), dtype=np.float32)
    emissive = np.where(rng.random((h, w, 1)) < 0.2, rng.random((h, w, 3)) * 0.5, 0.0).astype(np.float32)
    depth, nrg, mr = depth.copy(), nrg.copy(), mr.copy()
    if w >= 5 and h >= 1:
        depth[0, 0] = 1.0
        mr[0, 1, 1] = 0.0
        mr[0, 2, 0] = 0.0
        mr[0, 3, 0] = 1.0
        f = frame[0] if frame.ndim else frame
        M = np.asarray(f["InvProjView"], np.float64).reshape(4, 4)
        d = depth[0, 4] if depth[0, 4] != 1.0 else 0.99
        depth[0, 4] = d
        wp = np.array([(4.5 / w) * 2 - 1, (0.5 / h) * 2 - 1, d, 1.0]) @ M
        frag = wp[:3] / wp[3]
        to_lights = np.asarray(scene.lights["Position"], np.float64) - frag
        away = -np.sum(to_lights / np.linalg.norm(to_lights, axis=1, keepdims=True), 0)
        nrg[0, 4] = vxgi.encode_unit_vec(away / np.linalg.norm(away))
    return depth, nrg, albedo, mr, emissive


def deferred_settings(mode, is_ssao, is_vxgi):
    return capi.IdkPtDeferredSettings(mode, int(is_ssao), int(is_vxgi))


def rt_images(pt, scene, frame, g, shadows):
    """Shadow k's visibility image from idkpt_shadows_ray_traced for the light whose PointShadowIndex is k."""
    out = []
    for k in range(len(shadows)):
        li = int(np.nonzero(scene.lights["PointShadowIndex"] == k)[0][0])
        out.append(pt.ShadowsRayTraced(frame, g[0], g[1], li, samples=2, jitter=JITTER)[0])
    return out


@functools.lru_cache(maxsize=None)
def cone_trace_gi(W, H):
    """The cone-traced indirect light of deferred_setup("cornell") at W x H, voxelised with the lights unshadowed."""
    scene, cam, _ = deferred_setup("cornell")
    frame = scenes.camera_frame(cam, W, H)
    with PathTracer(16, 16) as pt:
        pt.SetScene(scene)
        g = gbuffer(pt, scene, frame, W, H)
    unshadowed = copy.deepcopy(scene)                                           # the voxeliser's lights without shadow maps
    unshadowed.lights["PointShadowIndex"][:] = -1
    with vxgi.Voxelizer(32, GRID_MIN, GRID_MAX) as vx:
        vx.SetScene(unshadowed)
        vx.Render()
        return vx.ConeTrace(frame, g[0], g[1], g[3])[0]


# ------------------------------------------------------------------------------------------------ VXGI grids
FILLS = ["random", "sparse", "zeros", "subnormal", "near_max", "inf"]


def level0_fill(shape, fill, seed=0):
    """A synthetic level 0 (float16 [d, h, w, 4]) of one of FILLS."""
    w, h, d = shape
    rng = np.random.default_rng(seed + 7919 * FILLS.index(fill))
    n = (d, h, w, 4)
    if fill == "random":
        return rng.uniform(0.0, 4.0, n).astype(np.float16)
    if fill == "sparse":                     # voxeliser-like: alpha 0 or 1, rgb only where occupied
        occ = rng.random((d, h, w)) < 0.15
        out = np.zeros(n, np.float16)
        out[occ, :3] = rng.uniform(0.0, 20.0, (int(occ.sum()), 3)).astype(np.float16)
        out[occ, 3] = 1.0
        return out
    if fill == "zeros":
        return np.zeros(n, np.float16)
    if fill == "subnormal":                  # every float16 subnormal is a bit pattern 1 .. 1023
        return rng.integers(0, 1024, n).astype(np.uint16).view(np.float16)
    if fill == "near_max":
        return rng.uniform(60000.0, 65504.0, n).astype(np.float16)
    if fill == "inf":
        out = rng.uniform(0.0, 8.0, n).astype(np.float16)
        out[rng.random(n) < 0.02] = np.inf
        return out
    raise ValueError(fill)


def synthetic_chain(ci, kind, seed=0):
    """A mip chain (levels, raw) from a synthetic level 0: 'sparse' (voxeliser-like occupancy), 'dense' (random alpha)."""
    w, h, d = ci.Width, ci.Height, ci.Depth
    if kind == "sparse":
        level0 = level0_fill((w, h, d), "sparse", seed)
        level0[..., :3] = (level0[..., :3].astype(np.float32) * 0.1).astype(np.float16)
    else:
        rng = np.random.default_rng(seed)
        level0 = np.concatenate([rng.uniform(0, 0.3, (d, h, w, 3)), rng.uniform(0, 0.2, (d, h, w, 1))], -1).astype(np.float16)
    return ol.vx_mipmap(ci, level0)


def write_level(vx, level, data):
    """Copies a float16 [d, h, w, 4] level into the context's grid with torch."""
    import torch
    from idkengine_b200 import multigpu
    ptr, nbytes = vx.LevelDevicePtr(level)
    data = np.ascontiguousarray(data, np.float16).reshape(-1).view(np.int16)
    assert nbytes == data.nbytes
    vx.ReadLevel(len(vx.sizes) - 1)          # synchronises the context's stream (the grid's initial clear runs on it)
    torch.as_tensor(multigpu.DeviceArray(ptr, (data.size,), "<i2"), device="cuda").copy_(torch.from_numpy(data))
    torch.cuda.synchronize()


def check_voxelized(level0, frags, v, max_ambiguous_fraction):
    """A voxelised level 0 and its fragment count against voxelize64's result v: occupancy equal on every unambiguous voxel,
    rgb there within 1 ulp, at most max_ambiguous_fraction of the occupied voxels ambiguous, and the fragment counts apart
    by no more than the ambiguous samples."""
    occ = level0[..., 3] != 0
    assert np.all(level0[occ][:, 3] == 1.0)
    clear = ~v["ambiguous"]
    assert np.array_equal(occ & clear, v["written"] & clear)
    both = occ & v["written"] & clear
    u = r.half_ulp_distance(level0[both][:, :3], v["level0"][both][:, :3])
    assert u.max() <= 1.0, u.max()
    amb = int((v["ambiguous"] & occ).sum())
    assert amb <= max_ambiguous_fraction * occ.sum(), (amb, int(occ.sum()))
    assert abs(frags - v["fragments"]) <= v["ambiguous_samples"], (frags, v["fragments"], v["ambiguous_samples"])


# ------------------------------------------------------------------------------------------------ skinned scenes
def skinning_setup(scene, blas_id, joints=6, seed=3):
    """Unskinned vertices for the vertex range of one BLAS (random joints / weights) + joint matrices of a gentle deformation."""
    rng = np.random.default_rng(seed)
    d = scene.blas_descs[blas_id]
    tris = scene.blas_triangles[d["TriangleOffset"]:d["TriangleOffset"] + d["TriangleCount"]]
    idx = np.concatenate([tris["X"], tris["Y"], tris["Z"]])
    v0, v1 = int(idx.min()), int(idx.max()) + 1
    n = v1 - v0
    u = np.zeros(n, gt.GpuUnskinnedVertex)
    u["JointIndices"] = rng.integers(0, joints, (n, 4))
    w = rng.uniform(0.0, 1.0, (n, 4)).astype(np.float32)
    u["JointWeights"] = w / w.sum(1, keepdims=True)
    u["Position"][:, 0] = scene.positions["x"][v0:v1]
    u["Position"][:, 1] = scene.positions["y"][v0:v1]
    u["Position"][:, 2] = scene.positions["z"][v0:v1]
    u["Normal"] = scene.vertices["Normal"][v0:v1]
    u["Tangent"] = scene.vertices["Tangent"][v0:v1]
    jm = np.zeros((joints + 2, 3, 4), np.float32)          # two unused leading matrices: exercises JointMatricesOffset
    for j in range(joints):
        a = rng.uniform(-0.25, 0.25)
        c, s = np.cos(a), np.sin(a)
        jm[2 + j, :, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], np.float32) * rng.uniform(0.9, 1.2)
        jm[2 + j, :, 3] = rng.uniform(-0.15, 0.15, 3)
    cmd = np.zeros(1, gt.IdkPtSkinningCmd)
    cmd["InputVertexOffset"], cmd["OutputVertexOffset"], cmd["JointMatricesOffset"], cmd["VertexCount"] = 0, v0, 2, n
    return u, jm, cmd
