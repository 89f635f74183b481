"""ctypes wrapper of oracle/liboracle.so -- imported by tests/, __graft_entry__.smoke() and bench.py's CPU legs only."""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "oracle"))

from idkengine_b200 import capi, gpu_types as gt  # noqa: E402

_lib = None


def lib():
    global _lib
    if _lib is None:
        import importlib.util
        spec = importlib.util.spec_from_file_location("oracle_build", os.path.join(REPO, "oracle", "build.py"))
        ob = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ob)
        path = ob.LIBORACLE if os.path.exists(ob.LIBORACLE) else ob.build()
        try:
            path = ob.build()
        except Exception:
            pass
        L = ctypes.CDLL(path)
        P = ctypes.POINTER
        vp, u64, i32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int32
        L.oracle_trace_rays.restype = i32
        L.oracle_trace_rays.argtypes = [P(capi.IdkPtSceneDesc), vp, u64, i32, vp, i32]
        L.oracle_brute_force.restype = i32
        L.oracle_brute_force.argtypes = [P(capi.IdkPtSceneDesc), vp, u64, vp, i32]
        L.oracle_cpu_intersect.restype = ctypes.c_double
        L.oracle_cpu_intersect.argtypes = [P(capi.IdkPtSceneDesc), vp, u64, vp, i32]
        L.oracle_gui_test_rays.restype = None
        L.oracle_gui_test_rays.argtypes = [vp, i32, i32, i32, i32, vp]
        L.oracle_path_trace.restype = i32
        L.oracle_path_trace.argtypes = [P(capi.IdkPtSceneDesc), P(capi.IdkPtSkyDesc), vp, P(capi.IdkPtSettings),
                                        i32, i32, i32, i32, i32, P(ctypes.c_uint32), vp, vp, vp, vp,
                                        P(capi.IdkPtStats), i32]
        L.oracle_det_sincos.argtypes = [vp, u64, vp, vp]
        L.oracle_det_exp.argtypes = [vp, u64, vp]
        L.oracle_encode_decode.argtypes = [vp, u64, vp, vp]
        L.oracle_pcg.restype = ctypes.c_uint32
        L.oracle_pcg.argtypes = [ctypes.c_uint32, P(ctypes.c_uint32)]
        _lib = L
    return _lib


def default_threads():
    return max(1, min(os.cpu_count() or 1, 64))


def make_rays(origins, directions, tmax=3.4028235e+38):
    r = np.zeros(len(origins), gt.IdkPtRay)
    r["Origin"] = origins
    r["Direction"] = directions
    r["TMax"] = tmax
    return r


def trace_rays(scene, rays, trace_lights=False, threads=None):
    d, keep = capi.scene_desc(scene)
    out = np.zeros(len(rays), gt.IdkPtHit)
    lib().oracle_trace_rays(ctypes.byref(d), rays.ctypes.data, len(rays), int(trace_lights), out.ctypes.data,
                            threads or default_threads())
    return out


def trace_rays_any(scene, rays, trace_lights=False, threads=None):
    d, keep = capi.scene_desc(scene)
    out = np.zeros(len(rays), gt.IdkPtHit)
    L = lib()
    L.oracle_trace_rays_any.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32]
    L.oracle_trace_rays_any(ctypes.byref(d), rays.ctypes.data, len(rays), int(trace_lights), out.ctypes.data, threads or default_threads())
    return out


def shadows_ray_traced(scene, frame, depth, normal_rg, light_index, samples=1, noise_index=0, jitter=(0.0, 0.0), visibility=None, threads=None):
    d, keep = capi.scene_desc(scene)
    h, w = depth.shape
    depth = np.ascontiguousarray(depth, np.float32)
    nrg = np.ascontiguousarray(normal_rg, np.float32)
    vis = np.zeros((h, w), np.float32) if visibility is None else np.ascontiguousarray(visibility, np.float32)
    jit = np.array(jitter, np.float32)
    L = lib()
    L.oracle_shadows_ray_traced.restype = ctypes.c_int32
    L.oracle_shadows_ray_traced.argtypes = [ctypes.POINTER(capi.IdkPtSceneDesc), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
                                            ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32]
    rc = L.oracle_shadows_ray_traced(ctypes.byref(d), frame.ctypes.data, depth.ctypes.data, nrg.ctypes.data, w, h, light_index, samples, noise_index,
                                     jit.ctypes.data, vis.ctypes.data, threads or default_threads())
    assert rc == 0
    return vis


def skin_vertices(unskinned, joint_matrices, positions, vertices, cmd):
    """In-place oracle_skin_vertices on numpy arrays (positions: PackedVec3, vertices: GpuVertex)."""
    L = lib()
    L.oracle_skin_vertices.restype = None
    L.oracle_skin_vertices.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_uint32] * 4
    jm = np.ascontiguousarray(joint_matrices, np.float32)
    L.oracle_skin_vertices(unskinned.ctypes.data, jm.ctypes.data, positions.ctypes.data, vertices.ctypes.data, int(cmd["InputVertexOffset"]),
                           int(cmd["OutputVertexOffset"]), int(cmd["JointMatricesOffset"]), int(cmd["VertexCount"]))


def blas_refit(scene, blas_id):
    """In-place BLAS.Refit of scene.blas_nodes for one BLAS from scene.positions."""
    L = lib()
    L.oracle_blas_refit.restype = None
    L.oracle_blas_refit.argtypes = [ctypes.c_void_p] * 4
    desc = np.ascontiguousarray(scene.blas_descs[blas_id:blas_id + 1])
    L.oracle_blas_refit(scene.blas_nodes.ctypes.data, desc.ctypes.data, scene.blas_triangles.ctypes.data, scene.positions.ctypes.data)


def post_process(result, settings=None, want_bloom=False, threads=None):
    """oracle_post_process on an rgba32f image [H, W, 4] -> rgba8 [H, W, 4] (and Bloom.Result [H//2, W//2, 3])."""
    st = settings if settings is not None else capi.default_post_settings()
    h, w = result.shape[:2]
    result = np.ascontiguousarray(result, np.float32)
    out = np.zeros((h, w, 4), np.uint8)
    bloom = np.zeros((max(h // 2, 1), max(w // 2, 1), 3), np.float32)
    L = lib()
    L.oracle_post_process.restype = ctypes.c_int32
    L.oracle_post_process.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(capi.IdkPtPostSettings), ctypes.c_void_p,
                                      ctypes.c_void_p, ctypes.c_int32]
    rc = L.oracle_post_process(result.ctypes.data, w, h, ctypes.byref(st), out.ctypes.data, bloom.ctypes.data if want_bloom else None,
                               threads or default_threads())
    assert rc == 0
    return (out, bloom) if want_bloom else out


def tex_sample(pixels, uv, srgb=False, wrap_s=10497, wrap_t=10497, flags=0):
    px = np.ascontiguousarray(pixels, np.uint8)
    uv = np.ascontiguousarray(uv, np.float32)
    t = capi.IdkPtTextureDesc(px.ctypes.data, px.shape[1], px.shape[0], 1 if srgb else 0, wrap_s, wrap_t, flags)
    out = np.zeros((len(uv), 4), np.float32)
    L = lib()
    L.oracle_tex_sample.restype = None
    L.oracle_tex_sample.argtypes = [ctypes.POINTER(capi.IdkPtTextureDesc), ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p]
    L.oracle_tex_sample(ctypes.byref(t), uv.ctypes.data, len(uv), out.ctypes.data)
    return out


def brute_force(scene, rays, threads=None):
    d, keep = capi.scene_desc(scene)
    out = np.zeros(len(rays), gt.IdkPtHit)
    lib().oracle_brute_force(ctypes.byref(d), rays.ctypes.data, len(rays), out.ctypes.data, threads or default_threads())
    return out


def cpu_intersect(scene, rays, threads=None, want_hits=True):
    d, keep = capi.scene_desc(scene)
    out = np.zeros(len(rays), gt.IdkPtHit) if want_hits else None
    secs = lib().oracle_cpu_intersect(ctypes.byref(d), rays.ctypes.data, len(rays),
                                      out.ctypes.data if want_hits else None, threads or default_threads())
    return out, secs


def gui_test_rays(frame, width, height, y0=0, y1=None):
    y1 = height if y1 is None else y1
    out = np.zeros((y1 - y0) * width, gt.IdkPtRay)
    lib().oracle_gui_test_rays(frame.ctypes.data, width, height, y0, y1, out.ctypes.data)
    return out


def primary_rays(frame, width, height, stride=1):
    """Pinhole rays through pixel centres (test inputs for the stand-alone traversal; not a reference code path)."""
    rays = gui_test_rays(frame, width, height)
    return rays[::stride].copy()


class PathTraceResult:
    pass


def path_trace(scene, frame, settings, width, height, sky=(0.6, 0.7, 0.9), tile=(8, 0, 1), accumulated=0,
               result=None, albedo=None, normal=None, want_rays=True, threads=None):
    d, keep = capi.scene_desc(scene)
    sk = capi.sky_desc(sky)
    res = np.zeros((height, width, 4), np.float32) if result is None else result
    alb = np.zeros((height, width, 4), np.float32) if albedo is None else albedo
    nrm = np.zeros((height, width, 4), np.float32) if normal is None else normal
    rays = np.zeros(width * height, gt.GpuWavefrontRay) if want_rays else None
    acc = ctypes.c_uint32(accumulated)
    stats = capi.IdkPtStats()
    rc = lib().oracle_path_trace(ctypes.byref(d), ctypes.byref(sk), frame.ctypes.data, ctypes.byref(settings),
                                 width, height, tile[0], tile[1], tile[2], ctypes.byref(acc),
                                 res.ctypes.data, alb.ctypes.data, nrm.ctypes.data,
                                 rays.ctypes.data if want_rays else None, ctypes.byref(stats),
                                 threads or default_threads())
    assert rc == 0, rc
    out = PathTraceResult()
    out.result, out.albedo, out.normal, out.rays, out.accumulated, out.stats = res, alb, nrm, rays, acc.value, stats
    return out


# ----------------------------------------------------------------------------------------------- VXGI
def _vx_declare():
    L = lib()
    from idkengine_b200 import vxgi
    P = ctypes.POINTER
    vp, u64, i32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int32
    L.oracle_vx_voxelize.restype = i32
    L.oracle_vx_voxelize.argtypes = [P(capi.IdkPtSceneDesc), P(vxgi.IdkVxCreateInfo), vp, u64, P(u64), i32]
    L.oracle_vx_cone_trace.restype = i32
    L.oracle_vx_cone_trace.argtypes = [P(vxgi.IdkVxCreateInfo), vp, vp, P(vxgi.IdkVxConeSettings), vp, vp, vp, i32, i32, vp, vp, P(u64), i32]
    L.oracle_vx_mipmap.restype = i32
    L.oracle_vx_mipmap.argtypes = [P(vxgi.IdkVxCreateInfo), vp, i32]
    L.oracle_half_roundtrip.argtypes = [vp, u64, vp, vp]
    L.oracle_det_log2.argtypes = [vp, u64, vp]
    return L


def _vx_split(raw, sizes):
    levels, off = [], 0
    for (w, h, dd) in sizes:
        k = w * h * dd * 4
        levels.append(raw[off:off + k].view(np.float16).reshape(dd, h, w, 4))
        off += k
    return levels


def vx_mipmap(ci, level0, threads=None):
    """Levels 1 .. n-1 of the mip chain built from a caller-supplied level 0 (float16 [d, h, w, 4]).
    Returns (list of float16 [d, h, w, 4] arrays per level, concatenated raw uint16 chain)."""
    from idkengine_b200 import vxgi
    L = _vx_declare()
    sizes = vxgi.level_sizes(ci)
    w, h, d = sizes[0]
    level0 = np.ascontiguousarray(level0, np.float16)
    assert level0.shape == (d, h, w, 4), level0.shape
    raw = np.zeros(sum(a * b * c for a, b, c in sizes) * 4, np.uint16)
    raw[:level0.size] = level0.reshape(-1).view(np.uint16)
    n = L.oracle_vx_mipmap(ctypes.byref(ci), raw.ctypes.data, threads or default_threads())
    assert n == len(sizes), n
    return _vx_split(raw, sizes), raw


def vx_voxelize(scene, ci, threads=None, raster_rule=0):
    """Returns (list of float16 [d,h,w,4] arrays per level, concatenated raw uint16 chain, fragment count).
    raster_rule: 0 = the product's coverage rule (what the GPU kernels implement), 1 = the GL model (1/256-pixel snapping +
    top-left fill rule) used only to measure the distance between the two."""
    from idkengine_b200 import vxgi
    L = _vx_declare()
    L.oracle_vx_set_raster_rule.restype = None
    L.oracle_vx_set_raster_rule.argtypes = [ctypes.c_int]
    L.oracle_vx_set_raster_rule(int(raster_rule))
    sizes = vxgi.level_sizes(ci)
    total = sum(w * h * d for w, h, d in sizes)
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    try:
        n = L.oracle_vx_voxelize(ctypes.byref(d), ctypes.byref(ci), raw.ctypes.data, total, ctypes.byref(frags), threads or default_threads())
    finally:
        L.oracle_vx_set_raster_rule(0)
    assert n == len(sizes), n
    return _vx_split(raw, sizes), raw, frags.value


def vx_cone_trace(ci, raw_chain, frame, settings, depth, normal_rg, metal_rough, sky=(0.6, 0.7, 0.9), threads=None):
    L = _vx_declare()
    h, w = depth.shape
    out = np.zeros((h, w, 4), np.float32)
    skyc = np.array(sky, np.float32)
    steps = ctypes.c_uint64()
    depth = np.ascontiguousarray(depth, np.float32)
    nrg = np.ascontiguousarray(normal_rg, np.float32)
    mr = np.ascontiguousarray(metal_rough, np.float32)
    rc = L.oracle_vx_cone_trace(ctypes.byref(ci), raw_chain.ctypes.data, frame.ctypes.data, ctypes.byref(settings), depth.ctypes.data,
                                nrg.ctypes.data, mr.ctypes.data, w, h, skyc.ctypes.data, out.ctypes.data, ctypes.byref(steps),
                                threads or default_threads())
    assert rc == 0
    return out, steps.value


def synth_gbuffer(scene, frame, width, height):
    """G-buffer for the cone tracer synthesised from the path tracer's first hit (SURVEY 8d config 5):
    depth = ProjView-projected hit point (1.0 = sky), normal = octahedral geometric normal facing the camera,
    metallic/roughness from the hit material."""
    rays = gui_test_rays(frame, width, height)
    # pixel centres instead of Gui.Test's pixel corners
    hits = trace_rays(scene, rays)
    hit = hits["TriangleId"] != 0xFFFFFFFF
    o = rays["Origin"].astype(np.float64)
    d = rays["Direction"].astype(np.float64)
    pos = o + d * hits["T"][:, None].astype(np.float64)
    pv = frame["ProjView"][0].astype(np.float64).reshape(4, 4)      # OpenTK rows: clip = [p,1] @ pv
    clip = np.concatenate([pos, np.ones((len(pos), 1))], 1) @ pv
    depth = np.where(hit, clip[:, 2] / clip[:, 3], 1.0).astype(np.float32)
    depth = np.where(hit & (depth >= 1.0), np.float32(0.999999), depth)
    tri = scene.blas_triangles[np.where(hit, hits["TriangleId"], 0)]
    P = scene.positions
    p0 = np.stack([P["x"][tri["X"]], P["y"][tri["X"]], P["z"][tri["X"]]], 1).astype(np.float64)
    p1 = np.stack([P["x"][tri["Y"]], P["y"][tri["Y"]], P["z"][tri["Y"]]], 1).astype(np.float64)
    p2 = np.stack([P["x"][tri["Z"]], P["y"][tri["Z"]], P["z"][tri["Z"]]], 1).astype(np.float64)
    n = np.cross(p1 - p0, p2 - p0)
    inv = scene.mesh_transforms["InvModelMatrix"][hits["MeshTransformId"]][:, :, :3].astype(np.float64)   # [N,3,3]
    n = np.einsum("nji,nj->ni", inv, n)                                # transpose(inv) * n
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-30)
    n = np.where((np.sum(n * d, 1) > 0)[:, None], -n, n)
    # EncodeUnitVec (Compression.glsl:54-61)
    m = n / np.sum(np.abs(n), 1, keepdims=True)
    wrap = (1.0 - np.abs(m[:, [1, 0]])) * np.where(m[:, :2] < 0, -1.0, 1.0)
    xy = np.where((m[:, 2] > 0)[:, None], m[:, :2], wrap)
    nrg = (xy * 0.5 + 0.5).astype(np.float32)
    mesh = scene.meshes[tri["MeshId"]]
    mat = scene.materials[mesh["MaterialId"]]
    mr = np.stack([np.clip(mat["MetallicFactor"] + mesh["SpecularBias"], 0, 1), np.clip(mat["RoughnessFactor"] + mesh["RoughnessBias"], 0, 1)], 1).astype(np.float32)
    return depth.reshape(height, width), nrg.reshape(height, width, 2), mr.reshape(height, width, 2)


def denoise(result, albedo, normal, settings=None, threads=None):
    """oracle_denoise: the guided a-trous filter of csrc/idk_post.cuh on rgba32f images [H, W, 4] -> denoised [H, W, 4]."""
    st = settings if settings is not None else capi.default_denoise_settings()
    h, w = result.shape[:2]
    r, a, n = (np.ascontiguousarray(x, np.float32) for x in (result, albedo, normal))
    out = np.zeros((h, w, 4), np.float32)
    L = lib()
    L.oracle_denoise.restype = ctypes.c_int32
    L.oracle_denoise.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(capi.IdkPtDenoiseSettings),
                                 ctypes.c_void_p, ctypes.c_int32]
    rc = L.oracle_denoise(r.ctypes.data, a.ctypes.data, n.ctypes.data, w, h, ctypes.byref(st), out.ctypes.data, threads or default_threads())
    assert rc == 0
    return out


def sample_sky(faces, dirs):
    """texture(samplerCube, dir).rgb for float32 faces [6, N, N, 4] and directions [M, 3]."""
    sk = capi.sky_desc((0.0, 0.0, 0.0), faces)
    d = np.ascontiguousarray(dirs, np.float32)
    out = np.zeros((len(d), 3), np.float32)
    L = lib()
    L.oracle_sample_sky.restype = None
    L.oracle_sample_sky.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p]
    L.oracle_sample_sky(ctypes.byref(sk), d.ctypes.data, len(d), out.ctypes.data)
    return out
