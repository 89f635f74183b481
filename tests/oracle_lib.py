"""ctypes wrapper of oracle/liboracle.so -- imported by tests/, __graft_entry__.smoke() and bench.py's CPU legs only.
The per-pass wrappers (tests/*_oracle.py) call the same library through lib()."""
import ctypes
import importlib.util
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "oracle"))

from idkengine_b200 import capi, gpu_types as gt, vxgi  # noqa: E402


def _signatures():
    """Every export of the library: name -> (restype, argtypes). tests/test_oracle_library.py checks it against the sources."""
    P = ctypes.POINTER
    vp, f32, i32, u32, u64 = ctypes.c_void_p, ctypes.c_float, ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint64
    SCENE, SKY, CI = P(capi.IdkPtSceneDesc), P(capi.IdkPtSkyDesc), P(vxgi.IdkVxCreateInfo)
    # oracle_deferred_lighting's arguments up to the output; the variable-rate entry points take the same ones first
    deferred = [vp, u64, vp, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, i32]
    return {
        # oracle.cpp
        "oracle_trace_rays": (i32, [SCENE, vp, u64, i32, vp, i32]),
        "oracle_trace_rays_any": (i32, [SCENE, vp, u64, i32, vp, i32]),
        "oracle_brute_force": (i32, [SCENE, vp, u64, vp, i32]),
        "oracle_cpu_intersect": (ctypes.c_double, [SCENE, vp, u64, vp, i32]),
        "oracle_gui_test_rays": (None, [vp, i32, i32, i32, i32, vp]),
        "oracle_path_trace": (i32, [SCENE, SKY, vp, P(capi.IdkPtSettings), i32, i32, i32, i32, i32, P(u32), vp, vp, vp, vp,
                                    P(capi.IdkPtStats), i32]),
        "oracle_sample_sky": (None, [vp, vp, u64, vp]),
        "oracle_det_sincos": (None, [vp, u64, vp, vp]),
        "oracle_det_exp": (None, [vp, u64, vp]),
        "oracle_encode_decode": (None, [vp, u64, vp, vp]),
        "oracle_pcg": (u32, [u32, P(u32)]),
        "oracle_shadows_ray_traced": (i32, [SCENE, vp, vp, vp, i32, i32, i32, i32, u32, vp, vp, i32]),
        "oracle_skin_vertices": (None, [vp] * 4 + [u32] * 4),
        "oracle_blas_refit": (None, [vp] * 4),
        "oracle_tex_sample": (None, [P(capi.IdkPtTextureDesc), vp, u64, vp]),
        # oracle_post.inc
        "oracle_post_process": (i32, [vp, i32, i32, P(capi.IdkPtPostSettings), vp, vp, i32]),
        "oracle_denoise": (i32, [vp, vp, vp, i32, i32, P(capi.IdkPtDenoiseSettings), vp, i32]),
        # oracle_vxgi.inc
        "oracle_vx_set_raster_rule": (None, [i32]),
        "oracle_vx_voxelize": (i32, [SCENE, CI, vp, u64, P(u64), i32]),
        "oracle_vx_mipmap": (i32, [CI, vp, i32]),
        "oracle_vx_cone_trace": (i32, [CI, vp, vp, P(vxgi.IdkVxConeSettings), vp, vp, vp, i32, i32, vp, vp, P(u64), i32]),
        "oracle_half_roundtrip": (None, [vp, u64, vp, vp]),
        "oracle_det_log2": (None, [vp, u64, vp]),
        # oracle_point_shadows.cpp
        "oracle_point_shadow_render": (None, [SCENE, vp, i32, u32, vp]),
        "oracle_point_shadow_visibility": (None, [vp, i32, vp, vp, u64, vp]),
        "oracle_vx_voxelize_shadow_maps": (i32, [SCENE, CI, vp, vp, vp, i32, vp, u64, P(u64), i32]),
        # oracle_deferred.cpp
        "oracle_ssao": (i32, [vp, P(capi.IdkPtSsaoSettings), vp, vp, i32, i32, vp]),
        "oracle_deferred_lighting": (i32, deferred + [vp]),
        "oracle_deferred_visibility": (None, [vp, i32, vp, vp, u64, vp]),
        "oracle_ggx_brdf": (None, [vp, u64, vp]),
        "oracle_store_r8": (None, [vp, u64, vp]),
        # oracle_vrs.cpp
        "oracle_shading_rate": (i32, [vp, P(capi.IdkPtShadingRateSettings), vp, vp, i32, i32, vp, vp]),
        "oracle_deferred_lighting_vrs": (i32, deferred + [vp, vp]),
        "oracle_deferred_samples": (i32, deferred + [vp, vp, u64, vp]),
        # oracle_ssr_taa.cpp
        "oracle_ssr": (i32, [vp, P(capi.IdkPtSsrSettings), SKY, vp, vp, vp, vp, vp, i32, i32, vp, vp]),
        "oracle_taa_resolve": (i32, [P(capi.IdkPtTaaSettings), vp, vp, vp, i32, i32, vp, i32, i32, vp]),
        # oracle_gbuffer.cpp
        "oracle_gbuffer": (i32, [SCENE, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32]),
        "oracle_gbuffer_store": (None, [i32, vp, u64, vp]),
        # oracle_transparency.cpp
        "oracle_transparency": (i32, [SCENE, SKY, vp, i32, i32, vp, vp, vp, i32, vp, vp, vp, vp, i32, i32, vp, i32, vp, vp, vp,
                                      vp, i32]),
        # oracle_lights_skybox.cpp
        "oracle_lights_skybox": (i32, [SCENE, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32]),
        "oracle_sphere_mesh": (None, [vp, vp]),
        # oracle_volumetric.cpp
        "oracle_volumetric_lighting": (i32, [vp, u64, vp, P(capi.IdkPtVolumetricSettings), vp, vp, vp, i32, vp, i32, i32, i32, i32,
                                             vp, vp, vp, vp]),
        "oracle_volumetric_upscale": (None, [vp, vp, i32, i32, vp, vp, i32, i32, i32, i32, vp]),
        "oracle_cube_nearest": (None, [vp, i32, vp, u64, vp]),
        # oracle_sky.cpp
        "oracle_sky_atmosphere": (i32, [P(capi.IdkPtAtmosphereSettings), i32, vp, i32]),
        "oracle_sky_equirect": (i32, [vp, i32, i32, vp, i32]),
        "oracle_sky_directions": (None, [i32, vp]),
        "oracle_det_atan2": (None, [vp, vp, u64, vp]),
        "oracle_det_asin": (None, [vp, u64, vp]),
        # oracle_vxgi_conservative.cpp
        "oracle_vx_voxelize_conservative": (i32, [SCENE, CI, vp, u64, P(u64), i32]),
        "oracle_vx_voxelize_conservative_shadow_maps": (i32, [SCENE, CI, vp, vp, vp, i32, vp, u64, P(u64), i32]),
        # oracle_vxgi_debug.cpp
        "oracle_vx_debug_render": (i32, [vp, vp, vp, vp, f32, f32, i32, i32, vp, P(u64), i32]),
    }


SIGNATURES = _signatures()

_lib = None


def lib():
    """oracle/liboracle.so, rebuilt first if an oracle source is newer than it, with every export's signature declared."""
    global _lib
    if _lib is None:
        spec = importlib.util.spec_from_file_location("oracle_build", os.path.join(REPO, "oracle", "build.py"))
        ob = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ob)
        L = ctypes.CDLL(ob.build())
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def pack_shadow_maps(shadows, maps):
    """GpuPointShadow records with one uint16 [6, N, N] cube map each -> (records, int32 sizes N, the maps' texels back to
    back), as the oracle takes them; without maps, sizes and texels are one-element placeholders."""
    records = np.ascontiguousarray(shadows, gt.GpuPointShadow).reshape(-1)
    sizes = np.array([m.shape[1] for m in maps] or [0], np.int32)
    texels = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(m, np.uint16).ravel() for m in maps]) if len(maps) else
                                  np.zeros(1, np.uint16))
    return records, sizes, texels


def split_levels(raw, ci):
    """A grid's raw uint16 mip chain -> the float16 [d, h, w, 4] view of each level."""
    levels, off = [], 0
    for (w, h, d) in vxgi.level_sizes(ci):
        k = w * h * d * 4
        levels.append(raw[off:off + k].view(np.float16).reshape(d, h, w, 4))
        off += k
    return levels


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
    lib().oracle_trace_rays_any(ctypes.byref(d), rays.ctypes.data, len(rays), int(trace_lights), out.ctypes.data, threads or default_threads())
    return out


def shadows_ray_traced(scene, frame, depth, normal_rg, light_index, samples=1, noise_index=0, jitter=(0.0, 0.0), visibility=None, threads=None):
    d, keep = capi.scene_desc(scene)
    h, w = depth.shape
    depth = np.ascontiguousarray(depth, np.float32)
    nrg = np.ascontiguousarray(normal_rg, np.float32)
    vis = np.zeros((h, w), np.float32) if visibility is None else np.ascontiguousarray(visibility, np.float32)
    jit = np.array(jitter, np.float32)
    rc = lib().oracle_shadows_ray_traced(ctypes.byref(d), frame.ctypes.data, depth.ctypes.data, nrg.ctypes.data, w, h, light_index, samples,
                                         noise_index, jit.ctypes.data, vis.ctypes.data, threads or default_threads())
    assert rc == 0
    return vis


def skin_vertices(unskinned, joint_matrices, positions, vertices, cmd):
    """In-place oracle_skin_vertices on numpy arrays (positions: PackedVec3, vertices: GpuVertex)."""
    jm = np.ascontiguousarray(joint_matrices, np.float32)
    lib().oracle_skin_vertices(unskinned.ctypes.data, jm.ctypes.data, positions.ctypes.data, vertices.ctypes.data, int(cmd["InputVertexOffset"]),
                               int(cmd["OutputVertexOffset"]), int(cmd["JointMatricesOffset"]), int(cmd["VertexCount"]))


def blas_refit(scene, blas_id):
    """In-place BLAS.Refit of scene.blas_nodes for one BLAS from scene.positions."""
    desc = np.ascontiguousarray(scene.blas_descs[blas_id:blas_id + 1])
    lib().oracle_blas_refit(scene.blas_nodes.ctypes.data, desc.ctypes.data, scene.blas_triangles.ctypes.data, scene.positions.ctypes.data)


def post_process(result, settings=None, want_bloom=False, threads=None):
    """oracle_post_process on an rgba32f image [H, W, 4] -> rgba8 [H, W, 4] (and Bloom.Result [H//2, W//2, 3])."""
    st = settings if settings is not None else capi.default_post_settings()
    h, w = result.shape[:2]
    result = np.ascontiguousarray(result, np.float32)
    out = np.zeros((h, w, 4), np.uint8)
    bloom = np.zeros((max(h // 2, 1), max(w // 2, 1), 3), np.float32)
    rc = lib().oracle_post_process(result.ctypes.data, w, h, ctypes.byref(st), out.ctypes.data, bloom.ctypes.data if want_bloom else None,
                                   threads or default_threads())
    assert rc == 0
    return (out, bloom) if want_bloom else out


def tex_sample(pixels, uv, srgb=False, wrap_s=10497, wrap_t=10497, flags=0):
    px = np.ascontiguousarray(pixels, np.uint8)
    uv = np.ascontiguousarray(uv, np.float32)
    t = capi.IdkPtTextureDesc(px.ctypes.data, px.shape[1], px.shape[0], 1 if srgb else 0, wrap_s, wrap_t, flags)
    out = np.zeros((len(uv), 4), np.float32)
    lib().oracle_tex_sample(ctypes.byref(t), uv.ctypes.data, len(uv), out.ctypes.data)
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
def vx_mipmap(ci, level0, threads=None):
    """Levels 1 .. n-1 of the mip chain built from a caller-supplied level 0 (float16 [d, h, w, 4]).
    Returns (list of float16 [d, h, w, 4] arrays per level, concatenated raw uint16 chain)."""
    sizes = vxgi.level_sizes(ci)
    w, h, d = sizes[0]
    level0 = np.ascontiguousarray(level0, np.float16)
    assert level0.shape == (d, h, w, 4), level0.shape
    raw = np.zeros(sum(a * b * c for a, b, c in sizes) * 4, np.uint16)
    raw[:level0.size] = level0.reshape(-1).view(np.uint16)
    n = lib().oracle_vx_mipmap(ctypes.byref(ci), raw.ctypes.data, threads or default_threads())
    assert n == len(sizes), n
    return split_levels(raw, ci), raw


def vx_voxelize(scene, ci, threads=None, raster_rule=0):
    """Returns (list of float16 [d,h,w,4] arrays per level, concatenated raw uint16 chain, fragment count).
    raster_rule: 0 = the product's coverage rule (what the GPU kernels implement), 1 = the GL model (1/256-pixel snapping +
    top-left fill rule) used only to measure the distance between the two."""
    L = lib()
    sizes = vxgi.level_sizes(ci)
    total = sum(w * h * d for w, h, d in sizes)
    raw = np.zeros(total * 4, np.uint16)
    d, keep = capi.scene_desc(scene)
    frags = ctypes.c_uint64()
    try:
        L.oracle_vx_set_raster_rule(int(raster_rule))   # process-wide: every other voxeliser entry point runs under rule 0
        n = L.oracle_vx_voxelize(ctypes.byref(d), ctypes.byref(ci), raw.ctypes.data, total, ctypes.byref(frags), threads or default_threads())
    finally:
        L.oracle_vx_set_raster_rule(0)
    assert n == len(sizes), n
    return split_levels(raw, ci), raw, frags.value


def vx_cone_trace(ci, raw_chain, frame, settings, depth, normal_rg, metal_rough, sky=(0.6, 0.7, 0.9), threads=None):
    h, w = depth.shape
    out = np.zeros((h, w, 4), np.float32)
    skyc = np.array(sky, np.float32)
    steps = ctypes.c_uint64()
    depth = np.ascontiguousarray(depth, np.float32)
    nrg = np.ascontiguousarray(normal_rg, np.float32)
    mr = np.ascontiguousarray(metal_rough, np.float32)
    rc = lib().oracle_vx_cone_trace(ctypes.byref(ci), raw_chain.ctypes.data, frame.ctypes.data, ctypes.byref(settings), depth.ctypes.data,
                                    nrg.ctypes.data, mr.ctypes.data, w, h, skyc.ctypes.data, out.ctypes.data, ctypes.byref(steps),
                                    threads or default_threads())
    assert rc == 0
    return out, steps.value


def synth_gbuffer(scene, frame, width, height):
    """vxgi.gbuffer_from_hits for the oracle's first hit through pixel centres (instead of Gui.Test's pixel corners)."""
    rays = gui_test_rays(frame, width, height)
    return vxgi.gbuffer_from_hits(scene, frame, rays, trace_rays(scene, rays), width, height)


def denoise(result, albedo, normal, settings=None, threads=None):
    """oracle_denoise: the guided a-trous filter of csrc/idk_post.cuh on rgba32f images [H, W, 4] -> denoised [H, W, 4]."""
    st = settings if settings is not None else capi.default_denoise_settings()
    h, w = result.shape[:2]
    r, a, n = (np.ascontiguousarray(x, np.float32) for x in (result, albedo, normal))
    out = np.zeros((h, w, 4), np.float32)
    rc = lib().oracle_denoise(r.ctypes.data, a.ctypes.data, n.ctypes.data, w, h, ctypes.byref(st), out.ctypes.data, threads or default_threads())
    assert rc == 0
    return out


def sample_sky(faces, dirs):
    """texture(samplerCube, dir).rgb for float32 faces [6, N, N, 4] and directions [M, 3]."""
    sk = capi.sky_desc((0.0, 0.0, 0.0), faces)
    d = np.ascontiguousarray(dirs, np.float32)
    out = np.zeros((len(d), 3), np.float32)
    lib().oracle_sample_sky(ctypes.byref(sk), d.ctypes.data, len(d), out.ctypes.data)
    return out
