"""ctypes wrapper of the G-buffer lighting oracle (oracle/oracle_deferred.cpp in oracle/liboracle.so), which tests/test_deferred*.py
use."""
import ctypes

import numpy as np

from idkengine_b200 import gpu_types as gt
from oracle_lib import _f32, lib, pack_shadow_maps


def ssao(frame, settings, depth, normal_rg):
    """SSAO.Compute: float32 depth [H, W], normal [H, W, 2] -> uint8 [H, W] (R8Unorm)."""
    d, n = _f32(depth), _f32(normal_rg)
    fr = np.ascontiguousarray(frame)
    out = np.zeros(d.shape, np.uint8)
    rc = lib().oracle_ssao(fr.ctypes.data, ctypes.byref(settings), d.ctypes.data, n.ctypes.data, d.shape[1], d.shape[0], out.ctypes.data)
    assert rc == 0, rc
    return out


def deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt):
    """oracle_deferred_lighting's arguments before its output, the arrays to keep alive while they are used, and (h, w)."""
    lt = np.ascontiguousarray(lights, gt.GpuLight)
    sh, sizes, texels = pack_shadow_maps(shadows, maps)
    assert len(sh) == len(maps)
    d, n, a, mr, e = [_f32(x) for x in gbuffer]
    h, w = d.shape
    fr = np.ascontiguousarray(frame)
    jit = None if jitter is None else _f32(jitter)
    ao = None if ssao is None else np.ascontiguousarray(ssao, np.uint8)
    gi = None if indirect is None else _f32(indirect)
    rts = [_f32(x) for x in (rt or [])]
    rt_ptrs = (ctypes.c_void_p * max(len(rts), 1))(*[x.ctypes.data for x in rts])
    keep = (lt, sh, sizes, texels, d, n, a, mr, e, fr, jit, ao, gi, rts, rt_ptrs)
    args = [lt.ctypes.data if len(lt) else None, len(lt), fr.ctypes.data, shadow_mode, sh.ctypes.data if len(sh) else None,
            sizes.ctypes.data, texels.ctypes.data, len(sh), d.ctypes.data, n.ctypes.data, a.ctypes.data, mr.ctypes.data, e.ctypes.data,
            w, h, jit.ctypes.data if jit is not None else None, ao.ctypes.data if ao is not None else None,
            gi.ctypes.data if gi is not None else None, rt_ptrs, len(rts)]
    return args, keep, (h, w)


def deferred_lighting(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter=None, ssao=None, indirect=None, rt=None):
    """The deferred lighting draw: gbuffer = (depth [H, W], normal [H, W, 2], albedo [H, W, 3], metallic/roughness [H, W, 2],
    emissive [H, W, 3]); shadows (GpuPointShadow) with one uint16 [6, N, N] map each; ssao uint8 [H, W] (IsSSAO) or None;
    indirect float32 [H, W, 4] (IsVXGI) or None; rt: one float32 [H, W] image per shadow (ShadowMode 2). -> float32 [H, W, 4]."""
    args, keep, (h, w) = deferred_args(lights, frame, shadow_mode, shadows, maps, gbuffer, jitter, ssao, indirect, rt)
    out = np.zeros((h, w, 4), np.float32)
    rc = lib().oracle_deferred_lighting(*args, out.ctypes.data)
    assert rc == 0, rc
    return out


def visibility(shadow, cube_map, light_to_sample):
    """The 21-tap PCF filter (Impl.glsl Visibility) for vectors [M, 3] into one uint16 [6, N, N] map."""
    m = np.ascontiguousarray(cube_map, np.uint16)
    v = _f32(light_to_sample).reshape(-1, 3)
    out = np.zeros(len(v), np.float32)
    s = np.ascontiguousarray(shadow, gt.GpuPointShadow).reshape(-1)
    lib().oracle_deferred_visibility(s.ctypes.data, m.shape[1], m.ctypes.data, v.ctypes.data, len(v), out.ctypes.data)
    return out


def ggx_brdf(albedo, metallic, roughness, normal, v, l):
    """GGXBrdf for rows of inputs -> (specular [M, 3], F [M, 3])."""
    rows = _f32(np.concatenate([np.asarray(albedo).reshape(-1, 3), np.asarray(metallic).reshape(-1, 1), np.asarray(roughness).reshape(-1, 1),
                                np.asarray(normal).reshape(-1, 3), np.asarray(v).reshape(-1, 3), np.asarray(l).reshape(-1, 3)], 1))
    out = np.zeros((len(rows), 6), np.float32)
    lib().oracle_ggx_brdf(rows.ctypes.data, len(rows), out.ctypes.data)
    return out[:, :3], out[:, 3:]


def store_r8(values):
    v = _f32(values).ravel()
    out = np.zeros(len(v), np.uint8)
    lib().oracle_store_r8(v.ctypes.data, len(v), out.ctypes.data)
    return out
