"""Voxelizer / ConeTracer: host-side mirrors of IDKEngine.Render.Voxelizer (SRC/Render/VXGI/Voxelizer/Voxelizer.cs) and
ConeTracer (SRC/Render/VXGI/ConeTracing/ConeTracer.cs) over the idkvx_* C ABI (include/idkvx.h)."""
import ctypes

import numpy as np

from . import capi
from . import gpu_types as gt

c_i32, c_u32, c_u64, c_f, c_vp = ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_float, ctypes.c_void_p


class IdkVxCreateInfo(ctypes.Structure):
    _fields_ = [("Device", c_i32), ("Width", c_i32), ("Height", c_i32), ("Depth", c_i32), ("GridMin", c_f * 3), ("GridMax", c_f * 3)]


class IdkVxConeSettings(ctypes.Structure):
    _fields_ = [("MaxSamples", c_i32), ("StepMultiplier", c_f), ("GIBoost", c_f), ("GISkyBoxBoost", c_f),
                ("NormalRayOffset", c_f), ("NoiseIndex", c_u32)]


class IdkVxStats(ctypes.Structure):
    _fields_ = [("ClearMs", c_f), ("VoxelizeMs", c_f), ("MipmapMs", c_f), ("ConeTraceMs", c_f), ("Fragments", c_u64),
                ("ConeSteps", c_u64), ("KernelLaunches", c_u32), ("_pad0", c_u32)]


VX_EXPORTS = ["idkvx_create", "idkvx_destroy", "idkvx_last_error", "idkvx_set_scene", "idkvx_set_scene_from", "idkvx_set_grid", "idkvx_level_count",
              "idkvx_voxelize", "idkvx_read_level", "idkvx_cone_trace", "idkvx_set_shadow_tracer",
              "idkvx_set_shadow_maps", "idkvx_set_slab", "idkvx_level_device_ptr", "idkvx_mipmap", "idkvx_cone_trace_rows",
              "idkvx_set_conservative_rasterization", "idkvx_debug_render", "idkvx_debug_device_ptr",
              "idkvx_cone_trace_gbuffer", "idkvx_cone_trace_device_ptr"]

DEFAULT_GRID_MIN = (-28.0, -3.0, -17.0)   # RasterPipeline.cs:213
DEFAULT_GRID_MAX = (28.0, 20.0, 17.0)


def default_cone_settings():
    """ConeTracer.GpuSettings defaults (ConeTracer.cs:10-22)."""
    return IdkVxConeSettings(4, 0.16, 1.3, 1.0 / 1.3, 1.0, 0)


def create_info(size, grid_min=DEFAULT_GRID_MIN, grid_max=DEFAULT_GRID_MAX, device=0):
    w, h, d = (size, size, size) if np.isscalar(size) else size
    ci = IdkVxCreateInfo(device, w, h, d)
    for i in range(3):
        ci.GridMin[i], ci.GridMax[i] = grid_min[i], grid_max[i]
    return ci


def level_sizes(ci):
    mx = max(ci.Width, ci.Height, ci.Depth)
    levels = 1
    while (mx >> levels) > 0:
        levels += 1
    return [(max(1, ci.Width >> l), max(1, ci.Height >> l), max(1, ci.Depth >> l)) for l in range(levels)]


def _declare(L):
    P = ctypes.POINTER
    L.idkvx_create.restype = c_i32
    L.idkvx_create.argtypes = [P(IdkVxCreateInfo), P(c_vp)]
    L.idkvx_destroy.restype = None
    L.idkvx_destroy.argtypes = [c_vp]
    L.idkvx_last_error.restype = ctypes.c_char_p
    L.idkvx_last_error.argtypes = [c_vp]
    L.idkvx_set_scene.restype = c_i32
    L.idkvx_set_scene.argtypes = [c_vp, P(capi.IdkPtSceneDesc)]
    L.idkvx_set_scene_from.restype = c_i32
    L.idkvx_set_scene_from.argtypes = [c_vp, c_vp]
    L.idkvx_set_grid.restype = c_i32
    L.idkvx_set_grid.argtypes = [c_vp, P(c_f * 3), P(c_f * 3)]
    L.idkvx_level_count.restype = c_i32
    L.idkvx_level_count.argtypes = [c_vp]
    L.idkvx_voxelize.restype = c_i32
    L.idkvx_voxelize.argtypes = [c_vp, P(IdkVxStats)]
    L.idkvx_set_conservative_rasterization.restype = c_i32
    L.idkvx_set_conservative_rasterization.argtypes = [c_vp, c_i32]
    L.idkvx_set_slab.restype = c_i32
    L.idkvx_set_slab.argtypes = [c_vp, c_i32, c_i32]
    L.idkvx_level_device_ptr.restype = c_i32
    L.idkvx_level_device_ptr.argtypes = [c_vp, c_i32, P(c_vp), P(c_u64)]
    L.idkvx_mipmap.restype = c_i32
    L.idkvx_mipmap.argtypes = [c_vp, P(IdkVxStats)]
    L.idkvx_cone_trace_rows.restype = c_i32
    L.idkvx_cone_trace_rows.argtypes = [c_vp, c_vp, P(IdkVxConeSettings), c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, P(c_f * 3), c_vp, P(IdkVxStats)]
    L.idkvx_set_shadow_tracer.restype = c_i32
    L.idkvx_set_shadow_tracer.argtypes = [c_vp, c_vp]
    L.idkvx_set_shadow_maps.restype = c_i32
    L.idkvx_set_shadow_maps.argtypes = [c_vp, c_vp]
    L.idkvx_read_level.restype = c_i32
    L.idkvx_read_level.argtypes = [c_vp, c_i32, c_vp, c_u64]
    L.idkvx_cone_trace.restype = c_i32
    L.idkvx_cone_trace.argtypes = [c_vp, c_vp, P(IdkVxConeSettings), c_vp, c_vp, c_vp, c_i32, c_i32, P(c_f * 3), c_vp, P(IdkVxStats)]
    L.idkvx_cone_trace_gbuffer.restype = c_i32
    L.idkvx_cone_trace_gbuffer.argtypes = [c_vp, c_vp, P(IdkVxConeSettings), P(capi.IdkPtGBuffer), P(c_f * 3), c_vp, P(IdkVxStats)]
    L.idkvx_cone_trace_device_ptr.restype = c_i32
    L.idkvx_cone_trace_device_ptr.argtypes = [c_vp, P(c_vp), P(c_u64)]
    L.idkvx_debug_render.restype = c_i32
    L.idkvx_debug_render.argtypes = [c_vp, c_vp, c_vp, c_f, c_f, c_i32, c_i32, c_vp, P(IdkVxStats)]
    L.idkvx_debug_device_ptr.restype = c_i32
    L.idkvx_debug_device_ptr.argtypes = [c_vp, P(c_vp), P(c_u64)]
    return L


class IdkVxError(RuntimeError):
    pass


class Voxelizer:
    def __init__(self, size=256, grid_min=DEFAULT_GRID_MIN, grid_max=DEFAULT_GRID_MAX, device=0, lib_path=None):
        self._lib = _declare(capi.load(lib_path))
        self.ci = create_info(size, grid_min, grid_max, device)
        self._ctx = c_vp()
        rc = self._lib.idkvx_create(ctypes.byref(self.ci), ctypes.byref(self._ctx))
        if rc != 0:
            raise IdkVxError(f"idkvx_create failed ({rc}): {(self._lib.idkvx_last_error(None) or b'').decode()}")
        self.sizes = level_sizes(self.ci)
        self._conservative = False
        self._source = None                # the PathTracer bound with SetSceneFrom, kept alive while bound
        self.DebugStepMultiplier = 0.4     # the constructor defaults of Voxelizer.cs:68 (DebugRender)
        self.DebugConeAngle = 0.0

    def _check(self, rc, what):
        if rc != 0:
            raise IdkVxError(f"{what} failed ({rc}): {(self._lib.idkvx_last_error(self._ctx) or b'').decode()}")

    def Dispose(self):
        if self._ctx:
            self._lib.idkvx_destroy(self._ctx)
            self._ctx = c_vp()
            self._source = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.Dispose()

    def SetScene(self, scene):
        d, keep = capi.scene_desc(scene)
        self._check(self._lib.idkvx_set_scene(self._ctx, ctypes.byref(d)), "idkvx_set_scene")
        self._source = None

    def SetSceneFrom(self, path_tracer):
        """Voxelise path_tracer's device scene as it stands at each Render, with no copy of it (idkvx_set_scene_from): skinning,
        UpdateRange and a new SetScene on the path tracer reach the next Render. None unbinds and leaves no scene."""
        self._check(self._lib.idkvx_set_scene_from(self._ctx, path_tracer._ctx if path_tracer is not None else None), "idkvx_set_scene_from")
        self._source = path_tracer

    def SetGrid(self, grid_min, grid_max):
        """Voxelizer.GridMin / GridMax setters (Voxelizer.cs:16-33); the next Render voxelises the new bounds."""
        self._check(self._lib.idkvx_set_grid(self._ctx, ctypes.byref((c_f * 3)(*grid_min)), ctypes.byref((c_f * 3)(*grid_max))), "idkvx_set_grid")

    def SetShadowTracer(self, path_tracer):
        """Shadow rays for lights with PointShadowIndex >= 0 go through this PathTracer's scene (None detaches)."""
        self._check(self._lib.idkvx_set_shadow_tracer(self._ctx, path_tracer._ctx if path_tracer is not None else None), "idkvx_set_shadow_tracer")

    def SetShadowMaps(self, path_tracer):
        """Lights with PointShadowIndex >= 0 are filtered through this PathTracer's point-shadow cube maps (PCF lookup;
        SetPointShadows / RenderPointShadows). Takes precedence over SetShadowTracer; None detaches."""
        self._check(self._lib.idkvx_set_shadow_maps(self._ctx, path_tracer._ctx if path_tracer is not None else None), "idkvx_set_shadow_maps")

    @property
    def IsConservativeRasterization(self):
        """Voxelizer.IsConservativeRasterization (Voxelizer.cs:41-56): False = a triangle writes the voxels of the pixel centres
        it covers; True = of every pixel it touches (thin geometry without gaps). Applies from the next Render on."""
        return self._conservative

    @IsConservativeRasterization.setter
    def IsConservativeRasterization(self, value):
        if not isinstance(value, (bool, np.bool_)):
            raise TypeError("IsConservativeRasterization is a bool")
        self._check(self._lib.idkvx_set_conservative_rasterization(self._ctx, int(bool(value))), "idkvx_set_conservative_rasterization")
        self._conservative = bool(value)

    # ---- multi-GPU: z-slab voxelisation, gather, mip chain, screen-tiled cone trace (include/idkvx.h)
    def SetSlab(self, z0, z1):
        self._check(self._lib.idkvx_set_slab(self._ctx, z0, z1), "idkvx_set_slab")

    def LevelDevicePtr(self, level):
        p, n = c_vp(), c_u64()
        self._check(self._lib.idkvx_level_device_ptr(self._ctx, level, ctypes.byref(p), ctypes.byref(n)), "idkvx_level_device_ptr")
        return p.value, n.value

    def Mipmap(self):
        st = IdkVxStats()
        self._check(self._lib.idkvx_mipmap(self._ctx, ctypes.byref(st)), "idkvx_mipmap")
        return st

    def ConeTraceRows(self, frame, depth, normal_rg, metallic_roughness, full_height, row_first, settings=None, sky=(0.6, 0.7, 0.9)):
        """ConeTracer.Compute on rows [row_first, row_first + depth.shape[0]) of a full_height-row G-buffer."""
        settings = settings or default_cone_settings()
        h, w = depth.shape
        depth = np.ascontiguousarray(depth, np.float32)
        nrg = np.ascontiguousarray(normal_rg, np.float32)
        mr = np.ascontiguousarray(metallic_roughness, np.float32)
        out = np.zeros((h, w, 4), np.float32)
        st = IdkVxStats()
        skyc = (c_f * 3)(*sky)
        frame = np.ascontiguousarray(frame)
        self._check(self._lib.idkvx_cone_trace_rows(self._ctx, frame.ctypes.data, ctypes.byref(settings), depth.ctypes.data, nrg.ctypes.data,
                                                    mr.ctypes.data, w, full_height, row_first, h, ctypes.byref(skyc), out.ctypes.data, ctypes.byref(st)), "idkvx_cone_trace_rows")
        return out, st

    def DebugRender(self, path_tracer, frame, width, height, out=True):
        """Voxelizer.DebugRender (Voxelizer.cs:230-244): the grid as it is now, marched per pixel with DebugConeAngle and
        DebugStepMultiplier and blended over path_tracer's sky (idkvx_debug_render). Returns (image float32 [h, w, 4] or None
        with out=False, when the image stays on the device: DebugDevicePtr), stats)."""
        frame = np.ascontiguousarray(frame)
        assert frame.dtype == gt.GpuPerFrameData
        img = np.empty((height, width, 4), np.float32) if out else None
        st = IdkVxStats()
        self._check(self._lib.idkvx_debug_render(self._ctx, path_tracer._ctx if path_tracer is not None else None, frame.ctypes.data,
                                                 float(self.DebugStepMultiplier), float(self.DebugConeAngle), int(width), int(height),
                                                 img.ctypes.data if out else None, ctypes.byref(st)), "idkvx_debug_render")
        return img, st

    def DebugDevicePtr(self):
        """(device pointer, bytes) of the last DebugRender's rgba32f image; (None, 0) before the first."""
        p, n = c_vp(), c_u64()
        self._check(self._lib.idkvx_debug_device_ptr(self._ctx, ctypes.byref(p), ctypes.byref(n)), "idkvx_debug_device_ptr")
        return p.value, n.value

    def Render(self):
        """Voxelizer.Render(modelManager): clear + voxelise + mipmap."""
        st = IdkVxStats()
        self._check(self._lib.idkvx_voxelize(self._ctx, ctypes.byref(st)), "idkvx_voxelize")
        return st

    def ReadLevel(self, level):
        w, h, d = self.sizes[level]
        out = np.zeros((d, h, w, 4), np.float16)
        self._check(self._lib.idkvx_read_level(self._ctx, level, out.ctypes.data, out.nbytes), "idkvx_read_level")
        return out

    def ConeTrace(self, frame, depth, normal_rg, metallic_roughness, settings=None, sky=(0.6, 0.7, 0.9)):
        """ConeTracer.Compute(voxels) on a G-buffer given as host arrays."""
        settings = settings or default_cone_settings()
        h, w = depth.shape
        depth = np.ascontiguousarray(depth, np.float32)
        nrg = np.ascontiguousarray(normal_rg, np.float32)
        mr = np.ascontiguousarray(metallic_roughness, np.float32)
        out = np.zeros((h, w, 4), np.float32)
        st = IdkVxStats()
        skyc = (c_f * 3)(*sky)
        frame = np.ascontiguousarray(frame)
        assert frame.dtype == gt.GpuPerFrameData
        self._check(self._lib.idkvx_cone_trace(self._ctx, frame.ctypes.data, ctypes.byref(settings), depth.ctypes.data, nrg.ctypes.data,
                                               mr.ctypes.data, w, h, ctypes.byref(skyc), out.ctypes.data, ctypes.byref(st)), "idkvx_cone_trace")
        return out, st

    def ConeTraceGBuffer(self, frame, gbuffer, settings=None, sky=(0.6, 0.7, 0.9), download=True):
        """ConeTracer.Compute(voxels) on a G-buffer: a capi.IdkPtGBuffer (e.g. PathTracer.GBufferDevicePtrs()'s, read in place)
        or arrays as PathTracer.gbuffer_arg takes them; Depth, NormalRG and MetallicRoughness are read. Returns (float32
        [H, W, 4] or None with download=False, when the image stays on the device: ConeTraceDevicePtr, stats)."""
        from .pathtracer import PathTracer
        g, keep = PathTracer.gbuffer_arg(gbuffer)
        settings = settings or default_cone_settings()
        out = np.zeros((g.Height, g.Width, 4), np.float32) if download else None
        st = IdkVxStats()
        skyc = (c_f * 3)(*sky)
        frame = np.ascontiguousarray(frame)
        assert frame.dtype == gt.GpuPerFrameData
        self._check(self._lib.idkvx_cone_trace_gbuffer(self._ctx, frame.ctypes.data, ctypes.byref(settings), ctypes.byref(g), ctypes.byref(skyc),
                                                       out.ctypes.data if download else None, ctypes.byref(st)), "idkvx_cone_trace_gbuffer")
        return out, st

    def ConeTraceDevicePtr(self):
        """(device pointer, bytes) of the last cone trace's rgba32f image: DeferredLighting's indirect light on the device."""
        p, n = c_vp(), c_u64()
        self._check(self._lib.idkvx_cone_trace_device_ptr(self._ctx, ctypes.byref(p), ctypes.byref(n)), "idkvx_cone_trace_device_ptr")
        return p.value, n.value


def camera_rays(frame, width, height):
    """Pinhole rays through the pixel grid, built like Ray.GetWorldSpaceRay (SRC/Shapes/Ray.cs:30-39) from GpuPerFrameData's
    InvProjection / InvView with ndc = (x, y) / resolution * 2 - 1 (the shape Gui.Test uses, Gui.cs:1484-1503)."""
    f = frame[0] if frame.ndim else frame
    ip = np.asarray(f["InvProjection"], np.float32).reshape(-1)
    iv = np.asarray(f["InvView"], np.float32).reshape(-1)
    xs = (np.arange(width, dtype=np.float32) / np.float32(width) * np.float32(2.0) - np.float32(1.0))[None, :]
    ys = (np.arange(height, dtype=np.float32) / np.float32(height) * np.float32(2.0) - np.float32(1.0))[:, None]
    vx = xs * ip[0] + ys * ip[4]
    vy = xs * ip[1] + ys * ip[5]
    w = np.stack([vx * iv[0] + vy * iv[4] - iv[8], vx * iv[1] + vy * iv[5] - iv[9], vx * iv[2] + vy * iv[6] - iv[10]], -1).astype(np.float32)
    w /= np.sqrt((w * w).sum(-1, keepdims=True, dtype=np.float32))
    rays = np.zeros(width * height, gt.IdkPtRay)
    rays["Origin"] = np.asarray(f["ViewPos"], np.float32).reshape(-1)[:3]
    rays["TMax"] = np.float32(3.4028235e38)
    rays["Direction"] = w.reshape(-1, 3)
    return rays


def encode_unit_vec(n):
    """EncodeUnitVec (Compression.glsl:54-61): unit vectors [..., 3] -> octahedral (x, y) in [0, 1], computed in n's precision
    and returned as float32."""
    m = n / np.sum(np.abs(n), -1, keepdims=True)
    wrap = (1.0 - np.abs(m[..., [1, 0]])) * np.where(m[..., :2] < 0, -1.0, 1.0)
    return (np.where((m[..., 2] > 0)[..., None], m[..., :2], wrap) * 0.5 + 0.5).astype(np.float32)


def gbuffer_from_hits(scene, frame, rays, hits, width, height):
    """The G-buffer attachments ConeTracer.Compute reads, from first hits of camera rays: depth = ProjView-projected hit point
    (1.0 = sky), normal = octahedral geometric normal facing the camera, metallic/roughness from the hit material."""
    hit = hits["TriangleId"] != 0xFFFFFFFF
    o = rays["Origin"].astype(np.float64)
    d = rays["Direction"].astype(np.float64)
    pos = o + d * hits["T"][:, None].astype(np.float64)
    f = frame[0] if frame.ndim else frame
    pv = np.asarray(f["ProjView"], np.float64).reshape(4, 4)            # OpenTK rows: clip = [p, 1] @ pv
    clip = np.concatenate([pos, np.ones((len(pos), 1))], 1) @ pv
    with np.errstate(all="ignore"):
        depth = np.where(hit, clip[:, 2] / clip[:, 3], 1.0).astype(np.float32)
    depth = np.where(hit & (depth >= 1.0), np.float32(0.999999), depth)
    tri = scene.blas_triangles[np.where(hit, hits["TriangleId"], 0)]
    P = scene.positions

    def pnt(k):
        return np.stack([P["x"][tri[k]], P["y"][tri[k]], P["z"][tri[k]]], 1).astype(np.float64)
    p0, p1, p2 = pnt("X"), pnt("Y"), pnt("Z")
    n = np.cross(p1 - p0, p2 - p0)
    inv = scene.mesh_transforms["InvModelMatrix"][hits["MeshTransformId"]][:, :, :3].astype(np.float64)
    n = np.einsum("nji,nj->ni", inv, n)                                # transpose(inv) * n
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-30)
    n = np.where((np.sum(n * d, 1) > 0)[:, None], -n, n)
    nrg = encode_unit_vec(n)
    mesh = scene.meshes[tri["MeshId"]]
    mat = scene.materials[mesh["MaterialId"]]
    mr = np.stack([np.clip(mat["MetallicFactor"] + mesh["SpecularBias"], 0, 1), np.clip(mat["RoughnessFactor"] + mesh["RoughnessBias"], 0, 1)], 1).astype(np.float32)
    return depth.reshape(height, width), nrg.reshape(height, width, 2), mr.reshape(height, width, 2)


def synth_gbuffer(pt, scene, frame, width, height):
    """gbuffer_from_hits for the path tracer's first hit on the GPU (`pt.TraceRays`), for scenes that have no rasteriser behind
    them (SURVEY 8d config 5)."""
    rays = camera_rays(frame, width, height)
    hits, _ = pt.TraceRays(rays)
    return gbuffer_from_hits(scene, frame, rays, hits, width, height)
