"""PathTracer: host-side mirror of IDKEngine.Render.PathTracer (SRC/Render/PathTracer.cs:10-346) whose body is the
libidkpt C ABI instead of GL dispatches -- the Python twin of the C# PathTracerNative class in INTEGRATION.md.

Same public members and meaning: ctor(width, height, settings), Compute(), SetSize(), ResetAccumulation(),
properties SamplesPerPixel, RayDepth, AccumulatedSamples, FocalLength, LenseRadius, DoDebugBVHTraversal,
DoTraceLights, DoRussianRoulette, DoRaySorting, OutputAOVs, images Result / AlbedoTexture / NormalTexture.
Setters reset the accumulation exactly where the C# setters do (PathTracer.cs:16-97).
Scene data the reference binds globally (SSBO/UBO slots) is handed over with SetScene()/SetSky()/SetFrame().
"""
import ctypes

import numpy as np

from . import capi
from . import gpu_types as gt
from . import host


class IdkPtError(RuntimeError):
    pass


class PathTracer:
    def __init__(self, width, height, settings=None, device=0, tile=(8, 0, 1), lib_path=None, lanes=0, global_slots=False):
        """global_slots: IDKPT_CREATE_GLOBAL_SLOTS -- a tiled (multi-GPU) context numbers its alive rays over the WHOLE image, so the
        N-GPU image is bit-identical to the 1-GPU image (needs EnablePeerGather / ConnectPeers)."""
        self._lib = capi.load(lib_path)
        self._ctx = ctypes.c_void_p()
        self._settings = settings or capi.default_settings()
        flags = ((int(lanes) & 15) << 8) | (capi.IDKPT_CREATE_GLOBAL_SLOTS if global_slots else 0)   # IDKPT_CREATE_LANES
        ci = capi.IdkPtCreateInfo(device, width, height, tile[0], tile[1], tile[2], flags)
        rc = self._lib.idkpt_create(ctypes.byref(ci), ctypes.byref(self._ctx))
        if rc != 0:
            msg = self._lib.idkpt_last_error(None)
            raise IdkPtError(f"idkpt_create failed ({rc}): {msg.decode() if msg else ''}")
        self.width, self.height = width, height
        self.tile = tile
        self._device = device
        self._frame = None
        self._keep = None
        self.last_stats = None
        self.last_blas_build_ms = None   # device time of the last BuildBlas
        self._export = False

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc, what):
        if rc != 0:
            msg = self._lib.idkpt_last_error(self._ctx)
            raise IdkPtError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")

    def _device_ptr(self, name, *args):
        """(device pointer, bytes) from the library's export `name` (an idkpt_*_device_ptr)."""
        p, n = ctypes.c_void_p(), ctypes.c_uint64()
        self._check(getattr(self._lib, name)(self._ctx, *args, ctypes.byref(p), ctypes.byref(n)), name)
        return p.value, n.value

    def Dispose(self):
        if self._ctx:
            self._lib.idkpt_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.Dispose()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.Dispose()

    # ------------------------------------------------------------------ scene hand-over
    def SetScene(self, scene):
        d, keep = capi.scene_desc(scene)
        self._check(self._lib.idkpt_set_scene(self._ctx, ctypes.byref(d)), "idkpt_set_scene")
        self._vertex_position_count = int(d.VertexPositionCount)

    def UpdateRange(self, which, first, data):
        data = np.ascontiguousarray(data)
        self._check(self._lib.idkpt_update_range(self._ctx, which, first, len(data), data.ctypes.data), "idkpt_update_range")

    _READ_DTYPES = {capi.IDKPT_ARRAY_TLAS_NODES: gt.GpuTlasNode, capi.IDKPT_ARRAY_BLAS_NODES: gt.GpuBlasNode,
                    capi.IDKPT_ARRAY_VERTEX_POSITIONS: gt.PackedVec3, capi.IDKPT_ARRAY_VERTICES: gt.GpuVertex,
                    capi.IDKPT_ARRAY_BLAS_TRIANGLES: gt.GpuBlasTriangle, capi.IDKPT_ARRAY_BLAS_DESCS: gt.GpuBlasDesc}

    def ReadRange(self, which, first, count):
        out = np.zeros(count, self._READ_DTYPES[which])
        self._check(self._lib.idkpt_read_range(self._ctx, which, first, count, out.ctypes.data), "idkpt_read_range")
        return out

    # ------------------------------------------------------------------ present chain (Application.cs:217-223)
    def PostProcess(self, settings=None, source=capi.IDKPT_IMAGE_RESULT, download=True):
        """Bloom + TonemapAndGammaCorrect of the accumulated frame. Returns (rgba8 [H, W, 4] or None, kernel ms)."""
        st = settings if settings is not None else capi.default_post_settings()
        out = np.zeros((self.height, self.width, 4), np.uint8) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_post_process(self._ctx, ctypes.byref(st), source, out.ctypes.data if download else None, ctypes.byref(ms)),
                    "idkpt_post_process")
        return out, ms.value

    # ------------------------------------------------------------------ denoise hand-off (PathTracerPipeline.Denoise, PathTracerPipeline.cs:165-194)
    def Denoise(self, settings=None):
        """Pack Result / Albedo / Normal into the OIDN-layout device buffers and run the built-in guided a-trous filter.
        Returns kernel ms; the output is `Denoised` (and PostProcess(source=IDKPT_IMAGE_DENOISED))."""
        st = settings if settings is not None else capi.default_denoise_settings()
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_denoise(self._ctx, ctypes.byref(st), ctypes.byref(ms)), "idkpt_denoise")
        return ms.value

    @property
    def Denoised(self):
        return self._read(capi.IDKPT_IMAGE_DENOISED)

    def DenoiseDevicePtrs(self):
        """(beauty, albedo, normal, output) device pointers of the packed-RGB float buffers (OIDN Format.Float3) and their size."""
        p = [ctypes.c_void_p() for _ in range(4)]
        n = ctypes.c_uint64()
        self._check(self._lib.idkpt_denoise_device_ptrs(self._ctx, *[ctypes.byref(x) for x in p], ctypes.byref(n)), "idkpt_denoise_device_ptrs")
        return [x.value for x in p], n.value

    def DenoiseImportOutput(self):
        self._check(self._lib.idkpt_denoise_import_output(self._ctx), "idkpt_denoise_import_output")

    # ------------------------------------------------------------------ dynamic geometry (ModelManager.Update, ModelManager.cs:236-261)
    def SetSkinningData(self, unskinned):
        unskinned = np.ascontiguousarray(unskinned)
        assert unskinned.dtype == gt.GpuUnskinnedVertex
        self._check(self._lib.idkpt_set_skinning_data(self._ctx, unskinned.ctypes.data, len(unskinned)), "idkpt_set_skinning_data")

    def SkinVertices(self, joint_matrices, cmds):
        """joint_matrices: [J, 3, 4] float32 (row-major mat4x3); cmds: IdkPtSkinningCmd array. Returns kernel ms."""
        jm = np.ascontiguousarray(joint_matrices, np.float32).reshape(-1, 3, 4)
        cmds = np.ascontiguousarray(cmds)
        assert cmds.dtype == gt.IdkPtSkinningCmd
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_skin_vertices(self._ctx, jm.ctypes.data, len(jm), cmds.ctypes.data, len(cmds), ctypes.byref(ms)), "idkpt_skin_vertices")
        return ms.value

    def BlasRefit(self, first, count=1):
        """BVH.GpuBlasesRefit (BVH.cs:472-489). Returns kernel ms."""
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_blas_refit(self._ctx, first, count, ctypes.byref(ms)), "idkpt_blas_refit")
        return ms.value

    def TlasBuild(self, search_radius=15):
        """BVH.TlasBuild on the device (BVH.cs:278-298, TLAS.cs:28-141) from the refitted roots and current transforms. Returns kernel ms."""
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_tlas_build(self._ctx, search_radius, ctypes.byref(ms)), "idkpt_tlas_build")
        return ms.value

    @staticmethod
    def _blas_settings(settings):
        """An IdkPtBlasBuildSettings from None (the defaults), an IdkPtBlasBuildSettings or a host.IdkBlasBuildSettings."""
        s = capi.default_blas_build_settings()
        if settings is not None:
            for name, _ in capi.IdkPtBlasBuildSettings._fields_:
                setattr(s, name, getattr(settings, name))
        return s

    def RebuildBlases(self, first, count=1, settings=None):
        """BVH.BlasesBuild(first, count) (BVH.cs:300-470) on the device scene in place, from its current positions
        (idkpt_blas_rebuild); a BLAS is pre-split when it is not refittable. Call TlasBuild afterwards. Returns kernel ms."""
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_blas_rebuild(self._ctx, first, count, ctypes.byref(self._blas_settings(settings)), ctypes.byref(ms)),
                    "idkpt_blas_rebuild")
        return ms.value

    def BlasSah(self, first, count=1, settings=None):
        """BLAS.ComputeGlobalSAH (BLAS.cs:629-656) of BLASes [first, first + count) as the device holds them now; float64 array.
        Only settings.TriangleCost is read."""
        out = np.zeros(count, np.float64)
        self._check(self._lib.idkpt_blas_sah(self._ctx, first, count, ctypes.byref(self._blas_settings(settings)), out.ctypes.data),
                    "idkpt_blas_sah")
        return out

    def BuildBlas(self, positions, triangles, presplit=True, settings=None):
        """BLAS.Build + PreSplitting.PreSplit on the device (idkpt_blas_build), with host.build_blas's signature and result:
        dict(nodes, triangles, required_stack_size, fragment_count, sah), equal to the host build. settings: an
        IdkPtBlasBuildSettings or host.IdkBlasBuildSettings (its Threads is ignored); DoPreSplit comes from `presplit`.
        The device time of the build (kernel_ms) is left in `last_blas_build_ms`."""
        positions = np.ascontiguousarray(positions)
        triangles = np.ascontiguousarray(triangles)
        assert positions.dtype == gt.PackedVec3 and triangles.dtype == gt.GpuBlasTriangle
        s = self._blas_settings(settings)
        s.DoPreSplit = 1 if presplit else 0
        h = ctypes.c_void_p()
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_blas_build(self._ctx, positions.ctypes.data, len(positions), triangles.ctypes.data, len(triangles),
                                               ctypes.byref(s), ctypes.byref(h), ctypes.byref(ms)), "idkpt_blas_build")
        try:
            nn, nt = ctypes.c_uint64(), ctypes.c_uint64()
            stack, frags, sah = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_double()
            self._check(self._lib.idkpt_blas_build_info(h, ctypes.byref(nn), ctypes.byref(nt), ctypes.byref(stack), ctypes.byref(frags),
                                                        ctypes.byref(sah)), "idkpt_blas_build_info")
            nodes = np.zeros(nn.value, gt.GpuBlasNode)
            tris = np.zeros(nt.value, gt.GpuBlasTriangle)
            self._check(self._lib.idkpt_blas_build_copy(h, nodes.ctypes.data, tris.ctypes.data), "idkpt_blas_build_copy")
        finally:
            self._lib.idkpt_blas_build_free(h)
        self.last_blas_build_ms = float(ms.value)
        return dict(nodes=nodes, triangles=tris, required_stack_size=int(stack.value), fragment_count=int(frags.value), sah=float(sah.value))

    def BuildBlases(self, positions, triangles, descs, settings=None):
        """BVH.BlasesBuild's loop (BVH.cs:315-377) over the BLASes of `descs` in one device call (idkpt_blas_build_batch): BLAS s
        is built from triangles[TriangleOffset, +TriangleCount) and pre-split when not IsRefittable; only those desc fields
        are read. settings as BuildBlas (DoPreSplit is ignored). Returns dict(descs, nodes, triangles, fragment_counts, sahs):
        the descs as BVH.cs:363-386 fills them, with offsets into the concatenated nodes and triangles; each BLAS equal to
        BuildBlas (and the host build) of it. The device time of the batch is left in `last_blas_build_ms`."""
        positions = np.ascontiguousarray(positions)
        triangles = np.ascontiguousarray(triangles)
        descs = np.ascontiguousarray(descs)
        assert positions.dtype == gt.PackedVec3 and triangles.dtype == gt.GpuBlasTriangle and descs.dtype == gt.GpuBlasDesc
        s = self._blas_settings(settings)
        h = ctypes.c_void_p()
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_blas_build_batch(self._ctx, positions.ctypes.data, len(positions), triangles.ctypes.data, len(triangles),
                                                     descs.ctypes.data, len(descs), ctypes.byref(s), ctypes.byref(h), ctypes.byref(ms)),
                    "idkpt_blas_build_batch")
        try:
            nn, nt = ctypes.c_uint64(), ctypes.c_uint64()
            self._check(self._lib.idkpt_blas_build_info(h, ctypes.byref(nn), ctypes.byref(nt), None, None, None), "idkpt_blas_build_info")
            out_descs = np.zeros(len(descs), gt.GpuBlasDesc)
            nodes = np.zeros(nn.value, gt.GpuBlasNode)
            tris = np.zeros(nt.value, gt.GpuBlasTriangle)
            frags = np.zeros(len(descs), np.int32)
            sahs = np.zeros(len(descs), np.float64)
            self._check(self._lib.idkpt_blas_build_batch_copy(h, out_descs.ctypes.data, nodes.ctypes.data, tris.ctypes.data,
                                                              frags.ctypes.data, sahs.ctypes.data), "idkpt_blas_build_batch_copy")
        finally:
            self._lib.idkpt_blas_build_free(h)
        self.last_blas_build_ms = float(ms.value)
        return dict(descs=out_descs, nodes=nodes, triangles=tris, fragment_counts=frags, sahs=sahs)

    def AddModels(self, *models, textures=(), unskinned=None, settings=None):
        """ModelManager.Add(models) (ModelManager.cs:128-216) on the device scene in place (idkpt_add_models): host.Model objects
        appended with host.model_records' call-local ids -- their material texture handles index `textures` (list of texture
        dicts as host.Scene.textures, 1-based, 0 = white) -- one BLAS and one instance per model, the BLASes built on the
        device, the TLAS rebuilt when the scene uses one. unskinned: GpuUnskinnedVertex records appended behind
        SetSkinningData's. settings as BuildBlas (DoPreSplit is ignored). Returns kernel ms."""
        if unskinned is not None:
            unskinned = np.ascontiguousarray(unskinned)
            assert unskinned.dtype == gt.GpuUnskinnedVertex
        d, keep = capi.add_models_desc(host.model_records(models), textures, unskinned)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_add_models(self._ctx, ctypes.byref(d), ctypes.byref(self._blas_settings(settings)), ctypes.byref(ms)),
                    "idkpt_add_models")
        return ms.value

    def SetTextures(self, textures):
        """Replace the material texture table (list of dict(pixels, srgb, wrap_s, wrap_t), as host.Scene.textures)."""
        arr, keep = capi.texture_descs(textures)
        self._check(self._lib.idkpt_set_textures(self._ctx, ctypes.addressof(arr) if textures else None, len(textures)), "idkpt_set_textures")

    def SetSky(self, color, faces=None):
        """Constant colour, or cubemap faces [6, N, N, 4] float32 (SkyBoxManager's samplerCube, UBO 5)."""
        s = capi.sky_desc(color, faces)
        self._check(self._lib.idkpt_set_sky(self._ctx, ctypes.byref(s)), "idkpt_set_sky")

    def SkyAtmosphere(self, settings=None, face_size=128):
        """AtmosphericScatterer.Compute on the device into the context's sky (DESIGN.md 8f.1j). settings:
        capi.IdkPtAtmosphereSettings (default: the engine's); face_size 128 is the engine's. Returns kernel ms."""
        st = settings if settings is not None else capi.default_atmosphere_settings()
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_sky_atmosphere(self._ctx, ctypes.byref(st), int(face_size), ctypes.byref(ms)), "idkpt_sky_atmosphere")
        return ms.value

    def SkyEquirectangular(self, rgb):
        """SkyBoxManager.LoadSkyBoxEquirectangular's unprojection on the device: rgb float32 [H, W, 3], row 0 first (what
        ImageLoader.Load(path, RGB, true) returns) -> faces of size W // 4 in the context's sky. Returns kernel ms."""
        img = np.ascontiguousarray(rgb, np.float32)
        if img.ndim != 3 or img.shape[2] != 3:
            raise ValueError("SkyEquirectangular: rgb must be [H, W, 3]")
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_sky_equirectangular(self._ctx, img.ctypes.data, img.shape[1], img.shape[0], ctypes.byref(ms)),
                    "idkpt_sky_equirectangular")
        return ms.value

    def read_sky(self):
        """The context's sky faces, float32 [6, n, n, 4] (+X,-X,+Y,-Y,+Z,-Z), or None for a constant sky."""
        n = ctypes.c_int32()
        self._check(self._lib.idkpt_read_sky(self._ctx, ctypes.byref(n), None, 0), "idkpt_read_sky")
        if n.value == 0:
            return None
        faces = np.empty((6, n.value, n.value, 4), np.float32)
        self._check(self._lib.idkpt_read_sky(self._ctx, ctypes.byref(n), faces.ctypes.data, faces.nbytes), "idkpt_read_sky")
        return faces

    def SetFrame(self, per_frame_data):
        """GpuPerFrameData (UBO 1). A changed camera resets the accumulation like Application.OnRender does
        (SRC/Application.cs:209-213)."""
        pf = np.ascontiguousarray(per_frame_data)
        assert pf.dtype == gt.GpuPerFrameData
        if self._frame is not None and pf.tobytes() != self._frame.tobytes():
            self.ResetAccumulation()
        self._frame = pf.copy()

    # ------------------------------------------------------------------ PathTracer surface
    def Compute(self, want_stats=True):
        if self._frame is None:
            raise IdkPtError("SetFrame() has not been called")
        stats = capi.IdkPtStats() if want_stats else None
        rc = self._lib.idkpt_compute(self._ctx, self._frame.ctypes.data, ctypes.byref(self._settings),
                                     ctypes.byref(stats) if want_stats else None)
        self._check(rc, "idkpt_compute")
        self.last_stats = stats
        return stats

    def ComputeAsync(self):
        """Queue one Compute() without waiting (stats == NULL): several samples stay in flight. Sync() waits."""
        if self._frame is None:
            raise IdkPtError("SetFrame() has not been called")
        self._check(self._lib.idkpt_compute(self._ctx, self._frame.ctypes.data, ctypes.byref(self._settings), None), "idkpt_compute")

    def StreamHandle(self):
        """cudaStream_t of the main (image) stream, e.g. for torch.cuda.ExternalStream."""
        h = ctypes.c_void_p()
        self._check(self._lib.idkpt_stream_handle(self._ctx, ctypes.byref(h)), "idkpt_stream_handle")
        return h.value

    def Sync(self):
        self._check(self._lib.idkpt_sync(self._ctx), "idkpt_sync")

    def SetSize(self, width, height):
        self._check(self._lib.idkpt_resize(self._ctx, width, height), "idkpt_resize")
        self.width, self.height = width, height

    def ResetAccumulation(self):
        self._check(self._lib.idkpt_reset_accumulation(self._ctx), "idkpt_reset_accumulation")

    @property
    def AccumulatedSamples(self):
        return int(self._lib.idkpt_accumulated_samples(self._ctx))

    def _read(self, which):
        img = np.zeros((self.height, self.width, 4), np.float32)
        self._check(self._lib.idkpt_read_result(self._ctx, which, img.ctypes.data, img.nbytes), "idkpt_read_result")
        return img

    @property
    def Result(self):
        return self._read(capi.IDKPT_IMAGE_RESULT)

    @property
    def AlbedoTexture(self):
        return self._read(capi.IDKPT_IMAGE_ALBEDO)

    @property
    def NormalTexture(self):
        return self._read(capi.IDKPT_IMAGE_NORMAL)

    def WriteResult(self, img, which=capi.IDKPT_IMAGE_RESULT, accumulated=None):
        img = np.ascontiguousarray(img, np.float32)
        self._check(self._lib.idkpt_write_result(self._ctx, which, img.ctypes.data, img.nbytes), "idkpt_write_result")
        if accumulated is not None:
            self._check(self._lib.idkpt_set_accumulated_samples(self._ctx, accumulated), "idkpt_set_accumulated_samples")

    def PresentAsync(self, host_ptr, nbytes, which=capi.IDKPT_IMAGE_RESULT):
        """Start copying the image of the last Compute() into host memory (pinned for full overlap) on a second stream;
        the next Compute() overlaps the transfer. PresentWait() blocks until it has landed."""
        self._check(self._lib.idkpt_present_async(self._ctx, which, host_ptr, nbytes), "idkpt_present_async")

    def PresentWait(self):
        self._check(self._lib.idkpt_present_wait(self._ctx), "idkpt_present_wait")

    def RegisterHostBuffer(self, host_ptr, nbytes):
        """Page-lock an engine-owned host buffer (e.g. the shared-memory frame every rank presents its stripes into)."""
        self._check(self._lib.idkpt_register_host_buffer(self._ctx, host_ptr, nbytes), "idkpt_register_host_buffer")

    def UnregisterHostBuffer(self, host_ptr):
        self._check(self._lib.idkpt_unregister_host_buffer(self._ctx, host_ptr), "idkpt_unregister_host_buffer")

    def EnablePeerGather(self, rank, world, exchange):
        """Multi-GPU: fuse the tile all-gather into Compute() over NVLink peer memory. `exchange(bytes) -> list[bytes]`
        must return every rank's blob in rank order (e.g. torch.distributed.all_gather_object)."""
        buf = (ctypes.c_uint8 * capi.IDKPT_GATHER_HANDLE_BYTES)()
        self._check(self._lib.idkpt_gather_export(self._ctx, buf, len(buf)), "idkpt_gather_export")
        blobs = exchange(bytes(buf))
        assert len(blobs) == world and all(len(b) == capi.IDKPT_GATHER_HANDLE_BYTES for b in blobs)
        allh = (ctypes.c_uint8 * (world * capi.IDKPT_GATHER_HANDLE_BYTES)).from_buffer_copy(b"".join(blobs))
        self._check(self._lib.idkpt_gather_import(self._ctx, rank, world, allh, len(allh)), "idkpt_gather_import")

    @staticmethod
    def ConnectPeers(tracers):
        """Single-process multi-GPU: wire the tile contexts (in tile order) to each other without IPC (idkpt_gather_connect)."""
        arr = (ctypes.c_void_p * len(tracers))(*[t._ctx.value for t in tracers])
        rc = tracers[0]._lib.idkpt_gather_connect(arr, len(tracers))
        if rc != 0:
            msgs = [t._lib.idkpt_last_error(t._ctx) for t in tracers]
            raise IdkPtError("idkpt_gather_connect failed (%d): %s" % (rc, "; ".join(m.decode() for m in msgs if m)))

    def GatheredDevicePtr(self):
        return self._device_ptr("idkpt_gather_device_ptr")

    def ResultDevicePtr(self, which=capi.IDKPT_IMAGE_RESULT):
        return self._device_ptr("idkpt_result_device_ptr", which)

    def TileRows(self):
        n = ctypes.c_int32()
        self._lib.idkpt_tile_rows(self._ctx, ctypes.byref(n), None, 0)
        rows = np.zeros(n.value, np.int32)
        self._lib.idkpt_tile_rows(self._ctx, ctypes.byref(n), rows.ctypes.data, n.value)
        return rows

    def EnableWavefrontExport(self, on=True):
        self._export = on
        self._check(self._lib.idkpt_read_wavefront_rays(self._ctx, None, 1 if on else 0), "idkpt_read_wavefront_rays")

    def ReadWavefrontRays(self):
        rays = np.zeros(self.width * self.height, gt.GpuWavefrontRay)
        self._check(self._lib.idkpt_read_wavefront_rays(self._ctx, rays.ctypes.data, len(rays)), "idkpt_read_wavefront_rays")
        return rays

    def TraceRays(self, rays, trace_lights=False):
        """Stand-alone closest-hit batch (GPU analogue of BVH.Intersect, SRC/Bvh/BVH.cs:162-193)."""
        rays = np.ascontiguousarray(rays)
        assert rays.dtype == gt.IdkPtRay
        hits = np.zeros(len(rays), gt.IdkPtHit)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_trace_rays(self._ctx, rays.ctypes.data, len(rays), int(trace_lights),
                                               hits.ctypes.data, ctypes.byref(ms)), "idkpt_trace_rays")
        return hits, ms.value

    def TraceRaysAny(self, rays, trace_lights=False):
        """Any-hit / occlusion batch (TraceRayAny, BVHIntersect.glsl:299-411). hits["NodePairFetches"] == 1 where occluded."""
        rays = np.ascontiguousarray(rays)
        assert rays.dtype == gt.IdkPtRay
        hits = np.zeros(len(rays), gt.IdkPtHit)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_trace_rays_any(self._ctx, rays.ctypes.data, len(rays), int(trace_lights),
                                                   hits.ctypes.data, ctypes.byref(ms)), "idkpt_trace_rays_any")
        return hits, ms.value

    def ShadowsRayTraced(self, frame, depth, normal_rg, light_index, samples=1, noise_index=0, jitter=(0.0, 0.0), visibility=None):
        """PointShadowManager.ComputeRayTracedShadowMaps for one light: visibility image from a G-buffer (host arrays)."""
        h, w = depth.shape
        depth = np.ascontiguousarray(depth, np.float32)
        nrg = np.ascontiguousarray(normal_rg, np.float32)
        vis = np.zeros((h, w), np.float32) if visibility is None else np.ascontiguousarray(visibility, np.float32)
        frame = np.ascontiguousarray(frame)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_shadows_ray_traced(self._ctx, frame.ctypes.data, depth.ctypes.data, nrg.ctypes.data, w, h, light_index,
                                                       samples, noise_index, self._jitter(jitter), vis.ctypes.data, ctypes.byref(ms)),
                    "idkpt_shadows_ray_traced")
        return vis, ms.value

    # ---- point-shadow cube maps (PointShadowManager.UpdateBuffer / RenderShadowMaps)
    def SetPointShadows(self, shadows, sizes):
        """GpuPointShadow records (gpu_types.GpuPointShadow) and the face size of each cube map. Same sizes as the last call:
        the maps are kept; otherwise they are reallocated and cleared to 65535."""
        shadows = np.ascontiguousarray(shadows, gt.GpuPointShadow)
        sizes = np.ascontiguousarray(sizes, np.int32)
        assert len(shadows) == len(sizes)
        self._point_shadow_sizes = [int(n) for n in sizes]
        self._check(self._lib.idkpt_set_point_shadows(self._ctx, shadows.ctypes.data if len(shadows) else None,
                                                      sizes.ctypes.data if len(sizes) else None, len(shadows)), "idkpt_set_point_shadows")

    def RenderPointShadows(self, first=0, count=None, face_masks=None):
        """Renders shadows [first, first + count) (default: all set ones); face_masks: one 6-bit mask per shadow (None = all
        faces). Returns the kernel time in ms."""
        if count is None:
            count = len(getattr(self, "_point_shadow_sizes", [])) - first
        masks = None if face_masks is None else np.ascontiguousarray(face_masks, np.uint32)
        if masks is not None:
            assert len(masks) == count
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_render_point_shadows(self._ctx, first, count, masks.ctypes.data if masks is not None else None,
                                                         ctypes.byref(ms)), "idkpt_render_point_shadows")
        return ms.value

    def ReadPointShadow(self, index):
        """One shadow's cube map as uint16 [6, N, N] (face +X,-X,+Y,-Y,+Z,-Z; row y = t; D16, 65535 = nothing)."""
        n = self._point_shadow_sizes[index] if 0 <= index < len(getattr(self, "_point_shadow_sizes", [])) else 1
        out = np.zeros((6, n, n), np.uint16)
        self._check(self._lib.idkpt_read_point_shadow(self._ctx, index, out.ctypes.data, out.nbytes), "idkpt_read_point_shadow")
        return out

    def PointShadowDevicePtr(self, index):
        return self._device_ptr("idkpt_point_shadow_device_ptr", index)

    # ---- volumetric lighting (VolumetricLighting.Compute)
    def VolumetricLighting(self, frame, depth, width, height, settings=None, jitter=None, download=True):
        """Volumetric point-light scattering through the point-shadow cube maps at width x height from the G-buffer depth
        (float32 [Hg, Wg], any size). settings: capi.IdkPtVolumetricSettings (default: the engine's). Returns float16
        [height, width, 4], or None with download=False (the image stays on the device: VolumetricDevicePtr). The kernel time
        in ms is left in last_volumetric_ms."""
        st = settings if settings is not None else capi.default_volumetric_settings()
        d = np.ascontiguousarray(depth, np.float32)
        frame = np.ascontiguousarray(frame)
        out = np.zeros((height, width, 4), np.float16) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_volumetric_lighting(self._ctx, frame.ctypes.data, ctypes.byref(st), d.ctypes.data, d.shape[1], d.shape[0],
                                                        width, height, self._jitter(jitter), out.ctypes.data if download else None,
                                                        ctypes.byref(ms)), "idkpt_volumetric_lighting")
        self.last_volumetric_ms = ms.value
        return out

    def VolumetricDevicePtr(self):
        """(device pointer, bytes) of the last VolumetricLighting image (rgba16f)."""
        return self._device_ptr("idkpt_volumetric_device_ptr")

    # ---- the ray-traced shadows and the volumetric light on a G-buffer (host or device)
    @classmethod
    def gbuffer_arg(cls, gbuffer):
        """A G-buffer argument: a capi.IdkPtGBuffer as it is, or GBufferDevicePtrs()'s (IdkPtGBuffer, velocity) pair, or the
        arrays (depth, normal_rg, albedo, metallic_roughness, emissive; trailing ones may be left out, None for one the call
        does not read) marshalled like the raster calls' arrays. Returns (IdkPtGBuffer, the arrays to keep alive)."""
        if isinstance(gbuffer, capi.IdkPtGBuffer):
            return gbuffer, None
        if isinstance(gbuffer, (tuple, list)) and gbuffer and isinstance(gbuffer[0], capi.IdkPtGBuffer):
            return gbuffer[0], None
        arrays = list(gbuffer) + [None] * (5 - len(gbuffer))
        g, _, keep = cls._gbuffer(arrays, [1, 2, 3, 2, 3])
        return g, keep

    def ShadowsRayTracedGBuffer(self, frame, gbuffer, light_index, slot, samples=1, noise_index=0, jitter=None, download=True):
        """ShadowsRayTraced on a G-buffer (gbuffer_arg: Depth and NormalRG are read) into the context's visibility image of
        `slot` (0 .. capi.IDKPT_MAX_POINT_SHADOWS - 1), which DeferredLighting takes as rt_visibility through ShadowsDevicePtr.
        Pixels with depth 1 keep the slot image's values (0 in a new image). Returns float32 [H, W], or None with
        download=False. Kernel ms in last_shadows_ms."""
        g, keep = self.gbuffer_arg(gbuffer)
        frame = np.ascontiguousarray(frame)
        out = np.zeros((g.Height, g.Width), np.float32) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_shadows_ray_traced_gbuffer(self._ctx, frame.ctypes.data, ctypes.byref(g), light_index, samples, noise_index,
                                                               self._jitter(jitter), slot, out.ctypes.data if download else None,
                                                               ctypes.byref(ms)), "idkpt_shadows_ray_traced_gbuffer")
        self.last_shadows_ms = ms.value
        return out

    def ShadowsDevicePtr(self, slot):
        """(device pointer, bytes) of the last ShadowsRayTracedGBuffer image of `slot` (float32 [H, W])."""
        return self._device_ptr("idkpt_shadows_device_ptr", slot)

    def VolumetricLightingGBuffer(self, frame, gbuffer, width, height, settings=None, jitter=None, download=True):
        """VolumetricLighting with the depth of a G-buffer (gbuffer_arg: only Depth is read, at the G-buffer's size). Returns
        float16 [height, width, 4], or None with download=False (VolumetricDevicePtr). Kernel ms in last_volumetric_ms."""
        st = settings if settings is not None else capi.default_volumetric_settings()
        g, keep = self.gbuffer_arg(gbuffer)
        frame = np.ascontiguousarray(frame)
        out = np.zeros((height, width, 4), np.float16) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_volumetric_lighting_gbuffer(self._ctx, frame.ctypes.data, ctypes.byref(st), ctypes.byref(g), width, height,
                                                                self._jitter(jitter), out.ctypes.data if download else None,
                                                                ctypes.byref(ms)), "idkpt_volumetric_lighting_gbuffer")
        self.last_volumetric_ms = ms.value
        return out

    # ---- the raster passes' marshalling
    @staticmethod
    def _gbuffer(arrays, channels):
        """The input images of a raster call: [H, W] (channels 1) or [H, W, c] arrays, or None; the first one sets H and W. numpy
        arrays are passed as host arrays, CUDA torch tensors in place (OnDevice = 1). Returns (IdkPtGBuffer over the first five,
        every array's pointer (None for None), the contiguous arrays to keep alive)."""
        on_device = type(arrays[0]).__module__.startswith("torch")
        if on_device and not all(a is None or (type(a).__module__.startswith("torch") and a.is_cuda) for a in arrays):
            raise TypeError("G-buffer: pass either all numpy arrays or all CUDA tensors")
        if on_device:
            import torch
        keep = []
        for a, c in zip(arrays, channels):
            if a is None:
                keep.append(None)
                continue
            keep.append(a.to(torch.float32).contiguous() if on_device else np.ascontiguousarray(a, np.float32))
            # the library copies or reads W * H * c floats of every array: a smaller one must never reach it
            want = tuple(keep[0].shape[:2]) + (() if c == 1 else (c,))
            if tuple(keep[-1].shape) != want or keep[0].ndim < 2:
                raise ValueError(f"G-buffer array of shape {tuple(keep[-1].shape)}: expected {want} (H and W from the first array)")
        h, w = keep[0].shape[:2]
        if on_device:   # the library's stream does not wait for torch's: let the tensors' producers finish
            torch.cuda.synchronize(keep[0].device)
        ptrs = [None if a is None else (a.data_ptr() if on_device else a.ctypes.data) for a in keep]
        return capi.IdkPtGBuffer(w, h, int(on_device), *ptrs[:5]), ptrs, keep

    @staticmethod
    def _jitter(jitter):
        """taaDataUBO.Jitter in NDC units as the two floats the library reads, or None (no jitter)."""
        if jitter is None:
            return None
        jit = np.ascontiguousarray(jitter, np.float32)
        if jit.size != 2:
            raise ValueError(f"jitter has two components, not {jit.size}")
        return (ctypes.c_float * 2)(*jit.ravel())

    # ---- G-buffer lighting (SSAO.Compute, the deferred lighting draw)
    def Ssao(self, frame, depth, normal_rg, settings=None, download=True):
        """SSAO.Compute on a G-buffer (depth [H, W], octahedral normal [H, W, 2]; numpy arrays or CUDA tensors). settings:
        capi.IdkPtSsaoSettings (default: the engine's). Returns uint8 [H, W] (R8Unorm), or None with download=False (the image
        stays on the device: SsaoDevicePtr, and DeferredLighting's IsSSAO reads it). Kernel ms in last_ssao_ms."""
        st = settings if settings is not None else capi.default_ssao_settings()
        g, _, keep = self._gbuffer([depth, normal_rg], [1, 2])
        frame = np.ascontiguousarray(frame)
        out = np.zeros((g.Height, g.Width), np.uint8) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_ssao(self._ctx, frame.ctypes.data, ctypes.byref(st), ctypes.byref(g), out.ctypes.data if download else None,
                                         ctypes.byref(ms)), "idkpt_ssao")
        self.last_ssao_ms = ms.value
        return out

    def SsaoDevicePtr(self):
        """(device pointer, bytes) of the last Ssao image (R8Unorm)."""
        return self._device_ptr("idkpt_ssao_device_ptr")

    def DeferredLighting(self, frame, depth, normal_rg, albedo, metallic_roughness, emissive, settings=None, jitter=None, indirect=None,
                         rt_visibility=None, download=True, vrs=False):
        """The deferred lighting pass on a G-buffer (depth [H, W], normal [H, W, 2], albedo [H, W, 3], metallic/roughness [H, W, 2],
        emissive [H, W, 3]; numpy arrays or CUDA tensors, and indirect ([H, W, 4], IsVXGI) and rt_visibility (one [H, W] image
        per point shadow, ShadowMode RayTraced) of the same kind). settings: capi.IdkPtDeferredSettings (default: the engine's).
        vrs=True sets IsVariableRateShading: the pass shades under the rate image of the last ShadingRate call (which must have
        the G-buffer's size). Returns float32 [H, W, 4] (alpha 1), or None with download=False (DeferredDevicePtr). Kernel ms
        in last_deferred_ms."""
        st = settings if settings is not None else capi.default_deferred_settings()
        if vrs:
            st = capi.IdkPtDeferredSettings.from_buffer_copy(st)
            st.IsVariableRateShading = 1
        rt = list(rt_visibility) if rt_visibility is not None else []
        g, ptrs, keep = self._gbuffer([depth, normal_rg, albedo, metallic_roughness, emissive, indirect] + rt, [1, 2, 3, 2, 3, 4] + [1] * len(rt))
        rt_ptrs = (ctypes.c_void_p * max(len(rt), 1))(*ptrs[6:])
        frame = np.ascontiguousarray(frame)
        out = np.zeros((g.Height, g.Width, 4), np.float32) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_deferred_lighting(self._ctx, frame.ctypes.data, ctypes.byref(st), ctypes.byref(g), self._jitter(jitter),
                                                      ptrs[5], rt_ptrs if rt else None, len(rt), out.ctypes.data if download else None,
                                                      ctypes.byref(ms)), "idkpt_deferred_lighting")
        self.last_deferred_ms = ms.value
        return out

    def DeferredDevicePtr(self):
        """(device pointer, bytes) of the last DeferredLighting image (rgba32f)."""
        return self._device_ptr("idkpt_deferred_device_ptr")

    # ---- the G-buffer pass (RasterPipeline.Render's "Fill G-Buffer" draws)
    GBUFFER_CHANNELS = (1, 2, 3, 2, 3, 2)   # depth, normal_rg, albedo, metallic_roughness, emissive, velocity_rg

    def GBuffer(self, frame, width, height, jitter=None, prev_positions=None, download=True):
        """Renders the G-buffer pass at width x height (DESIGN.md 8f.1g). jitter: taaDataUBO.Jitter in NDC units (None = 0);
        prev_positions: the previous frame's vertex positions, float32 [VertexPositionCount, 3], "kept" for the positions
        SkinVertices keeps on the device (PrevPositionsDevicePtr, read in place), or None for this frame's. Returns
        (depth [h, w], normal_rg [h, w, 2], albedo [h, w, 3], metallic_roughness [h, w, 2], emissive [h, w, 3], velocity_rg
        [h, w, 2]) as float32 numpy arrays, or None with download=False (the images stay on the device: GBufferDevicePtrs).
        Kernel ms in last_gbuffer_ms."""
        jit = self._jitter(jitter)
        if isinstance(prev_positions, str):
            if prev_positions != "kept":
                raise ValueError(f"GBuffer: prev_positions {prev_positions!r}: expected an array, 'kept' or None")
            prev_ptr = self.PrevPositionsDevicePtr()[0]
        else:
            prev = None if prev_positions is None else np.ascontiguousarray(prev_positions, np.float32)
            if prev is not None and (prev.ndim != 2 or prev.shape[1] != 3 or prev.shape[0] != self._vertex_position_count):
                raise ValueError(f"GBuffer: prev_positions {prev.shape}: expected ({self._vertex_position_count}, 3)")
            prev_ptr = prev.ctypes.data if prev is not None else None
        frame = np.ascontiguousarray(frame)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_gbuffer(self._ctx, frame.ctypes.data, width, height, jit, prev_ptr, ctypes.byref(ms)), "idkpt_gbuffer")
        self.last_gbuffer_ms = ms.value
        if not download:
            return None
        out = [np.zeros((height, width) if c == 1 else (height, width, c), np.float32) for c in self.GBUFFER_CHANNELS]
        self._check(self._lib.idkpt_read_gbuffer(self._ctx, *[a.ctypes.data for a in out]), "idkpt_read_gbuffer")
        return tuple(out)

    def PrevPositionsDevicePtr(self):
        """(device pointer, bytes) of the previous vertex positions SkinVertices keeps (prevVertexPositionSSBO: PackedVec3 per
        vertex position), valid until SetScene or Dispose."""
        return self._device_ptr("idkpt_prev_positions_device_ptr")

    def GBufferDevicePtrs(self, tensors=False):
        """The images of the last GBuffer call: (capi.IdkPtGBuffer with OnDevice = 1, velocity device pointer), or with
        tensors=True zero-copy CUDA tensors (depth, normal_rg, albedo, metallic_roughness, emissive, velocity_rg) over them,
        valid until the next GBuffer call with another size or SetScene."""
        g, v = capi.IdkPtGBuffer(), ctypes.c_void_p()
        self._check(self._lib.idkpt_gbuffer_device_ptrs(self._ctx, ctypes.byref(g), ctypes.byref(v)), "idkpt_gbuffer_device_ptrs")
        if not tensors:
            return g, v.value
        import torch
        from .multigpu import DeviceArray
        h, w = g.Height, g.Width
        ptrs = [g.Depth, g.NormalRG, g.AlbedoRGB, g.MetallicRoughness, g.EmissiveRGB, v.value]
        dev = torch.device("cuda", self._device)
        return tuple(torch.as_tensor(DeviceArray(p, (h, w) if c == 1 else (h, w, c)), device=dev)
                     for p, c in zip(ptrs, self.GBUFFER_CHANNELS))

    # ---- transparency (RasterPipeline.Render's "Record transparent fragments" + "Resolve transparent fragments")
    def Transparency(self, frame, depth, settings=None, jitter=None, color=None, source=None, voxelizer=None, cone=None,
                     download=True):
        """Ray-casts the blended layers along the G-buffer pass's rays, lights them and composites them front to back over the
        lit image, in place (DESIGN.md 8f.1h). depth: the opaque depth [H, W] (numpy array or CUDA tensor). The lit image is
        `color` (rgba32f [H, W, 4] of the same kind, LIT_SOURCE_ARRAY: composited in place, a numpy array included) or the
        last DeferredLighting image (LIT_SOURCE_DEFERRED: later DEFERRED reads see the composite). settings:
        capi.IdkPtTransparencySettings (default: the engine's); IsVXGI traces `voxelizer` (a voxelised vxgi.Voxelizer on the
        same device) with `cone` (vxgi.IdkVxConeSettings, default: the engine's). Returns the composited float32 [H, W, 4], or
        None with download=False. Kernel ms in last_transparency_ms."""
        st = settings if settings is not None else capi.default_transparency_settings()
        src = self._lit_source(source, color)
        g, ptrs, keep = self._gbuffer([depth, None, None, None, None, color], [1, 2, 3, 2, 3, 4])
        jit = self._jitter(jitter)
        cn = None
        if st.IsVXGI:
            from . import vxgi
            cn = cone if cone is not None else vxgi.default_cone_settings()
        frame = np.ascontiguousarray(frame)
        out = np.zeros((g.Height, g.Width, 4), np.float32) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_transparency(self._ctx, frame.ctypes.data, ctypes.byref(st), ctypes.byref(g), jit,
                                                 voxelizer._ctx if voxelizer is not None else None,
                                                 ctypes.byref(cn) if cn is not None else None, src, ptrs[5],
                                                 out.ctypes.data if download else None, ctypes.byref(ms)), "idkpt_transparency")
        self.last_transparency_ms = ms.value
        if color is not None and keep[5] is not color:
            if g.OnDevice:
                color.copy_(keep[5])
            else:
                np.copyto(color, keep[5], casting="unsafe")
        return out

    # ---- the light spheres and the skybox (RasterPipeline.Render's "Draw lights" + "Draw skybox")
    def LightsAndSkybox(self, frame, jitter=None, download=True):
        """Draws the light spheres and the skybox into the images of the last GBuffer call and the last DeferredLighting image
        (which must have the G-buffer's size), in place (DESIGN.md 8f.1i): later DEFERRED reads, GBufferDevicePtrs and
        GBuffer downloads see them. jitter: taaDataUBO.Jitter in NDC units (None = 0). Returns the lit image, float32 [H, W, 4],
        or None with download=False. Kernel ms in last_lights_and_skybox_ms."""
        jit = self._jitter(jitter)
        frame = np.ascontiguousarray(frame)
        out = None
        if download:
            g, _ = self.GBufferDevicePtrs()
            out = np.zeros((g.Height, g.Width, 4), np.float32)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_lights_and_skybox(self._ctx, frame.ctypes.data, jit, out.ctypes.data if download else None,
                                                      ctypes.byref(ms)), "idkpt_lights_and_skybox")
        self.last_lights_and_skybox_ms = ms.value
        return out

    # ---- variable-rate deferred lighting (LightingShadingRateClassifier.Compute)
    def ShadingRate(self, frame, velocity_rg, settings=None, color=None, source=None, download=True, debug=False):
        """LightingShadingRateClassifier.Compute over render-size inputs: velocity [h, w, 2] and the lit image `color` (rgba32f
        [h, w, 4]; LIT_SOURCE_ARRAY) or the last DeferredLighting image (LIT_SOURCE_DEFERRED); numpy arrays or CUDA tensors.
        frame's DeltaRenderTime divides the mean speed. settings: capi.IdkPtShadingRateSettings (default: the engine's). Returns
        the rate image, uint8 [ceil(h/16), ceil(w/16)] palette indices (capi.VRS_PALETTE), or None with download=False (the
        image stays on the device: ShadingRateDevicePtr, and DeferredLighting(vrs=True) reads it). debug=True (DebugMode 2..4)
        returns (rates, float32 debug image of the same size) instead. Kernel ms in last_shading_rate_ms."""
        st = settings if settings is not None else capi.default_shading_rate_settings()
        src = self._lit_source(source, color)
        g, ptrs, keep = self._gbuffer([velocity_rg, color], [2, 4])
        h, w = g.Height, g.Width
        inputs = capi.IdkPtShadingRateInputs(w, h, g.OnDevice, src, *ptrs)
        tiles = ((h + capi.VRS_TILE - 1) // capi.VRS_TILE, (w + capi.VRS_TILE - 1) // capi.VRS_TILE)
        rates = np.zeros(tiles, np.uint8) if download else None
        dbg = np.zeros(tiles, np.float32) if debug else None
        frame = np.ascontiguousarray(frame)
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_shading_rate(self._ctx, frame.ctypes.data, ctypes.byref(st), ctypes.byref(inputs),
                                                 rates.ctypes.data if download else None, dbg.ctypes.data if debug else None,
                                                 ctypes.byref(ms)), "idkpt_shading_rate")
        self.last_shading_rate_ms = ms.value
        return (rates, dbg) if debug else rates

    def ShadingRateDevicePtr(self):
        """(device pointer, bytes) of the last ShadingRate image (R8 palette indices, [ceil(h/16)][ceil(w/16)])."""
        return self._device_ptr("idkpt_shading_rate_device_ptr")

    # ---- the end of the raster frame (SSR.Compute, "Merge Textures", TaaResolve.Compute)
    @staticmethod
    def _lit_source(source, color):
        """The lit-image selector: ARRAY when a colour array is given, DEFERRED otherwise, unless `source` says."""
        if source is None:
            return capi.LIT_SOURCE_ARRAY if color is not None else capi.LIT_SOURCE_DEFERRED
        if (source == capi.LIT_SOURCE_ARRAY) != (color is not None):
            raise ValueError("a colour array goes with LIT_SOURCE_ARRAY, and only with it")
        return source

    def Ssr(self, frame, depth, normal_rg, albedo, metallic_roughness, settings=None, color=None, source=None, download=True):
        """SSR.Compute and the "Merge Textures" dispatch on a G-buffer (depth [H, W], normal [H, W, 2], albedo [H, W, 3],
        metallic/roughness [H, W, 2]; numpy arrays or CUDA tensors). The lit image is `color` (rgba32f [H, W, 4] of the same
        kind; LIT_SOURCE_ARRAY) or the last DeferredLighting image (LIT_SOURCE_DEFERRED). settings: capi.IdkPtSsrSettings
        (default: the engine's). Returns (merged float32 [H, W, 4], ssr float16 [H, W, 4]), or None with download=False (the
        images stay on the device: SsrDevicePtrs, and TaaResolve's LIT_SOURCE_MERGED reads the merged one). Kernel ms in
        last_ssr_ms."""
        st = settings if settings is not None else capi.default_ssr_settings()
        src = self._lit_source(source, color)
        g, ptrs, keep = self._gbuffer([depth, normal_rg, albedo, metallic_roughness, None, color], [1, 2, 3, 2, 3, 4])
        frame = np.ascontiguousarray(frame)
        merged = np.zeros((g.Height, g.Width, 4), np.float32) if download else None
        ssr = np.zeros((g.Height, g.Width, 4), np.float16) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_ssr(self._ctx, frame.ctypes.data, ctypes.byref(st), ctypes.byref(g), src, ptrs[5],
                                        merged.ctypes.data if download else None, ssr.ctypes.data if download else None,
                                        ctypes.byref(ms)), "idkpt_ssr")
        self.last_ssr_ms = ms.value
        return (merged, ssr) if download else None

    def SsrDevicePtrs(self):
        """((merged device pointer, bytes), (SSR device pointer, bytes)) of the last Ssr images (rgba32f, rgba16f)."""
        pm, ps, nm, ns = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_uint64()
        self._check(self._lib.idkpt_ssr_device_ptrs(self._ctx, ctypes.byref(pm), ctypes.byref(ps), ctypes.byref(nm), ctypes.byref(ns)),
                    "idkpt_ssr_device_ptrs")
        return (pm.value, nm.value), (ps.value, ns.value)

    def TaaResolve(self, depth, velocity_rg, width, height, settings=None, color=None, source=None, download=True):
        """TaaResolve.Compute at width x height (the presentation size) over render-size inputs: depth [h, w], velocity [h, w, 2]
        and the lit image `color` (rgba32f [h, w, 4]; LIT_SOURCE_ARRAY), or the last DeferredLighting (LIT_SOURCE_DEFERRED) or
        merged Ssr image (LIT_SOURCE_MERGED); numpy arrays or CUDA tensors. settings: capi.IdkPtTaaSettings (default: the
        engine's). The history is the context's. Returns float16 [height, width, 4], or None with download=False
        (TaaDevicePtr). Kernel ms in last_taa_ms."""
        st = settings if settings is not None else capi.default_taa_settings()
        src = self._lit_source(source, color)
        g, ptrs, keep = self._gbuffer([depth, velocity_rg, color], [1, 2, 4])
        inputs = capi.IdkPtTaaInputs(g.Width, g.Height, g.OnDevice, src, *ptrs)
        out = np.zeros((height, width, 4), np.float16) if download else None
        ms = ctypes.c_float()
        self._check(self._lib.idkpt_taa_resolve(self._ctx, ctypes.byref(st), ctypes.byref(inputs), width, height,
                                                out.ctypes.data if download else None, ctypes.byref(ms)), "idkpt_taa_resolve")
        self.last_taa_ms = ms.value
        return out

    def TaaDevicePtr(self):
        """(device pointer, bytes) of the image the last TaaResolve wrote (rgba16f)."""
        return self._device_ptr("idkpt_taa_device_ptr")

    # ---- properties with the reference's reset-on-set behaviour
    def _reset_prop(name, sub=None):  # noqa: N805
        def get(self):
            return getattr(self._settings.Gpu if sub else self._settings, name)

        def set_(self, v):
            setattr(self._settings.Gpu if sub else self._settings, name, v)
            self.ResetAccumulation()
        return property(get, set_)

    def _plain_prop(name):  # noqa: N805
        def get(self):
            return getattr(self._settings, name)

        def set_(self, v):
            setattr(self._settings, name, v)
        return property(get, set_)

    RayDepth = _reset_prop("RayDepth")                          # PathTracer.cs:16-25
    FocalLength = _reset_prop("FocalLength", True)              # :39-48
    LenseRadius = _reset_prop("LenseRadius", True)              # :50-59
    DoDebugBVHTraversal = _reset_prop("DoDebugBVHTraversal", True)  # :61-71
    DoTraceLights = _reset_prop("DoTraceLights", True)          # :73-84
    DoRussianRoulette = _reset_prop("DoRussianRoulette", True)  # :86-97
    SamplesPerPixel = _plain_prop("SamplesPerPixel")            # :12
    DoRaySorting = _plain_prop("DoRaySorting")                  # :101-111
    OutputAOVs = _plain_prop("OutputAOVs")                      # :113-125
    CollectStats = _plain_prop("CollectStats")

    def GetGpuSettings(self):
        return self._settings.Gpu
