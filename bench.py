#!/usr/bin/env python
"""bench.py -- Mrays/s of the wavefront path tracer on the Sponza-sized synthetic atrium, 1920x1080, 8 bounces.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

One "step" = one PathTracer.Compute() (1 sample per pixel, RayDepth 9) over the whole frame. With N GPUs the frame is
cut into 8-row stripes dealt round-robin to the ranks (scene replicated), followed by ONE all-gather of tile radiance.
Rank 0 prints ONE JSON line (see DESIGN.md "Measurement" for every field).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)

WORKLOAD_TRIS = 262144
WIDTH, HEIGHT = 1920, 1080
RAY_DEPTH = 9            # RayDepth = 1 + bounces (PathTracer.cs:228)
STRIPE = 8
SKY = (0.6, 0.7, 0.9)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--width", type=int, default=WIDTH)
    ap.add_argument("--height", type=int, default=HEIGHT)
    ap.add_argument("--tris", type=int, default=WORKLOAD_TRIS)
    ap.add_argument("--ray-depth", type=int, default=RAY_DEPTH)
    ap.add_argument("--sort", type=int, default=0)
    ap.add_argument("--workload", default="bench", choices=["bench", "config3", "config4"],
                    help="bench = BASELINE configs[1] scene at the headline depth (default); config3 = 9 M triangles 1080p sort on; "
                         "config4 = 3.9 M rotated triangles 3840x2160 (the 2/4/8-GPU configuration of BASELINE.json)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-parity", action="store_true", help="skip the CPU-oracle check of the first sample (the GPU-side digests still run)")
    ap.add_argument("--no-vxgi", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the image the timed path returned for its last step to DIR/*.npy (float32)")
    ap.add_argument("--global-slots", action="store_true",
                    help="N > 1: IDKPT_CREATE_GLOBAL_SLOTS -- per-bounce exchange of per-stripe alive counts over NVLink, the N-GPU image is "
                         "bit-identical to the 1-GPU image (SURVEY 8e option ii); parity_check then compares against a 1-GPU frame")
    return ap.parse_args()


def measured_peaks():
    p = os.path.join(REPO, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet 3.35 TB/s)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown," \
        "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, device):
        self.device = device
        self.proc = None
        self.path = None

    def start(self):
        try:
            f = tempfile.NamedTemporaryFile("w", suffix=".csv", delete=False)
            self.path = f.name
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(self.device)], stdout=f, stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for line in open(self.path):
            p = [x.strip() for x in line.split(",")]
            if len(p) < 9:
                continue
            try:
                sm.append(float(p[1]))
                mx.append(float(p[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), p[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        os.unlink(self.path)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(max(mx)), "reasons": sorted(reasons), "samples": len(sm)}


def gpu_info(device):
    """The card a number was measured on: name and power limit (a power-capped card runs lower clocks)."""
    import torch
    info = {"name": torch.cuda.get_device_name(device), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(device)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def build_scene(args):
    from idkengine_b200 import scenes
    if args.workload == "config3":
        args.tris, args.sort = 9_000_000, 1
        scene, cam = scenes.atrium(args.tris)
    elif args.workload == "config4":
        args.tris, args.width, args.height = 3_900_000, 3840, 2160
        scene, cam = scenes.street_canyon(args.tris)
    else:
        scene, cam = scenes.atrium(args.tris)
    frame = scenes.camera_frame(cam, args.width, args.height)
    return scene, cam, frame


def workload_config(args, world, scene):
    info = scene.build_info[0]
    return {
        "workload": f"{'street-canyon' if args.workload == 'config4' else 'atrium'}-{args.tris // 1000}k ({'Sponza-sized synthetic' if args.workload == 'bench' else 'BASELINE ' + args.workload}, seed 0x1D4E) {args.width}x{args.height} RayDepth {args.ray_depth} "
                    f"({args.ray_depth - 1} bounces) 1spp RR on, sort {'on' if args.sort else 'off'}, constant sky, constant textures",
        "triangles": int(info["source_triangles"]), "blas_triangles": int(info["triangles"]), "blas_nodes": int(info["nodes"]),
        "blas_stack_size": int(scene.blas_stack_size),
        "parallelism": f"screen tiles: {STRIPE}-row stripes round-robin over {world} GPU(s), scene replicated, tile gather fused into "
                       f"FinalDraw over NVLink peer memory (IDKPT_GATHER=nccl: one NCCL all-gather per frame)",
        "slots": ("global (IDKPT_CREATE_GLOBAL_SLOTS): per-stripe alive counts exchanged over NVLink every bounce, image == 1-GPU image"
                  if (getattr(args, "global_slots", False) and world > 1) else "tile-local (one collective per frame; image reproducible per GPU count)"),
        "l2": "per-step working set (2x64B path state + hits, ~330 MB at 1080p) exceeds the 50 MB L2; the 22 MB BVH is "
              "re-read every bounce and is L2-resident by design (SURVEY 8d)",
    }


# ----------------------------------------------------------------------------------------------- reference arm (CPU)
def run_reference(args, rank, world):
    """The reference's path on the host cores: the CPU restatement (oracle port: FirstHit/NHit/FinalDraw + BVHIntersect, all
    threads of a persistent pool with dynamic chunking) on the same workload. Each step = the WHOLE frame, one sample (on a
    box with fewer than 32 cores: 1/8 of the frame as an interleaved stripe tile, so that the run stays within minutes)."""
    if rank != 0:
        return
    sys.path.insert(0, os.path.join(REPO, "tests"))
    import oracle_lib as ol
    from idkengine_b200 import capi
    scene, cam, frame = build_scene(args)
    s = capi.default_settings()
    s.RayDepth = args.ray_depth
    s.DoRaySorting = args.sort
    threads = os.cpu_count() or 1
    tile = (STRIPE, 0, 1) if threads >= 32 else (STRIPE, 0, 8)
    img = np.zeros((args.height, args.width, 4), np.float32)
    acc, rays, secs = 0, 0, 0.0
    per_step = []
    for i in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        o = ol.path_trace(scene, frame, s, args.width, args.height, sky=SKY, tile=tile, accumulated=acc, result=img,
                          want_rays=False, threads=threads)
        dt = time.perf_counter() - t0
        acc = o.accumulated
        if i >= args.warmup:
            rays += o.stats.Rays
            secs += dt
            per_step.append(o.stats.Rays / dt / 1e6)
    value = rays / secs / 1e6
    sample = (f"{'the whole frame' if tile[2] == 1 else '1/8 of the frame (stripe tile %s)' % (tile,)} per step, {args.steps} steps, {rays} rays; "
              f"per-step Mrays/s min {min(per_step):.2f} / median {float(np.median(per_step)):.2f} / max {max(per_step):.2f}")
    line = {
        "impl": "reference", "metric": "Mrays/s Sponza-sized synthetic 1920x1080 8-bounce", "value": value, "unit": "Mrays/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": secs / args.steps * 1e3,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args, 1, scene),
        "cpu_baseline": {"value": value, "unit": "Mrays/s", "cores": threads, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": "Mrays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


def cpu_baseline(scene, frame, args):
    """The reference's own CPU traversal shape, Gui.Test (Gui.cs:1484-1503): one primary ray per pixel through
    BVH.Intersect -> BLAS.Intersect (C# semantics), rows in parallel on every host core."""
    sys.path.insert(0, os.path.join(REPO, "tests"))
    import oracle_lib as ol
    threads = os.cpu_count() or 1
    rays = ol.gui_test_rays(frame, args.width, args.height)
    best = None
    for _ in range(3):
        _, secs = ol.cpu_intersect(scene, rays, threads=threads, want_hits=False)
        best = secs if best is None else min(best, secs)
    return {"value": len(rays) / best / 1e6, "unit": "Mrays/s", "cores": threads, "kind": "port",
            "sample": f"{len(rays)} primary rays (one full {args.width}x{args.height} frame, Gui.Test shape), best of 3, "
                      f"restated BVH.Intersect/BLAS.Intersect (C# semantics)"}


# ----------------------------------------------------------------------------------------------- our arm (GPU)
def digest(arr):
    import hashlib
    return hashlib.sha1(np.ascontiguousarray(arr).tobytes()).hexdigest()[:16]


class HostFrame:
    """The frame the engine presents from: two full rgba32f images in host memory that EVERY rank can write.
    world == 1: plain pinned memory. world > 1: one POSIX shared-memory segment mapped by all ranks and page-locked in each
    (idkpt_register_host_buffer); every rank then delivers its own stripes over its own PCIe link."""

    def __init__(self, pt, height, width, rank, world, dist, rows=None):
        import torch
        self.pt, self.rank, self.world = pt, rank, world
        self.bytes_per_image = height * width * 16
        self.shm = None
        if world == 1:
            self.t = torch.empty((2, height, width, 4), dtype=torch.float32).pin_memory()
            self.np = self.t.numpy()
            self.base = self.t.data_ptr()
        else:
            from multiprocessing import shared_memory
            name = [None]
            if rank == 0:
                self.shm = shared_memory.SharedMemory(create=True, size=2 * self.bytes_per_image)
                name[0] = self.shm.name
            dist.broadcast_object_list(name, src=0)
            if rank != 0:
                self.shm = shared_memory.SharedMemory(name=name[0])
                try:      # only the creating rank owns the segment: keep Python's resource tracker from "cleaning it up" at exit
                    from multiprocessing import resource_tracker
                    resource_tracker.unregister(self.shm._name, "shared_memory")
                except Exception:
                    pass
            self.np = np.ndarray((2, height, width, 4), np.float32, buffer=self.shm.buf)
            # first touch decides the NUMA node of a page: every rank touches ITS OWN stripes (8 rows x 1920 x 16 B = 60 pages each),
            # so that its GPU's DMA writes land in the memory of the socket it hangs off instead of all on rank 0's node
            if rows is not None:
                self.np[:, rows] = 0.0
            dist.barrier()
            self.base = self.np.ctypes.data
            pt.RegisterHostBuffer(self.base, 2 * self.bytes_per_image)

    def ptr(self, k):
        return self.base + (k & 1) * self.bytes_per_image

    def close(self, dist):
        if self.shm is not None:
            self.pt.UnregisterHostBuffer(self.base)
            self.np = None
            dist.barrier()
            self.shm.close()
            if self.rank == 0:
                self.shm.unlink()


def vxgi_record(scene, frame, pt, args):
    """BASELINE configs[4] beside the headline: 384^3 rgba16f voxelise + mip chain + cone trace of the same scene with the
    reference's three lights, timed with the library's CUDA events (best of 3)."""
    from idkengine_b200 import vxgi
    import copy
    sc = copy.copy(scene)
    sc.lights = scene.lights.copy()
    for pos, col in (((-4.5, 5.7, -2.0), (429.8974, 22.459948, 28.425867)), ((-0.5, 5.7, -2.0), (8.773416, 506.7525, 28.425867)),
                     ((4.5, 5.7, -2.0), (8.773416, 22.459948, 533.77466))):      # Application.cs:488-490
        sc.add_light(pos, col, 0.3)
    depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, args.width, args.height)
    peak, _ = measured_peaks()
    with vxgi.Voxelizer(384) as vx:
        vx.SetScene(sc)
        vx.Render()
        best = None
        for _ in range(3):
            st = vx.Render()
            if best is None or st.ClearMs + st.VoxelizeMs + st.MipmapMs < best.ClearMs + best.VoxelizeMs + best.MipmapMs:
                best = st
        cone = None
        for _ in range(3):
            img, cs = vx.ConeTrace(frame, depth, nrg, mr)
            cone = cs if cone is None or cs.ConeTraceMs < cone.ConeTraceMs else cone
        sizes = vx.sizes
    vox = [w * h * d for (w, h, d) in sizes]
    mip_bytes = sum((vox[l - 1] + vox[l]) * 8 for l in range(1, len(vox)))           # unique bytes: read level l-1 once, write level l
    cone_bytes = cone.ConeSteps * 16 * 8                                             # 2 mip levels x 8 texels x 8 B per step
    gbs = lambda b, ms: b / 1e9 / (ms * 1e-3) if ms > 0 else None
    return {"grid": "384^3 rgba16f, 9 levels", "lights": 3, "fragments": int(best.Fragments),
            "clear_ms": best.ClearMs, "voxelize_ms": best.VoxelizeMs, "mipmap_ms": best.MipmapMs, "cone_trace_ms": cone.ConeTraceMs,
            "cone_steps": int(cone.ConeSteps), "cone_resolution": f"{args.width}x{args.height}",
            "clear_gbs": gbs(vox[0] * 8, best.ClearMs), "clear_frac": gbs(vox[0] * 8, best.ClearMs) / peak,
            "mipmap_unique_gbs": gbs(mip_bytes, best.MipmapMs), "mipmap_frac": gbs(mip_bytes, best.MipmapMs) / peak,
            "cone_texel_gbs": gbs(cone_bytes, cone.ConeTraceMs),
            "parity": "tests/test_configs_gpu.py::test_config5_vxgi_384_cubed (every level and the cone image == oracle)"}


DUMP_LIMIT = 64 << 20


def dump_outputs(out_dir, image):
    """image.npy: the rgba32f accumulated image, H x W x 4. A larger image (4K) is written as a fixed sample instead:
    image_sample.npy (n x 4) at the pixels image_sample_index.npy (row-major pixel index, float64), chosen with seed 0."""
    os.makedirs(out_dir, exist_ok=True)
    image = np.ascontiguousarray(image, np.float32)
    if image.nbytes <= DUMP_LIMIT:
        np.save(os.path.join(out_dir, "image.npy"), image)
        return
    flat = image.reshape(-1, image.shape[-1])
    n = DUMP_LIMIT // (flat.shape[1] * 4 + 8)
    idx = np.sort(np.random.default_rng(0).choice(len(flat), n, replace=False))
    np.save(os.path.join(out_dir, "image_sample.npy"), flat[idx])
    np.save(os.path.join(out_dir, "image_sample_index.npy"), idx.astype(np.float64))


def bind_to_gpu_numa_node(local_rank):
    """Best effort: run this rank on the CPUs of the NUMA node its GPU hangs off (its pinned pages and its share of the shared
    host frame are then first-touched there). Returns the node or None."""
    try:
        import torch
        p = torch.cuda.get_device_properties(local_rank)
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return node
    except Exception:
        pass
    return None


def run_ours(args, rank, world, local_rank):
    import torch
    import torch.distributed as dist
    from idkengine_b200 import capi, multigpu
    from idkengine_b200.pathtracer import PathTracer

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device -- libidkpt has no CPU fallback")
    torch.cuda.set_device(local_rank)
    numa_node = bind_to_gpu_numa_node(local_rank) if world > 1 else None
    dev = torch.device("cuda", local_rank)

    scene, cam, frame = build_scene(args)
    s = capi.default_settings()
    s.RayDepth = args.ray_depth
    s.DoRaySorting = args.sort
    tile = (STRIPE, rank, world)
    global_slots = bool(args.global_slots) and world > 1
    if global_slots and (args.sort or os.environ.get("IDKPT_GATHER", "peer") == "nccl"):
        raise SystemExit("bench.py: --global-slots needs the peer-memory gather and no ray sorting")
    pt = PathTracer(args.width, args.height, s, device=local_rank, tile=tile, global_slots=global_slots)
    pt.SetScene(scene)
    pt.SetSky(SKY)
    pt.SetFrame(frame)
    rows = pt.TileRows()
    ptr, nbytes = pt.ResultDevicePtr()
    local = torch.as_tensor(multigpu.DeviceArray(ptr, (len(rows), args.width, 4)), device=dev)
    host = HostFrame(pt, args.height, args.width, rank, world, dist, rows)
    copy_stream = torch.cuda.Stream(device=dev)
    # N > 1: the tile all-gather is fused into Compute() over NVLink peer memory (CUDA IPC); IDKPT_GATHER=nccl selects the
    # torch.distributed all_gather + de-interleave fallback instead.
    peer_gather = world > 1 and os.environ.get("IDKPT_GATHER", "peer") != "nccl"
    gatherer = multigpu.TileGatherer(args.height, args.width, 4, STRIPE, world, dev) if world > 1 else None
    if peer_gather:
        def exchange(blob):
            out = [None] * world
            dist.all_gather_object(out, blob)
            return out
        pt.EnablePeerGather(rank, world, exchange)
        dist.barrier()

    lanes = int(os.environ.get("IDKPT_LANES", "8"))      # the library default
    pipelined = lanes > 1 and (world == 1 or peer_gather)      # the NCCL fallback gathers between steps: one sample at a time

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def step(e2e, k=0):
        """e2e: the frame's GpuPerFrameData goes host->device inside Compute(); the finished image of EVERY step lands in the
        host frame (double-buffered, asynchronously, so the transfer overlaps the next step). With N ranks every rank
        presents its own stripes into the shared host frame (no root download); the NVLink gather still runs inside Compute()."""
        if pipelined:
            pt.ComputeAsync()         # stats == NULL: queued, up to `lanes` samples in flight
            st = None
        else:
            st = pt.Compute()
        if world > 1 and not peer_gather:
            torch.cuda.current_stream().wait_stream(copy_stream)
            gatherer.gather(local)
        if e2e:
            pt.PresentAsync(host.ptr(k), host.bytes_per_image)
        return st

    def e2e_drain():
        pt.PresentWait()
        pt.Sync()

    # ---- stats replay (untimed): exact S/T/I for the sample sequence the timed region will run
    pt.CollectStats = 1
    pt.ResetAccumulation()
    S = T = I = R = H = 0
    compact_slots = 0
    for _ in range(args.steps):
        rs = pt.Compute()
        S += rs.NodePairFetches; T += rs.TriangleTests; I += rs.InstanceVisits; R += rs.Rays; H += rs.Hits
        compact_slots += sum(rs.BounceRays[j] for j in range(args.ray_depth - 1))
    pt.CollectStats = 0

    for k in range(max(args.warmup, 3)):     # warm-up exercises the end-to-end path too (first present allocates the snapshot
        step(True, k)                        # buffer, the copy stream and touches the host pages)
    e2e_drain()

    # ---- timed region 1a: inputs resident in HBM, no read-back, ONE sample at a time with per-kernel CUDA events
    # (the roofline's kernel durations come from here; with pipelining off this is also `value`)
    pt.ResetAccumulation()
    sampler = ClockSampler(local_rank)
    barrier()
    if rank == 0:
        sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms = trav_ms = shade_ms = compact_ms = acc_ms = 0.0
    rays = launches = trav_launches = 0
    gather_ms = 0.0
    t0 = time.perf_counter()
    for _ in range(args.steps):
        st = pt.Compute()
        dev_ms += st.TotalMs; trav_ms += st.TraverseMs; shade_ms += st.ShadeMs; compact_ms += st.CompactMs; acc_ms += st.AccumulateMs
        rays += st.Rays; launches += st.KernelLaunches; trav_launches += st.TraverseLaunches
        if world > 1 and not peer_gather:
            ev0.record()
            gatherer.gather(local)
            ev1.record()
            ev1.synchronize()
            gather_ms += ev0.elapsed_time(ev1)
            launches += 1
        elif world > 1:
            gather_ms += st.OtherMs        # ray-gen + fused accumulate/scatter + arrival wait (inside Compute)
    barrier()
    wall_ms = (time.perf_counter() - t0) * 1e3
    assert rays == R, "timed region traced a different ray set than the stats replay"
    digest_serial = digest(pt.Result[rows])

    # ---- timed region 1b: the same K steps queued asynchronously (several samples in flight). Timed on the device with
    # events on the context's main stream: every sample's FinalDraw runs there in submission order.
    pipe_ms = None
    host_submit_ms = None
    digest_pipelined = None
    if pipelined:
        ext = torch.cuda.ExternalStream(pt.StreamHandle(), device=dev)
        pe0, pe1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        pt.ResetAccumulation()
        barrier()
        pe0.record(ext)
        th0 = time.perf_counter()
        for _ in range(args.steps):
            pt.ComputeAsync()
        host_submit_ms = (time.perf_counter() - th0) * 1e3      # host time to ENQUEUE the K steps (the device must not starve on it)
        pe1.record(ext)
        pt.Sync()
        barrier()
        pipe_ms = pe0.elapsed_time(pe1)
        assert pt.AccumulatedSamples == args.steps
        digest_pipelined = digest(pt.Result[rows])
    timed_image = pt.Result[rows] if args.dump_outputs else None      # what the pass behind `value` returned for its last step

    # ---- timed region 2: end to end through the public API with host buffers (frame H2D, result D2H every step)
    pt.ResetAccumulation()
    host.np[:, rows] = -1.0
    barrier()
    t0 = time.perf_counter()
    for k in range(args.steps):
        step(True, k)
    e2e_drain()
    barrier()
    e2e_ms = (time.perf_counter() - t0) * 1e3
    final_host = host.np[(args.steps - 1) & 1]
    if args.dump_outputs and rank == 0:     # N > 1: the full frame every rank presented into (parity_check: == the timed tiles)
        dump_outputs(args.dump_outputs, timed_image if world == 1 else final_host)

    # ---- parity of what was just timed (untimed). Everything is compared bit for bit.
    #  a) serial pass == pipelined pass == the image the e2e pass left in the host frame (same K samples from a reset);
    #  b) N > 1: the peer-gathered full frame on this GPU == an NCCL all-gather of the ranks' tiles == the shared host frame;
    #  c) the first sample of this rank's tile == the CPU oracle run with the same tile map (the checker, tests/oracle_lib.py).
    parity = {}
    ok_local = digest_serial == (digest_pipelined or digest_serial) == digest(final_host[rows])
    parity["serial_eq_pipelined_eq_host_frame"] = bool(ok_local)
    if world > 1:
        full_nccl = gatherer.gather(local)
        torch.cuda.synchronize()
        same = True
        if peer_gather:
            gp, gb = pt.GatheredDevicePtr()
            full_peer = torch.as_tensor(multigpu.DeviceArray(gp, (args.height, args.width, 4)), device=dev)
            same = bool(torch.equal(full_peer.view(torch.int32), full_nccl.view(torch.int32)))
        dist.barrier()           # every rank's present into the shared frame has completed (e2e_drain) before anyone reads it
        same_host = bool(np.array_equal(final_host.view(np.uint32), full_nccl.cpu().numpy().view(np.uint32)))
        parity["peer_gather_eq_nccl_gather"] = same
        parity["shared_host_frame_eq_gathered"] = same_host
        if global_slots:
            # strict multi-GPU parity: the frame the N ranks just produced == the same K samples traced by ONE GPU (an untiled context)
            with PathTracer(args.width, args.height, s, device=local_rank) as one:
                one.SetScene(scene)
                one.SetSky(SKY)
                one.SetFrame(frame)
                for _ in range(args.steps):
                    one.ComputeAsync()
                one.Sync()
                parity["n_gpu_frame_eq_one_gpu_frame"] = bool(np.array_equal(one.Result.view(np.uint32), full_nccl.cpu().numpy().view(np.uint32)))
    if not args.no_parity:
        sys.path.insert(0, os.path.join(REPO, "tests"))
        import oracle_lib as ol
        pt.ResetAccumulation()
        pt.Compute()
        mine = pt.Result[rows]
        ref = np.zeros((args.height, args.width, 4), np.float32)
        # global slots: the tile must equal the rows of the oracle's WHOLE-image run, not of a tile-local one
        o = ol.path_trace(scene, frame, s, args.width, args.height, sky=SKY, tile=(STRIPE, 0, 1) if global_slots else tile, result=ref, want_rays=False,
                          threads=max(1, (os.cpu_count() or 1) // world))
        parity["first_sample_tile_eq_cpu_oracle"] = bool(np.array_equal(mine.view(np.uint32), ref[rows].view(np.uint32)))
    flags = [bool(v) for v in parity.values()]
    if world > 1:
        t = torch.tensor([1.0 if all(flags) else 0.0], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        parity["all_ranks_ok"] = bool(t.item() == 1.0)
    parity["ok"] = all(bool(v) for v in parity.values())

    def reduce(x, op):
        if world == 1:
            return x
        t = torch.tensor([float(x)], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=op)
        return float(t.item())

    MAX, SUM = (dist.ReduceOp.MAX, dist.ReduceOp.SUM) if world > 1 else (None, None)
    serial_ms = reduce(dev_ms + (0.0 if peer_gather else gather_ms), MAX)     # device time of region 1a, max over ranks
    job_ms = reduce(pipe_ms, MAX) if pipelined else serial_ms                 # device time of the K timed steps, max over ranks
    # nvidia-smi samples every 100 ms but K steps may last only tens of ms: keep the identical load running (untimed) until
    # the sampler has seen ~0.6 s of it, then stop it. The step count is derived from the reduced time, i.e. equal on all ranks.
    extra_steps = int(min(600, max(0, 600.0 / max(job_ms / args.steps, 1e-3) - args.steps)))
    for k in range(extra_steps):
        step(False)
    if pipelined:
        pt.Sync()
    barrier()
    clocks = sampler.stop() if rank == 0 else None
    if clocks is not None:
        clocks["sampled_over"] = f"the {args.steps} timed steps + {extra_steps} identical untimed steps (nvidia-smi -lms 100)"
    per_rank = None
    if world > 1:      # per-rank device times: shows tile imbalance / a slow GPU behind the max-over-ranks figure
        mine = {"rank": rank, "pipelined_total": (pipe_ms / args.steps) if pipelined else None, "total": dev_ms / args.steps, "traverse": trav_ms / args.steps, "shade": shade_ms / args.steps,
                "gather": gather_ms / args.steps, "e2e_wall": e2e_ms / args.steps,
                "host_submit": (host_submit_ms / args.steps) if host_submit_ms is not None else None, "numa_node": numa_node, "rays": rays // args.steps}
        per_rank = [None] * world
        dist.all_gather_object(per_rank, mine)
    total_rays = reduce(rays, SUM)
    total_launches = int(reduce(launches, SUM))
    e2e_ms = reduce(e2e_ms, MAX)
    wall_ms = reduce(wall_ms, MAX)

    if rank == 0:
        peak, peak_src = measured_peaks()
        trav_bytes = 64 * S + 52 * T + 48 * I + 52 * R      # DESIGN.md: algorithmic bytes of k_traverse (rank 0's tile)
        achieved = trav_bytes / (trav_ms * 1e-3) / 1e9
        shade_only_ms = shade_ms - compact_ms
        shade_bytes = (84 + 64) * R + 260 * H              # DESIGN.md section 4: state + hit in, state out, surface / vertex gathers on a hit
        compact_bytes = 8 * compact_slots
        acc_bytes = 48 * len(rows) * args.width * args.steps
        gbs = lambda b, ms: b / (ms * 1e-3) / 1e9 if ms > 0 else None
        line = {
            "metric": "Mrays/s Sponza-sized synthetic 1920x1080 8-bounce", "value": total_rays / (job_ms * 1e-3) / 1e6, "unit": "Mrays/s",
            "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": job_ms / args.steps,
            "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args, world, scene),
            "rays_per_step": total_rays / args.steps,
            "serial_ms_per_step": serial_ms / args.steps,
            "pipeline": (f"{lanes} samples in flight: asynchronous Compute (stats == NULL), per-sample results and accumulation order identical to the "
                         f"serial path" if pipelined else "off: one sample at a time"),
            "wall_ms_per_step": wall_ms / args.steps,
            "host_submit_ms_per_step": (host_submit_ms / args.steps) if host_submit_ms is not None else None,
            "kernel_ms_per_step": {"measured_in": "serial pass (region 1a: one sample in flight, per-kernel CUDA events)", "traverse": trav_ms / args.steps, "shade": shade_only_ms / args.steps,
                                   "compact": compact_ms / args.steps, "accumulate": acc_ms / args.steps,
                                   "all_gather": gather_ms / args.steps, "total_device": dev_ms / args.steps},
            "roofline": {"kernel": "k_traverse2 (bounces) + k_traverse (primary rays)", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                         "frac": achieved / peak,
                         "frac_measured_in": "serial pass of the same K steps: algorithmic bytes / CUDA-event time of the traversal launches",
                         "frac_pipelined": (trav_bytes / (job_ms * 1e-3) / 1e9) / peak if world == 1 else None,
                         "frac_pipelined_is": "the same algorithmic bytes / the WHOLE pipelined step (traversal overlaps the shading of other samples): a lower bound for the kernel, the figure behind `value`",
                         "bound_note": "the BVH (26 MB) is kept L2-resident by a persisting access-policy window: the algorithmic bytes overstate the DRAM traffic",
                         "peak_source": peak_src,
                         "algorithmic_bytes_per_launch": trav_bytes / max(trav_launches, 1),
                         "launch_ms": trav_ms / max(trav_launches, 1),
                         "per_ray": {"node_pair_fetches": S / R, "triangle_tests": T / R, "instances": I / R},
                         "other_kernels": {
                             "k_shade": {"ms_per_step": shade_only_ms / args.steps, "algorithmic_gbs": gbs(shade_bytes, shade_only_ms), "frac": gbs(shade_bytes, shade_only_ms) / peak,
                                         "bytes_per_ray": shade_bytes / R},
                             "k_compact": {"ms_per_step": compact_ms / args.steps, "algorithmic_gbs": gbs(compact_bytes, compact_ms), "frac": (gbs(compact_bytes, compact_ms) or 0) / peak,
                                           "note": "8 launches per sample over 4-byte entries: launch-latency bound"},
                             "k_accumulate": {"ms_per_step": acc_ms / args.steps, "algorithmic_gbs": gbs(acc_bytes, acc_ms), "frac": (gbs(acc_bytes, acc_ms) or 0) / peak}}},
            "e2e": {"value": total_rays / (e2e_ms * 1e-3) / 1e6, "unit": "Mrays/s",
                    "h2d_bytes_per_step": (544 + 44) * world, "d2h_bytes_per_step": args.width * args.height * 16,
                    "how": ("every rank presents its own stripes into ONE shared pinned host frame (POSIX shm registered in every rank): "
                            f"{args.width * args.height * 16 // world} B per rank per step over its own PCIe link" if world > 1 else
                            "full rgba32f frame into pinned host memory every step, overlapping the next Compute")},
            "parity_check": parity,
            "gpu_launches": total_launches,
            "clocks": clocks,
            "gpu": gpu_info(local_rank),
        }
        if per_rank is not None:
            line["per_rank_ms"] = per_rank
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_baseline(scene, frame, args)
        if world == 1 and not args.no_vxgi:
            try:
                line["vxgi"] = vxgi_record(scene, frame, pt, args)
            except Exception as e:      # the headline must not depend on the side record
                line["vxgi"] = {"error": repr(e)}
        print(json.dumps(line))
    host.close(dist)
    pt.Dispose()


def main():
    args = parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        run_ours(args, rank, world, local_rank)
    finally:
        if world > 1:
            import torch.distributed as dist
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
