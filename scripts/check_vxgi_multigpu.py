"""torchrun check of the multi-GPU VXGI path (SURVEY 8e): z-slab voxelisation + one NCCL all-gather + replicated mip chain +
row-tiled cone trace on N GPUs == the single-GPU result on rank 0 (every level, the whole cone-trace image), with timings.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 scripts/check_vxgi_multigpu.py [size]
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from idkengine_b200 import capi, multigpu, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
size = int(sys.argv[1]) if len(sys.argv) > 1 else 384
scene, cam = scenes.atrium(262144)
w, h = 1920, 1080
frame = scenes.camera_frame(cam, w, h)
with PathTracer(64, 64, device=local) as pt:
    pt.SetScene(scene)
    depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, w, h)
for light in scenes.STARTUP_LIGHTS:
    scene.add_light(*light)
with vxgi.Voxelizer(size, device=local) as vx:
    vx.SetScene(scene)
    multigpu.voxelize_multi_gpu(vx, rank, world, dev)          # warm-up (allocations, NCCL channels)
    torch.cuda.synchronize(); (dist.barrier() if world > 1 else None)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    st, mst = multigpu.voxelize_multi_gpu(vx, rank, world, dev)
    e1.record(); e1.synchronize()
    total_ms = e0.elapsed_time(e1)
    # screen-tiled cone trace: ONE contiguous band of rows per rank (8-row stripes would be 68 tail-bound launches of 240 CTAs)
    r0, r1 = multigpu.slab_range(h, rank, world)
    out, cs = vx.ConeTraceRows(frame, depth[r0:r1], nrg[r0:r1], mr[r0:r1], h, int(r0))
    cone_ms, steps = cs.ConeTraceMs, cs.ConeSteps
    if world > 1:
        bands = [torch.empty((slab_range[1] - slab_range[0], w, 4), dtype=torch.float32, device=dev) for slab_range in (multigpu.slab_range(h, r, world) for r in range(world))]
        dist.all_gather(bands, torch.as_tensor(out, device=dev))
        gathered = torch.cat(bands).cpu().numpy()
    else:
        gathered = out
    levels = [vx.ReadLevel(l) for l in range(len(vx.sizes))]
    ok = True
    if rank == 0:
        with vxgi.Voxelizer(size, device=local) as ref:          # the single-GPU result
            ref.SetScene(scene)
            rst = ref.Render()
            for l in range(len(ref.sizes)):
                ok = ok and np.array_equal(ref.ReadLevel(l).view(np.uint16), levels[l].view(np.uint16))
            full, rcs = ref.ConeTrace(frame, depth, nrg, mr)
            ok = ok and np.array_equal(full, gathered)
        print(json.dumps({"check": "vxgi multi-GPU == single GPU (all levels, cone-trace image)", "ok": bool(ok), "n_gpus": world, "grid": size,
                          "voxelize_slab_ms_rank0": st.VoxelizeMs, "mipmap_ms": mst.MipmapMs, "voxelize_gather_mip_wall_ms": total_ms,
                          "cone_trace_ms_rank0": cone_ms, "single_gpu": {"voxelize_ms": rst.VoxelizeMs, "mipmap_ms": rst.MipmapMs, "cone_trace_ms": rcs.ConeTraceMs}}))
if world > 1:
    dist.destroy_process_group()
