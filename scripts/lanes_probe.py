"""Asynchronous Compute: throughput vs number of lanes, full frame and a 1/8 tile (the per-GPU share at N=8)."""
import json, os, sys, time
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch
import bench
from idkengine_b200 import capi
from idkengine_b200.pathtracer import PathTracer

sys.argv = sys.argv[:1]
args = bench.parse_args()
scene, cam, frame = bench.build_scene(args)
out = {}
K = 40
for tname, tile in (("full", (8, 0, 1)), ("eighth", (8, 0, 8))):
    for lanes in (1, 2, 3, 4, 6, 8):
        s = capi.default_settings(); s.RayDepth = args.ray_depth
        pt = PathTracer(args.width, args.height, s, device=0, tile=tile, lanes=lanes)
        pt.SetScene(scene); pt.SetSky(bench.SKY); pt.SetFrame(frame)
        rays = pt.Compute().Rays
        ext = torch.cuda.ExternalStream(pt.StreamHandle())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for rep in range(2):
            pt.ResetAccumulation()
            torch.cuda.synchronize()
            e0.record(ext)
            for _ in range(K if rep else 8):
                pt.ComputeAsync() if lanes > 1 else pt.Compute(want_stats=False)
            e1.record(ext)
            pt.Sync()
        ms = e0.elapsed_time(e1) / K
        key = f"{tname}_lanes{lanes}"
        out[key] = {"ms_per_sample": ms, "mrays_s": rays / ms / 1e3}
        print(key, out[key], flush=True)
        pt.Dispose()
json.dump(out, open("gpurun_out/lanes_probe.json", "w"), indent=1)
