"""Can two samples in flight hide the tail-bounce latency? Emulated with several contexts on one GPU, one host thread
each (idkpt_compute blocks, ctypes releases the GIL). Reports aggregate Mrays/s per context count."""
import json, os, sys, threading, time
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import bench
from idkengine_b200 import capi
from idkengine_b200.pathtracer import PathTracer

sys.argv = sys.argv[:1]
args = bench.parse_args()
scene, cam, frame = bench.build_scene(args)
K = 24
out = {}

def run(name, nctx, tile):
    s = capi.default_settings(); s.RayDepth = args.ray_depth
    pts = []
    for _ in range(nctx):
        pt = PathTracer(args.width, args.height, s, device=0, tile=tile)
        pt.SetScene(scene); pt.SetSky(bench.SKY); pt.SetFrame(frame)
        pts.append(pt)
    rays = [0] * nctx
    def worker(i, n):
        for _ in range(n):
            rays[i] += pts[i].Compute().Rays
    for n in (3, K):
        rays = [0] * nctx
        th = [threading.Thread(target=worker, args=(i, n)) for i in range(nctx)]
        t0 = time.perf_counter()
        for t in th: t.start()
        for t in th: t.join()
        dt = time.perf_counter() - t0
    out[name] = {"mrays_s": sum(rays) / dt / 1e6, "ms_per_sample": dt * 1e3 / (K * nctx)}
    print(name, out[name], flush=True)
    for pt in pts: pt.Dispose()

full, eighth = (8, 0, 1), (8, 0, 8)
run("full_1ctx", 1, full)
run("full_2ctx", 2, full)
run("full_3ctx", 3, full)
run("eighth_1ctx", 1, eighth)
run("eighth_2ctx", 2, eighth)
run("eighth_4ctx", 4, eighth)
json.dump(out, open("gpurun_out/overlap_probe.json", "w"), indent=1)
