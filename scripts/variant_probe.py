"""A/B harness for kernel experiments: build libidkpt with -D switches into side files (CPU), then
time every variant on the GPU in its own process (same scene, same samples) and check that all of them produce the
same image and the same S/T/I counters as the default build.

    python scripts/variant_probe.py --build name:-DIDK_REG_STACK=2 name2:-DIDK_TRI_STRIDE=3   (build machine)
    python scripts/variant_probe.py --run [--eighth]                                             (GPU machine)
"""
import hashlib
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
VDIR = os.path.join(REPO, "idkengine_b200", "csrc", "variants")


def build(specs):
    from idkengine_b200 import build as b
    os.makedirs(VDIR, exist_ok=True)
    srcs = b._sources(b.CSRC_DIR, (".cu",))
    srcs = [s for s in srcs if os.sep + "variants" + os.sep not in s]
    for spec in specs:
        name, _, flags = spec.partition(":")
        out = os.path.join(VDIR, f"libidkpt_{name}.so")
        cmd = [b.find_nvcc()] + b.NVCC_FLAGS + [f for f in flags.split(",") if f] + ["-I", b.INCLUDE_DIR, "-I", b.CSRC_DIR, "-o", out] + srcs
        print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)


def child(eighth):
    import torch
    import bench
    from idkengine_b200 import capi
    from idkengine_b200.pathtracer import PathTracer
    sys.argv = sys.argv[:1]
    args = bench.parse_args()
    scene, cam, frame = bench.build_scene(args)
    out = {"lib": os.path.basename(os.environ.get("IDKPT_LIB", "default"))}
    tiles = (("full", (8, 0, 1)),) + ((("eighth", (8, 0, 8)),) if eighth else ())
    for tname, tile in tiles:
        s = capi.default_settings()
        s.RayDepth = args.ray_depth
        pt = PathTracer(args.width, args.height, s, device=0, tile=tile)
        pt.SetScene(scene); pt.SetSky(bench.SKY); pt.SetFrame(frame)
        pt.CollectStats = 1
        st = pt.Compute()
        pt.CollectStats = 0
        out[tname + "_counters"] = [st.Rays, st.NodePairFetches, st.TriangleTests, st.InstanceVisits]
        out[tname + "_image"] = hashlib.sha1(pt.Result.tobytes()).hexdigest()[:16]
        for _ in range(3):
            pt.Compute()
        pt.ResetAccumulation()
        K = 10
        acc = {"TotalMs": 0.0, "TraverseMs": 0.0, "ShadeMs": 0.0}
        bt = [0.0] * args.ray_depth
        for _ in range(K):
            st = pt.Compute()
            for k in acc:
                acc[k] += getattr(st, k) / K
            for j in range(args.ray_depth):
                bt[j] += st.BounceTraverseMs[j] / K
        out[tname + "_serial"] = {k: round(v, 4) for k, v in acc.items()}
        out[tname + "_bounce_traverse_us"] = [round(v * 1e3, 1) for v in bt]
        ext = torch.cuda.ExternalStream(pt.StreamHandle())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        KP = 40
        for rep in range(2):
            pt.ResetAccumulation()
            torch.cuda.synchronize()
            e0.record(ext)
            for _ in range(KP if rep else 8):
                pt.ComputeAsync()
            e1.record(ext)
            pt.Sync()
        out[tname + "_pipelined_ms"] = round(e0.elapsed_time(e1) / KP, 4)
        out[tname + "_image40"] = hashlib.sha1(pt.Result.tobytes()).hexdigest()[:16]
        pt.Dispose()
    print("VARIANT " + json.dumps(out), flush=True)


def run(eighth):
    libs = [None] + sorted(os.path.join(VDIR, f) for f in os.listdir(VDIR) if f.endswith(".so")) if os.path.isdir(VDIR) else [None]
    jobs = [(lib, {}) for lib in libs]
    if "--sweep" in sys.argv:      # scheduling thresholds of the default build (IDKPT_TUNE_SETUP / IDKPT_TUNE_LEAF)
        jobs += [(None, {"IDKPT_PACK_CTA": str(v)}) for v in (0, 2, 4)]
    results = []
    for lib, extra in jobs:
        env = dict(os.environ)
        env.update(extra)
        if lib:
            env["IDKPT_LIB"] = lib
        else:
            env.pop("IDKPT_LIB", None)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"] + (["--eighth"] if eighth else []), env=env, capture_output=True, text=True)
        for line in p.stderr.splitlines():
            if "phase stats" in line:
                print(extra, line, flush=True)
        for line in p.stdout.splitlines():
            if line.startswith("VARIANT "):
                r = json.loads(line[8:])
                r["env"] = extra
                results.append(r)
        if p.returncode:
            print("FAILED", lib, p.stderr[-2000:], flush=True)
    ref = results[0] if results else None
    for r in results:
        r["same_as_default"] = all(r.get(k) == ref.get(k) for k in r if k.endswith(("_counters", "_image", "_image40")))
        print(json.dumps({k: v for k, v in r.items() if not k.endswith(("_counters", "_image", "_image40"))}), flush=True)
    os.makedirs(os.path.join(REPO, "gpurun_out"), exist_ok=True)
    json.dump(results, open(os.path.join(REPO, "gpurun_out", "variant_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    if "--build" in sys.argv:
        build(sys.argv[sys.argv.index("--build") + 1:])
    elif "--child" in sys.argv:
        child("--eighth" in sys.argv)
    else:
        run("--eighth" in sys.argv)
