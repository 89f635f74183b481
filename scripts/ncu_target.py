"""Small, fixed workloads for ncu captures (one process, few launches): `pt` = two synchronous samples of the bench workload
(sample 2's launches are the ones captured), `vxgi` = one voxelise + mip + cone trace at 384^3 / 1080p."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from idkengine_b200 import capi, scenes, vxgi  # noqa: E402
from idkengine_b200.pathtracer import PathTracer  # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "pt"
sys.argv = sys.argv[:1]
args = bench.parse_args()
scene, cam, frame = bench.build_scene(args)
s = capi.default_settings()
s.RayDepth = args.ray_depth
with PathTracer(args.width, args.height, s) as pt:
    pt.SetScene(scene); pt.SetSky(bench.SKY); pt.SetFrame(frame)
    if what == "pt":
        pt.Compute()
        pt.Compute()
    else:
        depth, nrg, mr = vxgi.synth_gbuffer(pt, scene, frame, args.width, args.height)
        for light in scenes.STARTUP_LIGHTS:
            scene.add_light(*light)
        with vxgi.Voxelizer(384) as vx:
            vx.SetScene(scene)
            vx.Render()
            vx.ConeTrace(frame, depth, nrg, mr)
