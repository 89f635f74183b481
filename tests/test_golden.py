"""Committed golden fixtures (tests/golden/path_trace_golden.json, made by tests/golden/make_golden.py from the oracle):
the oracle must keep reproducing them on CPU, and the CUDA path must hit the same digests on the GPU."""
import importlib.util
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "golden", "make_golden.py"))
mg = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mg)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "path_trace_golden.json")))


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_oracle_reproduces_golden(name):
    assert mg.run_case(GOLDEN[name]["case"]) == GOLDEN[name]["expect"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_gpu_reproduces_golden(name):
    from idkengine_b200 import scenes
    from idkengine_b200.pathtracer import PathTracer
    c, exp = GOLDEN[name]["case"], GOLDEN[name]["expect"]
    scene, cam = getattr(scenes, c["scene"])(threads=1)
    with PathTracer(c["w"], c["h"], mg.settings_for(c)) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.6, 0.7, 0.9))
        pt.SetFrame(scenes.camera_frame(cam, c["w"], c["h"]))
        pt.CollectStats = 1
        st = pt.Compute()
        assert mg.digest(pt.Result) == exp["result"]
        if c["aov"]:
            assert mg.digest(pt.AlbedoTexture) == exp["albedo"] and mg.digest(pt.NormalTexture) == exp["normal"]
        assert st.Rays == exp["rays"] and list(st.BounceRays)[: c["depth"]] == exp["bounce_rays"]
        assert st.NodePairFetches == exp["node_pair_fetches"] and st.TriangleTests == exp["triangle_tests"]


# next_rows_golden.json pins the present chain ("ldr", "ldr_mean") with Prefilter on bloom down levels 0 and 1, the two
# dispatches of Bloom.cs that upload Lod 0.
NEXT = json.load(open(os.path.join(HERE, "golden", "next_rows_golden.json")))


def test_oracle_reproduces_next_rows_golden_two_prefiltered_bloom_levels():
    assert mg.next_rows_expect() == NEXT


@pytest.mark.gpu
def test_gpu_reproduces_next_rows_golden_two_prefiltered_bloom_levels():
    from idkengine_b200 import capi
    from idkengine_b200.pathtracer import PathTracer
    x = mg.next_rows_inputs()
    scene = x["scene"]
    with PathTracer(80, 54) as pt:
        pt.SetScene(scene)
        vis, _ = pt.ShadowsRayTraced(x["frame"], x["depth"], x["nrg"], 0, samples=3, noise_index=6)
        anyh, _ = pt.TraceRaysAny(x["rays"], trace_lights=True)
        pt.WriteResult(x["hdr"])
        ldr, _ = pt.PostProcess()
        pt.SetSkinningData(x["unskinned"])
        pt.SkinVertices(x["joints"], x["cmd"])
        pt.BlasRefit(2, 1)
        pos = pt.ReadRange(capi.IDKPT_ARRAY_VERTEX_POSITIONS, 0, len(scene.positions))
        vtx = pt.ReadRange(capi.IDKPT_ARRAY_VERTICES, 0, len(scene.vertices))
        nodes = pt.ReadRange(capi.IDKPT_ARRAY_BLAS_NODES, 0, len(scene.blas_nodes))
    got = dict(shadows=mg.digest(vis), any_hit_flags=mg.digest(anyh["NodePairFetches"]), any_hit_t=mg.digest(anyh["T"]), ldr=mg.digest(ldr),
               skinned_positions=mg.digest(pos.view(np.float32)), skinned_vertices=mg.digest(vtx.view(np.uint32)),
               refit_nodes=mg.digest(nodes.view(np.uint32)))
    for k, v in got.items():
        assert v == NEXT[k], k
