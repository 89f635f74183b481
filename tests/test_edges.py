"""Traversal at its edges, CPU only: the oracle's closest-hit and any-hit queries against an independent float64 reference
(tests/edge_lib.py) on a battery of legal edge rays (axis-parallel and in-plane rays with +0.0 / -0.0, origins on node
planes, rays at vertices and shared edges, rays in a wall's plane, t == 0, boundary TMax, denormal and unnormalised
directions, far origins) plus random rays. A robust disagreement outside the slab-test artefact class is a bug."""
import numpy as np
import pytest

import edge_lib as el
import oracle_lib as ol
from idkengine_b200 import scenes

SCENES = ["cornell", "multi_blas", "multi_blas_tlas", "atrium_small"]


@pytest.fixture(scope="module")
def multi_blas_tlas():
    scene, cam = scenes.multi_blas(threads=1)
    scene.build_tlas()
    return scene, cam


def battery(scene, seed=7, n_random=20000):
    tris = el.world_triangles(scene)
    rays = np.concatenate([el.edge_rays(scene, seed, tris=tris), el.random_rays(n_random, scene, seed + 1, tris=tris)])
    return rays, tris


def check(scene, rays, hits, ref, any_hit, label):
    c = el.classify(scene, rays, hits, ref, any_hit=any_hit)
    print(f"{label}: {len(rays)} rays, robust hits {len(c['robust_hit'])}, robust misses {len(c['robust_miss'])}, "
          f"artefact class {len(c['artefact'])} (culled {len(c['culled'])}), robust disagreements {len(c['bad'])}")
    assert len(c["bad"]) == 0, (label, c["bad"][:10], rays[c["bad"][:5]], hits[c["bad"][:5]])
    return c


@pytest.mark.parametrize("name", SCENES)
def test_oracle_against_float64_reference(name, request):
    scene, _ = request.getfixturevalue(name)
    rays, tris = battery(scene)
    lights = [False, True] if len(scene.lights) else [False]
    for tl in lights:
        ref = el.ref64_closest(scene, rays, trace_lights=tl, tris=tris)
        c = check(scene, rays, ol.trace_rays(scene, rays, trace_lights=tl), ref, False, f"{name} closest lights={tl}")
        check(scene, rays, ol.trace_rays_any(scene, rays, trace_lights=tl), ref, True, f"{name} any lights={tl}")
        # the battery reaches both outcomes robustly, and the edge kinds are not all judged ambiguous
        assert len(c["robust_hit"]) > 0.2 * len(rays) and len(c["robust_miss"]) > 0
    assert el.artefact_class(scene, rays).sum() >= 50     # origins land exactly on node planes with a zero component


@pytest.mark.parametrize("name", SCENES)
def test_float64_reference_matches_brute_force_away_from_edges(name, request):
    """ref64 self-check: on random rays, wherever the float64 verdict is robust, the oracle's float32 brute force (every
    triangle, no BVH) agrees with it -- same hit / miss, the hit triangle in the lenient set, T within the bounds."""
    scene, _ = request.getfixturevalue(name)
    tris = el.world_triangles(scene)
    rays = el.random_rays(5000, scene, 99, tris=tris)
    ref = el.ref64_closest(scene, rays, tris=tris)
    bf = ol.brute_force(scene, rays)
    bf["NodePairFetches"] = 0
    c = check(scene, rays, bf, ref, False, f"{name} brute force")
    judged = len(c["robust_hit"]) + len(c["robust_miss"])
    assert judged > 0.99 * len(rays)            # random rays are almost never near an edge
