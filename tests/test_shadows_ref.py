"""The ray-traced point-shadow pass on the CPU oracle against the float64 restatement of tests/shadow_ref64.py: light sizes
from a 0.5 sphere down to a 0.001 one at distances 1 to 4 (and the verdict's independence of the light's slot), a light
that contains the fragment, another light's sphere in the way, penumbrae, masked and textured cut-out occluders, stacks of
blended panes around the 0.01 early stop and the 0.001 step, surfaces facing away, instanced geometry through the
instance loop and the TLAS, and the jitter, noise index and sample count settings. tests/test_shadows_ref_gpu.py holds
the device to the same bounds."""
import numpy as np
import pytest

import oracle_lib as ol
import pt_ref64 as pr
import shadow_ref64 as s6
import surface_ref64 as sr
from idkengine_b200 import scenes

W, H = 64, 48
SEED = 7.0                       # the visibility a depth == 1 pixel keeps
STAGE_CAM = dict(position=(0.0, 2.2, 3.2), view_dir=(0.0, -0.55, -1.0), fov_y_deg=60.0)
# lights no sample ray of the stage can reach: far below the floor, off to the sides
FAR_LIGHTS = [((40.0, -30.0, 40.0), (1.0, 1.0, 1.0), 0.2), ((-40.0, -30.0, 35.0), (1.0, 1.0, 1.0), 0.3)]


def light(pos, radius):
    return (pos, (10.0, 10.0, 10.0), radius)


def stage(lights, parts=(), specs=()):
    """A floor, a back wall and two boxes (mesh 0 grey, mesh 1 brown), plus `parts` ((positions, indices), mesh) whose
    meshes are 2, 3, ... with materials `specs`."""
    base = [dict(color=(0.7, 0.7, 0.7)), dict(color=(0.6, 0.3, 0.2))]
    geo = [(pr.floor(3.0), 0), (scenes.quad([-3, 0, -2], [3, 0, -2], [3, 3, -2], [-3, 3, -2]), 0),
           (pr.box_faces([-0.9, 0.0, -0.6], [-0.3, 0.7, 0.0]), 1), (pr.box_faces([0.3, 0.0, 0.2], [0.6, 1.2, 0.5]), 1)]
    return pr.build(geo + list(parts), base + list(specs), lights=lights)


def open_floor(lights, parts=(), specs=()):
    """A floor and a back wall only, plus `parts` (meshes 1, 2, ...)."""
    geo = [(pr.floor(3.0), 0), (scenes.quad([-3, 0, -2], [3, 0, -2], [3, 3, -2], [-3, 3, -2]), 0)]
    return pr.build(geo + list(parts), [dict(color=(0.7, 0.7, 0.7))] + list(specs), lights=lights)


def horizontal(y, x0=-1.0, x1=1.0, z0=-1.2, z1=0.8):
    """One triangle at height y that covers [x0, x1] x [z0, z1] with its edges outside it, so no ray through the rectangle
    passes near an edge (the ray test is double-sided)."""
    m = 0.5
    p = np.array([[x0 - m, y, z0 - m], [x0 - m, y, 2 * z1 - z0 + 3 * m], [2 * x1 - x0 + 3 * m, y, z0 - m]], np.float32)
    return p, np.array([[0, 1, 2]], np.uint32)


def gbuffer(scene, cam, w, h):
    frame = scenes.camera_frame(cam, w, h)
    depth, nrg, _ = ol.synth_gbuffer(scene, frame, w, h)
    return frame, depth, nrg


def oracle(scene, frame, depth, nrg, li, samples=4, noise_index=0, jitter=(0.0, 0.0)):
    seed = np.full(depth.shape, SEED, np.float32)
    return ol.shadows_ray_traced(scene, frame, depth, nrg, li, samples, noise_index, jitter, visibility=seed)


def judge(got, scene, frame, depth, nrg, li, tag, min_share, s64=None, **kw):
    """got against the float64 restatement; depth == 1 pixels must keep SEED. Returns the reference."""
    assert np.all(got[depth == 1.0] == SEED), tag
    ref = s6.shadows_ref(s64 or s6.Scene64(scene), frame, depth, nrg, li, **kw)
    s6.check(got, ref, tag, min_share)
    return ref


def run(scene, cam, li, tag, min_share=0.9, w=W, h=H, gscene=None, **kw):
    """The oracle on the G-buffer of gscene (default: the scene itself; the G-buffer pass leaves blended and cut-out cards
    out, so the tests that shadow with them take it from the scene without them) and its judgement."""
    frame, depth, nrg = gbuffer(gscene or scene, cam, w, h)
    got = oracle(scene, frame, depth, nrg, li, **kw)
    return got, judge(got, scene, frame, depth, nrg, li, tag, min_share, **kw)


# --------------------------------------------------------------------------------------------- light sizes and slots
RADII = (0.5, 0.05, 0.004, 0.001)
DISTANCES = (1.0, 2.5, 4.0)


def slot_scenes(radius, dist):
    """The same light at index 0 and at index 2 (behind two that no ray reaches)."""
    L = light((0.1, dist, -0.2), radius)
    return stage([L] + FAR_LIGHTS), stage(FAR_LIGHTS + [L])


@pytest.mark.parametrize("radius", RADII)
def test_light_radius_sweep_and_slot(radius):
    """A sample's verdict does not depend on which slot the light has. With the engine's float32 SampleSphere the sqrt's
    argument rounds below zero for small, far lights (radius 0.004 and 0.001 here), the distance is NaN, and the failed
    trace reads as a hit on light 0: visible when the light is light 0, occluded otherwise."""
    for dist in DISTANCES:
        s0, s2 = slot_scenes(radius, dist)
        frame, depth, nrg = gbuffer(s0, STAGE_CAM, W, H)
        v0 = oracle(s0, frame, depth, nrg, 0, samples=16)
        v2 = oracle(s2, frame, depth, nrg, 2, samples=16)
        assert np.array_equal(v0.view(np.uint32), v2.view(np.uint32)), (radius, dist, int((v0 != v2).sum()))
        ref = judge(v0, s0, frame, depth, nrg, 0, "radius %g distance %g" % (radius, dist), 0.9, samples=16)
        assert (ref["want"][ref["judged"]] == 0.0).sum() > 100 and (ref["want"][ref["judged"]] == 1.0).sum() > 100


def test_light_containing_the_fragment():
    """Fragments inside the light's sphere have a negative distance to it: nothing is traced and the sample is visible."""
    c, r = np.array([0.1, 0.25, 0.3]), 0.5
    scene = open_floor([light(tuple(c), r)])
    got, ref = run(scene, STAGE_CAM, 0, "inside the light", samples=4)
    frame, depth, nrg = gbuffer(scene, STAGE_CAM, W, H)
    P, _ = s6.frag_positions(frame, depth, (0.0, 0.0))
    inside = (np.linalg.norm(P + np.array([0.0, s6.BIAS, 0.0]) - c, axis=1) < r - 1e-3).reshape(H, W) & (depth < 1.0)
    assert inside.sum() > 50 and ref["judged"][inside].sum() > 25
    assert np.all(got[inside] == 1.0)


def test_another_light_in_the_way():
    """A second light's sphere between the fragment and the shadowed light occludes it (0, not 'visible')."""
    scene = open_floor([light((0.0, 3.0, 0.0), 0.3), light((0.2, 1.2, 0.1), 0.25)])
    got, ref = run(scene, STAGE_CAM, 0, "another light in the way", samples=8)
    j = ref["judged"] & ref["lit"]
    assert (got[j] == 0.0).sum() > 50 and ((got[j] > 0.0) & (got[j] < 1.0)).sum() > 20
    # the pixels the second light darkens see the first one without it
    alone = open_floor([light((0.0, 3.0, 0.0), 0.3)])
    got1, ref1 = run(alone, STAGE_CAM, 0, "the same light alone", samples=8)
    assert (j & ref1["judged"] & (got == 0.0) & (got1 == 1.0)).sum() > 10


def test_penumbra():
    """An opaque box partly covers a large light: judged pixels hold k / n exactly across the penumbra."""
    got, ref = run(stage([light((0.2, 2.0, 0.1), 0.5)]), STAGE_CAM, 0, "penumbra", samples=16)
    j = ref["judged"]
    partial = j & (got > 0.0) & (got < 1.0)
    assert partial.sum() > 150 and len(np.unique(got[partial])) >= 12


# --------------------------------------------------------------------------------------------- masked and textured
def test_masked_cutoff():
    """Alpha 129/255 over a 0.5 cutoff occludes, 126/255 does not (the ray goes on through the card)."""
    specs = [dict(color=(0.8, 0.2, 0.2, 129 / 255), cutoff=0.5), dict(color=(0.2, 0.8, 0.2, 126 / 255), cutoff=0.5)]
    parts = [(scenes.quad([-1.2, 0.8, -1.2], [-1.2, 0.8, 0.8], [-0.1, 0.8, 0.8], [-0.1, 0.8, -1.2]), 1),
             (scenes.quad([0.1, 0.8, -1.2], [0.1, 0.8, 0.8], [1.2, 0.8, 0.8], [1.2, 0.8, -1.2]), 2)]
    lights = [light((0.0, 2.6, -0.2), 0.05)]
    scene = open_floor(lights, parts, specs)
    got, ref = run(scene, STAGE_CAM, 0, "masked", 0.85, gscene=open_floor(lights), samples=4)
    frame, depth, nrg = gbuffer(open_floor(lights), STAGE_CAM, W, H)
    P, _ = s6.frag_positions(frame, depth, (0.0, 0.0))
    P = P.reshape(H, W, 3)
    j = ref["judged"] & (depth < 1.0) & (np.abs(P[..., 1]) < 0.05)
    band = j & (P[..., 2] > -0.9) & (P[..., 2] < 0.4)
    left, right = band & (P[..., 0] > -1.0) & (P[..., 0] < -0.5), band & (P[..., 0] > 0.5) & (P[..., 0] < 1.0)
    assert left.sum() > 20 and right.sum() > 20
    assert np.all(got[left] == 0.0) and np.all(got[right] == 1.0)


def textured():
    gpu, cpu, cam = sr.textured_scene()
    for s in (gpu, cpu):
        s.add_light((0.4, 2.8, 3.2), (10.0, 10.0, 10.0), 0.05)
    return gpu, cpu, cam


def test_textured_cutout():
    """The cut-out sphere of surface_ref64.textured_scene (BC7 alpha checker, cutoff 0.5) under a transform that mirrors,
    with every other textured mesh of that scene casting or receiving."""
    gpu, cpu, cam = textured()
    frame, depth, nrg = gbuffer(cpu, cam, W, H)
    got = oracle(cpu, frame, depth, nrg, 0, samples=4)
    ref = judge(got, gpu, frame, depth, nrg, 0, "textured", 0.4, samples=4)
    assert (ref["want"][ref["judged"]] == 0.0).sum() > 200


# --------------------------------------------------------------------------------------------- blended panes
PANES = [(1, 254, True), (2, 232, True), (3, 204, True), (4, 178, True), (3, 178, False)]


def panes_scene(heights, alpha_byte, wall=True):
    specs = [dict(color=(0.3, 0.5, 0.9, alpha_byte / 255), cutoff=2.0), dict(color=(0.5, 0.5, 0.5))]
    parts = [(horizontal(y), 1) for y in heights]
    if wall:
        parts.append((horizontal(1.2, -1.1, 1.1, -1.3, 0.9), 2))
    lights = [light((0.0, 2.5, -0.2), 0.05)]
    return open_floor(lights, parts, specs), open_floor(lights)


@pytest.mark.parametrize("count,alpha_byte,stops", PANES)
def test_blended_panes_and_the_early_stop(count, alpha_byte, stops):
    """Panes of alpha a over an opaque wall: the walk stops once the product (1 - a)^k falls below 0.01 and keeps it, so the
    wall never zeroes it; a product that stays above 0.01 reaches the wall and is 0."""
    scene, floor_only = panes_scene([0.5 + 0.1 * k for k in range(count)], alpha_byte)
    got, ref = run(scene, STAGE_CAM, 0, "%d panes of alpha %d/255" % (count, alpha_byte), 0.85, gscene=floor_only, samples=4)
    a = np.float64(np.float32(alpha_byte / 255))
    prod = np.prod([1.0 - a] * count)
    j = ref["judged"] & ref["blended"]
    under = np.abs(got - prod) <= 8 * count * s6.U32 * prod
    if stops:
        assert prod < 0.01 and (j & under).sum() > 200
    else:
        assert prod > 0.01 and (ref["judged"] & (got == 0.0)).sum() > 200 and not (j & under).any()


@pytest.mark.parametrize("gap,layers,share", [(0.0005, 1, 0.3), (0.01, 2, 0.9)])
def test_blended_panes_and_the_step(gap, layers, share):
    """After a blended hit the walk moves on by hit.T + 0.001: a second pane 0.0005 above the first is stepped over, one 0.01
    above it counts. (Two hits 0.0005 apart along the ray lie within the sampled direction's float32 bound of each other
    for many samples, so fewer pixels are judged there; one sample per pixel keeps enough of them.)"""
    scene, floor_only = panes_scene([0.6, 0.6 + gap], 128, wall=False)
    samples = 1 if layers == 1 else 4
    got, ref = run(scene, STAGE_CAM, 0, "two panes %g apart" % gap, share, gscene=floor_only, samples=samples)
    a = np.float64(np.float32(128 / 255))
    j = ref["judged"] & ref["blended"]
    one, two = np.abs(got - (1.0 - a)) <= 8 * s6.U32, np.abs(got - (1.0 - a) ** 2) <= 16 * s6.U32
    if layers == 1:
        assert (j & one).sum() > 100 and not two.any()
    else:
        assert (j & two).sum() > 200 and not (j & one).any()


# --------------------------------------------------------------------------------------------- facing away
def test_facing_away():
    """A light low at the side: box faces and floor beyond the light's horizon face away and store exactly 0."""
    got, ref = run(stage([light((3.5, 0.4, 0.0), 0.1)]), STAGE_CAM, 0, "facing away", samples=2)
    assert ref["facing_away"] > 50


# --------------------------------------------------------------------------------------------- instanced geometry
@pytest.mark.parametrize("tlas", [False, True])
def test_instances(tlas):
    """scenes.multi_blas: a room, a rotated and scaled sphere and a crate under a non-uniform scale and a 45 degree turn,
    walked by the instance loop or through the TLAS."""
    scene, cam = scenes.multi_blas(threads=1)
    if tlas:
        scene.build_tlas()
    run(scene, cam, 0, "instances, %s" % ("TLAS" if tlas else "instance loop"), 0.8, w=48, h=32, samples=4)


# --------------------------------------------------------------------------------------------- settings
@pytest.mark.parametrize("noise_index", [0, 7, 48, 1 << 20])
@pytest.mark.parametrize("samples", [1, 3, 16])
def test_settings(noise_index, samples):
    scene = stage([light((0.2, 2.2, 0.1), 0.3)])
    frame, depth, nrg = gbuffer(scene, STAGE_CAM, W, H)
    s64 = s6.Scene64(scene)
    for jitter in ((0.0, 0.0), (0.37 / W, -0.61 / H)):
        got = oracle(scene, frame, depth, nrg, 0, samples, noise_index, jitter)
        judge(got, scene, frame, depth, nrg, 0, "samples %d noise %d jitter %s" % (samples, noise_index, jitter), 0.9, s64,
              samples=samples, noise_index=noise_index, jitter=jitter)


def test_noise_is_float32():
    """The noise at index 2^20 differs from its float64 evaluation: x + 5.86e6 keeps half-pixel steps in float32."""
    x, y = np.arange(64, dtype=np.float32), np.full(64, 5.0, np.float32)
    n32 = s6.ign(x, y, 1 << 20).astype(np.float64)
    xs = x.astype(np.float64) + (1 << 20) * np.float64(np.float32(5.588238))
    a = np.float64(np.float32(0.06711056)) * xs + np.float64(np.float32(0.00583715)) * (5.0 + (1 << 20) * np.float64(np.float32(5.588238)))
    b = np.float64(np.float32(52.9829189)) * (a - np.floor(a))
    assert np.mean(np.abs(n32 - (b - np.floor(b))) > 1e-3) > 0.5
