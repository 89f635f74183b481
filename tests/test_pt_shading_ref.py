"""The path tracer's shading, bounce by bounce, against float64 geometry and closed-form scenes (tests/pt_ref64.py), run
on the CPU oracle. tests/test_pt_shading_ref_gpu.py runs the same checks on the device at larger sizes."""
import numpy as np
import pytest

import oracle_lib as ol
import pt_ref64 as pr
from idkengine_b200 import capi
from idkengine_b200 import gpu_types as gt

W = H = 128


def make_run(scene, frame, w, h, sky, rr=False, lights=False, aovs=False):
    def run(depth):
        s = capi.default_settings()
        s.RayDepth = depth
        s.Gpu.DoRussianRoulette = int(rr)
        s.Gpu.DoTraceLights = int(lights)
        s.OutputAOVs = int(aovs)
        r = ol.path_trace(scene, frame, s, w, h, sky=sky)
        return dict(rays=r.rays, bounce=list(r.stats.BounceRays), result=r.result, albedo=r.albedo, normal=r.normal)
    return run


def test_glass_and_thin_transmission_bounce_by_bounce():
    J = pr.check_glass(make_run, W, H)
    for case, least in (("bounce0", 3000), ("hit", 20000), ("miss", 2000), ("refract_in", 300), ("refract_out", 300),
                        ("tir", 100), ("mirror", 300), ("diffuse", 3000), ("thin", 300), ("absorbed", 500),
                        ("absorbed_to_zero", 50), ("from_inside", 500), ("throughput_exact", 10000)):
        assert J[case] >= least, (case, J[case])


def test_first_hit_from_inside_a_volumetric_mesh():
    J = pr.check_inside_glass(make_run, W, H)
    for case, least in (("bounce0", 8000), ("refract_out", 1000), ("tir", 1000), ("mirror", 50), ("absorbed", 8000)):
        assert J[case] >= least, (case, J[case])


def test_russian_roulette_divides_by_the_survival_probability():
    J = pr.check_roulette(make_run, W, H)
    for case, least in (("rr_survived", 5000), ("rr_terminated", 2000), ("diffuse", 10000)):
        assert J[case] >= least, (case, J[case])


def test_branch_counts_follow_schlick_fresnel():
    out = pr.check_branches(make_run, 192, 192)
    for name, r in out.items():
        assert r["judged"] >= 15000, (name, r["judged"])
        assert abs(r["zm"]) < 5.0 and abs(r["zt"]) < 5.0, (name, r["zm"], r["zt"])
    assert out["dielectric 1.5"]["mirror"] >= 500 and out["dielectric 1.0"]["mirror"] >= 100
    assert out["m+t>1 tinted"]["trans"] >= 5000 and out["m+t>1 tinted"]["J"]["diffuse"] == 0
    assert out["thin untinted"]["trans"] >= 3000 and out["biased"]["trans"] >= 1000


def test_cosine_sampling_and_camera_footprint():
    r = pr.check_cosine(make_run, 160, 160)
    assert r["n"] >= 15000
    assert r["ks_c"].pvalue > 1e-6 and r["ks_p"].pvalue > 1e-6
    assert r["footprint"].all(), (~r["footprint"]).sum()


def test_first_hit_aovs():
    r = pr.check_aovs(make_run, W, H)
    assert r["n"] >= 5000 and r["n_sky"] >= 500
    assert r["err_a"] <= 2e-7 and r["err_n"] <= 2e-6 and r["err_sa"] <= 6e-8 and r["err_sn"] == 0.0
    assert np.all(r["alpha"] == 1.0)


def test_light_spheres():
    r = pr.check_lights(make_run, W, H)
    assert r["ok"].sum() >= 300
    assert np.array_equal(r["ok"], r["lit"]) and np.all(r["lit"][r["near"]])


@pytest.mark.parametrize("metallic,roughness", [(0.0, 1.0), (1.0, 0.7)], ids=["diffuse", "rough-metal"])
def test_furnace(metallic, roughness):
    D = 4
    res, leak, want = pr.furnace(make_run, W, H, D, rr=False, metallic=metallic, roughness=roughness)
    rel = np.abs(res[~leak] - want).max() / want.max()
    print("furnace RR off: leaks %d / %d, max rel err %.3g" % (leak.sum(), len(leak), rel))
    assert leak.mean() <= 1e-3 and rel <= D * 2.0 ** -22
    D = 6
    res, leak, want = pr.furnace(make_run, W, H, D, rr=True, metallic=metallic, roughness=roughness)
    v = res[~leak]
    z = (v.mean(0) - want) / (v.std(0) / np.sqrt(len(v)))
    print("furnace RR on: mean %s want %s z %s" % (v.mean(0), want, z))
    assert leak.mean() <= 1e-3 and np.all(np.abs(z) < 5.0)


def test_sky_irradiance_of_a_diffuse_floor():
    faces = pr.cube_sky()
    tb, frame, states, alive, runs = pr.floor_run(make_run, dict(color=(0.6, 0.6, 0.6), roughness=1.0), W, H, depth=2,
                                                  cam=((0.0, 1.0, 0.0), (0.0, -1.0, -0.05), 60.0), rr=False)
    rad = states[1]["Radiance"].astype(np.float64)
    n = pr.unit(pr.decompress_normal(gt.compress_sr11g11b10(np.array([0.0, 1.0, 0.0], np.float32))))
    mean, band = pr.cosine_weighted_sky(n)
    want = tb.albedo[0] * mean
    sigma = rad.std(0) / np.sqrt(len(rad))
    allowance = tb.albedo[0] * band * np.ptp(faces[..., :3].reshape(-1, 3), 0) / 64.0
    z = (rad.mean(0) - want) / sigma
    print("sky irradiance: mean %s want %s z %s (edge allowance %s)" % (rad.mean(0), want, z, allowance))
    assert np.all(np.abs(rad.mean(0) - want) < 5.0 * sigma + allowance)
    assert int(runs[2]["bounce"][1]) == W * H                    # every camera ray hit the floor and bounced once more


def test_accumulation_is_the_running_mean():
    scene = pr.build([(pr.floor(), 0)], [dict(color=(0.6, 0.5, 0.4), roughness=1.0)])
    frame = pr._frame(*pr.FLOOR_CAM[:2], W, H, pr.FLOOR_CAM[2])
    s = capi.default_settings()
    s.RayDepth = 3
    res = np.zeros((H, W, 4), np.float32)
    samples = []
    for n in range(6):
        r = ol.path_trace(scene, frame, s, W, H, sky=pr.cube_sky(), accumulated=n, result=res)
        assert r.accumulated == n + 1
        samples.append(r.rays["Radiance"].reshape(H, W, 3).astype(np.float64))
        mean = np.mean(samples, 0)
        assert np.all(np.abs(res[..., :3] - mean) <= 1e-6 * np.abs(mean) + 1e-7), n
        assert np.all(res[..., 3] == 1.0)
    assert np.ptp(np.stack(samples), 0).max() > 0.1              # the samples differ, so the mean is not trivial
    # a changed frame restarts the mean: the first sample replaces whatever the image held
    other = pr._frame((0.0, 1.2, 0.0), (0.1, -0.5, -1.0), W, H, 90.0)
    r = ol.path_trace(scene, other, s, W, H, sky=pr.cube_sky(), accumulated=0, result=res)
    assert r.accumulated == 1 and np.array_equal(res[..., :3], r.rays["Radiance"].reshape(H, W, 3))
