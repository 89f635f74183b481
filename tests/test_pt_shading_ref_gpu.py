"""The checks of tests/test_pt_shading_ref.py on the device: the path tracer's shading, bounce by bounce, against float64
geometry and closed-form scenes (tests/pt_ref64.py), at 256 x 256 and above."""
import numpy as np
import pytest

import pt_ref64 as pr
from idkengine_b200 import capi
from idkengine_b200 import gpu_types as gt
from idkengine_b200.pathtracer import PathTracer

pytestmark = pytest.mark.gpu

W = H = 256


def _settings(depth, rr=False, lights=False, aovs=False):
    s = capi.default_settings()
    s.RayDepth = depth
    s.Gpu.DoRussianRoulette = int(rr)
    s.Gpu.DoTraceLights = int(lights)
    s.OutputAOVs = int(aovs)
    return s


def _set_sky(pt, sky):
    if isinstance(sky, np.ndarray):
        pt.SetSky((0.0, 0.0, 0.0), sky)
    else:
        pt.SetSky(sky)


def make_run(scene, frame, w, h, sky, rr=False, lights=False, aovs=False):
    """One fresh context per depth, so every run starts from the same accumulation state."""
    def run(depth):
        with PathTracer(w, h, _settings(depth, rr, lights, aovs)) as pt:
            pt.SetScene(scene)
            _set_sky(pt, sky)
            pt.SetFrame(frame)
            pt.EnableWavefrontExport(True)
            st = pt.Compute()
            return dict(rays=pt.ReadWavefrontRays(), bounce=list(st.BounceRays), result=pt.Result, albedo=pt.AlbedoTexture,
                        normal=pt.NormalTexture)
    return run


def test_glass_and_thin_transmission_bounce_by_bounce():
    J = pr.check_glass(make_run, W, H)
    for case, least in (("bounce0", 12000), ("hit", 80000), ("miss", 8000), ("refract_in", 1200), ("refract_out", 1200),
                        ("tir", 400), ("mirror", 1200), ("diffuse", 12000), ("thin", 1200), ("absorbed", 2000),
                        ("absorbed_to_zero", 200), ("from_inside", 2000), ("throughput_exact", 40000)):
        assert J[case] >= least, (case, J[case])


def test_first_hit_from_inside_a_volumetric_mesh():
    J = pr.check_inside_glass(make_run, W, H)
    for case, least in (("bounce0", 32000), ("refract_out", 4000), ("tir", 4000), ("mirror", 200), ("absorbed", 32000)):
        assert J[case] >= least, (case, J[case])


def test_russian_roulette_divides_by_the_survival_probability():
    J = pr.check_roulette(make_run, W, H)
    for case, least in (("rr_survived", 20000), ("rr_terminated", 8000), ("diffuse", 40000)):
        assert J[case] >= least, (case, J[case])


def test_branch_counts_follow_schlick_fresnel():
    out = pr.check_branches(make_run, 384, 384)
    for name, r in out.items():
        assert r["judged"] >= 60000, (name, r["judged"])
        assert abs(r["zm"]) < 5.0 and abs(r["zt"]) < 5.0, (name, r["zm"], r["zt"])
    assert out["dielectric 1.5"]["mirror"] >= 2000 and out["dielectric 1.0"]["mirror"] >= 400
    assert out["m+t>1 tinted"]["trans"] >= 20000 and out["m+t>1 tinted"]["J"]["diffuse"] == 0
    assert out["thin untinted"]["trans"] >= 12000 and out["biased"]["trans"] >= 4000


def test_cosine_sampling_and_camera_footprint():
    r = pr.check_cosine(make_run, 320, 320)
    assert r["n"] >= 60000
    assert r["ks_c"].pvalue > 1e-6 and r["ks_p"].pvalue > 1e-6
    assert r["footprint"].all(), (~r["footprint"]).sum()


def test_first_hit_aovs():
    r = pr.check_aovs(make_run, W, H)
    assert r["n"] >= 20000 and r["n_sky"] >= 2000
    assert r["err_a"] <= 2e-7 and r["err_n"] <= 2e-6 and r["err_sa"] <= 6e-8 and r["err_sn"] == 0.0
    assert np.all(r["alpha"] == 1.0)


def test_light_spheres():
    r = pr.check_lights(make_run, W, H)
    assert r["ok"].sum() >= 1200
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
    assert int(runs[2]["bounce"][1]) == W * H


def test_accumulation_is_the_running_mean():
    scene = pr.build([(pr.floor(), 0)], [dict(color=(0.6, 0.5, 0.4), roughness=1.0)])
    frame = pr._frame(*pr.FLOOR_CAM[:2], W, H, pr.FLOOR_CAM[2])
    with PathTracer(W, H, _settings(3, rr=True)) as pt:
        pt.SetScene(scene)
        pt.SetSky((0.0, 0.0, 0.0), pr.cube_sky())
        pt.SetFrame(frame)
        pt.EnableWavefrontExport(True)
        samples = []
        for n in range(6):
            pt.Compute()
            assert pt.AccumulatedSamples == n + 1
            samples.append(pt.ReadWavefrontRays()["Radiance"].reshape(H, W, 3).astype(np.float64))
            mean = np.mean(samples, 0)
            res = pt.Result
            assert np.all(np.abs(res[..., :3] - mean) <= 1e-6 * np.abs(mean) + 1e-7), n
            assert np.all(res[..., 3] == 1.0)
        assert np.ptp(np.stack(samples), 0).max() > 0.1
        # a changed frame restarts the mean
        pt.SetFrame(pr._frame((0.0, 1.2, 0.0), (0.1, -0.5, -1.0), W, H, 90.0))
        assert pt.AccumulatedSamples == 0
        pt.Compute()
        assert pt.AccumulatedSamples == 1
        assert np.array_equal(pt.Result[..., :3], pt.ReadWavefrontRays()["Radiance"].reshape(H, W, 3))
