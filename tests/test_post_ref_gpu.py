"""The present-chain kernels (k_bloom_down, k_bloom_up, k_agx_matrices, k_tonemap) on HDR images written through
PathTracer.WriteResult, at the shapes where a mip chain goes wrong: 1x1 levels, one-texel-high and one-texel-wide chains,
the fewest and the most levels, a full-HD frame, and the settings sweep. The LDR frame equals the oracle's bit for bit and
lies within the float64 bound of tests/test_post_ref.py against tests/post_ref64.py."""
import numpy as np
import pytest

import oracle_lib as ol
import post_ref64 as r
from test_post import synthetic_hdr
from test_post_ref import POST_SETTINGS, check_bloom, check_tonemap, out_of_gamut_hdr, post_settings

pytestmark = pytest.mark.gpu

SHAPE_CASES = [
    (2, 2, 3),          # two 1x1 levels
    (3, 3, 3),          # 3 / 2 = 1: two 1x1 levels again
    (4096, 2, 3),       # nine levels, every one a single row
    (2, 1500, 3),       # seven levels, every one a single column
    (250, 131, 0),      # the most levels at an odd size
    (250, 131, 30),     # the fewest: two
    (1920, 1080, 3),
]


def gpu_post(img, st):
    from idkengine_b200.pathtracer import PathTracer
    h, w = img.shape[:2]
    with PathTracer(w, h) as pt:
        pt.WriteResult(img)
        ldr, _ = pt.PostProcess(st)
    return ldr


def check_gpu_frame(img, st, what):
    ldr = gpu_post(img, st)
    want, bloom = ol.post_process(img, st, want_bloom=True)
    assert np.array_equal(ldr, want), f"{what}: {int((ldr != want).sum())} bytes differ from the oracle"
    if st.IsBloom:
        check_bloom(bloom, r.bloom64(img, st.BloomThreshold, st.BloomMaxColor, st.BloomMinusLods)[1][0], what)
    dev, outside = check_tonemap(ldr, img, bloom, st, what)
    print(f"{what}: largest |byte - 255 v64| {dev:.4f}, outside the position envelope {outside:.4f}")


@pytest.mark.parametrize("w,h,minus", SHAPE_CASES)
def test_gpu_present_chain_shapes(w, h, minus):
    st = post_settings(BloomMinusLods=minus)
    check_gpu_frame(synthetic_hdr(w, h, seed=w + h), st, f"{w}x{h} MinusLods {minus}")


@pytest.mark.parametrize("name", list(POST_SETTINGS))
@pytest.mark.parametrize("image", ["synthetic", "out_of_gamut"])
def test_gpu_present_chain_settings(image, name):
    st = post_settings(**POST_SETTINGS[name])
    w, h = 97, 33
    img = synthetic_hdr(w, h, seed=5) if image == "synthetic" else out_of_gamut_hdr(w, h)
    check_gpu_frame(img, st, f"{image} {name}")
