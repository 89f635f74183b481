"""k_first_hit starts from a pixel and needs the un-swizzled invocation the reference's FirstHit dispatch gives it: the closed-form
inverse of ReorderInvocations(20) (idkengine_b200/csrc/idk_reorder.h) against the forward map, for every 8x8 group."""
import os
import subprocess

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# 1080p and 4K (240 and 480 groups: full 20-group columns only), 1000 px = 125 groups (a last column 5 groups wide),
# 152 px = 19 groups (no full column), a single group, and a one-pixel-wide tall image
SIZES = ["1920x1080", "3840x2160", "1000x600", "152x8", "8x8", "1x1", "1x200", "168x16"]


def test_reorder_inverse_matches_forward_for_every_group(tmp_path):
    exe = str(tmp_path / "reorder_inverse")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(REPO, "idkengine_b200", "csrc"),
                    os.path.join(REPO, "tests", "cpp", "reorder_inverse.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe] + SIZES, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.endswith("OK\n") and r.stdout.count("groups OK") == len(SIZES), r.stdout
