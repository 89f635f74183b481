"""idk::PathTracer's animation calls (include/idkpt.hpp) compile, link and run: on a device a one-node animation moves a
transform; without one the constructor's IDKPT_ERR_NO_DEVICE is the expected outcome."""
import os
import subprocess

from idkengine_b200 import build

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_update_models_compiles_and_links(tmp_path):
    exe = str(tmp_path / "hpp_update_models")
    libdir = os.path.dirname(build.LIBIDKPT)
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-Wno-comment", "-I", os.path.join(REPO, "include"),
           os.path.join(REPO, "tests", "cpp", "hpp_update_models.cpp"), "-L", libdir, "-lidkpt", "-Wl,-rpath," + libdir, "-o", exe]
    subprocess.run(cmd, check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")
