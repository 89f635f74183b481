"""CPU side of the device BLAS build (idkpt_blas_build): the cube root its pre-splitting priorities use.

PreSplitting's priority is a cube root, and the host build takes libm's cbrtf, which is not correctly rounded. The device
build uses csrc/idk_cbrt.h, a restatement of that cbrtf. This compiles the same header for the CPU and compares it with the
running libm on every non-NaN float, so a machine whose libm rounds differently fails here instead of building other trees."""
import os
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "idkengine_b200", "csrc")

_CHECK = r"""
#include "idk_cbrt.h"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <atomic>
#include <thread>
#include <vector>
int main(int argc, char** argv) {
    const uint64_t step = strtoull(argv[1], nullptr, 10);
    const unsigned threads = std::max(1u, std::thread::hardware_concurrency());
    std::atomic<uint64_t> checked(0), bad(0);
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < threads; t++) pool.emplace_back([&, t]() {
        uint64_t c = 0, b = 0;
        for (uint64_t i = (uint64_t)t * step; i < (1ull << 32); i += (uint64_t)threads * step) {
            const float x = idk_cbrt_float((uint32_t)i);
            if (x != x) continue;
            const uint32_t want = idk_cbrt_bits(cbrtf(x)), got = idk_cbrt_bits(idk_cbrtf(x));
            if (want != got && b++ < 4) printf("x=0x%08x libm 0x%08x idk_cbrtf 0x%08x\n", (unsigned)i, want, got);
            c++;
        }
        checked += c;
        bad += b;
    });
    for (auto& th : pool) th.join();
    printf("checked %llu mismatches %llu\n", (unsigned long long)checked.load(), (unsigned long long)bad.load());
    return bad.load() != 0;
}
"""


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("cbrt")
    src, exe = d / "cbrt_check.cpp", d / "cbrt_check"
    src.write_text(_CHECK)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-pthread", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    return str(exe)


def _run(exe, step):
    r = subprocess.run([exe, str(step)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    checked = int(r.stdout.split("checked")[1].split()[0])
    return checked


def test_cube_root_equals_libm_on_every_float(checker):
    """All 2^32 bit patterns except the NaNs (2^32 - 2^24 + 2 of them)."""
    assert _run(checker, 1) == (1 << 32) - (1 << 24) + 2
