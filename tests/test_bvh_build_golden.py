"""The host BLAS and TLAS builds against their own past output (tests/golden/bvh_build_digests.json, made by
tests/golden/make_bvh_digests.py): node, triangle, stack-size, fragment-count and SAH bits of every case stay the same."""
import importlib.util
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("make_bvh_digests", os.path.join(HERE, "golden", "make_bvh_digests.py"))
mb = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mb)
GOLDEN = json.load(open(mb.OUT))


def test_host_builds_equal_their_digests():
    cases = mb.cases()
    assert sorted(cases) == sorted(GOLDEN)
    changed = [name for name, f in cases.items() if f() != GOLDEN[name]]
    assert not changed, changed
