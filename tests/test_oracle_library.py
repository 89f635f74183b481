"""CPU-only: oracle/liboracle.so exports what the oracle sources declare, and tests/oracle_lib.py declares a ctypes signature
for every one of them, so an export added without a signature fails here instead of truncating a pointer argument."""
import glob
import os
import re

import oracle_lib as ol


def test_signature_table_covers_every_export():
    names = set()
    for path in glob.glob(os.path.join(ol.REPO, "oracle", "*.cpp")) + glob.glob(os.path.join(ol.REPO, "oracle", "*.inc")):
        with open(path) as f:
            names |= set(re.findall(r"\bORACLE_API\b[^(;]*?\b(oracle_\w+)\(", f.read()))
    assert names == set(ol.SIGNATURES), names ^ set(ol.SIGNATURES)
    L = ol.lib()
    missing = sorted(name for name in names if not hasattr(L, name))
    assert not missing, missing
