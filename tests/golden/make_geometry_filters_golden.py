"""Generates tests/golden/geometry_filters_golden.npz from the UNMODIFIED geometry filters
(oracle/_ref/libgeometry_filters_ref.so): for the cases of test_geometry_filters.golden_cases(), each output buffer's
bytes with two bit planes, the bytes the reference writes and those of them that come from past the sources.
Run where the reference is built:  python tests/golden/make_geometry_filters_golden.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import test_geometry_filters as T  # noqa: E402

ref = T.ref_lib()
assert ref is not None, "build oracle/_ref first: make -C oracle ref && make -C oracle -f geometry_filters.mk"
out = {}
cases = T.golden_cases()
for case in cases:
    k = T.golden_key(case)
    for i, (got, written, dep) in enumerate(T.ref_run(ref, case)):
        n = got.size - 64
        assert not written[n:].any()
        out[f"{k}_{i}_out"] = np.where(written[:n], got[:n], 0).astype(np.uint8)
        out[f"{k}_{i}_flags"] = np.packbits(np.concatenate([written[:n], dep[:n]]))
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "geometry_filters_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases")
