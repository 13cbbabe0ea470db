"""Generates tests/golden/colour_filters_golden.npz from the UNMODIFIED colour capture filters
(oracle/_ref/libcolour_filters_ref.so): the bytes matrix, matrix2, grayscale and gamma write on a subset of
test_colour_filters.cases() and the mutant cases, gamma's four tables for every tested gamma, and matrix2's
y601_to_y709 coefficients.  Run where the reference is built:  python tests/golden/make_colour_filters_golden.py"""
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import test_colour_filters as T  # noqa: E402

ref = T.ref_lib()
assert ref is not None, "build oracle/_ref first: make -C oracle ref && make -C oracle -f colour_filters.mk"
FILT = ("matrix", "matrix2", "grayscale", "gamma")
out = {}
picked = [c for i, c in enumerate(T.cases()) if c[2] * c[3] <= 1000 and i % 3 == 0] + T.MUTANT_CASES
for case in picked:
    f, c, w, h, param, seed = case
    got, mask = T.ref_run(ref, case, T.got_src(case))
    n = int(mask.sum())
    assert mask[:n].all()
    p0, p1 = {"matrix": param, "matrix2": (param, 0), "grayscale": (0, 0), "gamma": param}[f] if param is not None else (0, 0)
    k = f"{f}_c{c}_{w}x{h}_s{seed}"
    out[k + "_out"] = got[:n]
    out[k + "_meta"] = np.array([FILT.index(f), c, w, h, p0, p1, seed])
for gi, g in enumerate(T.GAMMAS):
    for (ib, ob), t in T.ref_tables(ref, g).items():
        out[f"table_{gi}_{ib}_{ob}"] = t
m = (ctypes.c_double * 9)()
assert ref.ref_matrix2_init(b"y601_to_y709", m) == 0
out["y601_to_y709"] = np.array(list(m))
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "colour_filters_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(picked), "cases")
