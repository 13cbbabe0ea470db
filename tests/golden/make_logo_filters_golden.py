"""Generates tests/golden/logo_filters_golden.npz from the UNMODIFIED logo.c, r12l_to_y416_fake.c and
y416_to_r12l_fake.c (oracle/_ref/liblogo_filters_ref.so): for the cases of test_logo_filters.golden_logo_cases() and
golden_fake_cases(), the reference's output buffers under the fills the tests use.
Run where the reference is built:  python tests/golden/make_logo_filters_golden.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import test_logo_filters as T  # noqa: E402

ref = T.ref_lib()
assert ref is not None, "build oracle/_ref first: make -C oracle ref && make -C oracle -f logo_filters.mk"
out = T.golden_data(ref)
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "logo_filters_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(T.golden_logo_cases()), "logo cases,", len(T.golden_fake_cases()), "fake-pair cases")
