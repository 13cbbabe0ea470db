"""Generates tests/golden/resize_filter_golden.npz from the UNMODIFIED resize.c (oracle/_ref/libresize_filter_ref.so):
init() over test_resize_filter.PARSE_CORPUS, and filter() over route_cases(): the output descriptor, what it hands
resize_frame, and the bytes it hands it.
Run where the reference is built:  python tests/golden/make_resize_filter_golden.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import test_resize_filter as T  # noqa: E402

ref = T.ref_lib()
assert ref is not None, "build oracle/_ref first: make -C oracle ref && make -C oracle -f resize_filter.mk"
out = T.golden_data(ref)
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resize_filter_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(T.PARSE_CORPUS), "parse cases,", len(T.route_cases()), "route cases")
