"""Generates tests/golden/color601_golden.npz from the UNMODIFIED reference objects linked for `--param color-601`
(oracle/_ref/libugref601.so, built by oracle/color601.mk).  Run in the build container:  python tests/golden/make_color601_golden.py
The fixtures pin ugb200_pixfmt_convert_cs(..., UGB_CS_601, ...) on machines where oracle/_ref is absent; the sources are regenerated
from their seeds (tests/test_color601.py golden_cases)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import util  # noqa: E402
from test_color601 import golden_cases, golden_source, ref601_lib  # noqa: E402

ref = ref601_lib()
assert ref is not None, "build oracle/_ref/libugref601.so first: make -C oracle ref && make -C oracle -f color601.mk"
out = {}
for key, inc, outc, w, h, seed in golden_cases():
    out[key] = util.convert_cpu(ref, "ref_convert", inc, outc, golden_source(inc, w, h, seed), w, h, linesize=ref.ref_vc_get_linesize)
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "color601_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(out), "cases")
