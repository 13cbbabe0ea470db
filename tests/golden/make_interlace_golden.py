"""Generates tests/golden/interlace_golden.npz from the UNMODIFIED reference objects (oracle/_ref/libugref.so):
vc_deinterlace_ex, vc_deinterlace and il_upper_to_merged / il_merged_to_upper on small random frames.
Run where the reference is built:  python tests/golden/make_interlace_golden.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import interlace_ref as R  # noqa: E402
import util  # noqa: E402
from test_interlace import _bind, ref_ex, ref_legacy  # noqa: E402

ref = util.ref_cpu()
assert ref is not None, "build oracle/_ref first: make -C oracle ref"
ref = _bind(ref)
out = {}
n = 0
# kind 0: vc_deinterlace_ex (codec, L, lines, pitch, fill)
for c in R.NON_OPAQUE:
    for L, lines in ((36 * 3 + 20, 5), (48 * 6, 4), (100, 3), (14, 6), (1004, 1)):
        for fill in (0x00, 0xA5):
            pitch = L + (8 if fill else 0)
            src = util.rng_bytes(L * lines, 500 + n)
            got = ref_ex(ref, c, src, L, np.full(pitch * lines, fill, np.uint8), pitch, lines)
            n += 1
            if got is None:
                continue
            k = f"ex{c}_{L}x{lines}_{fill}"
            out[k + "_src"], out[k + "_out"], out[k + "_meta"] = src, got, np.array([0, c, L, lines, pitch, fill])
# kind 1: vc_deinterlace (L, lines, address offset)
for L, lines, off in ((16, 9, 0), (17, 8, 1), (40, 7, 4), (52, 12, 0), (300, 6, 1)):
    src = util.rng_bytes(L * lines, 900 + L)
    k = f"legacy_{L}x{lines}_{off}"
    out[k + "_src"], out[k + "_out"], out[k + "_meta"] = src, ref_legacy(ref, src, L, lines, off), np.array([1, L, lines, off])
# kinds 2 and 3: il_upper_to_merged, il_merged_to_upper
for kind, name in ((2, "il_upper_to_merged"), (3, "il_merged_to_upper")):
    for L, h in ((3, 7), (64, 6), (17, 1)):
        src = util.rng_bytes(L * h, 1300 + L + h)
        d = np.zeros(L * h, np.uint8)
        getattr(ref, name)(d.ctypes.data, src.ctypes.data, L, h, None)
        k = f"{name}_{L}x{h}"
        out[k + "_src"], out[k + "_out"], out[k + "_meta"] = src, d, np.array([kind, L, h])
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "interlace_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(out) // 3, "cases")
