"""Generates tests/golden/field_rate_golden.npz from the UNMODIFIED reference postprocessors
(oracle/_ref/libfield_rate_ref.so): double_framerate (with and without :d), deinterlace_bob, deinterlace_linear and
interlace on small random frames.  Run where the reference is built:  python tests/golden/make_field_rate_golden.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import test_field_rate as T  # noqa: E402
import util  # noqa: E402

ref = T.ref_lib()
assert ref is not None, "build oracle/_ref first: make -C oracle ref && make -C oracle -f field_rate.mk"
out = {}
n = 0
# meta: algo (0 DF, 1 bob, 2 linear, 3 interlace), codec, L, h, call, d, pitch, fill
for algo in (T.DF, T.BOB, T.LINEAR, 3):
    for c in T.CODECS:
        for w, h in ((5, 4), (21, 5)):
            for call in ((0, 1) if algo != 3 else (0,)):
                for d in ((0, 1) if algo == T.DF else (0,)):
                    L = T.vc_get_linesize(w, c)
                    fill = 0xA5 if n % 2 else 0x00
                    pitch = L + (8 if n % 3 else 0)
                    prev, cur = util.rng_bytes(L * h, 2000 + n), util.rng_bytes(L * h, 3000 + n)
                    got, _ = T.ref_run(ref, algo, c, w, h, call, prev, cur, np.full(pitch * h, fill, np.uint8), pitch, d)
                    k = f"a{algo}_c{c}_{L}x{h}_{call}{d}"
                    out[k + "_prev"], out[k + "_cur"], out[k + "_out"] = prev, cur, got
                    out[k + "_meta"] = np.array([algo, c, L, h, call, d, pitch, fill])
                    n += 1
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "field_rate_golden.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path), "bytes,", len(out) // 4, "cases")
