"""Generates tests/golden/ldgm_golden.npz: matrices written by the UNMODIFIED reference generator generate_ldgm_matrix and the buffers its
LDGM_session_cpu::encode_hdr_frame makes from them (oracle/_ref/libldgm_ref.so, built by oracle/ldgm.mk), so that the encode can be
checked where the reference tree is absent.  CPU only:
    python tests/golden/make_ldgm_golden.py [output.npz]
Keys: pcm_{k}_{m}_{c}_{seed}; hdr_, frame_ and enc_{k}_{m}_{c}_{seed}_{frame size}."""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import ldgm_cases as lc  # noqa: E402
import util  # noqa: E402

# c * k stays within the generator's work array (3 * 8192 entries)
SETS = [(64, 64, 2, 1), (512, 384, 5, 7), (256, 256, 63, 11)]
SIZES = [1, 999, 5003]

L = lc.ref_lib()
assert L is not None, "build oracle/_ref first: make -C oracle -f ldgm.mk"
out = {}
with tempfile.TemporaryDirectory() as tmp:
    for k, m, c, seed in SETS:
        path = os.path.join(tmp, f"{k}-{m}-{c}-{seed}.bin")
        assert L.ref_ldgm_generate(path.encode(), k, m, c, seed) == 0
        out[f"pcm_{k}_{m}_{c}_{seed}"] = lc.read_matrix_file(path)[2]
        s = lc.RefSession(L, path, k, m, c)
        for size in SIZES:
            key = f"{k}_{m}_{c}_{seed}_{size}"
            hdr, frame = util.rng_bytes(24, size), util.rng_bytes(size, size + seed)
            out[f"hdr_{key}"], out[f"frame_{key}"] = hdr, frame
            out[f"enc_{key}"] = s.encode(hdr.tobytes(), frame)
        s.close()
dst = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "ldgm_golden.npz")
np.savez_compressed(dst, **out)
print(dst, sum(v.nbytes for v in out.values()), "bytes")
