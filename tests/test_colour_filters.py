"""Colour capture filters on the GPU: gamma, matrix, matrix2 and grayscale (colour_filter_kernels.cu, ugb200_cf_*).

CPU: the numpy restatement (colour_filter_ref.py) equals the unmodified gamma.cpp, matrix.c, matrix2.c and
grayscale.c on every byte they write, with two sentinel fills of the output (and of matrix2's Y416 scratch) that
show which bytes those are; the module's own init / vo_pp paths run through the shims; mutants fail.  The golden
fixtures stand in for the reference where it is not built.  GPU: the kernels equal the restatement's contract form
everywhere, with sentinels around every buffer.
"""
import ctypes
import os

import numpy as np
import pytest

import colour_filter_ref as R
import util

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "colour_filters_golden.npz")
FILLS = (0x00, 0xA5)
UYVY, v210, RGB, RG48, Y416 = R.UYVY, R.v210, R.RGB, R.RG48, R.Y416
GAMMAS = (1 / 2.2, 1.0, 2.2, 0.0, -1.0, float("inf"), float("nan"), 1e-300)
_rng = np.random.default_rng(77)
MATRICES = [
    (1, 0, 0, 0, 1, 0, 0, 0, 1),
    R.Y601_TO_Y709,
    tuple(_rng.normal(0, 1.5, 9)),
    tuple(_rng.uniform(-1e6, 1e6, 9)),
    (1e300, -1e300, 1, 0.5, 1e300, 0, 0, 1, -1e300),
    (float("inf"), 1, 0, 0, float("-inf"), 1, 0, 0, 1),
    (float("nan"), 1, 0, 0, 1, 0, 0, 0, float("nan")),
    (-0.0, -0.0, -0.0, -0.0, 1, -0.0, -0.0, -0.0, 1),
    (3.7, -2.9, 1.3, 260.5, 0.01, -0.7, -1.9, 5.1, 2.2),  # wraps through the low 8 / 16 bits
    (0.1, 0.2, 0.7, 0.3, 0.3, 0.4, 0.7, 0.2, 0.1),  # rows summing to 1: near-integer sums on grey pixels
]
# matrix.c maps UYVY to RGB, the others keep their codec
CF_CODECS = {"matrix": (UYVY, RGB, RG48), "matrix2": (UYVY, v210, Y416), "grayscale": (UYVY,), "gamma": (RGB, RG48)}


def linesize(w, c):
    return {UYVY: (w + 1) // 2 * 4, RGB: 3 * w, RG48: 6 * w, Y416: 8 * w, v210: (w + 47) // 48 * 128}[c]


def src_frame(c, w, h, seed):
    """random bytes; seed < 0 gives grey pixels (equal 8-bit channels), where an FMA's rounding shows"""
    n = linesize(w, c) * h
    if seed < 0:
        return np.repeat(np.arange(n // 3 + 1) % 256, 3)[:n].astype(np.uint8)
    return util.rng_bytes(n, seed)


# ---- the reference ---------------------------------------------------------------------------------------------
def _bind(lib):
    vp, i, d, sz, s = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_size_t, ctypes.c_char_p
    lib.ref_matrix_filter.argtypes = [vp, i, i, i, i, vp, vp]
    lib.ref_matrix_init.argtypes = [s, vp, vp]
    lib.ref_matrix_vopp.argtypes = [s, i, i, i, vp, i, vp]
    lib.ref_matrix2_filter.argtypes = [vp, i, i, i, vp, vp, vp, sz]
    lib.ref_matrix2_filter.restype = None
    lib.ref_matrix2_init.argtypes = [s, vp]
    lib.ref_matrix2_vopp.argtypes = [s, i, i, i, vp, vp]
    lib.ref_grayscale_filter.argtypes = [i, i, i, vp, vp]
    lib.ref_grayscale_vopp.argtypes = [s, i, i, vp, vp]
    lib.ref_gamma_cpus.restype = ctypes.c_uint
    lib.ref_gamma_create.argtypes = [d, i]
    lib.ref_gamma_create.restype = vp
    lib.ref_gamma_destroy.argtypes = [vp]
    lib.ref_gamma_apply.argtypes = [vp, i, i, sz, vp, vp]
    lib.ref_gamma_filter.argtypes = [vp, i, i, i, vp, vp]
    lib.ref_gamma_init.argtypes = [s, vp]
    lib.ref_gamma_vopp.argtypes = [s, i, i, i, vp, i, vp]
    return lib


def ref_lib():
    path = os.path.join(util.ORACLE_DIR, "_ref", "libcolour_filters_ref.so")
    return _bind(ctypes.CDLL(path)) if os.path.exists(path) else None


@pytest.fixture(scope="module")
def ref():
    lib = ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libcolour_filters_ref.so not built (reference tree absent)")
    return lib


def _m9(m):
    return (ctypes.c_double * 9)(*m)


def ref_tables(ref, g):
    """the reference's four tables: apply_gamma on a ramp repeated once per task, so every task maps the whole ramp"""
    cpus = ref.ref_gamma_cpus()
    s = ref.ref_gamma_create(g, 0)
    out = {}
    try:
        for ib, ob in ((8, 8), (16, 16), (8, 16), (16, 8)):
            ramp = np.tile(np.arange(1 << ib, dtype=np.uint8 if ib == 8 else np.uint16), cpus)
            o = np.zeros(ramp.size, np.uint8 if ob == 8 else np.uint16)
            assert ref.ref_gamma_apply(s, ib, ob, ramp.nbytes, ramp.ctypes.data, o.ctypes.data) == 0
            out[(ib, ob)] = o[:1 << ib].copy()
    finally:
        ref.ref_gamma_destroy(s)
    return out


# A case: (filter, codec, w, h, param, seed); param is (matrix index, check_bounds) for matrix, the matrix index for
# matrix2, (gamma index, out_depth) for gamma, None for grayscale.
def out_len(f, c, w, h, param):
    if f == "matrix":
        return linesize(w, RGB if c == UYVY else c) * h
    if f == "gamma":
        ob = param[1] or (8 if c == RGB else 16)
        return linesize(w, RGB if ob == 8 else RG48) * h
    return linesize(w, c) * h


def ref_run(ref, case, src):
    """the reference's filter with two sentinel fills: (bytes of the output buffer from its start, mask of the bytes
    it wrote), over the frame plus slack"""
    f, c, w, h, param, _ = case
    n = out_len(f, c, w, h, param)
    pad = 8 * w * h + 64  # matrix2 v210 writes w * h * 8 bytes into the v210 frame
    runs = []
    for fill in FILLS:
        buf = np.full(n + pad, fill, np.uint8)
        inp = src.copy()
        if f == "matrix":
            assert ref.ref_matrix_filter(_m9(MATRICES[param[0]]), param[1], c, w, h, inp.ctypes.data, buf.ctypes.data) == 0
        elif f == "matrix2":
            tmp_len = 8 * w * h
            tmp = np.full(3 * tmp_len + 64, 0x3C, np.uint8)  # the same stale scratch in both runs
            ref.ref_matrix2_filter(_m9(MATRICES[param]), c, w, h, inp.ctypes.data, buf.ctypes.data, tmp.ctypes.data, tmp.size)
        elif f == "grayscale":
            assert ref.ref_grayscale_filter(c, w, h, inp.ctypes.data, buf.ctypes.data) == 0
        else:
            s = ref.ref_gamma_create(GAMMAS[param[0]], param[1])
            try:
                assert ref.ref_gamma_filter(s, c, w, h, inp.ctypes.data, buf.ctypes.data) == 0
            finally:
                ref.ref_gamma_destroy(s)
        runs.append(buf)
    return runs[0], runs[0] == runs[1]


def model(case, src, cpus, tables=None, **mutant):
    """(the restatement's stream, bytes the reference writes, bytes of those that are determinate)"""
    f, c, w, h, param, _ = case
    if f == "matrix":
        e = R.matrix(c, src, MATRICES[param[0]], param[1], **mutant)
        return e, e.size, e.size
    if f == "matrix2":
        e = R.matrix2(c, src, MATRICES[param], **mutant)
        return (e, 8 * w * h // 16 * 16, 16 * (w * h // 6)) if c == v210 else (e, e.size, e.size)
    if f == "grayscale":
        e = R.grayscale(src, w, h, **mutant)
        return e, e.size, e.size
    ib = 8 if c == RGB else 16
    ob = param[1] or ib
    t = tables if tables is not None else R.gamma_tables(GAMMAS[param[0]])
    e = R.gamma(t, ib, ob, src)
    n = src.size * 8 // ib
    written = (n - n % cpus) * ob // 8
    return e, written, written


def check(case, got, mask, cpus, tables=None, **mutant):
    e, written, det = model(case, got_src(case), cpus, tables, **mutant)
    want_mask = np.zeros(mask.size, bool)
    want_mask[:written] = True
    assert np.array_equal(mask, want_mask), f"{case}: the reference wrote other bytes than [0, {written})"
    assert np.array_equal(got[:det], e[:det]), f"{case}: bytes differ from the restatement"


def got_src(case):
    f, c, w, h, _, seed = case
    return src_frame(c, w, h, seed)


def cases():
    """every codec branch and out_depth at widths 1-131 (v210 on and off multiples of 48), heights 1-7, 1081"""
    k = 0
    for f, codecs in CF_CODECS.items():
        for c in codecs:
            params = {"matrix": [(mi, b) for mi in range(len(MATRICES)) for b in (1, 0)],
                      "matrix2": list(range(len(MATRICES))),
                      "grayscale": [None],
                      "gamma": [(gi, d) for gi in range(len(GAMMAS)) for d in (0, 8, 16)]}[f]
            for i, w in enumerate(range(1, 132)):
                yield (f, c, w, 1 + w % 7, params[i % len(params)], k)
                k += 1
            for h in range(1, 8):
                for j, p in enumerate(params):
                    yield (f, c, 5 + j % 4, h, p, k)
                    k += 1
            for w, h in ((1918, 1081), (1920, 1081), (47, 1081)):
                yield (f, c, w, h, params[k % len(params)], k)
                k += 1


# ---- CPU: the restatement against the unmodified filters --------------------------------------------------------
@pytest.mark.parametrize("filt", list(CF_CODECS))
def test_restatement_equals_reference(ref, filt):
    cpus = ref.ref_gamma_cpus()
    tables = {}
    n = 0
    for case in cases():
        if case[0] != filt:
            continue
        if filt == "gamma" and case[4][0] not in tables:
            tables[case[4][0]] = R.gamma_tables(GAMMAS[case[4][0]])
        got, mask = ref_run(ref, case, got_src(case))
        check(case, got, mask, cpus, tables.get(case[4][0]) if filt == "gamma" else None)
        n += 1
    assert n >= 141


def test_gamma_tables_equal_reference(ref):
    for g in GAMMAS:
        want = ref_tables(ref, g)
        got = R.gamma_tables(g)
        for k in want:
            assert np.array_equal(got[k], want[k]), f"gamma {g} table {k}"


def test_refusals_of_the_reference(ref):
    src = src_frame(RG48, 8, 2, 1)
    out = np.zeros(4096, np.uint8)
    assert ref.ref_matrix_filter(_m9(MATRICES[0]), 1, v210, 8, 2, src.ctypes.data, out.ctypes.data) == -1
    assert ref.ref_grayscale_filter(RGB, 8, 2, src.ctypes.data, out.ctypes.data) == 1  # returns its input
    s = ref.ref_gamma_create(2.2, 0)
    try:
        assert ref.ref_gamma_filter(s, UYVY, 8, 2, src.ctypes.data, out.ctypes.data) == -1
    finally:
        ref.ref_gamma_destroy(s)


def test_init_and_vo_pp_paths(ref):
    """the modules' own option parsing and the vo_pp wrapper: init -> reconfigure -> getf -> postprocess -> done"""
    m = (ctypes.c_double * 9)()
    cb = ctypes.c_int()
    assert ref.ref_matrix_init(b"1:2:3:4:5:6:7:8:9", m, ctypes.byref(cb)) == 0 and cb.value == 1 and list(m) == list(range(1, 10))
    assert ref.ref_matrix_init(b"1:2:3:4:5:6:7:8:9:no-bound-check", m, ctypes.byref(cb)) == 0 and cb.value == 0
    # the help text's spelling is only an excess initializer: the check stays on
    assert ref.ref_matrix_init(b"1:2:3:4:5:6:7:8:9:no-bounds-check", m, ctypes.byref(cb)) == 0 and cb.value == 1
    assert ref.ref_matrix_init(b"1:2:3", m, ctypes.byref(cb)) == -1
    assert ref.ref_matrix2_init(b"y601_to_y709", m) == 0 and tuple(m) == R.Y601_TO_Y709
    from ultragrid_b200 import api
    assert api.Y601_TO_Y709 == R.Y601_TO_Y709
    d = ctypes.c_int()
    assert ref.ref_gamma_init(b"2.2:16", ctypes.byref(d)) == 0 and d.value == 16
    assert ref.ref_gamma_init(b"2.2:12", ctypes.byref(d)) == -1
    cpus = ref.ref_gamma_cpus()
    w, h = 37, 3
    for cfg, c, oc, case in ((b"0.5:-1:2:3:0.25:1:-2:0.5:1:no-bound-check", UYVY, RGB, ("matrix", UYVY, w, h, None, 11)),
                             (b"0.5:-1:2:3:0.25:1:-2:0.5:1", RGB, RGB, ("matrix", RGB, w, h, None, 12)),
                             (b"0.5:-1:2:3:0.25:1:-2:0.5:1", RG48, RG48, ("matrix", RG48, w, h, None, 13))):
        src = got_src(case)
        o = np.zeros(out_len("matrix", c, w, h, (0, 1)) + 3 * h + 64, np.uint8)
        assert ref.ref_matrix_vopp(cfg, c, w, h, src.ctypes.data, oc, o.ctypes.data) == 0
        e = R.matrix(c, src, (0.5, -1, 2, 3, 0.25, 1, -2, 0.5, 1), not cfg.endswith(b"check"))
        assert np.array_equal(o[:e.size], e)
    for cfg, c in ((b"y601_to_y709", UYVY), (b"y601_to_y709", Y416)):
        src = src_frame(c, w, h, 14)
        o = np.zeros(src.size, np.uint8)
        assert ref.ref_matrix2_vopp(cfg, c, w, h, src.ctypes.data, o.ctypes.data) == 0
        assert np.array_equal(o, R.matrix2(c, src, R.Y601_TO_Y709))
    src = src_frame(UYVY, w, h, 15)
    o = np.zeros(src.size, np.uint8)
    assert ref.ref_grayscale_vopp(b"", w, h, src.ctypes.data, o.ctypes.data) == 0
    assert np.array_equal(o[:2 * w * h], R.grayscale(src, w, h))
    for cfg, c, oc in ((b"2.2", RGB, RGB), (b"0.45:16", RGB, RG48), (b"1.8:8", RG48, RGB)):
        src = src_frame(c, w, h, 16)
        o = np.zeros(linesize(w, oc) * h, np.uint8)
        assert ref.ref_gamma_vopp(cfg, c, w, h, src.ctypes.data, oc, o.ctypes.data) == 0
        ib, ob = (8 if c == RGB else 16), (8 if oc == RGB else 16)
        e = R.gamma(R.gamma_tables(float(cfg.split(b":")[0])), ib, ob, src)
        n = src.size * 8 // ib
        k = (n - n % cpus) * ob // 8
        assert np.array_equal(o[:k], e[:k])


MUTANT_CASES = [("matrix", RGB, 13, 3, (4, 0), 900), ("matrix", RG48, 13, 3, (8, 0), 901), ("matrix", RG48, 13, 3, (2, 1), 902),
                ("matrix2", UYVY, 13, 3, 4, 903), ("matrix2", v210, 48, 2, 2, 904), ("grayscale", UYVY, 13, 3, None, 905),
                ("matrix", RGB, 16, 16, (9, 1), -1)]
MUTANTS = {"saturate": ({"saturate": True}, ("matrix", "matrix2")), "fma": ({"fma": True}, ("matrix", "matrix2")),
           "rg48_65535": ({"rg48_max": 65535}, ("matrix",)), "chroma_128": ({"chroma": 128}, ("grayscale",))}


def _mutant_fails(name, outputs, cpus):
    kw, filters = MUTANTS[name]
    failed = False
    for case, got, mask in outputs:
        if case[0] not in filters or (name == "rg48_65535" and case[1] != RG48):
            continue
        try:
            check(case, got, mask, cpus, **kw)
        except AssertionError:
            failed = True
    return failed


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fail(ref, name):
    cpus = ref.ref_gamma_cpus()
    outputs = []
    for case in MUTANT_CASES:
        got, mask = ref_run(ref, case, got_src(case))
        check(case, got, mask, cpus)  # the restatement itself passes
        outputs.append((case, got, mask))
    assert _mutant_fails(name, outputs, cpus), f"mutant {name} still equals the reference"


# ---- CPU: the golden fixtures (the reference where it is not built) ---------------------------------------------
def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("golden fixtures absent")
    return np.load(GOLDEN)


def golden_outputs(g):
    """[(case, got, mask)] from the fixtures: `got` holds the bytes the reference wrote, mask covers them"""
    out = []
    for k in sorted(x[:-5] for x in g.files if x.endswith("_meta")):
        meta = g[k + "_meta"]
        f = ("matrix", "matrix2", "grayscale", "gamma")[int(meta[0])]
        p0, p1 = int(meta[4]), int(meta[5])
        param = {"matrix": (p0, p1), "matrix2": p0, "grayscale": None, "gamma": (p0, p1)}[f]
        case = (f, int(meta[1]), int(meta[2]), int(meta[3]), param, int(meta[6]))
        got = g[k + "_out"]
        mask = np.zeros(got.size + 64, bool)
        mask[:got.size] = True
        out.append((case, np.concatenate([got, np.zeros(64, np.uint8)]), mask))
    return out


def test_restatement_equals_golden():
    g = _golden()
    cpus_of = {}
    for case, got, mask in golden_outputs(g):
        # gamma's written length carries the reference's task count; derive it back
        cpus = 1
        if case[0] == "gamma":
            ib = 8 if case[1] == RGB else 16
            ob = case[4][1] or ib
            n = got_src(case).size * 8 // ib
            wn = int(mask.sum()) * 8 // ob
            cpus = next(c for c in range(1, 4097) if n - n % c == wn)
            cpus_of[case] = cpus
        check(case, got, mask, cpus)
    for gi, gv in enumerate(GAMMAS):
        t = R.gamma_tables(gv)
        for ib, ob in ((8, 8), (16, 16), (8, 16), (16, 8)):
            assert np.array_equal(g[f"table_{gi}_{ib}_{ob}"], t[(ib, ob)]), f"gamma {gv} table {(ib, ob)}"
    assert tuple(g["y601_to_y709"]) == R.Y601_TO_Y709


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fail_golden(name):
    outputs = [(c, got, mask) for c, got, mask in golden_outputs(_golden()) if c[0] != "gamma" and (c[5] >= 900 or c[5] < 0)]
    assert _mutant_fails(name, outputs, 1), f"mutant {name} still equals the reference"


def test_header_constant_matches():
    text = open(os.path.join(util.ROOT, "include", "ugb200.h")).read()
    line = next(x for x in text.splitlines() if x.startswith("#define UGB200_CF_Y601_TO_Y709"))
    vals = tuple(float(v) for v in line.split("{")[1].split("}")[0].split(","))
    assert vals == R.Y601_TO_Y709


# ---- GPU --------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Guarded:
    """a device buffer of n bytes at byte offset `off` inside a sentinel-filled allocation"""

    def __init__(self, n, off=0, fill=0x5A, data=None):
        import torch
        self.pad, self.off, self.n, self.fill = 256, off, n, fill
        self.buf = torch.full((n + 2 * self.pad + 16,), fill, dtype=torch.uint8, device="cuda")
        if data is not None:
            self.view.copy_(_dev(data))

    @property
    def view(self):
        a = self.pad + self.off
        return self.buf[a:a + self.n]

    def host(self):
        return self.buf.cpu().numpy()

    def check_outside(self):
        h = self.host()
        a = self.pad + self.off
        assert (h[:a] == self.fill).all() and (h[a + self.n:] == self.fill).all(), "wrote outside the buffer"
        return h[a:a + self.n]


def stream_model(f, c, w, h, param, src):
    """the contract form: what ugb200_cf_* write over their output frame (None where the frame byte is untouched),
    computed in slices of 48 * 65536 bytes (a whole number of units of every codec)"""
    step = 48 * 65536
    n = out_len(f, c, w, h, param)
    if f == "gamma":
        t = R.gamma_tables(GAMMAS[param[0]])
        ib = 8 if c == RGB else 16
        parts = [R.gamma(t, ib, param[1] or ib, src[i:i + step]) for i in range(0, src.size, step)]
    elif f == "matrix":
        parts = [R.matrix(c, src[i:i + step], MATRICES[param[0]], param[1]) for i in range(0, src.size, step)]
    elif f == "matrix2":
        parts = [R.matrix2(c, src[i:i + step], MATRICES[param]) for i in range(0, src.size, step)]
    else:
        parts = [R.grayscale(src[:2 * w * h], w, h)]
    return np.concatenate(parts)[:n]


def run_gpu(f, c, w, h, param, src, src_off=0, dst_off=0, stream=None):
    from ultragrid_b200 import api
    n = out_len(f, c, w, h, param)
    s = Guarded(src.size, src_off, 0x33, src)
    d = Guarded(n, dst_off, 0xC3)
    if f == "matrix":
        api.matrix(c, s.view, w, h, MATRICES[param[0]], param[1], dst=d.view, stream=stream)
    elif f == "matrix2":
        api.matrix2(c, s.view, w, h, MATRICES[param], dst=d.view, stream=stream)
    elif f == "grayscale":
        api.grayscale(s.view, w, h, dst=d.view, stream=stream)
    else:
        api.gamma(GAMMAS[param[0]])(c, s.view, w, h, param[1], dst=d.view, stream=stream)
    import torch
    torch.cuda.synchronize()
    assert np.array_equal(s.check_outside(), src), "the source changed"
    return d.check_outside()


def gpu_check(f, c, w, h, param, seed, src_off=0, dst_off=0, stream=None):
    src = src_frame(c, w, h, seed)
    got = run_gpu(f, c, w, h, param, src, src_off, dst_off, stream)
    e = stream_model(f, c, w, h, param, src)
    assert np.array_equal(got[:e.size], e), f"{(f, c, w, h, param)} differs from the restatement"
    assert (got[e.size:] == 0xC3).all(), f"{(f, c, w, h, param)} wrote past its output"


def _gpu_params(f):
    return {"matrix": [(mi, b) for mi in (1, 3, 6, 8) for b in (1, 0)], "matrix2": [1, 3, 6, 8], "grayscale": [None],
            "gamma": [(gi, d) for gi in (0, 5) for d in (0, 8, 16)]}[f]


@pytest.mark.gpu
@pytest.mark.parametrize("f,c", [(f, c) for f, cs in CF_CODECS.items() for c in cs])
def test_gpu_small_and_odd_sizes(f, c):
    """odd sizes, v210 widths on and off multiples of 48, and address offsets at the alignment limits"""
    params = _gpu_params(f)
    sizes = [(1, 1), (1, 7), (3, 5), (7, 3), (47, 2), (48, 3), (49, 1), (95, 2), (96, 5), (131, 7), (1918, 5), (1920, 1081)]
    align = {UYVY: 1, RGB: 1, RG48: 2, Y416: 2, v210: 4}[c]
    k = 0
    for w, h in sizes:
        for p in params:
            offs = ((0, 0), (align, 3 * align), (16 - align, 0)) if w * h < 5000 else ((0, 0),)
            for so, do in offs:
                if f == "gamma" and (p[1] or (8 if c == RGB else 16)) == 16:
                    do = do // 2 * 2 if do % 2 else do
                gpu_check(f, c, w, h, p, 10_000 + k, so, do)
                k += 1


@pytest.mark.gpu
@pytest.mark.parametrize("f,c", [(f, c) for f, cs in CF_CODECS.items() for c in cs])
def test_gpu_4k(f, c):
    for p in _gpu_params(f)[:2]:
        gpu_check(f, c, 3840, 2160, p, 20_000)


@pytest.mark.gpu
@pytest.mark.parametrize("f,c,p", [("matrix", UYVY, (1, 1)), ("matrix", RG48, (3, 0)), ("matrix2", v210, 1), ("matrix2", Y416, 8),
                                   ("grayscale", UYVY, None), ("gamma", RG48, (0, 16)), ("gamma", RGB, (2, 8))])
def test_gpu_8k(f, c, p):
    gpu_check(f, c, 7680, 4320, p, 30_000)


@pytest.mark.gpu
def test_gpu_gamma_tables():
    """every table entry through the kernels: a ramp over all input values, for every gamma"""
    import torch
    from ultragrid_b200 import api
    for gv in GAMMAS:
        t = R.gamma_tables(gv)
        g = api.gamma(gv)
        for ib, ob in ((8, 8), (16, 16), (8, 16), (16, 8)):
            ramp = np.arange(1 << ib, dtype=np.uint8 if ib == 8 else np.uint16).view(np.uint8)
            c = RGB if ib == 8 else RG48
            w = (1 << ib) // 3 + 1
            src = np.zeros(linesize(w, c), np.uint8)
            src[:ramp.size] = ramp
            out = g(c, _dev(src), w, 1, ob).cpu().numpy()
            got = out.view(np.uint8 if ob == 8 else np.uint16)[:1 << ib]
            assert np.array_equal(got, t[(ib, ob)]), f"gamma {gv} table {(ib, ob)}"
        g.close()
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gpu_matrix2_v210_equals_composed_route():
    """the fused v210 kernel equals v210 -> Y416 -> the Y416 matrix -> Y416 -> v210 through ugb200_pixfmt_convert, each
    run as one line over the whole frame (groups >= w * h / 6 included)"""
    from ultragrid_b200 import Codec, api
    for w, h, mi in ((47, 3, 1), (48, 5, 3), (131, 7, 8), (1918, 1081, 2), (7680, 4320, 1)):
        src = src_frame(v210, w, h, 40_000 + w)
        n = src.size
        s = _dev(src)
        fused = api.matrix2(v210, s, w, h, MATRICES[mi]).cpu().numpy()
        W = n // 16 * 6
        y416 = api.pixfmt_convert(Codec.v210, Codec.Y416, s, W, 1)
        y416 = api.matrix2(Codec.Y416, y416, W, 1, MATRICES[mi])
        composed = api.pixfmt_convert(Codec.Y416, Codec.v210, y416, W, 1, dst_len=n).cpu().numpy()
        assert np.array_equal(fused, composed[:n]), (w, h)


@pytest.mark.gpu
def test_gpu_side_stream():
    import torch
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for f, c, p in (("matrix", UYVY, (3, 1)), ("matrix2", v210, 1), ("grayscale", UYVY, None), ("gamma", RG48, (2, 8))):
            gpu_check(f, c, 1920, 1081, p, 50_000, stream=st)


@pytest.mark.gpu
def test_gpu_refusals_write_nothing():
    import torch
    from ultragrid_b200 import _lib
    L = _lib.load()
    w, h = 64, 4
    src = torch.randint(0, 256, (w * h * 8 + 64,), dtype=torch.uint8, device="cuda")
    dst = torch.full((w * h * 8 + 64,), 0x77, dtype=torch.uint8, device="cuda")
    sp, dp, st = ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    odd = ctypes.c_void_p(dst.data_ptr() + 1)
    m = _m9(MATRICES[1])
    g = L.ugb200_cf_gamma_create(2.2)
    assert g
    calls = [
        (-4, lambda: L.ugb200_cf_matrix(v210, w, h, m, 1, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_matrix(Y416, w, h, m, 1, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_matrix2(RGB, w, h, m, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_matrix2(RG48, w, h, m, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_gamma(g, UYVY, 0, w, h, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_gamma(g, RGB, 12, w, h, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_gamma(None, RGB, 0, w, h, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_matrix(RGB, w, h, None, 1, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_matrix(RGB, 0, h, m, 1, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_matrix2(UYVY, w, -1, m, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_grayscale(w, h, None, dp, st)),
        (-1, lambda: L.ugb200_cf_grayscale(w, h, sp, ctypes.c_void_p(src.data_ptr() + 8), st)),  # overlap
        (-1, lambda: L.ugb200_cf_matrix(RG48, w, h, m, 1, sp, odd, st)),
        (-1, lambda: L.ugb200_cf_matrix2(Y416, w, h, m, sp, odd, st)),
        (-1, lambda: L.ugb200_cf_matrix2(v210, w, h, m, sp, ctypes.c_void_p(dst.data_ptr() + 2), st)),
        (-1, lambda: L.ugb200_cf_gamma(g, RG48, 0, w, h, ctypes.c_void_p(src.data_ptr() + 1), dp, st)),
        (-1, lambda: L.ugb200_cf_gamma(g, RGB, 16, w, h, sp, odd, st)),
    ]
    for want, call in calls:
        assert call() == want
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 0x77).all(), "a refusal wrote"
    L.ugb200_cf_gamma_destroy(g)
