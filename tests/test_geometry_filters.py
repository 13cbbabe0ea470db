"""Geometry filters on the GPU: flip, mirror, crop, split, border and interlaced_3d (geometry_kernels.cu, ugb200_cf_* /
ugb200_pp_*).

CPU: the numpy restatement (geometry_filter_ref.py) equals the unmodified flip.c, mirror.c, crop.c, split.c (both),
vf_split.cpp, border.c and 3d-interlaced.c on every byte they write.  Three runs of the reference show which bytes
those are (two sentinel fills of the output) and which of them come from memory past the sources (two fills of the
input slack); both sets equal the restatement's, which DESIGN.md §8 lists.  The modules' own init / reconfigure
parse the options.  Mutants fail.  The golden fixtures stand in for the reference where it is not built.
GPU: the kernels equal the restatement's contract form, with sentinels around every buffer.
"""
import ctypes
import os

import numpy as np
import pytest

import geometry_filter_ref as R
import util

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geometry_filters_golden.npz")
OUT_FILLS = (0x00, 0xA5)
SLACK_FILLS = (0x11, 0xEE)
UYVY, v210, RGB, RGBA, R10k, R12L = R.UYVY, R.v210, R.RGB, R.RGBA, R.R10k, R.R12L
CODECS = list(R.BLOCK)
WIDTHS = list(range(1, 132)) + [1918, 1920, 7680]
FILTERS = ("flip", "mirror", "crop", "split", "border", "interlaced_3d")


def frame(c, w, h, seed):
    return util.rng_bytes(R.linesize(w, c) * h, seed)


# ---- the reference ---------------------------------------------------------------------------------------------
def _bind(lib):
    vp, i, s = ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p
    lib.ref_flip_filter.argtypes = [i, i, i, vp, vp]
    lib.ref_mirror_filter.argtypes = [i, i, i, vp, vp]
    lib.ref_crop_geometry.argtypes = [s, i, i, i, vp]
    lib.ref_crop.argtypes = [s, i, i, i, vp, vp, i]
    lib.ref_split_init.argtypes = [s, vp, vp]
    lib.ref_split_filter.argtypes = [s, i, i, i, vp, vp]
    lib.ref_split_vopp.argtypes = [s, i, i, i, vp, vp, vp]
    lib.ref_border_init.argtypes = [s, vp, vp]
    lib.ref_border.argtypes = [s, i, i, i, vp, vp]
    lib.ref_interlaced_3d.argtypes = [i, i, i, vp, vp, vp]
    return lib


def ref_lib():
    return util.ref_lib("libgeometry_filters_ref.so", _bind)


@pytest.fixture(scope="module")
def ref():
    lib = ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libgeometry_filters_ref.so not built (reference tree absent)")
    return lib


class Slacked:
    """a harness-owned input: the frame with `pre` and `post` bytes of slack around it"""

    def __init__(self, data, fill, pre=0, post=4096):
        self.pre = pre
        self.buf = np.full(pre + data.size + post, fill, np.uint8)
        self.buf[pre:pre + data.size] = data

    @property
    def ptr(self):
        return self.buf.ctypes.data + self.pre


def crop_cfg(p):
    width, height, xoff, yoff, _ = p
    return f"width={width}:height={height}:xoff={xoff}:yoff={yoff}".encode()


def border_cfg(p):
    return p[0].encode()


def out_sizes(case):
    """bytes of each output buffer the restatement covers (the reference's writes included)"""
    return [x[0].size for x in model(case)]


def ref_once(ref, case, out_fill, slack_fill):
    """one run of the reference: the output buffers, with 64 bytes of slack after each"""
    f, c, w, h, p, seed = case
    src = frame(c, w, h, seed)
    outs = [np.full(n + 64, out_fill, np.uint8) for n in out_sizes(case)]
    inp = Slacked(src, slack_fill)  # kept alive across the call
    if f == "flip":
        assert ref.ref_flip_filter(c, w, h, inp.ptr, outs[0].ctypes.data) == 0
    elif f == "mirror":
        assert ref.ref_mirror_filter(c, w, h, inp.ptr, outs[0].ctypes.data) == (0 if c == UYVY else 1)
    elif f == "crop":
        inp = Slacked(src, slack_fill, pre=src.size + 4096, post=src.size + 4096)
        assert ref.ref_crop(crop_cfg(p), c, w, h, inp.ptr, outs[0].ctypes.data, -1 if p[4] is None else p[4]) == 0
    elif f == "split":
        ptrs = (ctypes.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
        xy = (ctypes.c_int * 2)()
        assert ref.ref_split_vopp(f"{p[0]}:{p[1]}".encode(), c, w, h, inp.ptr, ptrs, xy) == 0
        assert tuple(xy) == p
    elif f == "border":
        rc = ref.ref_border(border_cfg(p), c, w, h, inp.ptr, outs[0].ctypes.data)
        assert rc == (0 if c in (UYVY, RGB, RGBA) else -1)
    else:
        right = Slacked(frame(c, w, h, seed + 1), slack_fill)
        assert ref.ref_interlaced_3d(c, w, h, inp.ptr, right.ptr, outs[0].ctypes.data) == 0
    return outs


def ref_run(ref, case):
    """[(bytes, written, from-slack)] per output buffer, from three runs: two output fills, two input slack fills"""
    a = ref_once(ref, case, OUT_FILLS[0], SLACK_FILLS[0])
    b = ref_once(ref, case, OUT_FILLS[1], SLACK_FILLS[0])
    s = ref_once(ref, case, OUT_FILLS[0], SLACK_FILLS[1])
    return [(x, x == y, (x != z) & (x == y)) for x, y, z in zip(a, b, s)]


def model(case, **mutant):
    """[(bytes, written, undefined)] per output buffer, from the restatement"""
    f, c, w, h, p, seed = case
    src = frame(c, w, h, seed)
    if f == "flip":
        return [R.flip(c, src, w, h)]
    if f == "mirror":
        return [R.mirror(c, src, w, h, swap=not mutant.get("no_swap"))]
    if f == "crop":
        width, height, xoff, yoff, pitch = p
        return [R.crop(c, src, w, h, width, height, xoff, yoff, pitch, xoff_in_pixels=mutant.get("xoff_pixels", False))]
    if f == "split":
        return R.split(c, src, w, h, p[0], p[1], rounded=mutant.get("rounded", False))
    if f == "border":
        color, bw, bh = R.border_init(p[0])
        return [R.border(c, src, w, h, color, bw, bh)]
    right = frame(c, w, h, seed + 1)
    return [R.interlaced_3d(c, src, right, w, h, drift=not mutant.get("pitch_L"), truncate=mutant.get("truncate", False))]


def check(case, got, **mutant):
    """the reference's (bytes, written, from-slack) per buffer equal the restatement's"""
    for (g, wr, dep), (e, ew, eu) in zip(got, model(case, **mutant)):
        n = e.size
        assert not wr[n:].any(), f"{case}: the reference wrote past the bytes the restatement covers"
        assert np.array_equal(wr[:n], ew), f"{case}: the reference wrote other bytes than the restatement"
        assert np.array_equal(dep[:n], eu), f"{case}: other bytes come from past the sources than DESIGN.md §8 lists"
        m = ew & ~eu
        assert np.array_equal(g[:n][m], e[m]), f"{case}: bytes differ from the restatement"


def check_fails(case, got, **mutant):
    try:
        check(case, got, **mutant)
    except AssertionError:
        return True
    return False


# ---- the cases ---------------------------------------------------------------------------------------------------
def flip_cases():
    return [("flip", c, w, h, None, 1000 + i) for i, (c, w, h) in
            enumerate([(c, w, 3 if w < 1000 else 5) for c in CODECS for w in WIDTHS[::7] + WIDTHS[-3:]] +
                      [(UYVY, w, 5) for w in WIDTHS])]


def mirror_cases():
    return [("mirror", UYVY, w, h, None, 2000 + w) for w in WIDTHS for h in (3,)] + \
           [("mirror", c, 37, 3, None, 2999) for c in (v210, RGB, RGBA, R.YUYV)]


def crop_windows(c, w, h):
    """(width, height, xoff, yoff, pitch): windows at every alignment, negative and oversized offsets, both pitches"""
    L = R.linesize(w, c)
    out = []
    for xo in (0, 1, 2, 3, 5, 7, 13, w // 3, w - 1, w + 5, -1, -2, -(w // 4) - 1, -w - 7, 1 << 31):
        for ww, hh, yo in ((w // 2 + 1, h // 2 + 1, 1), (w // 3, h - 1, 0), (0, 0, 0), (w + 9, 1, h - 1), (w // 2, h // 2, -1),
                           (w // 2, h // 2, -h), (1, 2, 1 << 20)):
            for pitch in (None, L + 48):
                out.append((ww, hh, xo, yo, pitch))
    return out


def crop_cases(ref_checks_negative=False):
    res = []
    k = 3000
    for c in CODECS:
        for w, h in ((37, 5), (131, 7), (1918, 3)):
            for p in crop_windows(c, w, h)[::3 if w > 1000 else 1]:
                first = R.crop_first_row_offset(c, w, h, *p[:4])
                if (first < 0) == ref_checks_negative:
                    res.append(("crop", c, w, h, p, k))
                k += 1
    return res


def split_cases():
    res = []
    k = 4000
    for c in (v210, R10k, R12L, RGB):
        for x in range(1, 9):
            for y in range(1, 5):
                for w in (x * 7 * 3, x * 48 + x, 840 if 840 % x == 0 else x * 100):
                    res.append(("split", c, w, y * 3, (x, y), k))
                    k += 1
    return res


BORDER_CFGS = ["", "color=ff8000", "color=#ff8000", "color=#1a2b3c:width=3:height=5", "width=0:height=0", "width=1:height=1",
               "width=7", "height=3", "color=00ff7f:width=4:height=2", "COLOR=a5a5a5:WIDTH=9:HEIGHT=0", "color=#0x1234",
               "color=zzzzzz:width=2"]


def border_cases():
    res = []
    k = 5000
    for c in (UYVY, RGB, RGBA, v210):
        for cfg in BORDER_CFGS:
            for w, h in ((37, 21), (64, 24), (131, 33)):
                res.append(("border", c, w, h, (cfg,), k))
                k += 1
    return res


def interlaced_cases():
    # line sizes off every multiple of 16: RGB widths 1..16 give every L % 16, UYVY every L % 16 in steps of 4
    res = [("interlaced_3d", RGB, w, h, None, 6000 + w) for w in range(1, 17) for h in (1, 4, 5)]
    res += [("interlaced_3d", c, w, h, None, 6100 + w) for c in (UYVY, v210, R12L) for w in (1, 3, 5, 7, 48, 131) for h in (2, 7)]
    return res


def cases():
    return flip_cases() + mirror_cases() + crop_cases() + split_cases() + border_cases() + interlaced_cases()


MUTANTS = {
    "mirror_without_luma_swap": ({"no_swap": True}, lambda c: c[0] == "mirror"),
    "crop_xoff_in_pixels": ({"xoff_pixels": True}, lambda c: c[0] == "crop"),
    "split_rounded_offsets": ({"rounded": True}, lambda c: c[0] == "split"),
    "interlaced_3d_at_pitch_L": ({"pitch_L": True}, lambda c: c[0] == "interlaced_3d"),
    "interlaced_3d_truncating_average": ({"truncate": True}, lambda c: c[0] == "interlaced_3d"),
}


# ---- CPU: the restatement against the reference -----------------------------------------------------------------
@pytest.mark.parametrize("filt", FILTERS)
def test_restatement_equals_reference(ref, filt):
    for case in [c for c in cases() if c[0] == filt]:
        check(case, ref_run(ref, case))


def test_crop_geometry_equals_reference(ref):
    """the output size and offsets of crop_postprocess_reconfigure / crop_postprocess, and the C entry's copy of them"""
    from ultragrid_b200 import _lib
    L = _lib.load()
    for c in CODECS:
        for w, h in ((37, 5), (1920, 1080), (7680, 4320)):
            for p in crop_windows(c, w, h):
                g = (ctypes.c_int * 4)()
                assert ref.ref_crop_geometry(crop_cfg(p), c, w, h, g) == 0
                assert tuple(g) == R.crop_geometry(c, w, h, *p[:4]), (c, w, h, p)
                d = (ctypes.c_int * 4)()
                assert L.ugb200_cf_crop_geometry(c, w, h, p[0], p[1], p[2], p[3], d) == 0
                assert tuple(d) == tuple(g), (c, w, h, p)


def test_crop_unclamped_negative_offsets_read_before_the_source(ref):
    """a negative offset within the window is not clamped: the reference's first row starts before the frame, so
    its bytes come from the slack before it (the device form refuses these with -1)"""
    cs = crop_cases(ref_checks_negative=True)
    assert len(cs) > 20
    for case in cs:
        f, c, w, h, p, seed = case
        src = frame(c, w, h, seed)
        outs = []
        for fill in SLACK_FILLS:
            o = np.zeros(R.crop(c, src, w, h, *p)[0].size, np.uint8)
            inp = Slacked(src, fill, pre=src.size + 4096, post=src.size + 4096)
            assert ref.ref_crop(crop_cfg(p), c, w, h, inp.ptr, o.ctypes.data, -1 if p[4] is None else p[4]) == 0
            outs.append(o)
        assert outs[0][0] != outs[1][0], case  # the first byte is read from before the frame


def test_module_options(ref):
    """split's two parsers and border_init, which the device form takes the results of"""
    for cfg, xy in (("2:2", (2, 2)), ("8:4", (8, 4)), ("3:1", (3, 1))):
        x, y = ctypes.c_int(), ctypes.c_int()
        assert ref.ref_split_init(cfg.encode(), ctypes.byref(x), ctypes.byref(y)) == 0
        assert (x.value, y.value) == xy
    for cfg in BORDER_CFGS + ["help", "color=12345", "depth=3", "color=#12345"]:
        col = (ctypes.c_ubyte * 4)()
        wh = (ctypes.c_uint * 2)()
        rc = ref.ref_border_init(cfg.encode(), col, wh)
        want = R.border_init(cfg)
        if want is None:
            assert rc == -2, cfg
        else:
            assert rc == 0 and (bytes(col), wh[0], wh[1]) == want, (cfg, bytes(col), tuple(wh), want)
    assert R.border_init("color=ff8000")[0] != bytes([0xFF, 0x80, 0x00, 0xFF])  # the parser's skipped character


def test_split_capture_filter_equals_postprocessor(ref):
    """split.c's filter() writes the same tile bytes as the postprocessor (its tiles come from malloc)"""
    for case in [c for c in split_cases() if c[4] in ((2, 2), (3, 4), (8, 1))][:12]:
        f, c, w, h, (x, y), seed = case
        want = model(case)
        tiles = [np.zeros(t[0].size, np.uint8) for t in want]
        ptrs = (ctypes.c_void_p * len(tiles))(*[t.ctypes.data for t in tiles])
        inp = Slacked(frame(c, w, h, seed), 0)
        assert ref.ref_split_filter(f"{x}:{y}".encode(), c, w, h, inp.ptr, ptrs) == 0
        for t, (e, ew, _) in zip(tiles, want):
            assert np.array_equal(t[ew], e[ew]), case


def _mutant_cases(name):
    return [c for c in cases() if MUTANTS[name][1](c)][::2]


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fail(ref, name):
    mut = MUTANTS[name][0]
    assert any(check_fails(case, ref_run(ref, case), **mut) for case in _mutant_cases(name)), f"mutant {name} still equals the reference"


# ---- CPU: the golden fixtures (the reference where it is not built) ---------------------------------------------
def golden_cases():
    """a subset of cases() small enough to keep as fixtures"""
    return [c for i, c in enumerate(cases()) if R.linesize(c[2], c[1]) * c[3] <= 4000 and i % 8 == 0]


def golden_key(case):
    f, c, w, h, p, seed = case
    return f"{f}_{c}_{w}x{h}_s{seed}"


def golden_run(g, case):
    k = golden_key(case)
    res = []
    for i in range(len(model(case))):
        a = g[f"{k}_{i}_out"]
        fl = np.unpackbits(g[f"{k}_{i}_flags"])[:2 * a.size].reshape(2, a.size).astype(bool)
        res.append((a, fl[0], fl[1]))
    return res


def test_restatement_equals_golden():
    g = util.golden(GOLDEN)
    cs = golden_cases()
    assert all(f"{golden_key(c)}_0_out" in g.files for c in cs), "fixtures out of date: run tests/golden/make_geometry_filters_golden.py"
    for case in cs:
        check(case, golden_run(g, case))


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fail_golden(name):
    g = util.golden(GOLDEN)
    cs = [c for c in golden_cases() if MUTANTS[name][1](c)]
    assert any(check_fails(case, golden_run(g, case), **MUTANTS[name][0]) for case in cs), f"mutant {name} still equals the reference"


# ---- GPU --------------------------------------------------------------------------------------------------------
def frame_len(case):
    """the output frame of each buffer: what the device may write"""
    f, c, w, h, p, seed = case
    if f == "crop":
        ow, oh, _, _ = R.crop_geometry(c, w, h, *p[:4])
        return [(p[4] or R.linesize(ow, c)) * oh]
    if f == "split":
        return [R.linesize(w // p[0], c) * (h // p[1])] * (p[0] * p[1])
    return [R.linesize(w, c) * h]


def contract(case):
    """[(bytes, mask)] per output frame: the bytes the device writes (mask) and their values"""
    res = []
    for (e, ew, eu), n in zip(model(case), frame_len(case)):
        m = np.zeros(n, bool)
        v = np.zeros(n, np.uint8)
        k = min(n, e.size)
        m[:k] = (ew & ~eu)[:k]
        v[:k] = e[:k]
        res.append((v, m))
    return res


def run_gpu(case, src_off=0, dst_off=0, stream=None):
    import torch
    from ultragrid_b200 import api
    f, c, w, h, p, seed = case
    src = frame(c, w, h, seed)
    s = util.Guarded(src.size, src_off, 0x33, src)
    outs = [util.Guarded(n, dst_off, 0xC3) for n in frame_len(case)]
    d = outs[0].view
    if f == "flip":
        api.flip(c, s.view, w, h, dst=d, stream=stream)
    elif f == "mirror":
        api.mirror(c, s.view, w, h, dst=d, stream=stream)
    elif f == "crop":
        api.crop(c, s.view, w, h, p[0], p[1], p[2], p[3], pitch=p[4] or 0, dst=d, stream=stream)
    elif f == "split":
        api.split(c, s.view, w, h, p[0], p[1], tiles=[o.view for o in outs], stream=stream)
    elif f == "border":
        color, bw, bh = R.border_init(p[0])
        api.border(c, s.view, w, h, color, bw, bh, dst=d, stream=stream)
    else:
        right = frame(c, w, h, seed + 1)
        r = util.Guarded(right.size, (src_off * 7) % 16, 0x44, right)
        api.interlaced_3d(c, s.view, r.view, w, h, dst=d, stream=stream)
        torch.cuda.synchronize()
        assert np.array_equal(r.check_outside(), right), "the right tile changed"
    torch.cuda.synchronize()
    assert np.array_equal(s.check_outside(), src), "the source changed"
    return [o.check_outside() for o in outs]


def gpu_check(case, src_off=0, dst_off=0, stream=None):
    got = run_gpu(case, src_off, dst_off, stream)
    for i, (g, (v, m)) in enumerate(zip(got, contract(case))):
        assert np.array_equal(g[m], v[m]), f"{case} buffer {i} (offsets {src_off}, {dst_off}) differs from the restatement"
        assert (g[~m] == 0xC3).all(), f"{case} buffer {i} (offsets {src_off}, {dst_off}) wrote bytes the contract leaves alone"


OFFSETS = ((0, 0), (1, 0), (0, 1), (3, 15), (15, 3), (1, 1))


def _gpu_small(filt):
    """the CPU corpus on the codecs each filter takes (the others are refusals, test_gpu_refusals_write_nothing)"""
    takes = {"mirror": (UYVY,), "border": (UYVY, RGB, RGBA)}
    cs = [c for c in cases() if c[0] == filt and c[1] in takes.get(filt, (c[1],))]
    return cs[::3] if len(cs) > 300 else cs


@pytest.mark.gpu
@pytest.mark.parametrize("filt", FILTERS)
def test_gpu_small_and_odd_sizes(filt):
    for i, case in enumerate(_gpu_small(filt)):
        so, do = OFFSETS[i % len(OFFSETS)]
        gpu_check(case, so, do)


@pytest.mark.gpu
@pytest.mark.parametrize("so,do", [(0, 0), (1, 3), (3, 1), (15, 0), (0, 15)])
def test_gpu_address_offsets(so, do):
    """every filter at source and destination offsets 0, 1, 3 and 15"""
    for case in (("flip", v210, 131, 7, None, 1), ("mirror", UYVY, 130, 5, None, 2), ("mirror", UYVY, 131, 5, None, 3),
                 ("crop", RGB, 131, 7, (64, 5, 3, 1, None), 4), ("crop", v210, 131, 7, (100, 5, 7, 1, 400), 5),
                 ("split", v210, 300, 8, (3, 2), 6), ("split", RGB, 35, 4, (5, 4), 7), ("border", UYVY, 37, 21, ("width=3:height=5",), 8),
                 ("border", RGB, 37, 21, ("",), 9), ("interlaced_3d", RGB, 7, 5, None, 10), ("interlaced_3d", UYVY, 64, 6, None, 11)):
        gpu_check(case, so, do)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)])
def test_gpu_4k_8k(w, h):
    for case in (("flip", UYVY, w, h, None, 1), ("flip", v210, w, h, None, 2), ("mirror", UYVY, w, h, None, 3),
                 ("crop", RGB, w, h, (w // 2, h // 2, 1001, 17, None), 4), ("crop", v210, w, h, (w // 2, h // 2, 1001, 17, None), 5),
                 ("split", v210, w, h, (4, 4), 6), ("split", RGB, w, h, (2, 2), 7), ("border", UYVY, w, h, ("",), 8),
                 ("border", RGBA, w, h, ("color=#123456:width=31:height=40",), 9), ("interlaced_3d", UYVY, w, h, None, 10)):
        gpu_check(case, 0, 0)
    gpu_check(("crop", UYVY, w, h, (w // 2, h // 2, 333, 9, None), 12), 1, 3)


@pytest.mark.gpu
def test_gpu_side_stream():
    import torch
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for case in (("flip", RGB, 1921, 1081, None, 1), ("mirror", UYVY, 1918, 1081, None, 2), ("crop", v210, 1920, 1080, (700, 500, 99, 3, None), 3),
                     ("split", v210, 1920, 1080, (8, 4), 4), ("border", UYVY, 1920, 1080, ("",), 5), ("interlaced_3d", RGB, 1921, 1081, None, 6)):
            gpu_check(case, 0, 0, stream=st)


@pytest.mark.gpu
def test_gpu_split_many_tiles():
    """tile counts far past any inline table: 64 x 2, and one tile per pixel column of a small frame"""
    gpu_check(("split", RGB, 128, 4, (64, 2), 1))
    gpu_check(("split", UYVY, 160, 3, (80, 3), 2))


@pytest.mark.gpu
def test_gpu_round_trips():
    """flip twice is the identity; split then a re-merge gives back the frame wherever the tiles cover it"""
    from ultragrid_b200 import api
    for c, w, h in ((UYVY, 1921, 1081), (v210, 1920, 1080), (RGB, 131, 7)):
        src = frame(c, w, h, 77)
        s = util.dev(src)
        assert np.array_equal(api.flip(c, api.flip(c, s, w, h), w, h).cpu().numpy(), src)
    for c, w, h, x, y in ((v210, 1920, 1080, 4, 4), (RGB, 1920, 1080, 3, 2), (R12L, 960, 540, 2, 2), (R10k, 640, 480, 5, 3)):
        src = frame(c, w, h, 78)
        tiles = [t.cpu().numpy() for t in api.split(c, util.dev(src), w, h, x, y)]
        L, tl, n = R.linesize(w, c), R.linesize(w // x, c), int((w // x) * R.bpp(c))
        offs = R.split_offsets(c, w, x)
        merged = np.zeros((h, L), np.uint8)
        cover = np.zeros((h, L), bool)
        for t, tile in enumerate(tiles):
            ty, tx = divmod(t, x)
            rows = tile.reshape(h // y, tl)[:, :n]
            merged[ty * (h // y):(ty + 1) * (h // y), offs[tx]:offs[tx] + n] = rows
            cover[ty * (h // y):(ty + 1) * (h // y), offs[tx]:offs[tx] + n] = True
        assert cover[:, :offs[-1] + n].all()
        assert np.array_equal(merged[cover], src.reshape(h, L)[cover]), (c, w, h, x, y)


@pytest.mark.gpu
def test_gpu_refusals_write_nothing():
    import torch
    from ultragrid_b200 import _lib
    L = _lib.load()
    w, h = 64, 8
    src = torch.randint(0, 256, (1 << 16,), dtype=torch.uint8, device="cuda")
    dst = torch.full((1 << 16,), 0x77, dtype=torch.uint8, device="cuda")
    sp, dp, st = ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    col = (ctypes.c_uint8 * 4)(1, 2, 3, 4)
    tiles = (ctypes.c_void_p * 4)(*[dst.data_ptr() + i * 4096 for i in range(4)])
    bad_tiles = (ctypes.c_void_p * 4)(dst.data_ptr(), None, dst.data_ptr() + 8192, dst.data_ptr() + 12288)
    ovl_tiles = (ctypes.c_void_p * 4)(dst.data_ptr(), src.data_ptr() + 100, dst.data_ptr() + 8192, dst.data_ptr() + 12288)
    calls = [
        (-4, lambda: L.ugb200_cf_mirror(RGB, w, h, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_mirror(v210, w, h, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_crop(9, w, h, 8, 8, 0, 0, sp, dp, 0, st)),  # DXT1
        (-4, lambda: L.ugb200_cf_crop(29, w, h, 8, 8, 0, 0, sp, dp, 0, st)),  # I420
        (-4, lambda: L.ugb200_cf_split(13, w, h, 2, 2, sp, tiles, st)),  # JPEG
        (-4, lambda: L.ugb200_pp_border(v210, w, h, col, 2, 2, sp, dp, st)),
        (-4, lambda: L.ugb200_pp_border(R.YUYV, w, h, col, 2, 2, sp, dp, st)),
        (-4, lambda: L.ugb200_cf_flip(0, w, h, sp, dp, st)),
        (-4, lambda: L.ugb200_pp_interlaced_3d(0, w, h, sp, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_split(v210, w, h, 3, 2, sp, tiles, st)),  # 64 % 3
        (-1, lambda: L.ugb200_cf_split(v210, w, h, 2, 3, sp, tiles, st)),  # 8 % 3
        (-1, lambda: L.ugb200_cf_split(RGB, w, h, 0, 2, sp, tiles, st)),
        (-1, lambda: L.ugb200_cf_split(RGB, w, h, 2, 2, sp, bad_tiles, st)),
        (-1, lambda: L.ugb200_cf_split(RGB, w, h, 2, 2, sp, ovl_tiles, st)),
        (-1, lambda: L.ugb200_pp_border(UYVY, w, h, col, 2, 5, sp, dp, st)),  # 2 * 5 > 8
        (-1, lambda: L.ugb200_pp_border(UYVY, w, h, col, 65, 2, sp, dp, st)),  # 33 groups > 32
        (-1, lambda: L.ugb200_pp_border(RGB, w, h, col, 65, 2, sp, dp, st)),
        (-1, lambda: L.ugb200_pp_border(RGBA, w, h, None, 2, 2, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_crop(RGB, w, h, 16, 4, -1, 0, sp, dp, 0, st)),  # first row before the source
        (-1, lambda: L.ugb200_cf_crop(RGB, w, h, 16, 4, 0, -1, sp, dp, 0, st)),
        (-1, lambda: L.ugb200_cf_crop(RGB, w, h, -3, 4, 0, 0, sp, dp, 0, st)),
        (-1, lambda: L.ugb200_cf_flip(RGB, w, 0, sp, dp, st)),
        (-1, lambda: L.ugb200_cf_flip(RGB, w, h, None, dp, st)),
        (-1, lambda: L.ugb200_cf_flip(RGB, w, h, sp, ctypes.c_void_p(src.data_ptr() + 5), st)),  # overlap
        (-1, lambda: L.ugb200_cf_mirror(UYVY, w, h, sp, ctypes.c_void_p(src.data_ptr() + 4), st)),
        (-1, lambda: L.ugb200_pp_interlaced_3d(RGB, w, h, sp, ctypes.c_void_p(dst.data_ptr() + 8), dp, st)),
        (-1, lambda: L.ugb200_pp_interlaced_3d(RGB, w, 0, sp, sp, dp, st)),
    ]
    for i, (want, call) in enumerate(calls):
        assert call() == want, i
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 0x77).all(), "a refusal wrote"
    # a crop clamped where the sum wraps is no refusal
    assert L.ugb200_cf_crop(RGB, w, h, 16, 4, -17, 0, sp, dp, 0, st) == 0
