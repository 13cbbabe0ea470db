"""The logo capture filter and the R12L <-> Y416 pass-through filters on the GPU (logo_kernels.cu, ugb200_cf_logo,
ugb200_cf_r12l_to_y416_fake, ugb200_pp_y416_to_r12l_fake).

CPU: the numpy restatement (logo_filter_ref.py) equals the unmodified logo.c, r12l_to_y416_fake.c and
y416_to_r12l_fake.c on every byte they write: a run on a random frame shows the bytes (the frame after the filter
equals the restatement's everywhere, slack included), and a run with every byte outside the restatement's written
span set to a second fill shows that none of them is written.  Logo widths whose segment the reference allocates
too short are checked against the reference run with the logo padded by transparent columns to the next width it
handles (DESIGN.md §8).  The module's own init loads 3- and 4-channel PAM files.  Mutants fail.  The golden fixtures
stand in for the reference where it is not built.
GPU: the kernels equal the restatement's contract form, with sentinels around every buffer.
"""
import ctypes
import os

import numpy as np
import pytest

import logo_filter_ref as R
import util

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "logo_filters_golden.npz")
FILLS = (0x00, 0xA5)
SLACK = 4096
RGB, RGBA, UYVY, RG48, R12L = R.RGB, R.RGBA, R.UYVY, R.RG48, R.R12L
CODECS = R.LOGO_CODECS


def logo_rgba(w, h, alpha, seed):
    """h x w x 4: random colours; alpha 0, 255, or random ("rnd") with 0 and 255 sprinkled in"""
    a = util.rng_bytes(w * h * 4, seed).reshape(h, w, 4)
    if alpha == "rnd":
        a[::3, ::2, 3] = 0
        a[1::3, 1::2, 3] = 255
    else:
        a[:, :, 3] = alpha
    return a


def frame(c, W, H, seed):
    return util.rng_bytes(R.linesize(W, c) * H, seed)


# ---- the reference ---------------------------------------------------------------------------------------------
def _bind(lib):
    vp, i, u, s = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_char_p
    lib.ref_logo_init.argtypes, lib.ref_logo_init.restype = [s], vp
    lib.ref_logo_state.argtypes = [vp, vp, vp]
    lib.ref_logo_make.argtypes, lib.ref_logo_make.restype = [vp, u, u, i, i], vp
    lib.ref_logo_done.argtypes = [vp]
    lib.ref_logo_filter.argtypes = [vp, i, i, i, vp]
    lib.ref_r12l_to_y416_task.argtypes = [i, i, i, vp, vp]
    lib.ref_r12l_to_y416_filter.argtypes = [s, i, i, vp, vp]
    lib.ref_y416_to_r12l_task.argtypes = [i, i, i, vp, vp, i]
    lib.ref_y416_to_r12l_postprocess.argtypes = [s, i, i, vp, vp, i]
    return lib


def ref_lib():
    return util.ref_lib("liblogo_filters_ref.so", _bind)


@pytest.fixture(scope="module")
def ref():
    lib = ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/liblogo_filters_ref.so not built (reference tree absent)")
    return lib


def ref_logo_once(ref, c, W, H, rgba, x, y, data, slack_fill):
    """the unmodified filter() on `data` (a frame) followed by SLACK bytes of slack: the bytes after it"""
    h, w, _ = rgba.shape
    buf = np.full(data.size + SLACK, slack_fill, np.uint8)
    buf[:data.size] = data
    lg = np.ascontiguousarray(rgba)
    st = ref.ref_logo_make(lg.ctypes.data, w, h, x, y)
    assert ref.ref_logo_filter(st, c, W, H, buf.ctypes.data) == 0
    ref.ref_logo_done(st)
    return buf


# ---- the cases: (codec, W, H, w, h, x, y, alpha, seed) --------------------------------------------------------------
def logo_cases():
    res = []
    k = 1
    alphas = (0, 255, "rnd")
    for c in CODECS:
        bp = R.block_px(c)
        # logo widths 1-150 and heights 1-5 at the default and an explicit position, over frames just wide enough
        # R12L handles only w % 72 in {0, 71}: more of those
        for w in list(range(1, 151)) + ([72 * k - j for k in range(3, 9) for j in (0, 1)] if c == R12L else []):
            h = 1 + w % 5
            wp = R.logo_padded_width(c, w)
            W = R.round_up(wp + 3 * bp + 17, bp) + (w % 3)
            res.append((c, W, h + 2, w, h, 5 + w % 7, 1, alphas[w % 3], k))
            res.append((c, W, h + 1, w, h, -1, -1, alphas[(w + 1) % 3], k + 1))
            k += 2
        # frame widths around each block boundary and at the usual sizes; positions inside, negative, too large
        for W in sorted({bp * 8 - 1, bp * 8, bp * 8 + 1, 36, 37, 71, 72, 73, 1918, 1920, 7680}):
            for w, h in ((1, 1), (5, 2), (16, 3), (33, 4), (W, 2), (W - 1, 3)):
                for x, y in ((-1, -1), (0, 0), (3, 1), (W - w, 0), (W, 9), (-5, -2), (W - w + 1, 1)):
                    if w >= 1:
                        res.append((c, W, 5, w, h, x, y, alphas[k % 3], k))
                        k += 1
    return res


def logo_run_case(case):
    """the restatement's result: None (refusal), or (frame after, written)"""
    c, W, H, w, h, x, y, alpha, seed = case
    return R.logo(c, frame(c, W, H, seed), W, H, logo_rgba(w, h, alpha, seed), x, y)


def ref_logo_case(ref, case):
    """(random-frame run, frame-and-slack after the fill run) of the reference, for a case it handles"""
    c, W, H, w, h, x, y, alpha, seed = case
    f = frame(c, W, H, seed)
    rgba = logo_rgba(w, h, alpha, seed)
    _, written = R.logo(c, f, W, H, rgba, x, y)
    a = ref_logo_once(ref, c, W, H, rgba, x, y, f, 0x11)
    g = np.where(written, f, FILLS[1]).astype(np.uint8)
    b = ref_logo_once(ref, c, W, H, rgba, x, y, g, FILLS[1])
    return a, b


def check_logo(case, a, b, **mutant):
    c, W, H, w, h, x, y, alpha, seed = case
    f = frame(c, W, H, seed)
    out, written = R.logo(c, f, W, H, logo_rgba(w, h, alpha, seed), x, y, **mutant)
    n = f.size
    assert (a[n:] == 0x11).all() and (b[n:] == FILLS[1]).all(), f"{case}: the reference wrote past the frame"
    assert np.array_equal(b[:n][~written], np.full((~written).sum(), FILLS[1], np.uint8)), f"{case}: the reference wrote outside the span"
    assert np.array_equal(a[:n], out), f"{case}: bytes differ from the restatement"


def check_logo_fails(case, a, b, **mutant):
    try:
        check_logo(case, a, b, **mutant)
    except AssertionError:
        return True
    return False


def ref_cases():
    """the cases the reference runs as they are: its own logo widths, placed inside the row"""
    return [cs for cs in logo_cases() if R.logo_handled(cs[0], cs[3]) and logo_run_case(cs) is not None]


# ---- CPU: logo against the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", CODECS)
def test_logo_restatement_equals_reference(ref, codec):
    cs = [c for c in ref_cases() if c[0] == codec]
    assert len(cs) > (150 if codec != R12L else 50)
    for case in cs:
        check_logo(case, *ref_logo_case(ref, case))


@pytest.mark.parametrize("codec", CODECS)
def test_logo_short_segment_widths_equal_padded_reference(ref, codec):
    """widths the reference's segment is too short for: the restatement's bytes equal the unmodified filter run with
    the logo padded by fully transparent columns to the next width it handles, on each row's written span"""
    n = 0
    for w in range(1, 151):
        if R.logo_handled(codec, w):
            continue
        wp = R.logo_padded_width(codec, w)
        for h, x, alpha in ((1 + w % 5, 3 + w % 11, "rnd"), (2, 0, 255)):
            bp = R.block_px(codec)
            W = R.round_up(x + wp + 2 * bp + 40, bp)
            H = h + 3
            case = (codec, W, H, w, h, x, 2, alpha, 7000 + w)
            f = frame(codec, W, H, case[-1])
            rgba = logo_rgba(w, h, alpha, case[-1])
            out, written = R.logo(codec, f, W, H, rgba, x, 2)
            padded = np.zeros((h, wp, 4), np.uint8)
            padded[:, :w] = rgba
            got = ref_logo_once(ref, codec, W, H, padded, x, 2, f, 0x11)
            assert np.array_equal(got[:f.size][written], out[written]), case
            assert np.array_equal(got[:f.size][~written], f[~written]) or wp > w, case
            n += 1
    assert n > 40 or codec == RGB and n > 20


def test_logo_span_past_the_row_is_written_by_the_reference(ref):
    """case (b) of DESIGN.md §8: a logo wider than the frame by less than one block lands at 0 and its span passes
    the row's end; on the last row (the default y) the reference writes past the frame, which the device refuses"""
    for c, W, w in ((RGB, 10, 11), (RGBA, 10, 12), (RG48, 12, 15), (R12L, 64, 70), (UYVY, 10, 12)):
        rc, rect_x, _, off, span = R.logo_place(c, W, 3, w, 2, -1, -1)
        assert rc == -1 and rect_x == 0, (c, W, w)
        if not R.logo_handled(c, w):
            continue
        got = ref_logo_once(ref, c, W, 3, logo_rgba(w, 2, 255, 3), -1, -1, frame(c, W, 3, 3), 0x11)
        assert (got[R.linesize(W, c) * 3:] != 0x11).any(), (c, W, w)


def _write_pam(path, rgba, channels):
    h, w, _ = rgba.shape
    data = rgba[:, :, :channels].tobytes()
    with open(path, "wb") as f:
        f.write(f"P7\nWIDTH {w}\nHEIGHT {h}\nDEPTH {channels}\nMAXVAL 255\nTUPLTYPE {'RGB_ALPHA' if channels == 4 else 'RGB'}\nENDHDR\n".encode())
        f.write(data)


@pytest.mark.parametrize("channels", (3, 4))
def test_logo_pam_loaded_by_init(ref, tmp_path, channels):
    """logo:<file>[:x[:y]] through the module's own init: 3-channel files are widened with alpha 0xFF"""
    for c, W, H, w, h, x, y in ((RGB, 64, 9, 17, 5, 3, 2), (UYVY, 100, 7, 24, 3, None, None), (R12L, 144, 6, 72, 4, 8, None),
                                 (RGBA, 33, 5, 7, 2, 20, 1), (RG48, 40, 4, 11, 3, -1, -1)):
        rgba = logo_rgba(w, h, "rnd", w)
        path = str(tmp_path / f"logo{c}.pam")
        _write_pam(path, rgba, channels)
        cfg = path + (f":{x}" if x is not None else "") + (f":{y}" if y is not None else "")
        st = ref.ref_logo_init(cfg.encode())
        assert st
        geom = (ctypes.c_int * 4)()
        got = np.zeros(w * h * 4, np.uint8)
        ref.ref_logo_state(st, geom, got.ctypes.data)
        want = rgba.copy()
        if channels == 3:
            want[:, :, 3] = 0xFF
        ex, ey = -1 if x is None else x, -1 if y is None else y
        assert tuple(geom) == (w, h, ex, ey)
        assert np.array_equal(got, want.reshape(-1))
        f = frame(c, W, H, 5)
        buf = np.concatenate([f, np.full(SLACK, 0x11, np.uint8)])
        assert ref.ref_logo_filter(st, c, W, H, buf.ctypes.data) == 0
        ref.ref_logo_done(st)
        out, _ = R.logo(c, f, W, H, want, ex, ey)
        assert np.array_equal(buf[:f.size], out), (c, channels)
    assert not ref.ref_logo_init(b"")  # help
    assert not ref.ref_logo_init(str(tmp_path / "logo.png").encode())


def test_logo_other_codecs_return_their_input(ref):
    for c in (R.v210, R.R10k, R.Y416, R.YUYV, R.BGR):
        f = frame(c, 64, 4, 1)
        buf = np.concatenate([f, np.zeros(SLACK, np.uint8)])
        lg = logo_rgba(8, 2, 255, 1)
        st = ref.ref_logo_make(lg.ctypes.data, 8, 2, -1, -1)
        assert ref.ref_logo_filter(st, c, 64, 4, buf.ctypes.data) == 1
        ref.ref_logo_done(st)
        assert np.array_equal(buf[:f.size], f)


# ---- CPU: the R12L <-> Y416 pair against the reference ----------------------------------------------------------------
FAKE_SIZES = [(w, h) for w in (8, 16, 48, 200) for h in range(1, 8)] + [(1920, 1080), (1920, 1081), (64, 1080), (64, 1081)]


def fake_cases():
    res = []
    k = 9000
    for full in (False, True):
        for w, h in FAKE_SIZES:
            for extra in (0, 20):
                res.append((full, w, h, extra, k))
                k += 1
    return res


def r12l_src(w, h, seed):
    return util.rng_bytes(R.linesize(w, R12L) * h, seed)


def y416_src(w, h, seed):
    return util.rng_bytes(8 * w * h, seed)


def ref_r12l_to_y416(ref, case):
    """(filter() output in full range, else None; task output with 64 bytes of slack, under two fills)"""
    full, w, h, _, seed = case
    src = r12l_src(w, h, seed)
    n = 8 * w * h
    out = None
    if full:  # init reaches only full range (test_module_options)
        out = np.zeros(n, np.uint8)
        assert ref.ref_r12l_to_y416_filter(b"", w, h, src.ctypes.data, out.ctypes.data) == 0
    tasks = []
    for fill in FILLS:
        t = np.full(n + 64, fill, np.uint8)
        ref.ref_r12l_to_y416_task(int(full), w, h, src.ctypes.data, t.ctypes.data)
        tasks.append(t)
    return out, tasks


def ref_y416_to_r12l(ref, case):
    """(postprocess() at pitch == linesize (the task there in limited range), the task at linesize + extra), each under
    two fills, with 64 bytes of slack"""
    full, w, h, extra, seed = case
    src = y416_src(w, h, seed)
    L = R.linesize(w, R12L)
    res = []
    for pitch, pp in ((L, full), (L + extra, False)):  # init reaches only full range (test_module_options)
        runs = []
        for fill in FILLS:
            o = np.full(pitch * h + 64, fill, np.uint8)
            if pp:
                assert ref.ref_y416_to_r12l_postprocess(b"", w, h, src.ctypes.data, o.ctypes.data, pitch) == 0
            else:
                ref.ref_y416_to_r12l_task(int(full), w, h, src.ctypes.data, o.ctypes.data, pitch)
            runs.append(o)
        res.append((pitch, runs))
    return res


def check_r12l_to_y416(case, got, c_scale=14):
    full, w, h, _, seed = case
    want = R.r12l_to_y416(r12l_src(w, h, seed), w, h, full, c_scale=c_scale)
    out, tasks = got
    assert out is None or np.array_equal(out, want), case
    for t in tasks:
        assert np.array_equal(t[:want.size], want) and (t[want.size:] == t[-1]).all(), case


def check_y416_to_r12l(case, got, c_scale=14):
    full, w, h, extra, seed = case
    src = y416_src(w, h, seed)
    for pitch, (a, b) in got:
        want, written = R.y416_to_r12l(src, w, h, full, pitch, c_scale=c_scale)
        n = want.size
        wr = a == b
        assert np.array_equal(wr[:n], written) and wr[n:].sum() == 0, (case, pitch)
        assert np.array_equal(a[:n][written], want[written]), (case, pitch)


def test_r12l_to_y416_restatement_equals_reference(ref):
    for case in fake_cases():
        if case[3] == 0:
            check_r12l_to_y416(case, ref_r12l_to_y416(ref, case))


def test_y416_to_r12l_restatement_equals_reference(ref):
    for case in fake_cases():
        check_y416_to_r12l(case, ref_y416_to_r12l(ref, case))


def test_module_options(ref):
    """both modules' init takes `full-range` by IS_PREFIX, for which the empty option is a prefix: without an option
    they run in full range, and no option reaches limited range (the entry points take the state's flag)"""
    w, h = 16, 2
    src = r12l_src(w, h, 3)
    full = R.r12l_to_y416(src, w, h, True)
    for cfg in (b"", b"full-range", b"full", b"f"):
        out = np.zeros(8 * w * h, np.uint8)
        assert ref.ref_r12l_to_y416_filter(cfg, w, h, src.ctypes.data, out.ctypes.data) == 0
        assert np.array_equal(out, full), cfg
        o = np.zeros(R.linesize(w, R12L) * h, np.uint8)
        assert ref.ref_y416_to_r12l_postprocess(cfg, w, h, full.ctypes.data, o.ctypes.data, R.linesize(w, R12L)) == 0
        assert np.array_equal(o, src), cfg
    for cfg in (b"limited", b"full-range-x", b"help"):
        out = np.zeros(8 * w * h, np.uint8)
        assert ref.ref_r12l_to_y416_filter(cfg, w, h, src.ctypes.data, out.ctypes.data) == -2, cfg
        assert ref.ref_y416_to_r12l_postprocess(cfg, w, h, full.ctypes.data, out.ctypes.data, R.linesize(w, R12L)) == -2, cfg


def test_fake_pair_round_trip_every_12_bit_value():
    """y416_to_r12l_fake(r12l_to_y416_fake(x)) == x for every 12-bit value in every component, both ranges"""
    w, h = 4096, 1
    i = np.arange(4096)
    px = np.stack([i, (i * 7 + 3) % 4096, 4095 - i], axis=1).reshape(1, w // 8, 8, 3)
    src = R.r12_pack(px).reshape(-1)
    for full in (False, True):
        y = R.r12l_to_y416(src, w, h, full)
        back, _ = R.y416_to_r12l(y, w, h, full, R.linesize(w, R12L))
        assert np.array_equal(back, src), full


# ---- mutants ---------------------------------------------------------------------------------------------------------
LOGO_MUTANTS = {
    "blend_rounding": ({"rounding": True}, lambda c: c[7] != 0),
    "rgba_alpha_kept": ({"keep_alpha": True}, lambda c: c[0] == RGBA),
    "rg48_low_byte_kept": ({"keep_low": True}, lambda c: c[0] == RG48),
    "rect_x_aligned_to_pixels": ({"pixel_align": True}, lambda c: c[0] in (RGB, RG48, R12L, UYVY) and c[5] in (3, -1)),
}


def _logo_mutant_cases(name):
    return [c for c in ref_cases() if LOGO_MUTANTS[name][1](c)][::5][:60]


@pytest.mark.parametrize("name", list(LOGO_MUTANTS))
def test_logo_mutants_fail(ref, name):
    mut = LOGO_MUTANTS[name][0]
    assert any(check_logo_fails(case, *ref_logo_case(ref, case), **mut) for case in _logo_mutant_cases(name)), name


def test_fake_pair_mutant_fails(ref):
    """/ 13 in place of / 14 for R and B"""
    case = fake_cases()[3]
    with pytest.raises(AssertionError):
        check_y416_to_r12l(case, ref_y416_to_r12l(ref, case), c_scale=13)
    with pytest.raises(AssertionError):
        check_r12l_to_y416(case, ref_r12l_to_y416(ref, case), c_scale=13)


# ---- CPU: the golden fixtures (the reference where it is not built) ------------------------------------------------
def golden_logo_cases():
    return [c for i, c in enumerate(ref_cases()) if R.linesize(c[1], c[0]) * c[2] <= 2000 and i % 6 == 0]


def golden_fake_cases():
    return [c for c in fake_cases() if c[1] * c[2] <= 400]


def golden_key(case):
    return "_".join(str(v) for v in case)


def golden_data(ref):
    """what the fixtures hold: the reference's outputs for the golden cases"""
    out = {}
    for case in golden_logo_cases():
        a, b = ref_logo_case(ref, case)
        out[f"logo_{golden_key(case)}_a"], out[f"logo_{golden_key(case)}_b"] = a, b
    for case in golden_fake_cases():
        k = golden_key(case)
        if case[3] == 0:
            o, (t0, t1) = ref_r12l_to_y416(ref, case)
            out[f"r12l_{k}_t0"], out[f"r12l_{k}_t1"] = t0, t1
            if o is not None:
                out[f"r12l_{k}"] = o
        for i, (pitch, (a, b)) in enumerate(ref_y416_to_r12l(ref, case)):
            out[f"y416_{k}_{i}_a"], out[f"y416_{k}_{i}_b"], out[f"y416_{k}_{i}_pitch"] = a, b, np.array(pitch)
    return out


def _golden_y416(g, case):
    k = golden_key(case)
    return [(int(g[f"y416_{k}_{i}_pitch"]), (g[f"y416_{k}_{i}_a"], g[f"y416_{k}_{i}_b"])) for i in range(2)]


def test_restatement_equals_golden():
    g = util.golden(GOLDEN)
    cs = golden_logo_cases()
    assert len(cs) > 100 and all(f"logo_{golden_key(c)}_a" in g.files for c in cs), "fixtures out of date: run tests/golden/make_logo_filters_golden.py"
    for case in cs:
        check_logo(case, g[f"logo_{golden_key(case)}_a"], g[f"logo_{golden_key(case)}_b"])
    for case in golden_fake_cases():
        k = golden_key(case)
        if case[3] == 0:
            check_r12l_to_y416(case, (g[f"r12l_{k}"] if case[0] else None, [g[f"r12l_{k}_t0"], g[f"r12l_{k}_t1"]]))
        check_y416_to_r12l(case, _golden_y416(g, case))


@pytest.mark.parametrize("name", list(LOGO_MUTANTS) + ["c_scale_13"])
def test_mutants_fail_golden(name):
    g = util.golden(GOLDEN)
    if name == "c_scale_13":
        case = golden_fake_cases()[3]
        with pytest.raises(AssertionError):
            check_y416_to_r12l(case, _golden_y416(g, case), c_scale=13)
        return
    mut, sel = LOGO_MUTANTS[name]
    cs = [c for c in golden_logo_cases() if sel(c)]
    assert any(check_logo_fails(c, g[f"logo_{golden_key(c)}_a"], g[f"logo_{golden_key(c)}_b"], **mut) for c in cs), name


# ---- GPU --------------------------------------------------------------------------------------------------------
def gpu_logo_check(case, off=0, stream=None):
    """the frame after the call equals the restatement's everywhere: its span, and nothing else, is written"""
    import torch
    from ultragrid_b200 import api
    c, W, H, w, h, x, y, alpha, seed = case
    f = frame(c, W, H, seed)
    rgba = logo_rgba(w, h, alpha, seed)
    want = R.logo(c, f, W, H, rgba, x, y)
    g = util.Guarded(f.size, off, 0xC3, f)
    lg = api.logo(rgba.reshape(-1), w, h)
    if want is None:
        with pytest.raises(RuntimeError, match="code -1"):
            lg(c, g.view, W, H, x, y, stream=stream)
        want = (f, None)
    else:
        lg(c, g.view, W, H, x, y, stream=stream)
    torch.cuda.synchronize()
    got = g.check_outside()
    lg.close()
    assert np.array_equal(got, want[0]), f"{case} (offset {off}) differs from the restatement"


def _offsets(c):
    return {RGB: (0, 1, 3), RGBA: (0, 1, 3), UYVY: (0, 1, 3), RG48: (0, 2, 6), R12L: (0, 4, 12)}[c]


@pytest.mark.gpu
@pytest.mark.parametrize("codec", CODECS)
def test_gpu_logo_small_and_odd_sizes(codec):
    """the whole CPU corpus of the codec: every logo width 1-150 (the short-segment ones included), refusals too"""
    for i, case in enumerate([c for c in logo_cases() if c[0] == codec]):
        gpu_logo_check(case, _offsets(codec)[i % 3])


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(3840, 2160), (7680, 4320)])
def test_gpu_logo_4k_8k(W, H):
    for c in CODECS:
        for w, h, x, y in ((256, 128, -1, -1), (1920, 1080, 1001, 17), (257, 3, 0, H - 3), (W, 2, -1, -1)):
            gpu_logo_check((c, W, H, w, h, x, y, "rnd", w + h + c), _offsets(c)[1])


@pytest.mark.gpu
def test_gpu_logo_side_stream():
    import torch
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for c in CODECS:
            gpu_logo_check((c, 1920, 1080, 131, 37, -1, -1, "rnd", c), 0, stream=st)


def _fake_gpu(case, src_off=0, dst_off=0, stream=None):
    import torch
    from ultragrid_b200 import api
    full, w, h, extra, seed = case
    L = R.linesize(w, R12L)
    src = r12l_src(w, h, seed)
    s = util.Guarded(src.size, src_off, 0x33, src)
    d = util.Guarded(8 * w * h, dst_off, 0xC3)
    api.r12l_to_y416_fake(s.view, w, h, full, dst=d.view, stream=stream)
    ysrc = y416_src(w, h, seed + 1)
    ys = util.Guarded(ysrc.size, dst_off, 0x44, ysrc)
    pitch = L + extra
    rd = util.Guarded((h - 1) * pitch + L, src_off, 0xC3)
    api.y416_to_r12l_fake(ys.view, w, h, full, pitch=pitch, dst=rd.view, stream=stream)
    torch.cuda.synchronize()
    assert np.array_equal(s.check_outside(), src) and np.array_equal(ys.check_outside(), ysrc), "a source changed"
    assert np.array_equal(d.check_outside(), R.r12l_to_y416(src, w, h, full)), case
    want, written = R.y416_to_r12l(ysrc, w, h, full, pitch)
    got = rd.check_outside()
    assert np.array_equal(got[written], want[written]) and (got[~written] == 0xC3).all(), case


@pytest.mark.gpu
def test_gpu_fake_pair_small_and_odd_sizes():
    for i, case in enumerate(fake_cases()):
        so, do = ((0, 0), (4, 2), (12, 6), (0, 16))[i % 4]
        _fake_gpu(case, so, do)


@pytest.mark.gpu
def test_gpu_fake_pair_4k_8k_and_side_stream():
    import torch
    _fake_gpu((False, 3840, 2160, 0, 1), 0, 0)
    _fake_gpu((True, 7680, 4320, 20, 2), 4, 2)
    _fake_gpu((False, 7680, 4320, 0, 3), 0, 0)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _fake_gpu((True, 1920, 1081, 20, 4), 0, 0, stream=st)


@pytest.mark.gpu
def test_gpu_fake_pair_8k_round_trip_is_the_identity():
    from ultragrid_b200 import api
    w, h = 7680, 4320
    src = util.dev(r12l_src(w, h, 11))
    for full in (False, True):
        back = api.y416_to_r12l_fake(api.r12l_to_y416_fake(src, w, h, full), w, h, full)
        assert bool((back == src).all()), full


@pytest.mark.gpu
def test_gpu_refusals_write_nothing():
    import torch
    from ultragrid_b200 import _lib
    L = _lib.load()
    buf = torch.full((1 << 16,), 0x77, dtype=torch.uint8, device="cuda")
    src = torch.randint(0, 256, (1 << 16,), dtype=torch.uint8, device="cuda")
    sp, st = ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    bp = lambda o=0: ctypes.c_void_p(buf.data_ptr() + o)  # noqa: E731
    rgba = (ctypes.c_uint8 * (16 * 4 * 4))(*([200] * 256))
    lg = L.ugb200_cf_logo_create(rgba, 16, 4)
    lg12 = L.ugb200_cf_logo_create(rgba, 12, 4)
    assert lg and not L.ugb200_cf_logo_create(rgba, 0, 4) and not L.ugb200_cf_logo_create(None, 16, 4)
    calls = [
        (-4, lambda: L.ugb200_cf_logo(lg, R.v210, 64, 8, -1, -1, bp(), st)),
        (-4, lambda: L.ugb200_cf_logo(lg, R.Y416, 64, 8, -1, -1, bp(), st)),
        (-4, lambda: L.ugb200_cf_logo(lg, R.BGR, 64, 8, -1, -1, bp(), st)),
        (-1, lambda: L.ugb200_cf_logo(None, RGB, 64, 8, -1, -1, bp(), st)),
        (-1, lambda: L.ugb200_cf_logo(lg, RGB, 64, 8, -1, -1, None, st)),
        (-1, lambda: L.ugb200_cf_logo(lg, RGB, 0, 8, -1, -1, bp(), st)),
        (-1, lambda: L.ugb200_cf_logo(lg, RGB, 64, -1, -1, -1, bp(), st)),
        (-1, lambda: L.ugb200_cf_logo(lg, RG48, 64, 8, -1, -1, bp(1), st)),
        (-1, lambda: L.ugb200_cf_logo(lg, R12L, 64, 8, -1, -1, bp(2), st)),
        (-1, lambda: L.ugb200_cf_logo(lg, RGB, 15, 8, -1, -1, bp(), st)),    # one pixel too narrow: the span passes the row
        (-1, lambda: L.ugb200_cf_logo(lg12, R12L, 48, 8, -1, -1, bp(), st)),  # rect_x 36 lands at pixel 40: its two groups pass the row's six
        (0, lambda: L.ugb200_cf_logo(lg, RGB, 12, 8, -1, -1, bp(), st)),     # rect_x -3 -> nothing written
        (0, lambda: L.ugb200_cf_logo(lg, RGB, 64, 3, -1, -1, bp(), st)),     # rect_y -1 -> nothing written
        (-1, lambda: L.ugb200_cf_r12l_to_y416_fake(12, 4, 0, sp, bp(), st)),  # width % 8
        (-1, lambda: L.ugb200_cf_r12l_to_y416_fake(16, 4, 0, ctypes.c_void_p(src.data_ptr() + 2), bp(), st)),
        (-1, lambda: L.ugb200_cf_r12l_to_y416_fake(16, 4, 0, sp, bp(1), st)),
        (-1, lambda: L.ugb200_cf_r12l_to_y416_fake(16, 0, 0, sp, bp(), st)),
        (-1, lambda: L.ugb200_cf_r12l_to_y416_fake(16, 4, 1, bp(), bp(100), st)),  # overlap
        (-1, lambda: L.ugb200_pp_y416_to_r12l_fake(12, 4, 0, sp, bp(), 54, st)),
        (-1, lambda: L.ugb200_pp_y416_to_r12l_fake(16, 4, 0, sp, bp(), 71, st)),  # pitch < 72
        (-1, lambda: L.ugb200_pp_y416_to_r12l_fake(16, 4, 0, ctypes.c_void_p(src.data_ptr() + 1), bp(), 72, st)),
        (-1, lambda: L.ugb200_pp_y416_to_r12l_fake(16, 4, 0, sp, bp(2), 72, st)),
        (-1, lambda: L.ugb200_pp_y416_to_r12l_fake(16, 4, 0, sp, None, 72, st)),
        (-1, lambda: L.ugb200_pp_y416_to_r12l_fake(16, 4, 0, bp(), bp(64), 72, st)),  # overlap
    ]
    for i, (want, call) in enumerate(calls):
        assert call() == want, i
    torch.cuda.synchronize()
    L.ugb200_cf_logo_destroy(lg)
    L.ugb200_cf_logo_destroy(lg12)
    assert (buf.cpu().numpy() == 0x77).all(), "a refusal wrote"
