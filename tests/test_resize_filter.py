"""The resize capture filter / postprocessor on the GPU (resize_kernels.cu, ugb200_cf_resize).

CPU, against the unmodified resize.c (oracle/resize_filter.mk, or the golden fixture where the reference is not
built): the module's init / parse_fmt equals the restatement's parse; for every codec, filter() picks the route codec
ugb200_cf_resize_geometry picks, gives the output codec and size it gives, and hands resize_frame exactly the pixfmt
oracle's conversion.  The letterbox comes from the restatement (resize_filter_ref.py).
CPU, the contract pinned without OpenCV: the colour stage against float64 BT.601, linear against a float64 bilinear,
invariants, and mutants that each fail one of those checks.
GPU: api.resize equals the restatement byte for byte, with sentinels around the exact output length.
"""
import ctypes
import os

import numpy as np
import pytest

import resize_filter_ref as R
import util

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_filter_golden.npz")
SLACK = 4096
PARSE_CORPUS = ["1/2", "0.5", ".5", "2", "3/0", "1280x720", "1280x", "x720", "algo=nearest", "a=area", "algorithm=help",
                "foo", "1/2:algo=cubic", "1/2:algo=nearest", "1/3:a=area", "1280x720:algorithm=linear", "1/2:algo=bogus",
                "=lanczos4:3/4", "help", "HELP", "0", "0/2", "1/-2", "2x0", "0x2", "-1", "1280x720:0.5", "0.5:1280x720",
                "1e-1", "7680x4320", "1/2:", "::1/2", "1/2:algo=help", "1.5", "3/2:al=area"]


def frame(c, w, h, seed):
    from ultragrid_b200 import vc_get_linesize
    n = R.frame_len(c, w, h) if c == R.I420 else vc_get_linesize(w, c) * h
    return util.rng_bytes(n, seed)


# ---- the reference -----------------------------------------------------------------------------------------------
def _bind(lib):
    vp, i, s = ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p
    lib.ref_resize_init.argtypes = [s, vp, vp, vp]
    lib.ref_resize_done.argtypes = [vp]
    lib.ref_resize_filter.argtypes = [vp, i, i, i, vp, vp]
    lib.ref_resize_last.argtypes, lib.ref_resize_last.restype = [vp, vp, ctypes.c_long], ctypes.c_long
    return lib


def ref_lib():
    return util.ref_lib("libresize_filter_ref.so", _bind)


def ref_parse(ref, cfg):
    """(rc, (mode, factor, tw, th, algo) or None) of the module's init()"""
    st, p, f = ctypes.c_void_p(), (ctypes.c_int * 4)(), ctypes.c_double()
    rc = ref.ref_resize_init(cfg.encode(), ctypes.byref(st), p, ctypes.byref(f))
    if rc != 0:
        return rc, None
    ref.ref_resize_done(st)
    return rc, (p[0], f.value, p[1], p[2], p[3])


def ref_filter(ref, cfg, c, w, h, data):
    """None (frame dropped) or (out codec, out w, out h, data_len, in_color, width, height, bytes handed)"""
    st, p, f = ctypes.c_void_p(), (ctypes.c_int * 4)(), ctypes.c_double()
    assert ref.ref_resize_init(cfg.encode(), ctypes.byref(st), p, ctypes.byref(f)) == 0
    buf = np.zeros(data.size + SLACK, np.uint8)
    buf[:data.size] = data
    out = (ctypes.c_long * 11)()
    rc = ref.ref_resize_filter(st, c, w, h, buf.ctypes.data, out)
    res = None
    if rc == 0:
        n = ref.ref_resize_last(ctypes.byref(f), None, 0)
        got = np.zeros(n, np.uint8)
        ref.ref_resize_last(ctypes.byref(f), got.ctypes.data, n)
        res = tuple(int(v) for v in out[:7]) + (got,)
    ref.ref_resize_done(st)
    return res


# ---- the cases -----------------------------------------------------------------------------------------------------
def all_codecs():
    from ultragrid_b200 import Codec
    return [int(c) for c in Codec if int(c) != 0]


ROUTE_CFGS = ["1/2", "0.7", "1280x720:algo=nearest"]
ROUTE_SIZES = [(16, 8), (17, 9), (48, 6), (96, 4), (3, 5)]


def route_cases():
    return [(cfg, c, w, h) for cfg in ROUTE_CFGS for c in all_codecs() for w, h in ROUTE_SIZES]


def lib_geometry(cfg, c, w, h):
    from ultragrid_b200 import api
    rc, p = R.parse(cfg)
    mode, factor, tw, th, algo = p
    r = api.Resize(factor=factor, algo=algo) if mode == R.FRACTION else api.Resize(size=(tw, th), algo=algo)
    try:
        return r.geometry(c, w, h)
    except RuntimeError as e:
        return int(str(e).rsplit(" ", 1)[1])
    finally:
        r.close()


def route_bytes(c, route, w, h, data):
    """what filter() hands resize_frame: the frame itself, or its conversion to the route codec (the pixfmt oracle)"""
    if c == route:
        return data[:R.frame_len(c, w, h)] if c == R.I420 else data
    return util.convert_cpu(util.oracle(), "orc_convert", c, route, data, w, h)


def check_route(case, res):
    """res: what the reference's filter() did (ref_filter's result, or the fixture's)"""
    cfg, c, w, h = case
    g = lib_geometry(cfg, c, w, h)
    if res is None:
        assert g == -4, f"{case}: the reference drops the frame, the library gives {g}"
        return
    oc, ow, oh, data_len, in_color, iw, ih, handed = res
    assert g != -4, f"{case}: the library finds no route"
    from ultragrid_b200 import vc_get_linesize
    p = R.parse(cfg)[1]
    assert (iw, ih) == (w, h)
    want_out = (R.RG48 if in_color == R.RG48 else R.RGB, int(w * p[1]) if p[0] == R.FRACTION else p[2],
                int(h * p[1]) if p[0] == R.FRACTION else p[3])
    assert (oc, ow, oh) == want_out, case
    assert data_len == vc_get_linesize(ow, oc) * oh
    if c == in_color or w % 48 == 0:
        # elsewhere some line decoders write past the row's length, into the next row, and which of the two writes
        # survives at parallel_pix_conv's task boundaries depends on the host's core count (DESIGN.md §8)
        want = route_bytes(c, in_color, w, h, frame(c, w, h, w * h + c))
        if c == R.I420:  # the Mat ug_to_rgb_mat wraps: h * 3 / 2 rows of w bytes (odd sizes are refused, DESIGN.md §8)
            want = want[:w * (h * 3 // 2)]
        assert np.array_equal(handed, want), f"{case}: bytes handed differ"
    if g == -1:  # odd sizes on 4:2:x routes, or an empty output
        assert (in_color in (R.UYVY, R.YUYV, R.I420) and (w % 2 or (in_color == R.I420 and h % 2))) or ow <= 0 or oh <= 0, case
        return
    route, out_c, gw, gh, rect = g
    assert (int(route), int(out_c), gw, gh) == (in_color, oc, ow, oh), case
    want = R.geometry(p, in_color, w, h)
    assert want is not None and (want[0], want[1], want[2], want[3]) == (oc, ow, oh, rect), case


@pytest.fixture(scope="module")
def ref():
    lib = ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libresize_filter_ref.so not built (reference tree absent)")
    return lib


def test_parse_equals_module(ref):
    for cfg in PARSE_CORPUS:
        assert ref_parse(ref, cfg) == R.parse(cfg), cfg


def test_route_output_and_bytes_equal_module(ref):
    for case in route_cases():
        cfg, c, w, h = case
        check_route(case, ref_filter(ref, cfg, c, w, h, frame(c, w, h, w * h + c)))


def test_route_is_get_best_decoder_from():
    from ultragrid_b200 import compress
    for c in all_codecs():
        g = lib_geometry("1/2", c, 16, 8)
        best = c if c in R.RESIZE_SET else compress.get_best_decoder_from(c, list(R.RESIZE_SET))
        assert (g == -4) == (best == 0), c
        if g != -4:
            assert int(g[0]) == best, c


# ---- golden fixtures ----------------------------------------------------------------------------------------------
def golden_data(ref):
    out = {}
    for i, cfg in enumerate(PARSE_CORPUS):
        rc, p = ref_parse(ref, cfg)
        out[f"parse_{i}"] = np.array([rc] + (list(p) if p else [0, 0, 0, 0, 0]), np.float64)
    for i, case in enumerate(route_cases()):
        cfg, c, w, h = case
        res = ref_filter(ref, cfg, c, w, h, frame(c, w, h, w * h + c))
        out[f"route_{i}"] = np.array([-1] if res is None else res[:7], np.int64)
        if res is not None:
            out[f"route_{i}_bytes"] = res[7]
    return out


def test_parse_equals_golden():
    g = util.golden(GOLDEN)
    for i, cfg in enumerate(PARSE_CORPUS):
        v = g[f"parse_{i}"]
        want = R.parse(cfg)
        assert int(v[0]) == want[0], cfg
        if want[0] == 0:
            assert (int(v[1]), v[2], int(v[3]), int(v[4]), int(v[5])) == want[1], cfg


def test_route_equals_golden():
    g = util.golden(GOLDEN)
    for i, case in enumerate(route_cases()):
        v = g[f"route_{i}"]
        check_route(case, None if v[0] == -1 else tuple(int(x) for x in v) + (g[f"route_{i}_bytes"],))


# ---- letterbox -----------------------------------------------------------------------------------------------------
def test_letterbox_branches():
    dims = (R.DIMENSIONS, 0.0, 1280, 720, 1)
    assert R.geometry(dims, R.UYVY, 1920, 1080)[3] == (0, 0, 1280, 720)  # equal aspect
    g = R.geometry(dims, R.RGB, 1919, 1080)[3]  # narrower: pillarbox
    assert g == (0, 0, 1279, 720) or (g[1] == 0 and g[3] == 720 and g[2] < 1280)
    g = R.geometry(dims, R.RGB, 1920, 1081)[3]  # taller: pillarbox
    assert g[1] == 0 and g[3] == 720 and g[2] < 1280
    g = R.geometry(dims, R.RGB, 1921, 1080)[3]  # wider: letterbox
    assert g[0] == 0 and g[2] == 1280 and g[3] < 720
    g = R.geometry((R.DIMENSIONS, 0.0, 720, 576, 1), R.UYVY, 1920, 1080)[3]
    assert g == (0, (576 - int(720 / (1920 / 1080))) // 2, 720, int(720 / (1920 / 1080)))


def test_letterbox_equals_library():
    from ultragrid_b200 import api
    for (w, h) in ((1920, 1080), (1919, 1080), (1920, 1081), (3840, 2160), (640, 480), (7, 3), (2, 100), (100, 2)):
        for (tw, th) in ((1280, 720), (720, 576), (3840, 2160), (5, 9), (1, 1)):
            r = api.Resize(size=(tw, th))
            want = R.geometry((R.DIMENSIONS, 0.0, tw, th, 1), R.RGB, w, h)
            try:
                got = r.geometry(R.RGB, w, h)
                assert want is not None and (got[2], got[3], got[4]) == (want[1], want[2], want[3]), (w, h, tw, th)
            except RuntimeError as e:
                assert want is None and "code -1" in str(e), (w, h, tw, th)
            r.close()


def test_refusal_codes():
    from ultragrid_b200 import api, Codec
    assert lib_geometry("1/2", int(Codec.UYVY), 17, 8) == -1
    assert lib_geometry("1/2", int(Codec.I420), 16, 9) == -1
    assert lib_geometry("1/4", int(Codec.RGB), 3, 8) == -1
    assert lib_geometry("1/2:algo=cubic", int(Codec.RGB), 16, 8) == -4
    assert lib_geometry("1/2:algo=lanczos4", int(Codec.RGB), 16, 8) == -4
    assert lib_geometry("0.75:algo=area", int(Codec.RGB), 16, 8) == -4
    assert lib_geometry("2:algo=area", int(Codec.RGB), 16, 8) == -4
    assert lib_geometry("1/2", int(Codec.DXT1), 16, 8) == -4
    for args in ((0, 0.5, 0, 0, 1), (1, 0.0, 0, 0, 1), (1, -1.0, 0, 0, 1), (2, 0.0, 0, 5, 1), (1, 0.5, 0, 0, 5), (1, float("inf"), 0, 0, 1)):
        assert not api._L.ugb200_cf_resize_create(*args), args


# ---- the contract, pinned without OpenCV ---------------------------------------------------------------------------
def colour_max_error(coeffs=None):
    """max |colour stage - float64 BT.601 limited range| over all 2^24 (Y, U, V)"""
    kw = {} if coeffs is None else {"coeffs": coeffs}
    U, V = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    worst = 0.0
    for Y in range(256):
        got = R.yuv_to_rgb(np.full_like(U, Y), U, V, **kw).astype(np.float64)
        y = 1.164 * max(0, Y - 16)
        f = np.stack([y + 1.596 * (V - 128), y - 0.813 * (V - 128) - 0.391 * (U - 128), y + 2.018 * (U - 128)], -1)
        worst = max(worst, float(np.abs(got - np.clip(f, 0, 255)).max()))
    return worst


def test_colour_within_one_of_float64():
    assert colour_max_error() <= 1.0


GEOMS = [(96, 64, 0.5), (96, 64, 1 / 3), (96, 64, 0.75), (96, 64, 1.5), (97, 63, 2.0), (33, 17, 0.3), (1920, 1080, 1280 / 1920),
         (7680, 4320, 0.5), (5, 3, 7.0), (2, 2, 0.5)]


def test_linear_coefficients_sum_to_2048(mut=()):
    for w, h, f in GEOMS:
        for n, zero in ((w, True), (h, False)):
            _, _, fr = R.linear_table(n, int(n * f), f, zero)
            a0, a1 = R.q11(fr, "truncated_coefficients" in mut)
            assert (a0 + a1 == 2048).all(), (w, h, f)


def bilinear64(rgb, rw, rh, isx, isy):
    h, w, _ = rgb.shape
    out = np.zeros((rh, rw, 3))

    def taps(n_src, n_dst, inv, zero):
        p = (np.arange(n_dst) + 0.5) / inv - 0.5
        s = np.floor(p).astype(np.int64)
        f = p - s
        if zero:
            f = np.where(s < 0, 0, f)
            s = np.where(s < 0, 0, s)
            f = np.where(s >= n_src - 1, 0, f)
            s = np.where(s >= n_src - 1, n_src - 1, s)
        return np.clip(s, 0, n_src - 1), np.clip(s + 1, 0, n_src - 1), f

    x0, x1, fx = taps(w, rw, isx, True)
    y0, y1, fy = taps(h, rh, isy, False)
    H0 = rgb[y0][:, x0] * (1 - fx)[None, :, None] + rgb[y0][:, x1] * fx[None, :, None]
    H1 = rgb[y1][:, x0] * (1 - fx)[None, :, None] + rgb[y1][:, x1] * fx[None, :, None]
    out = H0 * (1 - fy)[:, None, None] + H1 * fy[:, None, None]
    return out


def test_linear_within_one_of_float64_bilinear(mut=()):
    for i, (w, h, f) in enumerate(GEOMS[:7]):
        rgb = util.rng_bytes(w * h * 3, 100 + i).reshape(h, w, 3).astype(np.int32)
        rw, rh = int(w * f), int(h * f)
        got = R.resample(rgb, rw, rh, f, f, 1, False, mut)
        assert np.abs(got - bilinear64(rgb.astype(np.float64), rw, rh, f, f)).max() <= 1.0, (w, h, f)


def _rand(route, w, h, seed):
    from ultragrid_b200 import vc_get_linesize
    n = R.frame_len(route, w, h) if route == R.I420 else vc_get_linesize(w, route) * h
    return util.rng_bytes(n, seed)


def test_identity_at_scale_one():
    for route in R.RESIZE_SET:
        for algo in (0, 1, 3):
            d = _rand(route, 34, 18, route)
            rc, out = R.resize((R.FRACTION, 1.0, 0, 0, algo), route, d, 34, 18)
            assert rc == 0 and np.array_equal(out.reshape(18, 34, -1), _as_out(R.to_rgb(route, d, 34, 18), route == R.RG48)), (route, algo)


def _as_out(rgb, w16):
    return rgb.astype("<u2").view(np.uint8) if w16 else rgb.astype(np.uint8)


def test_constant_frame_stays_constant():
    rgb = np.full(60 * 40 * 3, 77, np.uint8)
    for f in (0.5, 1 / 3, 0.75, 1.5, 2.0, 0.3):
        for algo in (0, 1, 3):
            rc, out = R.resize((R.FRACTION, f, 0, 0, algo), R.RGB, rgb, 60, 40)
            assert rc == -4 or (rc == 0 and (out == 77).all()), (f, algo)


def test_linear_half_equals_area_2x2(mut=()):
    for route in (R.RGB, R.UYVY, R.I420, R.RGBA):
        for w, h in ((64, 32), (66, 34), (7680 // 8, 4320 // 8)):
            d = _rand(route, w, h, w + route)
            lin = R.resize((R.FRACTION, 0.5, 0, 0, 1), route, d, w, h, mut)
            area = R.resize((R.FRACTION, 0.5, 0, 0, 3), route, d, w, h, mut)
            assert np.array_equal(lin[1], area[1]), (route, w, h)


MUTANTS = {
    "no_rounding_term": test_linear_half_equals_area_2x2,
    "align_corners": test_linear_half_equals_area_2x2,
    "half_even_area": test_linear_half_equals_area_2x2,
    "truncated_coefficients": test_linear_coefficients_sum_to_2048,
}


@pytest.mark.parametrize("name", list(MUTANTS) + ["bt709"])
def test_mutants_fail(name):
    if name == "bt709":
        assert colour_max_error(R.BT709) > 1.0
        return
    with pytest.raises(AssertionError):
        MUTANTS[name](mut=(name,))


# ---- GPU -----------------------------------------------------------------------------------------------------------
def want_for(param, c, w, h, data):
    """the restatement's (code, bytes) for a frame of codec c"""
    from ultragrid_b200 import compress
    route = c if c in R.RESIZE_SET else compress.get_best_decoder_from(c, list(R.RESIZE_SET))
    return R.resize(param, route, route_bytes(c, route, w, h, data), w, h)


def gpu_check(param, c, w, h, seed=1, handle=None, stream=None):
    import torch
    from ultragrid_b200 import api
    mode, factor, tw, th, algo = param
    data = frame(c, w, h, seed)
    rc, want = want_for(param, c, w, h, data)
    r = handle or (api.Resize(factor=factor, algo=algo) if mode == R.FRACTION else api.Resize(size=(tw, th), algo=algo))
    n = want.size if rc == 0 else 64
    g = util.Guarded(n)
    if rc != 0:
        with pytest.raises(RuntimeError, match=f"code {rc}"):
            r(util.dev(data), c, w, h, dst=g.view, stream=stream)
        torch.cuda.synchronize()
        assert (g.check_outside() == g.fill).all(), "a refusal wrote"
    else:
        r(util.dev(data), c, w, h, dst=g.view, stream=stream)
        torch.cuda.synchronize()
        got = g.check_outside()
        assert np.array_equal(got, want), f"{param} codec {c} {w}x{h}: {int(np.count_nonzero(got != want))} bytes differ"
    if handle is None:
        r.close()
    return rc


FACTORS = [1.0, 0.5, 1 / 3, 0.25, 0.75, 1.5, 2.0]


@pytest.mark.gpu
@pytest.mark.parametrize("codec", R.RESIZE_SET)
@pytest.mark.parametrize("algo", [0, 1, 3])
def test_gpu_native_layouts_factors(codec, algo):
    sizes = [(96, 48), (2, 2), (98, 26)] + ([(97, 31), (1, 1), (35, 9)] if codec in (R.RGB, R.RGBA, R.RG48) else [(36, 8)])
    codes = []
    for w, h in sizes:
        for f in FACTORS:
            codes.append(gpu_check((R.FRACTION, f, 0, 0, algo), codec, w, h, seed=w + h + codec))
    assert codes.count(0) >= len(codes) // 3


@pytest.mark.gpu
@pytest.mark.parametrize("codec", R.RESIZE_SET)
def test_gpu_dimension_targets(codec):
    for algo in (0, 1, 3):
        for (w, h), (tw, th) in (((96, 54), (64, 36)), ((96, 54), (40, 40)), ((96, 54), (100, 30)), ((64, 48), (32, 24)),
                                 ((98, 54), (64, 36)), ((64, 36), (160, 90))):
            gpu_check((R.DIMENSIONS, 0.0, tw, th, algo), codec, w, h, seed=w * tw + algo)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v210", "R10k", "R12L", "Y416", "Y216", "BGR", "VUYA", "DVS10"])
def test_gpu_routed_codecs(name):
    from ultragrid_b200 import Codec
    c = int(Codec[name])
    for param in ((R.FRACTION, 0.5, 0, 0, 1), (R.FRACTION, 0.75, 0, 0, 0), (R.FRACTION, 0.5, 0, 0, 3), (R.DIMENSIONS, 0.0, 64, 64, 1)):
        assert gpu_check(param, c, 96, 54, seed=c) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v210", "R10k", "R12L", "Y416", "Y216", "BGR", "VUYA", "DVS10"])
def test_gpu_routed_codecs_at_spilling_widths(name):
    """widths where the route's line converter writes whole groups past the row on the staging frame's last row
    (v210 / DVS10: not a multiple of 6; R12L: not a multiple of 8; R10k, Y216: odd)"""
    from ultragrid_b200 import Codec, compress
    c = int(Codec[name])
    route = compress.get_best_decoder_from(c, list(R.RESIZE_SET))
    for w, h in ((50, 7), (64, 4), (1919, 5), (1366, 3), (94, 2), (13, 9)):
        for param in ((R.FRACTION, 0.5, 0, 0, 1), (R.DIMENSIONS, 0.0, 40, 40, 0)):
            rc = gpu_check(param, c, w, h, seed=w + c)  # == the restatement, refusals included
            # refused only for an odd width on a 4:2:2 route, or a letterbox rectangle of height 0 (1919 x 5 into 40 x 40)
            assert rc == 0 or (rc == -1 and R.geometry(param, route, w, h) is None), (name, w, h, rc)
            assert rc == 0 or param[0] == R.DIMENSIONS or (w % 2 and route in (R.UYVY, R.YUYV)), (name, w, h, rc)


@pytest.mark.gpu
@pytest.mark.parametrize("codec", [R.RGB, R.RG48, R.UYVY])
def test_gpu_area_boxes_of_65536_taps_and_more(codec):
    """boxes of kx * ky >= 65536 taps, whose sums take the 64-bit path"""
    for w, h, f in ((512, 512, 1 / 256), (1024, 300, 1 / 300), (600, 600, 1 / 300)):
        assert gpu_check((R.FRACTION, f, 0, 0, 3), codec, w, h, seed=w + codec) in (0, -4)
    assert gpu_check((R.FRACTION, 1 / 256, 0, 0, 3), codec, 512, 512, seed=codec) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,param", [(7680, 4320, (R.FRACTION, 0.5, 0, 0, 1)), (3840, 2160, (R.DIMENSIONS, 0.0, 1920, 1080, 3)),
                                       (3840, 2160, (R.DIMENSIONS, 0.0, 1280, 720, 1))])
def test_gpu_8k_4k(w, h, param):
    assert gpu_check(param, R.UYVY, w, h, seed=7) == 0


@pytest.mark.gpu
def test_gpu_one_handle_across_descriptors_and_side_stream():
    import torch
    from ultragrid_b200 import api, Codec
    r = api.Resize(factor=0.5)
    s = torch.cuda.Stream()
    seq = [(R.UYVY, 64, 32), (int(Codec.v210), 96, 54), (R.RGB, 33, 17), (R.RG48, 20, 10), (R.UYVY, 64, 32), (int(Codec.v210), 96, 54)]
    for i, (c, w, h) in enumerate(seq):
        assert gpu_check((R.FRACTION, 0.5, 0, 0, -1), c, w, h, seed=i, handle=r, stream=s if i % 2 else None) == 0
    r.close()


@pytest.mark.gpu
def test_gpu_refusals_write_nothing():
    import torch
    from ultragrid_b200 import api, Codec
    cases = [((R.FRACTION, 0.5, 0, 0, 1), R.UYVY, 17, 8), ((R.FRACTION, 0.5, 0, 0, 1), R.I420, 16, 9),
             ((R.FRACTION, 0.25, 0, 0, 1), R.RGB, 3, 8), ((R.FRACTION, 0.5, 0, 0, 2), R.RGB, 16, 8),
             ((R.FRACTION, 0.5, 0, 0, 4), R.RGB, 16, 8), ((R.FRACTION, 0.75, 0, 0, 3), R.RGB, 16, 8),
             ((R.FRACTION, 2.0, 0, 0, 3), R.RGB, 16, 8)]
    for param, c, w, h in cases:
        assert gpu_check(param, c, w, h) != 0
    r = api.Resize(factor=0.5)
    g = util.Guarded(64)
    with pytest.raises(RuntimeError, match="code -4"):  # no route
        r(util.dev(np.zeros(64, np.uint8)), Codec.DXT1, 16, 8, dst=g.view)
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="code -1"):  # dst overlapping src
        r(buf[:16 * 8 * 3], Codec.RGB, 16, 8, dst=buf[100:100 + 8 * 4 * 3])
    torch.cuda.synchronize()
    assert (g.check_outside() == g.fill).all() and (buf.cpu().numpy() == 0).all()
    r.close()
