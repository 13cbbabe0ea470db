"""numpy restatement of the resize filter (src/capture_filter/resize.c) and of the resampling contract of DESIGN.md §2
"Resize" (ugb200_cf_resize).  Independent of the device code: parse, route, geometry and letterbox are restated from
resize.c and resize_utils.cpp, and the tables are computed here in numpy.

Frames are flat uint8 arrays; RGB results are (h, w, 3) int arrays (0-255, or 0-65535 for RG48).
"""
import ctypes
import math
import sys

import numpy as np

RGBA, UYVY, YUYV, RGB, RG48, I420 = 1, 2, 3, 12, 27, 29
RESIZE_SET = (RGB, RGBA, I420, UYVY, YUYV, RG48)  # RESIZE_SUPPORTED_PIXFMT_INIT
ALGOS = {"nearest": 0, "linear": 1, "cubic": 2, "area": 3, "lanczos4": 4}
DFL, UNKN, HELP = -1, -2, -3
FRACTION, DIMENSIONS = 1, 2
DBL_EPSILON = sys.float_info.epsilon

_libc = ctypes.CDLL(None)
_libc.strtod.restype, _libc.strtod.argtypes = ctypes.c_double, [ctypes.c_char_p, ctypes.c_void_p]
_libc.strtol.restype, _libc.strtol.argtypes = ctypes.c_long, [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_int]


def _c_int(v):
    """a long stored into an int field (two's complement truncation)"""
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


# ---- init / parse_fmt (resize.c:107-164) -----------------------------------------------------------------------
def parse(cfg):
    """(rc, param): rc as init() returns it (0, 1 = help shown, -1); param = (mode, factor, tw, th, algo) on 0"""
    if cfg.lower() == "help":
        return 1, None
    mode, factor, tw, th, algo = 0, 0.0, 0, 0, DFL
    for item in [t for t in cfg.split(":") if t]:  # strtok_r skips empty tokens
        if "=" in item and "algorithm".startswith(item[:item.index("=")]):  # IS_KEY_PREFIX
            name = item[item.index("=") + 1:]
            algo = HELP if name == "help" else ALGOS.get(name, UNKN)
            if algo < 0:
                return (1 if algo == HELP else -1), None
            continue
        if not (item[0].isdigit() or item[0] == "."):
            return -1, None
        b = item.encode()
        if "x" in item:
            mode = DIMENSIONS
            tw = _c_int(_libc.strtol(b, None, 10))
            th = _c_int(_libc.strtol(item[item.index("x") + 1:].encode(), None, 10))
        else:
            mode = FRACTION
            factor = _libc.strtod(b, None)
            if "/" in item:
                den = _libc.strtol(item[item.index("/") + 1:].encode(), None, 10)
                factor = 0.0 if den <= 0 else factor / den
    if mode == DIMENSIONS and tw > 0 and th > 0:
        return 0, (mode, 0.0, tw, th, algo)
    if mode == FRACTION and factor > 0:
        return 0, (mode, factor, 0, 0, algo)
    return -1, None


# ---- geometry (resize.c:181-220, resize_utils.cpp:141-173) ---------------------------------------------------------
def geometry(param, route, w, h):
    """None (refused: -1) or (out codec, out_w, out_h, (rx, ry, rw, rh), inv_scale_x, inv_scale_y)"""
    mode, factor, tw, th, _ = param
    out_c = RG48 if route == RG48 else RGB
    if mode == DIMENSIONS:
        ow, oh = tw, th
        in_aspect, out_aspect = w / h, tw / th
        rx, ry, rw, rh = 0, 0, tw, th
        if in_aspect == out_aspect:
            pass
        elif in_aspect > out_aspect:
            rh = int(tw / in_aspect)
            ry = (th - rh) // 2  # non-negative operands: C division
        else:
            rw = int(th * in_aspect)
            rx = (tw - rw) // 2
        isx, isy = rw / w, rh / h
    else:
        ow, oh = int(w * factor), int(h * factor)
        rx, ry, rw, rh = 0, 0, ow, oh
        isx = isy = factor
    if ow <= 0 or oh <= 0 or rw <= 0 or rh <= 0:
        return None
    if (route in (UYVY, YUYV, I420) and w % 2) or (route == I420 and h % 2):
        return None
    return out_c, ow, oh, (rx, ry, rw, rh), isx, isy


def out_linesize(out_c, ow):
    return ow * (6 if out_c == RG48 else 3)


def frame_len(route, w, h):
    return {RGB: 3 * w * h, RGBA: 4 * w * h, UYVY: 2 * w * h, YUYV: 2 * w * h, RG48: 6 * w * h, I420: w * h * 3 // 2}[route]


# ---- colour stage (cvtColor) ---------------------------------------------------------------------------------
CY, CVR, CVG, CUG, CUB = 1220542, 1673527, -852492, -409993, 2116026  # round(2^20 * {1.164, 1.596, -0.813, -0.391, 2.018})


def yuv_to_rgb(Y, U, V, coeffs=(CY, CVR, CVG, CUG, CUB)):
    cy, cvr, cvg, cug, cub = coeffs
    Y, U, V = (np.asarray(a, np.int32) for a in (Y, U, V))  # |Yq + 1673527 v + 2^19| < 2^31
    yq = np.maximum(0, Y - 16) * cy
    u, v = U - 128, V - 128
    r = (yq + cvr * v + (1 << 19)) >> 20
    g = (yq + cvg * v + cug * u + (1 << 19)) >> 20
    b = (yq + cub * u + (1 << 19)) >> 20
    return np.clip(np.stack([r, g, b], -1), 0, 255)


def to_rgb(route, data, w, h, **kw):
    """(h, w, 3) int32: the frame as RGB, every pixel converted"""
    d = np.asarray(data, np.uint8)
    if route == RGB:
        return d[:3 * w * h].reshape(h, w, 3).astype(np.int32)
    if route == RGBA:
        return d[:4 * w * h].reshape(h, w, 4)[:, :, :3].astype(np.int32)
    if route == RG48:
        return d[:6 * w * h].view("<u2").reshape(h, w, 3).astype(np.int32)
    if route in (UYVY, YUYV):
        g = d[:2 * w * h].reshape(h, w // 2, 4).astype(np.int32)
        if route == UYVY:
            U, Y0, V, Y1 = (g[:, :, i] for i in range(4))
        else:
            Y0, U, Y1, V = (g[:, :, i] for i in range(4))
        Y = np.stack([Y0, Y1], -1).reshape(h, w)
        return yuv_to_rgb(Y, np.repeat(U, 2, 1), np.repeat(V, 2, 1), **kw)
    Y = d[:w * h].reshape(h, w)
    U = d[w * h:w * h + (w // 2) * (h // 2)].reshape(h // 2, w // 2)
    V = d[w * h + (w // 2) * (h // 2):w * h * 3 // 2].reshape(h // 2, w // 2)
    up = lambda p: np.repeat(np.repeat(p, 2, 0), 2, 1)  # noqa: E731
    return yuv_to_rgb(Y, up(U), up(V), **kw)


# ---- tables ------------------------------------------------------------------------------------------------------
def nearest_index(n_src, n_dst, inv_scale):
    ifs = 1.0 / inv_scale
    return np.minimum(np.floor(np.arange(n_dst) * ifs).astype(np.int64), n_src - 1)


def linear_table(n_src, n_dst, inv_scale, zero_frac, align_corners=False):
    """(s0, s1, f): positions and float32 fractions (DESIGN.md §2 "Resize")"""
    scale = 1.0 / inv_scale
    d = np.arange(n_dst, dtype=np.float64)
    if align_corners:  # mutant: maps corners to corners
        f = (d * ((n_src - 1) / max(n_dst - 1, 1))).astype(np.float32)
    else:
        f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if zero_frac:
        lo = s < 0
        s = np.where(lo, 0, s)
        f = np.where(lo, np.float32(0), f)
        hi = s >= n_src - 1
        s = np.where(hi, n_src - 1, s)
        f = np.where(hi, np.float32(0), f)
        s1 = np.minimum(s + 1, n_src - 1)
    else:
        s1 = np.clip(s + 1, 0, n_src - 1)
        s = np.clip(s, 0, n_src - 1)
    return s, s1, f.astype(np.float32)


def q11(f, truncate=False):
    """cvRound((1.0f - f) * 2048), cvRound(f * 2048), the products in float32 (np.rint: ties to even)"""
    one = (np.float32(1.0) - f).astype(np.float32) * np.float32(2048)
    two = f.astype(np.float32) * np.float32(2048)
    r = np.trunc if truncate else np.rint
    return r(one).astype(np.int32), r(two).astype(np.int32)  # b0 H0 + b1 H1 + 2^21 < 2^31


def area_factor(n_src, n_dst, inv_scale):
    scale = 1.0 / inv_scale
    k = int(math.floor(scale + 0.5))  # round(): the scales where it matters are within DBL_EPSILON of an integer
    return k if k >= 1 and abs(scale - k) < DBL_EPSILON and n_dst * k <= n_src else 0


# ---- resampling --------------------------------------------------------------------------------------------------
def resample(rgb, rw, rh, isx, isy, algo, w16, mut=()):
    """(rh, rw, 3) ints from (h, w, 3), or None where the algorithm is not built (-4)"""
    h, w, _ = rgb.shape
    if algo == 0:
        return rgb[nearest_index(h, rh, isy)][:, nearest_index(w, rw, isx)]
    if algo == 1:
        ac = "align_corners" in mut
        sx0, sx1, fx = linear_table(w, rw, isx, True, ac)
        sy0, sy1, fy = linear_table(h, rh, isy, False, ac)
        if w16:
            a0, a1 = (np.float32(1.0) - fx).astype(np.float32), fx
            b0, b1 = (np.float32(1.0) - fy).astype(np.float32), fy
            S = rgb.astype(np.float32)
            H0 = (S[sy0][:, sx0] * a0[None, :, None] + S[sy0][:, sx1] * a1[None, :, None]).astype(np.float32)
            H1 = (S[sy1][:, sx0] * a0[None, :, None] + S[sy1][:, sx1] * a1[None, :, None]).astype(np.float32)
            V = (H0 * b0[:, None, None] + H1 * b1[:, None, None]).astype(np.float32)
            return np.clip(np.rint(V), 0, 65535).astype(np.int32)
        tr = "truncated_coefficients" in mut
        a0, a1 = q11(fx, tr)
        b0, b1 = q11(fy, tr)
        H0 = rgb[sy0][:, sx0] * a0[None, :, None] + rgb[sy0][:, sx1] * a1[None, :, None]
        H1 = rgb[sy1][:, sx0] * a0[None, :, None] + rgb[sy1][:, sx1] * a1[None, :, None]
        rnd = 0 if "no_rounding_term" in mut else 1 << 21
        return np.clip((H0 * b0[:, None, None] + H1 * b1[:, None, None] + rnd) >> 22, 0, 255)
    if algo == 3:
        kx, ky = area_factor(w, rw, isx), area_factor(h, rh, isy)
        if not kx or not ky:
            return None
        s = rgb[:rh * ky, :rw * kx].reshape(rh, ky, rw, kx, 3).sum(axis=(1, 3), dtype=np.int64)
        n = kx * ky
        if "half_even_area" in mut:
            return np.rint(s / n).astype(np.int64)
        return (s + n // 2) // n
    return None


def resize(param, route, data, w, h, mut=()):
    """ugb200_cf_resize on a frame already in the route codec: (code, bytes).  code 0 with the output frame's bytes,
    or -1 / -4 with None"""
    g = geometry(param, route, w, h)
    if g is None:
        return -1, None
    out_c, ow, oh, (rx, ry, rw, rh), isx, isy = g
    algo = 1 if param[4] == DFL else param[4]
    w16 = route == RG48
    r = resample(to_rgb(route, data, w, h, **({"coeffs": BT709} if "bt709" in mut else {})), rw, rh, isx, isy, algo, w16, mut)
    if r is None:
        return -4, None
    out = np.zeros((oh, ow, 3), np.int32)
    out[ry:ry + rh, rx:rx + rw] = r
    return 0, (out.astype("<u2").view(np.uint8) if w16 else out.astype(np.uint8)).reshape(-1)


# mutant colour: BT.709 limited range in the same Q20 form
BT709 = tuple(int(round(c * 2 ** 20)) for c in (1.164, 1.793, -0.534, -0.213, 2.115))
