"""numpy restatement of the resize algorithms that ugb200_cf_resize_create2 handles add (DESIGN.md §2 "Resize"): cubic,
lanczos4, area at ratios that are not integer downscales, and area upscaling.  Parse, route, geometry, colour and the
algorithms built by every handle come from resize_filter_ref; the tables here are computed in numpy, float32 in the
contract's order, int64 for the 8-bit sums, and the C library's sin and cos through ctypes.
"""
import ctypes
import math

import numpy as np

import resize_filter_ref as R

CUBIC, AREA, LANCZOS4 = 2, 3, 4
F32 = np.float32

_libc = ctypes.CDLL(None)
_libc.sin.restype, _libc.sin.argtypes = ctypes.c_double, [ctypes.c_double]
_libc.cos.restype, _libc.cos.argtypes = ctypes.c_double, [ctypes.c_double]
S45 = 0.70710678118654752440084436210485
CS = ((1, 0), (-S45, -S45), (0, 1), (S45, -S45), (-1, 0), (S45, S45), (0, -1), (-S45, S45))


# ---- weights -------------------------------------------------------------------------------------------------------
def cubic_weights(f, A=-0.75):
    """interpolateCubic: (4,) float32 for one float32 fraction, each step one float32 operation"""
    x, A = F32(f), F32(A)
    one = F32(1)
    x1 = x + one
    c0 = ((A * x1 - F32(5) * A) * x1 + F32(8) * A) * x1 - F32(4) * A
    c1 = ((A + F32(2)) * x - (A + F32(3))) * x * x + one
    y = one - x
    c2 = ((A + F32(2)) * y - (A + F32(3))) * y * y + one
    c3 = one - c0 - c1 - c2
    return np.array([c0, c1, c2, c3], F32)


def lanczos4_weights(f, normalise=True):
    """interpolateLanczos4: (8,) float32 for one float32 fraction"""
    x3 = F32(f) + F32(3)
    y0 = float(-x3) * math.pi * 0.25
    s0, c0 = _libc.sin(y0), _libc.cos(y0)
    w = np.zeros(8, F32)
    for i in range(8):
        t = x3 - F32(i)
        if abs(t) >= F32(1e-6):
            y = float(-t) * math.pi * 0.25
            w[i] = F32((CS[i][0] * s0 + CS[i][1] * c0) / (y * y))
        else:
            w[i] = F32(1e30)
    if not normalise:
        return w
    s = F32(0)
    for i in range(8):
        s = F32(s + w[i])
    inv = F32(1) / s
    return (w * inv).astype(F32)


def q11(w):
    """saturate_cast<short>(w * 2048.0f): the product in float32, round half to even, saturated"""
    return np.clip(np.rint((np.asarray(w, F32) * F32(2048)).astype(F32)), -32768, 32767).astype(np.int64)


def fractions(n_dst, inv_scale):
    """(sx, f): f = (float) ((d + 0.5) * scale - 0.5), sx = floor(f), f -= sx (float)"""
    scale = 1.0 / inv_scale
    f = ((np.arange(n_dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    return s, (f - s.astype(F32)).astype(F32)


def multitap_table(n_dst, inv_scale, algo, mut=()):
    """(first, w): first tap sx - K / 2 + 1 (unclamped) and (n_dst, K) float32 weights"""
    s, f = fractions(n_dst, inv_scale)
    if algo == CUBIC:
        A = -0.5 if "cubic_a_half" in mut else -0.75
        w = np.array([cubic_weights(x, A) for x in f], F32).reshape(-1, 4)
    else:
        w = np.array([lanczos4_weights(x, "lanczos_unnormalised" not in mut) for x in f], F32).reshape(-1, 8)
    K = w.shape[1]
    return s - K // 2 + 1, w


def taps(first, K, n_src):
    """(n_dst, K) clamped source indices"""
    return np.clip(first[:, None] + np.arange(K)[None, :], 0, n_src - 1)


def area_tab(n_src, n_dst, scale, mut=()):
    """computeResizeAreaTab: a list per destination of (source index, float32 alpha), in order"""
    out = []
    for d in range(n_dst):
        fs1 = d * scale
        fs2 = fs1 + scale
        cw = min(scale, n_src - fs1)
        s1, s2 = math.ceil(fs1), math.floor(fs2)
        s2 = min(s2, n_src - 1)
        s1 = min(s1, s2)
        e = []
        if s1 - fs1 > 1e-3 and "area_no_partial" not in mut:
            e.append((s1 - 1, F32((s1 - fs1) / cw)))
        for s in range(s1, s2):
            e.append((s, F32(1.0 / cw)))
        if fs2 - s2 > 1e-3 and "area_no_partial" not in mut:
            e.append((s2, F32(min(min(fs2 - s2, 1.0), cw) / cw)))
        out.append(e)
    return out


def linear_area_table(n_src, n_dst, inv_scale, zero_frac):
    """(s0, s1, f) with area-mode positions: s = floor(d * scale), f = (float) ((d + 1) - (s + 1) * inv_scale),
    f = f <= 0 ? 0 : f - floor(f); columns set s = n - 1, f = 0 where s >= n - 1, rows clamp s, s + 1"""
    scale = 1.0 / inv_scale
    d = np.arange(n_dst, dtype=np.float64)
    s = np.floor(d * scale).astype(np.int64)
    f = ((d + 1) - (s + 1) * inv_scale).astype(F32)
    f = np.where(f <= 0, F32(0), (f - np.floor(f)).astype(F32)).astype(F32)
    if zero_frac:
        hi = s >= n_src - 1
        s = np.where(hi, n_src - 1, s)
        f = np.where(hi, F32(0), f)
        return s, np.minimum(s + 1, n_src - 1), f
    return np.clip(s, 0, n_src - 1), np.clip(s + 1, 0, n_src - 1), f


# ---- resampling ----------------------------------------------------------------------------------------------------
def area_mode(w, h, rw, rh, isx, isy):
    """'int' (integer downscale, resize_filter_ref's area), 'any' (both scales >= 1) or 'up'"""
    if R.area_factor(w, rw, isx) and R.area_factor(h, rh, isy):
        return "int"
    return "any" if 1.0 / isx >= 1 and 1.0 / isy >= 1 else "up"


def multitap(rgb, rw, rh, isx, isy, algo, w16, mut=()):
    h, w, _ = rgb.shape
    fx, ax = multitap_table(rw, isx, algo, mut)
    fy, ay = multitap_table(rh, isy, algo, mut)
    K = ax.shape[1]
    tx, ty = taps(fx, K, w), taps(fy, K, h)
    if w16:
        S = rgb.astype(F32)
        H = None
        for j in range(K):
            p = (S[:, tx[:, j]] * ax[None, :, j, None]).astype(F32)
            H = p if H is None else (H + p).astype(F32)
        V = None
        for k in range(K):
            p = (H[ty[:, k]] * ay[:, k, None, None]).astype(F32)
            V = p if V is None else (V + p).astype(F32)
        return np.clip(np.rint(V), 0, 65535).astype(np.int64)
    a, b = q11(ax), q11(ay)
    H = np.zeros((h, rw, 3), np.int64)
    for j in range(K):
        H += rgb[:, tx[:, j]].astype(np.int64) * a[None, :, j, None]
    V = np.zeros((rh, rw, 3), np.int64)
    for k in range(K):
        V += H[ty[:, k]] * b[:, k, None, None]
    if "wrap32" in mut:
        V = (V + 2 ** 31) % 2 ** 32 - 2 ** 31
    return np.clip((V + (1 << 21)) >> 22, 0, 255)


def _padded(tab):
    """(idx, alpha) (n, m) arrays, each row padded to the longest with (0, 0): the padding adds exact zeros at the end"""
    m = max(len(e) for e in tab)
    idx, al = np.zeros((len(tab), m), np.int64), np.zeros((len(tab), m), F32)
    for d, e in enumerate(tab):
        for i, (s, a) in enumerate(e):
            idx[d, i], al[d, i] = s, a
    return idx, al


def area_any(rgb, rw, rh, isx, isy, w16, mut=()):
    h, w, _ = rgb.shape
    xi, xa = _padded(area_tab(w, rw, 1.0 / isx, mut))
    yi, ya = _padded(area_tab(h, rh, 1.0 / isy, mut))
    S = rgb.astype(F32)
    buf = np.zeros((h, rw, 3), F32)  # buf of every source row
    for i in range(xi.shape[1]):
        buf = (buf + (S[:, xi[:, i]] * xa[None, :, i, None]).astype(F32)).astype(F32)
    s = (buf[yi[:, 0]] * ya[:, 0, None, None]).astype(F32)
    for j in range(1, yi.shape[1]):
        s = (s + (buf[yi[:, j]] * ya[:, j, None, None]).astype(F32)).astype(F32)
    return np.clip(np.rint(s), 0, 65535 if w16 else 255).astype(np.int64)


def area_up(rgb, rw, rh, isx, isy, w16, mut=()):
    h, w, _ = rgb.shape
    if "area_up_as_linear" in mut:
        sx0, sx1, fx = R.linear_table(w, rw, isx, True)
        sy0, sy1, fy = R.linear_table(h, rh, isy, False)
    else:
        sx0, sx1, fx = linear_area_table(w, rw, isx, True)
        sy0, sy1, fy = linear_area_table(h, rh, isy, False)
    if w16:
        a0, a1 = (F32(1.0) - fx).astype(F32), fx
        b0, b1 = (F32(1.0) - fy).astype(F32), fy
        S = rgb.astype(F32)
        H0 = (S[sy0][:, sx0] * a0[None, :, None] + S[sy0][:, sx1] * a1[None, :, None]).astype(F32)
        H1 = (S[sy1][:, sx0] * a0[None, :, None] + S[sy1][:, sx1] * a1[None, :, None]).astype(F32)
        V = (H0 * b0[:, None, None] + H1 * b1[:, None, None]).astype(F32)
        return np.clip(np.rint(V), 0, 65535).astype(np.int64)
    a0, a1 = R.q11(fx)
    b0, b1 = R.q11(fy)
    H0 = rgb[sy0][:, sx0] * a0[None, :, None] + rgb[sy0][:, sx1] * a1[None, :, None]
    H1 = rgb[sy1][:, sx0] * a0[None, :, None] + rgb[sy1][:, sx1] * a1[None, :, None]
    return np.clip((H0 * b0[:, None, None] + H1 * b1[:, None, None] + (1 << 21)) >> 22, 0, 255)


def resample(rgb, rw, rh, isx, isy, algo, w16, mut=()):
    """(rh, rw, 3) ints: every algorithm, as a ugb200_cf_resize_create2 handle resamples"""
    h, w, _ = rgb.shape
    if algo in (CUBIC, LANCZOS4):
        return multitap(rgb, rw, rh, isx, isy, algo, w16, mut)
    if algo == AREA:
        m = area_mode(w, h, rw, rh, isx, isy)
        if m == "any":
            return area_any(rgb, rw, rh, isx, isy, w16, mut)
        if m == "up":
            return area_up(rgb, rw, rh, isx, isy, w16, mut)
    return R.resample(rgb, rw, rh, isx, isy, algo, w16)


def resize(param, route, data, w, h, mut=()):
    """ugb200_cf_resize on a ugb200_cf_resize_create2 handle, frame already in the route codec: (code, bytes)"""
    g = R.geometry(param, route, w, h)
    if g is None:
        return -1, None
    out_c, ow, oh, (rx, ry, rw, rh), isx, isy = g
    algo = 1 if param[4] == R.DFL else param[4]
    w16 = route == R.RG48
    r = resample(R.to_rgb(route, data, w, h), rw, rh, isx, isy, algo, w16, mut)
    out = np.zeros((oh, ow, 3), np.int64)
    out[ry:ry + rh, rx:rx + rw] = r
    return 0, (out.astype("<u2").view(np.uint8) if w16 else out.astype(np.uint8)).reshape(-1)
