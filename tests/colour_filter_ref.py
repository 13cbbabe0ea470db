"""numpy restatement of UltraGrid's colour capture filters, quirks included.

  gamma      src/capture_filter/gamma.cpp:71-91 (the four tables), :96-136 (apply_lut)
  matrix     src/capture_filter/matrix.c:137-287 (filter)
  matrix2    src/capture_filter/matrix2.c:162-231 (apply_to_uyvy, convert_apply_y416), with the line converters
             vc_copylineV210toY416 / vc_copylineY416toV210 (src/pixfmt_conv.c:2834-2882, 3004-3031)
  grayscale  src/capture_filter/grayscale.c:86-90

Each function maps a flat input stream to the flat output stream over the whole length the reference loops over:
matrix on UYVY returns 6 bytes per 4 of the frame (3 * h bytes more than an RGB frame at odd widths), gamma every
sample, matrix2 on v210 every 16-byte group of the frame as a function of the same input group.  Which of those bytes
the reference leaves unwritten or indeterminate, and where ugb200_cf_* stop, is for the caller (DESIGN.md §8).

Every double -> integer conversion is x86's cvttsd2si into 32 bits (x86_i32), then the low 8 or 16 bits; sums are
float64 left to right, one numpy operation each, so none is fused.
"""
import ctypes
import ctypes.util

import numpy as np

UYVY, v210, RGB, RG48, Y416 = 2, 7, 12, 27, 31
Y601_TO_Y709 = (1, -0.11555, -0.207938, 0, 1.01864, 0.114618, 0, 0.075049, 1.025327)  # matrix2.c:66-70
INT_MIN = -(1 << 31)


def x86_i32(v, saturate=False):
    """cvttsd2si with a 32-bit destination: truncation toward zero; NaN and values outside int32 give INT_MIN.
    saturate=True is the mutant that clamps to the int32 range instead (__double2int_rz)"""
    v = np.asarray(v, np.float64)
    ok = (v > -2147483649.0) & (v < 2147483648.0)
    t = np.trunc(np.where(ok, v, 0.0)).astype(np.int64)
    if saturate:
        return np.where(ok, t, np.where(v > 0, (1 << 31) - 1, np.where(np.isnan(v), 0, INT_MIN)))
    return np.where(ok, t, INT_MIN)


def _dot(m, r, a0, a1, a2, off=None, fma=False):
    """(m[r] a0 + m[r+1] a1) + m[r+2] a2, or ((off + m[r] a0) + ...) for matrix2; fma=True is the mutant whose last
    step is one fused multiply-add (exact, through fractions)"""
    with np.errstate(invalid="ignore", over="ignore"):  # inf * 0 and 1e300 * 1e300 are part of the contract
        p0, p1 = m[r] * a0, m[r + 1] * a1
        s = p0 + p1 if off is None else (off + p0) + p1
        if not fma:
            return s + m[r + 2] * a2
    return _fma(np.broadcast_to(m[r + 2], np.shape(s)), np.broadcast_to(a2, np.shape(s)), s)


def _fma(a, b, c):
    from fractions import Fraction
    out = np.empty(np.shape(c), np.float64)
    for i, (x, y, z) in enumerate(zip(np.ravel(a), np.ravel(b), np.ravel(c))):
        if np.isfinite(x) and np.isfinite(y) and np.isfinite(z):
            out.flat[i] = float(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
        else:
            out.flat[i] = x * y + z
    return out


def _conv(v, bits, bound=False, saturate=False, clamp_max=255):
    i = x86_i32(v, saturate)
    if bound:
        i = np.clip(i, 0, clamp_max)
    return (i & ((1 << bits) - 1)).astype(np.uint8 if bits == 8 else np.uint16)


# ---- matrix ----------------------------------------------------------------------------------------------------
def matrix(codec, src, m, check_bounds=True, saturate=False, fma=False, rg48_max=255):
    """matrix.c filter over the whole input frame `src` (bytes); returns the output stream as bytes.
    saturate / fma / rg48_max=65535 are mutants."""
    m = np.asarray(m, np.float64)
    src = np.asarray(src, np.uint8)
    if codec == UYVY:
        q = src[:src.size // 4 * 4].reshape(-1, 4).astype(np.float64)
        u, v = q[:, 0] - 128, q[:, 2] - 128
        px = np.stack([np.stack([q[:, 1] - 16, u, v], 1), np.stack([q[:, 3] - 16, u, v], 1)], 1).reshape(-1, 3)
        bits = 8
    elif codec == RGB:
        px, bits = src[:src.size // 3 * 3].reshape(-1, 3).astype(np.float64), 8
    elif codec == RG48:
        px, bits = src[:src.size // 6 * 6].view(np.uint16).reshape(-1, 3).astype(np.float64), 16
    else:
        return None
    out = np.stack([_dot(m, 3 * r, px[:, 0], px[:, 1], px[:, 2], fma=fma) for r in range(3)], 1).reshape(-1)
    o = _conv(out, bits, check_bounds, saturate, rg48_max if codec == RG48 else 255)
    return o.view(np.uint8) if bits == 16 else o


# ---- matrix2 ---------------------------------------------------------------------------------------------------
def _y416_matrix(m, U, Y, V, fma=False, saturate=False):
    u, y, v = U.astype(np.float64) - (1 << 15), Y.astype(np.float64) - (1 << 12), V.astype(np.float64) - (1 << 15)
    return (_conv(_dot(m, 3, y, u, v, 32768.0, fma), 16, saturate=saturate),
            _conv(_dot(m, 0, y, u, v, 4096.0, fma), 16, saturate=saturate),
            _conv(_dot(m, 6, y, u, v, 32768.0, fma), 16, saturate=saturate))


def v210_to_y416(src):
    """vc_copylineV210toY416 over every whole 16-byte group: (groups * 6, 4) uint16 U Y V A"""
    w = np.asarray(src, np.uint8)[:src.size // 16 * 16].view(np.uint32).reshape(-1, 4)
    f = np.stack([(w >> s) & 0x3FF for s in (0, 10, 20)], 2).reshape(-1, 12).astype(np.uint16) << 6
    cb, cr, y = f[:, [0, 0, 4, 4, 8, 8]], f[:, [2, 2, 6, 6, 10, 10]], f[:, [1, 3, 5, 7, 9, 11]]
    return np.stack([cb, y, cr, np.full_like(y, 0xFFFF)], 2).reshape(-1, 4)


def y416_to_v210(px):
    """vc_copylineY416toV210 over whole groups of 6 pixels: chroma of each pair averaged, >> 6"""
    s = px[:px.shape[0] // 6 * 6].astype(np.uint32).reshape(-1, 6, 4)
    U = (s[:, 0::2, 0] + s[:, 1::2, 0]) // 2
    V = (s[:, 0::2, 2] + s[:, 1::2, 2]) // 2
    Y = s[:, :, 1]
    d = np.stack([U[:, 0] >> 6 | Y[:, 0] >> 6 << 10 | V[:, 0] >> 6 << 20,
                  Y[:, 1] >> 6 | U[:, 1] >> 6 << 10 | Y[:, 2] >> 6 << 20,
                  V[:, 1] >> 6 | Y[:, 3] >> 6 << 10 | U[:, 2] >> 6 << 20,
                  Y[:, 4] >> 6 | V[:, 2] >> 6 << 10 | Y[:, 5] >> 6 << 20], 1).astype(np.uint32)
    return d.reshape(-1).view(np.uint8)


def matrix2_y416(m, px, fma=False, saturate=False):
    U, Y, V = _y416_matrix(np.asarray(m, np.float64), px[:, 0], px[:, 1], px[:, 2], fma, saturate)
    return np.stack([U, Y, V, np.full_like(U, 0xFFFF)], 1)


def matrix2(codec, src, m, fma=False, saturate=False):
    """matrix2.c filter over the whole frame `src`: UYVY and Y416 per pixel, v210 per 16-byte group (the reference
    equals this on groups < w * h // 6 only); None for the codecs it refuses"""
    m = np.asarray(m, np.float64)
    src = np.asarray(src, np.uint8)
    if codec == UYVY:
        q = src.reshape(-1, 4).astype(np.int64)
        u, y1, v, y2 = (q[:, 0] - 128).astype(np.float64), (q[:, 1] - 16).astype(np.float64), \
            (q[:, 2] - 128).astype(np.float64), (q[:, 3] - 16).astype(np.float64)
        y = (y1 + y2) / 2
        return np.stack([_conv(_dot(m, 3, y, u, v, 128.0, fma), 8, saturate=saturate),
                         _conv(_dot(m, 0, y1, u, v, 16.0, fma), 8, saturate=saturate),
                         _conv(_dot(m, 6, y, u, v, 128.0, fma), 8, saturate=saturate),
                         _conv(_dot(m, 0, y2, u, v, 16.0, fma), 8, saturate=saturate)], 1).reshape(-1)
    if codec == Y416:
        return matrix2_y416(m, src.view(np.uint16).reshape(-1, 4), fma, saturate).reshape(-1).view(np.uint8)
    if codec == v210:
        return y416_to_v210(matrix2_y416(m, v210_to_y416(src), fma, saturate))
    return None


# ---- grayscale -------------------------------------------------------------------------------------------------
def grayscale(src, width, height, chroma=127):
    """grayscale.c over w * h pixels: bytes [0, 2 w h); chroma=128 is a mutant"""
    out = np.asarray(src, np.uint8)[:2 * width * height].copy()
    out[0::2] = chroma
    return out


# ---- gamma -----------------------------------------------------------------------------------------------------
_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.pow.restype = ctypes.c_double
_libm.pow.argtypes = [ctypes.c_double, ctypes.c_double]


def gamma_tables(g):
    """gamma.cpp:71-91 with the C library's pow: {(in_bits, out_bits): table}"""
    def table(n_in, max_in, max_out, bits):
        v = np.array([_libm.pow(float(i) / max_in, g) * max_out for i in range(n_in)], np.float64)
        return _conv(v, bits)
    return {(8, 8): table(256, 255.0, 255.0, 8), (16, 16): table(65536, 65535.0, 65535.0, 16),
            (8, 16): table(256, 255.0, 65535.0, 16), (16, 8): table(65536, 65535.0, 255.0, 8)}


def gamma(tables, in_bits, out_bits, src):
    """apply_lut over every sample of src (bytes); the reference leaves the last len % cpus samples unwritten"""
    s = np.asarray(src, np.uint8)
    s = s.view(np.uint16) if in_bits == 16 else s
    return tables[(in_bits, out_bits)][s].view(np.uint8)
