"""The libavcodec bridge (include/ugb200_lavc.h) against a plain numpy restatement of the reference conversions, with no C oracle in between.

Reference.  One vectorised numpy function per conversion, each citing the lines of src/libavcodec/to_lavc_vid_conv.c,
src/libavcodec/from_lavc_vid_conv.c or src/from_planar.c it restates.  Arithmetic is int64 with the reference's int32 comp_type_t emulated:
`>>` is arithmetic, stores wrap to the sample width, CLAMP_LIMITED_* are identities (color_space.h:93-94), and the tests confirm that no
intermediate leaves int32.  The Q14 coefficients are re-derived in float64 from kr, kb and the range scales with the C-cast rounding of
csrc/color_space.h, and equal its static_assert-pinned values (and the reference build's get_color_coeffs when oracle/_ref is built).

CPU pinning of the restatement (no GPU):
  * it equals oracle/lavc_oracle.c on random frames at ragged sizes;
  * identities through functions the tree does pin: v210 -> yuv422p10le -> yuv422p10le_to_v210 is the identity, yuv420p10le == v210_to_p010le
    >> 6, uyvy -> yuv422p -> yuv422p_to_uyvy and uyvy -> yuv444p -> yuv444p_to_uyvy are the identity, rgb -> gbrp -> gbrap_to_rgb is the
    identity; the from_planar restatements equal the unmodified from_planar.c objects when oracle/_ref is built;
  * the RGB-family outputs lie within a bound, derived in code, of the unrounded float64 BT.709 matrix on the same samples;
  * mutants (Cb/Cr swapped, G/B/R permuted, offset dropped, shift off by one, chroma from the odd pixel, YUV444P -> UYVY with alpha as luma)
    each fail a named check.

GPU: every pair the library admits, enumerated from ugb200_to_lavc_supported / ugb200_get_av_to_uv_conversion, equals the restatement byte
for byte, with sentinel bands around every plane and frame.  Bytes the reference's whole-group loops leave unwritten are derived as a mask:
to_lavc must leave them untouched; from_lavc routes through a line converter may fill them, so there they are excluded explicitly.

Two documented choices (DESIGN.md section 8):
  * the reference's yuv420p_to_v210 leaves the luma of word 3 unshifted (from_lavc_vid_conv.c:601-606); the bridge stores it shifted, and the
    restatement here pins the shifted value;
  * the reference's 8-bit from-lavc RGB conversions take matrix and range from the frame (cs_coeffs, lmt_rng); the CUDA hook signature
    (from_lavc_vid_conv_cuda.h:61-69) carries neither, so the bridge's BT.709 limited-range output (the UltraGrid line converters) is the
    contract for YUV -> RGB / RGBA / R10k, and those pairs are checked as planar stage + pinned line converter.
Not pinned: ugb200_lavc.h against libavcodec itself (FFmpeg is not part of the tree)."""
import ctypes

import numpy as np
import pytest

import util
from planar_cases import FromPlanarData, ToPlanarData
from test_jpeg_decode_color_exact import KR_KB, _c_limit, _y_limit, color_coeffs, pinned_values

RGBA, UYVY, VUYA, R10k, R12L, V210, RGB, RG48, Y216 = 1, 2, 4, 5, 6, 7, 12, 27, 30
AV_NAMES = ["NONE", "YUV420P", "YUV422P", "YUV444P", "NV12", "P010LE", "YUV420P10LE", "YUV422P10LE", "YUV444P10LE", "YUV422P12LE", "YUV444P12LE",
            "YUV422P16LE", "YUV444P16LE", "GBRP"]  # enum ugb200_av_pixfmt
AV = {n: i for i, n in enumerate(AV_NAMES)}
FILL, GUARD = 0xA5, 64
_vp, _i, _u = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint
I32 = 1 << 31


# ---- 1. coefficients --------------------------------------------------------------------------------------------------------------------
def coeffs(depth):
    """get_color_coeffs(CS_DFL, depth): BT.709 at the output depth, float64 with the C-cast rounding"""
    return color_coeffs(*KR_KB["Y709"], depth)


def test_coefficients_rederived_equal_header_pins_and_reference():
    pins, _ = pinned_values()
    for depth in (8, 10, 16):
        c = coeffs(depth)
        assert {f: c[f] for f in pins[depth]} == pins[depth], depth
    lib = util.ref_cpu()
    if lib is None:
        return  # only this comparison needs the reference build
    for depth in (8, 10, 12, 16):
        out = (_i * 14)()
        lib.ref_get_color_coeffs(0, depth, out)
        assert list(out)[:9] == [coeffs(depth)[f] for f in ("y_r", "y_g", "y_b", "cb_r", "cb_g", "cb_b", "cr_r", "cr_g", "cr_b")], depth


# ---- 2. the restatement: to_lavc ----------------------------------------------------------------------------------------------------------
def av_geom(fmt, w, h):
    """[(samples per row, rows)] and bytes per sample of each plane of `fmt`"""
    bps = 1 if fmt in ("YUV420P", "YUV422P", "YUV444P", "NV12", "GBRP") else 2
    hs = 0 if "444" in fmt or fmt == "GBRP" else 1
    vs = 1 if "420" in fmt or fmt in ("NV12", "P010LE") else 0
    cw, ch = (w + (1 << hs) - 1) >> hs, (h + (1 << vs) - 1) >> vs
    if fmt in ("NV12", "P010LE"):
        return [(w, h), (2 * cw, ch)], bps
    return [(w, h), (cw, ch), (cw, ch)], bps


def src_linesize(codec, w):
    """the source row stride each reference function uses: vc_get_linesize (R10k rows are padded to 64 pixels, video_codec.c:131), except
    uyvy_to_yuv422p / _yuv444p, whose source pointer runs on over (w + 1) / 2 pairs per row (:137-190), and rgb_rgba_to_gbrp (bpp * width,
    :1320)"""
    return {V210: (w + 47) // 48 * 128, UYVY: (w + 1) // 2 * 4, R10k: (w + 63) // 64 * 256, RG48: 6 * w, R12L: (w + 7) // 8 * 36, RGB: 3 * w,
            RGBA: 4 * w, Y216: (w + 1) // 2 * 8}[codec]


class Planes:
    """plane bodies (rows x linesize bytes) filled with FILL and a mask of the bytes written; put() clips at the row's linesize (the
    library writes no sample beyond it, ugb200_lavc.h)"""

    def __init__(self, shapes, bps):
        self.bps = bps
        self.buf = [np.full((rows, ls), FILL, np.uint8) for ls, rows in shapes]
        self.wr = [np.zeros((rows, ls), bool) for ls, rows in shapes]

    def put(self, i, rows, col0, vals):
        b, rows = self.bps, np.asarray(rows)
        n = max(0, min(vals.shape[1], self.buf[i].shape[1] // b - col0))
        if n == 0 or rows.size == 0:
            return
        v = (np.asarray(vals)[:, :n] & ((1 << (8 * b)) - 1)).astype("<u2" if b == 2 else np.uint8)
        self.buf[i][rows, col0 * b:(col0 + n) * b] = v.view(np.uint8).reshape(len(rows), n * b)
        self.wr[i][rows, col0 * b:(col0 + n) * b] = True


def _v210_fields(src, w, h):
    """Y (h x 6g), Cb and Cr (h x 3g) of the whole 6-pixel groups of a v210 frame (the bit layout comment of :215-226)"""
    ls, g = src_linesize(V210, w), w // 6
    W = src[:ls * h].view("<u4").reshape(h, ls // 4)[:, :4 * g].reshape(h, g, 4).astype(np.int64)
    f = lambda k, s: (W[:, :, k] >> s) & 0x3FF  # noqa: E731
    Y = np.stack([f(0, 10), f(1, 0), f(1, 20), f(2, 10), f(3, 0), f(3, 20)], 2).reshape(h, 6 * g)
    return Y, np.stack([f(0, 0), f(1, 10), f(2, 20)], 2).reshape(h, 3 * g), np.stack([f(0, 20), f(2, 0), f(3, 10)], 2).reshape(h, 3 * g)


def ref_v210(fmt, src, w, h, P):
    """v210_to_yuv420p10le (:197-262), _yuv422p10le (:264-301), _yuv444p10le (:303-346), _yuv444p16le (:348-385): whole groups only (x < width
    / 6).  4:2:0: chroma = (row0 + row1) / 2; an odd last row has no partner - the reference reads and writes one row beyond the frame
    there (:206-210), the bridge leaves that luma row and its chroma row alone."""
    Y, U, V = _v210_fields(src, w, h)
    rows = np.arange(h)
    if fmt == "YUV420P10LE":
        ev = np.arange(h // 2) * 2
        P.put(0, ev, 0, Y[ev]), P.put(0, ev + 1, 0, Y[ev + 1])
        P.put(1, ev // 2, 0, (U[ev] + U[ev + 1]) // 2), P.put(2, ev // 2, 0, (V[ev] + V[ev + 1]) // 2)
    elif fmt == "YUV422P10LE":
        P.put(0, rows, 0, Y), P.put(1, rows, 0, U), P.put(2, rows, 0, V)
    else:
        sh = 6 if fmt == "YUV444P16LE" else 0
        P.put(0, rows, 0, Y << sh), P.put(1, rows, 0, np.repeat(U, 2, 1) << sh), P.put(2, rows, 0, np.repeat(V, 2, 1) << sh)


def ref_uyvy(fmt, src, w, h, P):
    """uyvy_to_yuv422p (:137-151), uyvy_to_yuv444p (:174-190): two pixels per step while x < width, both written (an odd width writes one
    luma sample more, clipped at the linesize here); the source pointer runs on, (w + 1) / 2 pairs per row"""
    pairs = (w + 1) // 2
    S = src[:4 * pairs * h].reshape(h, pairs, 4).astype(np.int64)
    rows = np.arange(h)
    P.put(0, rows, 0, S[:, :, [1, 3]].reshape(h, 2 * pairs))
    rep = 2 if fmt == "YUV444P" else 1
    P.put(1, rows, 0, np.repeat(S[:, :, 0], rep, 1)), P.put(2, rows, 0, np.repeat(S[:, :, 2], rep, 1))


def rgb_samples(codec, src, w, h):
    """(r, g, b) int64 arrays (h x n) and the input depth; R12L gives whole groups of 8 (:790)"""
    ls = src_linesize(codec, w)
    rows = src[:ls * h].reshape(h, ls)
    if codec == R10k:  # big-endian 10:10:10:2 (:720-722)
        s = rows[:, :4 * w].reshape(h, w, 4).astype(np.int64)
        return s[..., 0] << 2 | s[..., 1] >> 6, (s[..., 1] & 0x3F) << 4 | s[..., 2] >> 4, (s[..., 2] & 0x0F) << 6 | s[..., 3] >> 2, 10
    if codec == RG48:  # (:1150-1152)
        s = rows[:, :6 * w].copy().view("<u2").reshape(h, w, 3).astype(np.int64)
        return s[..., 0], s[..., 1], s[..., 2], 16
    if codec == R12L:  # the byte picking of :798-860: field k even = s[o] | (s[o+1] & 0xF) << 8, odd = s[o+1] << 4 | s[o] >> 4, o = 12k / 8
        g = ls // 36
        B = rows.reshape(h, g, 36).astype(np.int64)
        f = [B[..., 3 * k // 2] | (B[..., 3 * k // 2 + 1] & 0xF) << 8 if k % 2 == 0 else B[..., 12 * k // 8 + 1] << 4 | B[..., 12 * k // 8] >> 4
             for k in range(24)]
        return tuple(np.stack(f[c::3], 2).reshape(h, 8 * g) for c in range(3)) + (12,)
    s = rows[:, :3 * w].reshape(h, w, 3).astype(np.int64)  # RGB, :1208-1210
    return s[..., 0], s[..., 1], s[..., 2], 8


def rgb_to_ycc(r, g, b, in_depth, depth, mutant=None):
    """RGB_TO_Y / _CB / _CR (color_space.h) >> (COMP_BASE + in_depth - depth), + 1 << (depth - 4) or + 1 << (depth - 1), in int32"""
    c = coeffs(depth)
    sh = 14 + in_depth - depth + (1 if mutant == "shift" else 0)
    acc = [r * c[k + "_r"] + g * c[k + "_g"] + b * c[k + "_b"] for k in ("y", "cb", "cr")]
    assert all(int(np.abs(a).max(initial=0)) < I32 for a in acc), "comp_type_t is int32_t"
    coff = 0 if mutant == "no_offset" else 1 << (depth - 1)
    y, cb, cr = (acc[0] >> sh) + (1 << (depth - 4)), (acc[1] >> sh) + coff, (acc[2] >> sh) + coff
    assert max(int(np.abs(v).max(initial=0)) for v in (y, cb, cr)) < I32
    return (y, cr, cb) if mutant == "swap_cbcr" else (y, cb, cr)


def ref_rgb(codec, fmt, src, w, h, P, mutant=None):
    """r10k_to_yuv444pXXle (:703-755), r12l_to_yuv4XXpYYle (:758-895; 4:2:2 chroma from the even pixel, :772), rg48_to_yuv444pXXle
    (:1133-1183), rgb_to_yuv444p (:1188-1227)"""
    r, g, b, in_depth = rgb_samples(codec, src, w, h)
    depth = 8 if fmt == "YUV444P" else int(fmt[7:9])
    y, cb, cr = rgb_to_ycc(r, g, b, in_depth, depth, mutant)
    rows = np.arange(h)
    P.put(0, rows, 0, y)
    if "422" in fmt:
        k = 1 if mutant == "odd_chroma" else 0
        cb, cr = cb[:, k::2], cr[:, k::2]
    P.put(1, rows, 0, cb), P.put(2, rows, 0, cr)


def ref_gbrp(codec, src, w, h, P, mutant=None):
    """rgb_rgba_to_gbrp (:1315-1333): planes G, B, R"""
    bpp = 4 if codec == RGBA else 3
    s = src[:bpp * w * h].reshape(h, w, bpp).astype(np.int64)
    order = (0, 1, 2) if mutant == "gbr_perm" else (1, 2, 0)
    for i, c in enumerate(order):
        P.put(i, np.arange(h), 0, s[..., c])


DELEGATED = {(UYVY, "YUV420P"): "uyvy_to_i420", (UYVY, "NV12"): "uyvy_to_nv12", (V210, "P010LE"): "v210_to_p010le", (Y216, "P010LE"): "y216_to_p010le"}


def ref_delegated(orc, inc, fmt, src, w, h, P):
    """the conversions the reference hands to src/to_planar.c (:132-135, :192-195, to_lavc_v210_to_p010le, to_lavc_y216_to_p010le): the CPU
    restatement of to_planar.c (oracle/planar_oracle.c, pinned to the unmodified objects by test_planar.py), run twice over different fills
    so that the bytes it writes are known.  Below one v210 group of width the reference writes past the end of a plane (a pair's group spans
    several rows); those bytes are not part of the plane and the library leaves them alone (the guard bands of the GPU tests)."""
    runs = []
    for fill in (FILL, FILL ^ 0xFF):
        bufs = [np.full(b.size + GUARD, fill, np.uint8) for b in P.buf]
        name = DELEGATED[(inc, fmt)]
        srcp = np.concatenate([src, np.zeros(4096, np.uint8)])
        if name == "v210_to_p010le":
            orc.orc_v210_to_p010le(w, h, bufs[0].ctypes.data, P.buf[0].shape[1], bufs[1].ctypes.data, P.buf[1].shape[1], srcp.ctypes.data)
        else:
            d = ToPlanarData()
            d.width, d.height, d.in_data = w, h, srcp.ctypes.data
            for i, b in enumerate(bufs):
                d.out_data[i], d.out_linesize[i] = b.ctypes.data, P.buf[i].shape[1]
            fn = getattr(orc, "orc_" + name)
            fn.argtypes, fn.restype = [ToPlanarData], None
            fn(d)
        runs.append(bufs)
    for i, b in enumerate(P.buf):
        a, c = runs[0][i], runs[1][i]
        wr = (a == c)[:b.size].reshape(b.shape)
        b[wr] = a[:b.size].reshape(b.shape)[wr]
        P.wr[i] |= wr


def ref_to_lavc(inc, fmt, src, w, h, lss, orc=None, mutant=None):
    """the numpy reference of one to_lavc conversion into planes of line sizes `lss`: (Planes with bodies and written masks)"""
    shapes, bps = av_geom(fmt, w, h)
    P = Planes([(ls, rows) for ls, (_, rows) in zip(lss, shapes)], bps)
    if (inc, fmt) in DELEGATED:
        ref_delegated(orc, inc, fmt, src, w, h, P)
    elif inc == V210:
        ref_v210(fmt, src, w, h, P)
    elif inc == UYVY:
        ref_uyvy(fmt, src, w, h, P)
    elif fmt == "GBRP":
        ref_gbrp(inc, src, w, h, P, mutant)
    else:
        ref_rgb(inc, fmt, src, w, h, P, mutant)
    return P


def make_source(inc, w, h, seed):
    ls = src_linesize(inc, w)
    if inc == V210:
        return util.v210_noise(w, h, seed)
    return util.rng_bytes(ls * h, seed)


# ---- 3. the restatement: from_lavc --------------------------------------------------------------------------------------------------------
def av_planes_in(fmt, w, h, seed, pad=0):
    """random decoder planes of `fmt`: [(array rows x ls bytes, ls)]; 10-bit samples below 1024; GBRP planes share linesize[0]"""
    shapes, bps = av_geom(fmt, w, h)
    rng = np.random.default_rng(seed)
    out = []
    for n, rows in shapes:
        ls = (shapes[0][0] if fmt == "GBRP" else n) * bps + pad * bps
        a = rng.integers(0, 256, (rows, ls), dtype=np.uint8)
        if bps == 2:
            a = (a.view("<u2") & 0x3FF).view(np.uint8)
        out.append((a, ls))
    return out


def _samples(planes, i, bps):
    a = planes[i][0]
    return (a.view("<u2") if bps == 2 else a).astype(np.int64)


class Frame:
    """a packed frame (rows x pitch bytes) filled with FILL and a mask of the bytes written"""

    def __init__(self, h, pitch):
        self.buf, self.wr = np.full((h, pitch), FILL, np.uint8), np.zeros((h, pitch), bool)

    def put(self, rows, col0, b):
        b = np.asarray(b, np.int64).astype(np.uint8) if b.dtype != np.uint8 else b
        self.buf[rows, col0:col0 + b.shape[1]], self.wr[rows, col0:col0 + b.shape[1]] = b, True


def _words(*ws):
    return np.stack(ws, -1).astype("<u4").view(np.uint8).reshape(ws[0].shape[0], -1)


def fp_yuv420p_to_uyvy(pl, w, h, F):
    """yuv420p_to_uyvy, from_planar.c:582-683: chroma row y / 2 serves rows y and y + 1 (an odd last row pairs with itself); pairs while
    x < width - 1, then an odd last pixel as Cb Y Cr 0"""
    Y, U, V = (_samples(pl, i, 1) for i in range(3))
    rows = np.arange(h)
    n = w // 2
    c = rows // 2
    out = np.stack([U[c][:, :n], Y[:, :2 * n:2], V[c][:, :n], Y[:, 1:2 * n:2]], 2).reshape(h, 4 * n)
    F.put(rows, 0, out)
    if w % 2:
        F.put(rows, 4 * n, np.stack([U[c][:, n], Y[:, w - 1], V[c][:, n], np.zeros(h, np.int64)], 1))


def fp_yuv422p_to_uyvy(pl, w, h, F, depth=8):
    """yuv422p_to_uyvy_yuyv (from_planar.c:392-417) and yuv422pXXle_to_uyvy_int (:425-441, samples >> depth - 8): width / 2 pairs"""
    Y, U, V = (_samples(pl, i, 1 if depth == 8 else 2) >> (depth - 8) for i in range(3))
    n = w // 2
    F.put(np.arange(h), 0, np.stack([U[:, :n], Y[:, 0:2 * n:2], V[:, :n], Y[:, 1:2 * n:2]], 2).reshape(h, 4 * n))


def fp_yuv444p_to_uyvy(pl, w, h, F, mutant=None):
    """yuv444p_to_uyvy, from_lavc_vid_conv.c:663-685: width / 2 pairs, chroma = (c[2x] + c[2x + 1]) / 2 (C truncation), luma copied"""
    Y, U, V = (_samples(pl, i, 1) for i in range(3))
    n = w // 2
    y1 = np.full((h, n), 0xFF, np.int64) if mutant == "alpha_luma" else Y[:, 1:2 * n:2]
    F.put(np.arange(h), 0, np.stack([(U[:, 0:2 * n:2] + U[:, 1:2 * n:2]) // 2, Y[:, 0:2 * n:2], (V[:, 0:2 * n:2] + V[:, 1:2 * n:2]) // 2, y1],
                                    2).reshape(h, 4 * n))


def fp_yuv444p_to_vuya(pl, w, h, F):
    """yuv444p_to_vuya, from_planar.c:565-580: V U Y 0xFF"""
    Y, U, V = (_samples(pl, i, 1)[:, :w] for i in range(3))
    F.put(np.arange(h), 0, np.stack([V, U, Y, np.full_like(Y, 0xFF)], 2).reshape(h, 4 * w))


def _v210_put(F, rows, Y, B, R):
    """whole 6-pixel groups: B0 | Y0 << 10 | R0 << 20, Y1 | B1 << 10 | Y2 << 20, R1 | Y3 << 10 | B2 << 20, Y4 | R2 << 10 | Y5 << 20"""
    g = Y.shape[1] // 6
    if g == 0 or len(rows) == 0:
        return
    Y, B, R = Y[:, :6 * g].reshape(-1, g, 6), B[:, :3 * g].reshape(-1, g, 3), R[:, :3 * g].reshape(-1, g, 3)
    F.put(rows, 0, _words(B[..., 0] | Y[..., 0] << 10 | R[..., 0] << 20, Y[..., 1] | B[..., 1] << 10 | Y[..., 2] << 20,
                          R[..., 1] | Y[..., 3] << 10 | B[..., 2] << 20, Y[..., 4] | R[..., 2] << 10 | Y[..., 5] << 20).reshape(len(rows), -1))


def fp_yuv422p10le_to_v210(pl, w, h, F):
    """yuv422p10le_to_v210, from_planar.c:295-333: x < width / 6"""
    Y, U, V = (_samples(pl, i, 2) for i in range(3))
    _v210_put(F, np.arange(h), Y[:, :w // 6 * 6], U, V)


def fl_yuv422p_to_v210(pl, w, h, F):
    """yuv422p_to_v210, from_lavc_vid_conv.c:622-661: 8-bit samples << 2, x < width / 6"""
    Y, U, V = (_samples(pl, i, 1) << 2 for i in range(3))
    _v210_put(F, np.arange(h), Y[:, :w // 6 * 6], U, V)


def fl_yuv420p_to_v210(pl, w, h, F, quirk=False):
    """yuv420p_to_v210, from_lavc_vid_conv.c:554-620: row pairs y < height / 2 (an odd last row is not written), chroma row y, 8-bit << 2.
    The reference leaves the luma of word 3 unshifted (:601-602); quirk=False pins the shifted value the bridge stores (DESIGN.md 8)."""
    Y, U, V = (_samples(pl, i, 1) << 2 for i in range(3))
    n = h // 2
    for k in (0, 1):
        rows = np.arange(n) * 2 + k
        Yk = Y[rows, :w // 6 * 6].copy()
        if quirk:
            Yk[:, 4::6] >>= 2
        _v210_put(F, rows, Yk, U[:n], V[:n])


def fl_gbrp_to_rgb(pl, w, h, F):
    """gbrp_to_rgb (from_lavc_vid_conv.c:222-237) = gbrap_to_rgb (from_planar.c:335-354): R G B from planes 2, 0, 1, all at linesize[0]"""
    G, B, R = (_samples(pl, i, 1)[:, :w] for i in range(3))
    F.put(np.arange(h), 0, np.stack([R, G, B], 2).reshape(h, 3 * w))


def fl_gbrp_to_rgba(pl, w, h, F, shifts):
    """gbrp_to_rgba, from_lavc_vid_conv.c:240-262: alpha_mask | R << rs | G << gs | B << bs"""
    rs, gs, bs = shifts
    G, B, R = (_samples(pl, i, 1)[:, :w] for i in range(3))
    amask = 0xFFFFFFFF ^ (0xFF << rs) ^ (0xFF << gs) ^ (0xFF << bs)
    F.put(np.arange(h), 0, _words((amask | R << rs | G << gs | B << bs) & 0xFFFFFFFF))


# the planar stage of each route (ugb200_av_to_uv_convert): the decoder's format -> the codec its kernel produces
PLANAR_STAGE = {"YUV420P": (UYVY, fp_yuv420p_to_uyvy), "YUV422P": (UYVY, fp_yuv422p_to_uyvy), "YUV444P": (VUYA, fp_yuv444p_to_vuya),
                "YUV422P10LE": (V210, fp_yuv422p10le_to_v210), "GBRP": (RGB, fl_gbrp_to_rgb)}
# av_to_uv_conversions[] entries (from_lavc_vid_conv.c:2050-2160) whose result the bridge reproduces exactly
DIRECT = {("YUV420P", UYVY): fp_yuv420p_to_uyvy, ("YUV422P", UYVY): fp_yuv422p_to_uyvy, ("YUV444P", UYVY): fp_yuv444p_to_uyvy,
          ("YUV444P", VUYA): fp_yuv444p_to_vuya, ("YUV422P10LE", V210): fp_yuv422p10le_to_v210,
          ("YUV422P10LE", UYVY): lambda pl, w, h, F: fp_yuv422p_to_uyvy(pl, w, h, F, depth=10),
          ("YUV420P", V210): fl_yuv420p_to_v210, ("YUV422P", V210): fl_yuv422p_to_v210, ("GBRP", RGB): fl_gbrp_to_rgb}


def v210_partial_group(pl, w, h, F):
    """the bridge's YUV422P10LE -> v210 intermediate also converts the partial last group of a row, which yuv422p10le_to_v210 leaves out
    (from_planar.c:308): the row's remaining samples, 0 beyond the width"""
    g = w // 6
    if w % 6 == 0:
        return
    Y, U, V = (_samples(pl, i, 2) for i in range(3))
    z = lambda a, n: np.concatenate([a[:, :n], np.zeros((h, 6 - n), np.int64)], 1)  # noqa: E731
    Yp, Up, Vp = z(Y[:, 6 * g:], w - 6 * g), z(U[:, 3 * g:], (w + 1) // 2 - 3 * g), z(V[:, 3 * g:], (w + 1) // 2 - 3 * g)
    P = Frame(h, 16)
    _v210_put(P, np.arange(h), Yp, Up, Vp)
    F.put(np.arange(h), 16 * g, P.buf)


def ref_from_lavc(orc, fmt, out, pl, w, h, pitch, shifts):
    """(expected frame rows x pitch, mask of the bytes compared).  A direct reference entry: its restatement, compared where it writes.
    Otherwise the planar stage, then the CPU line converter (orc_convert, pinned to pixfmt_conv.c by test_pixfmt_gpu.py) row by row into a
    frame of its own; the bytes the planar stage leaves unwritten are filled three ways and the converter's frame two ways, and only bytes
    equal in every run are compared: the rest depend on bytes nobody defines, or are bytes of the line the reference leaves unwritten.
    A v210 intermediate's line converters write whole 6-pixel groups: they convert the rounded-up width, the destination gets the line."""
    from ultragrid_b200.codec import vc_get_linesize
    F = Frame(h, pitch)
    if (fmt, out) == ("GBRP", RGBA):
        fl_gbrp_to_rgba(pl, w, h, F, shifts)
    elif (fmt, out) in DIRECT:
        DIRECT[(fmt, out)](pl, w, h, F)
    else:
        mid, stage = PLANAR_STAGE[fmt]
        wc = -(-w // 6) * 6 if mid == V210 else w
        mp, ls, lsc = vc_get_linesize(w, mid), vc_get_linesize(w, out), vc_get_linesize(wc, out)
        M = Frame(h, mp)
        stage(pl, w, h, M)
        if mid == V210:
            v210_partial_group(pl, w, h, M)
        outs = []
        for k, (fill, dfill) in enumerate(((0x00, FILL), (0xFF, FILL ^ 0xFF), (None, FILL))):
            m = M.buf.copy()
            m[~M.wr] = np.random.default_rng(k).integers(0, 256, int((~M.wr).sum()), dtype=np.uint8) if fill is None else fill
            src = np.concatenate([m.reshape(-1), np.zeros(4096, np.uint8)])
            dst = np.full(lsc * h + 4096, dfill, np.uint8)
            assert orc.orc_convert(mid, out, dst.ctypes.data, lsc, src.ctypes.data, mp, lsc, h, *shifts) == 0
            outs.append(dst[:lsc * h].reshape(h, lsc)[:, :ls])
        det = (outs[0] == outs[1]) & (outs[0] == outs[2])
        F.buf[:, :ls][det], F.wr[:, :ls][det] = outs[0][det], True
    assert_covers(fmt, out, w, h, F)
    return F


# out codec: (pixels, bytes) of its smallest whole unit
BLOCK = {UYVY: (2, 4), 3: (2, 4), Y216: (2, 8), V210: (6, 16), R12L: (8, 36), RGB: (1, 3), RGBA: (1, 4), RG48: (1, 6), 31: (1, 8), VUYA: (1, 4)}


def assert_covers(fmt, out, w, h, F):
    """the compared mask holds every byte of the whole output units the reference defines, so that a mistake in deriving it cannot exclude an
    output silently.  Defined pixels: the whole width, except that pixel-pair steps (a UYVY intermediate's line converters, and the direct
    UYVY / v210 entries) stop at the last whole pair or group; rows: all, except the odd last row yuv420p_to_v210 does not write (:561)."""
    mid = PLANAR_STAGE[fmt][0]
    px, bb = BLOCK[out]
    n = 2 * (w // 2) if mid == UYVY or (fmt, out) in DIRECT else w
    rows = h // 2 * 2 if (fmt, out) == ("YUV420P", V210) else h
    need = n // px * bb
    assert F.wr[:rows, :need].all(), (fmt, out, w, h, "bytes of defined output units excluded from the comparison")


# ---- 4. CPU pinning -----------------------------------------------------------------------------------------------------------------------
TO_PAIRS_KNOWN = [(V210, f) for f in ("YUV420P10LE", "YUV422P10LE", "YUV444P10LE", "YUV444P16LE")] + [(UYVY, "YUV422P"), (UYVY, "YUV444P")] + \
    [(c, f"YUV444P{d}LE") for c in (R10k, RG48, R12L) for d in (10, 12, 16)] + [(R12L, f"YUV422P{d}LE") for d in (10, 12, 16)] + \
    [(RGB, "YUV444P"), (RGB, "GBRP"), (RGBA, "GBRP")]


def orc_lavc(orc, inc, fmt, src, w, h, lss):
    """oracle/lavc_oracle.c into guard-banded host planes (it writes like the reference, whole groups included)"""
    shapes, _ = av_geom(fmt, w, h)
    bufs = [np.full(ls * rows + 4 * GUARD, FILL, np.uint8) for ls, (_, rows) in zip(lss, shapes)]
    p = (_vp * 3)(*[b.ctypes.data for b in bufs] + [None] * (3 - len(bufs)))
    ls = (_i * 3)(*lss)
    srcp = np.concatenate([src, np.zeros(4096, np.uint8)])
    s = srcp.ctypes.data
    for n in ("orc_lavc_v210", "orc_lavc_uyvy", "orc_lavc_gbrp"):
        getattr(orc, n).argtypes, getattr(orc, n).restype = [_i, _vp, _i, _i, _vp, _vp], None
    orc.orc_lavc_rgb.argtypes, orc.orc_lavc_rgb.restype = [_i, _i, _i, _vp, _vp, _i, _i, _vp, _vp], None
    if inc == V210:
        orc.orc_lavc_v210(["YUV420P10LE", "YUV422P10LE", "YUV444P10LE", "YUV444P16LE"].index(fmt), s, w, h, p, ls)
    elif inc == UYVY:
        orc.orc_lavc_uyvy(int(fmt == "YUV444P"), s, w, h, p, ls)
    elif fmt == "GBRP":
        orc.orc_lavc_gbrp(3 if inc == RGB else 4, s, w, h, p, ls)
    else:
        depth = 8 if fmt == "YUV444P" else int(fmt[7:9])
        c = coeffs(depth)
        cs = (_i * 9)(*[c[k] for k in ("y_r", "y_g", "y_b", "cb_r", "cb_g", "cb_b", "cr_r", "cr_g", "cr_b")])
        orc.orc_lavc_rgb({R10k: 0, RG48: 1, R12L: 2, RGB: 3}[inc], depth, int("422" in fmt), cs, s, w, h, p, ls)
    return [b[:ls_ * rows].reshape(rows, ls_) for b, ls_, (_, rows) in zip(bufs, lss, shapes)]


@pytest.mark.parametrize("inc,fmt", TO_PAIRS_KNOWN)
def test_restatement_equals_lavc_oracle(orc, inc, fmt):
    """the numpy restatement == oracle/lavc_oracle.c on random frames at ragged sizes, wherever the restatement writes (the oracle, like the
    reference, may also spill a whole group or an odd-width sample past a row; the restatement clips at the linesize)"""
    for k, (w, h) in enumerate([(48, 4), (49, 3), (47, 2), (6, 1), (8, 3), (1922, 3), (100, 5), (13, 7)]):
        if inc == V210 and fmt == "YUV420P10LE" and h % 2:
            h -= 1 if h > 1 else 0  # the oracle stops early on an odd last row like the bridge; compared on the even part
        shapes, bps = av_geom(fmt, w, h)
        lss = [n * bps + (k % 3) * 2 * bps for n, _ in shapes]
        src = make_source(inc, w, h, 40 + k)
        want = ref_to_lavc(inc, fmt, src, w, h, lss)
        got = orc_lavc(orc, inc, fmt, src, w, h, lss)
        for i, (g, b, wr) in enumerate(zip(got, want.buf, want.wr)):
            assert np.array_equal(g[wr], b[wr]), (w, h, i)


def test_restatement_no_int32_overflow_at_depth_16():
    """the extreme RG48 / R12L / R10k samples through the depth-16 matrix stay inside int32 (the asserts of rgb_to_ycc)"""
    for in_depth in (16, 12, 10):
        m = (1 << in_depth) - 1
        v = np.array([[0, m, m, 0, 0, m, m, 0]], np.int64)
        for r, g, b in [(v, v, v), (v, 0 * v, 0 * v), (0 * v, v, 0 * v), (0 * v, 0 * v, v), (v, v[:, ::-1], 0 * v)]:
            y, cb, cr = rgb_to_ycc(r, g, b, in_depth, 16)
            assert y.min() >= 0 and y.max() < 65536 and cb.min() >= 0 and cb.max() < 65536 and cr.min() >= 0 and cr.max() < 65536


def _ref_fp(ref_cpu, name, pl, w, h, out_pitch, depth=8):
    """an unmodified from_planar.c function on host planes"""
    out = np.full(out_pitch * h + GUARD, FILL, np.uint8)
    d = FromPlanarData()
    d.width, d.height, d.out_data, d.out_pitch, d.in_depth = w, h, out.ctypes.data, out_pitch, depth
    keep = [np.concatenate([a.reshape(-1), np.zeros(4096, np.uint8)]) for a, _ in pl]
    for i, ((_, ls), a) in enumerate(zip(pl, keep)):
        d.in_data[i], d.in_linesize[i] = a.ctypes.data, ls
    d.rgb_shift[0], d.rgb_shift[1], d.rgb_shift[2] = 0, 8, 16
    fn = getattr(ref_cpu, name)
    fn.argtypes, fn.restype = [FromPlanarData], None
    fn(d)
    assert np.all(out[out_pitch * h:] == FILL)
    return out[:out_pitch * h].reshape(h, out_pitch)


@pytest.mark.parametrize("fmt,name,fn", [("YUV420P", "yuv420p_to_uyvy", fp_yuv420p_to_uyvy), ("YUV422P", "yuv422p_to_uyvy", fp_yuv422p_to_uyvy),
                                         ("YUV444P", "yuv444p_to_vuya", fp_yuv444p_to_vuya), ("YUV422P10LE", "yuv422p10le_to_v210", fp_yuv422p10le_to_v210),
                                         ("YUV422P10LE", "yuv422p10le_to_uyvy", DIRECT[("YUV422P10LE", UYVY)]), ("GBRP", "gbrap_to_rgb", fl_gbrp_to_rgb)])
def test_from_planar_restatements_equal_reference_objects(ref_cpu, fmt, name, fn):
    """the planar stages restated here == the unmodified from_planar.c functions, wherever either writes (yuv420p_to_uyvy's SSE3 loop bound
    `width - 15` is unsigned, so its widths start at 15)"""
    for k, (w, h) in enumerate([(48, 4), (49, 3), (47, 5), (15, 1), (16, 2), (1922, 3), (100, 6)]):
        for pad in (0, 13):
            pl = av_planes_in(fmt, w, h, 70 + k, pad)
            pitch = 4 * w + 64 + pad
            F = Frame(h, pitch)
            fn(pl, w, h, F)
            ref = _ref_fp(ref_cpu, name, pl, w, h, pitch, 10 if "10" in fmt else 8)
            assert np.array_equal(ref, F.buf), (w, h, pad)


def check_v210_round_trip(ref, ref_cpu):
    """v210 -> yuv422p10le (restated) -> unmodified yuv422p10le_to_v210 (from_planar.c:295-333) == the frame, 30 valid bits per word"""
    w, h = 96, 6
    src = util.v210_noise(w, h, 4)
    P = ref(V210, "YUV422P10LE", src, w, h, [2 * w, w, w])
    back = np.zeros_like(src)
    ref_cpu.ref_yuv422p10le_to_v210.argtypes = [_i, _i, _vp, _u, _vp, _vp, _vp, _u, _u]
    ref_cpu.ref_yuv422p10le_to_v210(w, h, back.ctypes.data, len(src) // h, P.buf[0].ctypes.data, P.buf[1].ctypes.data, P.buf[2].ctypes.data,
                                    2 * w, w)
    assert np.array_equal(back, src)


def check_v210_420_is_p010_shifted(ref, ref_cpu):
    """v210 -> yuv420p10le == unmodified v210_to_p010le (to_planar.c:64-155) >> 6, chroma de-interleaved"""
    w, h = 96, 6
    src = util.v210_noise(w, h, 5)
    P = ref(V210, "YUV420P10LE", src, w, h, [2 * w, w, w])
    y, c = np.zeros(w * 2 * h, np.uint8), np.zeros(w * h, np.uint8)
    ref_cpu.ref_v210_to_p010le(w, h, y.ctypes.data, w * 2, c.ctypes.data, w * 2, src.ctypes.data)
    assert np.array_equal(P.buf[0].view("<u2"), y.view("<u2").reshape(h, w) >> 6)
    cc = (c.view("<u2") >> 6).reshape(h // 2, w)
    assert np.array_equal(P.buf[1].view("<u2"), cc[:, 0::2]) and np.array_equal(P.buf[2].view("<u2"), cc[:, 1::2])


def check_uyvy_planes_invert_to_uyvy(ref, fp444=fp_yuv444p_to_uyvy):
    """uyvy -> yuv422p, then yuv422p_to_uyvy (restated, pinned above), and uyvy -> yuv444p, then yuv444p_to_uyvy (from_lavc_vid_conv.c:663-685,
    the mean of two equal chroma samples is the sample) are the identity"""
    w, h = 50, 3
    src = util.rng_bytes(2 * w * h, 6)
    for fmt, back in (("YUV422P", fp_yuv422p_to_uyvy), ("YUV444P", fp444)):
        shapes, _ = av_geom(fmt, w, h)
        P = ref(UYVY, fmt, src, w, h, [n for n, _ in shapes])
        F = Frame(h, 2 * w)
        back([(b, b.shape[1]) for b in P.buf], w, h, F)
        assert np.array_equal(F.buf.reshape(-1), src), fmt


def check_gbrp_inverts_to_rgb(ref):
    """rgb -> gbrp, then gbrap_to_rgb (restated, pinned above) is the identity: the planes are G, B, R"""
    w, h = 33, 4
    src = util.rng_bytes(3 * w * h, 7)
    P = ref(RGB, "GBRP", src, w, h, [w, w, w])
    F = Frame(h, 3 * w)
    fl_gbrp_to_rgb([(b, w) for b in P.buf], w, h, F)
    assert np.array_equal(F.buf.reshape(-1), src)


def rgb_bound_violations(ref, inc, fmt, seed=8):
    """|output - unrounded float64 BT.709 on the same samples| beyond the bound derived from the arithmetic: the Q14 sum is within
    sum_j |c_j - 2^14 m_j| s_j / 2^sh of the exact value (the rounding error of each coefficient as color_space.c rounds it: up to 1/2, up to 1
    for cr_r and cr_b, whose +-0.5 has the opposite sign of the value), and `>>` floors (up to 1 - 2^-sh below).  Returns the number of
    samples outside."""
    w, h = 64, 6
    src = make_source(inc, w, h, seed)
    shapes, bps = av_geom(fmt, w, h)
    P = ref(inc, fmt, src, w, h, [n * bps for n, _ in shapes])
    r, g, b, in_depth = rgb_samples(inc, src, w, h)
    depth = 8 if fmt == "YUV444P" else int(fmt[7:9])
    kr, kb = KR_KB["Y709"]
    kg, yl, cl = 1 - kr - kb, _y_limit(depth), _c_limit(depth)
    M = np.array([[kr * yl, kg * yl, kb * yl], [-kr / (2 * (kr + kg)) * cl, -kg / (2 * (kr + kg)) * cl, (1 - kb) / (2 * (kr + kg)) * cl],
                  [(1 - kr) / (2 * (1 - kr)) * cl, -kg / (2 * (1 - kr)) * cl, -kb / (2 * (1 - kr)) * cl]])
    scale = 2.0 ** (depth - in_depth)
    off = [1 << (depth - 4), 1 << (depth - 1), 1 << (depth - 1)]
    n = r.shape[1] if inc == R12L else w
    rgb = np.stack([r[:, :n], g[:, :n], b[:, :n]], -1).astype(np.float64)
    sh = 14 + in_depth - depth
    c = coeffs(depth)
    Q = np.array([[c[k + s] for s in ("_r", "_g", "_b")] for k in ("y", "cb", "cr")], np.float64)
    bad = 0
    for i in range(3):
        exact = rgb @ M[i] * scale + off[i]
        err = rgb @ np.abs(Q[i] - 16384 * M[i]) / 2.0 ** sh
        got = P.buf[i].view("<u2" if bps == 2 else np.uint8).astype(np.float64)[:, :P.buf[i].shape[1] // bps]
        if i and "422" in fmt:
            exact, e = exact[:, 0::2], err[:, 0::2]
        else:
            e = err
        m = min(got.shape[1], exact.shape[1])
        d = got[:, :m] - exact[:, :m]
        bad += int(np.count_nonzero((d > e[:, :m]) | (d < -e[:, :m] - 1)))
    return bad


RGB_FAMILY = [p for p in TO_PAIRS_KNOWN if p[0] in (R10k, RG48, R12L, RGB) and p[1] != "GBRP"]


@pytest.mark.parametrize("inc,fmt", RGB_FAMILY)
def test_rgb_family_within_float64_bound(inc, fmt):
    assert rgb_bound_violations(ref_to_lavc, inc, fmt) == 0


def test_identities_through_reference_functions(ref_cpu):
    check_v210_round_trip(ref_to_lavc, ref_cpu)
    check_v210_420_is_p010_shifted(ref_to_lavc, ref_cpu)


def test_identities_of_the_planar_restatements():
    check_uyvy_planes_invert_to_uyvy(ref_to_lavc)
    check_gbrp_inverts_to_rgb(ref_to_lavc)


def _mut(m):
    return lambda inc, fmt, src, w, h, lss: ref_to_lavc(inc, fmt, src, w, h, lss, mutant=m)


@pytest.mark.parametrize("mutant,catcher", [
    ("swap_cbcr", lambda: rgb_bound_violations(_mut("swap_cbcr"), RG48, "YUV444P16LE") > 0),
    ("no_offset", lambda: rgb_bound_violations(_mut("no_offset"), R10k, "YUV444P10LE") > 0),
    ("shift", lambda: rgb_bound_violations(_mut("shift"), RGB, "YUV444P") > 0),
    ("odd_chroma", lambda: rgb_bound_violations(_mut("odd_chroma"), R12L, "YUV422P12LE") > 0),
    ("gbr_perm", lambda: _fails(check_gbrp_inverts_to_rgb, _mut("gbr_perm"))),
    ("alpha_luma", lambda: _fails(check_uyvy_planes_invert_to_uyvy, ref_to_lavc,
                                  lambda pl, w, h, F: fp_yuv444p_to_uyvy(pl, w, h, F, mutant="alpha_luma"))),
])
def test_mutants_are_reported(mutant, catcher):
    """each mutant of the restatement fails a named check: the float64 bound (test_rgb_family_within_float64_bound) or an identity
    (test_identities_of_the_planar_restatements); the alpha_luma mutant is today's YUV444P -> VUYA -> UYVY route, whose
    vc_copylineVUYAtoUYVY takes the second luma from the alpha byte (pixfmt_conv.c:2699)"""
    assert catcher(), mutant


def _fails(check, *args):
    try:
        check(*args)
    except AssertionError:
        return True
    return False


def _lib_built():
    import os
    return os.path.exists(os.path.join(util.ROOT, "ultragrid_b200", "libugb200.so"))


# ---- 5. GPU: to_lavc ----------------------------------------------------------------------------------------------------------------------
def lib_and_torch():
    import torch
    from ultragrid_b200 import _lib
    L = _lib.load()
    L.ugb200_to_lavc_convert.argtypes = [_i, _i, _vp, _vp, _i, _i, _vp]
    L.ugb200_to_lavc_vid_conv_init.restype = _vp
    L.ugb200_to_lavc_vid_conv_init.argtypes = [_i, _i, _i, _i]
    L.ugb200_to_lavc_vid_conv.restype = _vp
    L.ugb200_to_lavc_vid_conv.argtypes = [_vp, _vp, _i]
    L.ugb200_to_lavc_vid_conv_destroy.argtypes = [_vp]
    L.ugb200_get_av_to_uv_conversion.restype = _vp
    L.ugb200_get_av_to_uv_conversion.argtypes = [_i, _i]
    L.ugb200_av_to_uv_convert.argtypes = [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]
    L.ugb200_av_to_uv_conversion_destroy.argtypes = [_vp]
    return L, torch


def to_lavc_pairs():
    """every (in_codec, av_pixfmt) ugb200_to_lavc_supported admits"""
    from ultragrid_b200 import _lib
    L = _lib.load()
    return [(c, AV_NAMES[f]) for c in range(1, 64) for f in range(1, len(AV_NAMES)) if L.ugb200_to_lavc_supported(c, f)]


def from_lavc_pairs():
    """every (av_pixfmt, out_codec) ugb200_get_av_to_uv_conversion accepts"""
    L, _ = lib_and_torch()
    out = []
    for f in range(1, len(AV_NAMES)):
        for c in range(1, 64):
            st = L.ugb200_get_av_to_uv_conversion(f, c)
            if st:
                out.append((AV_NAMES[f], c))
                h = _vp(st)
                L.ugb200_av_to_uv_conversion_destroy(ctypes.byref(h))
    return out


def gpu_to_lavc(L, torch, inc, fmt, src, w, h, lss, plane_off=0, src_off=0):
    """(rc, [host copies of guard + plane + guard]) of ugb200_to_lavc_convert into sentinel-filled device planes"""
    from ultragrid_b200.api import AvPlanes
    shapes, _ = av_geom(fmt, w, h)
    bufs = [torch.full((2 * GUARD + plane_off + ls * rows,), FILL, dtype=torch.uint8, device="cuda") for ls, (_, rows) in zip(lss, shapes)]
    p = AvPlanes()
    for i, (b, ls) in enumerate(zip(bufs, lss)):
        p.data[i], p.linesize[i] = b.data_ptr() + GUARD + plane_off, ls
    s = torch.from_numpy(np.concatenate([np.zeros(16 + src_off, np.uint8), src, np.zeros(64, np.uint8)])).cuda()
    rc = L.ugb200_to_lavc_convert(inc, AV[fmt], ctypes.byref(p), s.data_ptr() + 16 + src_off, w, h, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, [b.cpu().numpy() for b in bufs]


def assert_planes(got, want, plane_off, what):
    for i, (g, b) in enumerate(zip(got, want.buf)):
        body = g[GUARD + plane_off:GUARD + plane_off + b.size].reshape(b.shape)
        assert np.all(g[:GUARD + plane_off] == FILL) and np.all(g[GUARD + plane_off + b.size:] == FILL), (what, i, "guard band written")
        bad = np.argwhere(body != b)
        assert bad.size == 0, (what, i, "first differing (row, byte)", bad[:4].tolist(), "of", len(bad),
                               "got", body[tuple(bad[0])], "want", b[tuple(bad[0])], "written by the reference", want.wr[i][tuple(bad[0])])


# every width at an even and an odd height; widths below one v210 group (1, 2, 4, 5) over several row pairs
TO_SIZES = [(1, 1), (1, 2), (1, 7), (2, 2), (2, 3), (2, 5), (4, 4), (5, 5), (6, 3), (6, 4), (8, 1), (8, 2), (47, 5), (47, 4), (48, 4), (48, 3),
            (49, 3), (49, 2), (1922, 2), (1922, 3), (7680, 3), (7680, 2)]


def plane_modes(fmt, w, h):
    """(name, linesizes, pointer offset): tight, padded to 64, padded by an odd number of samples, and tight 2 bytes into a larger buffer"""
    shapes, bps = av_geom(fmt, w, h)
    tight = [n * bps for n, _ in shapes]
    return [("tight", tight, 0), ("pad64", [(t + 63) // 64 * 64 for t in tight], 0), ("odd", [t + 7 * bps for t in tight], 0), ("offset2", tight, 2)]


@pytest.mark.gpu
def test_gpu_to_lavc_pair_enumeration_covers_known_pairs():
    pairs = to_lavc_pairs()
    assert set(TO_PAIRS_KNOWN) | set(DELEGATED) == set(pairs), pairs


@pytest.mark.gpu
@pytest.mark.parametrize("inc,fmt", to_lavc_pairs() if _lib_built() else [])
def test_gpu_to_lavc_exact(orc, inc, fmt):
    """every pair the library admits == the numpy reference, byte for byte, sentinels included: sizes from 1 x 1 to 7680 wide, odd heights
    (4:2:0 too), four plane layouts, and a source misaligned by 2 bytes (v210 refuses one, see the test below)"""
    L, torch = lib_and_torch()
    for k, (w, h) in enumerate(TO_SIZES):
        src = make_source(inc, w, h, 500 + k)
        for name, lss, off in plane_modes(fmt, w, h):
            want = ref_to_lavc(inc, fmt, src, w, h, lss, orc)
            rc, got = gpu_to_lavc(L, torch, inc, fmt, src, w, h, lss, off)
            assert rc == 0, (w, h, name, rc)
            assert_planes(got, want, off, (w, h, name))
        if inc != V210:
            lss = plane_modes(fmt, w, h)[0][1]
            rc, got = gpu_to_lavc(L, torch, inc, fmt, src, w, h, lss, 0, src_off=2)
            assert rc == 0
            assert_planes(got, ref_to_lavc(inc, fmt, src, w, h, lss, orc), 0, (w, h, "source + 2"))


@pytest.mark.gpu
@pytest.mark.parametrize("inc,fmt", to_lavc_pairs() if _lib_built() else [])
def test_gpu_to_lavc_taller_than_grid(orc, inc, fmt):
    """a thin frame of 2 * 16384 + 3 rows: the y grid-stride loops take more than one turn"""
    L, torch = lib_and_torch()
    w, h = (12 if inc == V210 else 10), 2 * 16384 + 3
    src = make_source(inc, w, h, 9)
    lss = plane_modes(fmt, w, h)[1][1]
    rc, got = gpu_to_lavc(L, torch, inc, fmt, src, w, h, lss)
    assert rc == 0
    assert_planes(got, ref_to_lavc(inc, fmt, src, w, h, lss, orc), 0, "tall")


@pytest.mark.gpu
def test_gpu_to_lavc_refusals_write_nothing():
    """v210 from a source that is not 4-byte aligned (the reference asserts it, :199) and 16-bit planes at an odd line size or address (the
    reference asserts linesize % 2 == 0, :200-202) return -1 and leave every plane untouched"""
    L, torch = lib_and_torch()
    w, h = 48, 4
    src = make_source(V210, w, h, 1)
    for fmt in ("YUV420P10LE", "YUV422P10LE", "YUV444P10LE", "YUV444P16LE", "P010LE"):
        lss = plane_modes(fmt, w, h)[0][1]
        rc, got = gpu_to_lavc(L, torch, V210, fmt, src, w, h, lss, 0, src_off=2)
        assert rc == -1 and all(np.all(g == FILL) for g in got), fmt
        rc, got = gpu_to_lavc(L, torch, V210, fmt, src, w, h, [ls + 1 for ls in lss])
        assert rc == -1 and all(np.all(g == FILL) for g in got), fmt
        rc, got = gpu_to_lavc(L, torch, V210, fmt, src, w, h, lss, plane_off=1)
        assert rc == -1 and all(np.all(g == FILL) for g in got), fmt
    src = make_source(RG48, w, h, 2)
    lss = plane_modes("YUV444P16LE", w, h)[0][1]
    rc, got = gpu_to_lavc(L, torch, RG48, "YUV444P16LE", src, w, h, [ls + 1 for ls in lss])
    assert rc == -1 and all(np.all(g == FILL) for g in got)


@pytest.mark.gpu
@pytest.mark.parametrize("inc,fmt", to_lavc_pairs() if _lib_built() else [])
def test_gpu_to_lavc_hook_host_and_device_frame(orc, inc, fmt):
    """the hook shape (ugb200_to_lavc_vid_conv_*): a host frame and a device frame give the reference's samples in the state's planes"""
    from ultragrid_b200.api import AvPlanes
    L, torch = lib_and_torch()
    w, h = 97, 5
    st = L.ugb200_to_lavc_vid_conv_init(inc, w, h, AV[fmt])
    assert st
    try:
        src = make_source(inc, w, h, 3)
        dev = torch.from_numpy(src).cuda()
        for frame, is_dev in ((src.ctypes.data, 0), (dev.data_ptr(), 1)):
            pp = L.ugb200_to_lavc_vid_conv(st, frame, is_dev)
            assert pp, is_dev
            p = AvPlanes.from_address(pp)
            shapes, _ = av_geom(fmt, w, h)
            lss = [p.linesize[i] for i in range(len(shapes))]
            want = ref_to_lavc(inc, fmt, src, w, h, lss, orc)
            for i, (b, wr) in enumerate(zip(want.buf, want.wr)):
                host = np.zeros(b.size, np.uint8)
                assert L.cuda_wrapper_memcpy(ctypes.c_void_p(host.ctypes.data), ctypes.c_void_p(p.data[i]), host.size, 1) == 0
                assert np.array_equal(host.reshape(b.shape)[wr], b[wr]), (is_dev, i)
    finally:
        hs = _vp(st)
        L.ugb200_to_lavc_vid_conv_destroy(ctypes.byref(hs))
        assert not hs.value


# ---- 6. GPU: from_lavc --------------------------------------------------------------------------------------------------------------------
def gpu_from_lavc(L, torch, st, fmt, out, pl, w, h, pitch, shifts):
    """one ugb200_av_to_uv_convert with state `st` into a sentinel-filled frame; returns the frame rows (h x pitch) and the trailing guard"""
    from ultragrid_b200.api import AvPlanes
    dev = [torch.from_numpy(a.reshape(-1).copy()).cuda() for a, _ in pl]
    p = AvPlanes()
    for i, (t, (_, ls)) in enumerate(zip(dev, pl)):
        p.data[i], p.linesize[i] = t.data_ptr(), ls
    dst = torch.full((pitch * h + GUARD,), FILL, dtype=torch.uint8, device="cuda")
    sh = None if shifts is None else (_i * 3)(*shifts)
    rc = L.ugb200_av_to_uv_convert(st, dst.data_ptr(), ctypes.byref(p), w, h, pitch, sh, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0, (fmt, out, w, h, rc)
    d = dst.cpu().numpy()
    return d[:pitch * h].reshape(h, pitch), d[pitch * h:]


def assert_frame(got, guard, F, ls, what):
    assert np.all(guard == FILL), (what, "sentinel after the last row written")
    assert np.all(got[:, ls:] == FILL), (what, "bytes beyond the line size written")
    bad = np.argwhere((got != F.buf) & F.wr)
    assert bad.size == 0, (what, "first differing (row, byte)", bad[:4].tolist(), "of", len(bad), "got", got[tuple(bad[0])], "want",
                           F.buf[tuple(bad[0])])


FROM_SIZES = [(2, 2), (15, 3), (47, 5), (48, 4), (49, 1), (1922, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,out", from_lavc_pairs() if _lib_built() else [])
def test_gpu_from_lavc_exact(orc, fmt, out):
    """every pair ugb200_get_av_to_uv_conversion accepts == the reference entry of av_to_uv_conversions[] restated, or == the planar stage
    restated + the pinned line converter; pitch tight and larger than the line, odd widths and heights, rgb_shift NULL / RGB / BGR order"""
    from ultragrid_b200.codec import vc_get_linesize
    L, torch = lib_and_torch()
    shift_set = [None, (0, 8, 16), (16, 8, 0)] if out == RGBA else [None]
    st = L.ugb200_get_av_to_uv_conversion(AV[fmt], out)
    assert st
    try:
        for k, (w, h) in enumerate(FROM_SIZES):
            ls = vc_get_linesize(w, out)
            for pitch, pad in ((ls, 0), (ls + 52, 9)):
                pl = av_planes_in(fmt, w, h, 900 + k, pad)
                for shifts in shift_set:
                    F = ref_from_lavc(orc, fmt, out, pl, w, h, pitch, shifts or (0, 8, 16))
                    got, guard = gpu_from_lavc(L, torch, st, fmt, out, pl, w, h, pitch, shifts)
                    assert_frame(got, guard, F, ls, (w, h, pitch, shifts))
    finally:
        hs = _vp(st)
        L.ugb200_av_to_uv_conversion_destroy(ctypes.byref(hs))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,out", [("YUV422P", RGBA), ("YUV444P", RGB), ("YUV422P10LE", UYVY), ("GBRP", UYVY)])
def test_gpu_from_lavc_state_reused_small_large_small(orc, fmt, out):
    """one state converts a small, a large and again a small frame: the intermediate buffer of a two-stage route grows and is reused"""
    from ultragrid_b200.codec import vc_get_linesize
    L, torch = lib_and_torch()
    st = L.ugb200_get_av_to_uv_conversion(AV[fmt], out)
    assert st
    try:
        for k, (w, h) in enumerate([(14, 3), (1923, 7), (11, 5)]):
            pitch = vc_get_linesize(w, out)
            pl = av_planes_in(fmt, w, h, 40 + k)
            got, guard = gpu_from_lavc(L, torch, st, fmt, out, pl, w, h, pitch, None)
            assert_frame(got, guard, ref_from_lavc(orc, fmt, out, pl, w, h, pitch, (0, 8, 16)), pitch, (w, h))
    finally:
        hs = _vp(st)
        L.ugb200_av_to_uv_conversion_destroy(ctypes.byref(hs))


def test_yuv420p_to_v210_keeps_the_shifted_luma():
    """documents the one deliberate difference from a reference entry: the reference's yuv420p_to_v210 stores the luma of word 3 unshifted
    (:601-602); the pinned value is << 2, like yuv422p_to_v210 (:651) and the route UYVY -> v210"""
    w, h = 12, 2
    pl = av_planes_in("YUV420P", w, h, 3)
    a, b = Frame(h, 32), Frame(h, 32)
    fl_yuv420p_to_v210(pl, w, h, a)
    fl_yuv420p_to_v210(pl, w, h, b, quirk=True)
    words = lambda F: F.buf.view("<u4")  # noqa: E731
    diff = words(a) != words(b)
    assert diff[:, 3::4].all() and not diff[:, [0, 1, 2]].any()
    assert np.array_equal(words(a)[:, 3] & 0x3FF, pl[0][0][:, 4].astype(np.uint32) << 2)
