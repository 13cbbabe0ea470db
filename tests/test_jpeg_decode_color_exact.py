"""The decoder's colour-space outputs (ugb200_jpeg_decode_cs, ugb200_jpeg_decode_to) pinned to the exact IDCT and the float64 colour matrices,
with no C restatement in between.  test_jpeg_decode_color.py and test_jpeg_decode_yuv.py compare these outputs with C oracles written together
with the kernels, on a narrow corpus; test_jpeg_exact.py pins the native samples to the exact IDCT on a broad one.  This file joins the two:

  * a plain numpy reference of the header contract (include/ugb200_jpeg.h): the Q14 coefficients derived in float64 from kr, kb and the range
    scales with the C-cast rounding of csrc/color_space.h, YCBCR_TO_R/G/B with chroma replicated from its pair or quad, the three Q14 YCbCr ->
    YCbCr formulas at the stream's own sampling, and the UYVY / I420 / VUYA / RGB / RGBA packings;
  * check A (exact): every colour output == that reference applied to the same decoder's native samples (decode_to NATIVE -> NATIVE into the
    lossless output), which in the same test equal clamp(round(exact IDCT)) outside the tie band (check_decoded);
  * check B (float64 bound): every output within a derived bound of the unrounded matrix applied to the clamped exact IDCT (see b_bound);
  * the corpus: every YCbCr stream of test_jpeg_exact.decoder_corpus, libjpeg's streams, grayscale with and without DRI, saturated and
    half-integer writer streams, each declared colour space, odd sizes up to 1921 x 1081, every Huffman route and marker scan, host and pitched
    device destinations, 4K and 8K (check A), and the decompress modules end to end on a stream without DRI;
  * on the CPU: the coefficient pins, the reference's self-checks, and mutants that A and B must report."""
import ctypes
import os
import re

import numpy as np
import pytest

import jpeg_exact as J
import util
from test_jpeg import RGB, UYVY, natural_rgb
from test_jpeg_alpha import al  # noqa: F401  (fixture: the alpha oracle, for decoder_corpus)
from test_jpeg_decode_color import JFIF, adobe, spiff, strip_app0, with_markers
from test_jpeg_decode_yuv import gray_image, gray_stream, i420_of_uyvy, matrices
from test_jpeg_exact import STD_TABLES, check_decoded, decoder_corpus, exact_planes, pil_stream
from test_jpeg_planar import pl  # noqa: F401  (fixture: the planar oracle, for decoder_corpus)

RGBA, VUYA, I420, DXT1, JPEG = 1, 4, 29, 9, 13
NATIVE, AUTO = 0, 5
SPACES = ["Y601", "Y601full", "Y709"]
CS = {"Y601": 1, "Y601full": 2, "Y709": 3}
PAIRS = [(a, b) for a in SPACES for b in SPACES if a != b]
SHIFTS = [None, (0, 8, 16), (16, 8, 0), (8, 16, 24)]  # None: RGB, else RGBA with these shifts
HERE = os.path.dirname(os.path.abspath(__file__))
COLOR_SPACE_H = os.path.join(os.path.dirname(HERE), "ultragrid_b200", "csrc", "color_space.h")
Q14_ERR = 0.5 / 16384 * (255 + 128 + 128)  # each Q14 coefficient off by at most 1/2 LSB, times the largest |Y - o|, |Cb - 128|, |Cr - 128|


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


# ---- 1. coefficients: compute_color_coeffs and compute_ycc_matrix of csrc/color_space.h, restated in float64 -----------------------------
KR_KB = {"Y709": (.212639, .072192), "Y601": (.299, .114), "Y601full": (.299, .114)}
DEPTH = {"Y709": 8, "Y601": 8, "Y601full": 0}
OFFSET = {"Y709": 16, "Y601": 16, "Y601full": 0}
RGB_FIELDS = ["y_r", "y_g", "y_b", "cb_r", "cb_g", "cb_b", "cr_r", "cr_g", "cr_b", "y_scale", "r_cr", "g_cb", "g_cr", "b_cb"]


def _y_limit(d):
    return 1.0 if d == 0 else 219. * (1 << (d - 8)) / ((1 << d) - 1)


def _c_limit(d):
    return 1.0 if d == 0 else 224. * (1 << (d - 8)) / ((1 << d) - 1)


def _scaled(x):
    """color_space.c:104-105: (int) (x * 2^14 +- 0.5), the C cast truncating toward zero"""
    return int(x * 16384 + (1. if x > 0 else -1.) * 0.5)


def color_coeffs(kr, kb, depth):
    """compute_color_coeffs: the RGB -> YCbCr rows and the YCbCr -> RGB inverse, as a dict of RGB_FIELDS"""
    kg, B = 1. - kr - kb, 16384.
    dd, ee = 2. * (kr + kg), 2. * (1. - kr)
    yl, cl = _y_limit(depth), _c_limit(depth)
    v = [int(kr * yl * B + 0.5), int(kg * yl * B + 0.5), int(kb * yl * B + 0.5),
         int(-kr / dd * cl * B - 0.5), int(-kg / dd * cl * B - 0.5), int((1 - kb) / dd * cl * B + 0.5),
         int((1 - kr) / ee * cl * B - 0.5), int(-kg / ee * cl * B - 0.5), int(-kb / ee * cl * B + 0.5),
         _scaled(1. / yl), _scaled((2. * (1. - kr)) / cl), _scaled((-kb * (2. * (kr + kg)) / kg) / cl), _scaled((-kr * (2. * (1. - kr)) / kg) / cl),
         _scaled((2. * (kr + kg)) / cl)]
    return dict(zip(RGB_FIELDS, v))


def rgb_coeffs(cs):
    """(y_scale, r_cr, g_cb, g_cr, b_cb, luma offset) of YCBCR_TO_R/G/B in the colour space: coeffs_709(8), coeffs_601(8), coeffs_601(0)"""
    c = color_coeffs(*KR_KB[cs], DEPTH[cs])
    return c["y_scale"], c["r_cr"], c["g_cb"], c["g_cr"], c["b_cb"], OFFSET[cs]


def ycc_coeffs(a, b):
    """compute_ycc_matrix from space a to space b: (yy, yb, yr, bb, br, rb, rr, o_in, o_out)"""
    (krs, kbs), ds, (krt, kbt), dt = KR_KB[a], DEPTH[a], KR_KB[b], DEPTH[b]
    ys, cs, kgs = 1. / _y_limit(ds), 1. / _c_limit(ds), 1. - krs - kbs
    dd = lambda kr, kb: 2. * (kr + (1. - kr - kb))
    r = [ys, 0., 2. * (1. - krs) * cs]
    g = [ys, -kbs * dd(krs, kbs) / kgs * cs, -krs * 2. * (1. - krs) / kgs * cs]
    bl = [ys, dd(krs, kbs) * cs, 0.]
    kgt = 1. - krt - kbt
    lum = [krt * r[i] + kgt * g[i] + kbt * bl[i] for i in range(3)]
    yt, cb, cr = _y_limit(dt), _c_limit(dt) / dd(krt, kbt), _c_limit(dt) / (2. * (1. - krt))
    return (_scaled(yt * lum[0]), _scaled(yt * lum[1]), _scaled(yt * lum[2]), _scaled(cb * (bl[1] - lum[1])), _scaled(cb * (bl[2] - lum[2])),
            _scaled(cr * (r[1] - lum[1])), _scaled(cr * (r[2] - lum[2])), OFFSET[a], OFFSET[b])


def ycc_matrix(a, b):
    """the unrounded float64 matrix over (Y - o_in, Cb - 128, Cr - 128): RGB -> YCbCr of b after YCbCr -> RGB of a"""
    return matrices(b)[0] @ matrices(a)[1]


def pinned_values():
    """the static_assert-pinned values of csrc/color_space.h: {depth: {field: value}} of coeffs_709 and {(cs_in, cs_out): 9 values} of
    ycc_matrix_between, read from the header itself"""
    src = open(COLOR_SPACE_H).read()
    depth_of = {n: int(d) for n, d in re.findall(r"\b(c\d+) = coeffs_709\((\d+)\)", src)}
    rgb = {}
    for n, f, v in re.findall(r"\b(c\d+)\.(\w+) == (-?\d+)", src):
        rgb.setdefault(depth_of[n], {})[f] = int(v)
    ycc = {(int(a), int(b)): [int(x) for x in vals.split(",")]
           for a, b, vals in re.findall(r"ycc_is\(ycc_matrix_between\((\d), (\d)\),([-\d, ]+)\)", src)}
    return rgb, ycc


# ---- the reference: samples -> colour outputs -------------------------------------------------------------------------------------------
def _chroma_at(c, n_rows, n_cols, sampling):
    """a chroma plane read at every luma position: the sample of the pixel's pair (4:2:2) or quad (4:2:0), no interpolation"""
    hs, vs = sampling
    return np.asarray(c)[np.arange(n_rows) // vs][:, np.arange(n_cols) // hs]


def rgb(planes, cs, sampling, w, shifts=None):
    """RGB (shifts None) or RGBA rows of decode_cs(cs): YCBCR_TO_R/G/B with `>>` a floor, clamped; only whole pixel pairs of a 4:2:2 / 4:2:0 row;
    RGBA places R, G, B at the shifts and sets every other bit.  planes: (Y, Cb, Cr) integer samples on the stream's grids."""
    ys, rc, gcb, gcr, bcb, o = rgb_coeffs(cs)
    n = w if sampling[0] == 1 else w // 2 * 2
    Y = np.asarray(planes[0])[:, :n].astype(np.int32)
    cb = _chroma_at(planes[1], Y.shape[0], n, sampling).astype(np.int32) - 128
    cr = _chroma_at(planes[2], Y.shape[0], n, sampling).astype(np.int32) - 128
    yy = ys * (Y - o)
    r, g, b = [np.clip(v >> 14, 0, 255).astype(np.uint32) for v in (yy + rc * cr, yy + gcb * cb + gcr * cr, yy + bcb * cb)]
    if shifts is None:
        return np.stack([r, g, b], 2).astype(np.uint8).reshape(Y.shape[0], -1)
    rs, gs, bs = (np.uint32(s) for s in shifts)
    rest = np.uint32(0xFFFFFFFF) ^ (np.uint32(255) << rs) ^ (np.uint32(255) << gs) ^ (np.uint32(255) << bs)
    v = np.ascontiguousarray(rest | (r << rs) | (g << gs) | (b << bs), "<u4")
    return v.view(np.uint8).reshape(Y.shape[0], -1)


def ycc(planes, a, b, sampling, rnd=8192):
    """decode_to's conversion from a to b at the stream's own sampling: Y' per luma sample with the chroma of its pair / quad, Cb' and Cr' per
    chroma sample (rnd: the rounding term, a parameter only so that a mutant can drop it)"""
    yy, yb, yr, bb, br, rb, rr, oi, oo = ycc_coeffs(a, b)
    Y = np.asarray(planes[0]).astype(np.int32)
    cb0, cr0 = (np.asarray(p).astype(np.int32) - 128 for p in planes[1:])
    cb, cr = _chroma_at(cb0, *Y.shape, sampling), _chroma_at(cr0, *Y.shape, sampling)
    clip = lambda v: np.clip(v, 0, 255).astype(np.uint8)
    return (clip(((yy * (Y - oi) + yb * cb + yr * cr + rnd) >> 14) + oo), clip(((bb * cb0 + br * cr0 + rnd) >> 14) + 128),
            clip(((rb * cb0 + rr * cr0 + rnd) >> 14) + 128))


def uyvy(planes, w, h, sampling):
    """UYVY of 4:2:2 / 4:2:0 / grayscale samples: a row of (w + 1) / 2 pairs, the chroma row y / V; the last pair of an odd width takes the
    luma sample past the width (the padded plane's, which the native UYVY holds)"""
    pairs = (w + 1) // 2
    Y = np.asarray(planes[0])
    assert Y.shape[1] >= 2 * pairs, "an odd width needs the luma sample past the width"
    rows = np.arange(h) // sampling[1]
    out = np.empty((h, pairs, 4), np.uint8)
    out[:, :, 0], out[:, :, 1] = np.asarray(planes[1])[rows, :pairs], Y[:h, 0:2 * pairs:2]
    out[:, :, 2], out[:, :, 3] = np.asarray(planes[2])[rows, :pairs], Y[:h, 1:2 * pairs:2]
    return out.reshape(h, -1)


def vuya(planes, w, h):
    Y, cb, cr = (np.asarray(p)[:h, :w] for p in planes)
    return np.stack([cr, cb, Y, np.full_like(Y, 255)], 2).reshape(h, -1)


def pack(planes, case, out_c):
    """the bytes of out_c for samples of the case's sampling: UYVY, I420 (uyvy_to_i420 of the UYVY: a 4:2:2 stream's chroma rows averaged
    (a + b + 1) >> 1, a 4:2:0 stream's chroma as it is) and, for 4:4:4 streams, VUYA; a 4:4:4 stream's UYVY and I420 need the VUYA -> UYVY line
    converter (pack_444, on the GPU)"""
    w, h = case.w, case.h
    if case.sampling[0] == 1:
        assert out_c == VUYA
        return vuya(planes, w, h).reshape(-1)
    u = uyvy(planes, w, h, case.sampling)
    if out_c == UYVY:
        return u.reshape(-1)
    assert out_c == I420
    return i420_of_uyvy(u, w, h)


def pack_444(planes, case, out_c):
    """UYVY / I420 of a 4:4:4 stream: its VUYA through the VUYA -> UYVY line converter (ugb200_pixfmt_convert, pinned to the reference by the
    pixfmt tests), as ugb200_jpeg_decode does"""
    import torch
    from ultragrid_b200 import Codec, api
    v = vuya(planes, case.w, case.h).reshape(-1)
    if out_c == VUYA:
        return v
    u = api.pixfmt_convert(Codec.VUYA, Codec.UYVY, torch.from_numpy(v.copy()).cuda(), case.w, case.h).cpu().numpy()
    return u if out_c == UYVY else i420_of_uyvy(u.reshape(case.h, -1), case.w, case.h)


def expected(planes, case, out_c):
    return pack_444(planes, case, out_c) if case.sampling[0] == 1 else pack(planes, case, out_c)


def check_a(got, want, what):
    """check A: byte for byte"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        i = tuple(int(v) for v in np.argwhere(got != want)[0])
        raise AssertionError(f"{what}: {int((got != want).sum())} bytes differ from the reference; first at {i}: got {got[i]}, want {want[i]}")


# ---- check B: the unrounded matrix on the clamped exact IDCT ---------------------------------------------------------------------------
def b_bound(m, bands, floor):
    """per output value: sum_j |m_ij| (1/2 + band_j) + the integer formula's own error.
    Derivation.  A decoded sample s_j is clamp(round(x_j)) of its exact IDCT value x_j, or one step away where x_j lies within band_j of a
    half-integer (jpeg_exact.py), so |s_j - clamp(x_j)| <= 1/2 + band_j (clamp is 1-Lipschitz).  The matrix row m_i carries that to at most
    sum_j |m_ij| (1/2 + band_j).  The integer formula applies round(2^14 m_ij) instead of m_ij: each off by at most 2^-15, times |Y - o| <= 255,
    |Cb - 128|, |Cr - 128| <= 128: Q14_ERR = 0.0156.  It then rounds to nearest (YCbCr -> YCbCr, + 8192 >> 14: 1/2, so 0.516 in all) or floors
    (YCbCr -> RGB, >> 14: below 1, so 1.016).  The final clamp to 0..255 is 1-Lipschitz again, so the output lies within the bound of
    clamp(m_i (clamp(x) - offsets) + offset, 0, 255)."""
    return sum(abs(m[j]) * (0.5 + bands[j]) for j in range(3)) + Q14_ERR + (1.0 if floor else 0.5)


def b_compare(channels, what, stats=None):
    """channels: [(name, got, exact, bound, bound without the band)]; raises when |got - exact| exceeds the bound.  Counts the values that need
    the band (beyond the band-free bound) and the worst excess |got - exact| - bound (negative: inside)"""
    for name, got, ex, bound, bound0 in channels:
        d = np.abs(np.asarray(got, np.float64) - ex)
        bad = d > bound
        if bad.any():
            i = tuple(int(v) for v in np.argwhere(bad)[0])
            raise AssertionError(f"{what} {name}: {int(bad.sum())} values beyond the float64 bound; first at {i}: got {np.asarray(got)[i]}, "
                                 f"exact {ex[i]!r}, bound {np.broadcast_to(bound, d.shape)[i]:.3f}")
        if stats is not None:
            stats["n"] += d.size
            stats["banded"] += int((d > bound0).sum())
            stats["worst"] = max(stats["worst"], float((d - bound).max()) if d.size else -9.0)


def exact_ycc(case):
    """clamp(exact IDCT) and the tie band of every sample on the stream's grids (grayscale: Cb = Cr = 128, band 0)"""
    ex = case.exact()
    Y, bY = np.clip(ex[0][0], 0, 255), ex[0][1]
    if len(ex) == 1:
        c = np.full((case.h, (case.w + 1) // 2), 128.0)
        return (Y, bY), (c, np.zeros_like(c)), (c, np.zeros_like(c))
    return (Y, bY), (np.clip(ex[1][0], 0, 255), ex[1][1]), (np.clip(ex[2][0], 0, 255), ex[2][1])


def b_channels_rgb(out, case, cs, shifts):
    """(name, got, exact, bound, bound0) of R, G, B of an RGB / RGBA output against the inverse matrix of cs on the clamped exact samples"""
    (Y, bY), (Cb, bCb), (Cr, bCr) = exact_ycc(case)
    inv, o = matrices(cs)[1], OFFSET[cs]
    h, w = case.h, case.w
    n = w if case.sampling[0] == 1 else w // 2 * 2
    v = [Y[:, :n] - o, _chroma_at(Cb, h, n, case.sampling) - 128, _chroma_at(Cr, h, n, case.sampling) - 128]
    bands = [bY[:, :n], _chroma_at(bCb, h, n, case.sampling), _chroma_at(bCr, h, n, case.sampling)]
    bpp = 3 if shifts is None else 4
    px = np.asarray(out).reshape(h, -1)[:, :n * bpp].reshape(h, n, bpp)
    if shifts is None:
        got = [px[:, :, k] for k in range(3)]
    else:
        word = px.astype(np.uint32) << (8 * np.arange(4, dtype=np.uint32))
        word = word.sum(2, dtype=np.uint32)
        got = [(word >> np.uint32(s)) & np.uint32(255) for s in shifts]
    out_ch = []
    for i, name in enumerate("RGB"):
        ex = np.clip(inv[i, 0] * v[0] + inv[i, 1] * v[1] + inv[i, 2] * v[2], 0, 255)
        out_ch.append((name, got[i], ex, b_bound(inv[i], bands, True), b_bound(inv[i], [0, 0, 0], True)))
    return out_ch


def b_channels_ycc(out, out_c, case, a, b):
    """(name, got, exact, bound, bound0) of Y', Cb', Cr' of a UYVY (4:2:x, grayscale) or VUYA (4:4:4) output of decode_to(a -> b)"""
    (Y, bY), (Cb, bCb), (Cr, bCr) = exact_ycc(case)
    m = ycc_matrix(a, b)
    oi, oo = OFFSET[a], OFFSET[b]
    h, w = case.h, case.w
    if out_c == VUYA:
        p = np.asarray(out).reshape(h, w, 4)
        gy, gcb, gcr, crow = p[:, :, 2], p[:, :, 1], p[:, :, 0], np.arange(h)
    else:
        gy, gcb, gcr = J.uyvy_planes(out, w, h)
        crow = np.arange(h) // case.sampling[1]
    cy = [Y[:h, :w] - oi, _chroma_at(Cb, h, w, case.sampling) - 128, _chroma_at(Cr, h, w, case.sampling) - 128]
    by = [bY[:h, :w], _chroma_at(bCb, h, w, case.sampling), _chroma_at(bCr, h, w, case.sampling)]
    cw = gcb.shape[1]
    cc = [None, Cb[crow][:, :cw] - 128, Cr[crow][:, :cw] - 128]
    bc = [np.zeros(1), bCb[crow][:, :cw], bCr[crow][:, :cw]]
    exy = np.clip(m[0, 0] * cy[0] + m[0, 1] * cy[1] + m[0, 2] * cy[2] + oo, 0, 255)
    # the target's chroma does not depend on the source's luma (|m[1:, 0]| < 1e-12, test_jpeg_decode_yuv.py): the luma term is left out
    exb = np.clip(m[1, 1] * cc[1] + m[1, 2] * cc[2] + 128, 0, 255)
    exr = np.clip(m[2, 1] * cc[1] + m[2, 2] * cc[2] + 128, 0, 255)
    mb, mr = np.array([0., m[1, 1], m[1, 2]]), np.array([0., m[2, 1], m[2, 2]])
    return [("Y'", gy, exy, b_bound(m[0], by, False), b_bound(m[0], [0, 0, 0], False)),
            ("Cb'", gcb, exb, b_bound(mb, bc, False), b_bound(mb, [0, 0, 0], False)),
            ("Cr'", gcr, exr, b_bound(mr, bc, False), b_bound(mr, [0, 0, 0], False))]


# ---- 3. corpus -------------------------------------------------------------------------------------------------------------------------
class Case:
    """a YCbCr or grayscale stream: name, bytes, size, sampling (H, V of luma; grayscale as 4:2:2 with Cb = Cr = 128), the space it declares,
    and its exact IDCT (computed once)"""

    def __init__(self, name, stream):
        self.name, self.stream = name, stream
        self.fr = J.read(stream)
        self.w, self.h = self.fr.w, self.fr.h
        self.gray = len(self.fr.components) == 1
        c0 = self.fr.components[0]
        self.sampling = (2, 1) if self.gray else (c0["h"], c0["v"])
        self._exact = None

    def exact(self):
        if self._exact is None:
            self._exact = exact_planes(self.fr)
        return self._exact

    def declared(self):
        from ultragrid_b200 import api
        return api.jpeg_stream_color_space(self.stream)


DECLARED = [("bare", None, "Y709"), ("jfif", JFIF, "Y601full"), ("spiff1", spiff(1), "Y709"), ("spiff3", spiff(3), "Y601full"),
            ("spiff4", spiff(4), "Y601"), ("spiff8", spiff(8), "Y601full"), ("adobe1", adobe(1), "Y601full")]


def declared_variants(name, s, gray):
    """the stream without its APP0, then with each declared space in front: (name, stream, the space AUTO must resolve to); SPIFF 8 (grayscale)
    only on one-component streams"""
    bare = strip_app0(s) if s[2:4] == b"\xff\xe0" else s
    return [(f"{name} {k}", bare if m is None else with_markers(bare, [m]), want) for k, m, want in DECLARED if k != "spiff8" or gray]


def saturated(hs, vs, il, seed):
    """YCbCr with flat blocks at the extremes: per MCU the DCs of Y, Cb and Cr run through every corner of {0, 255}^3 (DC +-127, +-150 at Q = 8:
    samples 1, 255 and clamped beyond), small AC on top; 93 x 45, restart interval 5, which leaves a partial last interval in every scan"""
    w, h, ri = 93, 45, 5
    rng = np.random.default_rng(seed)
    mw, mh = -(-w // (8 * hs)), -(-h // (8 * vs))
    m = np.arange(mh * mw).reshape(mh, mw)
    ext = lambda bit: np.where(bit, rng.choice([127, 150], bit.shape), rng.choice([-127, -150], bit.shape))
    dc = [np.repeat(np.repeat(ext((m >> 2) & 1), vs, 0), hs, 1), ext(m & 1), ext((m >> 1) & 1)]
    coef = []
    for c in range(3):
        a = np.zeros(dc[c].shape + (64,), np.int64)
        a[..., 0] = dc[c]
        a[..., 1], a[..., 8] = rng.integers(-5, 6, dc[c].shape), rng.integers(-5, 6, dc[c].shape)
        coef.append(a)
    comps = [(1, hs, vs, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
    scans = [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]] if il else [[(0, 0, 0)], [(1, 1, 1)], [(2, 1, 1)]]
    return J.write(w, h, comps, coef, {0: np.full(64, 8), 1: np.full(64, 8)}, STD_TABLES, scans, ri=ri)


def dc_half_420():
    """4:2:0 YCbCr, DC only at Q = 4 with odd DC: every sample an exact half-integer (128 + DC / 2), rounded either way by float32"""
    w, h = 37, 21
    rng = np.random.default_rng(21)
    coef = [np.zeros((4, 6, 64), np.int64), np.zeros((2, 3, 64), np.int64), np.zeros((2, 3, 64), np.int64)]
    for c in coef:
        c[..., 0] = rng.integers(-120, 120, c.shape[:2]) * 2 + 1
    return J.write(w, h, [(1, 2, 2, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef, {0: np.full(64, 4), 1: np.full(64, 4)}, STD_TABLES,
                   [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]])


def gray_2x2_dri3():
    """one component that declares 2 x 2 sampling (ignored, T.81 A.2.2), restart interval 3"""
    w, h = 41, 17
    rng = np.random.default_rng(5)
    coef = np.zeros((3, 6, 64), np.int64)
    coef[..., 0] = rng.integers(-300, 300, (3, 6))
    for k in range(1, 20):
        coef[..., J.ZIGZAG[k]] = rng.integers(-20, 21, (3, 6))
    return J.write(w, h, [(1, 2, 2, 0)], [coef], {0: J.scaled_qtable(J.Q_LUMA, 80)}, {(0, 0): J.DC_LUMA, (1, 0): J.AC_LUMA}, [[(0, 0, 0)]], ri=3)


def new_streams():
    """the writer streams of this file, grayscale, the declared spaces and the size sweep: (name, stream)"""
    out = [(f"sat-{'422' if vs == 1 else '420'}-{'il' if il else 'pc'}", saturated(2, vs, il, 10 * vs + il)) for vs in (1, 2) for il in (0, 1)]
    out += [("dc-half-420", dc_half_420()), ("gray-2x2-dri3", gray_2x2_dri3())]
    out += [(f"pil-L {w}x{h} ri{ri}", gray_stream(gray_image(w, h), 90, ri)) for (w, h), ri in (((41, 17), 0), ((63, 40), 3), ((24, 31), 1))]
    for name, s, gray in (("pil-420", pil_stream("420", 63, 40), False), ("pil-422", pil_stream("422", 41, 17), False),
                          ("pil-444", pil_stream("444", 17, 24), False), ("pil-L", gray_stream(gray_image(24, 31), 85), True)):
        out += [(n, v) for n, v, _ in declared_variants(name, s, gray)]
    for w, h in ((1, 1), (2, 1)):
        out += [(f"pil-{k} {w}x{h}", pil_stream(k, w, h)) for k in ("420", "422", "444")] + [(f"pil-L {w}x{h}", gray_stream(gray_image(w, h), 90))]
    out += [("pil-420 1921x1081", pil_stream("420", 1921, 1081)), ("pil-422-rst 1921x1081", pil_stream("422-rst-blocks", 1921, 1081))]
    return out


def is_ycc(s):
    from ultragrid_b200 import api
    return api.jpeg_image_info(s).native_codec not in (RGB, RGBA)


@pytest.fixture(scope="module")
def corpus(orc, pl, al):  # noqa: F811
    """every YCbCr member of decoder_corpus (this encoder's layouts, libjpeg's PIL_CASES, the YCbCr writer streams) and new_streams()"""
    return [Case(n, s) for n, s in decoder_corpus(orc, pl, al) + new_streams() if is_ycc(s)]


# ---- CPU: the coefficients ---------------------------------------------------------------------------------------------------------
def test_coefficients_are_the_pinned_ones():
    """the float64 derivation with the C-cast rounding gives the static_assert-pinned values of csrc/color_space.h (coeffs_709 at depths 8,
    10, 16 and full range; ycc_matrix_between of the pinned pairs), and the reference's get_color_coeffs for all three spaces where it is built"""
    rgb_pin, ycc_pin = pinned_values()
    assert sorted(rgb_pin) == [0, 8, 10, 16] and len(ycc_pin) == 7
    for depth, fields in rgb_pin.items():
        mine = color_coeffs(*KR_KB["Y709"], depth)
        assert sorted(fields) == sorted(RGB_FIELDS)
        assert {f: mine[f] for f in fields} == fields, depth
    name = {1: "Y601", 2: "Y601full", 3: "Y709"}
    for (a, b), vals in ycc_pin.items():
        assert list(ycc_coeffs(name[a], name[b])) == vals, (a, b)
    ref = util.ref_cpu()
    if ref is None:
        return
    for cs, which in (("Y709", 2), ("Y601", 1), ("Y601full", 1)):  # enum colorspace: CS_601 = 1, CS_709 = 2
        c = (ctypes.c_int * 14)()
        ref.ref_get_color_coeffs(which, DEPTH[cs], c)
        assert list(c) == [color_coeffs(*KR_KB[cs], DEPTH[cs])[f] for f in RGB_FIELDS], cs


@pytest.mark.parametrize("a", SPACES)
def test_coefficients_are_the_rounded_matrices(a):
    """each Q14 coefficient is the nearest integer to 2^14 times the float64 matrix formed independently (numpy inversion of the forward
    matrix of matrices()): the inverse rows for RGB, the product for every ordered pair; an equal pair is the identity"""
    inv = matrices(a)[1]
    ys, rc, gcb, gcr, bcb, o = rgb_coeffs(a)
    for q, x in ((ys, inv[0, 0]), (ys, inv[1, 0]), (ys, inv[2, 0]), (rc, inv[0, 2]), (gcb, inv[1, 1]), (gcr, inv[1, 2]), (bcb, inv[2, 1])):
        assert abs(q - 16384 * x) <= 0.5 + 1e-6, (a, q, 16384 * x)
    assert abs(inv[0, 1]) < 1e-12 and abs(inv[2, 2]) < 1e-12 and o == matrices(a)[2]
    for b in SPACES:
        m, c = ycc_matrix(a, b), ycc_coeffs(a, b)
        want = [m[0, 0], m[0, 1], m[0, 2], m[1, 1], m[1, 2], m[2, 1], m[2, 2]]
        assert all(abs(q - 16384 * x) <= 0.5 + 1e-6 for q, x in zip(c[:7], want)), (a, b, c, want)
        if a == b:
            assert list(c[:7]) == [16384, 0, 0, 16384, 0, 0, 16384]


# ---- CPU: the reference checks itself ------------------------------------------------------------------------------------------------
def _triples():
    y, cb, cr = [v.reshape(-1) for v in np.meshgrid(np.arange(256), np.arange(0, 256, 3), np.arange(0, 256, 5), indexing="ij")]
    return y, cb, cr


@pytest.mark.parametrize("cs", SPACES)
def test_reference_rgb_is_the_matrix(cs):
    """rgb() over a grid of (Y, Cb, Cr) triples (one pixel pair each, 4:2:2): within the floor's 1 + Q14_ERR below the unrounded inverse matrix,
    never above it by more than Q14_ERR; RGBA carries the same bytes at every shift with every other bit set"""
    y, cb, cr = _triples()
    planes = (np.repeat(y, 2)[None, :], cb[None, :], cr[None, :])
    got = rgb(planes, cs, (2, 1), 2 * len(y)).reshape(-1, 3)[0::2].astype(np.float64)
    inv, o = matrices(cs)[1], OFFSET[cs]
    ex = np.clip(np.stack([y - o, cb - 128, cr - 128], 1) @ inv.T, 0, 255)
    d = got - ex
    assert d.max() <= Q14_ERR and d.min() >= -1 - Q14_ERR, (d.min(), d.max())
    want = rgb(planes, cs, (2, 1), 2 * len(y)).reshape(-1, 3)
    for sh in SHIFTS[1:]:
        v = rgb(planes, cs, (2, 1), 2 * len(y), sh).reshape(-1, 4).astype(np.uint32)
        word = v[:, 0] | v[:, 1] << 8 | v[:, 2] << 16 | v[:, 3] << 24
        for k, s in enumerate(sh):
            assert np.array_equal((word >> s) & 255, want[:, k]), sh
        assert ((word | (255 << sh[0]) | (255 << sh[1]) | (255 << sh[2])) == 0xFFFFFFFF).all(), sh


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{p[0]}-{p[1]}")
def test_reference_ycc_is_the_matrix(pair):
    """ycc() over a grid of triples at 4:4:4: within 0.5 + Q14_ERR of the unrounded matrix wherever that lies inside 0..255 (the clamp
    elsewhere); the equal pair leaves every sample as it is"""
    a, b = pair
    y, cb, cr = _triples()
    got = np.stack([p.reshape(-1) for p in ycc((y[None, :], cb[None, :], cr[None, :]), a, b, (1, 1))], 1).astype(np.float64)
    m = ycc_matrix(a, b)
    ex = np.stack([y - OFFSET[a], cb - 128, cr - 128], 1) @ m.T + np.array([OFFSET[b], 128, 128])
    assert np.abs(got - np.clip(ex, 0, 255)).max() <= 0.5 + Q14_ERR
    same = ycc((y[None, :], cb[None, :], cr[None, :]), a, a, (1, 1))
    assert all(np.array_equal(s.reshape(-1), v) for s, v in zip(same, (y, cb, cr)))


def test_reference_packing():
    """UYVY / I420 / VUYA of known planes: J.uyvy_planes reads the UYVY back; I420 of a 4:2:0 stream is its planes; grayscale packs 128 chroma
    and converts its luma alone"""
    rng = np.random.default_rng(3)
    w, h = 7, 5
    Y = rng.integers(0, 256, (h, 8)).astype(np.uint8)
    cb, cr = rng.integers(0, 256, (3, 4)).astype(np.uint8), rng.integers(0, 256, (3, 4)).astype(np.uint8)

    class C:
        pass
    c = C()
    c.w, c.h, c.sampling = w, h, (2, 2)
    u = uyvy((Y, cb, cr), w, h, (2, 2))
    gy, gb, gr = J.uyvy_planes(u.reshape(-1), w, h)
    assert np.array_equal(gy, Y[:, :w]) and np.array_equal(gb, cb[np.arange(h) // 2]) and np.array_equal(gr, cr[np.arange(h) // 2])
    assert np.array_equal(u.reshape(h, 4, 4)[:, -1, 3], Y[:, 7])  # the luma sample past an odd width
    i = J.i420_planes(pack((Y, cb, cr), c, I420), w, h)
    assert np.array_equal(i[0], Y[:, :w]) and np.array_equal(i[1], cb) and np.array_equal(i[2], cr)
    c.sampling = (1, 1)
    v = pack((Y[:, :w], Y[:, :w] // 2, Y[:, :w] // 3), c, VUYA).reshape(h, w, 4)
    assert np.array_equal(v[:, :, 2], Y[:, :w]) and np.array_equal(v[:, :, 1], Y[:, :w] // 2) and np.array_equal(v[:, :, 0], Y[:, :w] // 3) and (v[:, :, 3] == 255).all()
    g = np.full((h, 4), 128, np.uint8)
    cy, cb2, cr2 = ycc((Y, g, g), "Y601full", "Y709", (2, 1))
    assert (cb2 == 128).all() and (cr2 == 128).all() and np.array_equal(cy, ((14071 * Y.astype(np.int32) + 8192) >> 14) + 16)
    assert np.array_equal(rgb((Y, g, g), "Y601full", (2, 1), w).reshape(h, -1, 3)[:, :, 1], Y[:, : w // 2 * 2])  # full range: R = G = B = Y


def test_saturated_streams_reach_every_clamp():
    """on the saturated writer streams the unrounded matrices leave 0..255 at both ends in every channel: R, G, B in each space, and Y', Cb', Cr'
    over the six pairs - so the corpus reaches every clamp of both conversions"""
    for vs in (1, 2):
        case = Case("sat", saturated(2, vs, 1, 3))
        (Y, _), (Cb, _), (Cr, _) = exact_ycc(case)
        assert Y.min() == 0 and Y.max() == 255 and Cb.min() == 0 and Cb.max() == 255
        cb, cr = _chroma_at(Cb, *Y.shape, case.sampling) - 128, _chroma_at(Cr, *Y.shape, case.sampling) - 128
        for cs in SPACES:
            raw = np.stack([Y - OFFSET[cs], cb, cr], -1) @ matrices(cs)[1].T
            assert (raw.min((0, 1)) < 0).all() and (raw.max((0, 1)) > 255).all(), cs
        lo, hi = np.zeros(3, bool), np.zeros(3, bool)
        for a, b in PAIRS:
            raw = np.stack([Y - OFFSET[a], cb, cr], -1) @ ycc_matrix(a, b).T + np.array([OFFSET[b], 128, 128])
            lo |= raw.min((0, 1)) < 0
            hi |= raw.max((0, 1)) > 255
        assert lo.all() and hi.all(), (lo, hi)


# ---- 5. teeth ---------------------------------------------------------------------------------------------------------------------------
def _synthetic(vs):
    """saturated planes: luma near 0 / 255 in bands, chroma alternating between the extremes from pair to pair and row to row; mid levels in the
    last rows"""
    w, h = 18, 6
    yy, xx = np.mgrid[0:h, 0:w]
    Y = np.where((xx // 3 + yy) % 2, 250, 5).astype(np.uint8)
    ch = -(-h // vs)
    cy, cx = np.mgrid[0:ch, 0:(w + 1) // 2]
    cb = np.where((cx + cy) % 2, 255, 0).astype(np.uint8)
    cr = np.where((cx // 2 + cy) % 2, 0, 255).astype(np.uint8)
    rng = np.random.default_rng(8)  # the last rows hold random mid levels, where the rounding terms show
    Y[-2:], cb[-1], cr[-1] = rng.integers(20, 236, Y[-2:].shape), rng.integers(20, 236, cb.shape[1]), rng.integers(20, 236, cr.shape[1])
    case = type("S", (), {})()
    case.w, case.h, case.sampling, case.gray = w, h, (2, vs), False
    f = lambda p: p.astype(np.float64)
    case.exact = lambda: [(f(Y), np.zeros(Y.shape)), (f(cb), np.zeros(cb.shape)), (f(cr), np.zeros(cr.shape))]
    return case, (Y, cb, cr)


def _mutant_planes(planes, vs, kind):
    """samples whose correct conversion is what a kernel with the fault would output: Cb / Cr swapped; chroma of the next pair; (4:2:0) the
    chroma row of the other half of the quad, as 4:2:2 planes with each luma row's chroma"""
    Y, cb, cr = planes
    if kind == "swap":
        return (Y, cr, cb), (2, vs)
    if kind == "pair":
        return (Y, np.roll(cb, -1, 1), np.roll(cr, -1, 1)), (2, vs)
    h = Y.shape[0]
    rows = np.minimum((np.arange(h) + 1) // 2, cb.shape[0] - 1)  # crow = (row + 1) >> 1: the odd row of a quad reads the next quad's chroma
    return (Y, cb[rows], cr[rows]), (2, 1)


@pytest.mark.parametrize("vs", [1, 2], ids=["422", "420"])
def test_check_a_and_b_report_each_mutant(vs):
    case, planes = _synthetic(vs)
    w, h = case.w, case.h
    kinds = ["swap", "pair"] + (["quad-row"] if vs == 2 else [])
    for cs in SPACES:
        for shifts in (None, (16, 8, 0)):
            want = rgb(planes, cs, case.sampling, w, shifts)
            check_a(want, want, "unmutated")
            b_compare(b_channels_rgb(want, case, cs, shifts), "unmutated")
            moved = want.copy()
            moved[h // 2, 7] ^= 1
            with pytest.raises(AssertionError, match="differ from the reference"):
                check_a(moved, want, "moved by one")
            for kind in kinds:
                p, smp = _mutant_planes(planes, vs, kind)
                bad = rgb(p, cs, smp, w, shifts)
                with pytest.raises(AssertionError, match="differ from the reference"):
                    check_a(bad, want, kind)
                with pytest.raises(AssertionError, match="beyond the float64 bound"):
                    b_compare(b_channels_rgb(bad, case, cs, shifts), kind)
    for a, b in PAIRS:
        conv = ycc(planes, a, b, case.sampling)
        want = pack(conv, case, UYVY)
        check_a(want, want, "unmutated")
        b_compare(b_channels_ycc(want, UYVY, case, a, b), "unmutated")
        for kind in kinds:
            p, smp = _mutant_planes(planes, vs, kind)
            bad = uyvy(ycc(p, a, b, smp), w, h, smp).reshape(-1)
            with pytest.raises(AssertionError, match="differ from the reference"):
                check_a(bad, want, kind)
            with pytest.raises(AssertionError, match="beyond the float64 bound"):
                b_compare(b_channels_ycc(bad, UYVY, case, a, b), kind)
        with pytest.raises(AssertionError, match="differ from the reference"):  # the + 8192 dropped: a floor where the formula rounds
            check_a(pack(ycc(planes, a, b, case.sampling, rnd=0), case, UYVY), want, "no rounding term")
        if vs == 1:  # I420 of a 4:2:2 stream whose chroma rows are averaged with truncation
            u = pack(conv, case, UYVY).reshape(h, -1)
            trunc = []
            for k in (0, 2):
                c = u[:, k::4].astype(np.int32)
                top, bot = c[0::2], c[1::2]
                trunc.append(np.concatenate([(top[: len(bot)] + bot) >> 1, top[len(bot):]]).astype(np.uint8).reshape(-1))
            bad = np.concatenate([u[:, 1::2][:, :w].reshape(-1)] + trunc)
            with pytest.raises(AssertionError, match="differ from the reference"):
                check_a(bad, pack(conv, case, I420), "truncating I420 average")


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------
def _decoder(monkeypatch, scan=None, sync=None):
    """a decoder created with UGB200_JPEG_MARKER_SCAN / UGB200_JPEG_SYNC set (None: unset), both read at creation"""
    from ultragrid_b200 import api
    for var, val in (("UGB200_JPEG_MARKER_SCAN", scan), ("UGB200_JPEG_SYNC", sync)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    dec = api.JpegDecoder()
    monkeypatch.delenv("UGB200_JPEG_MARKER_SCAN", raising=False)
    monkeypatch.delenv("UGB200_JPEG_SYNC", raising=False)
    return dec


def native(dec, case, pin=True):
    """the decoder's own samples (Y, Cb, Cr) through decode_to(NATIVE, NATIVE) into the lossless output: UYVY for 4:2:2 and grayscale, I420 for
    4:2:0 (with the luma past an odd width from its UYVY, whose samples must be the I420's), VUYA for 4:4:4.  pin: check_decoded against the
    exact IDCT."""
    s, w, h = case.stream, case.w, case.h
    if case.sampling[0] == 1:
        v = dec.decode_to(s, VUYA, NATIVE, NATIVE).reshape(h, w, 4)
        planes = (v[:, :, 2], v[:, :, 1], v[:, :, 0])
        assert (v[:, :, 3] == 255).all()
        comp = list(planes)
    else:
        u = dec.decode_to(s, UYVY, NATIVE, NATIVE).reshape(h, -1, 4)
        Yu = u[:, :, [1, 3]].reshape(h, -1)
        if case.sampling[1] == 1:
            planes = (Yu, u[:, :, 0], u[:, :, 2])
        else:
            i = J.i420_planes(dec.decode_to(s, I420, NATIVE, NATIVE), w, h)
            rows = np.arange(h) // 2
            assert np.array_equal(Yu[:, :w], i[0]) and np.array_equal(u[:, :, 0], i[1][rows]) and np.array_equal(u[:, :, 2], i[2][rows]), case.name
            planes = (Yu, i[1], i[2])
        comp = [Yu] if case.gray else list(planes)
        if case.gray:
            assert (u[:, :, 0] == 128).all() and (u[:, :, 2] == 128).all(), case.name
    if pin:
        check_decoded(case.stream, comp, case.name)
    return planes


def _get(dec, case, out_c, cs_in, cs_out=None, shifts=(0, 8, 16), device=False, pitch=0, fill=0x5A):
    """one decode: decode_cs (cs_out None; decode_to for grayscale, which decode_cs refuses) or decode_to; host, or device at `pitch` into a
    buffer filled with `fill`"""
    import torch
    if cs_out is None and case.gray:
        cs_out = NATIVE
    kw = {"color_space": cs_in} if cs_out is None else {"color_space": cs_in, "out_cs": cs_out}
    if not device:
        return dec.decode(case.stream, out_c, shifts=shifts, **kw)
    n = pitch * case.h if out_c != I420 else case.w * case.h + 2 * ((case.w + 1) // 2) * ((case.h + 1) // 2) + 64
    out = torch.full((n,), fill, dtype=torch.uint8, device="cuda")
    dec.decode(case.stream, out_c, shifts=shifts, device=True, pitch=0 if out_c == I420 else pitch, out=out, **kw)
    return out.cpu().numpy()


def _row_bytes(case, out_c):
    w = case.w
    if out_c in (RGB, RGBA):
        return (w if case.sampling[0] == 1 else w // 2 * 2) * (3 if out_c == RGB else 4)
    return (w + 1) // 2 * 4 if out_c == UYVY else w * 4


def check_device(got, want, case, out_c, pitch, what):
    """a device destination: the rows at `pitch`, nothing written behind them (the last pixel of an odd-width 4:2:x RGB / RGBA row included)"""
    if out_c == I420:
        check_a(got[:want.size], want, what)
        assert (got[want.size:] == 0x5A).all(), what
        return
    n = _row_bytes(case, out_c)
    g = got.reshape(case.h, pitch)
    check_a(g[:, :n], want.reshape(case.h, -1)[:, :n], what)
    assert (g[:, n:] == 0x5A).all(), (what, "bytes written behind the row")


def cs_name(cs, case):
    return case.declared() if cs == "auto" else cs


def sweep(dec, case, planes, full, stats=None):
    """every output of the case through `dec` against the reference of `planes` (check A), and the float64 bound (check B, when stats is given).
    full: every space, shift, pair and output, each to the host and to a pitched device buffer; else one of each kind, host only."""
    w, h = case.w, case.h
    spaces = SPACES + ["auto"] if full else ["Y601full", "auto"]
    for cs in spaces:
        eff = cs_name(cs, case)
        for shifts in (SHIFTS if full else [None, (8, 16, 24)]):
            out_c = RGB if shifts is None else RGBA
            want = rgb(planes, eff, case.sampling, w, shifts)
            n = want.shape[1]
            what = f"{case.name}: decode_cs({cs}) to {'RGB' if shifts is None else f'RGBA {shifts}'}"
            got = _get(dec, case, out_c, cs, shifts=shifts or (0, 8, 16))
            check_a(got.reshape(h, -1)[:, :n], want, what)
            if full:
                pitch = _row_bytes(case, out_c) + 48
                check_device(_get(dec, case, out_c, cs, shifts=shifts or (0, 8, 16), device=True, pitch=pitch), want, case, out_c, pitch, what + " (device)")
            if stats is not None and cs != "auto":
                b_compare(b_channels_rgb(got.reshape(h, -1)[:, :n], case, eff, shifts), what, stats.setdefault("rgb", _stats()))
        if eff == "Y709" and case.sampling[0] == 2 and not case.gray and full:  # Y709 RGB of a 4:2:x stream is ugb200_jpeg_decode's RGB
            n = _row_bytes(case, RGB)
            check_a(dec.decode(case.stream, RGB).reshape(h, -1)[:, :n], rgb(planes, "Y709", case.sampling, w), f"{case.name}: Y709 == ugb200_jpeg_decode")
    outs = [UYVY, I420] + ([VUYA] if case.sampling[0] == 1 else [])
    pairs = [(CS[a], CS[b]) for a, b in PAIRS] + [(CS["Y709"], CS["Y709"]), (NATIVE, CS["Y709"]), (AUTO, CS["Y709"])]
    if not full:
        pairs = [(CS["Y601full"], CS["Y709"]), (AUTO, CS["Y709"])]
    nat = {}
    for a, b in pairs:
        na = cs_name("auto", case) if a == AUTO else {v: k for k, v in CS.items()}.get(a)
        nb = {v: k for k, v in CS.items()}[b]
        conv = planes if a == NATIVE or na == nb else ycc(planes, na, nb, case.sampling)
        for out_c in (outs if full else outs[:2]):
            want = expected(conv, case, out_c)
            what = f"{case.name}: decode_to({a} -> {b}) to codec {out_c}"
            got = _get(dec, case, out_c, a, b)
            check_a(got, want, what)
            if a == NATIVE or na == nb:  # the native bytes
                nat.setdefault(out_c, got)
                check_a(got, nat[out_c], what + " (native bytes)")
            if full:
                pitch = _row_bytes(case, out_c) + 48
                check_device(_get(dec, case, out_c, a, b, device=True, pitch=pitch), want, case, out_c, pitch, what + " (device)")
            if stats is not None and a not in (NATIVE, AUTO) and na != nb and (out_c == VUYA or (out_c == UYVY and case.sampling[0] == 2)):
                b_compare(b_channels_ycc(got, out_c, case, na, nb), what, stats.setdefault("ycc", _stats()))


def _stats():
    return {"n": 0, "banded": 0, "worst": -9.0}


def _layout(case):
    return "gray" if case.gray else {(1, 1): "444", (2, 1): "422", (2, 2): "420"}[case.sampling]


@pytest.mark.gpu
def test_gpu_color_outputs_equal_the_reference(corpus, monkeypatch):
    """check A for every output of every corpus stream (host and pitched device destinations), check B for UYVY, VUYA, RGB and RGBA; the native
    samples pinned to the exact IDCT; prints the worst excess over the bound and the share of values that need the tie band, per layout"""
    dec = _decoder(monkeypatch)
    stats = {}
    for case in corpus:
        planes = native(dec, case)
        sweep(dec, case, planes, True, stats.setdefault(_layout(case), {}))
    dec.close()
    for lay, st in sorted(stats.items()):
        for kind, s in sorted(st.items()):
            print(f"[stats] check B {lay} {kind}: worst excess {s['worst']:.3f}, needs the band {s['banded']}/{s['n']} = {100 * s['banded'] / max(s['n'], 1):.4f} %")


@pytest.mark.gpu
def test_gpu_auto_reads_each_declared_space(corpus):
    """the declared-space variants resolve to the space the header's rules give; AUTO is then checked on them by the sweeps"""
    variants = [c for c in corpus if any(c.name.endswith(" " + k) for k, _, _ in DECLARED)]
    assert len(variants) == 4 * 6 + 1
    for c in variants:
        k = c.name.rsplit(" ", 1)[1]
        assert c.declared() == dict((n, want) for n, _, want in DECLARED)[k], c.name


@pytest.mark.gpu
@pytest.mark.parametrize("scan", ["host", "device"])
@pytest.mark.parametrize("sync", ["off", "on"])
def test_gpu_routes(corpus, monkeypatch, scan, sync):
    """both marker scans x one thread per segment / the self-synchronising route (the route taken asserted with last_sync), check A on one output
    of each kind; UGB200_JPEG_SYNC=on:8 (8-byte subsequences) on the no-DRI and saturated streams"""
    dec = _decoder(monkeypatch, scan, sync)
    for case in corpus:
        planes = native(dec, case)
        st = dec.last_sync()
        assert st["scans"] == (len(case.fr.scans) if sync == "on" else 0), (case.name, st)
        sweep(dec, case, planes, False)
        assert dec.last_sync()["scans"] == st["scans"], case.name
    dec.close()
    if scan == "device" and sync == "on":
        dec = _decoder(monkeypatch, scan, "on:8")
        few = [c for c in corpus if c.fr.ri == 0 or c.name.startswith("sat-")][:12]
        assert len(few) >= 8
        for case in few:
            planes = native(dec, case, pin=False)
            st = dec.last_sync()
            assert st["scans"] == len(case.fr.scans) and st["subsequences"] >= len(case.fr.scans), (case.name, st)
            sweep(dec, case, planes, False)
        dec.close()


def _encoder_stream(orc, kind, w, h):
    """this encoder's 4:2:2 (UYVY), its I420, and Y601full 4:2:0 in one scan per component, from the GPU encoder"""
    import torch
    from ultragrid_b200 import api
    rgb_src = natural_rgb(w, h, 3)
    enc = api.JpegEncoder()
    if kind == "rgb-y601full-420-pc":
        enc.encode_device(torch.from_numpy(np.ascontiguousarray(rgb_src).reshape(-1)).cuda(), w, h, RGB, quality=90, subsampling=420, color_space=2)
    else:
        u = util.convert_cpu(orc, "orc_convert", RGB, UYVY, rgb_src.reshape(-1), w, h)
        if kind == "uyvy422":
            enc.encode_device(torch.from_numpy(u).cuda(), w, h, UYVY, quality=90)
        else:
            src = np.concatenate([p.reshape(-1) for p in J.uyvy_to_i420_planes(u, w, h)])
            enc.encode_device(torch.from_numpy(src).cuda(), w, h, I420, quality=90)
    s = enc.result()
    enc.close()
    return s


class _Big(Case):
    """a large stream: header only (the Python reader is too slow for the exact IDCT of an 8K stream without DRI)"""

    def __init__(self, name, stream):
        from ultragrid_b200 import api
        info = api.jpeg_image_info(stream)
        self.name, self.stream, self.w, self.h, self.gray = name, stream, info.width, info.height, info.components == 1
        self.sampling = (info.h_samp, info.v_samp)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)], ids=["4K", "8K"])
def test_gpu_large_frames_check_a(orc, w, h):
    """check A at 4K and 8K: PIL 4:2:0 without DRI, this encoder's 4:2:2, its I420 and Y601full 4:2:0 per component; the native samples of such
    frames are pinned to the exact IDCT elsewhere (test_gpu_decoder_8k_equals_exact_idct, test_jpeg_decode_color.py)"""
    from ultragrid_b200 import api
    dec = api.JpegDecoder()
    streams = [("pil-420", pil_stream("420", w, h))] + [(k, _encoder_stream(orc, k, w, h)) for k in ("uyvy422", "i420", "rgb-y601full-420-pc")]
    for name, s in streams:
        case = _Big(f"{name} {w}x{h}", s)
        assert case.sampling[0] == 2
        planes = native(dec, case, pin=False)
        if name == "pil-420":
            assert dec.last_sync()["scans"] == 1
        for cs, shifts in (("Y601full", None), ("Y709", (16, 8, 0))):
            check_a(_get(dec, case, RGB if shifts is None else RGBA, cs, shifts=shifts or (0, 8, 16)).reshape(h, -1), rgb(planes, cs, case.sampling, w, shifts),
                    f"{case.name} decode_cs({cs})")
        for a, b, out_c in (("Y601full", "Y709", UYVY), ("Y709", "Y601", I420)):
            check_a(_get(dec, case, out_c, CS[a], CS[b]), pack(ycc(planes, a, b, case.sampling), case, out_c), f"{case.name} decode_to({a} -> {b}) {out_c}")
    dec.close()


@pytest.mark.gpu
def test_gpu_modules_on_a_stream_without_dri(monkeypatch):
    """the mirror-ABI gpujpeg and gpujpeg_to_dxt modules on a 1080p PIL 4:2:0 stream without DRI (the self-synchronising route), with
    UGB200_JPEG_DECODE_CS unset and `auto`: UYVY and RGB against the reference of the native samples; DXT1 against cuda_rgb_to_dxt1 of the
    reference RGB with the height mirrored, as the module encodes"""
    import torch
    from ultragrid_b200 import api
    from ultragrid_b200.compress import Decompress
    w, h = 1920, 1080
    case = Case("pil-420 1080p", pil_stream("420", w, h))
    assert case.fr.ri == 0 and case.declared() == "Y601full"
    dec = _decoder(monkeypatch)
    planes = native(dec, case)
    assert dec.last_sync()["scans"] == 1
    dec.close()

    def through(out_c):
        d = Decompress(JPEG, out_c)
        d.reconfigure(w, h, JPEG, out_c)
        st, out, _ = d.frame(case.stream)
        d.close()
        assert st == Decompress.GOT_FRAME
        return out

    for env in (None, "auto"):
        if env is None:
            monkeypatch.delenv("UGB200_JPEG_DECODE_CS", raising=False)
            want_uyvy, want_rgb = pack(planes, case, UYVY), rgb(planes, "Y709", case.sampling, w)
        else:
            monkeypatch.setenv("UGB200_JPEG_DECODE_CS", env)
            want_uyvy, want_rgb = pack(ycc(planes, "Y601full", "Y709", case.sampling), case, UYVY), rgb(planes, "Y601full", case.sampling, w)
        check_a(through(UYVY), want_uyvy, f"gpujpeg UYVY ({env})")
        check_a(through(RGB).reshape(h, -1), want_rgb, f"gpujpeg RGB ({env})")
        dxt = api.compat_to_dxt("cuda_rgb_to_dxt1", torch.from_numpy(want_rgb.reshape(-1).copy()).cuda(), w, -h).cpu().numpy()
        got = through(DXT1)
        assert got.size >= dxt.size
        check_a(got[:dxt.size], dxt, f"gpujpeg_to_dxt DXT1 ({env})")
    monkeypatch.delenv("UGB200_JPEG_DECODE_CS", raising=False)
