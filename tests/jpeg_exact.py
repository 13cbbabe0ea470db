"""Exact references for the JPEG encoder and decoder: the T.81 transforms in float64, an independent baseline stream reader, a
baseline stream writer, and the component planes as the encoder sees them.  numpy and the standard library only.

Transforms (T.81 A.3.3).  FDCT: F(v, u) = 1/4 C(u) C(v) sum_y sum_x s(y, x) cos((2x + 1) u pi / 16) cos((2y + 1) v pi / 16) of the
level-shifted samples s = p - 128, C(0) = 1/sqrt 2, else 1; as matrices F = M s M^T with M[u, x] = C(u) / 2 cos((2x + 1) u pi / 16)
(orthonormal), and the IDCT s = M^T F M.  Natural index n = 8 v + u.  What a coefficient of a stream must be: round_half_even(F / Q)
(AC clamped to +-1023, the 10-bit category limit); what a decoded sample must be: clamp(round(IDCT(coef x Q) + 128), 0, 255).

Tie band.  Both kernels compute the transforms in float32 (AAN, a fixed operation order), so a value lying very close to a
half-integer may round the other way.  Such a value is exempt: it may differ by 1 from the exact rounding, nothing else may.  The band
is derived, not guessed: `aan_fdct_f32` / `aan_idct_f32` restate the float32 operation order of oracle/jpeg_oracle.c and
oracle/jpeg_decode_oracle.c (test_jpeg_exact.py checks that they round to the oracles' integers), and their largest distance from the exact
value, over the CPU corpus of test_jpeg_exact.py (RGB noise, natural frames, extreme-AC and DC-swing frames; 64x64, 130x37 and 256x256;
q = 1, 50, 90, 100; decoder streams with Q = 255 and |coef| = 1023 as well), measured as a multiple of the block's magnitude:

  * encoder: |x_f32 - F / Q| <= E_ENC * S / Q with S = sum |s| of the block's 64 level-shifted samples.  Measured max ratio
    E_ENC = 4.65e-8 (float32 epsilon is 6.0e-8), and aan_fdct_f32 rounds to the oracle's integers for all 3.6 million coefficients.
    The band is about 4x that: ENC_BAND = 2e-7 * S / Q.  For a full-scale block (S = 8192) at Q = 1 this is 1.6e-3; for a typical
    block at q = 90 about 1e-5.
  * decoder: |px_f32 - px_exact| <= 3e-5 + E_DEC * D with D = sum |coef x Q| of the block's 64 dequantised coefficients; 3e-5 covers
    the level shift's own rounding (f + 128 in float32: half an ulp at 256 is 1.5e-5).  Measured max ratio E_DEC = 5.25e-8.  The band
    is about 4x that: DEC_BAND = 2.2e-7 * D + 3e-5.  Q = 255 with |coef| = 1023 everywhere gives D = 1.7e7 and a band of 3.7.
  * how the band is applied: it widens the UNCLAMPED exact value, and an exemption is one step, never more: a value may differ by 1 from
    clamp(round_half_even(x)), and only towards clamp(round(x - band)) or clamp(round(x + band)).  A sample whose exact value lies beyond
    0 or 255 by more than the band (almost every sample of the Q = 255 blocks) must equal the clamp; the AC clamp at +-1023 likewise.

Any real arithmetic error - a wrong constant, zig-zag entry, rounding rule or padding rule - moves values by far more than the band
around most coefficients and samples, and so shows as mismatches outside it (test_jpeg_exact.py demonstrates this per kind).

Reader.  `read(stream)` parses SOI, APPn, COM, DQT, DHT (tables may be redefined between scans), SOF0, DRI, SOS, RSTn and EOI and decodes
every scan into int16 coefficients per component, natural order, on the component's block grid (T.81 A.2: an interleaved scan covers
ceil(X / 8 Hmax) x ceil(Y / 8 Vmax) MCUs; a one-component scan ceil(ceil(X Hi / Hmax) / 8) x ceil(ceil(Y Vi / Vmax) / 8) blocks).
It asserts what a baseline stream must satisfy instead of tolerating it: 0xFF in entropy-coded data is followed by 0x00; the padding
before RSTn and EOI is 1-bits, fewer than 8; RSTn count modulo 8 and there is one per restart interval boundary; every code is defined
in its table; no run passes position 63; AC categories <= 10, DC difference categories <= 11.  Each restart segment is decoded from a
precomputed 16-bit window per bit position (one O(1) look-up per symbol); `segments=` decodes a chosen subset.
"""
import math

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# T.81 Annex K: K.1 / K.2 quantisation tables (natural order) and the typical Huffman tables K.3 - K.6 (BITS, HUFFVAL)
Q_LUMA = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
                   18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
                   103, 99])
Q_CHROMA = np.array([17, 18, 24, 47] + [99] * 4 + [18, 21, 26, 66] + [99] * 4 + [24, 26, 56] + [99] * 5 + [47, 66] + [99] * 38)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], list(bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a434445464748494a"
    "535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7"
    "c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")))
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], list(bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738393a434445464748"
    "494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3"
    "c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")))


def scaled_qtable(base, quality):
    """IJG quality scaling (jpeg_quality_scaling + jpeg_add_quant_table with the baseline clamp to 1..255)"""
    quality = min(max(quality, 1), 100)
    scale = 5000 // quality if quality < 50 else 200 - quality * 2
    return np.clip((np.asarray(base) * scale + 50) // 100, 1, 255)


# ---- exact transforms ----------------------------------------------------------------------------------------------------------
_u = np.arange(8)
M = np.cos((2 * _u[None, :] + 1) * _u[:, None] * np.pi / 16) * np.where(_u == 0, np.sqrt(0.5), 1.0)[:, None] / 2


def fdct(blocks):
    """(N, 8, 8) samples 0..255 -> (N, 64) float64 F in natural order, of the level-shifted samples"""
    s = np.asarray(blocks, np.float64).reshape(-1, 8, 8) - 128.0
    return np.einsum("vy,byx,ux->bvu", M, s, M).reshape(-1, 64)


def idct(F):
    """(N, 64) natural-order dequantised coefficients -> (N, 8, 8) float64 samples, level shift (+128) included, not rounded or clamped"""
    F = np.asarray(F, np.float64).reshape(-1, 8, 8)
    return np.einsum("vy,bvu,ux->byx", M, F, M) + 128.0


def half_dist(x):
    """distance of each value to the nearest half-integer (0 for n + 1/2)"""
    return np.abs(x - np.floor(x) - 0.5)


def enc_band(blocks, q):
    """(N, 64) tie band of the quotients F / Q of `blocks` (N, 8, 8 samples) for the natural-order table q"""
    S = np.abs(np.asarray(blocks, np.float64).reshape(-1, 64) - 128.0).sum(axis=1)
    return ENC_BAND * S[:, None] / np.asarray(q, np.float64)[None, :]


def dec_band(coef, q):
    """(N, 8, 8) tie band of the decoded samples of the natural-order coefficients coef (N, 64) under table q"""
    D = np.abs(np.asarray(coef, np.float64) * np.asarray(q, np.float64)[None, :]).sum(axis=1)
    return np.broadcast_to((DEC_BAND * D + DEC_BAND_ABS)[:, None, None], (len(D), 8, 8))


ENC_BAND = 2e-7
DEC_BAND = 2.2e-7
DEC_BAND_ABS = 3e-5


def expected_coefficients(x):
    """round_half_even(F / Q), AC clamped to the 10-bit category limit"""
    e = np.rint(x)
    e[:, 1:] = np.clip(e[:, 1:], -1023, 1023)
    return e


def _within_band(got, x, band, lo, hi):
    """got must equal clip(round_half_even(x), lo, hi); it may differ from that by 1 only towards clip(round(x -+ band)), i.e. only where a
    half-integer lies within the band of the UNCLAMPED exact value.  A value beyond the clamp limit by more than the band must equal the limit."""
    band = np.broadcast_to(band, x.shape)
    exp = np.clip(np.rint(x), lo, hi)
    alt_lo, alt_hi = np.clip(np.rint(x - band), lo, hi), np.clip(np.rint(x + band), lo, hi)
    ok = (got == exp) | ((np.abs(got - exp) == 1) & (got >= alt_lo) & (got <= alt_hi))
    return exp, ok


def compare_coefficients(got, x, band, what=""):
    """got (N, 64) integers against the exact quotients x: equal to round_half_even(x) (AC clamped to +-1023), or 1 away where the band of x
    reaches the half-integer between them.
    @returns dict(n, exempt, worst): number compared, values that differ from the exact rounding (all inside the band), largest |got - x| - 1/2"""
    got = np.asarray(got, np.int64).reshape(-1, 64)
    x = np.asarray(x, np.float64).reshape(-1, 64)
    lim = np.where(np.arange(64) == 0, np.inf, 1023.0)
    exp, ok = _within_band(got, x, band, -lim, lim)
    xc = np.clip(x, -lim, lim)
    diff = got != exp
    bad = ~ok
    if bad.any():
        b, n = np.argwhere(bad)[0]
        k = int(np.flatnonzero(ZIGZAG == n)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} coefficients off the exact value outside the tie band; first: block {b}, natural index {n} "
                             f"(zig-zag {k}), got {got[b, n]}, exact {x[b, n]!r}, band {np.broadcast_to(band, x.shape)[b, n]:.3g}")
    return {"n": int(x.size), "exempt": int(diff.sum()), "worst": float((np.abs(got - xc) - 0.5).max()) if x.size else 0.0}


def compare_samples(got, px, band, what=""):
    """got integers against exact samples px (same shape, before the clamp): equal to clamp(round(px), 0, 255), or 1 away where the band of px
    reaches the half-integer between them; a sample whose exact value lies beyond 0 or 255 by more than the band must equal the clamp"""
    got = np.asarray(got, np.int64)
    px = np.asarray(px, np.float64)
    exp, ok = _within_band(got, px, band, 0, 255)
    pc = np.clip(px, 0, 255)
    diff = got != exp
    bad = ~ok
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} samples off the exact value outside the tie band; first at {i}: got {got[i]}, "
                             f"exact {px[i]!r}, band {np.broadcast_to(band, px.shape)[i]:.3g}")
    return {"n": int(px.size), "exempt": int(diff.sum()), "worst": float((np.abs(got - pc) - 0.5).max()) if px.size else 0.0}


# ---- float32 restatements of the AAN operation order (to measure the band, and to show the comparators' teeth) --------------------------
AAN_FDCT = {"c707": 0.707106781, "c382": 0.382683433, "c541": 0.541196100, "c1306": 1.306562965}
AAN_SCALE = (1.0, 1.387039845, 1.306562965, 1.175875602, 1.0, 0.785694958, 0.541196100, 0.275899379)
_f = np.float32


def _fma(a, b, c):
    return (a.astype(np.float64) * np.float64(b) + c.astype(np.float64)).astype(_f) if np.ndim(b) == 0 else \
        (np.float64(a) * b.astype(np.float64) + c.astype(np.float64)).astype(_f)


def _fdct8(d, k):
    t0, t7 = d[0] + d[7], d[0] - d[7]
    t1, t6 = d[1] + d[6], d[1] - d[6]
    t2, t5 = d[2] + d[5], d[2] - d[5]
    t3, t4 = d[3] + d[4], d[3] - d[4]
    e0, e3, e1, e2 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = [None] * 8
    o[0], o[4] = e0 + e1, e0 - e1
    s1 = e2 + e3
    o[2], o[6] = _fma(s1, _f(k["c707"]), e3), _fma(s1, _f(-k["c707"]), e3)
    o0, o1, o2 = t4 + t5, t5 + t6, t6 + t7
    z5 = (o0 - o2) * _f(k["c382"])
    z2 = _fma(o0, _f(k["c541"]), z5)
    z4 = _fma(o2, _f(k["c1306"]), z5)
    z11, z13 = _fma(o1, _f(k["c707"]), t7), _fma(o1, _f(-k["c707"]), t7)
    o[5], o[3], o[1], o[7] = z13 + z2, z13 - z2, z11 + z4, z11 - z4
    return o


def aan_fdct_f32(blocks, q, consts=None):
    """(N, 8, 8) samples -> (N, 64) float64 values x_f32 that the float32 AAN forward transform of the oracle rounds (the exact product
    f32 coefficient x f32 multiplier, rounded half to even there); consts replaces AAN_FDCT entries"""
    k = dict(AAN_FDCT, **(consts or {}))
    f = (np.asarray(blocks, np.int64).reshape(-1, 8, 8) - 128).astype(_f)
    rows = _fdct8([f[:, :, x] for x in range(8)], k)            # along x, every row
    f = np.stack(rows, axis=2)
    cols = _fdct8([f[:, y, :] for y in range(8)], k)            # along y, every column
    f = np.stack(cols, axis=1).reshape(-1, 64)
    s = np.array(AAN_SCALE)
    qm = (1.0 / (np.asarray(q, np.float64).reshape(8, 8) * s[:, None] * s[None, :] * 8.0)).astype(_f).reshape(64)
    return f.astype(np.float64) * qm.astype(np.float64)


def _idct8(d):
    t0, t1, t2, t3 = d[0], d[2], d[4], d[6]
    e0, e1 = t0 + t2, t0 - t2
    e3 = t1 + t3
    e2 = (t1 - t3) * _f(1.414213562) - e3
    a0, a3, a1, a2 = e0 + e3, e0 - e3, e1 + e2, e1 - e2
    o4, o5, o6, o7 = d[1], d[3], d[5], d[7]
    z13, z10, z11, z12 = o6 + o5, o6 - o5, o4 + o7, o4 - o7
    b7 = z11 + z13
    b11 = (z11 - z13) * _f(1.414213562)
    z5 = (z10 + z12) * _f(1.847759065)
    b10 = _fma(z12, _f(1.082392200), -z5)
    b12 = _fma(z10, _f(-2.613125930), z5)
    b6 = b12 - b7
    b5 = b11 - b6
    b4 = b10 + b5
    return [a0 + b7, a1 + b6, a2 + b5, a3 - b4, a3 + b4, a2 - b5, a1 - b6, a0 - b7]


def aan_idct_f32(coef, q):
    """(N, 64) natural coefficients -> (N, 8, 8) float64 of the float32 values (f + 128) the oracle decoder rounds"""
    s = np.array(AAN_SCALE, _f)
    qq = np.asarray(q).reshape(8, 8).astype(_f)
    m = ((qq * s[:, None]) * s[None, :]) * _f(0.125)
    f = np.asarray(coef).reshape(-1, 8, 8).astype(_f) * m[None]
    f = np.stack(_idct8([f[:, v, :] for v in range(8)]), axis=1)  # columns (along v) first
    f = np.stack(_idct8([f[:, :, u] for u in range(8)]), axis=2)  # then rows
    return (f + _f(128.0)).astype(np.float64)


# ---- component planes as the encoder sees them ------------------------------------------------------------------------------------
def pad_blocks(plane, gh, gw):
    """(gh * gw, 8, 8) blocks of the plane on a gh x gw block grid, raster order; the plane is padded by edge replication (the rule of
    gather() in oracle/jpeg_oracle.c: a row or column beyond the plane repeats its last one)"""
    plane = np.asarray(plane)
    ph, pw = plane.shape
    yi = np.minimum(np.arange(gh * 8), ph - 1)
    xi = np.minimum(np.arange(gw * 8), pw - 1)
    p = plane[yi][:, xi]
    return p.reshape(gh, 8, gw, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)


def uyvy_planes(uyvy, w, h, pitch=None):
    """Y (h x w), Cb, Cr (h x ceil(w / 2)) of a UYVY frame"""
    pitch = pitch or (w + 1) // 2 * 4
    a = np.asarray(uyvy).reshape(-1)[:pitch * h].reshape(h, pitch)[:, :(w + 1) // 2 * 4].reshape(h, -1, 4)
    y = np.stack([a[:, :, 1], a[:, :, 3]], axis=2).reshape(h, -1)[:, :w]
    return [y, a[:, :, 0], a[:, :, 2]]


def packed_planes(src, w, h, n):
    """the n stored planes of a packed frame of n bytes per pixel (RGB: R G B, RGBA: R G B A)"""
    a = np.asarray(src).reshape(h, w, n)
    return [a[:, :, c] for c in range(n)]


def i420_planes(src, w, h):
    cw, ch = (w + 1) // 2, (h + 1) // 2
    a = np.asarray(src).reshape(-1)
    return [a[:w * h].reshape(h, w), a[w * h:w * h + cw * ch].reshape(ch, cw), a[w * h + cw * ch:w * h + 2 * cw * ch].reshape(ch, cw)]


def uyvy_to_i420_planes(uyvy, w, h):
    """uyvy_to_i420 (DESIGN.md section 2): Y copied; Cb, Cr = (a + b + 1) >> 1 of the two rows of a pair, the last row of an odd height with
    itself"""
    y, cb, cr = uyvy_planes(uyvy, w, h)
    r1 = np.minimum(np.arange(0, h, 2) + 1, h - 1)
    avg = [((c[0::2].astype(np.int32) + c[r1].astype(np.int32) + 1) >> 1).astype(np.uint8) for c in (cb, cr)]
    return [y] + avg


# ---- baseline reader ------------------------------------------------------------------------------------------------------------------
def _codes(bits, vals):
    """T.81 C.2: [(symbol, code, length)]"""
    out, code, k = [], 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            out.append((vals[k], code, ln))
            code += 1
            k += 1
        code <<= 1
    return out


def _lut(bits, vals):
    """65536 entries: (length << 8 | symbol) of the code that begins the 16-bit window, -1 where no code is defined"""
    assert sum(bits) == len(vals) <= 256
    lut = np.full(1 << 16, -1, np.int32)
    for sym, code, ln in _codes(bits, vals):
        assert code < (1 << ln), "over-subscribed Huffman table"
        lut[code << (16 - ln):(code + 1) << (16 - ln)] = ln << 8 | sym
    return lut


class Frame:
    """the parsed stream: w, h, components [{id, h, v, tq}], q {tq: natural table}, ri, adobe (transform or None), sof (marker byte),
    coef[c] (int16, grid rows x grid columns x 64, natural order), grid[c] (rows, cols) as coded, decoded[c] (bool per block), scans [{comps, nseg}]"""


def _extend(v, t):
    return v - (1 << t) + 1 if v < (1 << (t - 1)) else v


def _decode_segment(data, fr, scan, mcus, pred_reset=True):
    """entropy-coded bytes of one restart segment (stuffing in) -> fills fr.coef for the MCUs in `mcus`; asserts the padding"""
    a = np.frombuffer(data, np.uint8)
    ff = np.flatnonzero(a[:-1] == 0xFF) if len(a) > 1 else np.zeros(0, np.int64)
    assert len(a) == 0 or a[-1] != 0xFF, "0xFF at the end of a segment"
    assert (a[ff + 1] == 0).all(), "0xFF in entropy-coded data not followed by 0x00"
    keep = np.ones(len(a), bool)
    keep[ff + 1] = False
    bits = np.unpackbits(a[keep])
    nb = len(bits)
    b = np.concatenate([bits, np.zeros(16, np.uint8)]).astype(np.int32)
    win = np.zeros(nb + 1, np.int32)
    for k in range(16):
        win |= b[k:k + nb + 1] << (15 - k)
    win = win.tolist()
    pos = 0
    pred = [0] * len(scan["comps"])
    for m in mcus:
        for si, (c, blocks) in enumerate(scan["blocks_of"](m)):
            dc, ac = scan["dc"][si], scan["ac"][si]
            for (by, bx) in blocks:
                blk = np.zeros(64, np.int32)
                e = dc[win[pos]]
                assert e >= 0, f"undefined DC code at bit {pos}"
                pos += e >> 8
                t = e & 255
                assert t <= 11, f"DC category {t}"
                if t:
                    pred[si] += _extend(win[pos] >> (16 - t), t)
                    pos += t
                blk[0] = pred[si]
                k = 1
                while k < 64:
                    e = ac[win[pos]]
                    assert e >= 0, f"undefined AC code at bit {pos}"
                    pos += e >> 8
                    rs = e & 255
                    r, s = rs >> 4, rs & 15
                    if s == 0:
                        if r != 15:
                            break  # EOB
                        assert k + 16 <= 64, f"ZRL past position 63 (k = {k})"
                        k += 16
                        continue
                    assert s <= 10, f"AC category {s}"
                    k += r
                    assert k <= 63, f"run past position 63 (k = {k})"
                    blk[ZIGZAG[k]] = _extend(win[pos] >> (16 - s), s)
                    pos += s
                    k += 1
                assert pos <= nb, "read past the end of the segment"
                if by < fr.coef[c].shape[0] and bx < fr.coef[c].shape[1]:
                    fr.coef[c][by, bx] = blk
                    fr.decoded[c][by, bx] = True
    rest = nb - pos
    assert 0 <= rest < 8, f"{rest} bits left at the end of the segment"
    assert rest == 0 or bits[pos:].all(), "padding bits are not 1-bits"


def read(stream, segments=None):
    """parse and decode a baseline stream (see the module docstring).  segments: None (all), or a function (scan number, number of
    segments) -> the segment indices to decode"""
    s = bytes(stream)
    assert s[:2] == b"\xff\xd8", "no SOI"
    fr = Frame()
    fr.q, fr.ri, fr.adobe, fr.scans, fr.components, fr.sof = {}, 0, None, [], [], None
    huff = {}
    p = 2
    while True:
        assert p + 2 <= len(s) and s[p] == 0xFF, f"no marker at {p}"
        mk = s[p + 1]
        if mk == 0xD9:
            assert p + 2 == len(s), "bytes after EOI"
            break
        L = s[p + 2] << 8 | s[p + 3]
        d = s[p + 4:p + 2 + L]
        assert len(d) == L - 2
        if mk == 0xDB:
            i = 0
            while i < len(d):
                assert d[i] >> 4 == 0, "16-bit quantisation table"
                fr.q[d[i] & 15] = np.array([0] * 64)
                fr.q[d[i] & 15][ZIGZAG] = list(d[i + 1:i + 65])
                i += 65
        elif mk == 0xC4:
            i = 0
            while i < len(d):
                tc, th = d[i] >> 4, d[i] & 15
                assert tc <= 1 and th <= 1
                bits = list(d[i + 1:i + 17])
                n = sum(bits)
                huff[(tc, th)] = _lut(bits, list(d[i + 17:i + 17 + n]))
                i += 17 + n
        elif mk == 0xC0:
            assert fr.sof is None and d[0] == 8
            fr.sof = mk
            fr.h, fr.w, nc = d[1] << 8 | d[2], d[3] << 8 | d[4], d[5]
            for c in range(nc):
                fr.components.append({"id": d[6 + 3 * c], "h": d[7 + 3 * c] >> 4, "v": d[7 + 3 * c] & 15, "tq": d[8 + 3 * c]})
            hmax, vmax = max(c["h"] for c in fr.components), max(c["v"] for c in fr.components)
            mw, mh = math.ceil(fr.w / (8 * hmax)), math.ceil(fr.h / (8 * vmax))
            fr.coef = [np.zeros((mh * c["v"], mw * c["h"], 64), np.int16) for c in fr.components]
            fr.decoded = [np.zeros((mh * c["v"], mw * c["h"]), bool) for c in fr.components]
            fr.grid = [None] * nc
        elif mk == 0xDD:
            fr.ri = d[0] << 8 | d[1]
        elif mk == 0xEE and d[:5] == b"Adobe":
            fr.adobe = d[11]
        elif 0xE0 <= mk <= 0xEF or mk == 0xFE:
            pass
        elif mk == 0xDA:
            p = _scan(s, p + 2 + L, d, fr, huff, segments)
            continue
        else:
            raise AssertionError(f"marker FF{mk:02X} is not baseline")
        p += 2 + L
    assert fr.sof is not None and fr.scans
    return fr


def _scan(s, p, d, fr, huff, segments):
    ns = d[0]
    comps = []
    for i in range(ns):
        c = next(j for j, cc in enumerate(fr.components) if cc["id"] == d[1 + 2 * i])
        comps.append((c, d[2 + 2 * i] >> 4, d[2 + 2 * i] & 15))
    assert d[1 + 2 * ns:4 + 2 * ns] == bytes([0, 63, 0]), "not a sequential scan"
    hmax, vmax = max(c["h"] for c in fr.components), max(c["v"] for c in fr.components)
    if ns == 1:
        cc = fr.components[comps[0][0]]
        mcux = math.ceil(math.ceil(fr.w * cc["h"] / hmax) / 8)
        mcuy = math.ceil(math.ceil(fr.h * cc["v"] / vmax) / 8)
        c0 = comps[0][0]
        fr.grid[c0] = (mcuy, mcux)

        def blocks_of(m):
            return [(c0, [(m // mcux, m % mcux)])]
    else:
        mcux, mcuy = math.ceil(fr.w / (8 * hmax)), math.ceil(fr.h / (8 * vmax))
        for c, _, _ in comps:
            fr.grid[c] = (mcuy * fr.components[c]["v"], mcux * fr.components[c]["h"])

        def blocks_of(m):
            my, mx = divmod(m, mcux)
            out = []
            for c, _, _ in comps:
                hh, vv = fr.components[c]["h"], fr.components[c]["v"]
                out.append((c, [(my * vv + by, mx * hh + bx) for by in range(vv) for bx in range(hh)]))
            return out
    nmcu = mcux * mcuy
    nseg = math.ceil(nmcu / fr.ri) if fr.ri else 1
    # the scan's entropy-coded data: up to the first marker that is not RSTn
    a = np.frombuffer(s, np.uint8, offset=p)
    ff = np.flatnonzero(a[:-1] == 0xFF)
    nxt = a[ff + 1]
    mk = ff[nxt != 0]
    codes = a[mk + 1]
    stop = np.flatnonzero((codes < 0xD0) | (codes > 0xD7))
    assert len(stop), "scan without an end"
    end = int(mk[stop[0]])
    assert codes[stop[0]] in (0xC4, 0xD9, 0xDA, 0xDB, 0xDC, 0xDD, 0xFE) or 0xE0 <= codes[stop[0]] <= 0xEF, \
        f"0xFF in entropy-coded data not followed by 0x00 (FF{codes[stop[0]]:02X} is no marker that may follow a scan)"
    rst = mk[:stop[0]]
    assert len(rst) == nseg - 1, f"{len(rst)} RSTn for {nseg} restart intervals"
    assert (a[rst + 1] == 0xD0 + (np.arange(len(rst)) & 7)).all(), "RSTn do not count modulo 8"
    bounds = [0] + [int(r) + 2 for r in rst]
    ends = [int(r) for r in rst] + [end]
    scan = {"comps": [c for c, _, _ in comps], "blocks_of": blocks_of, "nseg": nseg,
            "dc": [huff[(0, td)] for _, td, _ in comps], "ac": [huff[(1, ta)] for _, _, ta in comps]}
    fr.scans.append({"comps": scan["comps"], "nseg": nseg, "nmcu": nmcu})
    which = range(nseg) if segments is None else segments(len(fr.scans) - 1, nseg)
    for k in which:
        m0 = k * fr.ri if fr.ri else 0
        m1 = min(m0 + fr.ri, nmcu) if fr.ri else nmcu
        _decode_segment(bytes(a[bounds[k]:ends[k]]), fr, scan, range(m0, m1))
    return p + end


def coefficients(fr, c):
    """coefficients of component c on the grid its scan coded, (rows * cols, 64) raster order, and the decoded mask"""
    gh, gw = fr.grid[c]
    return fr.coef[c][:gh, :gw].reshape(-1, 64).astype(np.int64), fr.decoded[c][:gh, :gw].reshape(-1)


# ---- baseline writer ------------------------------------------------------------------------------------------------------------------
class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, code, ln):
        self.acc = (self.acc << ln) | (code & ((1 << ln) - 1))
        self.n += ln
        while self.n >= 8:
            b = (self.acc >> (self.n - 8)) & 255
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)
            self.n -= 8
        self.acc &= (1 << self.n) - 1

    def flush(self, pad=1):
        if self.n:
            self.put(0x7F if pad else 0, 8 - self.n)


def _cat(v):
    return int(abs(int(v))).bit_length()


def _enc_block(bw, blk, pred, dc, ac, zrl_tail=False):
    """T.81 F.1.2 coding of one natural-order block; dc / ac: {symbol: (code, len)}.  zrl_tail: code trailing zeros as ZRL runs (and EOB
    only if positions remain), the corner cases a decoder must accept"""
    zz = [int(blk[n]) for n in ZIGZAG]
    diff = zz[0] - pred
    t = _cat(diff)
    bw.put(*dc[t])
    if t:
        bw.put(diff - 1 if diff < 0 else diff, t)
    run = 0
    for k in range(1, 64):
        v = zz[k]
        if v == 0:
            run += 1
            continue
        while run > 15:
            bw.put(*ac[0xF0])
            run -= 16
        s = _cat(v)
        bw.put(*ac[run << 4 | s])
        bw.put(v - 1 if v < 0 else v, s)
        run = 0
    if run:
        if zrl_tail:
            while run >= 16:
                bw.put(*ac[0xF0])
                run -= 16
            if run:
                bw.put(*ac[0x00])
        else:
            bw.put(*ac[0x00])
    return zz[0]


def _dht(tc, th, bits, vals):
    body = bytes([tc << 4 | th]) + bytes(bits) + bytes(vals)
    return b"\xff\xc4" + (2 + len(body)).to_bytes(2, "big") + body


def write(w, h, components, coef, qtables, tables, scans, ri=0, sof=0xC0, precision=8, adobe=None, between=None, zrl_tail=False, pad=1):
    """components: [(id, h, v, tq)]; coef[c]: (grid rows, grid cols, 64) natural order on the grid each scan codes; qtables {tq: natural 64};
    tables {(tc, th): (bits, vals)}; scans: [[(component index, td, ta), ...], ...]; between {scan number: {(tc, th): (bits, vals)}} = DHT
    segments in front of that scan (tables redefined); adobe: None or the APP14 transform; pad: the padding bit value (0 makes an invalid stream)."""
    out = bytearray(b"\xff\xd8")
    if adobe is not None:
        out += b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00" + bytes([adobe])
    for tq, q in sorted(qtables.items()):
        out += b"\xff\xdb\x00\x43" + bytes([tq]) + bytes(int(q[n]) for n in ZIGZAG)
    nc = len(components)
    out += bytes([0xFF, sof]) + (8 + 3 * nc).to_bytes(2, "big") + bytes([precision]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nc])
    for cid, hh, vv, tq in components:
        out += bytes([cid, hh << 4 | vv, tq])
    for (tc, th), (bits, vals) in sorted(tables.items()):
        out += _dht(tc, th, bits, vals)
    if ri:
        out += b"\xff\xdd\x00\x04" + ri.to_bytes(2, "big")
    hmax, vmax = max(c[1] for c in components), max(c[2] for c in components)
    cur = dict(tables)
    for sn, scan in enumerate(scans):
        for (tc, th), (bits, vals) in sorted((between or {}).get(sn, {}).items()):
            out += _dht(tc, th, bits, vals)
            cur[(tc, th)] = (bits, vals)
        out += b"\xff\xda" + (6 + 2 * len(scan)).to_bytes(2, "big") + bytes([len(scan)])
        for c, td, ta in scan:
            out += bytes([components[c][0], td << 4 | ta])
        out += b"\x00\x3f\x00"
        codes = {key: {sym: (code, ln) for sym, code, ln in _codes(*tv)} for key, tv in cur.items()}
        if len(scan) == 1:
            c = scan[0][0]
            mcux = math.ceil(math.ceil(w * components[c][1] / hmax) / 8)
            mcuy = math.ceil(math.ceil(h * components[c][2] / vmax) / 8)
        else:
            mcux, mcuy = math.ceil(w / (8 * hmax)), math.ceil(h / (8 * vmax))
        nmcu = mcux * mcuy
        bw = _Bits()
        pred = [0] * len(scan)
        for m in range(nmcu):
            if ri and m and m % ri == 0:
                bw.flush(pad)
                bw.out += bytes([0xFF, 0xD0 + ((m // ri - 1) & 7)])
                pred = [0] * len(scan)
            my, mx = divmod(m, mcux)
            for si, (c, td, ta) in enumerate(scan):
                hh, vv = (1, 1) if len(scan) == 1 else components[c][1:3]
                for by in range(vv):
                    for bx in range(hh):
                        pred[si] = _enc_block(bw, coef[c][my * vv + by, mx * hh + bx], pred[si], codes[(0, td)], codes[(1, ta)], zrl_tail)
        bw.flush(pad)
        out += bw.out
    out += b"\xff\xd9"
    return bytes(out)
