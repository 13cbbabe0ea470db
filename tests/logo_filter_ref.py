"""numpy restatement of the logo capture filter (logo.c) and the R12L <-> Y416 pass-through filters
(r12l_to_y416_fake.c, y416_to_r12l_fake.c), read from the reference's code and the line converters
(pixfmt_conv.c) logo.c takes from get_decoder_from_to.

logo() returns (frame, written) for a frame it changes in place: the frame after the filter and the bytes the
filter writes.  Logo widths whose RGB segment the reference allocates too short are given the reference's result
with a long enough segment (DESIGN.md §8); logo_handled() says which widths the reference itself handles.
"""
import numpy as np

from geometry_filter_ref import RGBA, UYVY, YUYV, R10k, R12L, v210, RGB, BGR, RG48, Y416, BLOCK, NAMES, c_div, linesize  # noqa: F401

LOGO_CODECS = (RGB, RGBA, UYVY, RG48, R12L)


# ---- colour_space.c's COEFFS at 8 bits (BT.709), Q14 ----------------------------------------------------------------
def _coeffs():
    kr, kb = .212639, .072192
    kg, B = 1. - kr - kb, 16384.
    dd, ee = 2. * (kr + kg), 2. * (1. - kr)
    yl, cl = 219. / 255, 224. / 255

    def scaled(x):
        return int(x * B + (1. if x > 0 else -1.) * 0.5)
    return dict(y_r=int(kr * yl * B + 0.5), y_g=int(kg * yl * B + 0.5), y_b=int(kb * yl * B + 0.5),
                cb_r=int(-kr / dd * cl * B - 0.5), cb_g=int(-kg / dd * cl * B - 0.5), cb_b=int((1 - kb) / dd * cl * B + 0.5),
                cr_r=int((1 - kr) / ee * cl * B - 0.5), cr_g=int(-kg / ee * cl * B - 0.5), cr_b=int(-kb / ee * cl * B + 0.5),
                y_scale=scaled(1. / yl), r_cr=scaled(2. * (1. - kr) / cl), g_cb=scaled((-kb * 2. * (kr + kg) / kg) / cl),
                g_cr=scaled((-kr * 2. * (1. - kr) / kg) / cl), b_cb=scaled(2. * (kr + kg) / cl))


K = _coeffs()


def _tdiv2(x):
    """C's x / 2 on int arrays: truncation toward zero"""
    return np.where(x < 0, -((-x) // 2), x // 2)


# ---- R12L: 8 pixels x (R, G, B) x 12 bits in 36 bytes, component k at bit 12k --------------------------------------
def r12_unpack(groups):
    """(..., 36) uint8 -> (..., 8, 3) int: the 12-bit samples"""
    g = groups.astype(np.int64)
    out = np.empty(g.shape[:-1] + (24,), np.int64)
    for k in range(24):
        b, sh = 12 * k // 8, 12 * k % 8
        out[..., k] = ((g[..., b] | g[..., b + 1] << 8) >> sh) & 0xFFF
    return out.reshape(g.shape[:-1] + (8, 3))


def r12_pack(px):
    """(..., 8, 3) 12-bit ints -> (..., 36) uint8"""
    v = px.reshape(px.shape[:-2] + (24,)).astype(np.int64)
    out = np.zeros(px.shape[:-2] + (36,), np.int64)
    for k in range(24):
        b, sh = 12 * k // 8, 12 * k % 8
        out[..., b] |= (v[..., k] << sh) & 0xFF
        out[..., b + 1] |= (v[..., k] << sh) >> 8
    return out.astype(np.uint8)


# ---- the line converters logo.c uses, over (rows, bytes) spans; default shifts ----------------------------------------
def decode(c, span, n, aux=None):
    """get_decoder_from_to(c, RGB) over the first n pixels of each row of `span` (rows, bytes): (rows, n, 3) int.
    RGBA: vc_copylineRGBAtoRGB's SSSE3 build, whose scalar tail (pixfmt_conv.c:889-895) never advances src, so every
    pixel from `aux` on is pixel aux"""
    s = span.astype(np.int64)
    rows = s.shape[0]
    if c == RGB:
        return s[:, :3 * n].reshape(rows, n, 3)
    if c == RGBA:
        idx = np.arange(n)
        if aux is not None:
            idx = np.minimum(idx, aux)
        return s[:, :4 * n].reshape(rows, n, 4)[:, idx, :3]
    if c == RG48:
        return s[:, :6 * n].reshape(rows, n, 6)[:, :, 1::2]
    if c == UYVY:  # copylineYUVtoRGB (:1065-1094)
        q = s[:, :2 * n].reshape(rows, n // 2, 4)
        u, v = q[..., 0] - 128, q[..., 2] - 128
        out = np.empty((rows, n // 2, 2, 3), np.int64)
        for i, yo in enumerate((1, 3)):
            y = K["y_scale"] * (q[..., yo] - 16)
            out[:, :, i, 0] = np.clip((y + v * K["r_cr"]) >> 14, 0, 255)
            out[:, :, i, 1] = np.clip((y + u * K["g_cb"] + v * K["g_cr"]) >> 14, 0, 255)
            out[:, :, i, 2] = np.clip((y + u * K["b_cb"]) >> 14, 0, 255)
        return out.reshape(rows, n, 3)
    if c == R12L:  # vc_copylineR12LtoRGB (:353-430): the high 8 bits
        return (r12_unpack(s[:, :36 * (n // 8)].reshape(rows, n // 8, 36)) >> 4).reshape(rows, n, 3)
    raise ValueError(c)


def encode(c, rgb, keep_alpha=None, keep_low=None):
    """get_decoder_from_to(RGB, c) over (rows, n, 3), n whole blocks of c: (rows, vc_get_linesize(n)) uint8.
    keep_alpha / keep_low (mutants): the frame's own alpha (RGBA) or low bytes (RG48) instead of 0xFF / 0"""
    rows, n, _ = rgb.shape
    if c == RGB:  # vc_copylineRGB: memcpy
        return rgb.reshape(rows, 3 * n).astype(np.uint8)
    if c == RGBA:  # vc_copylineRGBtoRGBA (:944-990): alpha 0xFF
        a = np.full((rows, n, 1), 0xFF, np.int64) if keep_alpha is None else keep_alpha[..., None]
        return np.concatenate([rgb, a], axis=2).reshape(rows, 4 * n).astype(np.uint8)
    if c == RG48:  # vc_copylineRGBtoRG48 (:1353-1363): the low byte 0
        lo = np.zeros_like(rgb) if keep_low is None else keep_low
        return np.stack([lo, rgb], axis=3).reshape(rows, 6 * n).astype(np.uint8)
    if c == UYVY:  # vc_copylineToUYVY (:1008-1053)
        p = rgb.reshape(rows, n // 2, 2, 3)
        r, g, b = p[..., 0], p[..., 1], p[..., 2]
        y = ((r * K["y_r"] + g * K["y_g"] + b * K["y_b"]) >> 14) + 16
        cb = (r * K["cb_r"] + g * K["cb_g"] + b * K["cb_b"]).sum(axis=2)
        cr = (r * K["cr_r"] + g * K["cr_g"] + b * K["cr_b"]).sum(axis=2)
        u, v = (_tdiv2(cb) >> 14) + 128, (_tdiv2(cr) >> 14) + 128
        return (np.stack([u, y[..., 0], v, y[..., 1]], axis=2) & 0xFF).reshape(rows, 2 * n).astype(np.uint8)
    if c == R12L:  # vc_copylineRGB_AtoR12L (:1258-1334): 8-bit << 4
        return r12_pack(rgb.reshape(rows, n // 8, 8, 3) << 4).reshape(rows, 36 * (n // 8))
    raise ValueError(c)


# ---- logo (logo.c:162-235) ----------------------------------------------------------------------------------------------
def block_px(c):
    return BLOCK[c][1]


def round_up(x, m):
    return (x + m - 1) // m * m


def logo_handled(c, w):
    """the logo widths whose segment rows, dec_width = (w + 1) / bb * bb pixels, hold round_up(w, block pixels)
    pixels and which the decoder fills: for the others the reference writes past its malloc"""
    bb = BLOCK[c][0]
    dec = (w + 1) // bb * bb
    n = round_up(w, block_px(c))
    if dec < n:
        return False
    return c != R12L or (3 * dec) % 24 == 0  # vc_copylineR12LtoRGB decodes whole 24-byte runs of dst_len


def logo_padded_width(c, w):
    """the next logo width >= w that the reference handles"""
    while not logo_handled(c, w):
        w += 1
    return w


def logo_place(c, W, H, w, h, x, y, pixel_align=False):
    """(rc, rect_x, rect_y, off, span): rc 0 writes, 1 returns without writing (a negative rect), -1 the span passes
    the end of the row (the device refuses it).  pixel_align (mutant): rect_x aligned to block pixels"""
    rect_x, rect_y = x, y
    if rect_x < 0 or rect_x + w > W:
        rect_x = W - w
    bb = block_px(c) if pixel_align else BLOCK[c][0]
    rect_x = c_div(rect_x, bb) * bb
    if rect_y < 0 or rect_y + h > H:
        rect_y = H - h
    if rect_x < 0 or rect_y < 0:
        return 1, rect_x, rect_y, 0, 0
    off, span = linesize(rect_x, c), linesize(w, c)
    if off + span > linesize(W, c):
        return -1, rect_x, rect_y, off, span
    return 0, rect_x, rect_y, off, span


def logo(c, frame, W, H, rgba, x=-1, y=-1, rounding=False, keep_alpha=False, keep_low=False, pixel_align=False):
    """(frame after the filter, written) for the h x w x 4 logo `rgba`, or None where the device refuses (-1).
    Mutants: rounding (+127 before / 255), keep_alpha, keep_low, pixel_align"""
    h, w, _ = rgba.shape
    L = linesize(W, c)
    out = frame.copy()
    written = np.zeros(frame.size, bool)
    rc, _, ry, off, span = logo_place(c, W, H, w, h, x, y, pixel_align)
    if rc == -1:
        return None
    if rc == 1:
        return out, written
    n = round_up(w, block_px(c))  # the pixels of the span
    rows = out.reshape(H, L)[ry:ry + h, off:off + span]
    aux = None
    if c == RGBA:  # vc_copylineRGBAtoRGB's first tail pixel at dst_len = 3 * d, d = w rounded up to whole blocks
        d = round_up(w, BLOCK[c][0])
        aux = ((3 * d - 24) // 12 + 1) * 4 if 3 * d >= 24 else 0
    rgb = decode(c, rows, n, aux)
    p = rgb[:, :w]
    a = rgba[:, :, 3:4].astype(np.int64)
    p[:] = (p * (255 - a) + rgba[:, :, :3].astype(np.int64) * a + (127 if rounding else 0)) // 255
    ka = rows.reshape(h, n, 4)[:, :, 3].astype(np.int64) if c == RGBA and keep_alpha else None
    kl = rows.reshape(h, n, 6)[:, :, 0::2].astype(np.int64) if c == RG48 and keep_low else None
    out.reshape(H, L)[ry:ry + h, off:off + span] = encode(c, rgb, ka, kl)
    written.reshape(H, L)[ry:ry + h, off:off + span] = True
    return out, written


# ---- r12l_to_y416_fake (r12l_to_y416_fake.c:85-191) and y416_to_r12l_fake (y416_to_r12l_fake.c:117-238) -------------
def r12l_to_y416(src, w, h, full_range, y_scale=13, c_scale=14):
    """tight R12L -> tight Y416 as uint8: (R', G', B', 0xFFFF) per pixel"""
    px = r12_unpack(src[:linesize(w, R12L) * h].reshape(-1, 36)).reshape(-1, 3)
    if full_range:
        v = px << 4
    else:
        v = px * np.array([c_scale, y_scale, c_scale]) + 4096
    out = np.concatenate([v, np.full((v.shape[0], 1), 0xFFFF)], axis=1).astype(np.uint16)
    return out.reshape(-1).view(np.uint8)


def y416_to_r12l(src, w, h, full_range, pitch, y_scale=13, c_scale=14):
    """tight Y416 -> R12L rows at `pitch` (row y at y * pitch, one task's layout): (bytes, written) over
    (h - 1) * pitch + vc_get_linesize(w, R12L) bytes"""
    L = linesize(w, R12L)
    v = src[:8 * w * h].view(np.uint16).reshape(-1, 4)[:, :3].astype(np.int64)
    if full_range:
        v = v >> 4
    else:
        v = (np.maximum(v, 4096) - 4096) // np.array([c_scale, y_scale, c_scale])
    packed = r12_pack(np.minimum(v, 4095).reshape(h, w // 8, 8, 3)).reshape(h, L)
    n = (h - 1) * pitch + L
    out = np.zeros(h * pitch, np.uint8)
    written = np.zeros(h * pitch, bool)
    out.reshape(h, pitch)[:, :L] = packed
    written.reshape(h, pitch)[:, :L] = True
    return out[:n], written[:n]
