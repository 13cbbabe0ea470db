"""numpy restatement of the geometry filters: flip.c, mirror.c, crop.c, vf_split.cpp (split), border.c and
3d-interlaced.c, read from the reference's code.

Each function returns (out, written, undefined) over an output buffer (or, for split, one triple per tile):
  out        the bytes the reference leaves there (0 where it writes nothing),
  written    the bytes it writes,
  undefined  the written bytes whose value comes from memory outside the sources (not defined by the inputs).
The device form writes `written & ~undefined` inside the output frame and nothing else (DESIGN.md §8).
"""
import numpy as np

RGBA, UYVY, YUYV, VUYA, R10k, R12L, v210, DVS10 = 1, 2, 3, 4, 5, 6, 7, 8
RGB, BGR, RG48, Y216, Y416 = 12, 20, 27, 30, 31

# codec_info[] (video_codec.c): block bytes, block pixels, h_align of the codecs with a pixel block
BLOCK = {RGBA: (4, 1, 1), UYVY: (4, 2, 2), YUYV: (4, 2, 2), VUYA: (4, 1, 1), R10k: (4, 1, 64), R12L: (36, 8, 8), v210: (16, 6, 48),
         DVS10: (16, 6, 48), RGB: (3, 1, 1), BGR: (3, 1, 1), RG48: (6, 1, 1), Y216: (8, 2, 2), Y416: (8, 1, 1)}
NAMES = {RGBA: "RGBA", UYVY: "UYVY", YUYV: "YUYV", VUYA: "VUYA", R10k: "R10k", R12L: "R12L", v210: "v210", DVS10: "DVS10", RGB: "RGB",
         BGR: "BGR", RG48: "RG48", Y216: "Y216", Y416: "Y416"}


def linesize(w, c):
    """vc_get_linesize"""
    bb, bp, al = BLOCK[c]
    if al:
        w = (w + al - 1) // al * al
    return (w + bp - 1) // bp * bb


def bpp(c):
    """get_bpp: a double"""
    bb, bp, _ = BLOCK[c]
    return float(bb) / bp


def c_int(x):
    """(int) of a double: truncation toward zero"""
    return int(x)


def c_div(a, b):
    """C integer division: truncation toward zero"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def u32(x):
    return x & 0xFFFFFFFF


def s32(x):
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >> 31 else x


def _gather(src, idx):
    """src[idx] where 0 <= idx < src.size; (values, undefined mask)"""
    bad = (idx < 0) | (idx >= src.size)
    return np.where(bad, 0, src[np.clip(idx, 0, max(src.size - 1, 0))]).astype(np.uint8), bad


# ---- flip (flip.c:77-80) ------------------------------------------------------------------------------------------
def flip(c, src, w, h):
    L = linesize(w, c)
    out = src[:L * h].reshape(h, L)[::-1].reshape(-1).copy()
    return out, np.ones(out.size, bool), np.zeros(out.size, bool)


# ---- mirror (mirror.c:61-79) ---------------------------------------------------------------------------------------
def mirror(c, src, w, h, swap=True):
    L = linesize(w, UYVY)
    if c != UYVY:
        z = np.zeros(L * h, np.uint8)
        return z, np.zeros(z.size, bool), np.zeros(z.size, bool)
    g = src[:L * h].reshape(h, L // 4, 4)[:, ::-1, :]
    out = g[:, :, [0, 3, 2, 1]] if swap else g
    out = np.ascontiguousarray(out).reshape(-1)
    return out, np.ones(out.size, bool), np.zeros(out.size, bool)


# ---- crop (crop.c:118-136, :160-185) ----------------------------------------------------------------------------
def crop_geometry(c, in_w, in_h, width=0, height=0, xoff=0, yoff=0):
    """(out_w, out_h, xoff, yoff) in the reference's arithmetic"""
    bb = BLOCK[c][0]
    ow = (min(width, in_w) if width else in_w)
    oh = (min(height, in_h) if height else in_h)
    ls = c_div(c_int(ow * bpp(c)), bb) * bb
    ow = int(ls / bpp(c))
    xo = (in_w - ow) if u32(u32(xoff) + ow) > in_w else s32(xoff)
    yo = (in_h - oh) if u32(u32(yoff) + oh) > in_h else s32(yoff)
    return ow, oh, xo, yo


def crop(c, src, in_w, in_h, width=0, height=0, xoff=0, yoff=0, pitch=None, xoff_in_pixels=False):
    """pitch None: the capture filter's vc_get_linesize(out_w).  src is the frame alone: reads outside it are undefined
    (before it included, which the device refuses)"""
    ow, oh, xo, yo = crop_geometry(c, in_w, in_h, width, height, xoff, yoff)
    bb = BLOCK[c][0]
    xb = xo if xoff_in_pixels else c_div(c_int(xo * bpp(c)), bb) * bb
    if pitch is None:
        pitch = linesize(ow, c)
    sl = linesize(in_w, c)
    y = np.arange(oh, dtype=np.int64)[:, None]
    j = np.arange(pitch, dtype=np.int64)[None, :]
    idx = ((yo + y) * sl + xb + j).reshape(-1)
    out, bad = _gather(src[:sl * in_h], idx)
    return out, np.ones(out.size, bool), bad


def crop_first_row_offset(c, in_w, in_h, width=0, height=0, xoff=0, yoff=0):
    """yoff * src_linesize + xoff_bytes: negative where the reference's first row starts before the source"""
    _, _, xo, yo = crop_geometry(c, in_w, in_h, width, height, xoff, yoff)
    bb = BLOCK[c][0]
    return yo * linesize(in_w, c) + c_div(c_int(xo * bpp(c)), bb) * bb


# ---- split (vf_split.cpp:14-84) ------------------------------------------------------------------------------------
def split_offsets(c, w, x, rounded=False):
    """the source byte offset of each tile column: `unsigned byte += tile_w * bpp`, truncated at every step"""
    tw = w // x
    offs, byte = [], 0
    for i in range(x):
        offs.append(int(round(i * tw * bpp(c))) if rounded else byte)
        byte = u32(int(float(byte) + tw * bpp(c)))
    return offs


def split(c, src, w, h, x, y, rounded=False):
    """[(tile, written, undefined)] in tile order (tile_row * x + i); each tile is vc_get_linesize(tile_w) * tile_h"""
    assert w % x == 0 and h % y == 0
    tw, th = w // x, h // y
    L, tl = linesize(w, c), linesize(tw, c)
    n = int(tw * bpp(c))
    offs = split_offsets(c, w, x, rounded)
    frame = src[:L * h].reshape(h, L)
    res = []
    for t in range(x * y):
        ty, tx = divmod(t, x)
        tile = np.zeros((th, tl), np.uint8)
        mask = np.zeros((th, tl), bool)
        rows = frame[ty * th:(ty + 1) * th]
        tile[:, :n] = rows[:, offs[tx]:offs[tx] + n]
        mask[:, :n] = True
        res.append((tile.reshape(-1), mask.reshape(-1), np.zeros(tile.size, bool)))
    return res


# ---- border (border.c:104-190) -------------------------------------------------------------------------------------
def border_init(cfg):
    """border_init's parsing: (color bytes, width, height), or None where it refuses cfg.  The colour parser skips one
    character too many: after an optional '#' it requires 6 characters, then reads pairs from the second one."""
    color, bw, bh = [0xFF, 0xFF, 0x00, 0xFF], 10, 10
    if cfg == "help":
        return None
    for item in [i for i in cfg.split(":") if i]:
        low = item.lower()
        if low.startswith("color="):
            col = item[6:]
            if col.startswith("#"):
                col = col[1:]
            if len(col) != 6:
                return None
            col = col[1:] + "\0"
            for i in range(3):
                pair = col[2 * i:2 * i + 2]
                color[i] = _strtol16(pair) & 0xFF
        elif low.startswith("width="):
            bw = u32(u32(_atoi(item[6:])) + 1) // 2 * 2  # unsigned arithmetic: s->width is unsigned
        elif low.startswith("height="):
            bh = u32(u32(_atoi(item[7:])) + 1) // 2 * 2
        else:
            return None
    return bytes(color), bw, bh


def _atoi(s):
    s = s.lstrip(" \t\n\r\f\v")
    m = 0
    sign = 1
    i = 0
    if i < len(s) and s[i] in "+-":
        sign = -1 if s[i] == "-" else 1
        i += 1
    while i < len(s) and s[i].isdigit():
        m = m * 10 + int(s[i])
        i += 1
    return sign * m


def _strtol16(s):
    s = s.split("\0")[0].lstrip(" \t\n\r\f\v")
    sign, i, v = 1, 0, 0
    if i < len(s) and s[i] in "+-":
        sign = -1 if s[i] == "-" else 1
        i += 1
    if s[i:i + 2].lower() == "0x" and len(s) > i + 2 and s[i + 2] in "0123456789abcdefABCDEF":
        i += 2
    while i < len(s) and s[i] in "0123456789abcdefABCDEF":
        v = v * 16 + int(s[i], 16)
        i += 1
    return sign * v


def rgba_to_uyvy_pair(color):
    """vc_copylineRGBAtoUYVY (pixfmt_conv.c:1008-1053 via :2316) over two pixels of the colour, with the BT.709 Q14
    coefficients of color_space.c's COEFFS (:116-128) at 8 bits"""
    kr, kb = .212639, .072192
    kg = 1. - kr - kb
    dd, ee = 2. * (kr + kg), 2. * (1. - kr)
    yl, cl, B = 219. * 1 / 255, 224. * 1 / 255, float(1 << 14)
    y_r, y_g, y_b = int(kr * yl * B + 0.5), int(kg * yl * B + 0.5), int(kb * yl * B + 0.5)
    cb_r, cb_g, cb_b = int(-kr / dd * cl * B - 0.5), int(-kg / dd * cl * B - 0.5), int((1 - kb) / dd * cl * B + 0.5)
    cr_r, cr_g, cr_b = int((1 - kr) / ee * cl * B - 0.5), int(-kg / ee * cl * B - 0.5), int(-kb / ee * cl * B + 0.5)
    r, g, b = color[0], color[1], color[2]
    y = ((r * y_r + g * y_g + b * y_b) >> 14) + 16
    u = (c_div(2 * (r * cb_r + g * cb_g + b * cb_b), 2) >> 14) + 128
    v = (c_div(2 * (r * cr_r + g * cr_g + b * cr_b), 2) >> 14) + 128
    return bytes([u & 0xFF, y & 0xFF, v & 0xFF, y & 0xFF])


def border(c, src, w, h, color, bw, bh):
    """rows [bh, h - bh) copied, then the fill over the top and bottom bh rows and the side bands"""
    L = linesize(w, c)
    out = np.zeros((h, L), np.uint8)
    written = np.zeros((h, L), bool)
    frame = src[:L * h].reshape(h, L)
    out[bh:h - bh] = frame[bh:h - bh]
    written[bh:h - bh] = True
    if c not in (UYVY, RGB, RGBA):
        return out.reshape(-1), written.reshape(-1), np.zeros(out.size, bool)
    if c == UYVY:
        pat = np.frombuffer(rgba_to_uyvy_pair(color), np.uint8)
        band = (bw + 1) // 2 * 4
    else:
        p = 3 if c == RGB else 4
        pat = np.frombuffer(bytes(color[:p]), np.uint8)
        band = bw * p
    fill = np.resize(pat, L)
    out[:bh] = fill
    out[h - bh:] = fill
    out[:, :band] = fill[:band]
    out[:, L - band:] = fill[L - band:]
    written[:] = True
    return out.reshape(-1), written.reshape(-1), np.zeros(out.size, bool)


def border_band_bytes(c, bw):
    return (bw + 1) // 2 * 4 if c == UYVY else bw * (3 if c == RGB else 4)


# ---- interlaced_3d (3d-interlaced.c:142-163) ----------------------------------------------------------------------
def interlaced_3d(c, left, right, w, h, drift=True, truncate=False):
    """over the h * ceil(L / 16) * 16 bytes the reference writes from the frame's start"""
    L = linesize(w, c)
    cpr = (L + 15) // 16
    pitch = cpr * 16 if drift else L
    n = (h - 1) * pitch + cpr * 16
    out = np.zeros(n, np.uint8)
    written = np.zeros(n, bool)
    undefined = np.zeros(n, bool)
    j = np.arange(cpr * 16, dtype=np.int64)
    for x in range(h):
        tile = (left if x % 2 == 0 else right)[:L * h]
        r = x // 2 * 2
        a, ba = _gather(tile, r * L + j)
        b, bb_ = _gather(tile, (r + 1) * L + j)
        s = a.astype(np.uint16) + b
        v = (s >> 1) if truncate else ((s + 1) >> 1)
        out[x * pitch:x * pitch + cpr * 16] = v.astype(np.uint8)
        written[x * pitch:x * pitch + cpr * 16] = True
        undefined[x * pitch:x * pitch + cpr * 16] = ba | bb_
    return out, written, undefined
