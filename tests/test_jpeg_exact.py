"""The JPEG encoder's DCT and the decoder's IDCT against the exact T.81 transforms, read through an independent stream reader
(tests/jpeg_exact.py).  Every other arithmetic test of the codec compares the kernels with the CPU oracles, which share the transform and
the entropy coder with them by design; these tests do not.  A coefficient must be round_half_even(F / Q) of the exact float64 DCT of the
edge-padded block, a decoded sample clamp(round(IDCT(coef x Q) + 128)); the only exemption is a value within the derived tie band of a
half-integer (jpeg_exact.py), where float32 may round the other way, and the share of such exemptions is bounded.
  * CPU: the reader against the oracle's coefficients and libjpeg (PIL), writer -> reader round trips, the CPU oracles against the exact
    transforms, the band's derivation re-measured, and perturbed transforms / arrays that the comparators must report;
  * GPU: the encoder's streams of every layout, size class, restart interval and route, and the decoder's output for the encoder's streams,
    libjpeg's streams and writer-made streams (extreme coefficients, ZRL / EOB corners, long and 9-bit codes, tables redefined between
    scans), through both marker scans; refusals."""
import ctypes
import io
import os
import re
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

import jpeg_exact as J
import util
from test_jpeg import RGB, UYVY, extreme_ac_frame, natural_rgb, orc_encode, orc_encode_interleaved_rgb
from test_jpeg_planar import I420, prep, source
from test_jpeg_planar import pl  # noqa: F401  (fixture: the planar oracle, for orc_jpeg_prep)
from test_jpeg_alpha import al, oracle_stream as alpha_stream, rgba_frame  # noqa: F401  (fixture al: the alpha oracle)
from test_jpeg_planar import oracle_stream as planar_stream

RGBA, VUYA = 1, 4
CS = {"native": 0, "Y601": 1, "Y601full": 2, "Y709": 3, "RGB": 4}
EXEMPT_SHARE = 0.01  # band exemptions per value compared; the CPU oracle reaches 0.36 % (RGB noise at q = 100), natural content far less


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


def dc_swing_frame(w, h, n=3):
    """alternating flat 0 and 255 blocks: DC differences of 2040 at q = 100 (category 11) in every component"""
    yy, xx = np.mgrid[0:h, 0:w]
    p = np.where(((xx // 8) + (yy // 8)) % 2 == 0, 0, 255).astype(np.uint8)
    return np.repeat(p[:, :, None], n, axis=2)


def natural_with_noise(w, h, seed, n=3):
    f = natural_rgb(w, h, seed)
    if n == 4:
        f = rgba_frame(w, h, seed)
    f = np.ascontiguousarray(f).copy()
    f[:min(h, 8)] = np.random.default_rng(seed).integers(0, 256, f[:min(h, 8)].shape, dtype=np.uint8)  # long codes, ZRL, 0xFF stuffing
    return f


# ---- checks --------------------------------------------------------------------------------------------------------------------
def check_encoded(stream, planes, quality=None, what="", segments=None, stats=None):
    """every coefficient of the stream == round_half_even(exact DCT / Q) of the edge-padded planes, outside the band"""
    fr = J.read(stream, segments)
    assert len(fr.components) == len(planes), what
    if quality is not None:
        assert np.array_equal(fr.q[0], J.scaled_qtable(J.Q_LUMA, quality)) and np.array_equal(fr.q[1], J.scaled_qtable(J.Q_CHROMA, quality)), what
    tot = {"n": 0, "exempt": 0, "worst": -1.0}
    for c, plane in enumerate(planes):
        got, mask = J.coefficients(fr, c)
        gh, gw = fr.grid[c]
        q = fr.q[fr.components[c]["tq"]]
        b = J.pad_blocks(plane, gh, gw)[mask]
        st = J.compare_coefficients(got[mask], J.fdct(b) / q, J.enc_band(b, q), f"{what} component {c}")
        tot["n"] += st["n"]
        tot["exempt"] += st["exempt"]
        tot["worst"] = max(tot["worst"], st["worst"])
    assert tot["exempt"] <= EXEMPT_SHARE * tot["n"], (what, tot)
    if stats is not None:
        stats.append((what, tot))
    return fr


def exact_planes(fr):
    """per component: (exact samples, band) on the component's sample grid ceil(X Hi / Hmax) x ceil(Y Vi / Vmax)"""
    hmax, vmax = max(c["h"] for c in fr.components), max(c["v"] for c in fr.components)
    out = []
    for c, cc in enumerate(fr.components):
        got, mask = J.coefficients(fr, c)
        assert mask.all()
        gh, gw = fr.grid[c]
        q = fr.q[cc["tq"]]
        px = J.idct(got * q[None, :]).reshape(gh, gw, 8, 8).transpose(0, 2, 1, 3).reshape(gh * 8, gw * 8)
        band = np.asarray(J.dec_band(got, q)).reshape(gh, gw, 8, 8).transpose(0, 2, 1, 3).reshape(gh * 8, gw * 8)
        ph, pw = -(-fr.h * cc["v"] // vmax), -(-fr.w * cc["h"] // hmax)
        out.append((px[:ph, :pw], band[:ph, :pw]))
    return out


def check_decoded(stream, planes, what=""):
    """decoded planes (the output's bytes, per component) against the exact IDCT of the stream's coefficients (the share of exemptions is
    not bounded for the stream made of exact ties)"""
    fr = J.read(stream)
    ex = exact_planes(fr)
    assert len(planes) == len(ex), what
    tot = {"n": 0, "exempt": 0, "worst": -1.0}
    for c, ((px, band), got) in enumerate(zip(ex, planes)):
        st = J.compare_samples(got[:px.shape[0], :px.shape[1]], px, band, f"{what} component {c}")
        assert got.shape[0] >= px.shape[0] and got.shape[1] >= px.shape[1], (what, c, got.shape, px.shape)
        for k in st:
            tot[k] = max(tot[k], st[k]) if k == "worst" else tot[k] + st[k]
    assert tot["exempt"] <= EXEMPT_SHARE * tot["n"] or what.startswith("dc-half"), (what, tot)
    return tot


def output_planes(out, fr, codec):
    """the component planes held by a decoder output of `codec` (the stream's native layout)"""
    w, h = fr.w, fr.h
    if codec == RGB:
        return J.packed_planes(out[:w * h * 3], w, h, 3)
    if codec == RGBA:
        return J.packed_planes(out[:w * h * 4], w, h, 4)
    if codec == VUYA:
        a = np.asarray(out[:w * h * 4]).reshape(h, w, 4)
        return [a[:, :, 2], a[:, :, 1], a[:, :, 0]]
    if codec == UYVY:
        return J.uyvy_planes(out, w, h)
    assert codec == I420
    return J.i420_planes(out, w, h)


# ---- stream corpus: (name, stream, component planes the encoder saw) -----------------------------------------------------------
LAYOUTS = ["uyvy422", "rgb", "rgb-il", "i420", "uyvy420"] + [f"{cs}-{sub}-{il}" for cs in ("Y709", "Y601full") for sub in (444, 422, 420) for il in (0, 1)] + \
          ["rgba", "rgba-il"]


def layout_params(name):
    """(codec, subsampling, colour space, interleaved)"""
    fixed = {"uyvy422": (UYVY, 0, "native", 0), "rgb": (RGB, 0, "native", 0), "rgb-il": (RGB, 0, "native", 1), "i420": (I420, 0, "native", 1),
             "uyvy420": (UYVY, 420, "native", 1), "rgba": (RGBA, 4444, "native", 0), "rgba-il": (RGBA, 4444, "native", 1)}
    if name in fixed:
        return fixed[name]
    cs, sub, il = name.split("-")
    return RGB, int(sub), cs, int(il)


def layout_source(orc, name, w, h, content, seed):
    """the source frame (flat uint8) of a layout"""
    codec, _, _, _ = layout_params(name)
    n = 4 if codec == RGBA else 3
    rgb = {"natural": lambda: natural_with_noise(w, h, seed, n), "noise": lambda: np.random.default_rng(seed).integers(0, 256, (h, w, n), dtype=np.uint8),
           "extreme": lambda: extreme_ac_frame(RGB, w, h).reshape(h, w, 3), "dcswing": lambda: dc_swing_frame(w, h, n)}[content]()
    if content == "extreme" and n == 4:
        rgb = np.dstack([rgb, rgb[:, :, :1]])
    rgb = np.ascontiguousarray(rgb)
    if codec in (RGB, RGBA):
        return rgb.reshape(-1).copy()
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, rgb.reshape(-1), w, h)
    if content in ("extreme", "dcswing"):  # the pattern straight into the planes, not through the colour conversion
        y = rgb[:, :, 0]
        u = uyvy.reshape(h, -1, 4)
        u[:, :, 1], u[:, :, 3] = y[:, 0::2][:, :u.shape[1]], np.pad(y[:, 1::2], ((0, 0), (0, u.shape[1] - y[:, 1::2].shape[1])), mode="edge")
        u[:, :, 0], u[:, :, 2] = y[:, 0::2][:, :u.shape[1]], 255 - y[:, 0::2][:, :u.shape[1]]
        uyvy = u.reshape(-1).copy()
    if codec == UYVY:
        return uyvy
    planes = J.uyvy_to_i420_planes(uyvy, w, h)
    return np.concatenate([p.reshape(-1) for p in planes])


def layout_planes(pl, name, src, w, h):
    codec, sub, cs, _ = layout_params(name)
    if name == "uyvy422":
        return J.uyvy_planes(src, w, h)
    if codec == RGB and cs == "native":
        return J.packed_planes(src, w, h, 3)
    if codec == RGBA:
        return J.packed_planes(src, w, h, 4)
    if codec == I420:
        return J.i420_planes(src, w, h)
    if codec == UYVY:
        return J.uyvy_to_i420_planes(src, w, h)
    hs, vs = (2 if sub in (422, 420) else 1), (2 if sub == 420 else 1)
    p = prep(pl, src, w, h, RGB, sub, cs)  # orc_jpeg_prep: pinned to rgb_to_yuv444p by test_jpeg_planar.py
    cw, ch = -(-w // hs), -(-h // vs)
    return [p[0].reshape(h, w), p[1].reshape(ch, cw), p[2].reshape(ch, cw)]


def oracle_layout_stream(orc, pl, al, name, src, w, h, q, ri):
    codec, sub, cs, il = layout_params(name)
    if name == "uyvy422":
        return orc_encode(orc, src, w, h, UYVY, q, ri, pitch=(w + 1) // 2 * 4)
    if name == "rgb":
        return orc_encode(orc, src, w, h, RGB, q, ri)
    if name == "rgb-il":
        return orc_encode_interleaved_rgb(orc, src, w, h, q, ri)
    if codec == RGBA:
        return alpha_stream(al, src, w, h, q, ri, il)
    return planar_stream(pl, src, w, h, codec, sub, cs, q, ri, il)


# ---- CPU: the reader -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", [UYVY, RGB])
@pytest.mark.parametrize("w,h", [(1, 1), (17, 9), (130, 37), (64, 64)])
def test_reader_equals_oracle_coefficients(orc, codec, w, h):
    """the one use of the oracle here: the reader's coefficients of an oracle stream are orc_jpeg_coefficients, block for block"""
    name = "uyvy422" if codec == UYVY else "rgb"
    src = layout_source(orc, name, w, h, "natural", w + h)
    pitch = (w + 1) // 2 * 4 if codec == UYVY else w * 3
    for q, ri in ((1, 0), (90, 3), (100, 1)):
        fr = J.read(orc_encode(orc, src, w, h, codec, q, ri, pitch=pitch))
        nblk = (-(-w // 16)) * (-(-h // 8)) * 4 if codec == UYVY else (-(-w // 8)) * (-(-h // 8)) * 3
        ref = np.zeros(nblk * 64, np.int16)
        orc.orc_jpeg_coefficients.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        orc.orc_jpeg_coefficients(src.ctypes.data, pitch, w, h, 0 if codec == UYVY else 1, q, ref.ctypes.data)
        nat = np.zeros((nblk, 64), np.int64)
        nat[:, J.ZIGZAG] = ref.reshape(-1, 64)
        if codec == RGB:
            mine = np.concatenate([J.coefficients(fr, c)[0] for c in range(3)])
        else:  # MCU order Y0 Y1 Cb Cr
            y, cb, cr = (fr.coef[c] for c in range(3))
            mh, mw = cb.shape[:2]
            mine = np.stack([y[:, 0::2].reshape(mh, mw, 64), y[:, 1::2].reshape(mh, mw, 64), cb, cr], axis=2).reshape(-1, 64)
        assert np.array_equal(mine, nat), (q, ri)


PIL_CASES = [("444", {"subsampling": 0}), ("422", {"subsampling": 1}), ("420", {"subsampling": 2}), ("420-opt", {"subsampling": 2, "optimize": True}),
             ("444-q1", {"subsampling": 0, "qtables": [[1] * 64] * 2}), ("420-q255", {"subsampling": 2, "qtables": [[255] * 64] * 2}),
             ("422-rst-blocks", {"subsampling": 1, "restart_marker_blocks": 3}), ("420-rst-rows", {"subsampling": 2, "restart_marker_rows": 1}),
             ("444-rst-rows", {"subsampling": 0, "restart_marker_rows": 2})]


def pil_stream(kind, w, h, seed=4, quality=85):
    kw = dict(PIL_CASES)[kind]
    b = io.BytesIO()
    Image.fromarray(natural_with_noise(w, h, seed)).save(b, "JPEG", quality=quality, **kw)
    return b.getvalue()


@pytest.mark.parametrize("kind", [k for k, _ in PIL_CASES])
def test_reader_on_libjpeg_streams(kind):
    """libjpeg's streams (its own Huffman tables with optimize, extreme quantisers, restart markers by blocks and by rows, no DRI): the exact
    IDCT of the reader's coefficients is within 1 of libjpeg's decode - luma always, all three components at 4:4:4 (libjpeg upsamples
    subsampled chroma with its own filter)"""
    for w, h in ((200, 120), (37, 21)):
        s = pil_stream(kind, w, h)
        fr = J.read(s)
        im = Image.open(io.BytesIO(s))
        im.draft("YCbCr", (w, h))
        lib = np.asarray(im).astype(np.int64)
        ex = exact_planes(fr)
        for c in (range(3) if kind.startswith("444") else range(1)):
            mine = np.clip(np.rint(ex[c][0]), 0, 255)
            assert np.abs(mine - lib[:, :, c]).max() <= 1, (kind, w, h, c)


def _writer_frame(w, h, hs=1, vs=1, rng=None, scale=30):
    rng = rng or np.random.default_rng(0)
    mw, mh = -(-w // (8 * hs)), -(-h // (8 * vs))
    shapes = [(mh * vs, mw * hs), (mh, mw), (mh, mw)]
    coef = []
    for gh, gw in shapes:
        c = np.zeros((gh, gw, 64), np.int64)
        c[..., 0] = rng.integers(-400, 400, (gh, gw))
        n = rng.integers(0, 64, (gh, gw))
        for k in range(1, 64):
            c[..., J.ZIGZAG[k]] = np.where(k < n, rng.integers(-scale, scale + 1, (gh, gw)), 0)
        coef.append(c)
    return coef


STD_TABLES = {(0, 0): J.DC_LUMA, (1, 0): J.AC_LUMA, (0, 1): J.DC_CHROMA, (1, 1): J.AC_CHROMA}


@pytest.mark.parametrize("hs,vs,il,ri", [(1, 1, 0, 0), (1, 1, 1, 3), (2, 1, 1, 1), (2, 2, 1, 7), (2, 2, 0, 5), (2, 1, 0, 0)])
def test_writer_reader_round_trip(hs, vs, il, ri):
    w, h = 45, 27
    coef = _writer_frame(w, h, hs, vs)
    comps = [(1, hs, vs, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
    scans = [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]] if il else [[(0, 0, 0)], [(1, 1, 1)], [(2, 1, 1)]]
    s = J.write(w, h, comps, coef, {0: np.full(64, 3), 1: np.full(64, 5)}, STD_TABLES, scans, ri=ri)
    fr = J.read(s)
    for c in range(3):
        got, mask = J.coefficients(fr, c)
        gh, gw = fr.grid[c]
        assert mask.all() and np.array_equal(got, coef[c][:gh, :gw].reshape(-1, 64)), c
    assert fr.scans[0]["nseg"] == (-(-fr.scans[0]["nmcu"] // ri) if ri else 1)


def test_reader_asserts_restart_markers(orc):
    """a misnumbered RSTn and a missing one are refused"""
    w, h = 64, 16
    src = layout_source(orc, "rgb", w, h, "noise", 3)
    s = bytearray(orc_encode(orc, src, w, h, RGB, 90, 1))
    J.read(bytes(s))
    rst = [i for i in range(len(s) - 1) if s[i] == 0xFF and 0xD0 <= s[i + 1] <= 0xD7]
    bad = bytearray(s)
    bad[rst[3] + 1] = 0xD0 + ((bad[rst[3] + 1] - 0xD0 + 1) & 7)
    with pytest.raises(AssertionError, match="modulo 8"):
        J.read(bytes(bad))
    with pytest.raises(AssertionError, match="RSTn for"):
        J.read(bytes(s[:rst[3]] + s[rst[3] + 2:]))


def test_reader_asserts_stuffing_and_padding():
    """an 0xFF of entropy-coded data without its stuffed 0x00, and 0-bit padding before RSTn / EOI, are refused"""
    w, h = 37, 21
    coef = _writer_frame(w, h, rng=np.random.default_rng(2), scale=300)
    args = (w, h, [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef, {0: np.full(64, 1), 1: np.full(64, 1)}, STD_TABLES, [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]])
    s = J.write(*args, ri=1)
    J.read(s)
    sos = s.index(b"\xff\xda")
    stuffed = s.index(b"\xff\x00", sos)
    with pytest.raises(AssertionError, match="not followed by 0x00"):
        J.read(s[:stuffed + 1] + b"\x12" + s[stuffed + 2:])
    with pytest.raises(AssertionError, match="padding bits are not 1-bits"):
        J.read(J.write(*args, ri=1, pad=0))


def _hand_coded(items, dc_table):
    """a 8x8 one-component stream whose single block is the given symbols: [("dc" | "ac" | "raw", symbol or bits, value, value bits)]"""
    ac_table = ([0] * 7 + [len(J.AC_LUMA[1]) + 1] + [0] * 8, J.AC_LUMA[1] + [0x0B])  # Annex K symbols and AC category 11, all 8 bits long
    tables = {(0, 0): dc_table, (1, 0): ac_table}
    head = J.write(8, 8, [(1, 1, 1, 0)], [np.zeros((1, 1, 64), np.int64)], {0: np.full(64, 1)}, tables, [[(0, 0, 0)]])
    sos = head.index(b"\xff\xda")
    data0 = sos + 2 + (head[sos + 2] << 8 | head[sos + 3])
    codes = {"dc": {v: (c, n) for v, c, n in J._codes(*dc_table)}, "ac": {v: (c, n) for v, c, n in J._codes(*ac_table)}}
    bw = J._Bits()
    for kind, sym, val, nbits in items:
        bw.put(*((sym, nbits) if kind == "raw" else codes[kind][sym]))
        if kind != "raw" and nbits:
            bw.put(val, nbits)
    bw.flush()
    return head[:data0] + bytes(bw.out) + b"\xff\xd9"


DC_13 = ([0, 0, 0, 13] + [0] * 12, list(range(13)))  # DC categories 0..12, all 4 bits long


@pytest.mark.parametrize("items,dc_table,message", [
    ([("dc", 0, 0, 0), ("ac", 0x01, 1, 1), ("ac", 0xF0, 0, 0), ("ac", 0xF0, 0, 0), ("ac", 0xF0, 0, 0), ("ac", 0xF1, 1, 1)], DC_13, "run past position 63"),
    ([("dc", 0, 0, 0), ("ac", 0x01, 1, 1)] + [("ac", 0xF0, 0, 0)] * 4, DC_13, "ZRL past position 63"),
    ([("dc", 0, 0, 0), ("ac", 0x0B, 1500, 11), ("ac", 0x00, 0, 0)], DC_13, "AC category 11"),
    ([("dc", 12, 3000, 12), ("ac", 0x00, 0, 0)], DC_13, "DC category 12"),
    ([("raw", 0b111, 0, 3)], ([0, 1] + [0] * 14, [0]), "undefined DC code"),
    ([("dc", 0, 0, 0), ("raw", 0xFF, 0, 8)], DC_13, "undefined AC code"),
])
def test_reader_asserts_symbols(items, dc_table, message):
    """a run past position 63, an AC category above 10, a DC category above 11 and a code undefined in its table are refused"""
    good = _hand_coded([("dc", 0, 0, 0), ("ac", 0x01, 1, 1), ("ac", 0x00, 0, 0)], DC_13)
    assert J.coefficients(J.read(good), 0)[0][0, 1] == 1
    with pytest.raises(AssertionError, match=message):
        J.read(_hand_coded(items, dc_table))


# ---- CPU: the oracles against the exact transforms ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", LAYOUTS)
def test_oracle_encoder_equals_exact_dct(orc, pl, al, name):  # noqa: F811
    stats = []
    for w, h in ((1, 1), (17, 9), (130, 37), (256, 256)):
        for k, q in enumerate((1, 50, 90, 100)):
            content = "noise" if (w, h, q) == (256, 256, 100) else "natural"
            if w == 256 and q in (1, 50):
                continue
            src = layout_source(orc, name, w, h, content, w + q)
            s = oracle_layout_stream(orc, pl, al, name, src, w, h, q, (0, 1, 3, 32)[k])
            check_encoded(s, layout_planes(pl, name, src, w, h), q, f"{name} {w}x{h} q{q}", stats=stats)
    for content in ("extreme", "dcswing"):
        src = layout_source(orc, name, 64, 32, content, 1)
        check_encoded(oracle_layout_stream(orc, pl, al, name, src, 64, 32, 100, 0), layout_planes(pl, name, src, 64, 32), 100, f"{name} {content}",
                      stats=stats)
    _log_stats(stats, "cpu-oracle", name)


def test_dc_swing_needs_category_11():
    """the DC-swing frame reaches DC differences of category 11 (|diff| = 2040) at q = 100 - the largest a baseline stream can carry"""
    b = J.pad_blocks(dc_swing_frame(32, 8)[:, :, 0], 1, 4)
    dc = np.rint(J.fdct(b)[:, 0])
    assert set(dc.tolist()) == {-1024.0, 1016.0} and int(abs(np.diff(dc)).max()).bit_length() == 11


def test_band_derivation_holds_on_the_corpus():
    """the float32 restatements stay within a quarter of the band over noise, natural, extreme-AC and DC-swing blocks (the measurement
    the band was derived from; jpeg_exact.py)"""
    rng = np.random.default_rng(11)
    blocks = np.concatenate([rng.integers(0, 256, (3000, 8, 8)), J.pad_blocks(natural_rgb(128, 64, 2)[:, :, 0], 8, 16),
                             J.pad_blocks(extreme_ac_frame(RGB, 64, 32).reshape(32, 64, 3)[:, :, 0], 4, 8), J.pad_blocks(dc_swing_frame(64, 16)[:, :, 0], 2, 8)])
    for q in (1, 50, 90, 100):
        Q = J.scaled_qtable(J.Q_LUMA, q)
        x = J.fdct(blocks) / Q
        assert (np.abs(J.aan_fdct_f32(blocks, Q) - x) <= J.enc_band(blocks, Q) / 4).all(), q
    for Q in (np.full(64, 1), J.scaled_qtable(J.Q_LUMA, 50), np.full(64, 255)):
        coef = rng.integers(-1023, 1024, (2000, 64)) * (rng.random((2000, 64)) < 0.3)
        coef[:, 0] = rng.integers(-2047, 2048, 2000)
        px = J.idct(coef * Q[None, :])
        assert (np.abs(J.aan_idct_f32(coef, Q) - px) <= (J.dec_band(coef, Q) - J.DEC_BAND_ABS) / 4 + J.DEC_BAND_ABS).all()


def test_restatements_round_to_the_oracles_integers(orc):
    """the band rests on aan_fdct_f32 / aan_idct_f32 being the oracles' float32 operation order: rounded, they give orc_jpeg_coefficients and
    orc_jpeg_decode exactly (the oracle used to validate the helpers)"""
    orc.orc_jpeg_coefficients.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    w, h = 96, 64
    frames = [np.random.default_rng(1).integers(0, 256, (h, w, 3), dtype=np.uint8), natural_rgb(w, h, 2), extreme_ac_frame(RGB, w, h).reshape(h, w, 3),
              dc_swing_frame(w, h)]
    for f in frames:
        src = np.ascontiguousarray(f).reshape(-1)
        for q in (1, 50, 90, 100):
            ref = np.zeros(3 * (w // 8) * (h // 8) * 64, np.int16)
            orc.orc_jpeg_coefficients(src.ctypes.data, w * 3, w, h, 1, q, ref.ctypes.data)
            ref = ref.reshape(3, -1, 64)
            for c in range(3):
                Q = J.scaled_qtable(J.Q_LUMA if c == 0 else J.Q_CHROMA, q)
                mine = J.expected_coefficients(J.aan_fdct_f32(J.pad_blocks(f[:, :, c], h // 8, w // 8), Q))
                assert np.array_equal(mine[:, J.ZIGZAG], ref[c]), (q, c)
            s = orc_encode(orc, src, w, h, RGB, q, 0)
            fr = J.read(s)
            got = _orc_decode_planes(orc, s, fr)
            for c in range(3):
                co, _ = J.coefficients(fr, c)
                px = J.aan_idct_f32(co, fr.q[fr.components[c]["tq"]]).reshape(h // 8, w // 8, 8, 8).transpose(0, 2, 1, 3).reshape(h, w)
                assert np.array_equal(np.clip(np.rint(px), 0, 255), got[c]), (q, c)
    for name, s in writer_streams():  # Q = 255 with |coef| = 1023, long codes, corners: the decoder's float32 order at its extremes
        fr = J.read(s)
        if fr.components[0]["h"] != 1:
            continue
        got = _orc_decode_planes(orc, s, fr)
        for c in range(3):
            co, _ = J.coefficients(fr, c)
            gh, gw = fr.grid[c]
            px = J.aan_idct_f32(co, fr.q[fr.components[c]["tq"]]).reshape(gh, gw, 8, 8).transpose(0, 2, 1, 3).reshape(gh * 8, gw * 8)
            assert np.array_equal(np.clip(np.rint(px[:fr.h, :fr.w]), 0, 255), got[c]), (name, c)


def test_clamped_samples_moved_are_reported():
    """the Q = 255 stream clamps most samples at 0 or 255, where the band is about 3.7: a clamped sample moved by 1 or 3 is still reported
    (the band widens the unclamped value, so a value far beyond a limit must equal it)"""
    s = dict(writer_streams())["q255-extreme"]
    fr = J.read(s)
    px, band = exact_planes(fr)[0]
    got = np.clip(np.rint(px), 0, 255)
    assert band.max() > 3 and J.compare_samples(got, px, band)["exempt"] == 0
    hi = np.argwhere(px > 255 + band + 1)
    lo = np.argwhere(px < -band - 1)
    assert len(hi) and len(lo)
    for idx, v in ((hi[0], 254), (hi[len(hi) // 2], 252), (lo[0], 1), (lo[-1], 3)):
        g = got.copy()
        g[tuple(idx)] = v
        with pytest.raises(AssertionError, match="outside the tie band"):
            J.compare_samples(g, px, band)


def test_one_step_only_inside_the_band():
    """inside a band wider than 1/2 an exemption is still one step: 2 away from the exact rounding is reported"""
    px = np.array([100.5, 100.2])
    band = np.array([0.01, 3.0])
    J.compare_samples(np.array([100, 101]), px, band)
    with pytest.raises(AssertionError, match="outside the tie band"):
        J.compare_samples(np.array([100, 102]), px, band)
    with pytest.raises(AssertionError, match="outside the tie band"):
        J.compare_samples(np.array([102, 100]), px, band)


def _orc_decode_planes(orc, s, fr):
    from test_jpeg_decode import orc_decode
    w, h = fr.w, fr.h
    if fr.components[0]["h"] == 2:
        _, out = orc_decode(orc, s, 0, w, h)
        y, cb, cr = J.uyvy_planes(out, w, h)
        return [y, cb[::fr.components[0]["v"]], cr[::fr.components[0]["v"]]]  # a chroma row serves V luma rows (nearest)
    _, out = orc_decode(orc, s, 1, w, h)
    return J.packed_planes(out, w, h, 3)


def writer_streams():
    """decoder inputs our encoder never makes: (name, stream)"""
    out = []
    rng = np.random.default_rng(7)
    w, h = 37, 21
    comps = [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
    il = [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]]
    three = [[(0, 0, 0)], [(1, 1, 1)], [(2, 1, 1)]]
    q_std = {0: J.scaled_qtable(J.Q_LUMA, 80), 1: J.scaled_qtable(J.Q_CHROMA, 80)}
    # Q = 255, AC = +-1023 at every zig-zag position, DC at the extremes: clamps at both ends
    ext = []
    for c in range(3):
        a = rng.choice([-1023, 1023], (3, 5, 64))
        a[..., 0] = np.where(rng.random((3, 5)) < 0.5, -1023, 1023)
        a[0, 0] = 0
        a[0, 0, 0] = -1023 if c else 1023
        ext.append(a)
    out.append(("q255-extreme", J.write(w, h, comps, ext, {0: np.full(64, 255), 1: np.full(64, 255)}, STD_TABLES, three, ri=2, adobe=0)))
    # DC only, at exact half-integer sample values (Q = 4: sample = 128 + DC / 2)
    dc = [np.zeros((3, 5, 64), np.int64) for _ in range(3)]
    for c in range(3):
        dc[c][..., 0] = rng.integers(-120, 120, (3, 5)) * 2 + 1
    out.append(("dc-half", J.write(w, h, comps, dc, {0: np.full(64, 4), 1: np.full(64, 4)}, STD_TABLES, il, adobe=0)))
    # the last coefficient at k = 63 (no EOB), ZRL runs that end exactly at 63, a ZRL followed by EOB
    corner = [np.zeros((3, 5, 64), np.int64) for _ in range(3)]
    for c in range(3):
        corner[c][..., 0] = rng.integers(-300, 300, (3, 5))
        corner[c][..., J.ZIGZAG[1]] = 5
        corner[c][0::2, :, J.ZIGZAG[63]] = -7           # k = 63 set: no EOB
        corner[c][1::2, 0::2, J.ZIGZAG[15]] = 9         # last at 15: 48 zeros = three ZRL ending at 63
        corner[c][1::2, 1::2, J.ZIGZAG[43]] = -3        # last at 43: 20 zeros = ZRL + EOB
    out.append(("zrl-eob-corners", J.write(w, h, comps, corner, q_std, STD_TABLES, il, ri=1, adobe=0, zrl_tail=True)))
    base = _writer_frame(w, h, rng=rng)
    # every code 10 - 16 bits long (the maxcode walk only); every code exactly 9 bits (the edge of the 9-bit look-up)
    dc_long = ([0] * 9 + [6, 0, 0, 0, 0, 0, 6], list(range(12)))
    ac_long = ([0] * 9 + [100, 0, 40, 0, 0, 0, 22], J.AC_LUMA[1])
    dc_9 = ([0] * 8 + [12] + [0] * 7, list(range(12)))
    ac_9 = ([0] * 8 + [150, 12] + [0] * 6, J.AC_CHROMA[1])
    for name, (d, a) in (("codes-10-16", (dc_long, ac_long)), ("codes-9", (dc_9, ac_9))):
        t = {(0, 0): d, (1, 0): a, (0, 1): d, (1, 1): a}
        out.append((name, J.write(w, h, comps, base, q_std, t, three, ri=3, adobe=0)))
        out.append((name + "-il", J.write(w, h, comps, base, q_std, t, il, ri=0, adobe=0)))
    # restart interval 1, a partial last interval, no DRI
    out.append(("ri1", J.write(w, h, comps, base, q_std, STD_TABLES, il, ri=1, adobe=0)))
    out.append(("ri-partial", J.write(w, h, comps, base, q_std, STD_TABLES, il, ri=4, adobe=0)))  # 15 MCUs: 4 + 4 + 4 + 3
    out.append(("no-dri", J.write(w, h, comps, base, q_std, STD_TABLES, three, ri=0, adobe=0)))
    # tables redefined between the scans of a three-scan stream: every scan codes with table 0 of each class, each time another one
    between = {1: {(0, 0): dc_long, (1, 0): ac_long}, 2: {(0, 0): dc_9, (1, 0): ac_9}}
    same_ids = [[(0, 0, 0)], [(1, 0, 0)], [(2, 0, 0)]]
    out.append(("dht-redefined", J.write(w, h, comps, base, q_std, STD_TABLES, same_ids, ri=2, adobe=0, between=between)))
    # YCbCr 4:4:4 without Adobe marker (VUYA), and 4:2:2 from the writer with custom tables
    out.append(("ycc444", J.write(w, h, comps, base, q_std, STD_TABLES, il, ri=2)))
    b422 = _writer_frame(w, h, 2, 1, rng=rng)
    out.append(("ycc422-long", J.write(w, h, [(1, 2, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)], b422, q_std, {(0, 0): dc_long, (1, 0): ac_long, (0, 1): dc_9, (1, 1): ac_9},
                                       il, ri=3)))
    return out


def test_oracle_decoder_equals_exact_idct(orc):
    """oracle/jpeg_decode_oracle.c on the encoder's streams, libjpeg's streams and the writer's streams"""
    streams = [(f"pil-{k}", pil_stream(k, 200, 120)) for k, _ in PIL_CASES] + writer_streams()
    w, h = 130, 37
    for q in (5, 50, 100):
        src = layout_source(orc, "rgb", w, h, "natural", q)
        streams.append((f"rgb q{q}", orc_encode(orc, src, w, h, RGB, q, 3)))
        uy = layout_source(orc, "uyvy422", w, h, "natural", q)
        streams.append((f"uyvy q{q}", orc_encode(orc, uy, w, h, UYVY, q, 1, pitch=(w + 1) // 2 * 4)))
    for name, s in streams:
        fr = J.read(s)
        check_decoded(s, _orc_decode_planes(orc, s, fr), name)


# ---- CPU: the comparators have teeth --------------------------------------------------------------------------------------------
def test_perturbed_aan_constant_is_reported():
    """each AAN constant changed in its 5th significant digit: the coefficients of natural and noise blocks leave the band"""
    blocks = np.concatenate([np.random.default_rng(3).integers(0, 256, (400, 8, 8)), J.pad_blocks(natural_rgb(64, 64, 1)[:, :, 1], 8, 8)])
    Q = J.scaled_qtable(J.Q_LUMA, 90)
    x = J.fdct(blocks) / Q
    J.compare_coefficients(np.rint(J.aan_fdct_f32(blocks, Q)), x, J.enc_band(blocks, Q), "unperturbed")
    for name, v in J.AAN_FDCT.items():
        bad = np.rint(J.aan_fdct_f32(blocks, Q, {name: v * (1 + 1e-4)}))
        with pytest.raises(AssertionError, match="outside the tie band"):
            J.compare_coefficients(bad, x, J.enc_band(blocks, Q), name)


def test_one_coefficient_moved_is_reported():
    blocks = J.pad_blocks(natural_rgb(64, 64, 5)[:, :, 0], 8, 8)
    Q = J.scaled_qtable(J.Q_LUMA, 75)
    x = J.fdct(blocks) / Q
    band = J.enc_band(blocks, Q)
    got = J.expected_coefficients(x.copy())
    J.compare_coefficients(got, x, band)
    i = np.argwhere(J.half_dist(x) > 0.01)[17]
    for d in (1, -1):
        g = got.copy()
        g[tuple(i)] += d
        with pytest.raises(AssertionError, match="outside the tie band"):
            J.compare_coefficients(g, x, band)


def test_one_sample_moved_is_reported():
    rng = np.random.default_rng(9)
    coef = rng.integers(-40, 41, (30, 64)) * (rng.random((30, 64)) < 0.2)
    Q = J.scaled_qtable(J.Q_LUMA, 50)
    px = J.idct(coef * Q[None, :])
    band = J.dec_band(coef, Q)
    got = np.clip(np.rint(px), 0, 255)
    J.compare_samples(got, px, band)
    inside = np.argwhere((J.half_dist(px) > 0.01) & (px > 2) & (px < 253))[5]
    g = got.copy()
    g[tuple(inside)] += 1
    with pytest.raises(AssertionError, match="outside the tie band"):
        J.compare_samples(g, px, band)


# ---- GPU: encoder ------------------------------------------------------------------------------------------------------------
GPU_SIZES = [(17, 24), (24, 31), (41, 17), (63, 40), (233, 120)]  # w % 16 in {1, 8, 9, 15}, h % 16 in {1, 8, 15}
GPU_RIS = [0, 1, 3, 32]


def gpu_encode(enc, name, src, w, h, q, ri):
    import torch
    codec, sub, cs, il = layout_params(name)
    pitch = (w + 1) // 2 * 4 if codec == UYVY else 0
    enc.encode_device(torch.from_numpy(src).cuda(), w, h, codec, quality=q, restart_interval=ri, pitch=pitch, interleaved=bool(il), subsampling=sub,
                      color_space=CS[cs])
    return enc.result()


def _log_stats(stats, tag, name):
    """one line per layout and route: the largest |value - exact| - 1/2 over everything compared (negative: every value within its rounding
    interval, 0 for an exact tie) and the share of band exemptions (printed; run with -s to see them)"""
    n, e, worst = sum(st["n"] for _, st in stats), sum(st["exempt"] for _, st in stats), max(st["worst"] for _, st in stats)
    print(f"[stats] {tag} {name}: worst {worst:.3g}, exempt {e}/{n} = {100 * e / n:.3f} %")


@pytest.mark.gpu
@pytest.mark.parametrize("name", LAYOUTS)
def test_gpu_encoder_equals_exact_dct(orc, pl, name):  # noqa: F811
    from ultragrid_b200 import api
    enc = api.JpegEncoder()
    stats = []
    for i, (w, h) in enumerate(GPU_SIZES):
        src = layout_source(orc, name, w, h, "natural", 3 * w + h)
        for k, q in enumerate((1, 90, 100)):
            ri = GPU_RIS[(i + k) % 4]
            check_encoded(gpu_encode(enc, name, src, w, h, q, ri), layout_planes(pl, name, src, w, h), q, f"{name} {w}x{h} q{q} ri{ri}", stats=stats)
    # noise twice (serial route, then the adapted cap); its quality keeps the stream inside the w * h * 3 bytes of output (4:4:4 noise at q = 100 codes
    # to more, which the encoder reports as an error, test_jpeg.py)
    _, sub, _, _ = layout_params(name)
    qn = 50 if sub == 4444 else 85 if sub == 444 or name in ("rgb", "rgb-il") else 100
    for content, (w, h), q in (("noise", (320, 96), qn), ("noise", (320, 96), qn), ("extreme", (64, 32), 100), ("dcswing", (72, 40), 100)):
        src = layout_source(orc, name, w, h, content, 5)
        check_encoded(gpu_encode(enc, name, src, w, h, q, 0), layout_planes(pl, name, src, w, h), q, f"{name} {content} q{q}", stats=stats)
    enc.close()
    _log_stats(stats, os.environ.get("UGB200_ROUTE", "default"), name)


def sampled_segments(seed=0):
    def pick(scan, nseg):
        rng = np.random.default_rng(seed + scan)
        spread = np.linspace(0, nseg - 1, min(nseg, 120)).astype(int)  # one per column band of the frame
        return sorted(set([0, nseg - 1] + spread.tolist() + rng.integers(0, nseg, min(nseg, 200)).tolist()))
    return pick


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["uyvy422", "rgb", "rgba"])
def test_gpu_encoder_8k_sampled_segments(orc, pl, name):  # noqa: F811
    from ultragrid_b200 import api
    w, h = 7680, 4320
    src = layout_source(orc, name, w, h, "natural", 8)
    enc = api.JpegEncoder()
    for q in (90, 100):
        check_encoded(gpu_encode(enc, name, src, w, h, q, 0), layout_planes(pl, name, src, w, h), q, f"{name} 8K q{q}", segments=sampled_segments(q))
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("knob,value", [("UGB200_JPEG_SPLIT", "1"), ("UGB200_JPEG_SINGLE_PASS", "1"), ("UGB200_JPEG_TWO_KERNELS", "1"),
                                        ("UGB200_JPEG_TWO_KERNELS", "8"), ("UGB200_JPEG_CAP", "12"), ("UGB200_JPEG_CAP", "24")])
def test_gpu_encoder_routes_equal_exact_dct(knob, value):
    """the process-wide route switches: the encoder tests once more in a child process with the switch set"""
    env = dict(os.environ, **{knob: value, "UGB200_ROUTE": f"{knob}={value}"})
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-q", "-x", "-s", "-k", "gpu_encoder_equals_exact_dct"],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    print("\n".join(re.findall(r"\[stats\][^\n]*", r.stdout)))


# ---- GPU: decoder ------------------------------------------------------------------------------------------------------------
def _decoders(monkeypatch):
    from ultragrid_b200 import api
    out = []
    for mode in ("host", "device"):
        monkeypatch.setenv("UGB200_JPEG_MARKER_SCAN", mode)  # read when the decoder is created
        out.append((mode, api.JpegDecoder()))
    monkeypatch.delenv("UGB200_JPEG_MARKER_SCAN")
    return out


def _decode_native(dec, s, fr):
    from ultragrid_b200 import api
    native = api.jpeg_image_info(s).native_codec
    codec = I420 if native == UYVY and fr.components[0]["v"] == 2 else native
    return codec, dec.decode(s, codec)


def four_scans_redefined():
    """R G B A in four scans, all coded with table 0 of each class, both redefined in front of scans 2, 3 and 4: four table versions per class"""
    w, h = 37, 21
    rng = np.random.default_rng(12)
    coef = _writer_frame(w, h, rng=rng) + _writer_frame(w, h, rng=rng)[:1]
    comps = [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1), (4, 1, 1, 1)]
    dc_long = ([0] * 9 + [6, 0, 0, 0, 0, 0, 6], list(range(12)))
    ac_long = ([0] * 9 + [100, 0, 40, 0, 0, 0, 22], J.AC_LUMA[1])
    dc_9 = ([0] * 8 + [12] + [0] * 7, list(range(12)))
    ac_9 = ([0] * 8 + [150, 12] + [0] * 6, J.AC_CHROMA[1])
    between = {1: {(0, 0): dc_long, (1, 0): ac_long}, 2: {(0, 0): dc_9, (1, 0): ac_9}, 3: {(0, 0): J.DC_CHROMA, (1, 0): J.AC_CHROMA}}
    q = {0: J.scaled_qtable(J.Q_LUMA, 80), 1: J.scaled_qtable(J.Q_CHROMA, 80)}
    return J.write(w, h, comps, coef, q, STD_TABLES, [[(c, 0, 0)] for c in range(4)], ri=2, adobe=0, between=between)


def test_decoder_parser_keeps_every_table_version():
    """host parser of the decoder: Huffman tables redefined before every scan of a four-scan stream (eight table versions in use) are accepted;
    a table no scan uses takes no slot"""
    from ultragrid_b200 import _lib
    lib = _lib.load()
    s = four_scans_redefined()
    fr = J.read(s)
    assert len(fr.scans) == 4
    begin, end = np.zeros(256, np.uint32), np.zeros(256, np.uint32)
    assert lib.ugb200_jpeg_debug_segments(s, len(s), begin.ctypes.data, end.ctypes.data, 256) == sum(sc["nseg"] for sc in fr.scans)


def decoder_corpus(orc, pl, al):  # noqa: F811
    out = []
    for i, name in enumerate(LAYOUTS):
        w, h = GPU_SIZES[i % len(GPU_SIZES)]
        src = layout_source(orc, name, w, h, "natural", i)
        for q, ri in ((90, 0), (100, 3)):
            out.append((f"{name} {w}x{h} q{q} ri{ri}", oracle_layout_stream(orc, pl, al, name, src, w, h, q, ri)))
    out += [(f"pil-{k}", pil_stream(k, 200, 120)) for k, _ in PIL_CASES]
    return out + writer_streams() + [("dht-redefined-4-scans", four_scans_redefined())]


@pytest.mark.gpu
def test_gpu_decoder_equals_exact_idct(orc, pl, al, monkeypatch):  # noqa: F811
    """every sample inside the image == clamp(round(exact IDCT)) outside the band, through both marker scans; 4:2:0 streams decode to I420,
    whose chroma planes are the decoded chroma planes (yuv420p_to_uyvy gives both rows of a pair the same chroma row, uyvy_to_i420 averages
    the two equal values)"""
    decs = _decoders(monkeypatch)
    for name, s in decoder_corpus(orc, pl, al):
        fr = J.read(s)
        for mode, dec in decs:
            codec, out = _decode_native(dec, s, fr)
            st = check_decoded(s, output_planes(out, fr, codec), f"{name} ({mode} scan, codec {codec})")
            print(f"[stats] decoder {name} ({mode} scan): worst {st['worst']:.3g}, exempt {st['exempt']}/{st['n']}")
    for _, dec in decs:
        dec.close()


@pytest.mark.gpu
def test_gpu_decoder_8k_equals_exact_idct(orc, monkeypatch):
    """8K UYVY and RGB streams: the blocks of a sample of restart segments (first, last, spread over the frame, random)"""
    decs = _decoders(monkeypatch)
    w, h = 7680, 4320
    for name in ("uyvy422", "rgb"):
        src = layout_source(orc, name, w, h, "natural", 2)
        codec = UYVY if name == "uyvy422" else RGB
        s = orc_encode(orc, src, w, h, codec, 90, 0, pitch=(w + 1) // 2 * 4 if codec == UYVY else 0)
        fr = J.read(s, sampled_segments(5))
        for mode, dec in decs:
            planes = output_planes(dec.decode(s, codec), fr, codec)
            hmax = max(c["h"] for c in fr.components)
            for c, cc in enumerate(fr.components):
                got, mask = J.coefficients(fr, c)
                gh, gw = fr.grid[c]
                q = fr.q[cc["tq"]]
                idx = np.flatnonzero(mask)
                px = J.idct(got[idx] * q[None, :])
                band = J.dec_band(got[idx], q)
                by, bx = idx // gw, idx % gw
                pw = -(-w * cc["h"] // hmax)
                ys = by[:, None, None] * 8 + np.arange(8)[None, :, None]
                xs = bx[:, None, None] * 8 + np.arange(8)[None, None, :]
                inside = (ys < h) & (xs < pw)
                ys, xs = np.broadcast_arrays(ys, xs)
                J.compare_samples(planes[c][ys[inside], xs[inside]], px[inside], np.asarray(band)[inside], f"{name} 8K {mode} c{c}")
    for _, dec in decs:
        dec.close()


@pytest.mark.gpu
def test_gpu_decoder_refuses_what_is_not_baseline():
    """SOF1, SOF2, SOF9, 12-bit precision, one component, luma sampled 1x2 or 4x1: -4, and the output buffer is not touched"""
    from ultragrid_b200 import _lib, api
    L = _lib.load()
    w, h = 32, 16
    base = _writer_frame(w, h)
    comps = [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)]
    il = [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]]
    q = {0: np.full(64, 2), 1: np.full(64, 3)}
    cases = [("sof1", J.write(w, h, comps, base, q, STD_TABLES, il, sof=0xC1)), ("sof2", J.write(w, h, comps, base, q, STD_TABLES, il, sof=0xC2)),
             ("sof9", J.write(w, h, comps, base, q, STD_TABLES, il, sof=0xC9)), ("12-bit", J.write(w, h, comps, base, q, STD_TABLES, il, precision=12)),
             ("one component", J.write(w, h, comps[:1], base[:1], q, STD_TABLES, [[(0, 0, 0)]]))]
    for name, hv in (("1x2", (1, 2)), ("4x1", (4, 1))):
        mw, mh = -(-w // (8 * hv[0])), -(-h // (8 * hv[1]))
        coef = [np.zeros((mh * hv[1], mw * hv[0], 64), np.int64), np.zeros((mh, mw, 64), np.int64), np.zeros((mh, mw, 64), np.int64)]
        cases.append((name, J.write(w, h, [(1, hv[0], hv[1], 0)] + comps[1:], coef, q, STD_TABLES, il)))
    dec = api.JpegDecoder()
    for name, s in cases:
        for codec in (UYVY, RGB):
            out = np.full(w * h * 4, 0xA5, np.uint8)
            rc = L.ugb200_jpeg_decode(dec._h, s, len(s), out.ctypes.data, 0, 0, codec, 0, 8, 16)
            assert rc == -4, (name, codec, rc)
            assert (out == 0xA5).all(), (name, codec)
    dec.close()
