"""JPEG decode in a colour space (ugb200_jpeg_decode_cs, ugb200_jpeg_stream_color_space) and the fused IDCT kernel behind ugb200_jpeg_decode.
  * CPU: the restatement tests/jpeg_color_oracle.c against the formula in numpy over every (Y, Cb, Cr), against the reference's unmodified
    vc_copylineUYVYtoRGB (Y709 == the line converter) and against libjpeg's own YCbCr -> RGB (Y601full on JFIF streams); the declared colour
    space of marker streams built with jpeg_exact.write.
  * GPU: ugb200_jpeg_decode to UYVY / RGB / RGBA == decode(UYVY) + pixfmt_convert (the route it replaces) for both Huffman routes and both marker
    scans, host and device destinations; decode_cs == the oracle for every colour space, sampling and packing; AUTO == the declared space."""
import ctypes
import io
import os
import subprocess
import tempfile

import numpy as np
import pytest
from PIL import Image

import jpeg_exact as J
import util
from test_jpeg import RGB, UYVY, natural_rgb, orc_encode, orc_encode_parallel

RGBA = 1
CS = {"Y601": 1, "Y601full": 2, "Y709": 3}
NATIVE, CS_RGB, AUTO = 0, 4, 5
HERE = os.path.dirname(os.path.abspath(__file__))
_vp, _i, _l = ctypes.c_void_p, ctypes.c_int, ctypes.c_long
STD_TABLES = {(0, 0): J.DC_LUMA, (1, 0): J.AC_LUMA, (0, 1): J.DC_CHROMA, (1, 1): J.AC_CHROMA}


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


@pytest.fixture(scope="module")
def co():
    """the colour oracle, compiled on its own (it includes oracle/jpeg_decode_oracle.c)"""
    d = tempfile.mkdtemp(prefix="ugb_color_oracle_")
    path = os.path.join(d, "libjpegcolor.so")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-fvisibility=hidden", "-o", path, os.path.join(HERE, "jpeg_color_oracle.c"), "-lm"],
                   check=True, capture_output=True)
    L = ctypes.CDLL(path)
    L.orc_cs_coeffs.argtypes = [_i, _vp]
    L.orc_cs_coeffs.restype = None
    L.orc_ycbcr_to_rgb.argtypes = [_i, _vp, _vp, _l]
    L.orc_ycbcr_to_rgb.restype = None
    L.orc_uyvy_to_rgb_cs.argtypes = [_i, _vp, _l, _i, _i, _i, _i, _i, _i, _vp, _l]
    L.orc_uyvy_to_rgb_cs.restype = None
    L.orc_jpeg_decode_cs.argtypes = [_vp, ctypes.c_size_t, _i, _i, _i, _i, _i, _vp, _l]
    return L


def coeffs(co, cs):
    c = (ctypes.c_int * 6)()
    co.orc_cs_coeffs(cs, c)
    return list(c)


def oracle_cs(co, s, cs, rgba, shifts, w, h, pitch=None, fill=0):
    bpp = 4 if rgba else 3
    pitch = pitch or w * bpp
    out = np.full(pitch * h, fill, np.uint8)
    b = np.frombuffer(s, np.uint8)
    assert co.orc_jpeg_decode_cs(b.ctypes.data, len(s), cs, rgba, *shifts, out.ctypes.data, pitch) == 0
    return out


def pil_stream(rgb, q, sub, ri=0):
    b = io.BytesIO()
    kw = {"restart_marker_blocks": ri} if ri else {}
    Image.fromarray(rgb).save(b, "JPEG", quality=q, subsampling=sub, **kw)
    return b.getvalue()


def bars(w, h):
    """saturated colour bars (the primaries, secondaries, black and white) over a natural frame's lower half"""
    cols = np.array([[255, 255, 255], [255, 255, 0], [0, 255, 255], [0, 255, 0], [255, 0, 255], [255, 0, 0], [0, 0, 255], [0, 0, 0]], np.uint8)
    img = natural_rgb(w, h, 3)
    img[: h // 2] = cols[(np.arange(w) * 8 // w)][None, :, :]
    return img


def with_markers(s, markers):
    """the stream with marker segments inserted after SOI"""
    return s[:2] + b"".join(markers) + s[2:]


def strip_app0(s):
    assert s[2:4] == b"\xff\xe0"
    n = int.from_bytes(s[4:6], "big")
    return s[:2] + s[4 + n:]


def spiff(code, truncate=False):
    body = b"SPIFF\x00" + b"\x01\x00" + b"\x00\x03" + (16).to_bytes(4, "big") + (16).to_bytes(4, "big") + bytes([code, 8, 5, 0]) + bytes(8)
    if truncate:
        body = body[:16]
    return b"\xff\xe8" + (len(body) + 2).to_bytes(2, "big") + body


JFIF = b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"


def adobe(t):
    return b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00" + bytes([t])


def written(w, h, ids=(1, 2, 3), hs=2, vs=1):
    comps = [(ids[0], hs, vs, 0), (ids[1], 1, 1, 1), (ids[2], 1, 1, 1)]
    mw, mh = -(-w // (8 * hs)), -(-h // (8 * vs))
    coef = [np.zeros((mh * vs, mw * hs, 64), np.int64), np.zeros((mh, mw, 64), np.int64), np.zeros((mh, mw, 64), np.int64)]
    return J.write(w, h, comps, coef, {0: np.full(64, 3), 1: np.full(64, 5)}, STD_TABLES, [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]])


# ---- CPU -----------------------------------------------------------------------------------------------------------------------------


def test_oracle_coefficients_are_color_space_h(co):
    """the oracle's inverse rows are compute_color_coeffs': the pinned BT.709 values of csrc/color_space.h, and all three from the reference
    where it is built"""
    assert coeffs(co, CS["Y709"]) == [19077, 29371, -3494, -8733, 34610, 16]
    assert coeffs(co, CS["Y601full"])[0] == 16384 and coeffs(co, CS["Y601full"])[5] == 0
    ref = util.ref_cpu()
    if ref is None:
        return
    for cs, (which, depth) in {"Y709": (2, 8), "Y601": (1, 8), "Y601full": (1, 0)}.items():  # enum colorspace: CS_601 = 1, CS_709 = 2
        c = (ctypes.c_int * 14)()
        ref.ref_get_color_coeffs(which, depth, c)
        assert list(c)[9:] == coeffs(co, CS[cs])[:5], cs


@pytest.mark.parametrize("cs", list(CS))
def test_oracle_conversion_equals_formula_for_every_triple(co, cs):
    ys, rc, gcb, gcr, bcb, o = coeffs(co, CS[cs])
    y, cb, cr = [a.reshape(-1) for a in np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij")]
    ycc = np.stack([y, cb, cr], 1).astype(np.uint8)
    got = np.empty_like(ycc)
    co.orc_ycbcr_to_rgb(CS[cs], ycc.ctypes.data, got.ctypes.data, len(ycc))
    yy = ys * (y.astype(np.int64) - o)
    want = np.stack([(yy + rc * (cr - 128)) >> 14, (yy + gcb * (cb - 128) + gcr * (cr - 128)) >> 14, (yy + bcb * (cb - 128)) >> 14], 1).clip(0, 255)
    assert np.array_equal(got, want.astype(np.uint8))


@pytest.mark.parametrize("w,h,sub", [(200, 120, 1), (131, 37, 2), (98, 50, 2), (17, 9, 1)])
def test_y709_rgb_equals_reference_line_converter(orc, co, w, h, sub):
    """Y709 RGB of a UYVY decode == the reference's unmodified vc_copylineUYVYtoRGB on the same UYVY (whole pixel pairs)"""
    ref = util.ref_cpu()
    if ref is None:
        pytest.skip("oracle/_ref not built")
    s = pil_stream(natural_rgb(w, h, 7), 90, sub)
    up = (w + 1) // 2 * 4
    uyvy = np.zeros(up * h + 64, np.uint8)
    info = (ctypes.c_int * 6)()
    orc.orc_jpeg_decode.argtypes = [_vp, ctypes.c_size_t, _i, _vp, _l, _vp]
    b = np.frombuffer(s, np.uint8)
    assert orc.orc_jpeg_decode(b.ctypes.data, len(s), 0, uyvy.ctypes.data, up, info) == 0
    uyvy = uyvy[:up * h]
    got = np.zeros(w * 3 * h, np.uint8)
    co.orc_uyvy_to_rgb_cs(CS["Y709"], uyvy.ctypes.data, up, w, h, 0, 0, 8, 16, got.ctypes.data, w * 3)
    want = util.convert_cpu(ref, "ref_convert", UYVY, RGB, uyvy, w, h, linesize=ref.ref_vc_get_linesize)
    n = (w // 2) * 6
    assert np.array_equal(got.reshape(h, -1)[:, :n], want.reshape(h, -1)[:, :n])
    assert np.array_equal(oracle_cs(co, s, CS["Y709"], 0, (0, 8, 16), w, h).reshape(h, -1)[:, :n], want.reshape(h, -1)[:, :n])


def _lib():
    from ultragrid_b200 import _lib
    return _lib.load()


def declared(L, s):
    return L.ugb200_jpeg_stream_color_space(s, len(s))


def test_stream_color_space_rules_and_precedence():
    L = _lib()
    plain, plain444, rgb_ids = written(40, 24), written(40, 24, hs=1), written(40, 24, ids=(ord("R"), ord("G"), ord("B")), hs=1)
    cases = [
        (plain, NATIVE + 3),                                             # no marker: Y709
        (with_markers(plain, [JFIF]), 2),                                # JFIF: Y601full
        (with_markers(plain, [adobe(1)]), 2),                            # Adobe transform 1
        (with_markers(plain444, [adobe(0)]), CS_RGB),                    # Adobe transform 0 on 4:4:4: an RGB stream
        (with_markers(plain, [adobe(0)]), 3),                            # 4:2:2 decodes as YCbCr whatever the transform says (native_codec)
        (rgb_ids, CS_RGB), (with_markers(rgb_ids, [spiff(1)]), CS_RGB),  # component ids R G B, whatever else it carries
        (with_markers(plain, [spiff(1)]), 3), (with_markers(plain, [spiff(4)]), 1), (with_markers(plain, [spiff(3)]), 2),
        (with_markers(plain, [spiff(10)]), CS_RGB),
        (with_markers(plain, [spiff(4), JFIF]), 1), (with_markers(plain, [JFIF, spiff(1)]), 3),   # SPIFF before JFIF
        (with_markers(plain, [adobe(1), spiff(4)]), 1),                                            # SPIFF before Adobe
        (with_markers(plain, [JFIF, adobe(2)]), 2), (with_markers(plain, [adobe(1), JFIF]), 2),
        (with_markers(plain, [spiff(5)]), -4), (with_markers(plain, [spiff(2)]), -4), (with_markers(plain, [spiff(12)]), -4),
        (with_markers(plain, [spiff(1, truncate=True)]), -3),
        (with_markers(plain444, [spiff(99), adobe(0)]), CS_RGB), (with_markers(plain444, [spiff(99)]), -4),
        (plain[:20], -3),
    ]
    for i, (s, want) in enumerate(cases):
        assert declared(L, s) == want, (i, declared(L, s), want)
    assert L.ugb200_jpeg_stream_color_space(None, 0) == -1
    four = J.write(16, 16, [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1), (4, 1, 1, 1)], [np.zeros((2, 2, 64), np.int64)] * 4, {0: np.full(64, 3), 1: np.full(64, 5)},
                   STD_TABLES, [[(0, 0, 0)], [(1, 1, 1)], [(2, 1, 1)], [(3, 1, 1)]])
    assert declared(L, with_markers(four, [JFIF])) == CS_RGB


def pil_rgb(s):
    return np.asarray(Image.open(io.BytesIO(s)).convert("RGB"))


def libjpeg_bound(co):
    """per channel: each decoded sample within 1 of libjpeg's (the IDCT bound) times the matrix gains, plus libjpeg's own round-to-nearest
    (0.5) and our floor (below 1), so |diff| < gain + 1.5; the Q14 coefficients add under 0.05"""
    ys, rc, gcb, gcr, bcb, _ = coeffs(co, CS["Y601full"])
    gains = [(ys + abs(rc)) / 16384, (ys + abs(gcb) + abs(gcr)) / 16384, (ys + abs(bcb)) / 16384]
    return np.array([int(np.floor(g + 1.5 + 0.05)) for g in gains])


@pytest.mark.parametrize("q", [75, 90, 100])
@pytest.mark.parametrize("content", ["natural", "bars"])
def test_y601full_matches_libjpeg_on_jfif_444(co, q, content):
    w, h = 160, 96
    img = natural_rgb(w, h, 11) if content == "natural" else bars(w, h)
    s = pil_stream(img, q, 0)
    want = pil_rgb(s).astype(np.int32)
    bound = libjpeg_bound(co)
    got = oracle_cs(co, s, CS["Y601full"], 0, (0, 8, 16), w, h).reshape(h, w, 3).astype(np.int32)
    worst = np.abs(got - want).reshape(-1, 3).max(0)
    assert (worst <= bound).all(), (worst, bound)
    if content == "bars":  # the same samples read as BT.709 limited range are far off: the test tells the matrices apart
        bad = oracle_cs(co, s, CS["Y709"], 0, (0, 8, 16), w, h).reshape(h, w, 3).astype(np.int32)
        assert (np.abs(bad - want).reshape(-1, 3).max(0) > bound).any()


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------

SHIFTS = [(0, 8, 16), (16, 8, 0)]


def make(orc, kind, w, h, q):
    if kind == "ours-422":
        rgb = natural_rgb(w, h, 5)
        uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, rgb.reshape(-1), w, h)
        enc = orc_encode_parallel if w * h > 1 << 20 else orc_encode
        return enc(orc, uyvy, w, h, UYVY, q)
    return pil_stream(natural_rgb(w, h, 9), q, {"pil-422": 1, "pil-420": 2, "pil-444": 0}[kind])


def old_route(api, Codec, dec, s, w, h, out_c, shifts):
    """decode to UYVY, then UltraGrid's line converter on the device: what ugb200_jpeg_decode did for these outputs"""
    uy = dec.decode(s, UYVY, device=True)
    if out_c == UYVY:
        return uy.cpu().numpy()
    return api.pixfmt_convert(Codec.UYVY, Codec(out_c), uy, w, h, shifts=shifts).cpu().numpy()


def row_bytes(w, out_c):
    return (w + 1) // 2 * 4 if out_c == UYVY else (w // 2) * 2 * (3 if out_c == RGB else 4)


def check_same(api, Codec, dec, s, w, h, want_uyvy=None):
    import torch
    for out_c in (UYVY, RGB, RGBA):
        for shifts in (SHIFTS if out_c == RGBA else SHIFTS[:1]):
            want = old_route(api, Codec, dec, s, w, h, out_c, shifts)
            ls = api.vc_get_linesize(w, Codec(out_c))
            n = row_bytes(w, out_c)
            w2 = want.reshape(h, ls)
            got = dec.decode(s, out_c, shifts=shifts)
            assert np.array_equal(got.reshape(h, ls)[:, :n], w2[:, :n]), (out_c, shifts)
            for cs in (None, NATIVE):
                for pitch in (ls, ls + 80):
                    out = torch.full((pitch * h,), 0xA5, dtype=torch.uint8, device="cuda")
                    dec.decode(s, out_c, shifts=shifts, device=True, pitch=pitch, out=out, color_space=cs)
                    g = out.cpu().numpy().reshape(h, pitch)
                    assert np.array_equal(g[:, :n], w2[:, :n]), (out_c, shifts, cs, pitch)
                    assert (g[:, n:] == 0xA5).all(), (out_c, shifts, cs, pitch)  # nothing written beyond the whole pixel pairs
            assert np.array_equal(dec.decode(s, out_c, shifts=shifts, color_space=NATIVE).reshape(h, ls)[:, :n], w2[:, :n])
    if want_uyvy is not None:
        assert np.array_equal(dec.decode(s, UYVY), want_uyvy)


@pytest.mark.gpu
@pytest.mark.parametrize("sync", ["on", "off"])
@pytest.mark.parametrize("scan", ["host", "device"])
def test_gpu_fused_route_same_bytes(orc, monkeypatch, sync, scan):
    from ultragrid_b200 import Codec, api
    from test_jpeg_decode import orc_decode
    monkeypatch.setenv("UGB200_JPEG_SYNC", sync)
    monkeypatch.setenv("UGB200_JPEG_MARKER_SCAN", scan)
    dec = api.JpegDecoder()
    cases = [(k, w, h, q) for k in ("ours-422", "pil-422", "pil-420") for (w, h) in ((200, 120), (98, 50)) for q in (1, 90, 100)]
    cases += [(k, w, h, 90) for k in ("pil-422", "pil-420") for (w, h) in ((131, 37), (17, 9), (33, 18), (1921, 1081))]
    cases += [("ours-422", 1920, 1080, 90), ("pil-420", 1920, 1080, 90)]
    for kind, w, h, q in cases:
        s = make(orc, kind, w, h, q)
        _, want_uyvy = orc_decode(orc, s, 0, w, h)
        check_same(api, Codec, dec, s, w, h, want_uyvy)
    dec.close()


@pytest.mark.gpu
def test_gpu_fused_route_same_bytes_large(orc):
    from ultragrid_b200 import Codec, api
    dec = api.JpegDecoder()
    for kind, w, h in [("ours-422", 3840, 2160), ("pil-420", 3840, 2160), ("pil-420", 7680, 4320), ("pil-422", 3839, 2161)]:
        check_same(api, Codec, dec, make(orc, kind, w, h, 90), w, h)
    dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pil-444", "pil-422", "pil-420", "ours-422"])
def test_gpu_decode_cs_equals_oracle(orc, co, kind):
    import torch
    from ultragrid_b200 import api
    dec = api.JpegDecoder()
    sizes = [(200, 120), (131, 37), (17, 9), (3840, 2160)] if kind != "ours-422" else [(200, 120), (98, 50)]
    for w, h in sizes:
        s = make(orc, kind, w, h, 90)
        whole = kind == "pil-444"
        for cs in CS:
            for out_c, shifts in [(RGB, (0, 8, 16)), (RGBA, SHIFTS[0]), (RGBA, SHIFTS[1])]:
                rgba = out_c == RGBA
                bpp = 4 if rgba else 3
                n = w * bpp if whole else row_bytes(w, out_c)
                want = oracle_cs(co, s, CS[cs], int(rgba), shifts, w, h).reshape(h, -1)
                got = dec.decode(s, out_c, shifts=shifts, color_space=cs).reshape(h, -1)
                assert np.array_equal(got[:, :n], want[:, :n]), (kind, w, h, cs, out_c, shifts)
                pitch = w * bpp + 48
                out = torch.full((pitch * h,), 0x5A, dtype=torch.uint8, device="cuda")
                dec.decode(s, out_c, shifts=shifts, device=True, pitch=pitch, out=out, color_space=CS[cs])
                g = out.cpu().numpy().reshape(h, pitch)
                assert np.array_equal(g[:, :n], want[:, :n]) and (g[:, n:] == 0x5A).all(), (kind, w, h, cs, out_c, shifts)
    dec.close()


@pytest.mark.gpu
def test_gpu_auto_equals_declared_space(orc):
    from ultragrid_b200 import api
    dec = api.JpegDecoder()
    base = pil_stream(natural_rgb(130, 66, 4), 90, 2)
    bare = strip_app0(base)
    streams = {"Y601full": base, "Y709": bare, "Y601": with_markers(bare, [spiff(4)]), "Y709 ": with_markers(base, [spiff(1)]),
               "Y601full ": with_markers(bare, [adobe(1)])}
    for name, s in streams.items():
        assert api.jpeg_stream_color_space(s) == name.strip()
        for out_c in (RGB, RGBA, UYVY):
            assert np.array_equal(dec.decode(s, out_c, color_space="auto"), dec.decode(s, out_c, color_space=name.strip())), (name, out_c)
    rgb_stream = orc_encode(orc, natural_rgb(64, 32, 2).reshape(-1).copy(), 64, 32, RGB, 90)
    assert api.jpeg_stream_color_space(rgb_stream) == "RGB"
    for cs in ("auto", "Y601full", "Y709"):  # RGB streams are never transformed
        assert np.array_equal(dec.decode(rgb_stream, RGBA, color_space=cs), dec.decode(rgb_stream, RGBA))
    dec.close()


@pytest.mark.gpu
def test_gpu_refusals_leave_output_untouched():
    import torch
    from ultragrid_b200 import _lib, api
    L = _lib.load()
    dec = api.JpegDecoder()
    bare = strip_app0(pil_stream(natural_rgb(64, 48, 4), 90, 2))
    out = torch.full((64 * 4 * 48,), 0x33, dtype=torch.uint8, device="cuda")
    b = api._bytes_ptr(bare)
    for cs, want in [(4, -1), (6, -1), (-1, -1)]:
        assert L.ugb200_jpeg_decode_cs(dec._h, b, len(bare), ctypes.c_void_p(out.data_ptr()), 1, 0, RGBA, 0, 8, 16, cs) == want
    bad = with_markers(bare, [spiff(7)])
    assert L.ugb200_jpeg_decode_cs(dec._h, api._bytes_ptr(bad), len(bad), ctypes.c_void_p(out.data_ptr()), 1, 0, RGBA, 0, 8, 16, AUTO) == -4
    host = np.full(64 * 4 * 48, 0x33, np.uint8)
    assert L.ugb200_jpeg_decode_cs(dec._h, api._bytes_ptr(bad), len(bad), ctypes.c_void_p(host.ctypes.data), 0, 0, RGB, 0, 8, 16, AUTO) == -4
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == 0x33).all() and (host == 0x33).all()
    dec.close()
