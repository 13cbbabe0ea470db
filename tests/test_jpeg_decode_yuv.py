"""JPEG decode to a YCbCr colour space (ugb200_jpeg_decode_to) and grayscale streams.
  * CPU: the restatement tests/jpeg_yuv_oracle.c - its coefficients against an independent float64 computation, the conversion over every
    (Y, Cb, Cr) against the integer formula and the unrounded matrix, against libjpeg (PIL) on JFIF streams; grayscale header rules and samples;
    refusals.
  * GPU: ugb200_jpeg_decode_to == the oracle for every sampling, output codec and pair of spaces, both Huffman routes and marker scans, host and
    pitched device destinations; the identities with ugb200_jpeg_decode and ugb200_jpeg_decode_cs."""
import ctypes
import io
import os
import subprocess
import tempfile

import numpy as np
import pytest
from PIL import Image

import util
from test_jpeg import RGB, UYVY, natural_rgb
from test_jpeg_decode_color import JFIF, RGBA, adobe, bars, co, make, pil_stream, spiff, strip_app0, with_markers  # noqa: F401 (co: fixture)

CS = {"Y601": 1, "Y601full": 2, "Y709": 3}
NATIVE, CS_RGB, AUTO = 0, 4, 5
PAIRS = [(a, b) for a in CS for b in CS if a != b]
HERE = os.path.dirname(os.path.abspath(__file__))
_vp, _i, _l = ctypes.c_void_p, ctypes.c_int, ctypes.c_long


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


@pytest.fixture(scope="module")
def yo():
    d = tempfile.mkdtemp(prefix="ugb_yuv_oracle_")
    path = os.path.join(d, "libjpegyuv.so")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-fvisibility=hidden", "-o", path, os.path.join(HERE, "jpeg_yuv_oracle.c"), "-lm"],
                   check=True, capture_output=True)
    L = ctypes.CDLL(path)
    L.orc_ycc_coeffs.argtypes = [_i, _i, _vp, _vp]
    L.orc_ycc_coeffs.restype = None
    L.orc_ycc_convert.argtypes = [_i, _i, _vp, _vp, _l]
    L.orc_ycc_convert.restype = None
    L.orc_jpeg_decode_yuv.argtypes = [_vp, ctypes.c_size_t, _i, _i, _vp, _l]
    return L


def coeffs(yo, a, b):
    c, z = (ctypes.c_int * 9)(), (ctypes.c_double * 2)()
    yo.orc_ycc_coeffs(CS[a], CS[b], c, z)
    return list(c), list(z)


def matrices(name):
    """float64 RGB -> YCbCr and YCbCr -> RGB (over Y - o, Cb - 128, Cr - 128) of a space, from kr, kb and the range scales"""
    kr, kb = (.212639, .072192) if name == "Y709" else (.299, .114)
    kg = 1 - kr - kb
    yl, cl, o = (1., 1., 0) if name == "Y601full" else (219 / 255, 224 / 255, 16)
    fwd = np.array([[kr, kg, kb], [-kr, -kg, 1 - kb], [1 - kr, -kg, -kb]], np.float64)
    fwd[0] *= yl
    fwd[1] *= cl / (2 * (1 - kb))
    fwd[2] *= cl / (2 * (1 - kr))
    return fwd, np.linalg.inv(fwd), o


def matrix(a, b):
    return matrices(b)[0] @ matrices(a)[1]


def triples():
    y, cb, cr = [a.reshape(-1) for a in np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij")]
    return np.stack([y, cb, cr], 1).astype(np.uint8)


def convert(yo, a, b, ycc):
    out = np.empty_like(ycc)
    yo.orc_ycc_convert(CS[a], CS[b], ycc.ctypes.data, out.ctypes.data, len(ycc))
    return out


def oracle_yuv(yo, s, cs_in, cs_out, w, h, hs):
    pitch = (w + 1) // 2 * 4 if hs != 1 else w * 3
    out = np.zeros(pitch * h, np.uint8)
    b = np.frombuffer(s, np.uint8)
    assert yo.orc_jpeg_decode_yuv(b.ctypes.data, len(s), cs_in, cs_out, out.ctypes.data, pitch) == 0
    return out.reshape(h, pitch)


def gray_stream(img, q, ri=0):
    b = io.BytesIO()
    kw = {"restart_marker_blocks": ri} if ri else {}
    Image.fromarray(img, "L").save(b, "JPEG", quality=q, **kw)
    return b.getvalue()


def gray_image(w, h, seed=4):
    return natural_rgb(w, h, seed)[:, :, 1].copy()


def i420_of_uyvy(u, w, h):
    """uyvy_to_i420 (to_planar.c:343-378): chroma of a row pair averaged (a + b + 1) / 2, a last row without a partner taken as it is"""
    cw = (w + 1) // 2
    y = u[:, 1::2][:, :w]
    planes = [y.reshape(-1)]
    for k in (0, 2):
        c = u[:, k::4][:, :cw].astype(np.int32)
        top, bot = c[0::2], c[1::2]
        avg = (top[: len(bot)] + bot + 1) >> 1
        planes.append(np.concatenate([avg, top[len(bot):]]).astype(np.uint8).reshape(-1))
    return np.concatenate(planes)


# ---- CPU -----------------------------------------------------------------------------------------------------------------------------


def test_coefficients_are_the_rounded_float64_matrix(yo):
    for a in CS:
        c, z = coeffs(yo, a, a)
        assert c[:7] == [16384, 0, 0, 16384, 0, 0, 16384]
    for a, b in PAIRS:
        m = matrix(a, b)
        c, z = coeffs(yo, a, b)
        want = [m[0, 0], m[0, 1], m[0, 2], m[1, 1], m[1, 2], m[2, 1], m[2, 2]]
        assert c[:7] == [int(np.floor(abs(x) * 16384 + .5) * np.sign(x)) for x in want], (a, b)
        assert c[7:] == [matrices(a)[2], matrices(b)[2]]
        assert abs(m[1, 0]) < 1e-12 and abs(m[2, 0]) < 1e-12 and max(abs(v) for v in z) < 1e-8  # target chroma does not depend on source luma
        # there and back: the product of the two Q14 matrices is the identity within 2 LSB of Q14
        back, _ = coeffs(yo, b, a)
        q = lambda k: np.array([[k[0], k[1], k[2]], [0, k[3], k[4]], [0, k[5], k[6]]], np.float64)
        assert np.abs(q(back) @ q(c) / 16384 - 16384 * np.eye(3)).max() <= 2, (a, b)
    assert coeffs(yo, "Y601full", "Y709")[0] == [14071, -1663, -2992, 14660, 1649, 1080, 14757, 0, 16]  # pinned in csrc/color_space.h too


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{p[0]}-{p[1]}")
def test_conversion_of_every_triple(yo, pair):
    a, b = pair
    ycc = triples()
    got = convert(yo, a, b, ycc).astype(np.int64)
    (yy, yb, yr, bb, br, rb, rr, oi, oo), _ = coeffs(yo, a, b)
    y, cb, cr = ycc[:, 0].astype(np.int64) - oi, ycc[:, 1].astype(np.int64) - 128, ycc[:, 2].astype(np.int64) - 128
    want = np.stack([((yy * y + yb * cb + yr * cr + 8192) >> 14) + oo, ((bb * cb + br * cr + 8192) >> 14) + 128, ((rb * cb + rr * cr + 8192) >> 14) + 128], 1)
    assert np.array_equal(got, want.clip(0, 255))
    # against the unrounded matrix: each coefficient is off by at most 0.5 * 2^-14 and multiplies at most 255, 128 and 128, so the sum is off by
    # under 0.5 * 2^-14 * 511 = 0.016; the result is then rounded to nearest (0.5).  Within 0.516 of the exact value, so never 1 or more away.
    m = matrix(a, b)
    exact = np.stack([y, cb, cr], 1).astype(np.float64) @ m.T + np.array([oo, 128, 128])
    inside = (exact >= 0) & (exact <= 255)
    err = np.abs(got - exact)[inside]
    assert err.max() <= 0.5 + 0.5 / 16384 * 511 + 1e-9, err.max()


def test_jfif_to_709_matches_the_reference_two_step_path(yo, co):
    """in-gamut triples: Y601FULL -> Y709 against the reference's RGB -> UYVY line converter applied to the full-range BT.601 RGB.  The two-step
    path rounds twice more (RGB floored to 8 bits: up to 1 LSB of R, G, B, which the BT.709 rows - gains below 1 - pass on as under 1; then its own
    floor), so the results differ by at most 2."""
    ref = util.ref_cpu()
    if ref is None:
        pytest.skip("reference converters are not built")
    ycc = triples()
    fwd, inv, _ = matrices("Y601full")
    rgbf = (ycc.astype(np.float64) - np.array([0, 128, 128])) @ inv.T
    ycc = ycc[((rgbf >= 0) & (rgbf <= 255)).all(1)]
    ycc = ycc[: len(ycc) // 2 * 2]
    rgb = np.empty_like(ycc)
    co.orc_ycbcr_to_rgb(2, ycc.ctypes.data, rgb.ctypes.data, len(ycc))
    n = len(ycc)
    uyvy = util.convert_cpu(ref, "ref_convert", RGB, UYVY, rgb.reshape(-1), n, 1).reshape(-1, 4).astype(np.int32)
    got = convert(yo, "Y601full", "Y709", ycc).astype(np.int32)
    worst_y = max(np.abs(uyvy[:, 1] - got[0::2, 0]).max(), np.abs(uyvy[:, 3] - got[1::2, 0]).max())
    assert worst_y <= 2, worst_y


def pil_ycc(s, mode="YCbCr"):
    im = Image.open(io.BytesIO(s))
    im.draft(mode, im.size)  # libjpeg's own samples, no colour conversion
    return np.asarray(im.convert(mode) if im.mode != mode else im)


@pytest.mark.parametrize("q", [75, 90, 100])
@pytest.mark.parametrize("sub", [0, 1, 2], ids=["444", "422", "420"])
def test_jfif_to_709_against_libjpeg(yo, q, sub):
    """oracle decode_to(Y601FULL -> Y709) against the float64 matrix applied to libjpeg's own YCbCr samples (PIL draft mode: no colour conversion).
    At q 100 each of our samples is within 1 of libjpeg's (the IDCT bound); the luma row's absolute sum is 0.859 + 0.102 + 0.183 = 1.14 and the
    conversion adds 0.516 of rounding: under 1.66 + the chroma rows' 1.0 + 0.516, so 2.5 bounds every component.  Lower qualities let the two IDCTs
    differ by more on ringing chroma, bound 6.  The unconverted samples miss by over 12 (black is 0 where BT.709 wants 16).  Luma only where chroma
    is subsampled (libjpeg interpolates chroma, this decoder replicates it)."""
    w, h = 160, 96
    s = pil_stream(bars(w, h), q, sub)
    m = matrix("Y601full", "Y709")
    src = pil_ycc(s).astype(np.float64)
    want = (src - np.array([0, 128, 128])) @ m.T + np.array([16, 128, 128])
    out = oracle_yuv(yo, s, 2, 3, w, h, 1 if sub == 0 else 2)
    raw = oracle_yuv(yo, s, 0, 0, w, h, 1 if sub == 0 else 2)
    if sub == 0:
        got, unconv = out.reshape(h, w, 3).astype(np.float64), raw.reshape(h, w, 3).astype(np.float64)
        if q == 100:  # chroma too, where quantisation leaves libjpeg's samples and ours within 1
            assert np.abs(got - want).max() <= 2.5
        got, unconv, want = got[:, :, 0], unconv[:, :, 0], want[:, :, 0]
    else:
        got, unconv, want = out[:, 1::2][:, :w].astype(np.float64), raw[:, 1::2][:, :w].astype(np.float64), want[:, :, 0]
        # luma takes the replicated chroma of its pair / quad where libjpeg's is interpolated: compare inside the flat bars only
        flat = np.zeros((h, w), bool)
        flat[2 : h // 2 - 2] = True
        for k in range(1, 8):
            flat[:, k * w // 8 - 18 : k * w // 8 + 18] = False
        got, unconv, want = got[flat], unconv[flat], want[flat]
    bound = 2.5 if q == 100 else 6  # lower qualities: chroma ringing between the two decoders' IDCTs is scaled by the luma row's chroma terms
    assert np.abs(got - want).max() <= bound, np.abs(got - want).max()
    assert np.abs(unconv - want).max() > 12  # the unconverted samples are far off: black is 0 where BT.709 wants 16


def _L():
    from ultragrid_b200 import _lib
    return _lib.load()


def test_grayscale_headers_and_declared_space():
    from ultragrid_b200 import api
    L = _L()
    s = gray_stream(gray_image(40, 24), 90)
    info = api.jpeg_image_info(s)
    assert (info.width, info.height, info.components, info.h_samp, info.v_samp, info.native_codec) == (40, 24, 1, 1, 1, UYVY)
    assert info.restart_interval == 0 and api.jpeg_image_info(gray_stream(gray_image(40, 24), 90, ri=2)).restart_interval == 2
    bare = strip_app0(s)
    two = bytearray(bare)  # sampling factors 2x2 on the one component have no effect (T.81 A.2.2)
    p = bytes(two).index(b"\xff\xc0")
    two[p + 11] = 0x22
    info2 = api.jpeg_image_info(bytes(two))
    assert (info2.h_samp, info2.v_samp, info2.components) == (1, 1, 1)
    d = lambda x: L.ugb200_jpeg_stream_color_space(x, len(x))
    assert d(s) == 2 and d(bare) == 3 and d(with_markers(bare, [adobe(1)])) == 2
    assert d(with_markers(bare, [spiff(8)])) == 2 and d(with_markers(bare, [spiff(8), JFIF])) == 2
    assert d(with_markers(bare, [spiff(1)])) == 3 and d(with_markers(bare, [spiff(4)])) == 1 and d(with_markers(bare, [spiff(3)])) == 2
    assert d(with_markers(bare, [spiff(10)])) == -4 and d(with_markers(bare, [spiff(2)])) == -4
    assert d(with_markers(bare, [adobe(0)])) == 3  # never RGB


@pytest.mark.parametrize("ri", [0, 3])
def test_grayscale_oracle_matches_libjpeg(yo, ri):
    for w, h in [(1, 1), (7, 5), (8, 8), (17, 9), (40, 24), (131, 37)]:
        img = gray_image(w, h)
        s = gray_stream(img, 90, ri)
        want = pil_ycc(s, "L").astype(np.int32)
        u = oracle_yuv(yo, s, 0, 0, w, h, 2)
        assert (u[:, 0::2] == 128).all()
        assert np.abs(u[:, 1::2][:, :w].astype(np.int32) - want).max() <= 1, (w, h)
        conv = oracle_yuv(yo, s, 2, 3, w, h, 2)[:, 1::2].astype(np.int32)
        assert np.array_equal(conv, ((14071 * u[:, 1::2].astype(np.int32) + 8192) >> 14) + 16)


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------


def stream_of(orc, kind, w, h, q=90):
    if kind == "pil-L":
        return gray_stream(gray_image(w, h), q), 2
    if kind == "pil-L-dri":
        return gray_stream(gray_image(w, h), q, ri=5), 2
    return make(orc, kind, w, h, q), (1 if kind == "pil-444" else 2)


def expected(api, Codec, yo, s, hs, cs_in, cs_out, w, h, out_c):
    """convert (oracle), then pack: UYVY words are the oracle's; I420 is uyvy_to_i420 of them; a 4:4:4 stream's VUYA is the
    oracle's triples reordered, its UYVY the VUYA -> UYVY line converter that ugb200_jpeg_decode uses (pinned to the reference by the pixfmt tests)"""
    import torch
    o = oracle_yuv(yo, s, cs_in, cs_out, w, h, hs)
    if hs == 1:
        t = o.reshape(h, w, 3)
        vuya = np.concatenate([t[:, :, 2:3], t[:, :, 1:2], t[:, :, 0:1], np.full((h, w, 1), 255, np.uint8)], 2).reshape(-1)
        if out_c == int(Codec.VUYA):
            return vuya
        uy = api.pixfmt_convert(Codec.VUYA, Codec.UYVY, torch.from_numpy(vuya).cuda(), w, h).cpu().numpy()
        return uy if out_c == UYVY else i420_of_uyvy(uy.reshape(h, -1), w, h)
    if out_c == UYVY:
        return o.reshape(-1)
    if out_c == int(Codec.I420):
        return i420_of_uyvy(o, w, h)
    raise AssertionError("VUYA is an output of 4:4:4 streams only (ugb200_jpeg_decode refuses it for the others)")


KINDS = ["pil-444", "pil-422", "pil-420", "pil-L", "pil-L-dri", "ours-422"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_decode_to_equals_oracle(orc, yo, kind):
    import torch
    from ultragrid_b200 import Codec, api
    dec = api.JpegDecoder()
    sizes = [(200, 120), (131, 37), (17, 9), (33, 18), (1, 1)]
    for w, h in sizes:
        s, hs = stream_of(orc, kind, w, h)
        declared = api.JPEG_CS[api.jpeg_stream_color_space(s)]
        for cs_in, cs_out in [(CS[a], CS[b]) for a, b in PAIRS] + [(NATIVE, 3), (3, NATIVE), (2, 2), (AUTO, 3), (AUTO, 1)]:
            eff = declared if cs_in == AUTO else cs_in
            for out_c in (UYVY, int(Codec.I420)) + ((int(Codec.VUYA),) if hs == 1 else ()):
                want = expected(api, Codec, yo, s, hs, eff, cs_out, w, h, out_c)
                got = dec.decode_to(s, out_c, cs_in, cs_out)
                assert np.array_equal(got, want), (kind, w, h, cs_in, cs_out, out_c)
            ls = (w + 1) // 2 * 4
            pitch = ls + 48
            out = torch.full((pitch * h,), 0x5A, dtype=torch.uint8, device="cuda")
            dec.decode_to(s, UYVY, cs_in, cs_out, device=True, pitch=pitch, out=out)
            g = out.cpu().numpy().reshape(h, pitch)
            want = expected(api, Codec, yo, s, hs, eff, cs_out, w, h, UYVY).reshape(h, ls)
            assert np.array_equal(g[:, :ls], want) and (g[:, ls:] == 0x5A).all(), (kind, w, h, cs_in, cs_out)
    dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("sync", ["on", "off"])
@pytest.mark.parametrize("scan", ["host", "device"])
def test_gpu_decode_to_routes(orc, yo, monkeypatch, sync, scan):
    from ultragrid_b200 import Codec, api
    monkeypatch.setenv("UGB200_JPEG_SYNC", sync)
    monkeypatch.setenv("UGB200_JPEG_MARKER_SCAN", scan)
    dec = api.JpegDecoder()
    for kind in KINDS:
        for w, h in [(200, 120), (131, 37)]:
            s, hs = stream_of(orc, kind, w, h)
            for out_c in (UYVY, int(Codec.I420)):
                assert np.array_equal(dec.decode_to(s, out_c, 2, 3), expected(api, Codec, yo, s, hs, 2, 3, w, h, out_c)), (kind, w, h, out_c)
    dec.close()


@pytest.mark.gpu
def test_gpu_decode_to_4k(orc, yo):
    from ultragrid_b200 import Codec, api
    dec = api.JpegDecoder()
    for kind in ("pil-422", "pil-420", "pil-L"):
        w, h = 3840, 2160
        s, hs = stream_of(orc, kind, w, h)
        for out_c in (UYVY, int(Codec.I420)):
            assert np.array_equal(dec.decode_to(s, out_c, AUTO, 3), expected(api, Codec, yo, s, hs, 2, 3, w, h, out_c)), (kind, out_c)
    dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_identities(orc, yo, co, kind):
    """decode_to(NATIVE, NATIVE) == ugb200_jpeg_decode; RGB / RGBA of decode_to == ugb200_jpeg_decode_cs whatever out_cs says.  Grayscale, which the
    two older calls refuse as before: RGB / RGBA == the colour oracle's conversion of the UYVY words with Cb = Cr = 128"""
    from ultragrid_b200 import Codec, api
    dec = api.JpegDecoder()
    gray = kind.startswith("pil-L")
    for w, h in [(200, 120), (131, 37), (17, 9)]:
        s, hs = stream_of(orc, kind, w, h)
        for out_c in (UYVY, int(Codec.I420), RGB, RGBA) + ((int(Codec.VUYA),) if hs == 1 else ()):
            try:
                want = dec.decode(s, out_c)
            except RuntimeError as e:  # grayscale, or an output ugb200_jpeg_decode has no line converter for
                assert "-4" in str(e)
                if not gray:
                    with pytest.raises(RuntimeError):
                        dec.decode_to(s, out_c, NATIVE, NATIVE)
                continue
            assert not gray
            assert np.array_equal(dec.decode_to(s, out_c, NATIVE, NATIVE), want), (kind, w, h, out_c)
            assert np.array_equal(dec.decode_to(s, out_c, NATIVE, 3), want), (kind, w, h, out_c)
        for cs in (1, 2, 3, AUTO):
            for out_c, shifts in [(RGB, (0, 8, 16)), (RGBA, (0, 8, 16)), (RGBA, (16, 8, 0)), (RGBA, (8, 16, 24))]:
                got = dec.decode_to(s, out_c, cs, 1, shifts=shifts)
                if not gray:
                    assert np.array_equal(got, dec.decode(s, out_c, shifts=shifts, color_space=cs)), (kind, w, h, cs, out_c)
                elif cs != AUTO:
                    u = oracle_yuv(yo, s, 0, 0, w, h, 2)
                    bpp = 4 if out_c == RGBA else 3
                    want = np.zeros(w * bpp * h, np.uint8)
                    co.orc_uyvy_to_rgb_cs(cs, u.ctypes.data, u.shape[1], w, h, int(out_c == RGBA), *shifts, want.ctypes.data, w * bpp)
                    n = (w // 2) * 2 * bpp
                    assert np.array_equal(got.reshape(h, -1)[:, :n], want.reshape(h, -1)[:, :n]), (w, h, cs, out_c, shifts)
                    if cs == 2 and out_c == RGB:  # full range: R = G = B = Y
                        assert np.array_equal(got.reshape(h, -1)[:, 0:n:3], u[:, 1::2][:, : w // 2 * 2])
    dec.close()


@pytest.mark.gpu
def test_gpu_refusals_leave_output_untouched(orc):
    import torch
    from ultragrid_b200 import Codec, api
    from test_jpeg import orc_encode
    L = _L()
    dec = api.JpegDecoder()
    w, h = 64, 32
    rgb_stream = orc_encode(orc, natural_rgb(w, h, 2).reshape(-1), w, h, RGB, 90)
    ycc = pil_stream(natural_rgb(w, h, 2), 90, 1)
    out = torch.full((w * h * 4,), 0xC3, dtype=torch.uint8, device="cuda")
    host = np.full(w * h * 4, 0xC3, np.uint8)
    call = lambda s, out_c, a, b, dev=1: L.ugb200_jpeg_decode_to(dec._h, api._bytes_ptr(s), len(s), ctypes.c_void_p(out.data_ptr() if dev else host.ctypes.data), dev, 0,
                                                                 out_c, 0, 8, 16, a, b)
    for dev in (1, 0):
        assert call(ycc, UYVY, 2, 4, dev) == -1 and call(ycc, UYVY, 2, AUTO, dev) == -1 and call(ycc, UYVY, 2, 7, dev) == -1 and call(ycc, UYVY, 9, 3, dev) == -1
        assert call(rgb_stream, UYVY, NATIVE, 1, dev) == -4 and call(rgb_stream, int(Codec.I420), AUTO, 2, dev) == -4
        assert call(with_markers(strip_app0(ycc), [spiff(10)]), UYVY, AUTO, 1, dev) == -4  # declares RGB: never matrixed, so no BT.601 output
    assert (out.cpu().numpy() == 0xC3).all() and (host == 0xC3).all()
    assert np.array_equal(dec.decode_to(rgb_stream, UYVY, AUTO, 3), dec.decode(rgb_stream, UYVY))
    assert np.array_equal(dec.decode_to(rgb_stream, UYVY, NATIVE, NATIVE), dec.decode(rgb_stream, UYVY))
    dec.close()


def i420_planes(torch, w, h):
    cw, ch = (w + 1) // 2, (h + 1) // 2
    buf = torch.full((w * h + 2 * cw * ch,), 0x3C, dtype=torch.uint8, device="cuda")
    return buf, [buf[: w * h], buf[w * h : w * h + cw * ch], buf[w * h + cw * ch :]], [w, cw, cw]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pil-422", "pil-420", "ours-422", "pil-L"])
def test_gpu_planar_epilogue_equals_uyvy_then_uyvy_to_i420(orc, kind):
    """I420 written by the fused kernel's planar epilogue == the same decode to UYVY followed by ugb200_uyvy_to_i420 (the two-pass route it replaces,
    pinned to the reference's to_planar.c by test_planar.py): odd and even sizes, with and without the matrix, host and device destinations,
    through ugb200_jpeg_decode as well"""
    import torch
    from ultragrid_b200 import Codec, api
    dec = api.JpegDecoder()
    sizes = [(200, 120), (208, 64), (98, 50)] + ([] if kind == "ours-422" else [(131, 37), (17, 9), (33, 18), (2, 1), (1, 1), (1921, 1081)])
    for w, h in sizes:
        s, _ = stream_of(orc, kind, w, h)
        for cs_in, cs_out in [(NATIVE, NATIVE), (2, 3), (3, 1)]:
            uy = dec.decode_to(s, UYVY, cs_in, cs_out, device=True)
            buf, planes, ls = i420_planes(torch, w, h)
            api.to_planar("uyvy_to_i420", uy, w, h, planes, ls)
            torch.cuda.synchronize()
            want = buf.cpu().numpy()
            assert np.array_equal(dec.decode_to(s, int(Codec.I420), cs_in, cs_out), want), (kind, w, h, cs_in, cs_out)
            out = torch.full((want.size + 32,), 0x77, dtype=torch.uint8, device="cuda")
            dec.decode_to(s, int(Codec.I420), cs_in, cs_out, device=True, out=out)
            g = out.cpu().numpy()
            assert np.array_equal(g[: want.size], want) and (g[want.size:] == 0x77).all(), (kind, w, h, cs_in, cs_out)
            if cs_in == NATIVE and kind != "pil-L":
                assert np.array_equal(dec.decode(s, int(Codec.I420)), want), (kind, w, h)
    dec.close()


@pytest.mark.gpu
def test_gpu_modules_with_and_without_the_colour_space_switch(orc, monkeypatch):
    """the mirror-ABI gpujpeg module: UGB200_JPEG_DECODE_CS=auto gives decode_to(AUTO -> Y709) for UYVY and decode_cs(AUTO) for RGB; unset, the bytes of
    ugb200_jpeg_decode; a grayscale stream decodes either way; gpujpeg_to_dxt encodes the RGB the switch selects"""
    from ultragrid_b200 import api
    from ultragrid_b200.compress import Decompress
    JPEG, DXT1 = 13, 9
    w, h = 320, 200
    s = pil_stream(bars(w, h), 90, 1)
    gray = gray_stream(gray_image(w, h), 90)
    dec = api.JpegDecoder()

    def through(stream, out_c):
        d = Decompress(JPEG, out_c)
        d.reconfigure(w, h, JPEG, out_c)
        st, out, _ = d.frame(stream)
        d.close()
        assert st == Decompress.GOT_FRAME
        return out

    monkeypatch.delenv("UGB200_JPEG_DECODE_CS", raising=False)
    assert np.array_equal(through(s, UYVY), dec.decode(s, UYVY)) and np.array_equal(through(s, RGB), dec.decode(s, RGB))
    assert np.array_equal(through(gray, UYVY), dec.decode_to(gray, UYVY, NATIVE, NATIVE))
    assert np.array_equal(through(gray, RGB), dec.decode_to(gray, RGB, NATIVE, NATIVE))
    plain_dxt = through(s, DXT1)
    monkeypatch.setenv("UGB200_JPEG_DECODE_CS", "auto")
    conv = through(s, UYVY)
    assert np.array_equal(conv, dec.decode_to(s, UYVY, AUTO, 3)) and not np.array_equal(conv, dec.decode(s, UYVY))
    assert np.array_equal(through(s, RGB), dec.decode(s, RGB, color_space="auto"))
    assert np.array_equal(through(gray, UYVY), dec.decode_to(gray, UYVY, AUTO, 3))
    assert np.array_equal(through(gray, RGB), dec.decode_to(gray, RGB, AUTO, 3))
    assert not np.array_equal(through(s, DXT1), plain_dxt)
    monkeypatch.setenv("UGB200_JPEG_DECODE_CS", "y709")
    assert np.array_equal(through(s, UYVY), dec.decode(s, UYVY))  # Y709 -> Y709: the stream's samples
    dec.close()
