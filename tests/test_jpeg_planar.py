"""JPEG encoder, planar layouts (ugb200_jpeg_encode_device_ex / _into_ex): I420 input, UYVY -> 4:2:0, RGB -> YCbCr 4:4:4 / 4:2:2 / 4:2:0.
GPUJPEG's own pre-processor and bitstream are absent here (parity unpinned against them); pinned instead:
  * CPU: the restatement tests/jpeg_planar_oracle.c (orc_jpeg_prep, orc_jpeg_encode_planar) against what the tree pins: the RGB_TO_* rows
    of rgb_to_yuv444p (oracle/lavc_oracle.c), uyvy_to_i420 (oracle/planar_oracle.c and, when built, the unmodified reference), libjpeg (PIL)
    decoding the streams, and PSNR within a fraction of a dB of libjpeg's own encoder;
  * GPU: the product's stream == orc_jpeg_encode_planar(orc_jpeg_prep(src)) byte for byte; native _ex parameters == the plain calls;
    the project's decoder reads the 4:2:0 streams back like the CPU decode oracle does."""
import ctypes
import io
import os
import subprocess
import tempfile

import numpy as np
import pytest
from PIL import Image

import util
from test_jpeg import RGB, UYVY, natural_rgb, orc_encode, psnr

I420 = 29
CS = {"native": 0, "Y601": 1, "Y601full": 2, "Y709": 3, "RGB": 4}
_vp, _i, _l = ctypes.c_void_p, ctypes.c_int, ctypes.c_long
HERE = os.path.dirname(os.path.abspath(__file__))

# the new rows of the supported matrix: (input codec, subsampling, colour space, interleaved)
ROWS = [(UYVY, 420, "native", 1), (UYVY, 420, "Y709", 1), (I420, 0, "native", 1), (I420, 420, "Y709", 1)] + \
       [(RGB, sub, cs, il) for sub in (0, 422, 420) for cs in ("Y709", "Y601", "Y601full") for il in (0, 1)]
SIZES = [(1, 1), (17, 9), (100, 52), (130, 37), (640, 360)]
RIS = [0, 1, 3, 7]


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


@pytest.fixture(scope="module")
def pl():
    """the planar oracle, compiled on its own (it includes oracle/jpeg_oracle.c)"""
    d = tempfile.mkdtemp(prefix="ugb_planar_oracle_")
    path = os.path.join(d, "libjpegplanar.so")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fvisibility=hidden", "-o", path,
                    os.path.join(HERE, "jpeg_planar_oracle.c"), "-lm"], check=True, capture_output=True)
    L = ctypes.CDLL(path)
    L.orc_jpeg_prep.argtypes = [_vp, _l, _i, _i, _i, _i, _i, _vp, _vp]
    L.orc_jpeg_prep_coeffs.argtypes = [_i, _vp]
    L.orc_jpeg_prep_coeffs.restype = None
    L.orc_jpeg_encode_planar.argtypes = [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, ctypes.c_size_t]
    L.orc_jpeg_encode_planar.restype = ctypes.c_size_t
    return L


def sampling(codec, sub):
    if codec != RGB:
        return 2, 2
    return (2 if sub in (422, 420) else 1), (2 if sub == 420 else 1)


def layout(codec, sub, ri, interleaved):
    """restart interval and scan layout as the encoder resolves them (gpujpeg.cpp:303,351)"""
    return (ri or (8 if codec == RGB else 4)), (interleaved if codec == RGB else 1)


def prep(pl, src, w, h, codec, sub, cs, pitch=0):
    hs, vs = sampling(codec, sub)
    cw, ch = (w + hs - 1) // hs, (h + vs - 1) // vs
    pitch = pitch or (w * 3 if codec == RGB else (w + 1) // 2 * 4)
    planes = [np.zeros(w * h, np.uint8), np.zeros(cw * ch, np.uint8), np.zeros(cw * ch, np.uint8)]
    p = (_vp * 3)(*[a.ctypes.data for a in planes])
    ls = (_i * 3)(w, cw, cw)
    rc = pl.orc_jpeg_prep(src.ctypes.data, pitch, w, h, codec, sub, CS[cs], p, ls)
    assert rc == 0, rc
    return planes


def encode_planar(pl, planes, w, h, hs, vs, q, ri, interleaved):
    cw = (w + hs - 1) // hs
    p = (_vp * 3)(*[a.ctypes.data for a in planes])
    ls = (_i * 3)(w, cw, cw)
    cap = 4096 + ((w + 15) // 16 + 1) * ((h + 15) // 16 + 1) * 6 * 418 + ((w + 7) // 8 + 1) * ((h + 7) // 8 + 1) * 3 * 418
    out = np.zeros(cap, np.uint8)
    n = pl.orc_jpeg_encode_planar(p, ls, w, h, hs, vs, q, ri, interleaved, out.ctypes.data, cap)
    assert n > 0
    return out[:n].tobytes()


def oracle_stream(pl, src, w, h, codec, sub, cs, q, ri, interleaved, pitch=0):
    hs, vs = sampling(codec, sub)
    ri, il = layout(codec, sub, ri, interleaved)
    return encode_planar(pl, prep(pl, src, w, h, codec, sub, cs, pitch), w, h, hs, vs, q, ri, il)


def source(orc, codec, w, h, seed, noise=False):
    rgb = util.rng_bytes(w * h * 3, seed).reshape(h, w, 3) if noise else natural_rgb(w, h, seed)
    if codec == RGB:
        return np.ascontiguousarray(rgb).reshape(-1)
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, np.ascontiguousarray(rgb).reshape(-1), w, h)
    if codec == UYVY:
        return uyvy
    cw, ch = (w + 1) // 2, (h + 1) // 2  # I420 = uyvy_to_i420 of the UYVY frame
    planes = [np.zeros(w * h, np.uint8), np.zeros(cw * ch, np.uint8), np.zeros(cw * ch, np.uint8)]
    orc_uyvy_to_i420(orc, uyvy, w, h, planes)
    return np.concatenate(planes)


class ToPlanarData(ctypes.Structure):
    _fields_ = [("width", _i), ("height", _i), ("out_data", _vp * 4), ("out_linesize", ctypes.c_uint * 4), ("in_data", _vp)]


def orc_uyvy_to_i420(lib, uyvy, w, h, planes, name="orc_uyvy_to_i420"):
    d = ToPlanarData()
    d.width, d.height, d.in_data = w, h, uyvy.ctypes.data
    cw = (w + 1) // 2
    for k, (a, ls) in enumerate(zip(planes, (w, cw, cw))):
        d.out_data[k], d.out_linesize[k] = a.ctypes.data, ls
    fn = getattr(lib, name)
    fn.argtypes, fn.restype = [ToPlanarData], None
    fn(d)


def coeffs(pl, cs):
    c = (_i * 9)()
    pl.orc_jpeg_prep_coeffs(CS[cs], c)
    return np.array(list(c), np.int64)


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_prep_coefficients_are_the_color_space_ones(pl, orc):
    """Y709 = coeffs_709(8), Y601 = coeffs_601(8), Y601full = coeffs_601(0) of csrc/color_space.h (as the pixfmt oracle computes them)"""
    for cs, (which, depth) in (("Y709", (0, 8)), ("Y601", (1, 8)), ("Y601full", (1, 0))):
        out = (_i * 14)()
        orc.orc_get_color_coeffs(which, depth, out)
        assert list(coeffs(pl, cs)) == list(out)[:9], cs
    assert list(coeffs(pl, "Y709")[:3]) == [2992, 10063, 1016]  # pinned in color_space.h


@pytest.mark.parametrize("cs", ["Y709", "Y601", "Y601full"])
def test_colour_transform_stays_in_range_over_the_rgb_cube(pl, cs):
    """every RGB value maps into 0..255 (no clamp needed); prep at 4:4:4 equals the formula over the whole cube"""
    c = coeffs(pl, cs)
    off_y = 0 if cs == "Y601full" else 16
    v = np.arange(1 << 24, dtype=np.int64)
    cube = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], axis=1)
    w = h = 4096
    planes = prep(pl, cube.astype(np.uint8).reshape(-1), w, h, RGB, 0, cs)
    for k, base in ((0, off_y), (1, 128), (2, 128)):
        for s in range(0, 1 << 24, 1 << 22):
            x = cube[s:s + (1 << 22)]
            val = ((x[:, 0] * c[3 * k] + x[:, 1] * c[3 * k + 1] + x[:, 2] * c[3 * k + 2]) >> 14) + base
            assert val.min() >= 0 and val.max() <= 255, (cs, k, val.min(), val.max())
            assert np.array_equal(planes[k][s:s + (1 << 22)], val.astype(np.uint8)), (cs, k, s)


def test_prep_rgb_444_y709_equals_rgb_to_yuv444p(pl, orc):
    """the RGB_TO_* expressions of rgb_to_yuv444p (to_lavc_vid_conv.c:1206-1214) as oracle/lavc_oracle.c restates them"""
    class Coeffs(ctypes.Structure):
        _fields_ = [(n, _i) for n in ("y_r", "y_g", "y_b", "cb_r", "cb_g", "cb_b", "cr_r", "cr_g", "cr_b")]
    for w, h in ((1, 1), (17, 9), (130, 37)):
        rgb = util.rng_bytes(w * h * 3, w + h)
        got = prep(pl, rgb, w, h, RGB, 444, "Y709")
        want = [np.zeros(w * h, np.uint8) for _ in range(3)]
        p, ls = (_vp * 3)(*[a.ctypes.data for a in want]), (_i * 3)(w, w, w)
        orc.orc_lavc_rgb(3, 8, 0, ctypes.byref(Coeffs(*coeffs(pl, "Y709").tolist())), rgb.ctypes.data, w, h, p, ls)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), (w, h)


@pytest.mark.parametrize("w,h", [(1, 1), (2, 1), (17, 9), (18, 3), (101, 52), (130, 37)])
def test_prep_uyvy_420_equals_uyvy_to_i420(pl, orc, w, h):
    uyvy = util.rng_bytes((w + 1) // 2 * 4 * h, 7 * w + h)
    got = prep(pl, uyvy, w, h, UYVY, 420, "native")
    cw, ch = (w + 1) // 2, (h + 1) // 2
    for lib, name in ((orc, "orc_uyvy_to_i420"), (util.ref_cpu(), "uyvy_to_i420")):
        if lib is None:
            continue  # the unmodified reference objects are not built here (oracle/_ref)
        want = [np.zeros(w * h, np.uint8), np.zeros(cw * ch, np.uint8), np.zeros(cw * ch, np.uint8)]
        orc_uyvy_to_i420(lib, uyvy, w, h, want, name)
        for k, (a, b) in enumerate(zip(got, want)):
            assert np.array_equal(a, b), (name, k)


def test_prep_refuses_what_the_encoder_refuses(pl):
    src = np.zeros(64 * 3, np.uint8)
    planes = [np.zeros(64, np.uint8) for _ in range(3)]
    p, ls = (_vp * 3)(*[a.ctypes.data for a in planes]), (_i * 3)(8, 8, 8)
    assert pl.orc_jpeg_prep(src.ctypes.data, 0, 8, 8, UYVY, 444, 0, p, ls) == -4
    assert pl.orc_jpeg_prep(src.ctypes.data, 0, 8, 8, I420, 422, 0, p, ls) == -4
    assert pl.orc_jpeg_prep(src.ctypes.data, 0, 8, 8, RGB, 420, CS["native"], p, ls) == -4


@pytest.mark.parametrize("codec,sub,cs,il", ROWS)
def test_oracle_streams_decode_with_libjpeg(pl, orc, codec, sub, cs, il):
    for w, h in SIZES:
        src = source(orc, codec, w, h, w + h)
        for ri in RIS:
            s = oracle_stream(pl, src, w, h, codec, sub, cs, 75, ri, il)
            im = Image.open(io.BytesIO(s))
            im.load()
            assert im.size == (w, h) and im.mode == "RGB", (w, h, ri)
            hs, vs = sampling(codec, sub)
            assert s[s.index(b"\xff\xc0") + 11] == (hs << 4 | vs)
            assert (b"JFIF" in s[:32]) and (b"Adobe" not in s[:64])


def _y_psnr_vs_libjpeg(pl, w, h, q, ri, interleaved):
    rgb = natural_rgb(w, h, 9)
    planes = prep(pl, np.ascontiguousarray(rgb).reshape(-1), w, h, RGB, 420, "Y601full")
    ours = encode_planar(pl, planes, w, h, 2, 2, q, ri, interleaved)
    cw, ch = (w + 1) // 2, (h + 1) // 2
    ycc = np.stack([planes[0].reshape(h, w), np.repeat(np.repeat(planes[1].reshape(ch, cw), 2, 0), 2, 1)[:h, :w],
                    np.repeat(np.repeat(planes[2].reshape(ch, cw), 2, 0), 2, 1)[:h, :w]], axis=2)
    b = io.BytesIO()
    Image.fromarray(ycc, "YCbCr").save(b, "JPEG", quality=q, subsampling="4:2:0")
    y0 = planes[0].reshape(h, w)

    def y_of(stream):
        im = Image.open(io.BytesIO(stream))
        im.draft("YCbCr", (w, h))
        return np.asarray(im)[:, :, 0]
    return psnr(y_of(ours), y0), psnr(y_of(b.getvalue()), y0)


@pytest.mark.parametrize("q", [50, 75, 90])
def test_oracle_420_luma_psnr_close_to_libjpeg(pl, q):
    """the Y plane of our 4:2:0 stream is as good as libjpeg's own encoder on the same planes (Annex K tables, same quality scaling)"""
    for interleaved in (0, 1):
        ours, lib = _y_psnr_vs_libjpeg(pl, 640, 360, q, 8, interleaved)
        assert ours >= lib - 0.3, (q, interleaved, ours, lib)


@pytest.mark.parametrize("q", [50, 75, 90])
def test_oracle_y601full_rgb_close_to_libjpeg(pl, q):
    """JFIF both: PIL's RGB decode of our RGB -> Y601full 4:2:0 stream against PIL's own encode of the same RGB"""
    w, h = 640, 360
    rgb = natural_rgb(w, h, 3)
    ours = oracle_stream(pl, np.ascontiguousarray(rgb).reshape(-1), w, h, RGB, 420, "Y601full", q, 0, 0)
    b = io.BytesIO()
    Image.fromarray(rgb).save(b, "JPEG", quality=q, subsampling="4:2:0")
    p_ours = psnr(np.asarray(Image.open(io.BytesIO(ours)).convert("RGB")), rgb)
    p_lib = psnr(np.asarray(Image.open(io.BytesIO(b.getvalue())).convert("RGB")), rgb)
    assert p_ours >= p_lib - 0.5, (q, p_ours, p_lib)


# ---- GPU ------------------------------------------------------------------------------------------------------------------
def _enc():
    from ultragrid_b200 import api
    return api.JpegEncoder()


def _gpu_stream(enc, src, w, h, codec, sub, cs, q, ri, il, pitch=0, device=True):
    import torch
    if codec == UYVY and not pitch:
        pitch = (w + 1) // 2 * 4  # the frames here are vc_get_linesize wide; pitch 0 means 2 * w bytes, as for the 4:2:2 stream
    if device:
        t = torch.from_numpy(src).cuda()
        enc.encode_device(t, w, h, codec, quality=q, restart_interval=ri, pitch=pitch, interleaved=bool(il), subsampling=sub, color_space=CS[cs])
        return enc.result()
    return enc.encode(src, w, h, codec, quality=q, restart_interval=ri, pitch=pitch, interleaved=bool(il), subsampling=sub, color_space=CS[cs])


@pytest.mark.gpu
@pytest.mark.parametrize("codec,sub,cs,il", ROWS)
def test_gpu_planar_equals_oracle_bytes(pl, orc, codec, sub, cs, il):
    enc = _enc()
    for w, h in SIZES + [(1920, 1080)]:
        src = source(orc, codec, w, h, 3 * w + h)
        for q in (1, 90, 100) if w < 1000 else (90,):
            for ri in RIS if w < 1000 else (0,):
                want = oracle_stream(pl, src, w, h, codec, sub, cs, q, ri, il)
                assert _gpu_stream(enc, src, w, h, codec, sub, cs, q, ri, il) == want, (w, h, q, ri)
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("codec,sub,cs,il", [(UYVY, 420, "native", 1), (I420, 0, "native", 1), (RGB, 420, "Y709", 0), (RGB, 420, "Y709", 1),
                                             (RGB, 422, "Y601", 0), (RGB, 0, "Y601full", 1)])
def test_gpu_planar_large_frames(pl, orc, codec, sub, cs, il):
    enc = _enc()
    for w, h in ((3840, 2160), (7680, 4320)):
        src = source(orc, codec, w, h, 11)
        assert _gpu_stream(enc, src, w, h, codec, sub, cs, 90, 0, il) == oracle_stream(pl, src, w, h, codec, sub, cs, 90, 0, il), (w, h)
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("codec,sub,cs,il", [(I420, 0, "native", 1), (RGB, 420, "Y601full", 0), (UYVY, 420, "native", 1)])
def test_gpu_planar_8k_noise_q100(pl, orc, codec, sub, cs, il):
    w, h = 7680, 4320
    src = source(orc, codec, w, h, 21, noise=True)
    enc = _enc()
    assert _gpu_stream(enc, src, w, h, codec, sub, cs, 100, 0, il) == oracle_stream(pl, src, w, h, codec, sub, cs, 100, 0, il)
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("codec,sub,cs,il", [(UYVY, 420, "native", 1), (RGB, 420, "Y709", 0), (RGB, 422, "Y601full", 1)])
def test_gpu_planar_padded_pitch_and_8_byte_aligned_source(pl, orc, codec, sub, cs, il):
    import torch
    enc = _enc()
    for w, h in ((130, 37), (640, 360)):
        bpp = 3 if codec == RGB else 2
        ls = w * bpp if codec == RGB else (w + 1) // 2 * 4
        src = source(orc, codec, w, h, w)
        pitch = ls + 40
        padded = np.full((h, pitch), 0xA5, np.uint8)
        padded[:, :ls] = src.reshape(h, ls)
        want = oracle_stream(pl, src, w, h, codec, sub, cs, 90, 0, il, pitch=ls)
        assert _gpu_stream(enc, padded.reshape(-1), w, h, codec, sub, cs, 90, 0, il, pitch=pitch) == want, ("pitch", w, h)
        buf = torch.zeros(ls * h + 64, dtype=torch.uint8, device="cuda")  # 8 bytes past a 256-byte aligned allocation
        buf[8:8 + ls * h] = torch.from_numpy(src).cuda()
        enc.encode_device(buf[8:], w, h, codec, quality=90, pitch=ls, interleaved=bool(il), subsampling=sub, color_space=CS[cs])
        assert enc.result() == want, ("aligned 8", w, h)
    enc.close()


@pytest.mark.gpu
def test_gpu_i420_from_host_and_device(pl, orc):
    enc = _enc()
    for w, h in ((17, 9), (130, 37), (1920, 1080)):
        src = source(orc, I420, w, h, 5)
        want = oracle_stream(pl, src, w, h, I420, 0, "native", 80, 0, 1)
        assert _gpu_stream(enc, src, w, h, I420, 0, "native", 80, 0, 1, device=False) == want
        assert _gpu_stream(enc, src, w, h, I420, 0, "native", 80, 0, 1, device=True) == want
    enc.close()


@pytest.mark.gpu
def test_gpu_ex_with_native_parameters_gives_the_plain_bytes(orc):
    import torch
    from ultragrid_b200 import api, _lib
    L = _lib.load()
    enc = _enc()
    for codec, w, h in ((UYVY, 640, 360), (UYVY, 130, 37), (RGB, 640, 360), (RGB, 17, 9)):
        src = source(orc, codec, w, h, 2)
        plain = enc.encode(src, w, h, codec, quality=90)
        for cs in ("native", "Y709" if codec == UYVY else "RGB"):
            for sub in (0, 422 if codec == UYVY else 444):
                px = api.JpegParamsEx()
                L.ugb200_jpeg_default_params_ex(ctypes.byref(px))
                px.base.quality, px.subsampling, px.color_space = 90, sub, CS[cs]
                dst, n = np.zeros(w * h * 3 + 4096, np.uint8), ctypes.c_size_t()
                assert L.ugb200_jpeg_encode_into_ex(enc._h, src.ctypes.data, 0, 0, w, h, codec, ctypes.byref(px), dst.ctypes.data, dst.size, ctypes.byref(n)) == 0
                assert dst[:n.value].tobytes() == plain, (codec, w, h, cs, sub)
                t = torch.from_numpy(src).cuda()
                assert L.ugb200_jpeg_encode_device_ex(enc._h, t.data_ptr(), 0, w, h, codec, ctypes.byref(px)) == 0
                assert enc.result() == plain
    # what needs upsampling, a YCbCr -> RGB transform, another matrix or subsampled RGB is refused with -4
    t = torch.zeros(64 * 64 * 3, dtype=torch.uint8, device="cuda")
    for codec, sub, cs in ((UYVY, 444, "native"), (I420, 422, "native"), (UYVY, 0, "RGB"), (I420, 0, "Y601"), (RGB, 420, "RGB"), (RGB, 420, "native")):
        px = api.JpegParamsEx()
        L.ugb200_jpeg_default_params_ex(ctypes.byref(px))
        px.subsampling, px.color_space = sub, CS[cs]
        assert L.ugb200_jpeg_encode_device_ex(enc._h, t.data_ptr(), 0, 64, 64, codec, ctypes.byref(px)) == -4, (codec, sub, cs)
    assert L.ugb200_jpeg_encode_device(enc._h, t.data_ptr(), 0, 64, 64, I420, ctypes.byref(api.JpegParams(75, 0, 0))) == -4  # plain call unchanged
    enc.close()


ALTERNATING = [(UYVY, 0, "native", 0), (I420, 0, "native", 1), (RGB, 420, "Y601full", 0), (RGB, 0, "RGB", 0)]


def _alt_want(pl, orc, w, h, k):
    codec, sub, cs, il = ALTERNATING[k]
    src = source(orc, codec, w, h, 40 + k)
    if sub == 0 and cs in ("native", "RGB") and codec != I420:
        return src, orc_encode(orc, src, w, h, codec, 90, 0)
    return src, oracle_stream(pl, src, w, h, codec, sub, cs, 90, 0, il)


@pytest.mark.gpu
def test_gpu_one_encoder_alternating_layouts(pl, orc):
    """the configure() cache key covers subsampling and colour space: no stale geometry, tables or planes"""
    w, h = 320, 184
    cases = [_alt_want(pl, orc, w, h, k) for k in range(4)]
    enc = _enc()
    for _ in range(3):
        for k, (src, want) in enumerate(cases):
            codec, sub, cs, il = ALTERNATING[k]
            assert _gpu_stream(enc, src, w, h, codec, sub, cs, 90, 0, il) == want, k
    enc.close()


@pytest.mark.gpu
def test_gpu_two_encoders_on_two_streams(pl, orc):
    import torch
    from ultragrid_b200 import api
    w, h = 1920, 1080
    a = [_alt_want(pl, orc, w, h, k) for k in (1, 2)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    e1, e2 = api.JpegEncoder(s1), api.JpegEncoder(s2)
    d = [torch.from_numpy(src).cuda() for src, _ in a]
    torch.cuda.synchronize()
    for _ in range(3):
        e1.encode_device(d[0], w, h, I420, quality=90)
        e2.encode_device(d[1], w, h, RGB, quality=90, subsampling=420, color_space=CS["Y601full"])
        assert e1.result() == a[0][1] and e2.result() == a[1][1]
    e1.close(), e2.close()


@pytest.mark.gpu
@pytest.mark.parametrize("il", [0, 1])
def test_gpu_420_round_trip_through_the_decoder(pl, orc, il):
    """decode each 4:2:0 stream to I420 with the project's decoder: equal to the CPU decode oracle, and close to the source"""
    from test_jpeg_decode import orc_decode
    from ultragrid_b200 import api
    w, h = 1920, 1080
    rgb = np.ascontiguousarray(natural_rgb(w, h, 12))
    s = oracle_stream(pl, rgb.reshape(-1), w, h, RGB, 420, "Y709", 90, 0, il)
    enc = _enc()
    assert _gpu_stream(enc, rgb.reshape(-1), w, h, RGB, 420, "Y709", 90, 0, il) == s
    dec = api.JpegDecoder()
    got = dec.decode(s, I420)
    _, uyvy = orc_decode(orc, s, 0, w, h)  # the oracle's native output (UYVY); I420 output = uyvy_to_i420 of it, as the decoder documents
    cw, ch = (w + 1) // 2, (h + 1) // 2
    want = [np.zeros(w * h, np.uint8), np.zeros(cw * ch, np.uint8), np.zeros(cw * ch, np.uint8)]
    orc_uyvy_to_i420(orc, uyvy, w, h, want)
    assert np.array_equal(got, np.concatenate(want))
    y_src = prep(pl, rgb.reshape(-1), w, h, RGB, 420, "Y709")[0]
    assert psnr(got[:w * h].reshape(h, w), y_src.reshape(h, w)) > 35
    also = orc_uyvy_to_i420  # the same for the UYVY -> 4:2:0 stream
    uyvy_src = source(orc, UYVY, w, h, 12)
    s2 = oracle_stream(pl, uyvy_src, w, h, UYVY, 420, "native", 90, 0, 1)
    _, u2 = orc_decode(orc, s2, 0, w, h)
    want2 = [np.zeros(w * h, np.uint8), np.zeros(cw * ch, np.uint8), np.zeros(cw * ch, np.uint8)]
    also(orc, u2, w, h, want2)
    assert np.array_equal(dec.decode(s2, I420), np.concatenate(want2))
    enc.close(), dec.close()


@pytest.mark.gpu
def test_gpujpeg_module_takes_i420(pl, orc):
    """I420 frames go straight into the encoder (gpujpeg.cpp:262-266, :332), host and device memory; subsampling=422 on I420 drops the frame"""
    import torch
    from ultragrid_b200 import compress
    w, h = 320, 184
    src = source(orc, I420, w, h, 8)
    want = oracle_stream(pl, src, w, h, I420, 0, "native", 90, 0, 1)
    c = compress.Compress("GPUJPEG:q=90")
    c.push(src, w, h, I420)
    got, _, _ = c.pop(w * h * 3 + 4096)
    assert got.tobytes() == want
    c.push(torch.from_numpy(src).cuda(), w, h, I420)
    got, _, _ = c.pop(w * h * 3 + 4096)
    assert got.tobytes() == want
    c.close()
    c = compress.Compress("GPUJPEG:q=90:Y709:subsampling=420:lanes=1")
    c.push(src, w, h, I420)
    got, _, _ = c.pop(w * h * 3 + 4096)
    assert got.tobytes() == want
    c.close()
    for cfg in ("GPUJPEG:subsampling=422:lanes=1", "GPUJPEG:Y601:lanes=1"):
        c = compress.Compress(cfg)
        c.push(src, w, h, I420)
        c.push(None, 0, 0, 0)
        assert c.pop(w * h * 3 + 4096) is None
        c.close()
