"""JPEG stage.  CPU part pins the oracle (oracle/jpeg_oracle.c) with an INDEPENDENT decoder (libjpeg through PIL):
valid baseline stream, PSNR equal to libjpeg's own encoder at the same quality/tables, the reference's flat-grey
round-trip criterion (test/gpujpeg_test.cpp:68-106).  GPU part: the CUDA encoder emits the oracle's bytes exactly."""
import ctypes
import io
import os

import numpy as np
import pytest

import util

PIL = pytest.importorskip("PIL.Image")
UYVY, RGB = 2, 12


def orc_encode(orc, src, w, h, codec, quality, ri=0, pitch=0):
    orc.orc_jpeg_encode.restype = ctypes.c_size_t
    orc.orc_jpeg_encode.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_void_p, ctypes.c_size_t]
    out = np.zeros(((w + 15) // 16 * 16) * ((h + 7) // 8 * 8) * 3 // 64 * 418 + 4096, dtype=np.uint8)  # worst case, see orc_jpeg_encode
    pitch = pitch or w * (2 if codec == UYVY else 3)
    n = orc.orc_jpeg_encode(src.ctypes.data, pitch, w, h, 0 if codec == UYVY else 1, quality, ri, out.ctypes.data, out.size)
    assert n > 0
    return out[:n].tobytes()


def orc_encode_interleaved_rgb(orc, src, w, h, quality, ri=0):
    """RGB stored as one interleaved scan (the `interleaved` option of the GPUJPEG module, gpujpeg.cpp:303,397-398)"""
    orc.orc_jpeg_encode_ex.restype = ctypes.c_size_t
    orc.orc_jpeg_encode_ex.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_void_p, ctypes.c_size_t]
    out = np.zeros(((w + 15) // 16 * 16) * ((h + 7) // 8 * 8) * 3 // 64 * 418 + 4096, dtype=np.uint8)
    n = orc.orc_jpeg_encode_ex(src.ctypes.data, w * 3, w, h, 1, quality, ri, 1, out.ctypes.data, out.size)
    assert n > 0
    return out[:n].tobytes()


def orc_encode_parallel(orc, src, w, h, codec, quality, ri=0, pitch=0):
    """the all-threads CPU port (bench.py's cpu_baseline for the JPEG workloads)"""
    orc.orc_jpeg_encode_parallel.restype = ctypes.c_size_t
    orc.orc_jpeg_encode_parallel.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_void_p, ctypes.c_size_t]
    out = np.zeros(((w + 15) // 16 * 16) * ((h + 7) // 8 * 8) * 3 // 64 * 418 + 4096, dtype=np.uint8)
    pitch = pitch or w * (2 if codec == UYVY else 3)
    n = orc.orc_jpeg_encode_parallel(src.ctypes.data, pitch, w, h, 0 if codec == UYVY else 1, quality, ri, out.ctypes.data, out.size)
    assert n > 0
    return out[:n].tobytes()


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else 10 * np.log10(255 ** 2 / mse)


def natural_rgb(w, h, seed=1):
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) % 256], axis=2).astype(np.int32)
    img += np.random.default_rng(seed).integers(-6, 7, img.shape)
    return img.clip(0, 255).astype(np.uint8)


def decode_ycc(data, w, h):
    im = PIL.open(io.BytesIO(data))
    im.draft("YCbCr", (w, h))
    im.load()
    assert im.mode == "YCbCr" and im.size == (w, h)
    return np.asarray(im)


def uyvy_planes(uyvy, w, h):
    u = uyvy.reshape(h, w // 2, 4)
    return np.stack([u[:, :, 1], u[:, :, 3]], axis=2).reshape(h, w), u[:, :, 0], u[:, :, 2]


@pytest.mark.parametrize("q", [50, 75, 90])
def test_oracle_uyvy_stream_decodes_and_matches_libjpeg_psnr(orc, q):
    w, h = 640, 360
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, natural_rgb(w, h).reshape(-1), w, h)
    Y, Cb, Cr = uyvy_planes(uyvy, w, h)
    dec = decode_ycc(orc_encode(orc, uyvy, w, h, UYVY, q), w, h)
    full = np.stack([Y, np.repeat(Cb, 2, axis=1), np.repeat(Cr, 2, axis=1)], axis=2)
    b = io.BytesIO()
    PIL.fromarray(full, mode="YCbCr").save(b, format="JPEG", quality=q, subsampling="4:2:2")
    lib = decode_ycc(b.getvalue(), w, h)
    for name, mine, theirs, want in (("Y", dec[:, :, 0], lib[:, :, 0], Y), ("Cb", dec[:, ::2, 1], lib[:, ::2, 1], Cb)):
        assert abs(psnr(mine, want) - psnr(theirs, want)) < 0.3, (name, psnr(mine, want), psnr(theirs, want))
    assert psnr(dec[:, :, 0], Y) > 34


@pytest.mark.parametrize("w,h", [(16, 8), (48, 24), (100, 52), (130, 37), (1920, 1080)])
def test_oracle_rgb_stream_is_rgb_and_close(orc, w, h):
    rgb = natural_rgb(w, h, 3)
    data = orc_encode(orc, rgb.reshape(-1), w, h, RGB, 90)
    im = PIL.open(io.BytesIO(data))
    im.load()
    assert im.mode == "RGB" and im.size == (w, h)  # Adobe APP14 transform 0: no YCbCr->RGB applied by the decoder
    assert psnr(np.asarray(im), rgb) > 33


@pytest.mark.parametrize("w,h,ri", [(16, 8, 0), (100, 52, 0), (130, 37, 3), (640, 360, 8)])
def test_oracle_interleaved_rgb_stream(orc, w, h, ri):
    """one scan with three components, 1x1 sampling: an independent decoder reads it as RGB, and it carries the same pixels as the three-scan form"""
    rgb = natural_rgb(w, h, 8)
    a = orc_encode_interleaved_rgb(orc, rgb.reshape(-1), w, h, 90, ri)
    b = orc_encode(orc, rgb.reshape(-1), w, h, RGB, 90, ri)
    assert a.count(b"\xff\xda") == 1 and b.count(b"\xff\xda") >= 3
    ia, ib = PIL.open(io.BytesIO(a)), PIL.open(io.BytesIO(b))
    ia.load(), ib.load()
    assert ia.mode == "RGB" and ia.size == (w, h)
    assert np.array_equal(np.asarray(ia), np.asarray(ib))  # same coefficients, another scan order


def test_flat_grey_roundtrip_like_reference_test(orc):
    """gpujpeg_test_simple (test/gpujpeg_test.cpp:68-106): 1920x1080 RGB all-127, default quality, max |diff| <= 1"""
    w, h = 1920, 1080
    rgb = np.full((h, w, 3), 127, dtype=np.uint8)
    im = PIL.open(io.BytesIO(orc_encode(orc, rgb.reshape(-1), w, h, RGB, 75)))
    im.load()
    assert np.abs(np.asarray(im).astype(int) - 127).max() <= 1


def test_restart_markers_and_header_layout(orc):
    w, h = 64, 32
    uyvy = util.rng_bytes(w * h * 2, 9)
    data = orc_encode(orc, uyvy, w, h, UYVY, 90, ri=2)
    assert data[:2] == b"\xff\xd8" and data[-2:] == b"\xff\xd9"
    assert data.count(b"\xff\xdb") >= 2 and b"\xff\xc0" in data and data.count(b"\xff\xc4") >= 4 and b"\xff\xdd\x00\x04\x00\x02" in data
    nm = (w // 16) * (h // 8)
    body = data[data.index(b"\xff\xda"):]
    rst = sum(body.count(bytes([0xFF, 0xD0 + k])) for k in range(8))
    assert rst == (nm + 1) // 2 - 1
    decode_ycc(data, w, h)


@pytest.mark.parametrize("codec,w,h,q,ri", [(UYVY, 16, 8, 90, 0), (UYVY, 100, 52, 75, 3), (UYVY, 1920, 1080, 90, 0), (RGB, 8, 8, 90, 0), (RGB, 130, 37, 50, 3),
                                            (RGB, 640, 360, 90, 0), (UYVY, 640, 360, 100, 1)])
def test_parallel_cpu_port_equals_serial_oracle(orc, codec, w, h, q, ri):
    """the OpenMP form that bench.py times as the CPU baseline is the same encoder: identical bytes for any thread count"""
    src = util.rng_bytes(w * h * (2 if codec == UYVY else 3), 31)
    src[len(src) // 3:] = 128  # part noise, part flat
    want = orc_encode(orc, src, w, h, codec, q, ri)
    for threads in (1, 3, 0):
        orc.orc_set_threads(threads)
        assert orc_encode_parallel(orc, src, w, h, codec, q, ri) == want, threads
    orc.orc_set_threads(0)


def dqt_tables(data):
    """{table id: 64 values in natural order} from the DQT segments of a stream"""
    zig = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43,
           36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]
    out, i = {}, 2
    while i + 4 <= len(data) and data[i] == 0xFF and data[i + 1] != 0xDA:
        L = data[i + 2] << 8 | data[i + 3]
        if data[i + 1] == 0xDB:
            d = data[i + 4:i + 2 + L]
            while len(d) >= 65:
                t = [0] * 64
                for k in range(64):
                    t[zig[k]] = d[1 + k]
                out[d[0] & 15] = t
                d = d[65:]
        i += 2 + L
    return out


@pytest.mark.parametrize("q", [1, 25, 50, 75, 90, 95, 100])
def test_quant_tables_equal_libjpegs_entry_by_entry(orc, q):
    """Annex K.1 / K.2 scaled by the IJG quality rule: both tables of the UYVY stream and both tables of the RGB stream (component 0 -> table 0 =
    K.1, components 1, 2 -> table 1 = K.2, the assignment DESIGN.md section 2 states) equal the tables libjpeg itself writes at that quality"""
    w, h = 32, 16
    b = io.BytesIO()
    PIL.fromarray(natural_rgb(w, h), mode="RGB").save(b, format="JPEG", quality=q, subsampling="4:2:2")
    theirs = dqt_tables(b.getvalue())
    assert set(theirs) == {0, 1}
    uy = orc_encode(orc, util.rng_bytes(w * h * 2, 1), w, h, UYVY, q)
    rgb = orc_encode(orc, util.rng_bytes(w * h * 3, 1), w, h, RGB, q)
    for mine in (dqt_tables(uy), dqt_tables(rgb)):
        assert mine[0] == theirs[0] and mine[1] == theirs[1]
    # SOF0 of the RGB stream: three components, 1x1 sampling each, quantiser tables 0, 1, 1
    i = rgb.index(b"\xff\xc0")
    assert rgb[i + 9] == 3 and [rgb[i + 10 + 3 * c + 2] for c in range(3)] == [0, 1, 1] and [rgb[i + 10 + 3 * c + 1] for c in range(3)] == [0x11] * 3


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("codec,w,h,q,ri", [(UYVY, 16, 8, 90, 0), (UYVY, 64, 32, 75, 2), (UYVY, 100, 52, 90, 0), (UYVY, 1920, 1080, 90, 0),
                                            (UYVY, 3840, 2160, 90, 0), (RGB, 8, 8, 90, 0), (RGB, 130, 37, 50, 3), (RGB, 1920, 1080, 90, 0),
                                            (UYVY, 100, 52, 90, 5), (UYVY, 1920, 1080, 75, 8), (UYVY, 640, 360, 90, 1), (RGB, 200, 120, 90, 32),
                                            (RGB, 64, 64, 100, 4), (UYVY, 48, 24, 100, 16)])
def test_gpu_encoder_equals_oracle_bytes(orc, codec, w, h, q, ri):
    import torch
    from ultragrid_b200 import api
    if codec == UYVY:
        src = util.convert_cpu(orc, "orc_convert", RGB, UYVY, natural_rgb(w, h, 5).reshape(-1), w, h)
        src[: w * 2 * min(h, 8)] = util.rng_bytes(w * 2 * min(h, 8), 1)  # a band of noise: long codes, ZRL, 0xFF stuffing
    else:
        src = natural_rgb(w, h, 7).reshape(-1).copy()
        src[: w * 3 * min(h, 8)] = util.rng_bytes(w * 3 * min(h, 8), 2)
    want = orc_encode(orc, src, w, h, codec, q, ri)
    enc = api.JpegEncoder()
    got = enc.encode(src, w, h, codec, quality=q, restart_interval=ri)  # host buffer in, pinned host buffer out
    if got != want:
        fmt = 0 if codec == UYVY else 1
        nblk = ((w + 15) // 16) * ((h + 7) // 8) * 4 if codec == UYVY else ((w + 7) // 8) * ((h + 7) // 8) * 3
        ref = np.zeros(nblk * 64, dtype=np.int16)
        orc.orc_jpeg_coefficients.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        orc.orc_jpeg_coefficients(src.ctypes.data, w * (2 if codec == UYVY else 3), w, h, fmt, q, ref.ctypes.data)
        co = enc.coefficients()
        bad = np.nonzero(co != ref)[0]
        pytest.fail(f"stream differs (len {len(got)} vs {len(want)}); coefficient mismatches: {len(bad)} first {bad[:8].tolist()}")
    # device-resident input path gives the same bytes
    enc.encode_device(torch.from_numpy(src).cuda(), w, h, codec, quality=q, restart_interval=ri)
    assert enc.result() == want
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,q,ri", [(16, 8, 90, 0), (130, 37, 50, 3), (640, 360, 90, 0), (1920, 1080, 90, 8), (200, 120, 100, 1)])
def test_gpu_interleaved_rgb_equals_oracle_bytes(orc, w, h, q, ri):
    import torch
    from ultragrid_b200 import api
    src = natural_rgb(w, h, 21).reshape(-1).copy()
    src[: w * 3 * min(h, 8)] = util.rng_bytes(w * 3 * min(h, 8), 3)
    want = orc_encode_interleaved_rgb(orc, src, w, h, q, ri)
    enc = api.JpegEncoder()
    assert enc.encode(src, w, h, RGB, quality=q, restart_interval=ri, interleaved=True) == want
    enc.encode_device(torch.from_numpy(src).cuda(), w, h, RGB, quality=q, restart_interval=ri, interleaved=True)
    assert enc.result() == want
    assert enc.encode(src, w, h, RGB, quality=q, restart_interval=ri) == orc_encode(orc, src, w, h, RGB, q, ri)  # and back to three scans
    enc.close()


def extreme_ac_frame(codec, w, h):
    """samples +-full scale in the sign pattern of cos((2x+1) 4 pi / 16) in x, y or both: the largest AC coefficients a block can have
    (F(4,4) = F(4,0) = F(0,4) = 1020 in magnitude at quantiser step 1), in every block and every component"""
    sgn = np.array([1, -1, -1, 1, 1, -1, -1, 1])
    yy, xx = np.mgrid[0:h, 0:w]
    kind = ((xx // 8) + (yy // 8)) % 4
    pat = np.where(kind == 0, sgn[xx % 8] * sgn[yy % 8], np.where(kind == 1, sgn[xx % 8], np.where(kind == 2, sgn[yy % 8], -sgn[xx % 8] * sgn[yy % 8])))
    plane = np.where(pat > 0, 255, 0).astype(np.uint8)
    if codec == RGB:
        return np.repeat(plane[:, :, None], 3, axis=2).reshape(-1).copy()
    out = np.empty((h, w, 2), np.uint8)
    out[:, :, 1] = plane                 # luma
    cx = np.where(sgn[(xx // 2) % 8] * sgn[yy % 8] > 0, 255, 0).astype(np.uint8)  # chroma samples sit at every second pixel
    out[:, :, 0] = cx
    return out.reshape(-1).copy()


@pytest.mark.parametrize("codec", [UYVY, RGB])
def test_oracle_largest_ac_coefficients_stay_in_range(orc, codec):
    """the fused kernel does not clamp AC coefficients to the 10-bit categories: the bound is 1020 (jpeg_kernels.cu); the oracle's own
    coefficients of the worst-case frame confirm it at quality 100 (all quantiser steps 1)"""
    w, h = 64, 32
    src = extreme_ac_frame(codec, w, h)
    nblk = (w // 16) * (h // 8) * 4 if codec == UYVY else (w // 8) * (h // 8) * 3
    co = np.zeros(nblk * 64, dtype=np.int16)
    orc.orc_jpeg_coefficients.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    orc.orc_jpeg_coefficients(src.ctypes.data, w * (2 if codec == UYVY else 3), w, h, 0 if codec == UYVY else 1, 100, co.ctypes.data)
    ac = co.reshape(-1, 64)[:, 1:]
    assert 1015 <= np.abs(ac).max() <= 1020, np.abs(ac).max()


@pytest.mark.gpu
@pytest.mark.parametrize("codec", [UYVY, RGB])
def test_gpu_largest_ac_coefficients_equal_oracle_bytes(orc, codec):
    import torch
    from ultragrid_b200 import api
    w, h = 64, 32
    src = extreme_ac_frame(codec, w, h)
    enc = api.JpegEncoder()
    for q in (100, 97):
        enc.encode_device(torch.from_numpy(src).cuda(), w, h, codec, quality=q)
        assert enc.result() == orc_encode(orc, src, w, h, codec, q, 0), q
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("codec,q", [(UYVY, 100), (UYVY, 85), (RGB, 90)])
def test_gpu_noise_takes_serial_route_then_adapts(orc, codec, q):
    """Pure noise overflows the capped per-block bit buffers of the fused kernel: the first frame goes through the serial route of the
    overflowing CTAs, the following ones through a larger cap chosen from the first frame's statistics; calm content shrinks it again."""
    import torch
    from ultragrid_b200 import api
    w, h = 320, 96
    noise = util.rng_bytes(w * h * (2 if codec == UYVY else 3), 9)
    calm = np.full_like(noise, 100)
    enc = api.JpegEncoder()
    for src in (noise, noise, noise, calm, calm, noise):
        want = orc_encode(orc, src, w, h, codec, q, 0)
        enc.encode_device(torch.from_numpy(src).cuda(), w, h, codec, quality=q)
        assert enc.result() == want
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("codec,w,h,pad", [(UYVY, 100, 52, 24), (UYVY, 1920, 64, 64), (RGB, 77, 33, 5), (UYVY, 98, 50, 4)])
def test_gpu_encoder_honours_the_source_pitch(orc, codec, w, h, pad):
    """rows further apart than one line (device and host input): the same stream as from the tight frame"""
    import torch
    from ultragrid_b200 import api
    bpp = 2 if codec == UYVY else 3
    tight = util.rng_bytes(w * bpp * h, 21) if codec == RGB else util.convert_cpu(orc, "orc_convert", RGB, UYVY, natural_rgb(w, h, 9).reshape(-1), w, h)
    row = len(tight) // h
    pitch = row + pad
    padded = np.full(pitch * h, 0xEE, np.uint8)
    padded.reshape(h, pitch)[:, :row] = tight.reshape(h, row)
    want = orc_encode(orc, tight, w, h, codec, 85)
    assert orc_encode(orc, padded, w, h, codec, 85, pitch=pitch) == want
    enc = api.JpegEncoder()
    assert enc.encode(padded, w, h, codec, quality=85, pitch=pitch) == want
    assert enc.encode(torch.from_numpy(padded).cuda(), w, h, codec, quality=85, pitch=pitch) == want
    enc.close()


@pytest.mark.gpu
def test_gpu_two_encoders_with_different_quality_interleaved(orc):
    """no module-level table state: encoders of different quality (and format) share a device, their launches interleave on two streams"""
    import torch
    from ultragrid_b200 import api
    w, h = 640, 360
    uy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, natural_rgb(w, h, 11).reshape(-1), w, h)
    rgb = natural_rgb(w, h, 12).reshape(-1).copy()
    d_uy, d_rgb = torch.from_numpy(uy).cuda(), torch.from_numpy(rgb).cuda()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a, b = api.JpegEncoder(stream=s1), api.JpegEncoder(stream=s2)
    want_a, want_b = orc_encode(orc, uy, w, h, UYVY, 50), orc_encode(orc, rgb, w, h, RGB, 95)
    for _ in range(4):
        a.encode_device(d_uy, w, h, UYVY, quality=50)
        b.encode_device(d_rgb, w, h, RGB, quality=95)
        assert a.result() == want_a
        assert b.result() == want_b
    a.close(), b.close()


@pytest.mark.gpu
def test_gpu_stream_larger_than_output_buffer_is_an_error(orc):
    """RGB noise at quality 100 codes to more than w * h * 3 bytes (the capacity the reference hands libgpujpeg, gpujpeg.cpp:355)"""
    import torch
    from ultragrid_b200 import api
    w, h = 320, 96
    enc = api.JpegEncoder()
    enc.encode_device(torch.from_numpy(util.rng_bytes(w * h * 3, 3)).cuda(), w, h, RGB, quality=100)
    with pytest.raises(RuntimeError):
        enc.result()
    enc.encode_device(torch.from_numpy(np.full(w * h * 3, 90, np.uint8)).cuda(), w, h, RGB, quality=100)  # the encoder stays usable
    assert len(enc.result()) > 600
    enc.close()


@pytest.mark.gpu
def test_gpu_8k_uyvy_jpeg_decodes_with_expected_psnr(orc):
    """config 3 / metric at full size: size-independent checks (valid stream, PSNR on luma vs source)"""
    import torch
    from ultragrid_b200 import api
    w, h = 7680, 4320
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, natural_rgb(w, h, 11).reshape(-1), w, h)
    enc = api.JpegEncoder()
    enc.encode_device(torch.from_numpy(uyvy).cuda(), w, h, UYVY, quality=90)
    data = enc.result()
    PIL.MAX_IMAGE_PIXELS = None
    dec = decode_ycc(data, w, h)
    Y, Cb, _ = uyvy_planes(uyvy, w, h)
    assert psnr(dec[:, :, 0], Y) > 36 and psnr(dec[:, ::2, 1], Cb) > 36
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)])
def test_gpu_rgb_jpeg_config3_sizes(orc, w, h):
    """BASELINE config 3 (RGB -> JPEG q = 90: stored as RGB, three scans, gpujpeg.cpp:303-305) at 4K and at the full 8K size: the stream equals
    the CPU restatement byte for byte, libjpeg decodes it as RGB, and its PSNR is within 0.3 dB of libjpeg's own encoder with the same tables"""
    import torch
    from ultragrid_b200 import api
    PIL.MAX_IMAGE_PIXELS = None
    rgb = natural_rgb(w, h, 13)
    src = rgb.reshape(-1)
    enc = api.JpegEncoder()
    enc.encode_device(torch.from_numpy(src).cuda(), w, h, RGB, quality=90)
    got = enc.result()
    enc.close()
    orc.orc_set_threads(0)
    assert got == orc_encode_parallel(orc, src, w, h, RGB, 90)
    im = PIL.open(io.BytesIO(got))
    im.load()
    assert im.mode == "RGB" and im.size == (w, h)
    mine = psnr(np.asarray(im), rgb)
    b = io.BytesIO()
    # libjpeg's encoder on the same samples with the same colour handling (no transform: the planes go in as if they were YCbCr, 4:4:4)
    PIL.fromarray(rgb, mode="YCbCr").save(b, format="JPEG", quality=90, subsampling="4:4:4")
    lib = PIL.open(io.BytesIO(b.getvalue()))
    lib.draft("YCbCr", (w, h))
    lib.load()
    theirs = psnr(np.asarray(lib), rgb)
    assert abs(mine - theirs) < 0.3, (mine, theirs)
    assert mine > 36


@pytest.mark.gpu
@pytest.mark.parametrize("knob,value", [("UGB200_JPEG_SINGLE_PASS", "1"), ("UGB200_JPEG_SPLIT", "1"), ("UGB200_JPEG_CAP", "12"),
                                        ("UGB200_JPEG_CAP", "8"), ("UGB200_JPEG_CAP", "24")])
def test_gpu_alternative_routes_give_the_same_bytes(knob, value):
    """the single-pass compaction (decoupled look-back), the forced split path and the bit-buffer cap (12 words and fewer = the instantiation
    for seven CTAs per SM, with the input tile reaching into the segment images; 24 = a larger cap) are process-wide switches: the
    byte-exactness tests run once more in a child process with the switch set"""
    import subprocess
    import sys
    env = dict(os.environ, **{knob: value})
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-q", "-x", "-k",
                        "equals_oracle_bytes or serial_route or source_pitch or larger_than_output or largest_ac"], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
