"""JPEG with alpha: RGBA input with subsampling 4444 (the GPUJPEG module's `alpha` option, gpujpeg.cpp:227-236,316-328,335) -> a four-component
stream R G B A, and its decode back to RGBA (src/video_decompress/gpujpeg.c:122-129,254-260).
GPUJPEG's own table choice for the alpha component is unpinned (the library is absent); the stream is pinned instead:
  * CPU: the restatement tests/jpeg_alpha_oracle.c against the existing RGB oracle exactly (scans 1-3 = the RGB stream's scans, scan 4 = the
    third scan of the RGB stream of (R, G, A)), its headers, libjpeg (PIL) decoding it and the host-only image info;
  * GPU: the product's stream == the oracle byte for byte, the decompress module's probe, the decoder == the oracle's four-component decode, the modules end to end."""
import ctypes
import io
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
from PIL import Image

import util
from test_jpeg import RGB, UYVY, natural_rgb, orc_encode, psnr

RGBA, I420, JPEG, NONE = 1, 29, 13, 0
_vp, _i, _l, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_size_t
HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [(1, 1), (17, 9), (130, 37), (640, 360)]
RIS = [0, 1, 3, 7]
QS = [1, 90, 100]


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


@pytest.fixture(scope="module")
def al():
    """the alpha oracle, compiled on its own (it includes oracle/jpeg_oracle.c and oracle/jpeg_decode_oracle.c)"""
    d = tempfile.mkdtemp(prefix="ugb_alpha_oracle_")
    path = os.path.join(d, "libjpegalpha.so")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fvisibility=hidden", "-o", path,
                    os.path.join(HERE, "jpeg_alpha_oracle.c"), "-lm"], check=True, capture_output=True)
    L = ctypes.CDLL(path)
    L.orc_jpeg_encode_rgba.argtypes = [_vp, _l, _i, _i, _i, _i, _i, _vp, _sz]
    L.orc_jpeg_encode_rgba.restype = _sz
    L.orc_jpeg_decode_rgba.argtypes = [_vp, _sz, _vp, _l, _vp]
    return L


def rgba_frame(w, h, seed=1):
    """the natural frame of test_jpeg with a natural alpha plane: a soft-edged elliptic key whose edge wanders with a seeded wave"""
    rgb = natural_rgb(w, h, seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    rng = np.random.default_rng(seed + 100)
    ph, amp = rng.uniform(0, 2 * np.pi), rng.uniform(0.02, 0.08)
    r = np.hypot((xx - w * 0.5) / max(w * 0.35, 1), (yy - h * 0.5) / max(h * 0.35, 1)) + amp * np.sin(6 * np.arctan2(yy - h * 0.5, xx - w * 0.5) + ph)
    a = np.clip((1.15 - r) / 0.3, 0, 1) * 255
    return np.ascontiguousarray(np.dstack([rgb, a.round().astype(np.uint8)]))


def oracle_stream(al, src, w, h, q, ri=0, il=0, pitch=0):
    src = np.ascontiguousarray(src).reshape(-1)
    out = np.zeros(((w + 7) // 8) * ((h + 7) // 8) * 4 * 418 + 4096, np.uint8)
    n = al.orc_jpeg_encode_rgba(src.ctypes.data, pitch or w * 4, w, h, q, ri, il, out.ctypes.data, out.size)
    assert n > 0
    return out[:n].tobytes()


def oracle_decode(al, stream, w, h):
    out = np.zeros(w * h * 4, np.uint8)
    b = np.frombuffer(stream, np.uint8)
    info = (_i * 2)()
    assert al.orc_jpeg_decode_rgba(b.ctypes.data, len(stream), out.ctypes.data, w * 4, info) == 0
    assert tuple(info) == (w, h)
    return out.reshape(h, w, 4)


def scans(stream):
    """entropy-coded data of every scan (from behind its SOS header to the marker that ends it; RSTn stay in)"""
    out, p = [], 2
    while p + 4 <= len(stream):
        mk, L = stream[p + 1], stream[p + 2] << 8 | stream[p + 3]
        if mk == 0xD9:
            break
        if mk != 0xDA:
            p += 2 + L
            continue
        b = e = p + 2 + L
        while not (stream[e] == 0xFF and stream[e + 1] not in (0,) and not 0xD0 <= stream[e + 1] <= 0xD7):
            e += 1
        out.append(stream[b:e])
        p = e
    return out


def segment(stream, marker):
    p = 2
    while p + 4 <= len(stream):
        mk, L = stream[p + 1], stream[p + 2] << 8 | stream[p + 3]
        if mk == marker:
            return p
        if mk == 0xDA:
            return -1
        p += 2 + L
    return -1


# ---- CPU ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("ri", RIS)
@pytest.mark.parametrize("q", QS)
def test_oracle_four_scans_are_the_rgb_oracles_scans(al, orc, w, h, ri, q):
    """scans 1-3 = orc_encode of the frame's RGB bytes; scan 4 = the third scan of orc_encode of (R, G, A)"""
    f = rgba_frame(w, h, w + h + q)
    s = scans(oracle_stream(al, f, w, h, q, ri))
    assert len(s) == 4
    rgb = scans(orc_encode(orc, np.ascontiguousarray(f[..., :3]).reshape(-1), w, h, RGB, q, ri))
    rga = scans(orc_encode(orc, np.ascontiguousarray(f[..., [0, 1, 3]]).reshape(-1), w, h, RGB, q, ri))
    assert s[:3] == rgb
    assert s[3] == rga[2]


@pytest.mark.parametrize("il,ri", [(0, 0), (1, 0), (0, 5), (1, 3)])
def test_oracle_headers(al, il, ri):
    w, h = 130, 37
    s = oracle_stream(al, rgba_frame(w, h), w, h, 90, ri, il)
    a = segment(s, 0xEE)
    assert a > 0 and s[a + 4:a + 9] == b"Adobe" and s[a + 15] == 0  # transform 0: stored as is
    f = segment(s, 0xC0)
    assert s[f + 2:f + 4] == bytes([0, 20]) and s[f + 4] == 8 and s[f + 9] == 4
    assert s[f + 10:f + 22] == bytes([1, 0x11, 0, 2, 0x11, 1, 3, 0x11, 1, 4, 0x11, 1])
    d = segment(s, 0xDD)
    assert d > 0 and (s[d + 4] << 8 | s[d + 5]) == (ri or 8)
    assert len(scans(s)) == (1 if il else 4)
    sos = s.index(b"\xff\xda")
    assert s[sos + 4] == (4 if il else 1)
    if il:
        assert s[sos + 5:sos + 13] == bytes([1, 0x00, 2, 0x11, 3, 0x11, 4, 0x11])


@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("w,h,q", [(17, 9, 90), (130, 37, 75), (640, 360, 95)])
def test_libjpeg_decodes_the_stream(al, il, w, h, q):
    """PIL opens a four-component Adobe JPEG as CMYK and inverts it ("CMYK;I"): 255 - PIL is the stored R G B A, within 1 of the oracle's float IDCT"""
    f = rgba_frame(w, h, 3)
    s = oracle_stream(al, f, w, h, q, 0, il)
    im = Image.open(io.BytesIO(s))
    assert im.mode == "CMYK" and im.size == (w, h)
    lib = 255 - np.asarray(im).astype(np.int32)
    ours = oracle_decode(al, s, w, h).astype(np.int32)
    assert np.abs(lib - ours).max() <= 1
    assert psnr(ours[..., 3], f[..., 3]) > 30


def _info(s):
    from ultragrid_b200 import _lib
    lib = _lib.load()

    class Info(ctypes.Structure):
        _fields_ = [(n, ctypes.c_int) for n in ("width", "height", "components", "h_samp", "v_samp", "adobe", "ri", "native")]
    info = Info()
    rc = lib.ugb200_jpeg_get_image_info((ctypes.c_uint8 * len(s)).from_buffer_copy(s), len(s), ctypes.byref(info))
    return rc, info


@pytest.mark.parametrize("il", [0, 1])
def test_image_info_and_refused_four_component_streams(al, il):
    w, h = 130, 37
    s = oracle_stream(al, rgba_frame(w, h), w, h, 90, 0, il)
    rc, info = _info(s)
    assert rc == 0 and (info.width, info.height, info.components, info.h_samp, info.v_samp, info.adobe, info.ri) == (w, h, 4, 1, 1, 0, 8)
    assert info.native == RGBA
    ycck = bytearray(s)
    ycck[segment(s, 0xEE) + 15] = 2  # Adobe transform 2: YCCK
    assert _info(bytes(ycck))[0] == -4
    sub = bytearray(s)
    sub[segment(s, 0xC0) + 11] = 0x22  # component 0 sampled 2x2
    assert _info(bytes(sub))[0] == -4
    no_adobe = s[:segment(s, 0xEE)] + s[segment(s, 0xEE) + 16:]  # no Adobe marker: samples as stored
    rc, info = _info(no_adobe)
    assert rc == 0 and info.native == RGBA and info.adobe == -1


@pytest.mark.gpu
def test_decompress_module_probe_reports_4444(al):
    """the module's init selects a CUDA device, so this runs where there is one; the probe itself reads the headers on the host"""
    from ultragrid_b200.compress import Decompress
    w, h = 64, 48
    s = oracle_stream(al, rgba_frame(w, h), w, h, 90)
    probe = Decompress(JPEG, NONE)
    assert probe.module == "gpujpeg"
    probe.reconfigure(w, h, JPEG, NONE)
    st, _, props = probe.frame(s)
    assert st == Decompress.GOT_CODEC and props == [8, 4444, 1]
    probe.close()


# ---- GPU ------------------------------------------------------------------------------------------------------------------
def _enc(stream=None):
    from ultragrid_b200 import api
    return api.JpegEncoder(stream)


def _gpu(enc, src, w, h, q, ri=0, il=0, pitch=0, device=True):
    import torch
    if device:
        enc.encode_device(torch.from_numpy(np.ascontiguousarray(src).reshape(-1)).cuda(), w, h, RGBA, quality=q, restart_interval=ri, pitch=pitch,
                          interleaved=bool(il), subsampling=4444)
        return enc.result()
    return enc.encode(np.ascontiguousarray(src).reshape(-1), w, h, RGBA, quality=q, restart_interval=ri, pitch=pitch, interleaved=bool(il), subsampling=4444)


@pytest.mark.gpu
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("q", QS)
def test_gpu_rgba_equals_oracle_bytes(al, il, q):
    enc = _enc()
    for w, h in SIZES:
        f = rgba_frame(w, h, w + q)
        for ri in RIS:
            want = oracle_stream(al, f, w, h, q, ri, il)
            assert _gpu(enc, f, w, h, q, ri, il) == want, (w, h, ri)
        assert _gpu(enc, f, w, h, q, 0, il, device=False) == oracle_stream(al, f, w, h, q, 0, il), (w, h, "host")
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)])
def test_gpu_rgba_large_frames_equal_oracle_bytes(al, il, w, h):
    enc = _enc()
    f = rgba_frame(w, h, 4)
    for q, ri in ((90, 0), (100, 3)):
        assert _gpu(enc, f, w, h, q, ri, il) == oracle_stream(al, f, w, h, q, ri, il), (q, ri)
    assert _gpu(enc, f, w, h, 90, 0, il, device=False) == oracle_stream(al, f, w, h, 90, 0, il)
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("il", [0, 1])
def test_gpu_rgba_padded_pitch_and_8_byte_aligned_source(al, il):
    import torch
    enc = _enc()
    for w, h in ((130, 37), (640, 360), (1920, 1080)):
        f = rgba_frame(w, h, 9)
        want = oracle_stream(al, f, w, h, 90, 0, il)
        pitch = w * 4 + 40
        padded = np.full((h, pitch), 0xA5, np.uint8)
        padded[:, :w * 4] = f.reshape(h, -1)
        assert _gpu(enc, padded, w, h, 90, 0, il, pitch=pitch) == want, ("pitch", w, h)
        assert _gpu(enc, padded, w, h, 90, 0, il, pitch=pitch, device=False) == want, ("host pitch", w, h)
        buf = torch.zeros(w * h * 4 + 64, dtype=torch.uint8, device="cuda")  # 8 bytes past a 256-byte aligned allocation
        buf[8:8 + w * h * 4] = torch.from_numpy(f.reshape(-1)).cuda()
        enc.encode_device(buf[8:], w, h, RGBA, quality=90, interleaved=bool(il), subsampling=4444)
        assert enc.result() == want, ("aligned 8", w, h)
    enc.close()


@pytest.mark.gpu
def test_gpu_rgba_refusals():
    import torch
    from ultragrid_b200 import api, _lib
    L = _lib.load()
    enc = _enc()
    t = torch.zeros(64 * 64 * 4, dtype=torch.uint8, device="cuda")
    assert L.ugb200_jpeg_encode_device(enc._h, t.data_ptr(), 0, 64, 64, RGBA, ctypes.byref(api.JpegParams(75, 0, 0))) == -4  # plain call: no RGBA
    for codec, sub, cs in ((RGBA, 0, 0), (RGBA, 444, 0), (RGBA, 4444, 3), (RGBA, 420, 0), (RGB, 4444, 0), (UYVY, 4444, 0), (I420, 4444, 0), (RGBA, 4444, 1)):
        px = api.JpegParamsEx()
        L.ugb200_jpeg_default_params_ex(ctypes.byref(px))
        px.subsampling, px.color_space = sub, cs
        assert L.ugb200_jpeg_encode_device_ex(enc._h, t.data_ptr(), 0, 64, 64, codec, ctypes.byref(px)) == -4, (codec, sub, cs)
    for cs in (0, 4):  # native and RGB are accepted
        px = api.JpegParamsEx()
        L.ugb200_jpeg_default_params_ex(ctypes.byref(px))
        px.subsampling, px.color_space = 4444, cs
        assert L.ugb200_jpeg_encode_device_ex(enc._h, t.data_ptr(), 0, 64, 64, RGBA, ctypes.byref(px)) == 0
        enc.result()
    enc.close()


@pytest.mark.gpu
def test_gpu_one_encoder_alternating_rgb_rgba_uyvy(al, orc):
    """the configure() cache key tells RGB and RGBA apart: no stale header or geometry"""
    w, h = 320, 184
    f = rgba_frame(w, h, 21)
    rgb = np.ascontiguousarray(f[..., :3]).reshape(-1)
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, rgb, w, h)
    want = [orc_encode(orc, rgb, w, h, RGB, 90), oracle_stream(al, f, w, h, 90), orc_encode(orc, uyvy, w, h, UYVY, 90), oracle_stream(al, f, w, h, 90, 0, 1)]
    enc = _enc()
    import torch
    for _ in range(3):
        enc.encode_device(torch.from_numpy(rgb).cuda(), w, h, RGB, quality=90)
        assert enc.result() == want[0]
        assert _gpu(enc, f, w, h, 90) == want[1]
        enc.encode_device(torch.from_numpy(uyvy).cuda(), w, h, UYVY, quality=90)
        assert enc.result() == want[2]
        assert _gpu(enc, f, w, h, 90, il=1) == want[3]
    enc.close()


@pytest.mark.gpu
def test_gpu_two_encoders_on_two_streams(al, orc):
    import torch
    w, h = 1920, 1080
    f1, f2 = rgba_frame(w, h, 31), rgba_frame(w, h, 32)
    w1, w2 = oracle_stream(al, f1, w, h, 90), oracle_stream(al, f2, w, h, 75, 0, 1)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    e1, e2 = _enc(s1), _enc(s2)
    d1, d2 = torch.from_numpy(f1.reshape(-1)).cuda(), torch.from_numpy(f2.reshape(-1)).cuda()
    torch.cuda.synchronize()
    for _ in range(3):
        e1.encode_device(d1, w, h, RGBA, quality=90, subsampling=4444)
        e2.encode_device(d2, w, h, RGBA, quality=75, interleaved=True, subsampling=4444)
        assert e1.result() == w1 and e2.result() == w2
    e1.close(), e2.close()


@pytest.mark.gpu
@pytest.mark.parametrize("knob,value", [("UGB200_JPEG_SPLIT", "1"), ("UGB200_JPEG_SINGLE_PASS", "1"), ("UGB200_JPEG_CAP", "12")])
def test_gpu_alternative_routes_give_the_same_bytes(knob, value):
    """process-wide switches: the byte-exactness tests once more in a child process (the split path takes every RGBA stream there)"""
    env = dict(os.environ, **{knob: value})
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-q", "-x", "-k",
                        "equals_oracle_bytes or padded_pitch"], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:]


@pytest.mark.gpu
@pytest.mark.parametrize("il", [0, 1])
def test_gpu_decoder_equals_oracle(al, orc, il):
    import torch
    from ultragrid_b200 import api
    dec = api.JpegDecoder()
    for w, h in SIZES + [(7680, 4320)]:
        f = rgba_frame(w, h, 50 + w)
        s = oracle_stream(al, f, w, h, 90, 0, il)
        want = oracle_decode(al, s, w, h)
        assert np.array_equal(dec.decode(s, RGBA).reshape(h, w, 4), want), (w, h, "host")
        got = dec.decode(s, RGBA, device=True)
        torch.cuda.synchronize()
        assert np.array_equal(got.cpu().numpy().reshape(h, w, 4), want), (w, h, "device")
        if w * h > 1920 * 1080:
            continue
        pitch = w * 4 + 36
        got = dec.decode(s, RGBA, pitch=pitch).reshape(h, pitch)
        assert np.array_equal(got[:, :w * 4].reshape(h, w, 4), want), (w, h, "pitch")
        got = dec.decode(s, RGBA, pitch=pitch, device=True)
        torch.cuda.synchronize()
        assert np.array_equal(got.cpu().numpy().reshape(h, pitch)[:, :w * 4].reshape(h, w, 4), want), (w, h, "device pitch")
        for shifts in ((16, 8, 0), (8, 16, 24), (24, 16, 8)):  # vc_copylineRGBA of the (0, 8, 16) result: alpha becomes 0xFF
            conv = util.convert_cpu(orc, "orc_convert", RGBA, RGBA, want.reshape(-1), w, h, shifts=shifts)
            assert np.array_equal(dec.decode(s, RGBA, shifts=shifts), conv), (w, h, shifts)
            assert np.array_equal(dec.decode(s, RGBA, shifts=shifts, device=True).cpu().numpy().reshape(-1), conv), (w, h, shifts, "device")
        assert np.array_equal(dec.decode(s, RGB).reshape(h, w, 3), want[..., :3]), (w, h, "RGB")
        rgb_stream = orc_encode(orc, np.ascontiguousarray(f[..., :3]).reshape(-1), w, h, RGB, 90)  # the same R G B samples once decoded
        for out_c in (UYVY, I420):
            assert np.array_equal(dec.decode(s, out_c), dec.decode(rgb_stream, out_c)), (w, h, out_c)
    from ultragrid_b200 import _lib
    L = _lib.load()
    s = oracle_stream(al, rgba_frame(64, 48), 64, 48, 90, 0, il)
    assert L.ugb200_jpeg_decoder_expect(dec._h, 64, 40) == 0
    out = np.zeros(64 * 48 * 4, np.uint8)
    assert L.ugb200_jpeg_decode(dec._h, s, len(s), out.ctypes.data, 0, 0, RGBA, 0, 8, 16) == -3  # another size: refused
    assert L.ugb200_jpeg_decoder_expect(dec._h, 64, 48) == 0
    assert L.ugb200_jpeg_decode(dec._h, s, len(s), out.ctypes.data, 0, 0, RGBA, 0, 8, 16) == 0
    dec.close()


def _pop_all(c, n, cap):
    out = []
    for _ in range(n):
        r = c.pop(cap)
        out.append(None if r is None else r[0].tobytes())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 3])
def test_gpujpeg_module_alpha(al, orc, lanes):
    """`alpha` with RGBA frames from host and device memory: the four-component stream, in order"""
    import torch
    from ultragrid_b200 import compress
    w, h = 320, 184
    frames = [rgba_frame(w, h, 60 + k) for k in range(4)]
    want = [oracle_stream(al, f, w, h, 90) for f in frames]
    c = compress.Compress(f"GPUJPEG:q=90:alpha:lanes={lanes}")
    for k, f in enumerate(frames):
        c.push(f.reshape(-1) if k % 2 == 0 else torch.from_numpy(f.reshape(-1)).cuda(), w, h, RGBA)
    assert _pop_all(c, 4, w * h * 3 + 4096) == want
    c.close()


@pytest.mark.gpu
def test_gpujpeg_module_alpha_with_other_inputs_and_refusals(al, orc):
    from ultragrid_b200 import compress
    w, h = 320, 184
    f = rgba_frame(w, h, 70)
    rgb = np.ascontiguousarray(f[..., :3]).reshape(-1)
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, rgb, w, h)
    for cfg in ("GPUJPEG:q=90:lanes=1", "GPUJPEG:q=90:alpha:lanes=1"):  # UYVY: `alpha` changes nothing
        c = compress.Compress(cfg)
        c.push(uyvy, w, h, UYVY)
        assert c.pop(w * h * 3 + 4096)[0].tobytes() == orc_encode(orc, uyvy, w, h, UYVY, 90), cfg
        c.close()
    # RGBA without `alpha`: the line converter to RGB, then the RGB stream (the route of the parent version)
    c = compress.Compress("GPUJPEG:q=90:lanes=1")
    c.push(f.reshape(-1), w, h, RGBA)
    conv = util.convert_cpu(orc, "orc_convert", RGBA, RGB, f.reshape(-1), w, h)
    assert c.pop(w * h * 3 + 4096)[0].tobytes() == orc_encode(orc, conv, w, h, RGB, 90)
    c.close()
    c = compress.Compress("GPUJPEG:q=90:alpha:RGB:subsampling=444:lanes=1")  # the input's own options are accepted
    c.push(f.reshape(-1), w, h, RGBA)
    assert c.pop(w * h * 3 + 4096)[0].tobytes() == oracle_stream(al, f, w, h, 90)
    c.close()
    for cfg in ("GPUJPEG:alpha:Y709:lanes=1", "GPUJPEG:alpha:subsampling=420:lanes=1"):
        c = compress.Compress(cfg)
        c.push(f.reshape(-1), w, h, RGBA)
        c.push(None, 0, 0, 0)
        assert c.pop(w * h * 3 + 4096) is None, cfg
        c.close()


ALPHA_PSNR_DB = 30  # q = 90 on the soft-edged key: the alpha plane comes back well above this


@pytest.mark.gpu
def test_round_trip_through_the_modules(al):
    from ultragrid_b200 import compress
    from ultragrid_b200.compress import Decompress
    w, h = 640, 360
    f = rgba_frame(w, h, 80)
    c = compress.Compress("GPUJPEG:q=90:alpha:lanes=1")
    c.push(f.reshape(-1), w, h, RGBA)
    s = c.pop(w * h * 3 + 4096)[0].tobytes()
    c.close()
    d = Decompress(JPEG, RGBA)
    assert d.module == "gpujpeg"
    d.reconfigure(w, h, JPEG, RGBA)
    st, out, _ = d.frame(s)
    assert st == Decompress.GOT_FRAME
    got = out.reshape(h, w, 4)
    assert np.array_equal(got, oracle_decode(al, s, w, h))
    assert psnr(got[..., 3], f[..., 3]) > ALPHA_PSNR_DB
    d.close()


@pytest.mark.gpu
def test_alpha_through_the_reference_framework(al):
    """the real-ABI compress and decompress modules inside the reference's unmodified framework (tests/test_real_module.py): an RGBA frame with
    `alpha` gives the four-component stream; the decompress module probes it as 4:4:4:4 RGB and decodes it to RGBA with the alpha kept"""
    from test_real_module import dec_frame, framework, pop
    fw = framework()
    w, h = 640, 360
    f = rgba_frame(w, h, 90)
    want = oracle_stream(al, f, w, h, 90)
    st = fw.fwd_init(b"gpujpeg:q=90:alpha:lanes=1")
    assert st
    src = np.ascontiguousarray(f.reshape(-1))
    fw.fwd_frame(st, src.ctypes.data, 0, w, h, RGBA, 60.0)
    fw.fwd_frame(st, None, 0, 0, 0, 0, 0.0)
    got, codec, seq, ow, oh = pop(fw, st, w * h * 3 + 4096)
    assert codec == JPEG and (ow, oh) == (w, h) and got.tobytes() == want
    assert pop(fw, st, 16) is None
    fw.fwd_done(st)
    probe = fw.fwd_dec_init(JPEG, 0)
    assert probe and fw.fwd_dec_reconfigure(probe, w, h, JPEG, 0, 8, 16, 0, 0)
    rc, _, props = dec_frame(fw, probe, want, 0)
    assert rc == 2 and props == [8, 4444, 1]
    fw.fwd_dec_done(probe)
    d = fw.fwd_dec_init(JPEG, RGBA)
    assert d and fw.fwd_dec_reconfigure(d, w, h, JPEG, 0, 8, 16, w * 4, RGBA)
    rc, out, _ = dec_frame(fw, d, want, w * h * 4)
    assert rc == 1 and np.array_equal(out.reshape(h, w, 4), oracle_decode(al, want, w, h))
    fw.fwd_dec_done(d)
