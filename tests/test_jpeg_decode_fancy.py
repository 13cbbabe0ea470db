"""Interpolated chroma (ugb200_jpeg_decoder_set_upsampling(FANCY)): RGB and RGBA output of 4:2:2 and 4:2:0 streams in a colour space with
libjpeg-turbo's triangle-filter upsampling instead of replicated chroma.

  * CPU: a numpy restatement of the header contract (upsample) equals libjpeg's own YCbCr output (PIL draft mode) sample for sample on streams
    whose IDCT is exact, so the filter and its edge rules are pinned to libjpeg independently of this decoder;
  * GPU, check A: FANCY output == fancy_rgb() of the decoder's own native samples, byte for byte, on the colour-exact corpus and sizes that cross
    CTA boundaries and MCU rows, every space, shift set, destination, Huffman route and marker scan, 4K and 8K;
  * GPU, against libjpeg end to end: within the bound of the 4:4:4 comparison, which replicated chroma exceeds on saturated content;
  * GPU: every output outside the scope is byte-identical to a REPLICATE decoder, the setter's refusals, and the decompress modules."""
import ctypes
import io

import numpy as np
import pytest
from PIL import Image

import jpeg_exact as J
import util
from test_jpeg import RGB, UYVY, natural_rgb
from test_jpeg_alpha import al  # noqa: F401  (fixture: the alpha oracle, for the corpus)
from test_jpeg_decode_color import bars, co, libjpeg_bound, pil_rgb  # noqa: F401  (co: fixture, the colour oracle)
from test_jpeg_decode_color import pil_stream as pil_rgb_stream
from test_jpeg_decode_color_exact import (AUTO, CS, DXT1, I420, JPEG, NATIVE, RGBA, SHIFTS, SPACES, VUYA, Case, _Big, _decoder, _encoder_stream, _get,
                                          check_a, corpus, cs_name, native, rgb)  # noqa: F401  (corpus: fixture)
from test_jpeg_exact import STD_TABLES, pil_stream
from test_jpeg_planar import pl  # noqa: F401  (fixture: the planar oracle, for the corpus)

SX = np.array([1, -1, -1, 1, 1, -1, -1, 1])  # sign of the exact IDCT of coefficient 4 along one axis: (cos((2x + 1) pi / 4) * sqrt 2)


@pytest.fixture(scope="module")
def orc():
    return util.oracle()


# ---- the restatement ---------------------------------------------------------------------------------------------------------------------
def upsample(c, w, h, vs):
    """a chroma plane of cw = ceil(w / 2) columns and ch rows (h for 4:2:2, ceil(h / 2) for 4:2:0) to w x h as libjpeg-turbo upsamples it: the
    triangle filter with neighbours clamped to the plane's edge; planes of at most two columns are replicated (libjpeg-turbo's jdsample.c
    filters only wider ones)"""
    c = np.asarray(c, np.int32)
    ch, cw = c.shape
    assert cw == (w + 1) // 2 and ch == (h if vs == 1 else (h + 1) // 2), (c.shape, w, h, vs)
    if cw <= 2:
        return np.repeat(np.repeat(c, vs, 0), 2, 1)[:h, :w]
    xm, xp = np.maximum(np.arange(cw) - 1, 0), np.minimum(np.arange(cw) + 1, cw - 1)
    if vs == 1:
        o = np.empty((ch, 2 * cw), np.int32)
        o[:, 0::2] = (3 * c + c[:, xm] + 1) >> 2
        o[:, 1::2] = (3 * c + c[:, xp] + 2) >> 2
        return o[:h, :w]
    ym, yp = np.maximum(np.arange(ch) - 1, 0), np.minimum(np.arange(ch) + 1, ch - 1)
    o = np.empty((2 * ch, 2 * cw), np.int32)
    for par, n in ((0, c[ym]), (1, c[yp])):
        s = 3 * c + n
        o[par::2, 0::2] = (3 * s + s[:, xm] + 8) >> 4
        o[par::2, 1::2] = (3 * s + s[:, xp] + 7) >> 4
    return o[:h, :w]


def fancy_rgb(planes, cs, sampling, w, h, shifts=None):
    """FANCY RGB / RGBA rows of decode_cs(cs): every pixel, YCBCR_TO_R/G/B of its own luma and its own upsampled chroma.  planes: the stream's
    samples, luma at least w x h, chroma of at least cw x ch (the native planes)."""
    cw, ch = (w + 1) // 2, h if sampling[1] == 1 else (h + 1) // 2
    Y = np.asarray(planes[0])[:h, :w]
    cb, cr = (upsample(np.asarray(p)[:ch, :cw], w, h, sampling[1]) for p in planes[1:])
    return rgb((Y, cb, cr), cs, (1, 1), w, shifts)


# ---- CPU: the restatement against libjpeg ------------------------------------------------------------------------------------------------
def exact_stream(w, h, vs, seed):
    """4:2:2 (vs 1) or 4:2:0 YCbCr whose every IDCT is exact in integers: Q = 8 and per block a DC and the coefficients (0, 4), (4, 0), whose
    exact IDCT is +-coef at every sample (SX), so no IDCT rounds, ours or libjpeg's; each block its own values.  Returns the stream and the
    sample planes on the block grids."""
    rng = np.random.default_rng(seed)
    mw, mh = -(-w // 16), -(-h // (8 * vs))
    coef, planes = [], []
    for c in range(3):
        shape = (mh * vs, mw * 2) if c == 0 else (mh, mw)
        a = np.zeros(shape + (64,), np.int64)
        dc, hx, vy = rng.integers(-60, 61, shape), rng.integers(-30, 31, shape), rng.integers(-30, 31, shape)
        a[..., 0], a[..., 4], a[..., 32] = dc, hx, vy
        coef.append(a)
        blk = 128 + dc[..., None, None] + hx[..., None, None] * SX[None, None, None, :] + vy[..., None, None] * SX[None, None, :, None]
        planes.append(blk.transpose(0, 2, 1, 3).reshape(shape[0] * 8, shape[1] * 8))
    s = J.write(w, h, [(1, 2, vs, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef, {0: np.full(64, 8), 1: np.full(64, 8)}, STD_TABLES,
                [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]])
    return s, planes


# chroma widths and heights 1, 2, 3 and 9; planes that end inside a block; 1 x N and N x 1; a few hundred pixels
PIN_SIZES = [(1, 1), (2, 2), (3, 3), (4, 4), (5, 5), (6, 6), (17, 17), (18, 9), (17, 33), (33, 37), (45, 37), (1, 40), (2, 40), (40, 1), (40, 2),
             (3, 17), (300, 200), (257, 131)]


@pytest.mark.parametrize("vs", [1, 2], ids=["422", "420"])
def test_restatement_equals_libjpeg(vs):
    """libjpeg-turbo's YCbCr output (PIL draft mode: its upsampler, no colour conversion) == the stream's exact samples for luma and
    upsample() of them for Cb and Cr, at every pixel.  At two chroma columns libjpeg replicates: the plain filter would differ there."""
    for w, h in PIN_SIZES:
        s, pl_ = exact_stream(w, h, vs, 1000 * w + h + vs)
        im = Image.open(io.BytesIO(s))
        im.draft("YCbCr", (w, h))
        assert im.mode == "YCbCr" and im.size == (w, h)
        lib = np.asarray(im).astype(np.int32)
        cw, ch = (w + 1) // 2, h if vs == 1 else (h + 1) // 2
        assert np.array_equal(lib[:, :, 0], pl_[0][:h, :w]), (w, h, "luma: the IDCT is not exact")
        for k in (1, 2):
            want = upsample(pl_[k][:ch, :cw], w, h, vs)
            assert np.array_equal(lib[:, :, k], want), (w, h, vs, k, np.argwhere(lib[:, :, k] != want)[:4])
            if cw == 2:
                c = pl_[k][:ch, :2].astype(np.int32)
                filt = np.stack([(3 * c[:, 0] + c[:, 0] + 1) >> 2, (3 * c[:, 0] + c[:, 1] + 2) >> 2], 1)
                assert not np.array_equal(np.repeat(filt, vs, 0)[:h], lib[:, :2, k]), (w, h)


def test_upsample_softens_a_step():
    """a flat chroma plane upsamples to itself; at a vertical step from 77 to 200 the two pixels next to the edge get a quarter of the step,
    (3 * 77 + 200 + 2) >> 2 = 108 and (3 * 200 + 77 + 1) >> 2 = 169 (4:2:0, s = 4 c: (3 * 308 + 800 + 7) >> 4 and (3 * 800 + 308 + 8) >> 4, the
    same), where replication keeps 77 and 200"""
    for vs in (1, 2):
        h = 5 if vs == 1 else 10
        c = np.full((5, 7), 77)
        assert (upsample(c, 13, h, vs) == 77).all()
        c[:, 3:] = 200
        o = upsample(c, 14, h, vs)
        assert (o == [77] * 5 + [108, 169] + [200] * 7).all(), o[0]


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------------
def _fancy(monkeypatch, scan=None, sync=None):
    dec = _decoder(monkeypatch, scan, sync)
    dec.set_upsampling("fancy")
    return dec


def _row(case, out_c):
    return case.w * (3 if out_c == RGB else 4)


def sweep(dec, case, planes, full):
    """FANCY RGB / RGBA of the case against fancy_rgb of its native planes; full: every space, shift set and destination (host, pitched device
    behind a sentinel), decode_cs and decode_to; else one of each kind, host only"""
    w, h = case.w, case.h
    for cs in (SPACES + ["auto"] if full else ["Y601full", "auto"]):
        eff = cs_name(cs, case)
        for shifts in (SHIFTS if full else [None, (8, 16, 24)]):
            out_c = RGB if shifts is None else RGBA
            want = fancy_rgb(planes, eff, case.sampling, w, h, shifts)
            what = f"{case.name}: FANCY decode_cs({cs}) to {'RGB' if shifts is None else f'RGBA {shifts}'}"
            check_a(_get(dec, case, out_c, cs, shifts=shifts or (0, 8, 16)).reshape(h, -1), want, what)
            if full:
                pitch = _row(case, out_c) + 48
                got = _get(dec, case, out_c, cs, shifts=shifts or (0, 8, 16), device=True, pitch=pitch).reshape(h, pitch)
                check_a(got[:, :_row(case, out_c)], want, what + " (device)")
                assert (got[:, _row(case, out_c):] == 0x5A).all(), (what, "bytes written behind the row")
                to = dec.decode(case.stream, out_c, shifts=shifts or (0, 8, 16), color_space=cs, out_cs="Y709")
                check_a(to.reshape(h, -1), want, what + " (decode_to)")


def fancy_cases(corpus):
    return [c for c in corpus if c.sampling[0] == 2 and not c.gray]


def size_cases():
    """widths across CTA boundaries (a CTA holds 32 MCUs = 512 pixels), heights across several MCU rows, odd sizes, 1 x 1 .. 3 x 3"""
    out = []
    for kind in ("420", "422"):
        for w, h in ((513, 37), (1041, 50), (1553, 33), (31, 67), (97, 129), (1, 1), (2, 2), (3, 3), (5, 17), (17, 1)):
            out.append(Case(f"pil-{kind} {w}x{h}", pil_stream(kind, w, h, seed=w + h)))
    out.append(Case("pil-420-rst-rows 1041x77", pil_stream("420-rst-rows", 1041, 77)))
    out.append(Case("pil-422-rst-blocks 1553x19", pil_stream("422-rst-blocks", 1553, 19)))
    return out


@pytest.mark.gpu
def test_gpu_fancy_equals_the_restatement(corpus, monkeypatch):
    """check A on every 4:2:2 / 4:2:0 stream of the colour-exact corpus and the size sweep: every space, shift set and destination"""
    dec, nat = _fancy(monkeypatch), _decoder(monkeypatch)
    cases = fancy_cases(corpus) + size_cases()
    assert len(cases) >= 30
    for case in cases:
        sweep(dec, case, native(nat, case, pin=False), True)
    dec.close(), nat.close()


@pytest.mark.gpu
@pytest.mark.parametrize("scan", ["host", "device"])
@pytest.mark.parametrize("sync", ["off", "on"])
def test_gpu_fancy_routes(corpus, monkeypatch, scan, sync):
    """both marker scans x both Huffman routes (the route taken asserted with last_sync), check A on one output of each kind"""
    dec, nat = _fancy(monkeypatch, scan, sync), _decoder(monkeypatch, scan, sync)
    for case in fancy_cases(corpus) + size_cases()[:6]:
        planes = native(nat, case, pin=False)
        sweep(dec, case, planes, False)
        assert dec.last_sync()["scans"] == (len(case.fr.scans) if sync == "on" else 0), case.name
    dec.close(), nat.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)], ids=["4K", "8K"])
def test_gpu_fancy_large_frames(orc, w, h):
    """check A at 4K (PIL 4:2:0 without DRI) and 8K (this encoder's 4:2:2 and PIL 4:2:0 without DRI)"""
    from ultragrid_b200 import api
    dec, nat = api.JpegDecoder(), api.JpegDecoder()
    dec.set_upsampling("fancy")
    streams = [("pil-420", pil_stream("420", w, h))] + ([("uyvy422", _encoder_stream(orc, "uyvy422", w, h))] if w > 4000 else [])
    for name, s in streams:
        case = _Big(f"{name} {w}x{h}", s)
        planes = native(nat, case, pin=False)
        for cs, shifts in (("Y601full", None), ("Y709", (16, 8, 0))):
            got = _get(dec, case, RGB if shifts is None else RGBA, cs, shifts=shifts or (0, 8, 16))
            check_a(got.reshape(h, -1), fancy_rgb(planes, cs, case.sampling, w, h, shifts), f"{case.name} FANCY decode_cs({cs})")
    dec.close(), nat.close()


def _encoder_rgb_stream(w, h, sub):
    """this encoder's RGB -> Y601full YCbCr stream (JFIF) at 4:2:0 or 4:2:2"""
    import torch
    from ultragrid_b200 import api
    enc = api.JpegEncoder()
    enc.encode_device(torch.from_numpy(np.ascontiguousarray(bars(w, h)).reshape(-1)).cuda(), w, h, RGB, quality=90, subsampling=sub, color_space=2)
    s = enc.result()
    enc.close()
    return s


@pytest.mark.gpu
def test_gpu_fancy_matches_libjpeg(co):
    """FANCY Y601full RGB within libjpeg_bound (the 4:4:4 comparison's (3, 3, 4): the upsampled chroma is within 1 of libjpeg's, both filters
    taking inputs within 1 with non-negative weights of the same sum and bias) of PIL's RGB, on PIL's own 4:2:0 / 4:2:2 streams and this encoder's
    RGB -> Y601full streams; on saturated bars the replicated chroma exceeds that bound, so the comparison tells the two modes apart"""
    from ultragrid_b200 import api
    bound = libjpeg_bound(co)
    w, h = 161, 97
    dec, rep = api.JpegDecoder(), api.JpegDecoder()
    dec.set_upsampling("fancy")
    streams = [(f"pil {content} q{q} sub{sub}", pil_rgb_stream(natural_rgb(w, h, 11) if content == "natural" else bars(w, h), q, sub), content)
               for q in (75, 90, 100) for sub in (1, 2) for content in ("natural", "bars")]
    streams += [(f"ours sub{sub}", _encoder_rgb_stream(w, h, sub), "bars") for sub in (420, 422)]
    for name, s, content in streams:
        assert api.jpeg_image_info(s).h_samp == 2, name
        want = pil_rgb(s).astype(np.int32)
        got = dec.decode(s, RGB, color_space="Y601full").reshape(h, w, 3).astype(np.int32)
        worst = np.abs(got - want).reshape(-1, 3).max(0)
        assert (worst <= bound).all(), (name, worst, bound)
        if content == "bars":
            n = w // 2 * 2
            old = rep.decode(s, RGB, color_space="Y601full").reshape(h, w, 3)[:, :n].astype(np.int32)
            assert (np.abs(old - want[:, :n]).reshape(-1, 3).max(0) > bound).any(), name
    dec.close(), rep.close()


@pytest.mark.gpu
def test_gpu_out_of_scope_outputs_do_not_move(corpus, monkeypatch):
    """with FANCY set, ugb200_jpeg_decode, colour space NATIVE, UYVY / I420 / VUYA output, 4:4:4 and grayscale streams of the colour-exact corpus
    are byte-identical to a REPLICATE decoder"""
    from ultragrid_b200 import api
    dec, rep = _fancy(monkeypatch), _decoder(monkeypatch)

    def outcome(f, d):  # the output, or the refusal's message (4:4:4 YCbCr to RGBA without a colour space is -4 in both modes)
        try:
            return f(d)
        except RuntimeError as e:
            return str(e)

    both = lambda f: (outcome(f, dec), outcome(f, rep))
    for name, s in [(c.name, c.stream) for c in corpus]:
        info = api.jpeg_image_info(s)
        gray = info.components == 1
        calls = []
        if not gray:
            calls += [(f"decode {oc}", lambda d, oc=oc, sh=sh: d.decode(s, oc, shifts=sh)) for oc, sh in ((UYVY, (0, 8, 16)), (RGB, (0, 8, 16)), (RGBA, (16, 8, 0)), (I420, (0, 8, 16)))]
            calls += [(f"decode_cs native {oc}", lambda d, oc=oc: d.decode(s, oc, color_space="native")) for oc in (RGB, RGBA)]
        if info.h_samp == 1 and not gray:
            calls += [(f"decode_cs {cs} {oc} 444", lambda d, cs=cs, oc=oc: d.decode(s, oc, color_space=cs)) for cs in SPACES + ["auto"] for oc in (RGB, RGBA)]
            calls += [("decode_to VUYA", lambda d: d.decode(s, VUYA, color_space="Y601full", out_cs="Y709"))]
        calls += [(f"decode_to {a}->{b} {oc}", lambda d, a=a, b=b, oc=oc: d.decode(s, oc, color_space=a, out_cs=b))
                  for a, b in (("Y601full", "Y709"), ("auto", "Y709"), ("native", "native")) for oc in (UYVY, I420)]
        if gray:
            calls += [(f"gray decode_to {cs} {RGB}", lambda d, cs=cs: d.decode(s, RGB, color_space=cs, out_cs="native")) for cs in ("Y601full", "auto")]
        for what, f in calls:
            a, b = both(f)
            if isinstance(a, str) or isinstance(b, str):
                assert a == b, (name, what, a, b)
                continue
            if what.split()[-1] in (str(RGB), str(RGBA)) and (info.h_samp == 2 or gray) and info.width % 2:  # whole pixel pairs only
                a, b = (v.reshape(info.height, -1)[:, :-(3 if what.endswith(str(RGB)) else 4)] for v in (a, b))
            check_a(a, b, f"{name}: {what}")
    dec.close(), rep.close()


@pytest.mark.gpu
def test_gpu_rgb_streams_and_refusals_do_not_move(orc, monkeypatch):
    """RGB and four-component streams (AUTO resolves to RGB) and the refusals: the same under FANCY as under REPLICATE; the setter refuses a
    bad mode and a NULL decoder"""
    from test_jpeg import orc_encode, orc_encode_interleaved_rgb
    from test_jpeg_decode_yuv import gray_image, gray_stream
    from ultragrid_b200 import _lib, api
    dec, rep = _fancy(monkeypatch), _decoder(monkeypatch)
    w, h = 130, 45
    rgb_src = natural_rgb(w, h, 7).reshape(-1).copy()
    streams = [("rgb", orc_encode(orc, rgb_src, w, h, RGB, 90)), ("rgb-il", orc_encode_interleaved_rgb(orc, rgb_src, w, h, 90))]
    for name, s in streams:
        assert api.jpeg_stream_color_space(s) == "RGB"
        for cs in ("auto", "Y601full", "native"):
            for oc in (RGB, RGBA, UYVY):
                check_a(dec.decode(s, oc, color_space=cs), rep.decode(s, oc, color_space=cs), f"{name} {cs} {oc}")
    gray = gray_stream(gray_image(41, 17), 90)
    for d in (dec, rep):  # decode_cs refuses grayscale with -4 in both modes
        with pytest.raises(RuntimeError, match="code -4"):
            d.decode(gray, RGB, color_space="Y601full")
        with pytest.raises(RuntimeError, match="code -3|code -4"):
            d.decode(b"\xff\xd8\xff\xd9", RGB, color_space="Y601full")
    L = _lib.load()
    assert L.ugb200_jpeg_decoder_set_upsampling(None, 1) == -1
    for bad in (-1, 2, 7):
        assert L.ugb200_jpeg_decoder_set_upsampling(dec._h, bad) == -1
    with pytest.raises(KeyError):
        dec.set_upsampling("bilinear")
    dec.set_upsampling("replicate")
    s = pil_stream("420", 63, 40)
    check_a(dec.decode(s, RGB, color_space="Y601full"), rep.decode(s, RGB, color_space="Y601full"), "back to replicate")
    dec.close(), rep.close()


@pytest.mark.gpu
def test_gpu_modules_fancy(monkeypatch):
    """UGB200_JPEG_DECODE_UPSAMPLE=fancy with UGB200_JPEG_DECODE_CS=y601full: the mirror-ABI gpujpeg module's RGB and RGBA == the library call
    with FANCY, gpujpeg_to_dxt == cuda_rgb_to_dxt1 of that RGB with the height mirrored; without a colour space, or with an unknown value, the
    modules keep today's bytes"""
    import torch
    from ultragrid_b200 import api
    from ultragrid_b200.compress import Decompress
    w, h = 1920, 1080
    s = pil_rgb_stream(bars(w, h), 90, 2)
    dec = api.JpegDecoder()
    dec.set_upsampling("fancy")
    want = {RGB: dec.decode(s, RGB, color_space="Y601full"), RGBA: dec.decode(s, RGBA, shifts=(16, 8, 0), color_space="Y601full")}
    dec.close()
    rep = api.JpegDecoder()
    plain = rep.decode(s, RGB)
    rep.close()

    def through(out_c, shifts=(0, 8, 16)):
        d = Decompress(JPEG, out_c)
        d.reconfigure(w, h, JPEG, out_c, shifts=shifts)
        st, out, _ = d.frame(s)
        d.close()
        assert st == Decompress.GOT_FRAME
        return out

    monkeypatch.setenv("UGB200_JPEG_DECODE_CS", "y601full")
    monkeypatch.setenv("UGB200_JPEG_DECODE_UPSAMPLE", "fancy")
    check_a(through(RGB)[:want[RGB].size], want[RGB], "gpujpeg RGB (fancy)")
    check_a(through(RGBA, (16, 8, 0))[:want[RGBA].size], want[RGBA], "gpujpeg RGBA (fancy)")
    dxt = api.compat_to_dxt("cuda_rgb_to_dxt1", torch.from_numpy(want[RGB].copy()).cuda(), w, -h).cpu().numpy()
    got = through(DXT1)
    check_a(got[:dxt.size], dxt, "gpujpeg_to_dxt DXT1 (fancy)")
    for cs, up in ((None, "fancy"), ("", "fancy"), (None, "bogus")):
        monkeypatch.delenv("UGB200_JPEG_DECODE_CS", raising=False)
        monkeypatch.setenv("UGB200_JPEG_DECODE_UPSAMPLE", up)
        check_a(through(RGB)[:plain.size], plain, f"gpujpeg RGB (UPSAMPLE={up}, no colour space)")
    monkeypatch.delenv("UGB200_JPEG_DECODE_UPSAMPLE", raising=False)


@pytest.mark.gpu
def test_gpu_real_abi_module_fancy(monkeypatch):
    """the real-ABI gpujpeg module in the reference's own framework, with UGB200_JPEG_DECODE_UPSAMPLE=fancy and UGB200_JPEG_DECODE_CS=y601full
    (skipped where the reference framework was not built)"""
    from test_real_module import dec_frame, framework
    from ultragrid_b200 import api
    fw = framework()
    w, h = 640, 360
    s = pil_rgb_stream(bars(w, h), 90, 2)
    dec = api.JpegDecoder()
    dec.set_upsampling("fancy")
    want = dec.decode(s, RGB, color_space="Y601full")
    dec.close()
    monkeypatch.setenv("UGB200_JPEG_DECODE_CS", "y601full")
    monkeypatch.setenv("UGB200_JPEG_DECODE_UPSAMPLE", "fancy")
    st = fw.fwd_dec_init(JPEG, RGB)
    assert st
    assert fw.fwd_dec_reconfigure(st, w, h, JPEG, 0, 8, 16, w * 3, RGB)
    rc, out, _ = dec_frame(fw, st, s, w * 3 * h)
    fw.fwd_dec_done(st)
    assert rc == 1
    check_a(out, want, "real-ABI gpujpeg RGB (fancy)")
