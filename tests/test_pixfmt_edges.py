"""The whole-buffer line converters (ugb200_pixfmt_convert, ugb200_vc_copyline) and the packed<->planar converters at their edges.

Every destination lies between guards of G sentinel bytes, and the whole buffer is compared, guards included: bytes a converter must not
write (pitch gaps, past a ragged dst_len, the rest of a 16-byte unit) keep the sentinel, and the spill the reference writes past the last
row (the `row == height - 1` rule of line_conv_kernel) is compared too.  Sources sit at unaligned base addresses where asked, and the
bytes after src_size are poison: include/ugb200.h promises that reads past src_size give 0, so poison must never reach the output.
Frames of 2 * 65 535 + 7 rows make every row loop take three turns (grid.y stops at 65 535), and a case per converter runs on a side
stream whose source arrives only after a sleep.

The expectation is the CPU restatement (oracle/libugoracle.so) run on the same framed buffer, with zeros after src_size.  The CPU part
checks that framed expectation against the unmodified reference objects (oracle/_ref/libugref.so) on the same geometries."""
import collections
import ctypes
import itertools

import numpy as np
import pytest

import planar_cases as pc
import util
from test_oracle_pinning import BGR, PAIRS, R10K, RG48, RGBA, UYVY, VUYA, Y416

from ultragrid_b200.codec import Codec

G = 64                    # guard bytes on each side of a destination (>= MAX_PADDING, video_codec.h:61)
SENT = 0xCD               # destination sentinel
POISON = 0xEE             # source bytes after src_size on the GPU
SLACK = 4096              # zeros after src_size on the CPU
TALL = 2 * 65535 + 7      # grid.y is capped at 65 535: every row loop takes three turns
DFL = (0, 8, 16)
SHIFTS = (DFL, (16, 8, 0), (8, 16, 24))
FORMS = (-1, 0, 1, 2, 3)  # ugb200_pixfmt_staged_mode: per converter, never staged (lean or general kernel), staged in + out, out only, in only
CHUNKS = (16, 32, 48, 64, 96, 128, 144, 192, 256)  # every C::OUT of pixfmt_kernels.cu, rgb_line_conv.cuh, yuv_rgb_conv.cuh, rgb_to_uyvy.cuh
SLEEP_CYCLES = 10_000_000  # a few ms of torch.cuda._sleep ahead of the side-stream upload

# the lean_default converters of pixfmt_kernels.cu with their (C::IN, C::OUT): line_conv_lean_kernel runs for them when pointers and pitches are
# 16-byte aligned, out_len(dst_len) is a whole number of chunks no longer than dst_pitch and every chunk of every row lies inside src_size
LEAN = {(UYVY, RGBA): (16, 32), (R10K, RGBA): (16, 16), (UYVY, RG48): (16, 48), (RGBA, VUYA): (16, 16), (BGR, UYVY): (48, 32),
        (RGBA, UYVY): (32, 16), (RGBA, R10K): (16, 16), (Y416, R10K): (32, 16), (Y416, RGBA): (32, 16), (VUYA, UYVY): (32, 16)}

# every codec_t from UGB_RGBA to UGB_DRM_PRIME (include/ugb200.h); ugb200_pixfmt_supported(c, c) admits each, through vc_memcpy
IDENTITY = list(range(1, 42))

LINE_FUNCS = {"ABGRtoRGB": (1, 4, 3), "BGRAtoRGB": (2, 4, 3), "ToRGBA_inplace": (3, 4, 4), "UYVYtoGrayscale": (4, 2, 1)}  # id, bytes/px in, out

Geo = collections.namedtuple("Geo", "w h sp dp dl off_s off_d src_size shifts")

_VP, _I, _L = ctypes.c_void_p, ctypes.c_int, ctypes.c_long


def _a16(n):
    return (n + 15) // 16 * 16


def _name(c):
    try:
        return Codec(c).name
    except ValueError:
        return f"codec{c}"


# ---- the conversions ------------------------------------------------------------------------------------------------------------------
class Pair:
    """ugb200_pixfmt_convert(inc, outc); with copy=True the plain copy of codec inc, whose `width` counts bytes"""
    inplace = False

    def __init__(self, inc, outc, copy=False):
        self.inc, self.outc, self.identity = inc, outc, copy
        self.id = f"copy-{_name(inc)}" if copy else f"{_name(inc)}-{_name(outc)}"

    def li(self, w):
        return w if self.identity else util.oracle().orc_vc_get_linesize(w, self.inc)

    def lo(self, w):
        return w if self.identity else util.oracle().orc_vc_get_linesize(w, self.outc)

    def size(self, w):
        return w if self.identity else util.oracle().orc_vc_get_size(w, self.outc)

    def ragged(self, w):
        """dst_len values of the existing suites: vc_get_size, and a whole number of words below it"""
        return [self.size(w), max(self.size(w) - 4, 0) // 4 * 4] if not self.identity else [w - 1, w - 5]

    def shift_sets(self):
        return (DFL,) if self.identity else SHIFTS  # RGB -> RGB and RGBA -> RGBA take the copy only with the default shifts

    def cpu(self, lib, dst, dp, src, sp, dl, h, shifts):
        fn = lib.orc_convert if hasattr(lib, "orc_convert") else lib.ref_convert
        return fn(self.inc, self.outc, dst, dp, src, sp, dl, h, *shifts)

    def admitted_by(self, ref):
        return ref.ref_has_decoder(self.inc, self.outc)

    def gpu(self, api, src, dst, g, stream=None):
        # the C ABI itself: most codecs of IDENTITY have no name in ultragrid_b200.codec
        rc = api._L.ugb200_pixfmt_convert(self.inc, self.outc, api._ptr(dst), g.dp, api._ptr(src), g.sp, g.dl, g.h, src.numel(), *g.shifts,
                                          api._stream(stream))
        assert rc == 0, (self.id, g, rc)


class Line:
    """ugb200_vc_copyline(func); ToRGBA_inplace also with dst == src"""

    def __init__(self, name, inplace=False):
        self.name, self.inplace = name, inplace
        self.fid, self.bi, self.bo = LINE_FUNCS[name]
        self.id = f"line-{name}" + ("-inplace" if inplace else "")

    def li(self, w):
        return w * self.bi

    def lo(self, w):
        return w * self.bo

    def size(self, w):
        return w * self.bo

    def ragged(self, w):
        return [self.lo(w) - 2, self.lo(w) - self.bo]  # as tests/test_named_line_converters.py

    def shift_sets(self):
        return SHIFTS if self.name == "ToRGBA_inplace" else (DFL,)

    def cpu(self, lib, dst, dp, src, sp, dl, h, shifts):
        fn = getattr(lib, "orc_copyline_named" if hasattr(lib, "orc_copyline_named") else "ref_copyline_named")
        fn.argtypes = [_I, _VP, _L, _VP, _L, _I, _I, _I, _I, _I]
        return fn(self.fid, dst, dp, src, sp, dl, h, *shifts)

    def admitted_by(self, ref):
        return hasattr(ref, "ref_copyline_named")

    def gpu(self, api, src, dst, g, stream=None):
        api.vc_copyline(self.name, src, dst, g.dl, g.h, g.sp, g.dp, shifts=g.shifts, stream=stream)


PAIR_CONVS = [Pair(i, o) for i, o in PAIRS]
LINE_CONVS = [Line(n) for n in LINE_FUNCS] + [Line("ToRGBA_inplace", inplace=True)]
CHUNKED = PAIR_CONVS + LINE_CONVS                       # everything launch_line runs
ALL = CHUNKED + [Pair(c, c, copy=True) for c in IDENTITY]  # plus copy_rows


def _ids(convs):
    return [c.id for c in convs]


# ---- geometries ------------------------------------------------------------------------------------------------------------------------
def make_geo(conv, w, h, sp, dp, dl=None, off=(0, 0), short=False, src_size=None, shifts=DFL):
    """short: src_size = (h - 1) * sp + line size, so the last row's over-read meets what lies after src_size; src_size: a source that
    ends earlier still, inside a row"""
    if conv.inplace:
        sp, off, short, src_size = dp, (off[1], off[1]), False, None  # one buffer, one pitch
    dl = conv.lo(w) if dl is None else dl
    if src_size is None:
        src_size = (h - 1) * sp + conv.li(w) if short else sp * h
    return Geo(w, h, sp, dp, dl, off[0], off[1], src_size, shifts)


def aligned(g):
    return g.off_s % 16 == 0 and g.off_d % 16 == 0 and g.sp % 16 == 0 and g.dp % 16 == 0


def _pitch(line, p):
    """p: bytes added to the line size, or 'a' / 'a16' / 'a64' for the 16-byte aligned pitch plus 0 / 16 / 64"""
    if isinstance(p, str):
        return _a16(line) + {"a": 0, "a16": 16, "a64": 64}[p]
    return line + p


# source / destination pitch: tight, +1, +4, +16, +64 on each side, and 16-byte aligned pitches
PITCH_PAIRS = [(0, 0), (1, 1), (4, 4), (16, 16), (64, 64), (0, 64), (64, 0), (1, 16), (16, 1), (4, 0), (0, 4), ("a", "a"), ("a16", "a"), ("a", "a64"),
               ("a64", "a16")]
OFFSETS = list(itertools.product((0, 1, 4, 8), (0, 1, 3, 8)))  # (off_s, off_d)


def geometries(conv):
    out = []
    for i, (ps, pd) in enumerate(PITCH_PAIRS):
        w, h = ((17, 1), (50, 2), (130, 5))[i % 3]
        out.append(make_geo(conv, w, h, _pitch(conv.li(w), ps), _pitch(conv.lo(w), pd)))
    for j, off in enumerate(OFFSETS):  # base offsets crossed with pitches that keep (16-byte multiples) or break 16-byte alignment
        w, h = ((48, 2), (17, 5))[j % 2]
        out.append(make_geo(conv, w, h, _a16(conv.li(w)), _a16(conv.lo(w)), off=off))
        out.append(make_geo(conv, w, h, conv.li(w) + 4, conv.lo(w) + 1, off=off))
    for w, h in ((17, 2), (50, 5), (130, 1)):  # dst_len: line size, vc_get_size, ragged, and one ending inside a 16-byte unit
        for dl in sorted({conv.lo(w), *conv.ragged(w), max(conv.lo(w) - 20, 0) // 4 * 4} - {0}):
            out.append(make_geo(conv, w, h, _a16(conv.li(w)), _a16(conv.lo(w)), dl))
            out.append(make_geo(conv, w, h, conv.li(w), conv.lo(w), dl))
    for w in (17, 50):  # short sources, aligned and not
        out.append(make_geo(conv, w, 5, _a16(conv.li(w)) + 16, _a16(conv.lo(w)), short=True))
        out.append(make_geo(conv, w, 5, conv.li(w) + 5, conv.lo(w) + 4, off=(1, 3), short=True))
        out.append(make_geo(conv, w, 1, conv.li(w), conv.lo(w), off=(4, 8), short=True))
        sp = _a16(conv.li(w)) + 16  # sources that end inside the last row, and inside the second
        out.append(make_geo(conv, w, 5, sp, _a16(conv.lo(w)), src_size=4 * sp + conv.li(w) // 2))
        out.append(make_geo(conv, w, 5, sp + 1, conv.lo(w) + 4, off=(8, 1), src_size=sp + 1 + conv.li(w) // 3))
    for shifts in conv.shift_sets()[1:]:
        out.append(make_geo(conv, 50, 2, _a16(conv.li(50)), _a16(conv.lo(50)), shifts=shifts))
        out.append(make_geo(conv, 17, 5, conv.li(17) + 1, conv.lo(17) + 4, off=(4, 1), shifts=shifts))
    return out


def _first_width(lo, target):
    a, b = 1, 1
    while lo(b) < target:
        b *= 2
    while a < b:
        m = (a + b) // 2
        a, b = (m + 1, b) if lo(m) < target else (a, m)
    return a


def chunk_geometries(conv):
    """Widths whose output line first reaches k * c bytes, k = 1, 127, 128, 129, for every chunk size c: the chunk count of every converter
    crosses one block (128 threads) at some of them.  Pointers and pitches are 16-byte aligned, dst_len is the line size and the source is
    whole, so where the line is exactly k * C::OUT bytes the lean_default converters take line_conv_lean_kernel (for instance UYVY -> RGBA,
    C::OUT = 32, at every width that is a multiple of 8); the width one pixel wider leaves a partial chunk (wlen % C::OUT != 0) and takes
    the general or the staged kernel.  The input line gets widths of its own for k = 1 and 128: where the output line is padded (R10k to 64
    pixels), only a width at which the source line covers it (a multiple of 64 pixels for RGBA -> R10k and Y416 -> R10k) reaches the lean form."""
    ws = set()
    for c in CHUNKS:
        for k in (1, 127, 128, 129):
            w = _first_width(conv.lo, k * c)
            ws.add(w)
            if k == 128:
                ws.add(w + 1)
        for k in (1, 128):
            ws.add(_first_width(conv.li, k * c))
    return [make_geo(conv, w, 2, _a16(conv.li(w)), _a16(conv.lo(w))) for w in sorted(ws)]


def lean_runs(conv, g):
    """whether launch_line picks line_conv_lean_kernel for g when not forced to a staged form"""
    key = (getattr(conv, "inc", None), getattr(conv, "outc", None))
    if key not in LEAN or not aligned(g) or g.dl != conv.lo(g.w):
        return False
    cin, cout = LEAN[key]
    return g.dl % cout == 0 and g.dl <= g.dp and (g.h - 1) * g.sp + g.dl // cout * cin <= g.src_size


def tall_geometries(conv):
    """a narrow frame (at least 512 output bytes per row, so two chunks of every size) of TALL rows: aligned for the staged and lean forms,
    and at odd offsets and pitches for the general kernel's byte paths"""
    w = next((w for w in range(1, 4096) if conv.lo(w) >= 512 and conv.lo(w) % 192 == 0), None) or _first_width(conv.lo, 512)
    return [(make_geo(conv, w, TALL, _a16(conv.li(w)), _a16(conv.lo(w))), FORMS),
            (make_geo(conv, w, TALL, conv.li(w) + 1, conv.lo(w) + 4, off=(1, 3)), (-1,))]


# ---- CPU expectation -----------------------------------------------------------------------------------------------------------------
def source_bytes(g, seed):
    return util.rng_bytes(g.sp * g.h, seed)


def expect(conv, lib, g, src):
    """G sentinel bytes, the dst_pitch * height frame, G more; the source is its first src_size bytes followed by zeros"""
    out = np.full(2 * G + g.dp * g.h, SENT, np.uint8)
    if conv.inplace:
        out[G:G + g.dp * g.h] = src[:g.dp * g.h]
        sptr = out.ctypes.data + G
    else:
        srcp = np.zeros(g.src_size + SLACK, np.uint8)
        srcp[:g.src_size] = src[:g.src_size]
        sptr = srcp.ctypes.data
    rc = conv.cpu(lib, out.ctypes.data + G, g.dp, sptr, g.sp, g.dl, g.h, g.shifts)
    assert rc == 0, (conv.id, g, rc)
    return out


# ---- CPU part: the framed expectation against the unmodified reference ------------------------------------------------------------------
def _cpu_geometries(conv):
    """the geometries the reference can run: many of its loops assert 2- or 4-byte aligned rows (pixfmt_conv.c), so pitches here are multiples of 4"""
    seen, out = set(), []
    for g in geometries(conv) + chunk_geometries(conv):
        key = g._replace(off_s=0, off_d=0)  # base offsets do not change what the CPU writes
        if key not in seen and g.sp % 4 == 0 and g.dp % 4 == 0:
            seen.add(key)
            out.append(key)
    return out


@pytest.mark.parametrize("conv", ALL, ids=_ids(ALL))
def test_framed_restatement_equals_reference(orc, ref_cpu, conv):
    if not conv.admitted_by(ref_cpu):
        pytest.skip(f"the reference has no decoder for {conv.id}")
    for i, g in enumerate(_cpu_geometries(conv)):
        src = source_bytes(g, 5000 + i)
        a, b = expect(conv, orc, g, src), expect(conv, ref_cpu, g, src)
        assert np.array_equal(a, b), (conv.id, g, np.flatnonzero(a != b)[:8])


def test_every_lean_converter_gets_lean_and_general_geometries():
    for conv in PAIR_CONVS:
        if (conv.inc, conv.outc) in LEAN:
            geos = geometries(conv) + chunk_geometries(conv)
            n = sum(lean_runs(conv, g) for g in geos)
            assert 0 < n < len(geos), (conv.id, n, len(geos))


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def api():
    from ultragrid_b200 import api as a
    return a


def _source_buffer(g, src):
    b = np.full(g.off_s + g.src_size + SLACK, POISON, np.uint8)
    b[g.off_s:g.off_s + g.src_size] = src[:g.src_size]
    return b


def _inplace_init(g, src):
    b = np.full(g.off_d + 2 * G + g.dp * g.h, SENT, np.uint8)
    b[g.off_d + G:g.off_d + G + g.dp * g.h] = src[:g.dp * g.h]
    return b


def _assert_same(torch, got, want, what):
    if not torch.equal(got, want):
        bad = torch.nonzero(got != want).flatten()[:8].cpu().tolist()
        pytest.fail(f"{what}: bytes differ at {bad} (the frame starts at {G})")


def run_forms(api, conv, g, src, want_d, forms):
    """run g in every form of `forms` and compare the whole framed destination on the device"""
    import torch
    frame0 = g.off_d + G
    if conv.inplace:
        init = torch.from_numpy(_inplace_init(g, src)).cuda()
        d_dst = torch.empty_like(init)
    else:
        d_src = torch.from_numpy(_source_buffer(g, src)).cuda()
        d_dst = torch.empty(g.off_d + 2 * G + g.dp * g.h, dtype=torch.uint8, device="cuda")
    frame = d_dst[frame0:frame0 + g.dp * g.h]
    for form in forms:
        api.pixfmt_staged_mode(form)
        if conv.inplace:
            d_dst.copy_(init)
            s_view = frame[:g.src_size]
        else:
            d_dst.fill_(SENT)
            s_view = d_src[g.off_s:g.off_s + g.src_size]
        conv.gpu(api, s_view, frame, g)
        _assert_same(torch, d_dst[g.off_d:], want_d, f"{conv.id} {g} form {form}")


@pytest.mark.gpu
@pytest.mark.parametrize("conv", ALL, ids=_ids(ALL))
def test_edges_vs_restatement(api, orc, conv):
    """every geometry in every launch form that can apply: the forms only differ where pointers and pitches are 16-byte aligned"""
    import torch
    if isinstance(conv, Pair):
        assert api.pixfmt_supported(conv.inc, conv.outc)
        assert not api.pixfmt_supported(IDENTITY[-1] + 1, IDENTITY[-1] + 1)  # IDENTITY is every admitted codec
    try:
        for i, g in enumerate(geometries(conv) + chunk_geometries(conv)):
            src = source_bytes(g, 6000 + i)
            want = torch.from_numpy(expect(conv, orc, g, src)).cuda()
            run_forms(api, conv, g, src, want, FORMS if aligned(g) else (-1,))
    finally:
        api.pixfmt_staged_mode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("conv", CHUNKED, ids=_ids(CHUNKED))
def test_tall_frames(api, orc, conv):
    """TALL rows: the row loops of the general, lean and staged kernels take three turns; one expectation per geometry, reused across forms"""
    import torch
    try:
        for i, (g, forms) in enumerate(tall_geometries(conv)):
            src = source_bytes(g, 7000 + i)
            want = torch.from_numpy(expect(conv, orc, g, src)).cuda()
            run_forms(api, conv, g, src, want, forms)
            del want
    finally:
        api.pixfmt_staged_mode(-1)


def _side_stream(torch, fill_and_launch):
    """queue a sleep on a fresh stream, then fill_and_launch(stream) there; the caller's buffers hold stale data written before"""
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        keep = fill_and_launch(s)
    s.synchronize()
    return keep


@pytest.mark.gpu
@pytest.mark.parametrize("conv", ALL, ids=_ids(ALL))
def test_side_stream(api, orc, conv):
    """the source arrives on the caller's stream after a sleep; a launch on any other stream reads the stale source"""
    import torch
    w = 50
    for i, g in enumerate((make_geo(conv, w, 5, _a16(conv.li(w)), _a16(conv.lo(w))),
                           make_geo(conv, w, 5, conv.li(w) + 1, conv.lo(w) + 4, off=(1, 3)))):
        src = source_bytes(g, 8000 + i)
        want = torch.from_numpy(expect(conv, orc, g, src)).cuda()
        framed = _inplace_init(g, src) if conv.inplace else np.full(g.off_d + 2 * G + g.dp * g.h, SENT, np.uint8)
        h_dst = torch.from_numpy(framed).pin_memory()
        h_src = torch.from_numpy(_source_buffer(g, src)).pin_memory()
        d_dst = torch.full((h_dst.numel(),), 0x11, dtype=torch.uint8, device="cuda")  # stale
        d_src = torch.full((h_src.numel(),), 0x5A, dtype=torch.uint8, device="cuda")  # stale
        frame = d_dst[g.off_d + G:g.off_d + G + g.dp * g.h]

        def launch(s):
            d_src.copy_(h_src, non_blocking=True)
            d_dst.copy_(h_dst, non_blocking=True)
            s_view = frame[:g.src_size] if conv.inplace else d_src[g.off_s:g.off_s + g.src_size]
            conv.gpu(api, s_view, frame, g, stream=s)
            return h_src, h_dst

        _side_stream(torch, launch)
        _assert_same(torch, d_dst[g.off_d:], want, f"{conv.id} {g} side stream")


# ---- packed <-> planar and v210 -> P010 ------------------------------------------------------------------------------------------------
PLANAR = pc.all_cases()


def _planar_height(name, h):
    return h + 1 if name == "yuv420_to_i420" and h % 2 else h  # the reference asserts even sizes there (from_planar.c:371-372)


def _planar_fn(lib, name):
    fn = getattr(lib, "ugb200_" + name)
    fn.argtypes = [_VP, _VP]
    fn.restype = _I
    return fn


@pytest.mark.gpu
@pytest.mark.parametrize("name,depth", PLANAR)
def test_planar_tall_frames(orc, name, depth):
    """TALL rows (TALL + 1 for yuv420_to_i420): the 4:2:0 functions loop over row pairs, so their loops take a second turn too"""
    import torch
    from ultragrid_b200 import _lib
    fn = _planar_fn(_lib.load(), name)
    for mode in (0, 2):  # 16-byte aligned pitches, and pitches that are only 2-byte aligned
        c = pc.Case(name, 48, _planar_height(name, TALL), seed=90 + mode, mode=mode, depth=depth)
        want = c.run_cpu(orc, "orc_")
        ins = [torch.from_numpy(a).cuda() for a in c.inputs()]
        outs = [torch.from_numpy(o).cuda() for o in c.alloc_out()]
        d = c.struct([t.data_ptr() for t in ins], [t.data_ptr() for t in outs])
        assert fn(ctypes.byref(d), _VP(torch.cuda.current_stream().cuda_stream)) == 0
        for k, (o, x) in enumerate(zip(outs, want)):
            _assert_same(torch, o, torch.from_numpy(x).cuda(), f"{name} {depth} mode {mode} plane {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,depth", PLANAR)
def test_planar_side_stream(orc, name, depth):
    import torch
    from ultragrid_b200 import _lib
    fn = _planar_fn(_lib.load(), name)
    c = pc.Case(name, 50 if name != "yuv420_to_i420" else 48, 6, seed=3, mode=1, depth=depth)
    want = c.run_cpu(orc, "orc_")
    h_ins = [torch.from_numpy(a).pin_memory() for a in c.inputs()]
    h_outs = [torch.from_numpy(o).pin_memory() for o in c.alloc_out()]
    ins = [torch.full((t.numel(),), 0x5A, dtype=torch.uint8, device="cuda") for t in h_ins]    # stale
    outs = [torch.full((t.numel(),), 0x11, dtype=torch.uint8, device="cuda") for t in h_outs]  # stale
    d = c.struct([t.data_ptr() for t in ins], [t.data_ptr() for t in outs])

    def launch(s):
        for dv, hv in zip(ins + outs, h_ins + h_outs):
            dv.copy_(hv, non_blocking=True)
        assert fn(ctypes.byref(d), _VP(s.cuda_stream)) == 0
        return h_ins, h_outs

    _side_stream(torch, launch)
    for k, (o, x) in enumerate(zip(outs, want)):
        _assert_same(torch, o, torch.from_numpy(x).cuda(), f"{name} {depth} side stream plane {k}")


@pytest.mark.gpu
def test_v210_to_p010le_tall(api, orc):
    """v210_to_p010le loops over row pairs: TALL rows, odd, with a partial 6-pixel group and sentinel guards around both planes"""
    import torch
    w, h = 100, TALL
    ls_y, ls_c = w * 2 + 40, w * 2 + 24
    src = util.v210_noise(w, h, 17)
    y = np.full(2 * G + ls_y * h, SENT, np.uint8)
    c = np.full(2 * G + ls_c * ((h + 1) // 2), SENT, np.uint8)
    orc.orc_v210_to_p010le(w, h, y.ctypes.data + G, ls_y, c.ctypes.data + G, ls_c, src.ctypes.data)
    dy = torch.full((y.size,), SENT, dtype=torch.uint8, device="cuda")
    dc = torch.full((c.size,), SENT, dtype=torch.uint8, device="cuda")
    api.v210_to_p010le(torch.from_numpy(src).cuda(), w, h, out_y=dy[G:], out_c=dc[G:], ls_y=ls_y, ls_c=ls_c)
    _assert_same(torch, dy, torch.from_numpy(y).cuda(), "v210_to_p010le luma")
    _assert_same(torch, dc, torch.from_numpy(c).cuda(), "v210_to_p010le chroma")
