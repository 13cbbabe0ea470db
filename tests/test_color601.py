"""BT.601 in the colour conversions: ugb200_pixfmt_convert_cs and ugb200_to_lavc_convert_cs with UGB_CS_601 against UltraGrid run with
`--param color-601`.

The oracle is the unmodified reference built a second time (oracle/color601.mk -> oracle/_ref/libugref601.so): the same objects as
libugref.so, linked with a host stub whose get_commandline_param("color-601") is non-NULL, so every get_color_coeffs(CS_DFL, depth) there
returns the BT.601 set.  tests/golden/color601_golden.npz holds its outputs for machines without oracle/_ref.

CPU (no GPU):
  * the 601 build's get_color_coeffs(CS_DFL, d), d in {0, 8, 10, 12, 16}, is the BT.601 set re-derived in float64 and the static_assert pins
    of csrc/color_space.h;
  * the selection line of get_color_coeffs, `cs != (CS_DFL ? cs : dfl_cs) - 1` (color_space.c:157), restated, agrees with both builds for
    every (default, cs, depth): callers passing CS_DFL get the default space, and an explicit CS_601 under color-601 gets BT.709;
  * the pairs whose output differs between the two builds are exactly the converters the library instantiates per coefficient set;
  * the framed expectation used on the GPU (the 601 build run row by row where the reference cannot take the pitches) equals the 601 build
    run directly wherever it can;
  * the to_lavc restatement of test_lavc_exact.py with the BT.601 sets equals oracle/lavc_oracle.c given those sets, and its RGB family lies
    within the derived bound of the float64 BT.601 matrix; mutants (BT.709 under 601, the depth-8 set at 10 / 16 bits, Cb and Cr swapped) fail.

GPU: every pair ugb200_pixfmt_supported admits, in every launch form, at the edge geometries of test_pixfmt_edges.py (sentinels around every
buffer, unaligned bases, ragged dst_len, short sources), at 1080p and 8K widths and on a side stream, equals the 601 build; CS_DFL and CS_709
equal ugb200_pixfmt_convert; every to_lavc pair under CS_601 equals the restatement inside sentinel bands, in the call and the hook form; an
invalid colour space writes nothing."""
import contextlib
import ctypes
import os
import re

import numpy as np
import pytest

import test_lavc_exact as tle
import test_pixfmt_edges as pe
import util
from test_jpeg_decode_color_exact import KR_KB, RGB_FIELDS, _c_limit, _y_limit, color_coeffs
from test_oracle_pinning import BGR, PAIRS, R10K, R12L, RG48, RGB, RGBA, UYVY, V210, VUYA, Y216, Y416, YUYV

CS_DFL, CS_601, CS_709 = 0, 1, 2
DEPTHS = (0, 8, 10, 12, 16)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "color601_golden.npz")
GOLDEN_SIZES = ((50, 3), (193, 2))
_vp, _i, _l = ctypes.c_void_p, ctypes.c_int, ctypes.c_long
EPS = 1e-6

# the decoders whose reference body reads get_color_coeffs (pixfmt_conv.c): the converters pixfmt_kernels.cu instantiates per coefficient set
COEFF_PAIRS = {(UYVY, RGB), (YUYV, RGB), (UYVY, RG48), (RGB, UYVY), (BGR, UYVY), (RGBA, UYVY), (RG48, UYVY), (R10K, UYVY), (R10K, Y416),
               (R12L, Y416), (R12L, UYVY), (Y416, R12L), (Y416, RG48), (Y416, RGB), (Y416, RGBA), (Y416, R10K), (RGBA, VUYA), (VUYA, RGB),
               (RG48, V210), (RG48, Y216), (RG48, Y416), (V210, RGB), (V210, RG48)}


def space(cs):
    return "Y601" if cs == CS_601 else "Y709"


def ref601_lib():
    """oracle/_ref/libugref601.so (its own dfl_cs: ctypes loads it RTLD_LOCAL), or None when it is not built"""
    def bind(L):
        L.ref_convert.argtypes = [_i, _i, _vp, _l, _vp, _l, _i, _i, _i, _i, _i]
        L.ref_has_decoder.argtypes = [_i, _i]
        L.ref_vc_get_linesize.argtypes = [ctypes.c_uint, _i]
        L.ref_get_color_coeffs.argtypes, L.ref_get_color_coeffs.restype = [_i, _i, _vp], None
        return L
    return util.ref_lib("libugref601.so", bind)


@pytest.fixture(scope="module")
def ref601():
    lib = ref601_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libugref601.so not built (reference tree absent)")
    return lib


def probe(lib, cs, depth):
    out = (_i * 14)()
    lib.ref_get_color_coeffs(cs, depth, out)
    return dict(zip(RGB_FIELDS, out))


# ---- coefficients and their selection -------------------------------------------------------------------------------------------------
def test_601_build_returns_bt601_for_cs_dfl(ref601):
    pins = {}
    src = open(os.path.join(util.ROOT, "ultragrid_b200", "csrc", "color_space.h")).read()
    depth_of = {n: int(d) for n, d in re.findall(r"\b(s\d+) = coeffs_601\((\d+)\)", src)}
    for n, f, v in re.findall(r"\b(s\d+)\.(\w+) == (-?\d+)", src):
        pins.setdefault(depth_of[n], {})[f] = int(v)
    assert set(pins) == {8, 10, 16} and all(len(p) == 14 for p in pins.values())
    for d in DEPTHS:
        want = color_coeffs(*KR_KB["Y601"], d)
        assert probe(ref601, CS_DFL, d) == {f: want[f] for f in RGB_FIELDS}, d
        if d in pins:
            assert {f: want[f] for f in pins[d]} == pins[d], d


def selects_709(dfl_cs, cs):
    """color_space.c:157: cs_idx = cs != (CS_DFL ? cs : dfl_cs) - 1; CS_DFL is 0, so the condition always takes dfl_cs; index 1 is BT.709"""
    return cs != (cs if CS_DFL else dfl_cs) - 1


def test_selection_line_agrees_with_both_builds(ref_cpu, ref601):
    for dfl, lib in ((CS_709, ref_cpu), (CS_601, ref601)):
        for cs in (CS_DFL, CS_601, CS_709):
            for d in DEPTHS:
                want = color_coeffs(*KR_KB["Y709" if selects_709(dfl, cs) else "Y601"], d)
                assert probe(lib, cs, d) == {f: want[f] for f in RGB_FIELDS}, (dfl, cs, d)
        assert selects_709(dfl, CS_DFL) == (dfl == CS_709)  # CS_DFL callers (every converter) get the default space
    assert selects_709(CS_601, CS_601)  # the quirk: an explicit CS_601 under color-601 selects BT.709


def test_coefficient_reading_pairs_are_the_instantiated_ones(ref_cpu, ref601):
    """the two builds differ on random frames exactly where the library has a per-set converter; elsewhere the bytes are the same"""
    differ = set()
    for n, (inc, outc) in enumerate(PAIRS):
        assert ref601.ref_has_decoder(inc, outc)
        for w, h in ((50, 3), (193, 2)):
            src = util.rng_bytes(ref_cpu.ref_vc_get_linesize(w, inc) * h, 300 + n)
            a = util.convert_cpu(ref_cpu, "ref_convert", inc, outc, src, w, h, linesize=ref_cpu.ref_vc_get_linesize)
            b = util.convert_cpu(ref601, "ref_convert", inc, outc, src, w, h, linesize=ref_cpu.ref_vc_get_linesize)
            if not np.array_equal(a, b):
                differ.add((inc, outc))
    assert differ == COEFF_PAIRS


# ---- the framed expectation ----------------------------------------------------------------------------------------------------------------
def expect_rows(conv, lib, g, src):
    """pe.expect with the reference `lib` run one row at a time from aligned copies, in row order (a row's spill is overwritten by the next
    row, as in the row loop); a row's written bytes are those where a run over 0x00 or a run over 0xFF left its fill"""
    out = np.full(2 * pe.G + g.dp * g.h, pe.SENT, np.uint8)
    srcp = np.zeros(g.src_size + pe.SLACK, np.uint8)
    srcp[:g.src_size] = src[:g.src_size]
    span = g.dl + 512
    for y in range(g.h):
        row = srcp[y * g.sp:].copy()
        runs = []
        for fill in (0x00, 0xFF):
            d = np.full(span, fill, np.uint8)
            assert conv.cpu(lib, d.ctypes.data, span, row.ctypes.data, span, g.dl, 1, g.shifts) == 0
            runs.append(d)
        wr = (runs[0] != 0x00) | (runs[1] != 0xFF)
        at = pe.G + y * g.dp
        n = min(span, out.size - at)
        out[at:at + n][wr[:n]] = np.where(runs[0] != 0x00, runs[0], runs[1])[:n][wr[:n]]
    return out


def expect_cs(conv, lib, g, src):
    """the framed expectation of g: the reference run directly where both pitches are multiples of 4 (it asserts aligned rows elsewhere),
    row by row otherwise"""
    return pe.expect(conv, lib, g, src) if g.sp % 4 == 0 and g.dp % 4 == 0 else expect_rows(conv, lib, g, src)


@pytest.mark.parametrize("conv", pe.PAIR_CONVS, ids=pe._ids(pe.PAIR_CONVS))
def test_row_by_row_expectation_equals_the_reference(ref601, conv):
    for i, g in enumerate(pe._cpu_geometries(conv)):
        src = pe.source_bytes(g, 5000 + i)
        assert np.array_equal(pe.expect(conv, ref601, g, src), expect_rows(conv, ref601, g, src)), (conv.id, g)


def golden_cases():
    """(key, inc, outc, w, h, seed): the cases of tests/golden/make_color601_golden.py"""
    return [(f"c{inc}_{outc}_{w}x{h}", inc, outc, w, h, 9100 + n) for n, (inc, outc) in enumerate(PAIRS) for w, h in GOLDEN_SIZES]


def golden_source(inc, w, h, seed):
    return util.rng_bytes(util.oracle().orc_vc_get_linesize(w, inc) * h, seed)


def test_golden_fixtures_equal_the_601_build(ref601):
    gold = util.golden(GOLDEN)
    for key, inc, outc, w, h, seed in golden_cases():
        src = golden_source(inc, w, h, seed)
        want = util.convert_cpu(ref601, "ref_convert", inc, outc, src, w, h, linesize=ref601.ref_vc_get_linesize)
        assert np.array_equal(gold[key], want), key


# ---- to_lavc: the restatement of test_lavc_exact.py with a colour space -----------------------------------------------------------------
@contextlib.contextmanager
def lavc_coeffs(fn):
    """test_lavc_exact's restatement with get_color_coeffs(CS_DFL, depth) := fn(depth)"""
    saved = tle.coeffs
    tle.coeffs = fn
    try:
        yield
    finally:
        tle.coeffs = saved


def coeffs_of(cs):
    return lambda depth: color_coeffs(*KR_KB[space(cs)], depth)


MUTANTS = {
    "709_under_601": coeffs_of(CS_709),
    "depth8_set": lambda depth: color_coeffs(*KR_KB["Y601"], 8),
    "cb_cr_swapped": lambda depth: {**color_coeffs(*KR_KB["Y601"], depth),
                                    **{f"cb{s}": color_coeffs(*KR_KB["Y601"], depth)[f"cr{s}"] for s in ("_r", "_g", "_b")},
                                    **{f"cr{s}": color_coeffs(*KR_KB["Y601"], depth)[f"cb{s}"] for s in ("_r", "_g", "_b")}},
}


def ref_to_lavc_cs(inc, fmt, src, w, h, lss, orc=None, cs=CS_601, fn=None):
    with lavc_coeffs(fn or coeffs_of(cs)):
        return tle.ref_to_lavc(inc, fmt, src, w, h, lss, orc)


def orc_lavc_cs(orc, inc, fmt, src, w, h, lss, cs=CS_601):
    with lavc_coeffs(coeffs_of(cs)):
        return tle.orc_lavc(orc, inc, fmt, src, w, h, lss)


def _restatement_differs(orc, inc, fmt, fn):
    for k, (w, h) in enumerate([(48, 4), (49, 3), (47, 2), (6, 1), (8, 3), (1922, 3), (100, 5), (13, 7)]):
        shapes, bps = tle.av_geom(fmt, w, h)
        lss = [n * bps + (k % 3) * 2 * bps for n, _ in shapes]
        src = tle.make_source(inc, w, h, 40 + k)
        want = ref_to_lavc_cs(inc, fmt, src, w, h, lss, fn=fn)
        got = orc_lavc_cs(orc, inc, fmt, src, w, h, lss)
        if any(not np.array_equal(g[wr], b[wr]) for g, b, wr in zip(got, want.buf, want.wr)):
            return True
    return False


@pytest.mark.parametrize("inc,fmt", tle.TO_PAIRS_KNOWN)
def test_lavc_restatement_601_equals_lavc_oracle(orc, inc, fmt):
    """the restatement with the BT.601 sets == oracle/lavc_oracle.c given the same sets (orc_lavc_rgb takes them as an argument)"""
    assert not _restatement_differs(orc, inc, fmt, coeffs_of(CS_601))


def bound_violations(inc, fmt, cs, fn=None, seed=8):
    """tle.rgb_bound_violations against the float64 matrix of `cs`: |output - exact| within the Q14 rounding of each coefficient and the floor.
    The bound is reached exactly where the floor takes nothing off; EPS absorbs the float64 rounding of `exact` and `err` there."""
    w, h = 64, 6
    src = tle.make_source(inc, w, h, seed)
    shapes, bps = tle.av_geom(fmt, w, h)
    P = ref_to_lavc_cs(inc, fmt, src, w, h, [n * bps for n, _ in shapes], cs=cs, fn=fn)
    r, g, b, in_depth = tle.rgb_samples(inc, src, w, h)
    depth = 8 if fmt == "YUV444P" else int(fmt[7:9])
    kr, kb = KR_KB[space(cs)]
    kg, yl, cl = 1 - kr - kb, _y_limit(depth), _c_limit(depth)
    M = np.array([[kr * yl, kg * yl, kb * yl], [-kr / (2 * (kr + kg)) * cl, -kg / (2 * (kr + kg)) * cl, (1 - kb) / (2 * (kr + kg)) * cl],
                  [(1 - kr) / (2 * (1 - kr)) * cl, -kg / (2 * (1 - kr)) * cl, -kb / (2 * (1 - kr)) * cl]])
    off = [1 << (depth - 4), 1 << (depth - 1), 1 << (depth - 1)]
    n = r.shape[1] if inc == R12L else w
    rgb = np.stack([r[:, :n], g[:, :n], b[:, :n]], -1).astype(np.float64)
    sh = 14 + in_depth - depth
    c = coeffs_of(cs)(depth)  # the bound is that of the true set, whatever the restatement used
    Q = np.array([[c[k + s] for s in ("_r", "_g", "_b")] for k in ("y", "cb", "cr")], np.float64)
    bad = 0
    for i in range(3):
        exact = rgb @ M[i] * 2.0 ** (depth - in_depth) + off[i]
        err = rgb @ np.abs(Q[i] - 16384 * M[i]) / 2.0 ** sh
        got = P.buf[i].view("<u2" if bps == 2 else np.uint8).astype(np.float64)[:, :P.buf[i].shape[1] // bps]
        if i and "422" in fmt:
            exact, err = exact[:, 0::2], err[:, 0::2]
        m = min(got.shape[1], exact.shape[1])
        d = got[:, :m] - exact[:, :m]
        bad += int(np.count_nonzero((d > err[:, :m] + EPS) | (d < -err[:, :m] - 1 - EPS)))
    return bad


@pytest.mark.parametrize("inc,fmt", tle.RGB_FAMILY)
def test_lavc_rgb_family_within_float64_bt601_bound(inc, fmt):
    assert bound_violations(inc, fmt, CS_601) == 0


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutants_fail(orc, mutant):
    """each mutant of the coefficient choice is caught: by the float64 BT.601 bound on every RGB-family pair, and by lavc_oracle.c"""
    fn = MUTANTS[mutant]
    assert all(bound_violations(inc, fmt, CS_601, fn) > 0 for inc, fmt in tle.RGB_FAMILY if mutant != "depth8_set" or fmt != "YUV444P"), mutant
    assert _restatement_differs(orc, RG48, "YUV444P16LE", fn), mutant
    if mutant == "depth8_set":
        assert bound_violations(RG48, "YUV444P10LE", CS_601, fn) > 0 and bound_violations(R10K, "YUV444P16LE", CS_601, fn) > 0


# ---- GPU: line converters --------------------------------------------------------------------------------------------------------------------
class PairCS(pe.Pair):
    """pe.Pair through ugb200_pixfmt_convert_cs"""

    def __init__(self, inc, outc, cs):
        super().__init__(inc, outc)
        self.cs = cs
        self.id += f"-cs{cs}"

    def gpu(self, api, src, dst, g, stream=None):
        rc = api._L.ugb200_pixfmt_convert_cs(self.inc, self.outc, api._ptr(dst), g.dp, api._ptr(src), g.sp, g.dl, g.h, src.numel(), *g.shifts,
                                             self.cs, api._stream(stream))
        assert rc == 0, (self.id, g, rc)


CONVS_601 = [PairCS(i, o, CS_601) for i, o in PAIRS]


@pytest.fixture(scope="module")
def api():
    from ultragrid_b200 import api as a
    return a


@pytest.mark.gpu
def test_gpu_pairs_are_those_admitted(api):
    """PAIRS holds every pair of distinct codecs ugb200_pixfmt_supported admits (the other identities are plain copies, the same for every cs)"""
    assert {(i, o) for i in range(1, 42) for o in range(1, 42) if i != o and api.pixfmt_supported(i, o)} == {p for p in PAIRS if p[0] != p[1]}


@pytest.mark.gpu
@pytest.mark.parametrize("conv", CONVS_601, ids=pe._ids(CONVS_601))
def test_gpu_601_edges(api, ref601, conv):
    """the edge geometries of test_pixfmt_edges.py in every launch form that applies, against the 601 build"""
    import torch
    try:
        for i, g in enumerate(pe.geometries(conv) + pe.chunk_geometries(conv)):
            src = pe.source_bytes(g, 6000 + i)
            want = torch.from_numpy(expect_cs(conv, ref601, g, src)).cuda()
            pe.run_forms(api, conv, g, src, want, pe.FORMS if pe.aligned(g) else (-1,))
    finally:
        api.pixfmt_staged_mode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("conv", CONVS_601, ids=pe._ids(CONVS_601))
def test_gpu_601_wide_and_side_stream(api, ref601, conv):
    """1080p and 8K widths in every launch form, and a side stream whose source arrives after a sleep"""
    import torch
    try:
        for i, (w, h) in enumerate(((1920, 6), (7680, 3))):
            g = pe.make_geo(conv, w, h, pe._a16(conv.li(w)), pe._a16(conv.lo(w)))
            src = pe.source_bytes(g, 6500 + i)
            pe.run_forms(api, conv, g, src, torch.from_numpy(expect_cs(conv, ref601, g, src)).cuda(), pe.FORMS)
    finally:
        api.pixfmt_staged_mode(-1)
    g = pe.make_geo(conv, 50, 5, conv.li(50) + 1, conv.lo(50) + 4, off=(1, 3))
    src = pe.source_bytes(g, 6600)
    want = torch.from_numpy(expect_cs(conv, ref601, g, src)).cuda()
    h_src = torch.from_numpy(pe._source_buffer(g, src)).pin_memory()
    h_dst = torch.from_numpy(np.full(g.off_d + 2 * pe.G + g.dp * g.h, pe.SENT, np.uint8)).pin_memory()
    d_src = torch.full((h_src.numel(),), 0x5A, dtype=torch.uint8, device="cuda")
    d_dst = torch.full((h_dst.numel(),), 0x11, dtype=torch.uint8, device="cuda")

    def launch(s):
        d_src.copy_(h_src, non_blocking=True)
        d_dst.copy_(h_dst, non_blocking=True)
        conv.gpu(api, d_src[g.off_s:g.off_s + g.src_size], d_dst[g.off_d + pe.G:g.off_d + pe.G + g.dp * g.h], g, stream=s)
        return h_src, h_dst

    pe._side_stream(torch, launch)
    pe._assert_same(torch, d_dst[g.off_d:], want, f"{conv.id} side stream")


@pytest.mark.gpu
@pytest.mark.parametrize("key,inc,outc,w,h,seed", golden_cases(), ids=[c[0] for c in golden_cases()])
def test_gpu_601_golden(api, key, inc, outc, w, h, seed):
    """the fixtures of the 601 build: what pins the GPU path where oracle/_ref is absent"""
    gold = util.golden(GOLDEN)
    src = golden_source(inc, w, h, seed)
    got = api.pixfmt_convert(inc, outc, util.dev(src), w, h, cs=CS_601).cpu().numpy()
    assert np.array_equal(got, gold[key]), key


@pytest.mark.gpu
@pytest.mark.parametrize("inc,outc", PAIRS)
def test_gpu_dfl_and_709_equal_the_plain_entry(api, inc, outc):
    import torch
    for i, (w, h) in enumerate(((50, 3), (1921, 2))):
        src = util.dev(util.rng_bytes(util.oracle().orc_vc_get_linesize(w, inc) * h, 77 + i))
        plain = torch.zeros(util.oracle().orc_vc_get_linesize(w, outc) * h, dtype=torch.uint8, device="cuda")
        from ultragrid_b200.codec import vc_get_linesize
        ls_i, ls_o = vc_get_linesize(w, inc), vc_get_linesize(w, outc)
        assert api._L.ugb200_pixfmt_convert(inc, outc, api._ptr(plain), ls_o, api._ptr(src), ls_i, ls_o, h, src.numel(), 0, 8, 16, api._stream()) == 0
        for cs in (CS_DFL, CS_709):
            assert torch.equal(api.pixfmt_convert(inc, outc, src, w, h, cs=cs), plain), (inc, outc, cs)


@pytest.mark.gpu
def test_gpu_invalid_colour_space_writes_nothing(api):
    import torch
    w, h = 64, 2
    src = util.dev(util.rng_bytes(w * 2 * h, 1))
    for cs in (-1, 3, 7, 1 << 20):
        dst = torch.full((w * 3 * h,), 0xCD, dtype=torch.uint8, device="cuda")
        rc = api._L.ugb200_pixfmt_convert_cs(UYVY, RGB, api._ptr(dst), w * 3, api._ptr(src), w * 2, w * 3, h, src.numel(), 0, 8, 16, cs, api._stream())
        torch.cuda.synchronize()
        assert rc == -1 and bool((dst == 0xCD).all()), cs
        with pytest.raises(RuntimeError):
            api.pixfmt_convert(UYVY, RGB, src, w, h, cs=cs)
        planes = [torch.full((w * h * 2,), 0xCD, dtype=torch.uint8, device="cuda") for _ in range(3)]
        rgb = util.dev(util.rng_bytes(w * 3 * h, 2))
        with pytest.raises(RuntimeError):
            api.to_lavc(RGB, "YUV444P", rgb, w, h, planes=planes, cs=cs)
        torch.cuda.synchronize()
        assert all(bool((p == 0xCD).all()) for p in planes), cs
        assert not api._L.ugb200_to_lavc_vid_conv_init_cs(RGB, w, h, tle.AV["YUV444P"], cs)


# ---- GPU: to_lavc ------------------------------------------------------------------------------------------------------------------------------
def gpu_to_lavc_cs(L, torch, inc, fmt, src, w, h, lss, cs, plane_off=0):
    """tle.gpu_to_lavc through ugb200_to_lavc_convert_cs"""
    from ultragrid_b200.api import AvPlanes
    shapes, _ = tle.av_geom(fmt, w, h)
    bufs = [torch.full((2 * tle.GUARD + plane_off + ls * rows,), tle.FILL, dtype=torch.uint8, device="cuda") for ls, (_, rows) in zip(lss, shapes)]
    p = AvPlanes()
    for i, (b, ls) in enumerate(zip(bufs, lss)):
        p.data[i], p.linesize[i] = b.data_ptr() + tle.GUARD + plane_off, ls
    s = torch.from_numpy(np.concatenate([np.zeros(16, np.uint8), src, np.zeros(64, np.uint8)])).cuda()
    rc = L.ugb200_to_lavc_convert_cs(inc, tle.AV[fmt], ctypes.byref(p), s.data_ptr() + 16, w, h, cs, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, [b.cpu().numpy() for b in bufs]


def _lavc_lib():
    L, torch = tle.lib_and_torch()
    L.ugb200_to_lavc_convert_cs.argtypes = [_i, _i, _vp, _vp, _i, _i, _i, _vp]
    L.ugb200_to_lavc_vid_conv_init_cs.restype = _vp
    L.ugb200_to_lavc_vid_conv_init_cs.argtypes = [_i, _i, _i, _i, _i]
    return L, torch


@pytest.mark.gpu
@pytest.mark.parametrize("inc,fmt", tle.to_lavc_pairs() if tle._lib_built() else [])
def test_gpu_to_lavc_601(orc, inc, fmt):
    """every admitted pair under CS_601 == the restatement with the BT.601 sets, sentinel bands included; the YCbCr sources are unchanged"""
    L, torch = _lavc_lib()
    for k, (w, h) in enumerate(tle.TO_SIZES):
        src = tle.make_source(inc, w, h, 700 + k)
        for name, lss, off in tle.plane_modes(fmt, w, h):
            want = ref_to_lavc_cs(inc, fmt, src, w, h, lss, orc)
            rc, got = gpu_to_lavc_cs(L, torch, inc, fmt, src, w, h, lss, CS_601, off)
            assert rc == 0, (w, h, name, rc)
            tle.assert_planes(got, want, off, (w, h, name))
        lss = tle.plane_modes(fmt, w, h)[0][1]
        for cs in (CS_DFL, CS_709):
            rc, got = gpu_to_lavc_cs(L, torch, inc, fmt, src, w, h, lss, cs)
            assert rc == 0
            tle.assert_planes(got, tle.ref_to_lavc(inc, fmt, src, w, h, lss, orc), 0, (w, h, cs))


@pytest.mark.gpu
@pytest.mark.parametrize("inc,fmt", tle.to_lavc_pairs() if tle._lib_built() else [])
def test_gpu_to_lavc_601_hook_host_and_device_frame(orc, inc, fmt):
    from ultragrid_b200.api import AvPlanes
    L, torch = _lavc_lib()
    w, h = 97, 5
    st = L.ugb200_to_lavc_vid_conv_init_cs(inc, w, h, tle.AV[fmt], CS_601)
    assert st
    try:
        src = tle.make_source(inc, w, h, 3)
        dev = torch.from_numpy(src).cuda()
        for frame, is_dev in ((src.ctypes.data, 0), (dev.data_ptr(), 1)):
            pp = L.ugb200_to_lavc_vid_conv(st, frame, is_dev)
            assert pp, is_dev
            p = AvPlanes.from_address(pp)
            shapes, _ = tle.av_geom(fmt, w, h)
            lss = [p.linesize[i] for i in range(len(shapes))]
            want = ref_to_lavc_cs(inc, fmt, src, w, h, lss, orc)
            for i, (b, wr) in enumerate(zip(want.buf, want.wr)):
                host = np.zeros(b.size, np.uint8)
                assert L.cuda_wrapper_memcpy(ctypes.c_void_p(host.ctypes.data), ctypes.c_void_p(p.data[i]), host.size, 1) == 0
                assert np.array_equal(host.reshape(b.shape)[wr], b[wr]), (is_dev, i)
    finally:
        hs = _vp(st)
        L.ugb200_to_lavc_vid_conv_destroy(ctypes.byref(hs))
