"""Interlaced video: the linear-blend deinterlacers and field-order converters on the GPU (interlace_kernels.cu).

CPU: the numpy restatement (interlace_ref.py) equals the unmodified reference objects byte for byte, with two
sentinel fills of dst that reveal which bytes the reference writes; the golden fixtures stand in for the reference
where it is not built.  GPU: the kernels equal the restatement's contract form everywhere, with sentinels around
every buffer, and the reference where it is present.
"""
import ctypes
import os

import numpy as np
import pytest

import interlace_ref as R
import util
from ultragrid_b200.codec import vc_get_linesize

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "interlace_golden.npz")
FILLS = (0x00, 0xA5)
WIDTHS = (1, 2, 3, 5, 6, 7, 47, 48, 1918, 1920)
RAW_LS = (14, 17, 44, 52, 100, 172, 300, 1004)  # not multiples of 16, 36 or 128
LINES = (1, 2, 3, 4, 5, 6, 7)
LEGACY_LS = (16, 17, 31, 36, 40, 52, 3840, 5760, 23040)


def _bind(lib):
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.vc_deinterlace_ex.argtypes = [ctypes.c_int, vp, sz, vp, sz, sz]
    lib.vc_deinterlace_ex.restype = ctypes.c_bool
    lib.vc_deinterlace.argtypes = [vp, ctypes.c_long, ctypes.c_int]
    lib.vc_deinterlace.restype = None
    for n in ("il_upper_to_merged", "il_merged_to_upper"):
        getattr(lib, n).argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, vp]
        getattr(lib, n).restype = None
    lib.get_bits_per_component.argtypes = [ctypes.c_int]
    lib.is_codec_opaque.argtypes = [ctypes.c_int]
    lib.is_codec_opaque.restype = ctypes.c_bool
    return lib


@pytest.fixture(scope="module")
def ref():
    lib = util.ref_cpu()
    if lib is None:
        pytest.skip("oracle/_ref/libugref.so not built (reference tree absent)")
    return _bind(lib)


def ref_ex(ref, codec, src, L, dst, pitch, lines, in_place=False):
    """the reference on copies; returns the new dst or None when it refuses"""
    if in_place:
        m = src.copy()
        ok = ref.vc_deinterlace_ex(codec, m.ctypes.data, L, m.ctypes.data, L, lines)
        return m if ok else None
    d = dst.copy()
    ok = ref.vc_deinterlace_ex(codec, src.ctypes.data, L, d.ctypes.data, pitch, lines)
    return d if ok else None


def ref_legacy(ref, data, L, lines, offset):
    """vc_deinterlace at a 64-byte-aligned address + offset; the bytes around the frame must stay"""
    raw = np.full(L * lines + 256, 0x5A, np.uint8)
    base = (-raw.ctypes.data) % 64 + offset
    raw[base:base + L * lines] = data
    ref.vc_deinterlace(raw.ctypes.data + base, L, lines)
    assert (raw[:base] == 0x5A).all() and (raw[base + L * lines:] == 0x5A).all(), "reference wrote outside the frame"
    return raw[base:base + L * lines].copy()


def ex_cases():
    """(codec, L, lines, pitch pad) for every non-opaque codec: codec widths, raw line sizes, lines 1-7"""
    for c in R.NON_OPAQUE:
        sizes = sorted({vc_get_linesize(w, c) for w in WIDTHS} | set(RAW_LS))
        for L in sizes:
            for lines in LINES:
                yield c, L, lines, 0 if lines % 2 else 20


def src_for(c, L, lines, seed):
    return util.rng_bytes(L * lines, seed)  # random bytes: v210 / R10k padding bits included


# ---- CPU: restatement vs reference ---------------------------------------------------------------------------
def test_codec_table_matches_reference(ref):
    assert [ref.get_bits_per_component(c) for c in range(1, R.CODEC_COUNT)] == R.BITS[1:]
    assert [c for c in range(1, R.CODEC_COUNT) if not ref.is_codec_opaque(c)] == list(R.NON_OPAQUE)


@pytest.mark.parametrize("codec", range(1, R.CODEC_COUNT))
def test_ex_acceptance_matches_reference(ref, codec):
    src = util.rng_bytes(64 * 3, codec)
    for lines in (1, 3):
        got = ref_ex(ref, codec, src, 64, np.zeros(64 * 3, np.uint8), 64, lines)
        want = R.deinterlace_ex(codec, src, 64, np.zeros(64 * 3, np.uint8), 64, lines)
        assert (got is None) == (want is None), (codec, lines)
        if got is not None:
            assert np.array_equal(got, want)


@pytest.mark.parametrize("codec", R.NON_OPAQUE)
def test_ex_restatement_equals_reference(ref, codec):
    n = 0
    for c, L, lines, pad in ex_cases():
        if c != codec:
            continue
        src = src_for(c, L, lines, n)
        pitch = L + pad
        for fill in FILLS:
            dst = np.full(pitch * lines + 32, fill, np.uint8)
            got = ref_ex(ref, c, src, L, dst, pitch, lines)
            want = R.deinterlace_ex(c, src, L, dst, pitch, lines)
            assert (got is None) == (want is None), (c, L, lines)
            if got is not None:
                assert np.array_equal(got, want), (c, L, lines, fill, np.flatnonzero(got != want)[:8])
        got = ref_ex(ref, c, src, L, None, L, lines, in_place=True)
        want = R.deinterlace_ex(c, src, L, src, L, lines)
        assert (got is None) == (want is None)
        if got is not None:
            assert np.array_equal(got, want), ("in place", c, L, lines)
        n += 1


@pytest.mark.parametrize("codec,w", [(R.UYVY, 1920), (R.v210, 1920), (R.RG48, 1918), (R.R12L, 1920), (R.R10k, 1918)])
@pytest.mark.parametrize("lines", (1080, 1081))
def test_ex_full_frames_equal_reference(ref, codec, w, lines):
    L = vc_get_linesize(w, codec)
    src = util.rng_bytes(L * lines, w + lines)
    for fill in FILLS:
        dst = np.full(L * lines, fill, np.uint8)
        assert np.array_equal(ref_ex(ref, codec, src, L, dst, L, lines), R.deinterlace_ex(codec, src, L, dst, L, lines))
    assert np.array_equal(ref_ex(ref, codec, src, L, None, L, lines, in_place=True), R.deinterlace_ex(codec, src, L, src, L, lines))


def test_opaque_codecs_blend_compressed_bytes_in_the_reference(ref):
    src = util.rng_bytes(100 * 4, 3)
    got = ref_ex(ref, 13, src, 100, np.zeros(400, np.uint8), 100, 4)  # JPEG, depth 8
    assert got is not None and np.array_equal(got, R.deinterlace_ex(13, src, 100, np.zeros(400, np.uint8), 100, 4))
    assert R.deinterlace_ex(13, src, 100, np.zeros(400, np.uint8), 100, 4, contract=True) is None


def written(c, L, lines, pitch, contract):
    """mask of dst bytes a call writes, from two sentinel fills of the restatement"""
    src = src_for(c, L, lines, 99)
    a = R.deinterlace_ex(c, src, L, np.full(pitch * lines, 0x00, np.uint8), pitch, lines, contract)
    b = R.deinterlace_ex(c, src, L, np.full(pitch * lines, 0xFF, np.uint8), pitch, lines, contract)
    return (a == b), a


@pytest.mark.parametrize("codec,L", [(R.RG48, vc_get_linesize(1918, R.RG48)), (R.Y216, 1004), (R.Y416, 172), (R.R12L, vc_get_linesize(1920, R.R12L)),
                                     (R.R12L, 36 * 7 + 8), (R.R12L, 36 * 6), (R.v210, 1004), (R.UYVY, 1918 * 2)])
def test_deliberate_differences_are_exactly_the_quirk_list(codec, L):
    lines, pitch = 5, L + 12
    wr_ref, ref_out = written(codec, L, lines, pitch, False)
    wr_ctr, ctr_out = written(codec, L, lines, pitch, True)
    row_ref, row_ctr = np.zeros(pitch, bool), np.zeros(pitch, bool)
    if R.BITS[codec] == 16:
        row_ref[:L // 16 * 16 if L >= 16 else L // 2 * 2] = True  # whole 16-byte chunks only
        row_ctr[:L // 2 * 2] = True
    elif codec == R.R12L:
        g = L // 36
        row_ref[:32 * g if g % 3 == 0 else max(32 * g - 4, 0)] = True  # the first 8 of every 9 words, last word pending
        row_ctr[:36 * g] = True
    elif codec in (R.v210, R.R10k):
        row_ref[:L // 16 * 16] = row_ctr[:L // 16 * 16] = True
    else:
        row_ref[:L] = row_ctr[:L] = True
    assert np.array_equal(wr_ref.reshape(lines, pitch)[:-1], np.tile(row_ref, (lines - 1, 1)))
    assert np.array_equal(wr_ctr.reshape(lines, pitch)[:-1], np.tile(row_ctr, (lines - 1, 1)))
    # wherever the reference writes, the contract writes the same bytes
    assert np.array_equal(ctr_out[wr_ref], ref_out[wr_ref])
    # on the rest it holds the per-sample blend of the two rows (the 16-bit / 12-bit samples, whole)
    src = src_for(codec, L, lines, 99)
    extra = wr_ctr & ~wr_ref
    if extra.any():
        rows = src.reshape(lines, L)
        for y in range(lines - 1):
            e = np.flatnonzero(extra.reshape(lines, pitch)[y])
            if codec == R.R12L:
                blend = R._r12l_pack(R._avg(R._r12l_unpack(rows[y, :L // 36 * 36]), R._r12l_unpack(rows[y + 1, :L // 36 * 36])))
            else:
                blend = R._avg(rows[y, :L // 2 * 2].view(np.uint16), rows[y + 1, :L // 2 * 2].view(np.uint16)).astype(np.uint16).view(np.uint8)
            assert np.array_equal(ctr_out.reshape(lines, pitch)[y, e], blend[e])
    else:
        assert codec not in (R.RG48, R.Y216, R.Y416, R.R12L) or L < 16


def test_legacy_restatement_equals_reference(ref):
    for L in LEGACY_LS:
        for lines in LINES + (8, 9, 12, 13):
            if L * lines > 23040 * 13:
                continue
            for off in (0, 1, 4):
                data = util.rng_bytes(L * lines, L + lines + off)
                assert np.array_equal(ref_legacy(ref, data, L, lines, off), R.deinterlace(data, L, lines)), (L, lines, off)


@pytest.mark.parametrize("lines", (1080, 1081))
def test_legacy_restatement_equals_reference_full_frames(ref, lines):
    for L in (3840, 5760, 3844):
        data = util.rng_bytes(L * lines, lines)
        assert np.array_equal(ref_legacy(ref, data, L, lines, 0), R.deinterlace(data, L, lines))


def test_il_restatement_equals_reference(ref):
    for L in (1, 3, 16, 3840):
        for h in (1, 2, 3, 4, 7, 1080, 1081):
            src = util.rng_bytes(L * h, L + h)
            for name in ("il_upper_to_merged", "il_merged_to_upper"):
                d = np.zeros(L * h, np.uint8)
                getattr(ref, name)(d.ctypes.data, src.ctypes.data, L, h, None)
                assert np.array_equal(d, getattr(R, name)(src, L, h)), (name, L, h)
                m = src.copy()
                getattr(ref, name)(m.ctypes.data, m.ctypes.data, L, h, None)
                assert np.array_equal(m, d)


def test_il_round_trip_is_identity():
    for L, h in ((5, 1), (7, 6), (3, 9)):
        src = util.rng_bytes(L * h, h)
        assert np.array_equal(R.il_merged_to_upper(R.il_upper_to_merged(src, L, h), L, h), src)


# ---- golden fixtures (made from the reference by tests/golden/make_interlace_golden.py) ------------------------
def test_restatement_equals_golden():
    g = util.golden(GOLDEN)
    n = 0
    for k in g.files:
        if k.endswith("_meta"):
            p = k[:-5]
            kind, *meta = g[k].tolist()
            if kind == 0:
                c, L, lines, pitch, fill = meta
                dst = np.full(pitch * lines, fill, np.uint8)
                assert np.array_equal(R.deinterlace_ex(c, g[p + "_src"], L, dst, pitch, lines), g[p + "_out"]), p
            elif kind == 1:
                L, lines = meta[:2]
                assert np.array_equal(R.deinterlace(g[p + "_src"], L, lines), g[p + "_out"]), p
            else:
                L, h = meta[:2]
                fn = R.il_upper_to_merged if kind == 2 else R.il_merged_to_upper
                assert np.array_equal(fn(g[p + "_src"], L, h), g[p + "_out"]), p
            n += 1
    assert n >= 40


# ---- GPU ----------------------------------------------------------------------------------------------------
GUARD = 64
SENT = 0x3C


def gpu_ex(codec, src, L, dst_init, pitch, lines, in_place=False):
    """ugb200_vc_deinterlace_ex between sentinels; returns (rc, dst bytes)"""
    from ultragrid_b200 import _lib, api
    import torch
    lib = _lib.load()
    s = util.Guarded(src.size, 0, SENT, src, GUARD)
    d = s if in_place else util.Guarded(dst_init.size, 0, SENT, dst_init, GUARD)
    rc = lib.ugb200_vc_deinterlace_ex(codec, ctypes.c_void_p(s.view.data_ptr()), L, ctypes.c_void_p(d.view.data_ptr()), pitch, lines, api._stream())
    torch.cuda.synchronize()
    got = d.check_outside()
    if not in_place:
        assert np.array_equal(s.check_outside(), src), "source changed"
    return rc, got


@pytest.mark.gpu
@pytest.mark.parametrize("codec", R.NON_OPAQUE)
def test_gpu_ex_exact(codec):
    ref = util.ref_cpu()
    ref = _bind(ref) if ref is not None else None
    n = 0
    for c, L, lines, pad in ex_cases():
        if c != codec:
            continue
        src = src_for(c, L, lines, n)
        n += 1
        pitch = L + pad
        word = c in (R.v210, R.R10k, R.R12L)
        align = 4 if word else 2 if R.BITS[c] == 16 else 1
        for fill in FILLS:
            dst = np.full(pitch * (lines - 1) + L, fill, np.uint8)
            rc, got = gpu_ex(c, src, L, dst, pitch, lines)
            want = R.deinterlace_ex(c, src, L, dst, pitch, lines, contract=True)
            if L % align or pitch % align:
                assert rc == -1 and np.array_equal(got, dst), (c, L, lines)
                continue
            if want is None:
                assert rc == -4 and np.array_equal(got, dst), (c, L, lines)
                continue
            assert rc == 0, (c, L, lines, rc)
            assert np.array_equal(got, want), (c, L, lines, fill, np.flatnonzero(got != want)[:8])
            if ref is not None and fill == FILLS[0]:
                r = ref_ex(ref, c, src, L, dst, pitch, lines)
                wr = written(c, L, lines, pitch, False)[0][:dst.size]
                assert np.array_equal(got[wr], r[wr])
        if L % align == 0 and R.deinterlace_ex(c, src, L, src, L, lines, contract=True) is not None:
            rc, got = gpu_ex(c, src, L, None, L, lines, in_place=True)
            assert rc == 0 and np.array_equal(got, R.deinterlace_ex(c, src, L, src, L, lines, contract=True)), ("in place", c, L, lines)


@pytest.mark.gpu
@pytest.mark.parametrize("codec,w,h", [(R.UYVY, 1920, 1080), (R.UYVY, 1920, 1081), (R.v210, 1920, 1080), (R.RG48, 1918, 1080),
                                       (R.R12L, 1920, 1080), (R.R10k, 1918, 1081), (R.Y216, 1920, 1080), (R.RGB, 3840, 2160),
                                       (R.UYVY, 7680, 4320), (R.R12L, 3840, 2161), (R.v210, 7680, 4320)])
def test_gpu_ex_frames(codec, w, h):
    L = vc_get_linesize(w, codec)
    src = util.rng_bytes(L * h, w + h)
    dst = np.full(L * h, 0xA5, np.uint8)
    rc, got = gpu_ex(codec, src, L, dst, L, h)
    want = R.deinterlace_ex(codec, src, L, dst, L, h, contract=True)
    assert rc == 0 and np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    rc, got_ip = gpu_ex(codec, src, L, None, L, h, in_place=True)
    assert rc == 0 and np.array_equal(got_ip, R.deinterlace_ex(codec, src, L, src, L, h, contract=True))
    ref = util.ref_cpu()
    if ref is not None and h <= 2161:
        r = ref_ex(_bind(ref), codec, src, L, dst, L, h)
        wr = written(codec, L, h, L, False)[0]
        assert np.array_equal(got[wr], r[wr])


@pytest.mark.gpu
def test_gpu_ex_side_stream_and_api():
    import torch
    from ultragrid_b200 import api
    L, h = vc_get_linesize(1920, R.UYVY), 1080
    src = util.rng_bytes(L * h, 5)
    want = R.deinterlace_ex(R.UYVY, src, L, np.zeros(L * h, np.uint8), L, h, contract=True)
    s = torch.cuda.Stream()
    t = util.dev(src)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = api.deinterlace_ex(R.UYVY, t, L, h, stream=s)
        api.deinterlace_ex(R.UYVY, t, L, h, dst=t, stream=s)  # in place, after the out-of-place read on the same stream
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)
    assert np.array_equal(t.cpu().numpy(), want)


@pytest.mark.gpu
def test_gpu_ex_refusals_write_nothing():
    from ultragrid_b200 import _lib, api
    import torch
    lib = _lib.load()
    L, lines = 384, 6
    src = util.rng_bytes(L * lines, 1)

    def call(codec, s_off, L_, d_off, pitch, n, writes=False):
        buf = torch.full((L * lines * 3 + 256,), SENT, dtype=torch.uint8, device="cuda")
        buf[64:64 + src.size] = torch.from_numpy(src).cuda()
        before = buf.cpu().numpy()
        rc = lib.ugb200_vc_deinterlace_ex(codec, ctypes.c_void_p(buf.data_ptr() + s_off), L_, ctypes.c_void_p(buf.data_ptr() + d_off), pitch, n,
                                          api._stream())
        torch.cuda.synchronize()
        assert np.array_equal(buf.cpu().numpy(), before) != writes, (codec, s_off, d_off, pitch, n)
        return rc

    far = 64 + L * lines + 64
    assert call(13, 64, L, far, L, lines) == -4           # JPEG: opaque
    assert call(R.DVS10, 64, L, far, L, lines) == -4      # no DVS10 branch
    assert call(R.UYVY, 64, L, far, L, 0) == -1           # lines == 0
    assert call(R.UYVY, 64, L, far, L - 2, lines) == -1   # dst_pitch < src_linesize
    assert call(R.UYVY, 64, L, 64 + L, L, lines) == -1    # partial overlap
    assert call(R.UYVY, 64, L, 64, L + 4, lines) == -1    # same start, other pitch
    assert call(R.RG48, 65, L, far, L, lines) == -1       # 16-bit at an odd address
    assert call(R.v210, 64, L, far + 2, L, lines) == -1   # word codec at a 2-byte address
    assert call(R.R12L, 64, L, far, L + 2, lines) == -1   # word codec, pitch not a multiple of 4
    assert call(R.R10k, 64, L - 2, far, L, lines) == -1   # word codec, line size not a multiple of 4
    assert lib.ugb200_vc_deinterlace(None, 64, 8, api._stream()) == -1
    assert call(R.UYVY, 64, L, far, L, lines, writes=True) == 0  # and the good call works


@pytest.mark.gpu
def test_gpu_legacy_exact():
    import torch
    from ultragrid_b200 import _lib, api
    lib = _lib.load()
    ref = util.ref_cpu()
    ref = _bind(ref) if ref is not None else None
    for L in LEGACY_LS:
        for lines in LINES + (8, 9, 12, 13, 1080, 1081):
            if L * lines > 23040 * 13 and lines < 1080:
                continue
            for off in (0, 1, 4):
                data = util.rng_bytes(L * lines, L * 7 + lines + off)
                buf = util.Guarded(data.size, off, SENT, data, GUARD)
                assert lib.ugb200_vc_deinterlace(ctypes.c_void_p(buf.view.data_ptr()), L, lines, api._stream()) == 0
                torch.cuda.synchronize()
                got = buf.check_outside()
                want = R.deinterlace(data, L, lines)
                assert np.array_equal(got, want), (L, lines, off, np.flatnonzero(got != want)[:8])
                if ref is not None and lines < 1080:
                    assert np.array_equal(want, ref_legacy(ref, data, L, lines, off))
    assert lib.ugb200_vc_deinterlace(ctypes.c_void_p(buf.buf.data_ptr() + GUARD), 15, 8, api._stream()) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,bpp", [(7680, 4320, 2), (3840, 2160, 3), (1919, 1081, 3)])
def test_gpu_legacy_frames(w, h, bpp):
    from ultragrid_b200 import api
    data = util.rng_bytes(w * bpp * h, w)
    t = util.dev(data)
    api.deinterlace(t, w * bpp, h)
    assert np.array_equal(t.cpu().numpy(), R.deinterlace(data, w * bpp, h))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ("il_upper_to_merged", "il_merged_to_upper"))
def test_gpu_il_exact(name):
    import torch
    from ultragrid_b200 import _lib, api
    lib = _lib.load()
    fn = getattr(lib, "ugb200_" + name)
    for L in (1, 3, 16, 17, 3840, 7680 * 2):
        for h in (1, 2, 3, 4, 7, 1080, 1081):
            src = util.rng_bytes(L * h, L + h)
            want = getattr(R, name)(src, L, h)
            for off in (0, 1, 4):
                s = util.Guarded(src.size, off, SENT, src, GUARD)
                d = util.Guarded(L * h, 0, SENT, np.zeros(L * h, np.uint8), GUARD)
                sp, dp = ctypes.c_void_p(s.view.data_ptr()), ctypes.c_void_p(d.view.data_ptr())
                assert fn(dp, sp, L, h, api._stream()) == 0
                assert fn(sp, sp, L, h, api._stream()) == 0
                torch.cuda.synchronize()
                assert np.array_equal(d.check_outside(), want), (name, L, h, off)
                assert np.array_equal(s.check_outside(), want), ("in place", name, L, h, off)
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    assert fn(ctypes.c_void_p(buf.data_ptr() + 16), ctypes.c_void_p(buf.data_ptr()), 64, 8, api._stream()) == -1  # partial overlap
    assert (buf == 0).all()


@pytest.mark.gpu
def test_gpu_il_round_trip_on_a_side_stream():
    import torch
    from ultragrid_b200 import api
    for L, h in ((3840, 1080), (7680 * 2, 4321), (5, 7)):
        src = util.rng_bytes(L * h, h)
        t = util.dev(src)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            api.il_merged_to_upper(t, L, h, stream=s)
            up = t.clone()
            api.il_upper_to_merged(t, L, h, stream=s)
        s.synchronize()
        assert np.array_equal(up.cpu().numpy(), R.il_merged_to_upper(src, L, h))
        assert np.array_equal(t.cpu().numpy(), src)


@pytest.mark.gpu
def test_gpu_matches_golden():
    import torch
    from ultragrid_b200 import api
    g = util.golden(GOLDEN)
    for k in g.files:
        if not k.endswith("_meta"):
            continue
        p = k[:-5]
        kind, *meta = g[k].tolist()
        src, want = g[p + "_src"], g[p + "_out"]
        if kind == 0:
            c, L, lines, pitch, fill = meta
            if R.BITS[c] == 16 or c == R.R12L:
                continue  # the reference leaves those tails unwritten; checked against the restatement above
            if (c in (R.v210, R.R10k) and (L % 4 or pitch % 4)):
                continue
            dst = util.dev(np.full(pitch * lines, fill, np.uint8))
            api.deinterlace_ex(c, util.dev(src), L, lines, dst=dst, dst_pitch=pitch)
            assert np.array_equal(dst.cpu().numpy(), want), p
        elif kind == 1:
            L, lines = meta[:2]
            t = util.dev(src)
            api.deinterlace(t, L, lines)
            assert np.array_equal(t.cpu().numpy(), want), p
        else:
            L, h = meta[:2]
            t = util.dev(src)
            (api.il_upper_to_merged if kind == 2 else api.il_merged_to_upper)(t, L, h)
            torch.cuda.synchronize()
            assert np.array_equal(t.cpu().numpy(), want), p
