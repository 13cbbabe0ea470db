"""Field-rate postprocessors on the GPU: double_framerate (with and without `:d`), deinterlace_bob,
deinterlace_linear and interlace (interlace_kernels.cu, ugb200_pp_*).

CPU: the numpy restatement (field_rate_ref.py) equals the unmodified temporal-deint.c and interlace.c on the bytes
[0, L) of every row, with two sentinel fills of dst that show which bytes the reference writes; the module's own
init / getf / postprocess sequence pins the call-0 / call-1 and prev / cur model; mutants that "fix" a quirk fail.
The golden fixtures stand in for the reference where it is not built.  GPU: the kernels equal the restatement's
contract form everywhere, with sentinels around every buffer.
"""
import ctypes
import os

import numpy as np
import pytest

import field_rate_ref as F
import interlace_ref as IR
import util
from ultragrid_b200.codec import vc_get_linesize

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "field_rate_golden.npz")
FILLS = (0x00, 0xA5)
CODECS = (IR.UYVY, IR.RGB, IR.RGBA, IR.I420, IR.DVS10, IR.RG48, IR.Y216, IR.Y416, IR.v210, IR.R10k, IR.R12L)
WIDTHS = (1, 2, 3, 5, 7, 8, 13, 47, 49, 100, 131)
HEIGHTS = (2, 3, 4, 5, 6, 7)
DF, BOB, LINEAR = 0, 1, 2


# ---- the reference ---------------------------------------------------------------------------------------------
def _bind(lib):
    vp, i = ctypes.c_void_p, ctypes.c_int
    lib.ref_tdi_perform.argtypes = [i, i, i, i, vp, vp, i, i, vp, i]
    lib.ref_tdi_perform.restype = None
    lib.ref_tdi_avg_lines.argtypes = [i, ctypes.c_size_t, vp, vp, vp]
    lib.ref_tdi_sequence.argtypes = [i, ctypes.c_char_p, i, i, i, vp, i, vp, i]
    lib.ref_interlace_weave.argtypes = [i, i, i, vp, vp, vp, i]
    lib.ref_interlace_sequence.argtypes = [i, i, i, vp, i, vp, i]
    return lib


def ref_lib():
    return util.ref_lib("libfield_rate_ref.so", _bind)


@pytest.fixture(scope="module")
def ref():
    lib = ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libfield_rate_ref.so not built (reference tree absent)")
    return lib


class Slack:
    """a harness-owned copy of `data` with 3 rows + 64 bytes of slack on both sides (the reference writes past rows)"""

    def __init__(self, data, row, fill=0):
        self.pad = 3 * row + 64
        self.buf = np.full(data.size + 2 * self.pad, fill, np.uint8)
        self.buf[self.pad:self.pad + data.size] = data
        self.n = data.size

    @property
    def ptr(self):
        return self.buf.ctypes.data + self.pad

    def get(self):
        return self.buf[self.pad:self.pad + self.n].copy()

    def outside(self):
        return np.concatenate([self.buf[:self.pad], self.buf[self.pad + self.n:]])


def ref_run(ref, algo, c, w, h, call, prev, cur, dst, pitch, d=0):
    """perform_* on harness copies; returns (dst bytes of the frame, dst bytes around it)"""
    L = vc_get_linesize(w, c)
    row = max(L, pitch)
    p, q, o = Slack(prev, row, 0x5A), Slack(cur, row, 0x5A), Slack(dst, row, fill=int(dst[0]) if dst.size else 0)
    if algo == 3:
        ref.ref_interlace_weave(c, w, h, q.ptr, p.ptr, o.ptr, pitch)  # `first` = cur, `second` = prev
    else:
        ref.ref_tdi_perform(algo, c, w, h, p.ptr, q.ptr, call, d, o.ptr, pitch)
    return o.get(), o.outside()


def model(algo, c, L, h, call, prev, cur, dst, pitch, d=0, contract=False):
    if algo == DF:
        return F.double_framerate(c, prev, cur, L, h, call, dst, pitch, d, contract)
    if algo == BOB:
        return F.bob(cur, L, h, call, dst, pitch, contract)
    if algo == LINEAR:
        return F.linear(c, cur, L, h, call, dst, pitch, contract)
    return F.interlace(cur, prev, L, h, dst, pitch, contract)


def frame_mask(L, h, pitch, blend_all=False):
    """the bytes the restatement answers for: [0, L) of rows [0, h); `:d` off pitch L also blends [0, L*h)"""
    m = np.zeros((h, pitch), bool)
    m[:, :L] = True
    m = m.reshape(-1)
    if blend_all:
        m[:L * h] = True
    return m


def cases():
    for algo in (DF, BOB, LINEAR, 3):
        for c in CODECS:
            for w in WIDTHS:
                for h in HEIGHTS:
                    for call in ((0, 1) if algo != 3 else (0,)):
                        for d in ((0, 1) if algo == DF else (0,)):
                            yield algo, c, w, h, call, d


def inputs(L, h, seed):
    return util.rng_bytes(L * h, seed), util.rng_bytes(L * h, seed + 1)


# ---- CPU: restatement vs reference -------------------------------------------------------------------------------
@pytest.mark.parametrize("algo", (DF, BOB, LINEAR, 3), ids=("df", "bob", "linear", "interlace"))
def test_restatement_equals_reference(ref, algo):
    n = 0
    for a, c, w, h, call, d in cases():
        if a != algo:
            continue
        L = vc_get_linesize(w, c)
        prev, cur = inputs(L, h, n)
        n += 1
        for pad in (0, 20):
            pitch = L + pad
            for fill in FILLS:
                dst = np.full(pitch * h, fill, np.uint8)
                got, _ = ref_run(ref, algo, c, w, h, call, prev, cur, dst, pitch, d)
                want = model(algo, c, L, h, call, prev, cur, dst, pitch, d)
                m = frame_mask(L, h, pitch, algo == DF and d and pad)
                assert np.array_equal(got[m], want[m]), (algo, c, w, L, h, call, d, pad, fill, np.flatnonzero((got != want) & m)[:8])
    assert n > 100


@pytest.mark.parametrize("algo,codec,w", [(DF, IR.UYVY, 1920), (DF, IR.v210, 1920), (BOB, IR.RGB, 1918), (LINEAR, IR.UYVY, 1920),
                                          (LINEAR, IR.v210, 1920), (LINEAR, IR.RG48, 1918), (LINEAR, IR.R10k, 1918), (LINEAR, IR.R12L, 1920),
                                          (3, IR.UYVY, 1920)])
@pytest.mark.parametrize("h", (1080, 1081))
def test_restatement_equals_reference_full_frames(ref, algo, codec, w, h):
    L = vc_get_linesize(w, codec)
    prev, cur = inputs(L, h, w + h)
    for call in ((0, 1) if algo != 3 else (0,)):
        for d in ((0, 1) if algo == DF else (0,)):
            dst = np.full(L * h, 0xA5, np.uint8)
            got, _ = ref_run(ref, algo, codec, w, h, call, prev, cur, dst, L, d)
            assert np.array_equal(got, model(algo, codec, L, h, call, prev, cur, dst, L, d)), (algo, call, d)


RAW_LS = (4, 6, 8, 12, 20, 36, 44, 48, 52, 100, 128, 140, 172, 252, 260, 300, 1004)  # off multiples of 16, 36 and 256


@pytest.mark.parametrize("codec", CODECS)
def test_avg_lines_at_raw_line_sizes(ref, codec):
    """avg_lines alone at line sizes no width gives: bytes written (two fills) and their values"""
    for L in RAW_LS:
        if (IR.BITS[codec] == 16 and L % 2) or (codec in (IR.v210, IR.R10k, IR.R12L) and L % 4):
            continue
        a, b = util.rng_bytes(L * 4, L), util.rng_bytes(L * 4, L + 1)  # R10k reads 4 x L
        want = F.avg_lines(codec, a[:L], b[:L])
        for fill in FILLS:
            d = np.full(L * 4 + 64, fill, np.uint8)
            ok = ref.ref_tdi_avg_lines(codec, L, a.ctypes.data, b.ctypes.data, d.ctypes.data)
            assert bool(ok) == (want is not None), (codec, L)
            if want is not None:
                assert np.array_equal(d[:want.size], want), (codec, L, np.flatnonzero(d[:want.size] != want)[:8])
                assert (d[want.size:L] == fill).all(), (codec, L, "bytes after the blended ones must stay")


def test_module_sequence_pins_the_call_and_buffer_model(ref):
    """init / reconfigure / getf / postprocess of the module itself over f1..f5, both calls each, `nodelay`"""
    for algo in (DF, BOB, LINEAR):
        for c, w, h in ((IR.UYVY, 24, 7), (IR.UYVY, 40, 8), (IR.v210, 48, 6), (IR.v210, 96, 9)):
            L = vc_get_linesize(w, c)
            frames = [util.rng_bytes(L * h, 40 + i + algo) for i in range(5)]
            pitch = L + 8
            out = np.full(2 * 5 * pitch * h, 0x77, np.uint8)
            assert ref.ref_tdi_sequence(algo, b"nodelay", c, w, h, np.concatenate(frames).ctypes.data, 5, out.ctypes.data, pitch) == 0
            out = out.reshape(10, pitch * h)
            for i in range(5):
                # the module's buffers start as malloc'd memory: before f2 there is no prev, so skip f1's call 0
                prev = frames[i - 1] if i else None
                for call in (0, 1):
                    if prev is None and call == 0 and algo == DF:
                        continue
                    want = model(algo, c, L, h, call, prev, frames[i], out[2 * i + call], pitch)
                    m = frame_mask(L, h, pitch)
                    assert np.array_equal(out[2 * i + call][m], want[m]), (algo, c, w, h, i, call)


def test_interlace_sequence_pins_the_buffer_model(ref):
    for c, w, h in ((IR.UYVY, 24, 7), (IR.v210, 48, 6)):
        L = vc_get_linesize(w, c)
        frames = [util.rng_bytes(L * h, 60 + i) for i in range(4)]
        out = np.zeros(2 * L * h, np.uint8)
        assert ref.ref_interlace_sequence(c, w, h, np.concatenate(frames).ctypes.data, 4, out.ctypes.data, L) == 2
        for k in range(2):
            want = F.interlace(frames[2 * k], frames[2 * k + 1], L, h, np.zeros(L * h, np.uint8), L)
            assert np.array_equal(out[k * L * h:(k + 1) * L * h], want)


# ---- the deliberate differences (DESIGN.md §8) -------------------------------------------------------------------
def test_reference_writes_outside_the_frame_only_where_listed(ref):
    """quirks 2, 3 and 6: the reference's writes past L or past row h-1 are the listed ones and no others; the
    contract never writes there"""
    for algo, c, w, h, call, d in cases():
        if w not in (5, 47) or h not in (4, 5):
            continue
        L = vc_get_linesize(w, c)
        prev, cur = inputs(L, h, w + h)
        pitch = L + 20
        dst = np.zeros(pitch * h, np.uint8)
        got, around = ref_run(ref, algo, c, w, h, call, prev, cur, dst, pitch, d)
        pad = ~frame_mask(L, h, pitch, algo == DF and d)
        wrote_pad = bool((got[pad] != 0).any())
        wrote_after = bool(around.any())  # slack is 0-filled; the slack before the frame is never written
        linear_avg = algo == LINEAR and not IR.opaque(c) and (IR.BITS[c] in (8, 16) or c == IR.R10k) and h > 2 + call
        df_row_h = algo == DF and call == 0 and h % 2
        if IR.BITS[c] in (8, 16) and linear_avg:
            assert wrote_pad == (L % 16 != 0), (algo, c, w, h, call)  # rounded up to 16 bytes
        elif c == IR.R10k and linear_avg:
            assert wrote_pad or wrote_after  # 4 x L
        elif df_row_h:
            assert wrote_after and not wrote_pad, (c, w, h)  # row h from prev row h
        else:
            assert not wrote_pad and not wrote_after, (algo, c, w, h, call, d)
        want = model(algo, c, L, h, call, prev, cur, dst, pitch, d, contract=True)
        if want is not None:
            assert not want[pad].any()
        assert around[:3 * max(L, pitch) + 64].sum() == 0


def test_refusals_in_the_contract():
    L, h = 64, 4
    prev, cur = inputs(L, h, 1)
    dst = np.zeros(L * h, np.uint8)
    assert F.bob(cur, L, 1, 0, dst, L, contract=True) is None  # quirk 7
    assert F.linear(IR.UYVY, cur, L, 1, 0, dst, L, contract=True) is None
    assert F.linear(13, cur, L, h, 0, dst, L, contract=True) is None  # quirk 8: JPEG
    assert F.linear(13, cur, L, h, 0, dst, L) is not None  # the reference blends its bytes
    assert F.double_framerate(13, prev, cur, L, h, 0, dst, L, True, contract=True) is None
    assert F.double_framerate(13, prev, cur, L, h, 0, dst, L, False, contract=True) is not None
    assert F.interlace(cur, prev, L, h, dst, L - 1, contract=True) is None


# ---- mutants: restatements that "fix" a quirk fail against the reference -----------------------------------------
def _fixed_rounding(codec, a, b):
    if IR.BITS[codec] == 8:
        return IR._avg(a, b).astype(np.uint8)
    return IR._avg(a.view(np.uint16), b.view(np.uint16)).astype(np.uint16).view(np.uint8)


def _fixed_r10k(codec, a, b):
    o = F.avg_lines(codec, a, b)
    return o.view(np.uint32).byteswap().view(np.uint8)


def _fixed_v210(codec, a, b):
    o = F.avg_lines(codec, a, b)
    return (o.view(np.uint32) & 0x3FFFFFFF).view(np.uint8)


def _fixed_r12l(codec, a, b):
    g = a.size // 16
    n = 16 * g
    k = (n + 2) // 3 * 3 - n
    return IR._r12l_pack(IR._avg(IR._r12l_unpack(np.pad(a[:n], (0, k))), IR._r12l_unpack(np.pad(b[:n], (0, k)))))[:n]  # every word stored


@pytest.mark.parametrize("name,codec,mutant", [("rounding 8-bit", IR.UYVY, _fixed_rounding), ("rounding 16-bit", IR.RG48, _fixed_rounding),
                                               ("R10k swap", IR.R10k, _fixed_r10k), ("v210 padding cleared", IR.v210, _fixed_v210),
                                               ("R12L last word", IR.R12L, _fixed_r12l)])
def test_mutant_avg_lines_fails(ref, name, codec, mutant):
    L = {IR.UYVY: 64, IR.RG48: 96, IR.R10k: 64, IR.v210: 128, IR.R12L: 160}[codec]  # R12L: 10 groups, the last word pending
    a, b = util.rng_bytes(L * 4, 7), util.rng_bytes(L * 4, 8)
    d = np.zeros(L * 4 + 64, np.uint8)
    ref.ref_tdi_avg_lines(codec, L, a.ctypes.data, b.ctypes.data, d.ctypes.data)
    assert np.array_equal(d[:F.avg_lines(codec, a[:L], b[:L]).size], F.avg_lines(codec, a[:L], b[:L]))
    m = mutant(codec, a[:L], b[:L])
    assert not np.array_equal(d[:m.size], m), name


def test_mutant_row_rules_fail(ref):
    c, w = IR.UYVY, 8
    L = vc_get_linesize(w, c)
    # quirk 6: at odd h a "fixed" double_framerate would fill row h-1 from cur
    h = 5
    prev, cur = inputs(L, h, 3)
    dst = np.full(L * h, 0xA5, np.uint8)
    got, _ = ref_run(ref, DF, c, w, h, 0, prev, cur, dst, L)
    fixed = F.double_framerate(c, prev, cur, L, h, 0, dst, L)
    fixed[(h - 1) * L:h * L] = cur[(h - 1) * L:h * L]
    assert not np.array_equal(got, fixed)
    assert np.array_equal(got, F.double_framerate(c, prev, cur, L, h, 0, dst, L))
    # the bob last-row rule: a "fixed" bob would double source row h-1 at even h in call 1
    h = 6
    prev, cur = inputs(L, h, 4)
    dst = np.zeros(L * h, np.uint8)
    got, _ = ref_run(ref, BOB, c, w, h, 1, prev, cur, dst, L)
    fixed = F.bob(cur, L, h, 1, dst, L)
    fixed[(h - 1) * L:] = cur[(h - 1) * L:h * L]
    assert not np.array_equal(got, fixed)
    assert np.array_equal(got, F.bob(cur, L, h, 1, dst, L))


# ---- golden fixtures (made from the reference by tests/golden/make_field_rate_golden.py) -------------------------
def test_restatement_equals_golden():
    g = util.golden(GOLDEN)
    n = 0
    for k in g.files:
        if not k.endswith("_meta"):
            continue
        p = k[:-5]
        algo, c, L, h, call, d, pitch, fill = g[k].tolist()
        dst = np.full(pitch * h, fill, np.uint8)
        want = model(algo, c, L, h, call, g[p + "_prev"], g[p + "_cur"], dst, pitch, d)
        m = frame_mask(L, h, pitch, algo == DF and d and pitch != L)
        assert np.array_equal(want[m], g[p + "_out"][m]), p
        n += 1
    assert n >= 100


# ---- GPU ------------------------------------------------------------------------------------------------------
GUARD = 64
SENT = 0x3C


def gpu_run(algo, c, L, h, call, prev, cur, dst_init, pitch, d=0, offset=0):
    """ugb200_pp_* between sentinels; returns (rc, dst bytes)"""
    import torch
    from ultragrid_b200 import _lib, api
    lib = _lib.load()
    p, q, o = (util.Guarded(a.size, offset, SENT, a, GUARD) for a in (prev, cur, dst_init))
    P, Q, O = (ctypes.c_void_p(g.view.data_ptr()) for g in (p, q, o))
    st = api._stream()
    if algo == DF:
        rc = lib.ugb200_pp_double_framerate(c, P, Q, L, h, call, d, O, pitch, st)
    elif algo == BOB:
        rc = lib.ugb200_pp_bob(Q, L, h, call, O, pitch, st)
    elif algo == LINEAR:
        rc = lib.ugb200_pp_linear(c, Q, L, h, call, O, pitch, st)
    else:
        rc = lib.ugb200_pp_interlace(Q, P, L, h, O, pitch, st)
    torch.cuda.synchronize()
    for g, src in ((p, prev), (q, cur)):
        assert np.array_equal(g.check_outside(), src), "a source changed"
    return rc, o.check_outside()


def _align(algo, c, d):
    if algo == LINEAR or (algo == DF and d):
        return 4 if c in (IR.v210, IR.R10k, IR.R12L) else 2 if IR.BITS[c] == 16 else 1
    return 1


@pytest.mark.gpu
@pytest.mark.parametrize("algo", (DF, BOB, LINEAR, 3), ids=("df", "bob", "linear", "interlace"))
def test_gpu_exact(algo):
    n = 0
    for a, c, w, h, call, d in cases():
        if a != algo:
            continue
        L = vc_get_linesize(w, c)
        for pad, off in ((0, 0), (20, 0), (6, 1)):
            for fill in FILLS:
                _check_gpu(algo, c, L, h, call, d, pad, off, fill, n)
        n += 1


def _check_gpu(algo, c, L, h, call, d, pad, off, fill, seed):
    """one ugb200_pp_* call between sentinels against the restatement's contract form (or the refusal it must give)"""
    prev, cur = inputs(L, h, seed)
    pitch = L + pad
    dst = np.full(pitch * (h - 1) + L, fill, np.uint8)  # tight: ends at row h-1's L bytes
    rc, got = gpu_run(algo, c, L, h, call, prev, cur, dst, pitch, d, off)
    want = model(algo, c, L, h, call, prev, cur, dst, pitch, d, contract=True)
    al = _align(algo, c, d)
    if (L % al or pitch % al or off % al) and want is not None:
        assert rc == -1 and np.array_equal(got, dst), (algo, c, L, h, call, d, pad, off)
        return
    if want is None:
        assert rc == -4 and np.array_equal(got, dst), (algo, c, L, h, call, d)
        return
    assert rc == 0, (algo, c, L, h, call, d, rc)
    assert np.array_equal(got, want), (algo, c, L, h, call, d, pad, off, fill, np.flatnonzero(got != want)[:8])


# line sizes no width gives: partial v210 / R10k 16-byte groups and R12L 36-byte groups at the end of every row
GPU_RAW_LS = (4, 12, 20, 36, 44, 52, 68, 100, 112, 136, 140, 172, 188, 252, 260, 300, 1004)


@pytest.mark.gpu
@pytest.mark.parametrize("codec", (IR.v210, IR.R10k, IR.R12L, IR.UYVY, IR.RG48))
def test_gpu_exact_raw_line_sizes(codec):
    n = 0
    for L in GPU_RAW_LS:
        for h in (2, 3, 5, 6):
            for algo in (DF, BOB, LINEAR, 3):
                for call in ((0, 1) if algo != 3 else (0,)):
                    for d in ((0, 1) if algo == DF else (0,)):
                        for pad in (0, 20):
                            _check_gpu(algo, codec, L, h, call, d, pad, 0, FILLS[n % 2], 500 + n)
                            n += 1


@pytest.mark.gpu
@pytest.mark.parametrize("codec,w,h", [(IR.UYVY, 3840, 2160), (IR.UYVY, 7680, 4320), (IR.v210, 3840, 2161), (IR.v210, 7680, 4320),
                                       (IR.RG48, 3840, 2160), (IR.R10k, 7680, 4321), (IR.R12L, 3840, 2160), (IR.R12L, 7680, 4320),
                                       (IR.UYVY, 1920, 1081)])
def test_gpu_frames(codec, w, h):
    L = vc_get_linesize(w, codec)
    prev, cur = inputs(L, h, w + h)
    dst = np.full(L * h, 0xA5, np.uint8)
    for algo in (DF, BOB, LINEAR, 3):
        for call in ((0, 1) if algo != 3 else (0,)):
            for d in ((0, 1) if algo == DF else (0,)):
                rc, got = gpu_run(algo, codec, L, h, call, prev, cur, dst, L, d)
                want = model(algo, codec, L, h, call, prev, cur, dst, L, d, contract=True)
                assert rc == 0 and np.array_equal(got, want), (algo, call, d, np.flatnonzero(got != want)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("codec", (IR.UYVY, IR.RG48, IR.v210, IR.R10k, IR.R12L, IR.Y416))
def test_gpu_fused_d_equals_weave_then_deinterlace_ex(codec):
    """`:d` at pitch L (one pass) against the two steps: the copy (deinterlace=False), then ugb200_vc_deinterlace_ex in
    place at pitch L; at line sizes from widths and off every multiple of 16 and 36 (partial groups), both calls.
    Off pitch L the two steps are what runs, so there it is checked against the restatement."""
    import torch
    from ultragrid_b200 import api
    al = 4 if codec in (IR.v210, IR.R10k, IR.R12L) else 2 if IR.BITS[codec] == 16 else 1
    shapes = [(vc_get_linesize(w, codec), h) for w, h in ((1920, 1080), (1918, 1081), (100, 7), (47, 5))]
    shapes += [(L, h) for L in (68, 136, 188, 112, 260, 1004) if L % al == 0 for h in (4, 5)]
    for L, h in shapes:
        prev, cur = inputs(L, h, L + h)
        P, Q = torch.from_numpy(prev).cuda(), torch.from_numpy(cur).cuda()
        for pad in (0, 64, 4):
            pitch = L + pad
            for call in (0, 1):
                init = util.rng_bytes(pitch * h, 9)
                fused = torch.from_numpy(init).cuda()
                api.double_framerate(codec, P, Q, L, h, call, True, dst=fused, pitch=pitch)
                if pad == 0:
                    composed = torch.from_numpy(init).cuda()
                    api.double_framerate(codec, P, Q, L, h, call, False, dst=composed, pitch=pitch)
                    api.deinterlace_ex(codec, composed, L, h, dst=composed)
                    assert torch.equal(fused, composed), (codec, L, h, call)
                want = F.double_framerate(codec, prev, cur, L, h, call, init, pitch, True, contract=True)
                assert np.array_equal(fused.cpu().numpy(), want), (codec, L, h, pad, call)


@pytest.mark.gpu
def test_gpu_side_stream_and_api():
    import torch
    from ultragrid_b200 import api
    L, h = vc_get_linesize(1920, IR.UYVY), 1080
    prev, cur = inputs(L, h, 5)
    s = torch.cuda.Stream()
    P, Q = torch.from_numpy(prev).cuda(), torch.from_numpy(cur).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        outs = [api.double_framerate(IR.UYVY, P, Q, L, h, 0, True, stream=s), api.deinterlace_bob(Q, L, h, 1, stream=s),
                api.deinterlace_linear(IR.UYVY, Q, L, h, 0, stream=s), api.interlace(Q, P, L, h, stream=s)]
    s.synchronize()
    z = np.zeros(L * h, np.uint8)
    wants = [F.double_framerate(IR.UYVY, prev, cur, L, h, 0, z, L, True, True), F.bob(cur, L, h, 1, z, L, True),
             F.linear(IR.UYVY, cur, L, h, 0, z, L, True), F.interlace(cur, prev, L, h, z, L, True)]
    for o, want in zip(outs, wants):
        assert np.array_equal(o.cpu().numpy(), want)


@pytest.mark.gpu
def test_gpu_refusals_write_nothing():
    import torch
    from ultragrid_b200 import _lib, api
    lib = _lib.load()
    L, h = 384, 6
    src = util.rng_bytes(L * h, 1)
    buf = torch.full((L * h * 4 + 512,), SENT, dtype=torch.uint8, device="cuda")
    buf[64:64 + src.size] = torch.from_numpy(src).cuda()
    before = buf.cpu().numpy()
    base = buf.data_ptr()
    S, far = 64, 64 + L * h + 64
    st = api._stream()
    vp = ctypes.c_void_p

    def df(codec, d, off, pitch, hh=h, call=0, dst=None, prev=None):
        return lib.ugb200_pp_double_framerate(codec, vp(base + (prev if prev is not None else S)), vp(base + S), L, hh, call, d,
                                              vp(base + (dst if dst is not None else far + off)), pitch, st)

    rcs = [
        (df(13, 1, 0, L), -4),                  # JPEG `:d`: opaque
        (df(IR.DVS10, 1, 0, L), -4),            # no DVS10 blend
        (df(IR.UYVY, 0, 0, L, hh=1), -1),       # h < 2
        (df(IR.UYVY, 0, 0, L - 2), -1),         # pitch < L
        (df(IR.UYVY, 0, 0, L, call=2), -1),     # no such call
        (df(IR.UYVY, 0, 0, L, dst=S + L), -1),  # dst overlaps cur
        (df(IR.v210, 1, 2, L), -1),             # word codec at a 2-byte address
        (lib.ugb200_pp_linear(13, vp(base + S), L, h, 0, vp(base + far), L, st), -4),
        (lib.ugb200_pp_linear(IR.R12L, vp(base + S), L, h, 0, vp(base + far), L + 2, st), -1),
        (lib.ugb200_pp_linear(IR.RG48, vp(base + S + 1), L, h, 0, vp(base + far), L, st), -1),
        (lib.ugb200_pp_linear(IR.UYVY, vp(base + S), L, 1, 0, vp(base + far), L, st), -1),
        (lib.ugb200_pp_bob(vp(base + S), L, 1, 0, vp(base + far), L, st), -1),
        (lib.ugb200_pp_bob(vp(base + S), L, h, 0, vp(base + S + 8), L, st), -1),
        (lib.ugb200_pp_bob(None, L, h, 0, vp(base + far), L, st), -1),
        (lib.ugb200_pp_interlace(vp(base + S), vp(base + far), L, h, vp(base + far + 16), L, st), -1),
        (lib.ugb200_pp_interlace(vp(base + S), vp(base + S), 0, h, vp(base + far), L, st), -1),
    ]
    torch.cuda.synchronize()
    assert [r for r, _ in rcs] == [w for _, w in rcs]
    assert np.array_equal(buf.cpu().numpy(), before), "a refusal wrote"
    assert lib.ugb200_pp_bob(vp(base + S), L, h, 0, vp(base + far), L, st) == 0  # and the good call works
    torch.cuda.synchronize()
    assert not np.array_equal(buf.cpu().numpy(), before)


@pytest.mark.gpu
def test_gpu_matches_golden():
    g = util.golden(GOLDEN)
    for k in g.files:
        if not k.endswith("_meta"):
            continue
        p = k[:-5]
        algo, c, L, h, call, d, pitch, fill = g[k].tolist()
        if algo == DF and d and (IR.BITS[c] == 16 or c == IR.R12L):
            continue  # vc_deinterlace_ex's own differences (test_interlace.py); checked against the restatement above
        dst = np.full(pitch * h, fill, np.uint8)
        rc, got = gpu_run(algo, c, L, h, call, g[p + "_prev"], g[p + "_cur"], dst, pitch, d)
        if (IR.opaque(c) and (algo == LINEAR or d)) or (d and c == IR.DVS10):
            assert rc == -4 and np.array_equal(got, dst)  # the reference logs and keeps the weave; vc_deinterlace_ex refuses DVS10
            continue
        m = frame_mask(L, h, pitch, algo == DF and d and pitch != L)
        assert rc == 0 and np.array_equal(got[m], g[p + "_out"][m]), p
