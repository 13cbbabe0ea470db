"""The resize algorithms of ugb200_cf_resize_create2 handles: cubic, lanczos4, area at any downscale ratio, and area
upscaling (resize_kernels.cu multitap_kernel and resize_kernel, DESIGN.md §2 "Resize").

CPU: the contract pinned without OpenCV, through the restatement (resize_algos_ref.py) against independent float64
models: weights, area tabs, accuracy on random frames, identity, constant frames, the 8-bit lanczos4 worst case, and
mutants that each fail one of those checks.
GPU: api.resize(..., all_algos=True) equals the restatement byte for byte, with sentinels around the exact output length.
"""
import math

import numpy as np
import pytest

import resize_algos_ref as A
import resize_filter_ref as R
import util
from test_resize_filter import frame, route_bytes

RATIOS = [0.5, 1 / 3, 0.75, 2 / 3, 1.5, 2.0, 0.3]
FRACS = np.linspace(0, 1, 1001, dtype=np.float32)[:-1]


# ---- float64 models ------------------------------------------------------------------------------------------------
def keys64(f, A_=-0.75):
    """Keys' cubic convolution kernel at the distances of taps -1, 0, 1, 2 from a fraction f"""
    def k(x):
        x = abs(x)
        if x <= 1:
            return (A_ + 2) * x ** 3 - (A_ + 3) * x ** 2 + 1
        if x < 2:
            return A_ * x ** 3 - 5 * A_ * x ** 2 + 8 * A_ * x - 4 * A_
        return 0.0
    return np.array([k(f + 1), k(f), k(1 - f), k(2 - f)])


def lanczos64(f):
    """the normalised Lanczos-4 kernel, sinc(t) sinc(t / 4), at taps -3 .. 4 from a fraction f"""
    t = np.array([f + 3 - i for i in range(8)], np.float64)
    w = np.sinc(t) * np.sinc(t / 4)
    return w / w.sum()


def weights64(n_dst, inv, algo):
    """(first, (n_dst, K) float64 weights) at float64 positions"""
    p = (np.arange(n_dst) + 0.5) / inv - 0.5
    s = np.floor(p).astype(np.int64)
    f = p - s
    w = np.array([keys64(x) if algo == A.CUBIC else lanczos64(x) for x in f])
    K = w.shape[1]
    return s - K // 2 + 1, w


def multitap64(rgb, rw, rh, isx, isy, algo):
    h, w, _ = rgb.shape
    fx, ax = weights64(rw, isx, algo)
    fy, ay = weights64(rh, isy, algo)
    K = ax.shape[1]
    tx, ty = A.taps(fx, K, w), A.taps(fy, K, h)
    H = sum(rgb[:, tx[:, j]] * ax[None, :, j, None] for j in range(K))
    return sum(H[ty[:, k]] * ay[:, k, None, None] for k in range(K)), (ax, ay)


def box64(rgb, rw, rh, isx, isy):
    """the exact coverage-weighted mean over [d scale, (d + 1) scale) on each axis, clipped to the frame"""
    h, w, _ = rgb.shape

    def cover(n_src, n_dst, scale):
        m = np.zeros((n_dst, n_src))
        for d in range(n_dst):
            a, b = d * scale, min((d + 1) * scale, n_src)
            for s in range(int(math.floor(a)), int(math.ceil(b))):
                m[d, s] = max(0.0, min(b, s + 1) - max(a, s))
            m[d] /= m[d].sum()
        return m

    mx, my = cover(w, rw, 1 / isx), cover(h, rh, 1 / isy)
    return np.einsum("yi,ijc,xj->yxc", my, rgb.astype(np.float64), mx)


def area_bilinear64(rgb, rw, rh, isx, isy):
    """bilinear at the area-mode positions, in float64"""
    h, w, _ = rgb.shape

    def taps(n_src, n_dst, inv, zero):
        d = np.arange(n_dst, dtype=np.float64)
        s = np.floor(d / inv).astype(np.int64)
        f = (d + 1) - (s + 1) * inv
        f = np.where(f <= 0, 0, f - np.floor(f))
        if zero:
            f = np.where(s >= n_src - 1, 0, f)
            s = np.where(s >= n_src - 1, n_src - 1, s)
        return np.clip(s, 0, n_src - 1), np.clip(s + 1, 0, n_src - 1), f

    x0, x1, fx = taps(w, rw, isx, True)
    y0, y1, fy = taps(h, rh, isy, False)
    H0 = rgb[y0][:, x0] * (1 - fx)[None, :, None] + rgb[y0][:, x1] * fx[None, :, None]
    H1 = rgb[y1][:, x0] * (1 - fx)[None, :, None] + rgb[y1][:, x1] * fx[None, :, None]
    return H0 * (1 - fy)[:, None, None] + H1 * fy[:, None, None]


# ---- weights and tabs ----------------------------------------------------------------------------------------------
def test_cubic_weights_equal_keys():
    # c1, c2 are within 2^-22 of Keys.  c0's Horner form cancels terms near 3 (ulp 2^-22) down to about -0.002, and c3
    # = 1 - c0 - c1 - c2 inherits that error: up to 1.21e-6 (1.27 * 2^-20) over 200 000 fractions, so 2^-19 here
    for f in FRACS:
        w = A.cubic_weights(f)
        e = np.abs(w.astype(np.float64) - keys64(float(f)))
        assert e[1:3].max() <= 2 ** -22 and e.max() <= 2 ** -19, f
        assert abs(float(w.astype(np.float64).sum()) - 1) <= 4 * 2 ** -24, f
    assert A.cubic_weights(0).tolist() == [0, 1, 0, 0]


def test_lanczos4_weights_equal_lanczos(mut=()):
    for f in FRACS:
        w = A.lanczos4_weights(f, "lanczos_unnormalised" not in mut)
        assert np.abs(w.astype(np.float64) - lanczos64(float(f))).max() <= 1e-6, f
    assert A.q11(A.lanczos4_weights(0)).tolist() == [0, 0, 0, 2048, 0, 0, 0, 0]


def test_area_tab_alphas_sum_to_one():
    for n in (7, 33, 97, 1919, 1920):
        for r in (1.0, 0.75, 2 / 3, 0.5, 0.3, 1 / 3, 1280 / 1920, 0.1):
            nd = max(1, int(n * r))
            scale = n / nd
            for d, e in enumerate(A.area_tab(n, nd, scale)):
                cw = min(scale, n - d * scale)
                s = sum(float(a) for _, a in e)
                assert abs(s - 1) <= 1e-3 / cw + len(e) * 2 ** -23, (n, nd, d, s)


# ---- accuracy against float64 models -------------------------------------------------------------------------------
SIZES = [(97, 31), (64, 48), (33, 17)]


def _cases():
    for i, (w, h) in enumerate(SIZES):
        for r in RATIOS:
            rw, rh = int(w * r), int(h * r)
            if rw and rh:
                yield i, w, h, rw, rh, r


def test_multitap_8bit_within_q11_bound(mut=()):
    for i, w, h, rw, rh, r in _cases():
        rgb = util.rng_bytes(w * h * 3, 300 + i).reshape(h, w, 3).astype(np.int64)
        for algo in (A.CUBIC, A.LANCZOS4):
            got = A.resample(rgb, rw, rh, r, r, algo, False, mut)
            want, (ax, ay) = multitap64(rgb.astype(np.float64), rw, rh, r, r, algo)
            # the Q11 tables' own rounding: |Vq - V64| <= 255 (sum|a_q| sum|b_q - b64| + sum|a_q - a64| sum|b64|), + 1/2
            qa, qb = A.q11(A.multitap_table(rw, r, algo)[1]) / 2048, A.q11(A.multitap_table(rh, r, algo)[1]) / 2048
            ea, eb = np.abs(qa - ax).sum(1), np.abs(qb - ay).sum(1)
            bound = 0.5 + 255 * (np.abs(qa).sum(1)[None, :] * eb[:, None] + ea[None, :] * np.abs(ay).sum(1)[:, None])
            err = np.abs(got - np.clip(want, 0, 255)).max(axis=2)
            assert (err <= bound + 1e-9).all(), (algo, w, h, r, float((err - bound).max()))


def test_multitap_rg48_within_one(mut=()):
    for i, w, h, rw, rh, r in _cases():
        rgb = util.rng_bytes(w * h * 6, 400 + i).view("<u2").reshape(h, w, 3).astype(np.int64)
        for algo in (A.CUBIC, A.LANCZOS4):
            got = A.resample(rgb, rw, rh, r, r, algo, True, mut)
            want = np.clip(multitap64(rgb.astype(np.float64), rw, rh, r, r, algo)[0], 0, 65535)
            assert np.abs(got - want).max() <= 1.0, (algo, w, h, r)


def test_area_any_within_one_of_box_mean(mut=()):
    for i, w, h, rw, rh, r in _cases():
        if r >= 1 or A.area_mode(w, h, rw, rh, r, r) != "any":
            continue
        for w16 in (False, True):
            n = 2 if w16 else 1
            rgb = util.rng_bytes(w * h * 3 * n, 500 + i)
            rgb = (rgb.view("<u2") if w16 else rgb).reshape(h, w, 3).astype(np.int64)
            got = A.resample(rgb, rw, rh, r, r, A.AREA, w16, mut)
            assert np.abs(got - box64(rgb, rw, rh, r, r)).max() <= 1.0, (w, h, r, w16)


def test_area_up_within_one_of_area_bilinear(mut=()):
    for i, w, h, rw, rh, r in list(_cases()) + [(9, 3, 2, 4, 2, None)]:
        isx, isy = (rw / w, rh / h) if r is None else (r, r)
        if A.area_mode(w, h, rw, rh, isx, isy) != "up":
            continue
        for w16 in (False, True):
            n = 2 if w16 else 1
            rgb = util.rng_bytes(w * h * 3 * n, 600 + i)
            rgb = (rgb.view("<u2") if w16 else rgb).reshape(h, w, 3).astype(np.int64)
            got = A.resample(rgb, rw, rh, isx, isy, A.AREA, w16, mut)
            assert np.abs(got - area_bilinear64(rgb.astype(np.float64), rw, rh, isx, isy)).max() <= 1.0, (w, h, r, w16)


def test_area_up_integer_is_replication(mut=()):
    for k in (2, 3, 4):
        for w16 in (False, True):
            rgb = util.rng_bytes(13 * 7 * 3 * (2 if w16 else 1), k)
            rgb = (rgb.view("<u2") if w16 else rgb).reshape(7, 13, 3).astype(np.int64)
            got = A.resample(rgb, 13 * k, 7 * k, float(k), float(k), A.AREA, w16, mut)
            assert np.array_equal(got, np.repeat(np.repeat(rgb, k, 0), k, 1)), (k, w16)


def test_identity_at_scale_one():
    for route in R.RESIZE_SET:
        for algo in (A.CUBIC, A.AREA, A.LANCZOS4):
            w, h = 34, 18
            d = util.rng_bytes(R.frame_len(route, w, h), route + algo)
            rc, out = A.resize((R.FRACTION, 1.0, 0, 0, algo), route, d, w, h)
            rgb = R.to_rgb(route, d, w, h)
            want = rgb.astype("<u2").view(np.uint8) if route == R.RG48 else rgb.astype(np.uint8)
            assert rc == 0 and np.array_equal(out.reshape(h, w, -1), want), (route, algo)


def _constant_movers():
    """(algo, ratio, n, sum a, sum b, value) for every 8-bit value that a pair of table entries moves"""
    moved = []
    for algo in (A.CUBIC, A.LANCZOS4):
        for r in RATIOS + [1.0, 0.25, 0.1]:
            for n in (33, 97, 1920):
                q = A.q11(A.multitap_table(max(1, int(n * r)), r, algo)[1]).sum(1)
                for sa in np.unique(q):
                    for sb in np.unique(q):
                        v = np.arange(256, dtype=np.int64)
                        out = np.clip((v * int(sa) * int(sb) + (1 << 21)) >> 22, 0, 255)
                        moved += [(algo, r, n, int(sa), int(sb), int(c)) for c in v[out != v]]
    return moved


def test_constant_frames_stay_constant():
    # every sum of Q11 weights in these tables lies in [2046, 2049], and no pair of them moves any 8-bit value
    assert _constant_movers() == []
    for f in (0.5, 1 / 3, 0.75, 1.5, 2.0, 0.3, 2 / 3):
        for algo in (A.CUBIC, A.AREA, A.LANCZOS4):
            for route, vals in ((R.RGB, (0, 1, 77, 254, 255)), (R.RG48, (0, 1, 32768, 65534, 65535))):
                for c in vals:
                    d = np.full(40 * 30 * 3, c, "<u2" if route == R.RG48 else np.uint8).view(np.uint8)
                    rc, out = A.resize((R.FRACTION, f, 0, 0, algo), route, d, 40, 30)
                    got = out.view("<u2") if route == R.RG48 else out
                    assert rc == 0 and (got == c).all(), (f, algo, route, c)


def worst_case_lanczos(n=64, r=0.5):
    """an RGB frame of 0 and 255 on the signs of a_j b_k around the interior pair of table entries with the largest
    sum of positive products; (frame, (x, y), exact result, V)"""
    first, w = A.multitap_table(int(n * r), r, A.LANCZOS4)
    q = A.q11(w)
    pos = np.where(q > 0, q, 0).sum(1)
    inner = [d for d in range(len(first)) if first[d] >= 0 and first[d] + 8 <= n]
    d = max(inner, key=lambda i: int(pos[i]))
    outer = np.outer(q[d], q[d])  # b_k a_j, rows k, columns j
    img = np.zeros((n, n, 3), np.int64)
    img[first[d]:first[d] + 8, first[d]:first[d] + 8] = np.where(outer > 0, 255, 0)[:, :, None]
    V = int(255 * outer[outer > 0].sum())
    return img, (d, d), min(255, (V + (1 << 21)) >> 22), V


def test_lanczos4_8bit_worst_case_exact(mut=()):
    img, (x, y), want, V = worst_case_lanczos()
    got = A.resample(img, 32, 32, 0.5, 0.5, A.LANCZOS4, False, mut)
    assert (got[y, x] == want).all()
    # the largest V of any pair of Q11 lanczos4 entries, plus the rounding term, stays below 2^31 (an int suffices)
    assert V + (1 << 21) < 2 ** 31


MUTANTS = {
    "cubic_a_half": test_multitap_8bit_within_q11_bound,
    "lanczos_unnormalised": test_lanczos4_weights_equal_lanczos,
    "area_up_as_linear": test_area_up_within_one_of_area_bilinear,
    "area_no_partial": test_area_any_within_one_of_box_mean,
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fail(name):
    with pytest.raises(AssertionError):
        MUTANTS[name](mut=(name,))


def test_wrap32_mutant_is_equivalent():
    """8-bit sums wrapped at 32 bits give the exact bytes: no lanczos4 or cubic Q11 table reaches 2^31 (the worst case
    above), so the wrap cannot show.  The kernel still bounds V from the handle's tables before it sums in 32 bits."""
    img, (x, y), want, _ = worst_case_lanczos()
    got = A.resample(img, 32, 32, 0.5, 0.5, A.LANCZOS4, False, ("wrap32",))
    assert (got[y, x] == want).all()


# ---- GPU -----------------------------------------------------------------------------------------------------------
def want_for(param, c, w, h, data):
    from ultragrid_b200 import compress
    route = c if c in R.RESIZE_SET else compress.get_best_decoder_from(c, list(R.RESIZE_SET))
    return A.resize(param, route, route_bytes(c, route, w, h, data), w, h)


def gpu_check(param, c, w, h, seed=1, handle=None, stream=None, data=None):
    import torch
    from ultragrid_b200 import api
    mode, factor, tw, th, algo = param
    data = frame(c, w, h, seed) if data is None else data
    rc, want = want_for(param, c, w, h, data)
    kw = dict(factor=factor) if mode == R.FRACTION else dict(size=(tw, th))
    r = handle or api.Resize(algo=algo, all_algos=True, **kw)
    g = util.Guarded(want.size if rc == 0 else 64)
    if rc != 0:
        with pytest.raises(RuntimeError, match=f"code {rc}"):
            r(util.dev(data), c, w, h, dst=g.view, stream=stream)
        torch.cuda.synchronize()
        assert (g.check_outside() == g.fill).all(), "a refusal wrote"
    else:
        r(util.dev(data), c, w, h, dst=g.view, stream=stream)
        torch.cuda.synchronize()
        got = g.check_outside()
        assert np.array_equal(got, want), f"{param} codec {c} {w}x{h}: {int(np.count_nonzero(got != want))} bytes differ"
    if handle is None:
        r.close()
    return rc


FACTORS = [1.0, 0.5, 1 / 3, 0.25, 0.75, 2 / 3, 1.5, 2.0, 0.3]


@pytest.mark.gpu
@pytest.mark.parametrize("codec", R.RESIZE_SET)
@pytest.mark.parametrize("algo", ["cubic", "lanczos4", "area"])
def test_gpu_native_layouts_factors(codec, algo):
    a = R.ALGOS[algo]
    odd = codec in (R.RGB, R.RGBA, R.RG48)
    sizes = [(2, 2), (98, 26), (36, 8)] + ([(1, 1), (97, 31), (35, 9)] if odd else [(96, 30)])
    codes = []
    for w, h in sizes:
        for f in FACTORS:
            codes.append(gpu_check((R.FRACTION, f, 0, 0, a), codec, w, h, seed=w + h + codec + a))
    assert codes.count(0) >= len(codes) // 2


@pytest.mark.gpu
@pytest.mark.parametrize("codec", R.RESIZE_SET)
def test_gpu_dimension_targets(codec):
    for algo in (A.CUBIC, A.AREA, A.LANCZOS4):
        for (w, h), (tw, th) in (((96, 54), (64, 36)), ((96, 54), (40, 40)), ((96, 54), (100, 30)), ((64, 48), (32, 24)),
                                 ((98, 54), (64, 36)), ((64, 36), (160, 90)), ((96, 54), (72, 41))):
            gpu_check((R.DIMENSIONS, 0.0, tw, th, algo), codec, w, h, seed=w * tw + algo)


@pytest.mark.gpu
@pytest.mark.parametrize("codec", [R.RGB, R.RG48])
def test_gpu_unequal_and_mixed_area(codec):
    # 1919x1080 -> 1280x720: generic area with scales 1.5004 and 1.5; 3x2 -> 4x3: mixed axes (rw 4, rh 2), area upscale
    assert gpu_check((R.DIMENSIONS, 0.0, 1280, 720, A.AREA), codec, 1919, 1080, seed=3) == 0
    assert gpu_check((R.DIMENSIONS, 0.0, 4, 3, A.AREA), codec, 3, 2, seed=4) == 0
    for algo in (A.CUBIC, A.LANCZOS4):
        assert gpu_check((R.DIMENSIONS, 0.0, 1280, 720, algo), codec, 1919, 1080, seed=5) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v210", "R10k", "R12L", "Y416", "Y216", "BGR", "VUYA", "DVS10"])
def test_gpu_routed_codecs(name):
    from ultragrid_b200 import Codec
    c = int(Codec[name])
    for w, h in ((96, 54), (50, 7), (1366, 3), (13, 9)):
        for algo, f in ((A.CUBIC, 0.5), (A.LANCZOS4, 0.75), (A.AREA, 2 / 3), (A.AREA, 1.5)):
            gpu_check((R.FRACTION, f, 0, 0, algo), c, w, h, seed=w + c + algo)


@pytest.mark.gpu
@pytest.mark.parametrize("codec", [R.RGB, R.UYVY, R.RG48])
def test_gpu_dense_and_sparse_staging(codec):
    """scale_x below and above K: the multi-tap kernel stages a dense span or K taps per column (chosen per block from
    the span's width); 0.3 and 0.2 fall on either side for cubic (K = 4), 0.15 and 0.1 for lanczos4 (K = 8)"""
    for algo, fs in ((A.CUBIC, (0.3, 0.26, 0.2, 0.1)), (A.LANCZOS4, (0.15, 0.13, 0.1, 0.05))):
        for f in fs:
            assert gpu_check((R.FRACTION, f, 0, 0, algo), codec, 1000, 120, seed=int(f * 100)) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,c,param", [(7680, 4320, R.UYVY, (R.FRACTION, 0.5, 0, 0, A.LANCZOS4)),
                                         (3840, 2160, R.UYVY, (R.DIMENSIONS, 0.0, 1920, 1080, A.CUBIC)),
                                         (1920, 1080, R.UYVY, (R.DIMENSIONS, 0.0, 1280, 720, A.AREA)),
                                         (1920, 1080, R.UYVY, (R.DIMENSIONS, 0.0, 3840, 2160, A.AREA))])
def test_gpu_8k_4k_1080p(w, h, c, param):
    assert gpu_check(param, c, w, h, seed=7) == 0


@pytest.mark.gpu
def test_gpu_lanczos4_8bit_worst_case():
    img, (x, y), want, _ = worst_case_lanczos()
    d = img.astype(np.uint8).reshape(-1)
    assert gpu_check((R.FRACTION, 0.5, 0, 0, A.LANCZOS4), R.RGB, 64, 64, data=d) == 0
    rc, out = A.resize((R.FRACTION, 0.5, 0, 0, A.LANCZOS4), R.RGB, d, 64, 64)
    assert (out.reshape(32, 32, 3)[y, x] == want).all()


@pytest.mark.gpu
def test_gpu_one_handle_across_descriptors_and_side_stream():
    import torch
    from ultragrid_b200 import api, Codec
    s = torch.cuda.Stream()
    seq = [(R.UYVY, 64, 32), (int(Codec.v210), 96, 54), (R.RGB, 33, 17), (R.RG48, 20, 10), (R.UYVY, 64, 32)]
    for algo in (A.CUBIC, A.LANCZOS4, A.AREA):
        for f in (0.75, 1.5):
            r = api.Resize(factor=f, algo=algo, all_algos=True)
            for i, (c, w, h) in enumerate(seq):
                assert gpu_check((R.FRACTION, f, 0, 0, algo), c, w, h, seed=i, handle=r, stream=s if i % 2 else None) == 0
            r.close()


@pytest.mark.gpu
def test_gpu_built_algorithms_equal_create_handles():
    import torch
    from ultragrid_b200 import api
    for algo in ("nearest", "linear", "area"):
        for c, w, h in ((R.RGB, 97, 31), (R.UYVY, 96, 48), (R.I420, 64, 32), (R.RG48, 35, 9)):
            for kw in (dict(factor=0.5), dict(factor=0.25), dict(factor=1.5), dict(size=(40, 40))):
                src = util.dev(frame(c, w, h, w + c))
                outs = []
                for all_algos in (False, True):
                    try:
                        outs.append(api.resize(src, c, w, h, algo=algo, all_algos=all_algos, **kw)[0].cpu().numpy())
                    except RuntimeError as e:
                        outs.append(str(e))
                torch.cuda.synchronize()
                if isinstance(outs[0], str):  # refused by _create: area at other than integer downscales
                    assert algo == "area" and "code -4" in outs[0], (algo, c, kw)
                else:
                    assert np.array_equal(outs[0], outs[1]), (algo, c, w, h, kw)


@pytest.mark.gpu
def test_gpu_create_handles_still_refuse():
    import torch
    from test_resize_filter import gpu_check as create_check
    for param in ((R.FRACTION, 0.5, 0, 0, A.CUBIC), (R.FRACTION, 0.5, 0, 0, A.LANCZOS4), (R.FRACTION, 0.75, 0, 0, A.AREA),
                  (R.FRACTION, 2.0, 0, 0, A.AREA)):
        assert create_check(param, R.RGB, 16, 8) == -4
    torch.cuda.synchronize()
