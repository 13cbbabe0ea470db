"""Fused UYVY -> DXT1 across the launcher's choices, bit for bit against the unmodified reference kernels (oracle/_ref:
cuda_yuv422_to_yuv444 + cuda_yuv_to_dxt1, as src/video_compress/cuda_dxt.cpp runs them).

An even block count with 16-byte aligned rows runs two blocks per thread, their encodes interleaved one phase apart; an odd block count, an
8-byte aligned buffer or a pitch of 8 (mod 16) takes the one-block-per-thread kernel.  The cases cover both, with a last CTA of a block row
that is partly idle, one-CTA frames and 8K frames, mirrored frames, padded rows, and three streams at once.
"""
import ctypes

import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def api():
    from ultragrid_b200 import api as a
    return a


@pytest.fixture(scope="module")
def ref():
    lib = util.ref_gpu()
    if lib is None:
        pytest.skip("oracle/_ref/libcuda_dxt_ref.so not present")
    return lib


def frame(w, h, seed):
    """noise with every third block row flat grey (the flat-block path) and every fifth one of low amplitude"""
    f = util.rng_bytes(w * h * 2, seed).reshape(h, w * 2)
    for by in range(h // 4):
        rows = f[4 * by:4 * by + 4]
        if by % 3 == 1:
            rows[:] = 0x80
        elif by % 5 == 2:
            rows[:] = 0x70 + (rows & 3)
    return f.reshape(-1)


def reference(ref, orc, uyvy, w, h):
    """cuda_yuv422_to_yuv444 then cuda_yuv_to_dxt1 (the expander needs a pixel count divisible by 256; otherwise the CPU oracle expands)"""
    ah = abs(h)
    if (w * ah) % 256 == 0:
        src = torch.from_numpy(uyvy).cuda()
        yuv444 = torch.empty(w * ah * 3, dtype=torch.uint8, device="cuda")
        assert ref.cuda_yuv422_to_yuv444(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(yuv444.data_ptr()), w * ah, None) == 0
    else:
        e = np.zeros(w * ah * 3, dtype=np.uint8)
        orc.orc_yuv422_to_yuv444(uyvy.ctypes.data, e.ctypes.data, w * ah)
        yuv444 = torch.from_numpy(e).cuda()
    out = torch.empty(w * ah // 2, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert ref.cuda_yuv_to_dxt1(ctypes.c_void_p(yuv444.data_ptr()), ctypes.c_void_p(out.data_ptr()), w, h, None) == 0
    return out


def assert_same(mine, theirs):
    if not torch.equal(mine, theirs):
        a = mine.cpu().numpy().view(np.uint32).reshape(-1, 2)
        b = theirs.cpu().numpy().view(np.uint32).reshape(-1, 2)
        bad = np.nonzero((a != b).any(axis=1))[0]
        pytest.fail(f"{len(bad)} of {len(a)} blocks differ; first block numbers {bad[:8].tolist()}")


# (width, height): block pairs per row = w / 8, 64 per CTA.  8 x 4 / 16 x 8: one CTA with one or two busy threads; 256: 32 pairs; 264: 33;
# 1288: 161 (two full CTAs and one with 33 pairs); 7688 x 4320: 961 pairs per row at 8K height; 7680 x 4320: the benchmark's frame (960 pairs,
# 15 full CTAs per row); negative heights: mirrored.
SHAPES = [(8, 4), (16, 8), (256, 4), (264, 8), (264, 4320), (1288, 36), (7688, 4320), (7680, 4320), (264, -8), (7688, -4320), (1288, -36)]


@pytest.mark.parametrize("w,h", SHAPES)
def test_two_block_kernel_vs_reference(api, ref, orc, w, h):
    uyvy = frame(w, abs(h), w + abs(h))
    assert_same(api.uyvy_to_dxt(torch.from_numpy(uyvy).cuda(), w, h), reference(ref, orc, uyvy, w, h))


@pytest.mark.parametrize("w,h,pad", [(264, 8, 16), (1288, -36, 48), (7688, 4320, 16), (264, 8, 8), (1288, 36, 24)])
def test_padded_pitch_vs_reference(api, ref, orc, w, h, pad):
    """a pitch that is a multiple of 16 keeps the two-block kernel; 8 (mod 16) takes the one-block kernel"""
    ah = abs(h)
    uyvy = frame(w, ah, 7 * w + ah)
    pitch = w * 2 + pad
    padded = np.full((ah, pitch), 0xA5, dtype=np.uint8)
    padded[:, :w * 2] = uyvy.reshape(ah, w * 2)
    mine = api.uyvy_to_dxt(torch.from_numpy(padded.reshape(-1)).cuda(), w, h, pitch=pitch)
    assert_same(mine, reference(ref, orc, uyvy, w, h))


@pytest.mark.parametrize("w,h", [(36, 16), (7684, 4320), (7684, -8)])
def test_odd_block_count_vs_reference(api, ref, orc, w, h):
    uyvy = frame(w, abs(h), 3 * w + abs(h))
    assert_same(api.uyvy_to_dxt(torch.from_numpy(uyvy).cuda(), w, h), reference(ref, orc, uyvy, w, h))


@pytest.mark.parametrize("w,h", [(264, 8), (7680, 4320)])
def test_eight_byte_aligned_source_vs_reference(api, ref, orc, w, h):
    uyvy = frame(w, h, 5 * w + h)
    buf = torch.zeros(uyvy.size + 16, dtype=torch.uint8, device="cuda")
    src = buf[8:8 + uyvy.size]
    src.copy_(torch.from_numpy(uyvy))
    assert src.data_ptr() % 16 == 8
    assert_same(api.uyvy_to_dxt(src, w, h), reference(ref, orc, uyvy, w, h))


def test_three_streams_at_once(api, ref, orc):
    """three frames of different shapes encoded concurrently on three streams, each launch enqueued before any completes, twice over"""
    shapes = [(7680, 4320), (7688, -4320), (1288, 36)]
    frames = [frame(w, abs(h), 11 + i) for i, (w, h) in enumerate(shapes)]
    want = [reference(ref, orc, f, w, h) for f, (w, h) in zip(frames, shapes)]
    srcs = [torch.from_numpy(f).cuda() for f in frames]
    streams = [torch.cuda.Stream() for _ in shapes]
    outs = [[torch.full((w * abs(h) // 2,), 0xEE, dtype=torch.uint8, device="cuda") for _ in range(2)] for w, h in shapes]
    torch.cuda.synchronize()
    for rep in range(2):
        for i, ((w, h), st) in enumerate(zip(shapes, streams)):
            with torch.cuda.stream(st):
                api.uyvy_to_dxt(srcs[i], w, h, out=outs[i][rep], stream=st)
    torch.cuda.synchronize()
    for i in range(len(shapes)):
        for rep in range(2):
            assert_same(outs[i][rep], want[i])
