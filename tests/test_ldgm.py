"""LDGM FEC (include/ugb200_ldgm.h, csrc/ldgm_kernels.cu) against the unmodified reference coder LDGM_session_cpu
(oracle/_ref/libldgm_ref.so) and, where the reference tree is absent, against tests/golden/ldgm_golden.npz."""
import ctypes
import os

import numpy as np
import pytest

import ldgm_cases as lc
import util


@pytest.fixture(scope="module")
def ref():
    L = lc.ref_lib()
    if L is None:
        pytest.skip("oracle/_ref/libldgm_ref.so not built (reference tree absent)")
    return L


_SESSIONS = {}


def ref_session(L, tmp_dir, k, m, c, seed):
    key = (k, m, c, seed)
    if key not in _SESSIONS:
        pcm = lc.matrix(k, m, c, seed)
        path = os.path.join(tmp_dir, f"ldgm_matrix-{k}-{m}-{c}-{seed}.bin")
        lc.write_matrix_file(path, pcm, k, m)
        _SESSIONS[key] = (pcm, lc.RefSession(L, path, k, m, c))
    return _SESSIONS[key]


@pytest.fixture(scope="module")
def mdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("ldgm"))


# ---------------------------------------------------------------- CPU ----------------------------------------------------------------

@pytest.mark.parametrize("k,m,c,seed", [(64, 64, 2, 1), (512, 384, 5, 7), (512, 384, 63, 3), (256, 256, 63, 11), (1024, 1024, 3, 5)])
@pytest.mark.parametrize("ps", [4, 20, 64, 600])
def test_ref_encode_equals_encode_naive_and_model(ref, mdir, k, m, c, seed, ps):
    pcm, s = ref_session(ref, mdir, k, m, c, seed)
    data = np.ascontiguousarray(util.rng_bytes(k * ps, seed * 31 + ps))
    fast, naive = s.encode_raw(data, ps, False), s.encode_raw(data, ps, True)
    assert np.array_equal(fast, naive), "encode != encode_naive (parity packets)"
    assert np.array_equal(fast, lc.model_parity(pcm, k, data.reshape(k, ps)).reshape(-1)), "encode != model (parity packets)"


@pytest.mark.parametrize("k,m,c,seed", [(64, 64, 2, 1), (512, 384, 5, 7), (8191, 8191, 2, 9)])
def test_ref_decode_no_loss_recovers_everything(ref, mdir, k, m, c, seed):
    pcm, s = ref_session(ref, mdir, k, m, c, seed)
    frame = util.rng_bytes(30011, seed)
    buf = s.encode(b"HDR12345", frame)
    got = buf.copy()
    fs = s.decode(got, [(0, buf.size)])
    assert fs == 8 + frame.size, "*frame_size"
    assert np.array_equal(got, buf), "whole buffer"


@pytest.mark.parametrize("k,m,c,seed", [(64, 64, 2, 1), (512, 384, 5, 7), (256, 64, 7, 100), (1000, 300, 3, 12345)])
def test_matrix_reader_equals_set_pcMatrix(ref, tmp_path, k, m, c, seed):
    """generate_ldgm_matrix writes the file; the reader below and set_pcMatrix must see the same pcm (kept to c * k <= 3 * 8192,
    the size of the generator's work array)"""
    path = str(tmp_path / "m.bin")
    assert ref.ref_ldgm_generate(path.encode(), k, m, c, seed) == 0
    kf, mf, pcm = lc.read_matrix_file(path)
    assert (kf, mf) == (k, m)
    s = lc.RefSession(ref, path, k, m, c)
    try:
        assert np.array_equal(pcm, s.pcm())
    finally:
        s.close()


def test_golden_matrices_are_the_generators(ref, tmp_path):
    g = np.load(lc.GOLDEN)
    for name in g.files:
        if not name.startswith("pcm_"):
            continue
        k, m, c, seed = (int(t) for t in name.split("_")[1:])
        path = str(tmp_path / f"{name}.bin")
        assert ref.ref_ldgm_generate(path.encode(), k, m, c, seed) == 0
        assert np.array_equal(lc.read_matrix_file(path)[2], g[name]), name


def test_golden_buffers_equal_model():
    """the stored encode_hdr_frame buffers of the reference equal the numpy model (runs without the reference tree)"""
    g = np.load(lc.GOLDEN)
    for name in g.files:
        if not name.startswith("enc_"):
            continue
        k, m, c, seed, size = (int(t) for t in name.split("_")[1:])
        hdr, frame = g[f"hdr_{k}_{m}_{c}_{seed}_{size}"], g[f"frame_{k}_{m}_{c}_{seed}_{size}"]
        assert np.array_equal(lc.model_encode(g[f"pcm_{k}_{m}_{c}_{seed}"], k, m, hdr.tobytes(), frame), g[name]), name


def test_c_abi_refuses_bad_matrices():
    """argument checks happen before any CUDA call, so they hold without a device"""
    from ultragrid_b200 import _lib
    L = _lib.load()
    h = L.ugb200_ldgm_create(None)
    assert h
    try:
        good = lc.matrix(64, 64, 2, 1)
        for pcm, k, m in [(good, 0, 64), (good, 64, 0), (good, 8192, 64), (good, 64, 8192)]:
            assert L.ugb200_ldgm_set_matrix(h, pcm.ctypes.data, k, m, pcm.shape[1]) == -1, (k, m)
        for bad in (-2, 128):  # an index below -1 or past k + m
            pcm = good.copy()
            pcm[5, 0] = bad
            assert L.ugb200_ldgm_set_matrix(h, pcm.ctypes.data, 64, 64, pcm.shape[1]) == -1, bad
        assert L.ugb200_ldgm_set_matrix(h, good.ctypes.data, 64, 64, 1) == -1
        assert L.ugb200_ldgm_set_matrix(h, good.ctypes.data, 64, 64, 129) == -1
        ps = ctypes.c_int()
        assert L.ugb200_ldgm_buffer_size(h, 100, ctypes.byref(ps)) == -3, "no matrix set"
        assert L.ugb200_ldgm_encode(h, good.ctypes.data, good.ctypes.data, 6) == -1, "packet size not a multiple of 4"
        fs = ctypes.c_int()
        assert L.ugb200_ldgm_decode(h, good.ctypes.data, 1000, None, 0, ctypes.byref(fs)) == -3, "no matrix set"
    finally:
        L.ugb200_ldgm_destroy(h)


# ---------------------------------------------------------------- GPU: encode ----------------------------------------------------------

def _coder(pcm, k, m, stream=None):
    from ultragrid_b200.api import LdgmCoder
    return LdgmCoder(pcm, k, m, stream=stream)


# set_pcMatrix refuses rows of more than 126 packets (MAX_W = 128 columns), so k * c / m stays well below that: k = 8191 with m = 64,
# or c = 63 with k = 512 and m = 64, is no configuration the reference can run
ENC_PARAMS = sorted({(k, m, c) for k in (64, 512, 8191) for m in (64, 384, k) for c in (2, 5, 63) if c <= m and k * c <= 100 * m})


def _frame_sizes(k):
    """1 B, a ps that is a multiple of 4 but not of 8 or 16, a 1080p JPEG, a 4K JPEG and an 8K UYVY frame; sizes that put ps at
    65532 (the largest multiple of 4 below 65535) where the buffers stay small enough for the CPU coder"""
    sizes = [1, 4 * k * 5 - 4 - 24, 300_000 + 17, 1_200_000 + 3]
    if k == 8191:
        sizes.append(7680 * 4320 * 2)
    if k <= 512:
        sizes.append(65532 * k - 4 - 24)
    return sizes


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,c", ENC_PARAMS)
def test_encode_host_equals_reference(ref, mdir, k, m, c):
    seeds = (1, 2) if k < 8191 else (3,)
    for seed in seeds:
        pcm, s = ref_session(ref, mdir, k, m, c, seed)
        assert pcm.shape[1] <= 128
        coder = _coder(pcm, k, m)
        for size in _frame_sizes(k):
            if k == 8191 and c == 63 and size > 2_000_000 and seed != 3:
                continue
            hdr = util.rng_bytes(24, size).tobytes()
            frame = util.rng_bytes(size, seed + size)
            want = s.encode(hdr, frame)
            got = coder.encode(frame, hdr)
            dbytes, ps = lc.layout(k, len(hdr) + size)
            assert got.size == want.size, (k, m, c, seed, size, "buffer length")
            assert np.array_equal(got[:dbytes], want[:dbytes]), (k, m, c, seed, size, ps, "header + frame + padding [0, k*ps)")
            assert np.array_equal(got[dbytes:], want[dbytes:]), (k, m, c, seed, size, ps, "parity [k*ps, (k+m)*ps)")
        coder.close()


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 4, 8, 1])
@pytest.mark.parametrize("k,m,c", [(64, 64, 2), (512, 384, 5), (8191, 8191, 63), (8191, 8191, 5)])
def test_encode_device_equals_reference(ref, mdir, k, m, c, offset):
    import torch
    pcm, s = ref_session(ref, mdir, k, m, c, 4)
    coder = _coder(pcm, k, m)
    for size in (1, 300_017, 4 * k * 3 - 4 - 16, 7680 * 4320 * 2 if k == 8191 else 2_000_000):
        hdr = util.rng_bytes(16, size + 1).tobytes()
        frame = util.rng_bytes(size, size + offset)
        dev = torch.zeros(size + 16, dtype=torch.uint8, device="cuda")
        dev[offset:offset + size] = torch.from_numpy(frame).cuda()
        got = coder.encode(dev[offset:offset + size], hdr)
        torch.cuda.synchronize()
        got = got.cpu().numpy()
        want = s.encode(hdr, frame)
        dbytes, ps = lc.layout(k, len(hdr) + size)
        assert got.size == want.size
        assert np.array_equal(got[:dbytes], want[:dbytes]), (size, offset, "header + frame + padding [0, k*ps)")
        assert np.array_equal(got[dbytes:], want[dbytes:]), (size, offset, "parity [k*ps, (k+m)*ps)")
    coder.close()


@pytest.mark.gpu
def test_encode_raw_equals_encode_naive(ref, mdir):
    """ugb200_ldgm_encode against encode_naive, at packet sizes of every word width (4, 8, 16 bytes)"""
    from ultragrid_b200 import _lib
    L = _lib.load()
    pcm, s = ref_session(ref, mdir, 512, 384, 5, 7)
    coder = _coder(pcm, 512, 384)
    for ps in (4, 8, 12, 16, 20, 600, 608, 8192, 65532):
        data = np.ascontiguousarray(util.rng_bytes(512 * ps, ps))
        got = np.zeros(384 * ps, dtype=np.uint8)
        assert L.ugb200_ldgm_encode(coder._h, data.ctypes.data, got.ctypes.data, ps) == 0
        assert np.array_equal(got, s.encode_raw(data, ps, True)), (ps, "parity packets")
    coder.close()


@pytest.mark.gpu
def test_encode_golden_without_reference():
    g = np.load(lc.GOLDEN)
    for name in g.files:
        if not name.startswith("enc_"):
            continue
        k, m, c, seed, size = (int(t) for t in name.split("_")[1:])
        key = f"{k}_{m}_{c}_{seed}_{size}"
        coder = _coder(g[f"pcm_{k}_{m}_{c}_{seed}"], k, m)
        got = coder.encode(g[f"frame_{key}"], g[f"hdr_{key}"].tobytes())
        assert np.array_equal(got, g[name]), (name, "whole buffer")
        coder.close()


@pytest.mark.gpu
def test_two_sessions_two_streams_alternating_matrices(ref, mdir):
    import torch
    cases = [(512, 384, 5, 1), (64, 64, 2, 2), (8191, 384, 2, 3), (512, 512, 63, 4)]
    mats = {cs: ref_session(ref, mdir, *cs) for cs in cases}
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    coders = [_coder(mats[cases[0]][0], 512, 384, stream=streams[0]), _coder(mats[cases[1]][0], 64, 64, stream=streams[1])]
    frames = [util.rng_bytes(n, n) for n in (310_001, 1_000_003, 77, 5_000_000)]
    for rnd in range(4):
        pending = []
        for i, coder in enumerate(coders):
            cs = cases[(rnd + 2 * i) % len(cases)]
            coder.set_matrix(mats[cs][0], cs[0], cs[1])
            frame = frames[(rnd + i) % len(frames)]
            src = torch.from_numpy(frame).cuda()
            torch.cuda.synchronize()
            with torch.cuda.stream(streams[i]):
                out = coder.encode(src, b"hd")
            pending.append((cs, frame, out))
        torch.cuda.synchronize()
        for cs, frame, out in pending:
            want = mats[cs][1].encode(b"hd", frame)
            assert np.array_equal(out.cpu().numpy(), want), (rnd, cs, "whole buffer")
    for c in coders:
        c.close()


# ---------------------------------------------------------------- GPU: decode ----------------------------------------------------------

def _patterns(k, m, ps, rng):
    n = k + m
    total = n * ps
    pats = {"no loss": [(0, total)]}
    for pct in (5, 10, 20, 30):
        keep = rng.random(n) >= pct / 100
        pats[f"{pct}% random"] = lc.packets_received(n, ps, keep)
    keep = np.ones(n, bool)
    for start in rng.integers(0, n - 8, size=max(2, n // 64)):
        keep[start:start + int(rng.integers(2, 8))] = False
    pats["bursts"] = lc.packets_received(n, ps, keep)
    keep = np.ones(n, bool)
    keep[k:] = False
    pats["all parity lost"] = lc.packets_received(n, ps, keep)
    keep = np.ones(n, bool)
    keep[k:] = False
    keep[rng.integers(0, k, size=max(1, k // 50))] = False
    pats["all parity and some data lost"] = lc.packets_received(n, ps, keep)
    drop = set(rng.integers(0, total // 1400 + 1, size=max(1, total // 1400 // 12)).tolist())
    pats["1400 B datagrams, some lost (partial packets)"] = lc.rtp_ranges(total, 1400, lambda i: i not in drop)
    halves = []  # adjacent halves merge; a lone first half leaves the packet lost
    for i in range(n):
        r = rng.random()
        if r < 0.85:
            halves += [(i * ps, ps // 2), (i * ps + ps // 2, ps - ps // 2)]
        elif r < 0.95:
            halves.append((i * ps, ps // 2))
    pats["split packets"] = halves
    keep = rng.random(n) >= 0.6
    pats["60% random (beyond peeling)"] = lc.packets_received(n, ps, keep)
    pats["nothing received"] = []
    return pats


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,c,size", [(64, 64, 2, 20_000), (512, 384, 5, 300_017), (512, 512, 63, 1_200_003), (256, 64, 5, 100_000),
                                        (8191, 8191, 5, 7680 * 4320 * 2), (8191, 384, 2, 2_000_000)])
def test_decode_equals_reference(ref, mdir, k, m, c, size):
    pcm, s = ref_session(ref, mdir, k, m, c, 5)
    assert _compare_decodes(s, _coder(pcm, k, m), k, m, size) >= 2  # no loss, and all parity lost, recover at any redundancy


def _compare_decodes(s, coder, k, m, size):
    """every loss pattern decoded by the reference session s and by coder; returns how many patterns recovered the frame"""
    frame = util.rng_bytes(size, size)
    enc = s.encode(b"video-hdr", frame)
    dbytes, ps = lc.layout(k, 9 + size)
    rng = np.random.default_rng(size + k)
    recovered = 0
    for name, ranges in _patterns(k, m, ps, rng).items():
        # lost packets carry garbage, as a receive buffer would
        received = np.frombuffer(rng.bytes(enc.size), dtype=np.uint8).copy()
        for o, n in ranges:
            received[o:o + n] = enc[o:o + n]
        want = received.copy()
        fs_want = s.decode(want, ranges)
        got = received.copy()
        fs_got = coder.decode(got, ranges)
        assert fs_got == fs_want, (name, "*frame_size")
        assert np.array_equal(got[:dbytes], want[:dbytes]), (name, "data packets [0, k*ps)")
        assert np.array_equal(got[dbytes:], want[dbytes:]), (name, "parity packets [k*ps, (k+m)*ps)")
        if fs_want:
            recovered += 1
            assert np.array_equal(got[4 + 9:4 + 9 + size], frame), (name, "recovered frame")
    return recovered


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,c,seed", [(512, 384, 5, 1), (1000, 500, 5, 2), (256, 256, 63, 3)])
def test_decode_generator_matrix_equals_reference(ref, tmp_path, k, m, c, seed):
    """the matrices ldgm.cpp deploys: written by the reference's generate_ldgm_matrix and read by set_pcMatrix (the default
    (512, 384, 5) first)"""
    path = str(tmp_path / "gen.bin")
    assert ref.ref_ldgm_generate(path.encode(), k, m, c, seed) == 0
    s = lc.RefSession(ref, path, k, m, c)
    try:
        assert _compare_decodes(s, _coder(s.pcm(), k, m), k, m, 300_017) >= 2
    finally:
        s.close()


@pytest.mark.gpu
def test_sessions_of_different_sizes_decode_in_turn(ref, mdir):
    """a session with a large matrix (the schedule kernel needs 164 KB of shared memory) keeps decoding after a session with a small
    matrix is set up, and the other way round"""
    big, s_big = ref_session(ref, mdir, 8191, 8191, 5, 6)
    small, s_small = ref_session(ref, mdir, 64, 64, 2, 6)
    c_big = _coder(big, 8191, 8191)
    c_small = _coder(small, 64, 64)
    assert _compare_decodes(s_big, c_big, 8191, 8191, 2_000_000) >= 2
    assert _compare_decodes(s_small, c_small, 64, 64, 20_000) >= 2
    c_small.set_matrix(lc.matrix(512, 384, 5, 6), 512, 384)
    assert _compare_decodes(s_big, c_big, 8191, 8191, 1_000_003) >= 2
    c_big.close(), c_small.close()


@pytest.mark.gpu
def test_decode_uneven_buffer_and_odd_packet_size(ref, mdir):
    """buf_size / (k + m) not a multiple of 4, and bytes past (k + m) * ps, which decode_frame leaves alone"""
    pcm, s = ref_session(ref, mdir, 64, 64, 2, 8)
    coder = _coder(pcm, 64, 64)
    rng = np.random.default_rng(0)
    for ps, extra in ((6, 5), (9, 0), (64, 100)):
        buf = np.frombuffer(rng.bytes(128 * ps + extra), dtype=np.uint8).copy()
        ranges = lc.packets_received(128, ps, rng.random(128) >= 0.15)
        want, got = buf.copy(), buf.copy()
        assert coder.decode(got, ranges) == s.decode(want, ranges), (ps, "*frame_size")
        assert np.array_equal(got, want), (ps, "whole buffer")
    coder.close()


# ---------------------------------------------------------------- GPU: real ABI ---------------------------------------------------------

@pytest.mark.gpu
def test_real_abi_module_in_reference_framework(mdir):
    """ultragrid_b200/modules/ultragrid_ldgm_gpu.so loaded into the unmodified lib_common.cpp registry and found by load_library("ldgm_gpu",
    LIBRARY_CLASS_UNDEFINED, 1) as src/rtp/ldgm.cpp does; it and LDGM_session_cpu driven only through LDGM_session *, compared byte for byte"""
    fw = os.path.join(util.ORACLE_DIR, "_ref", "libldgm_fw.so")
    mod = os.path.join(util.ROOT, "ultragrid_b200", "modules", "ultragrid_ldgm_gpu.so")
    if not (os.path.exists(fw) and os.path.exists(mod) and os.path.exists(lc.REF_PATH)):
        pytest.skip("oracle/_ref/libldgm_fw.so, libldgm_ref.so or the module not built (reference tree absent)")
    L = ctypes.CDLL(fw, mode=ctypes.RTLD_GLOBAL)  # the host binary: the module takes LDGM_session and register_library from it
    vp, i = ctypes.c_void_p, ctypes.c_int
    L.ldf_load_module.argtypes = [ctypes.c_char_p]
    L.ldf_create.argtypes, L.ldf_create.restype = [i], vp
    L.ldf_destroy.argtypes, L.ldf_destroy.restype = [vp], None
    L.ldf_set.argtypes = [vp, i, i, i, ctypes.c_char_p]
    L.ldf_encode.argtypes = [vp, vp, i, vp, i, vp, ctypes.c_long]
    L.ldf_decode.argtypes = [vp, vp, i, vp, i]
    assert L.ldf_load_module(mod.encode()) == 0
    gpu, cpu = L.ldf_create(1), L.ldf_create(0)
    assert gpu, "load_library(\"ldgm_gpu\", LIBRARY_CLASS_UNDEFINED, 1) found no module"
    rng = np.random.default_rng(9)
    ref = lc.ref_lib()
    for k, m, c, seed, generated in ((512, 384, 5, 1, True), (512, 384, 5, 1, False), (256, 256, 63, 2, False), (8191, 8191, 5, 3, False),
                                     (512, 384, 5, 4, False)):
        path = os.path.join(mdir, f"fw-{k}-{m}-{c}-{seed}-{int(generated)}.bin")
        if generated:  # the file ldgm.cpp makes with generate_ldgm_matrix
            assert ref.ref_ldgm_generate(path.encode(), k, m, c, seed) == 0
        else:
            lc.write_matrix_file(path, lc.matrix(k, m, c, seed), k, m)
        assert L.ldf_set(gpu, k, m, c, path.encode()) == 0 and L.ldf_set(cpu, k, m, c, path.encode()) == 0
        for size in (1, 300_017, 1_200_003):
            hdr, frame = util.rng_bytes(24, size).tobytes(), util.rng_bytes(size, size + seed)
            dbytes, ps = lc.layout(k, 24 + size)
            total = dbytes + m * ps
            a, b = np.zeros(total, np.uint8), np.zeros(total, np.uint8)
            assert L.ldf_encode(gpu, hdr, 24, frame.ctypes.data, size, a.ctypes.data, total) == total
            assert L.ldf_encode(cpu, hdr, 24, frame.ctypes.data, size, b.ctypes.data, total) == total
            assert np.array_equal(a, b), (k, m, c, size, "encode_hdr_frame buffer (whole)")
            for loss in (0.0, 0.1, 0.3):
                keep = rng.random(k + m) >= loss
                r = np.array(lc.packets_received(k + m, ps, keep) or [(0, 0)], dtype=np.int32).reshape(-1, 2)
                ga, gb = np.where(np.repeat(keep, ps), a, 0).astype(np.uint8), np.where(np.repeat(keep, ps), b, 0).astype(np.uint8)
                fa = L.ldf_decode(gpu, ga.ctypes.data, total, r.ctypes.data, len(r))
                fb = L.ldf_decode(cpu, gb.ctypes.data, total, r.ctypes.data, len(r))
                assert fa == fb, (k, m, c, size, loss, "*frame_size")
                assert np.array_equal(ga, gb), (k, m, c, size, loss, "decode_frame buffer (whole)")
    L.ldf_destroy(gpu)
    L.ldf_destroy(cpu)


@pytest.mark.gpu
def test_encode_equals_reference_gpu_coder(ref, mdir, tmp_path):
    """the reference's own GPU coder (gpu.cu + ldgm-session-gpu.cpp, built for sm_90a), run in a child process because it exits on a
    CUDA error: its encode_hdr_frame bytes, ours and LDGM_session_cpu's agree"""
    import subprocess
    import sys
    if not os.path.exists(lc.REF_GPU_PATH):
        pytest.skip("oracle/_ref/libldgm_gpu_ref.so not built (reference tree absent)")
    cases = [(512, 384, 5, 1, 1), (512, 384, 5, 1, 300_017), (512, 384, 5, 1, 1_200_003), (64, 64, 2, 2, 20_000), (256, 256, 63, 3, 100_000),
             (8191, 8191, 5, 4, 2_000_000)]
    out = str(tmp_path / "refgpu.npz")
    code = f"import sys; sys.path.insert(0, {os.path.dirname(__file__)!r}); import ldgm_cases; ldgm_cases.refgpu_encode_cases({mdir!r}, {cases!r}, {out!r})"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    got_ref = np.load(out)
    for k, m, c, seed, size in cases:
        pcm, s = ref_session(ref, mdir, k, m, c, seed)
        hdr, frame = lc.ref_frame(size, seed)
        cpu = s.encode(hdr, frame)
        coder = _coder(pcm, k, m)
        ours = coder.encode(frame, hdr)
        coder.close()
        dbytes, _ = lc.layout(k, len(hdr) + size)
        g = got_ref[f"{k}_{m}_{c}_{seed}_{size}"]
        assert np.array_equal(g[dbytes:], cpu[dbytes:]), (k, m, c, size, "reference GPU vs CPU coder: parity [k*ps, (k+m)*ps)")
        assert np.array_equal(ours, g), (k, m, c, size, "ours vs reference GPU coder: whole buffer")
