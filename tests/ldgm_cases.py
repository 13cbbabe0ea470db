"""Helpers of tests/test_ldgm.py: LDGM matrices, the reference coder's extern "C" shim (oracle/_ref/libldgm_ref.so), a numpy model of
the encode, and loss patterns as (offset, length) ranges."""
import ctypes
import os

import numpy as np

import util

_vp, _i, _l, _u = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_uint
REF_PATH = os.path.join(util.ORACLE_DIR, "_ref", "libldgm_ref.so")
GOLDEN = os.path.join(util.ROOT, "tests", "golden", "ldgm_golden.npz")


def ref_lib():
    """the unmodified reference coder, or None when it has not been built (reference tree absent)"""
    if not os.path.exists(REF_PATH):
        return None
    L = ctypes.CDLL(REF_PATH)
    L.ref_ldgm_generate.argtypes = [ctypes.c_char_p, _u, _u, _u, _u]
    L.ref_ldgm_create.argtypes = [ctypes.c_char_p, _i, _i, _i]
    L.ref_ldgm_create.restype = _vp
    L.ref_ldgm_destroy.argtypes = [_vp]
    L.ref_ldgm_destroy.restype = None
    L.ref_ldgm_pcm.argtypes = [_vp, _i, _vp, _l]
    L.ref_ldgm_encode_hdr_frame.argtypes = [_vp, _vp, _i, _vp, _i, _vp, _l]
    L.ref_ldgm_encode_raw.argtypes = [_vp, _vp, _vp, _i, _i]
    L.ref_ldgm_encode_raw.restype = None
    L.ref_ldgm_decode.argtypes = [_vp, _vp, _i, _vp, _i]
    return L


def matrix(k, m, c, seed):
    """an LDGM matrix in set_pcMatrix's compact form (m rows of w_f = max row weight + 2 ints): c ones per data column in distinct
    random rows, data indices ascending, then the staircase k+j and k+j-1, padded with -1 - the shape generate_ldgm_matrix writes,
    from numpy's generator so that every (k, m, c) of the coder's range can be made"""
    rng = np.random.default_rng(seed)
    rows = [[] for _ in range(m)]
    for col in range(k):
        for j in rng.choice(m, size=min(c, m), replace=False):
            rows[j].append(col)
    for j in range(m):  # no row with fewer than two data packets, as left_matrix_init ensures
        while len(rows[j]) < min(2, k):
            col = int(rng.integers(k))
            if col not in rows[j]:
                rows[j].append(col)
    w_f = max(len(r) for r in rows) + 2
    pcm = np.full((m, w_f), -1, dtype=np.int32)
    for j, r in enumerate(rows):
        e = sorted(r) + [k + j] + ([k + j - 1] if j else [])
        pcm[j, :len(e)] = e
    return pcm


def write_matrix_file(path, pcm, k, m):
    """the file format generate_ldgm_matrix writes and set_pcMatrix reads: "k m w_f\\n" then m*w_f native ints"""
    with open(path, "wb") as f:
        f.write(f"{k} {m} {pcm.shape[1]}\n".encode())
        f.write(np.ascontiguousarray(pcm, dtype=np.int32).tobytes())


def read_matrix_file(path):
    """(k, m, pcm) of a matrix file, parsed as set_pcMatrix does (three integers, one separator byte, the ints)"""
    raw = open(path, "rb").read()
    nl = raw.index(b"\n")
    k, m, w_f = (int(t) for t in raw[:nl].split())
    pcm = np.frombuffer(raw[nl + 1:nl + 1 + 4 * m * w_f], dtype=np.int32).reshape(m, w_f)
    return k, m, pcm.copy()


def layout(k, payload):
    """(data bytes, packet size) of encode_hdr_frame for a header + frame of payload bytes"""
    align = 4 * k
    data = (payload + 4 + align - 1) // align * align
    return data, data // k


def model_parity(pcm, k, data):
    """parity[j] = parity[j-1] ^ XOR{ data[i] : i in row j, 0 <= i < k } with data as (k, ps) uint8"""
    m = pcm.shape[0]
    r = np.zeros((m, data.shape[1]), dtype=np.uint8)
    for e in range(pcm.shape[1]):
        col = pcm[:, e]
        sel = (col > -1) & (col < k)
        r[sel] ^= data[col[sel]]
    return np.bitwise_xor.accumulate(r, axis=0)


def model_encode(pcm, k, m, hdr, frame):
    """the whole encode_hdr_frame buffer"""
    payload = len(hdr) + len(frame)
    dbytes, ps = layout(k, payload)
    buf = np.zeros(dbytes + m * ps, dtype=np.uint8)
    buf[:4] = np.frombuffer(np.int32(payload).tobytes(), dtype=np.uint8)
    buf[4:4 + len(hdr)] = np.frombuffer(bytes(hdr), dtype=np.uint8)
    buf[4 + len(hdr):4 + payload] = np.frombuffer(bytes(frame), dtype=np.uint8) if isinstance(frame, (bytes, bytearray)) else frame
    buf[dbytes:] = model_parity(pcm, k, buf[:dbytes].reshape(k, ps)).reshape(-1)
    return buf


class RefSession:
    """LDGM_session_cpu of the reference with set_params + set_pcMatrix on a matrix file"""

    def __init__(self, L, path, k, m, c):
        self.L, self.k, self.m = L, k, m
        self.h = L.ref_ldgm_create(path.encode(), k, m, c)
        assert self.h, "set_pcMatrix refused the matrix file"

    def close(self):
        if self.h:
            self.L.ref_ldgm_destroy(self.h)
        self.h = None

    def pcm(self):
        w_f = self.L.ref_ldgm_pcm(self.h, self.m, None, 0)
        out = np.empty((self.m, w_f), dtype=np.int32)
        self.L.ref_ldgm_pcm(self.h, self.m, out.ctypes.data, out.size)
        return out

    def encode(self, hdr, frame):
        payload = len(hdr) + len(frame)
        dbytes, ps = layout(self.k, payload)
        out = np.empty(dbytes + self.m * ps, dtype=np.uint8)
        hdr_b, frame_b = bytes(hdr), np.ascontiguousarray(np.frombuffer(bytes(frame), dtype=np.uint8))
        n = self.L.ref_ldgm_encode_hdr_frame(self.h, hdr_b, len(hdr_b), frame_b.ctypes.data, frame_b.size, out.ctypes.data, out.size)
        assert n == out.size
        return out

    def encode_raw(self, data, ps, naive):
        parity = np.zeros(self.m * ps, dtype=np.uint8)
        self.L.ref_ldgm_encode_raw(self.h, data.ctypes.data, parity.ctypes.data, ps, 1 if naive else 0)
        return parity

    def decode(self, buf, ranges):
        r = np.ascontiguousarray(np.array(ranges, dtype=np.int32).reshape(-1, 2))
        return self.L.ref_ldgm_decode(self.h, buf.ctypes.data, buf.size, r.ctypes.data, len(r))


def packets_received(n_packets, ps, keep):
    """one range per received packet (keep: bool array over the k + m packets)"""
    return [(i * ps, ps) for i in range(n_packets) if keep[i]]


def rtp_ranges(total, chunk, keep_chunk):
    """the buffer cut into chunk-byte datagrams as RTP would carry it, with the datagrams keep_chunk(i) accepts: packets straddling a
    lost datagram are partially received"""
    return [(o, min(chunk, total - o)) for i, o in enumerate(range(0, total, chunk)) if keep_chunk(i)]


REF_GPU_PATH = os.path.join(util.ORACLE_DIR, "_ref", "libldgm_gpu_ref.so")


def refgpu_encode_cases(matrix_dir, cases, out_npz):
    """child-process side of the reference GPU coder (it exits the process on a CUDA error): encode_hdr_frame of every
    (k, m, c, seed, size) case, with the frames and headers of ref_frame(), into out_npz"""
    L = ctypes.CDLL(REF_GPU_PATH)
    L.refgpu_ldgm_create.argtypes, L.refgpu_ldgm_create.restype = [ctypes.c_char_p, _i, _i, _i], _vp
    L.refgpu_ldgm_destroy.argtypes, L.refgpu_ldgm_destroy.restype = [_vp], None
    L.refgpu_ldgm_encode_hdr_frame.argtypes = [_vp, _vp, _i, _vp, _i, _vp, _l]
    out = {}
    for k, m, c, seed, size in cases:
        path = os.path.join(matrix_dir, f"gpuref-{k}-{m}-{c}-{seed}.bin")
        write_matrix_file(path, matrix(k, m, c, seed), k, m)
        h = L.refgpu_ldgm_create(path.encode(), k, m, c)
        hdr, frame = ref_frame(size, seed)
        dbytes, ps = layout(k, len(hdr) + size)
        buf = np.zeros(dbytes + m * ps, dtype=np.uint8)
        assert L.refgpu_ldgm_encode_hdr_frame(h, hdr, len(hdr), frame.ctypes.data, size, buf.ctypes.data, buf.size) == buf.size
        out[f"{k}_{m}_{c}_{seed}_{size}"] = buf
        L.refgpu_ldgm_destroy(h)
    np.savez(out_npz, **out)


def ref_frame(size, seed):
    return util.rng_bytes(24, seed).tobytes(), util.rng_bytes(size, size + seed)
