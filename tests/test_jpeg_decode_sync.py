"""The self-synchronising Huffman route of the JPEG decoder (ultragrid_b200/csrc/jpeg_huffman_step.cuh, jpeg_sync_*_kernel): the same coefficients as
the one-thread-per-segment route for ANY bytes.

CPU: the shared header compiled for the host; a shim runs the route's phases sequentially (one simulated thread per subsequence, the same rounds,
counts and prefix sums) and a plain serial loop over the same header.  Valid streams are also compared with jpeg_exact.read.
GPU: ugb200_jpeg_decode with the route against the forced one-thread route (UGB200_JPEG_SYNC=off) and the CPU oracle."""
import ctypes
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

import jpeg_exact as J
import util
from test_jpeg import natural_rgb
from test_jpeg_exact import STD_TABLES, _writer_frame, four_scans_redefined, writer_streams

SHIM = r'''
#include <vector>
#include "jpeg_huffman_step.cuh"
using namespace ugb;

struct host_sink {
        int16_t *blk;
        bool inside;
        void dc(uint32_t p) { if (inside) blk[0] = (int16_t) p; }
        void operator()(int i, int v) { static const uint8_t zz[64] = { 0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48,
                41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                61, 54, 47, 55, 62, 63 }; if (inside) blk[zz[i]] = (int16_t) v; }
};

static void geometry(const int *geo, dec_geom &g)
{
        g = dec_geom{};
        g.w = geo[0], g.h = geo[1], g.ncomp = geo[2], g.ri = geo[3], g.nscans = geo[4];
        g.hmax = g.vmax = 1;
        for (int i = 0; i < g.ncomp; ++i) {
                g.c[i].h = geo[5 + 2 * i], g.c[i].v = geo[6 + 2 * i];
                g.hmax = g.c[i].h > g.hmax ? g.c[i].h : g.hmax, g.vmax = g.c[i].v > g.vmax ? g.c[i].v : g.vmax;
        }
        int blk = 0, seg = 0;
        for (int i = 0; i < g.ncomp; ++i) {
                dec_comp &c = g.c[i];
                c.bw = (g.w + 8 * g.hmax - 1) / (8 * g.hmax) * c.h, c.bh = (g.h + 8 * g.vmax - 1) / (8 * g.vmax) * c.v;
                c.blk_off = blk, blk += c.bw * c.bh;
        }
        g.nblocks = blk;
        const int *sp = geo + 5 + 2 * g.ncomp;
        for (int j = 0; j < g.nscans; ++j, sp += 13) {
                dec_scan &S = g.s[j];
                S.ns = sp[0];
                for (int k = 0; k < 4; ++k) {
                        S.comp[k] = sp[1 + k], S.td[k] = sp[5 + k], S.ta[k] = sp[9 + k];
                }
                int mcuy;
                if (S.ns == 1) {
                        const dec_comp &c = g.c[S.comp[0]];
                        S.mcux = ((g.w * c.h + g.hmax - 1) / g.hmax + 7) / 8, mcuy = ((g.h * c.v + g.vmax - 1) / g.vmax + 7) / 8;
                } else {
                        S.mcux = (g.w + 8 * g.hmax - 1) / (8 * g.hmax), mcuy = (g.h + 8 * g.vmax - 1) / (8 * g.vmax);
                }
                S.nmcu = S.mcux * mcuy;
                S.seg0 = seg, S.nseg = g.ri ? (S.nmcu + g.ri - 1) / g.ri : 1;
                seg += S.nseg;
        }
}

static void segment_scan(const dec_geom &g, int s, dec_scan &S, int &m0, int &m1)
{
        int sc = 0;
        while (s >= g.s[sc].seg0 + g.s[sc].nseg) {
                ++sc;
        }
        S = g.s[sc];
        const int ls = s - S.seg0;
        m0 = g.ri ? ls * g.ri : 0, m1 = g.ri ? (m0 + g.ri < S.nmcu ? m0 + g.ri : S.nmcu) : S.nmcu;
}

static host_sink sink_at(const dec_geom &g, const dec_scan &S, const mcu_layout &L, int16_t *coef, int m, int b)
{
        const int k = L.k[b], mx = m % S.mcux, my = m / S.mcux;
        const dec_comp &c = g.c[S.comp[k]];
        const int nh = S.ns == 1 ? 1 : c.h, nv = S.ns == 1 ? 1 : c.v, X = mx * nh + L.bx[b], Y = my * nv + L.by[b];
        return { coef + ((long) c.blk_off + (long) Y * c.bw + X) * 64, X < c.bw && Y < c.bh };
}

/// sub == 0: the plain serial loop; otherwise the self-synchronising route with subsequences of `sub` bytes.  coef: zeroed [nblocks][64]
extern "C" int sim(const uint8_t *s, int ntab, const uint8_t *tabs, const int *geo, const uint32_t *sb, const uint32_t *se, int nseg, int sub, int16_t *coef)
{
        static dec_tables T;
        memset(&T, 0, sizeof T);
        for (int k = 0; k < ntab; ++k) {
                int n = 0;
                for (int i = 0; i < 16; ++i) {
                        n += tabs[272 * k + i];
                }
                build_table(T, k, tabs + 272 * k, tabs + 272 * k + 16, n);
        }
        dec_geom g;
        geometry(geo, g);
        if (sub == 0) {
                for (int seg = 0; seg < nseg; ++seg) {
                        dec_scan S;
                        int m0, m1;
                        segment_scan(g, seg, S, m0, m1);
                        const mcu_layout L = layout_of(g, S);
                        pos_reader r;
                        r.s = s, r.end = se[seg];
                        r.start(sb[seg], 0);
                        uint32_t pred[4] = { 0, 0, 0, 0 };
                        for (int m = m0; m < m1; ++m) {
                                for (int b = 0; b < L.bpm; ++b) {
                                        decode_block(r, &T, S.td[L.k[b]], S.ta[L.k[b]], pred[L.k[b]], sink_at(g, S, L, coef, m, b));
                                }
                        }
                }
                return 0;
        }
        // the phases of jpeg_sync_kernel / jpeg_sync_write_kernel, one simulated thread after the other
        std::vector<uint32_t> first(nseg + 1, 0);
        for (int seg = 0; seg < nseg; ++seg) {
                first[seg + 1] = first[seg] + (uint32_t) sub_count(se[seg] - sb[seg], sub);
        }
        const uint32_t nsub = first[nseg];
        std::vector<int> segof(nsub);
        for (int seg = 0; seg < nseg; ++seg) {
                for (uint32_t j = first[seg]; j < first[seg + 1]; ++j) {
                        segof[j] = seg;
                }
        }
        std::vector<sync_point> entry(nsub), exitp(nsub);
        std::vector<uint32_t> res(5 * (size_t) nsub, 0), dirty(nsub, 1);
        for (uint32_t j = 0; j < nsub; ++j) {
                const int seg = segof[j];
                entry[j] = make_point(sub_start(s, sb[seg], se[seg], (int) (j - first[seg]), sub), 0, 0);
        }
        int round = 0;
        for (;; ++round) {
                for (uint32_t j = 0; j < nsub; ++j) {
                        const int seg = segof[j];
                        if (!dirty[j] || j + 1 == first[seg + 1]) {
                                continue;
                        }
                        dec_scan S;
                        int m0, m1;
                        segment_scan(g, seg, S, m0, m1);
                        const mcu_layout L = layout_of(g, S);
                        pos_reader r;
                        r.s = s, r.end = se[seg];
                        r.start(entry[j].byte, (int) (entry[j].tag >> 16));
                        int blk = (entry[j].tag >> 8) & 0xff, zz = entry[j].tag & 0xff;
                        uint32_t count = 0, sum[4] = { 0, 0, 0, 0 };
                        walk_count(r, &T, S.td, S.ta, L, sub_start(s, sb[seg], se[seg], (int) (j + 1 - first[seg]), sub), blk, zz, count, sum);
                        exitp[j] = make_point(r.pos(), blk, zz);
                        res[j] = count;
                        for (int v = 0; v < 4; ++v) {
                                res[(v + 1) * (size_t) nsub + j] = sum[v];
                        }
                }
                uint32_t changed = 0;
                for (uint32_t j = 0; j < nsub; ++j) {
                        const int seg = segof[j];
                        if (j == first[seg]) {
                                dirty[j] = 0;
                        }
                        if (j + 1 == first[seg + 1]) {
                                continue;
                        }
                        const bool moved = exitp[j].byte != entry[j + 1].byte || exitp[j].tag != entry[j + 1].tag;
                        if (moved) {
                                entry[j + 1] = exitp[j];
                        }
                        dirty[j + 1] = moved;
                        changed += moved;
                }
                if (changed == 0) {
                        break;
                }
        }
        std::vector<uint32_t> scan(5 * (size_t) nsub);
        for (int v = 0; v < 5; ++v) {
                uint32_t run = 0;
                for (uint32_t j = 0; j < nsub; ++j) {
                        scan[v * (size_t) nsub + j] = run;
                        run += res[v * (size_t) nsub + j];
                }
        }
        for (uint32_t j = 0; j < nsub; ++j) {
                const int seg = segof[j];
                dec_scan S;
                int m0, m1;
                segment_scan(g, seg, S, m0, m1);
                const mcu_layout L = layout_of(g, S);
                const uint32_t f = first[seg], nblk = (uint32_t) (m1 - m0) * (uint32_t) L.bpm;
                uint32_t idx = scan[j] - scan[f], pred[4];
                for (int v = 0; v < 4; ++v) {
                        pred[v] = scan[(v + 1) * (size_t) nsub + j] - scan[(v + 1) * (size_t) nsub + f];
                }
                if (idx >= nblk) {
                        continue;
                }
                pos_reader r;
                r.s = s, r.end = se[seg];
                r.start(entry[j].byte, (int) (entry[j].tag >> 16));
                const int zz = entry[j].tag & 0xff;
                if (zz) {
                        finish_block(r, &T, S.ta[L.k[(entry[j].tag >> 8) & 0xff]], zz);
                }
                const uint64_t limit = j + 1 == first[seg + 1] ? ~(uint64_t) 0 : sub_start(s, sb[seg], se[seg], (int) (j + 1 - f), sub);
                while (idx < nblk && r.pos() < limit) {
                        const int m = m0 + (int) (idx / (uint32_t) L.bpm), b = (int) (idx % (uint32_t) L.bpm);
                        decode_block(r, &T, S.td[L.k[b]], S.ta[L.k[b]], pred[L.k[b]], sink_at(g, S, L, coef, m, b));
                        ++idx;
                }
        }
        return round + 1;
}
'''


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("huffman_sync")
    src, so = d / "shim.cpp", d / "libshim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(util.ROOT, "ultragrid_b200", "csrc"), str(src), "-o", str(so)],
                   check=True, capture_output=True)
    lib = ctypes.CDLL(str(so))
    lib.sim.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return lib


def headers(s):
    """what the decoder's parser takes from the stream: geometry, restart interval and per scan its components and Huffman tables (as they stand at
    its SOS); the tables become slots, one per distinct definition"""
    a = np.frombuffer(s, np.uint8)
    p, huff, comps, scans, ri, wh, slots = 2, {}, [], [], 0, None, []
    while p + 4 <= len(a):
        mk = int(a[p + 1])
        if mk == 0xD9:
            break
        if mk == 0xFF:
            p += 1
            continue
        L = int(a[p + 2]) << 8 | int(a[p + 3])
        d = bytes(a[p + 4:p + 2 + L])
        if mk == 0xC4:
            i = 0
            while i < len(d):
                n = sum(d[i + 1:i + 17])
                huff[(d[i] >> 4, d[i] & 15)] = d[i + 1:i + 17] + d[i + 17:i + 17 + n]
                i += 17 + n
        elif mk == 0xC0:
            wh = (d[3] << 8 | d[4], d[1] << 8 | d[2])
            comps = [(d[6 + 3 * c], d[7 + 3 * c] >> 4, d[7 + 3 * c] & 15) for c in range(d[5])]
        elif mk == 0xDD:
            ri = d[0] << 8 | d[1]
        elif mk == 0xDA:
            sc = []
            for i in range(d[0]):
                ci = next(j for j, c in enumerate(comps) if c[0] == d[1 + 2 * i])
                ids = []
                for key in ((0, d[2 + 2 * i] >> 4), (1, d[2 + 2 * i] & 15)):
                    if huff[key] not in slots:
                        slots.append(huff[key])
                    ids.append(slots.index(huff[key]))
                sc.append((ci, ids[0], ids[1]))
            scans.append(sc)
            p += 2 + L
            while p + 1 < len(a) and not (a[p] == 0xFF and a[p + 1] not in (0x00, 0xFF) and not 0xD0 <= a[p + 1] <= 0xD7):
                p += 1
            continue
        p += 2 + L
    geo = [wh[0], wh[1], len(comps), ri, len(scans)] + [x for c in comps for x in c[1:]]
    for sc in scans:
        geo += [len(sc)] + [c[0] for c in sc] + [0] * (4 - len(sc)) + [c[1] for c in sc] + [0] * (4 - len(sc)) + [c[2] for c in sc] + [0] * (4 - len(sc))
    tabs = np.zeros((max(1, len(slots)), 272), np.uint8)
    for k, t in enumerate(slots):
        tabs[k, :len(t)] = np.frombuffer(t, np.uint8)
    assert len(slots) <= 8
    return np.array(geo, np.int32), tabs, len(slots), comps, wh


def run(shim, s, sub, hdr=None):
    """coefficients [nblocks, 64] (natural order) of the shim, and the rounds it needed (0 for the serial loop)"""
    from ultragrid_b200 import _lib
    lib = _lib.load()
    geo, tabs, ntab, comps, (w, h) = hdr or headers(s)
    a = np.frombuffer(s, np.uint8).copy()
    cap = 1 << 16
    sb, se = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    nseg = lib.ugb200_jpeg_debug_segments(a.ctypes.data, len(a), sb.ctypes.data, se.ctypes.data, cap)
    assert 0 < nseg <= cap, nseg
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    nblocks = sum(-(-w // (8 * hmax)) * c[1] * -(-h // (8 * vmax)) * c[2] for c in comps)
    coef = np.zeros((nblocks, 64), np.int16)
    rounds = shim.sim(a.ctypes.data, ntab, tabs.ctypes.data, geo.ctypes.data, sb.ctypes.data, se.ctypes.data, nseg, sub, coef.ctypes.data)
    return coef, rounds


def reader_coefficients(s, comps, wh):
    """jpeg_exact.read's coefficients in the decoder's [block][64] layout (padded planes, blocks no scan codes stay zero)"""
    fr = J.read(s)
    w, h = wh
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    out = []
    for ci, c in enumerate(comps):
        bw, bh = -(-w // (8 * hmax)) * c[1], -(-h // (8 * vmax)) * c[2]
        plane = np.zeros((bh, bw, 64), np.int64)
        gh, gw = fr.grid[ci]
        plane[:gh, :gw] = fr.coef[ci][:gh, :gw]
        out.append(plane.reshape(-1, 64))
    return np.concatenate(out)


SUBS = (4, 5, 8, 64, 1024)


def pil(rgb, q, subsampling, optimize=False, restart_blocks=0):
    b = io.BytesIO()
    kw = {"restart_marker_blocks": restart_blocks} if restart_blocks else {}
    Image.fromarray(rgb).save(b, "JPEG", quality=q, subsampling=subsampling, optimize=optimize, **kw)
    return b.getvalue()


def valid_corpus():
    rgb = natural_rgb(77, 45, 3)
    out = [(f"pil ss{ss} q{q} opt{int(o)}", pil(rgb, q, ss, o)) for ss in (0, 1, 2) for q in (5, 50, 95, 100) for o in (False, True)]
    names = {"codes-10-16-il", "codes-9-il", "zrl-eob-corners", "q255-extreme", "no-dri", "dht-redefined", "ycc422-long"}
    out += [(n, s) for n, s in writer_streams() if n in names]
    out.append(("dht-redefined-4-scans", four_scans_redefined()))
    # per-component scans of 4:2:0 without DRI: the chroma grids are smaller than the padded planes (MCU padding, non-FULL)
    w, h = 45, 27
    coef = _writer_frame(w, h, 2, 2)
    out.append(("420-three-scans", J.write(w, h, [(1, 2, 2, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef, {0: np.full(64, 3), 1: np.full(64, 5)}, STD_TABLES,
                                            [[(0, 0, 0)], [(1, 1, 1)], [(2, 1, 1)]], ri=0)))
    return out


def test_sync_route_equals_reader_and_serial_loop_on_valid_streams(shim):
    """every subsequence length puts boundaries at other bit phases and inside other kinds of symbol"""
    for name, s in valid_corpus():
        hdr = headers(s)
        want = reader_coefficients(s, hdr[3], hdr[4])
        ser, _ = run(shim, s, 0, hdr)
        assert np.array_equal(ser, want), name
        for sub in SUBS:
            got, rounds = run(shim, s, sub, hdr)
            assert rounds >= 1 and np.array_equal(got, want), (name, sub)


def stuffed_everywhere():
    """a stream whose entropy-coded data is mostly 0xFF 0x00 pairs: with 5-byte subsequences some boundary falls on every byte of a pair, plus
    one lone 0xFF inside the data (a damaged stream the decoder still reads)"""
    w, h = 64, 32
    dc = ([0, 2] + [0] * 14, [0, 1])
    # one code of every length 1..16: the 16-bit one, 1111111111111110, codes AC +1 (value bit 1), so the data is mostly 0xFF 0x00 pairs
    ac = ([1] * 16, [0x00, 0x02, 0x03, 0x04, 0x05, 0x06, 0x07, 0x08, 0x09, 0x0A, 0x11, 0x12, 0x13, 0x14, 0x15, 0x01])
    coef2 = [np.zeros((4, 8, 64), np.int64) for _ in range(3)]
    for c in coef2:
        c[..., 1:] = 1
    tables = {(0, 0): dc, (1, 0): ac, (0, 1): dc, (1, 1): ac}
    s = J.write(w, h, [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef2, {0: np.full(64, 2), 1: np.full(64, 2)}, tables,
                [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]], ri=0)
    a = bytearray(s)
    pairs = sum(1 for i in range(len(a) - 1) if a[i] == 0xFF and a[i + 1] == 0)
    assert pairs > 100
    sos = a.index(b"\xff\xda")
    i = sos + 200
    while not (a[i] == 0xFF and a[i + 1] == 0):
        i += 1
    a.insert(i, 0xFF)  # a lone 0xFF in front of a stuffed pair: FF FF 00 reads as FF FF
    return bytes(a)


def test_stuffed_pairs_at_every_boundary(shim):
    s = stuffed_everywhere()
    want, _ = run(shim, s, 0)
    for sub in (1, 2, 3, 4, 5, 7, 8, 64):
        got, _ = run(shim, s, sub)
        assert np.array_equal(got, want), sub


def damaged_corpus(seed=0):
    rng = np.random.default_rng(seed)
    base = pil(natural_rgb(120, 72, 9), 85, 2)
    a0 = np.frombuffer(base, np.uint8)
    sos = int(np.flatnonzero((a0[:-1] == 0xFF) & (a0[1:] == 0xDA))[0])
    begin = sos + 2 + (int(a0[sos + 2]) << 8 | int(a0[sos + 3]))
    out = []
    for k in range(12):  # truncation at random points (the data runs out: the rest decodes from zero bits)
        out.append((f"truncated {k}", bytes(a0[:int(rng.integers(begin + 1, len(a0) - 2))])))
    for k in range(12):  # random bytes inside the scan
        a = a0.copy()
        for _ in range(int(rng.integers(1, 6))):
            a[int(rng.integers(begin, len(a) - 2))] = rng.integers(0, 256)
        out.append((f"bytes {k}", bytes(a)))
    a = a0.copy()  # a run of 0xFE 0xFF...: codes that are in no table
    p = begin + (len(a) - begin) // 3
    a[p:p + 40] = 0xFE
    out.append(("undefined codes", bytes(a)))
    out.append(("trailing garbage", bytes(a0[:-2]) + bytes(rng.integers(0, 255, 3000, dtype=np.uint8)) + b"\xff\xd9"))
    return out


def test_sync_route_equals_serial_loop_on_damaged_streams(shim):
    for name, s in damaged_corpus():
        hdr = headers(s)
        want, _ = run(shim, s, 0, hdr)
        for sub in (4, 5, 64):
            got, _ = run(shim, s, sub, hdr)
            assert np.array_equal(got, want), (name, sub)


def adversarial_stream():
    """Synchronisation is slow when a wrong start state never meets the right one: all data bits are zero, a block is an 8-bit DC code and 63
    AC units of a 9-bit code and one value bit (638 bits, a period incommensurate with the byte-aligned subsequence starts).  A guessed state stays
    out of phase with the true one, so each round proves one more subsequence only."""
    w, h = 64, 16
    dc = ([0] * 7 + [12] + [0] * 8, list(range(12)))
    ac = ([0] * 8 + [2] + [0] * 7, [0x01, 0x00])
    coef = [np.zeros((h // 8, w // 8, 64), np.int64) for _ in range(3)]
    for c in coef:
        c[..., 1:] = -1
    tables = {(0, 0): dc, (1, 0): ac, (0, 1): dc, (1, 1): ac}
    return J.write(w, h, [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef, {0: np.full(64, 2), 1: np.full(64, 2)}, tables,
                   [[(0, 0, 0), (1, 1, 1), (2, 1, 1)]], ri=0)


ADVERSARIAL_MIN_ROUNDS = 8


def test_adversarial_stream_needs_many_rounds_and_stays_exact(shim):
    s = adversarial_stream()
    hdr = headers(s)
    want = reader_coefficients(s, hdr[3], hdr[4])
    got, _ = run(shim, s, 0, hdr)
    assert np.array_equal(got, want)
    got, rounds = run(shim, s, 8, hdr)
    assert np.array_equal(got, want)
    assert rounds > ADVERSARIAL_MIN_ROUNDS, rounds


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------------------
def _decoder(monkeypatch, sync=None, scan=None):
    from ultragrid_b200 import api
    for var, val in (("UGB200_JPEG_SYNC", sync), ("UGB200_JPEG_MARKER_SCAN", scan)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)  # read when the decoder is created
    dec = api.JpegDecoder()
    monkeypatch.delenv("UGB200_JPEG_SYNC", raising=False)
    monkeypatch.delenv("UGB200_JPEG_MARKER_SCAN", raising=False)
    return dec


def _decode(dec, s, codec, device=False, shifts=(0, 8, 16)):
    from ultragrid_b200 import api
    try:
        out = dec.decode(s, codec, shifts=shifts, device=device)
    except RuntimeError as e:
        return str(e)
    return out.cpu().numpy() if device else out


def _outputs(info):
    from test_jpeg_decode import I420, RGBA, VUYA
    from test_jpeg import RGB, UYVY
    out = [(info.native_codec, (0, 8, 16)), (UYVY, (0, 8, 16)), (RGB, (0, 8, 16)), (RGBA, (0, 8, 16)), (RGBA, (16, 8, 0)), (VUYA, (0, 8, 16))]
    if info.h_samp == 2:
        out.append((I420, (0, 8, 16)))
    return out


def gpu_corpus():
    out = []
    for (w, h) in ((1, 1), (17, 9), (333, 211), (1919, 1081)):
        rgb = natural_rgb(w, h, 11)
        for ss in (0, 1, 2):
            out.append((f"pil {w}x{h} ss{ss} q90", pil(rgb, 90, ss)))
        out.append((f"pil {w}x{h} ss2 q5 opt", pil(rgb, 5, 2, True)))
    rgb = natural_rgb(3840, 2160, 12)
    out += [(f"pil 4K ss{ss}", pil(rgb, 90, ss)) for ss in (1, 2)]
    out += valid_corpus()[24:]
    return out


@pytest.mark.gpu
def test_gpu_sync_route_equals_serial_route_and_oracle(orc, monkeypatch):
    from test_jpeg_decode import orc_decode
    from ultragrid_b200 import api
    sync, serial, forced = _decoder(monkeypatch), _decoder(monkeypatch, "off"), _decoder(monkeypatch, "on")
    for name, s in gpu_corpus():
        info = api.jpeg_image_info(s)
        for codec, shifts in _outputs(info):
            # to a host buffer, a 4:2:2 frame of odd width converted to RGBA keeps the last pixel of each row from the decoder's staging buffer
            # (the line converter writes whole pixel pairs), whatever the route: those outputs are compared on the device only
            odd_rgba = codec == 1 and info.width % 2 == 1 and info.h_samp == 2
            for device in ((True,) if odd_rgba else (False, True)):
                a, b, c = (_decode(d, s, codec, device, shifts) for d in (sync, serial, forced))
                for x in (a, c):
                    assert type(x) is type(b) and (isinstance(x, str) and x == b or np.array_equal(x, b)), (name, codec, shifts, device)
        st = sync.last_sync()
        if info.restart_interval == 0:  # the writer's streams with short intervals take the route only when it is forced
            assert st["scans"] >= 1 and (st["subsequences"] > 1 or info.width * info.height < 1000), (name, st)
        assert forced.last_sync()["scans"] >= 1, name
        if name.startswith("pil") and info.h_samp == 2 and info.v_samp == 1:  # the CPU decode oracle, byte for byte (as test_gpu_decoder_equals_oracle)
            from test_jpeg import UYVY
            _, want = orc_decode(orc, s, 0, info.width, info.height)
            assert np.array_equal(_decode(sync, s, UYVY), want), name
    sync.close(), serial.close(), forced.close()


@pytest.mark.gpu
def test_gpu_8k_and_forced_small_subsequences(monkeypatch):
    from test_jpeg import UYVY
    rgb8 = natural_rgb(7680, 4320, 13)
    noise = np.random.default_rng(3).integers(0, 256, (4320, 7680, 3), dtype=np.uint8)
    streams = [("8K natural 420 q90", pil(rgb8, 90, 2)), ("8K noise 420 q90", pil(noise, 90, 2)),
               ("1080p 422 q75", pil(natural_rgb(1920, 1080, 14), 75, 1))]
    serial = _decoder(monkeypatch, "off")
    sync, small = _decoder(monkeypatch), _decoder(monkeypatch, "on:8")
    for name, s in streams:
        want = _decode(serial, s, UYVY, True)
        assert np.array_equal(_decode(sync, s, UYVY, True), want), name
        st = sync.last_sync()
        assert st["subsequences"] > 1000, (name, st)
        if name.startswith("1080p"):
            assert np.array_equal(_decode(small, s, UYVY, True), want), name
            st8 = small.last_sync()
            print(f"[stats] {name}: 64 B {st}, 8 B {st8}")
            assert st8["subsequences"] > 7 * st["subsequences"]
    for d in (serial, sync, small):
        d.close()


@pytest.mark.gpu
def test_gpu_route_selection(monkeypatch):
    from test_jpeg import UYVY
    rgb = natural_rgb(640, 360, 15)
    dec = _decoder(monkeypatch)
    _decode(dec, pil(rgb, 85, 1), UYVY)
    assert dec.last_sync()["scans"] == 1
    _decode(dec, pil(rgb, 85, 1, restart_blocks=4), UYVY)  # 4 blocks = 1 MCU per interval: one thread per segment
    assert dec.last_sync() == {"scans": 0, "subsequences": 0, "rounds": 0}
    dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("scan", ["host", "device"])
def test_gpu_both_marker_scans_on_large_streams(orc, monkeypatch, scan):
    from test_jpeg import RGB, UYVY
    s422 = pil(natural_rgb(3840, 2160, 16), 90, 1)
    assert len(s422) >= 1 << 20
    # one scan per component in component order, no DRI, Adobe transform 0: the device multi-scan path (forced "device" takes it at any size)
    w, h = 640, 360
    coef = _writer_frame(w, h, rng=np.random.default_rng(16))
    three = J.write(w, h, [(1, 1, 1, 0), (2, 1, 1, 1), (3, 1, 1, 1)], coef, {0: np.full(64, 3), 1: np.full(64, 5)}, STD_TABLES,
                    [[(0, 0, 0)], [(1, 1, 1)], [(2, 1, 1)]], ri=0, adobe=0)
    serial = _decoder(monkeypatch, "off", scan)
    sync = _decoder(monkeypatch, None, scan)
    for s, codec in ((s422, UYVY), (three, RGB)):
        assert np.array_equal(_decode(sync, s, codec, True), _decode(serial, s, codec, True))
        st = sync.last_sync()
        assert st["scans"] == (1 if codec == UYVY else 3) and st["subsequences"] > 100, st
    sync.close(), serial.close()


@pytest.mark.gpu
def test_gpu_damaged_and_adversarial_streams(monkeypatch):
    from test_jpeg import UYVY, RGB
    serial, sync, small = _decoder(monkeypatch, "off"), _decoder(monkeypatch), _decoder(monkeypatch, "on:8")
    for name, s in damaged_corpus(1) + [("adversarial", adversarial_stream()), ("stuffed", stuffed_everywhere())]:
        for codec in (UYVY, RGB):
            want = _decode(serial, s, codec)
            for d in (sync, small):
                got = _decode(d, s, codec)
                assert type(got) is type(want) and (isinstance(got, str) and got == want or np.array_equal(got, want)), (name, codec)
        if name == "adversarial":
            assert small.last_sync()["rounds"] > ADVERSARIAL_MIN_ROUNDS
    for d in (serial, sync, small):
        d.close()


@pytest.mark.gpu
def test_gpu_two_decoders_alternating_frames(monkeypatch):
    """scratch buffers that grow and shrink between frames of different size and route, on two streams"""
    import torch
    from test_jpeg import UYVY
    frames = [pil(natural_rgb(w, h, w), 85, 1, restart_blocks=rb) for (w, h, rb) in ((1920, 1080, 0), (640, 360, 4), (3840, 2160, 0), (320, 200, 0), (1280, 720, 8))]
    serial = _decoder(monkeypatch, "off")
    want = [_decode(serial, s, UYVY, True) for s in frames]
    from ultragrid_b200 import api
    decs = [api.JpegDecoder(torch.cuda.Stream()), api.JpegDecoder(torch.cuda.Stream())]
    for rep in range(3):
        for i, s in enumerate(frames):
            d = decs[(i + rep) % 2]
            assert np.array_equal(_decode(d, s, UYVY, True), want[i]), (rep, i)
    for d in decs + [serial]:
        d.close()
