// Baseline JPEG decoder (include/ugb200_jpeg.h, decode part): the stage libgpujpeg performs for UltraGrid's
// src/video_decompress/gpujpeg.c:268-330 and gpujpeg_to_dxt.cpp:117-166 (SURVEY.md section 8f rank 1).
//
//   host   parse_stream     markers up to each SOS (tables, frame, scans) and ONE pass over the entropy-coded bytes that records
//                           where every restart segment starts (what GPUJPEG's reader does when the stream carries no segment info)
//   K0     jpeg_marker_*_kernel   the same segment table built on the device for the two regular stream shapes (one interleaved scan, or one scan
//                           per component): the host then only reads the headers in front of the first SOS
//   K1     jpeg_decode_huffman_kernel   one thread per restart segment: T.81 F.2.2 Huffman decoding with a 9-bit look-ahead
//                           table per Huffman table in shared memory (longer codes: min/max-code walk), DC prediction; every block is
//                           built in shared memory and written as 128 bytes into the int16 [block][64] buffer (or, when the scans do
//                           not cover every block, scattered into a cleared buffer)
//   K2     jpeg_idct_kernel one thread per 8x8 block: dequantise, float AAN inverse DCT (fixed operation order = bit-exact with
//                           oracle/jpeg_decode_oracle.c), level shift, clamp, 8 x 8-byte stores into the component plane
//   pack   the component planes go through the from_planar kernels that already exist (planar_conv_kernels.cu):
//                           4:2:2 -> UYVY (yuv422p_to_uyvy), 4:2:0 -> UYVY (yuv420p_to_uyvy), 4:4:4 YCbCr -> VUYA (yuv444p_to_vuya),
//                           RGB -> RGB (rgbpXX_to_rgb), then ugb200_pixfmt_convert when another output codec was asked for.
// Restart intervals are the unit of parallelism; a stream without DRI decodes correctly but on one thread per scan.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <emmintrin.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <chrono>
#include <cstdio>
#include <new>
#include <thread>
#include <vector>

#include "../../include/ugb200.h"
#include "../../include/ugb200_jpeg.h"
#include "jpeg_marker_bounds.cuh"
#include "../../include/cuda_wrapper.h"

namespace ugb {

static const uint8_t kZigzag[64] = { 0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

constexpr int kLook = 9;
/// Huffman table slots.  A DHT definition is built into a slot when a scan first uses it: table id k (DC Th 0, 1 = 0, 1; AC Th 0, 1 = 2, 3)
/// goes to slot k when that slot is free, otherwise to the lowest free one.  A table redefined between scans (T.81 B.2.4.2) thus gets a slot
/// of its own, and every scan keeps the tables it was coded with.  In a valid stream each component appears in one scan and uses one DC and
/// one AC table, and only definitions that a scan uses take a slot: four components never need more than eight.
constexpr int kTables = 8;

struct dec_tables {
        uint16_t lut[kTables][1 << kLook];  // (length << 8) | symbol for codes of up to kLook bits, 0 = longer code
        int maxcode[kTables][18];           // T.81 F.2.2.3, -1 = no code of that length
        int valoff[kTables][17];            // valptr - mincode
        uint8_t vals[kTables][256];
        uint8_t zz[64];
        float m[4][64];               // dequantisation x AAN scale, natural order
};

struct dec_comp {
        int h, v, tq;
        int bw, bh;     // blocks per row / rows of the padded plane
        int blk_off;    // first block of the component in the coefficient buffer
        long plane_off; // first byte of the plane in the plane buffer
};
struct dec_scan {
        int ns, comp[4], td[4], ta[4];  // td, ta: table slots of dec_tables
        int mcux, nmcu;
        int seg0, nseg;  // segments [seg0, seg0 + nseg)
};
struct dec_geom {
        int w, h, ncomp, hmax, vmax, ri, nscans, nblocks;  // ncomp 3, or 4 (R G B A, all 1x1)
        int ntables;  // Huffman table slots in use: [0, ntables) (the Huffman kernel copies only those to shared memory)
        dec_comp c[4];
        dec_scan s[4];
};

struct bit_reader {  // MSB-first, removes stuffed zero bytes, feeds zeros beyond `end`
        const uint8_t *p, *end;
        uint64_t acc;
        int nbits;
        // the two aligned words that hold bytes p .. p + 3, fetched one refill AHEAD of their use: the thread's next four bytes are already in registers when
        // it needs them (ncu of the byte-wise reader: `long_scoreboard` on top of the stall list - every refill waited for its own loads with ~13 warps per SM)
        const uint32_t *wa;
        uint32_t w0, w1;
        /// the stream buffer is 16 bytes longer than the stream: the aligned loads around any p <= end stay inside the allocation
        __device__ __forceinline__ void prime()
        {
                wa = (const uint32_t *) ((size_t) p & ~(size_t) 3);
                w0 = __ldg(wa), w1 = __ldg(wa + 1);
        }
        /// after the call at least 33 bits are valid (code of up to 16 bits + up to 15 value bits), zeros beyond `end`.
        /// Fast path: four stream bytes at once when none of them is 0xFF (entropy-coded data holds one 0xFF in ~256 bytes).
        __device__ __forceinline__ void refill()
        {
                if (nbits > 32) {
                        return;
                }
                if (p + 4 <= end) {
                        const uint32_t le = __funnelshift_r(w0, w1, 8 * (unsigned) ((size_t) p & 3));  // bytes p[0..3], p[0] lowest
                        if (__vcmpeq4(le, 0xffffffffu) == 0) {
                                acc |= (uint64_t) __byte_perm(le, 0, 0x0123) << (32 - nbits);
                                nbits += 32, p += 4;
                                ++wa, w0 = w1, w1 = __ldg(wa + 1);  // for the next refill
                                return;
                        }
                }
                while (nbits <= 56) {
                        uint32_t b = 0;
                        if (p < end) {
                                b = __ldg(p++);
                                if (b == 0xFF && p < end && __ldg(p) == 0) {
                                        ++p;
                                }
                        }
                        acc |= (uint64_t) b << (56 - nbits);
                        nbits += 8;
                }
                prime();
        }
        __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t) (acc >> (64 - n)); }
        __device__ __forceinline__ void skip(int n) { acc <<= n, nbits -= n; }
};

__device__ __forceinline__ int decode_symbol(bit_reader &r, const dec_tables *t, int tab)
{
        const uint32_t e = t->lut[tab][r.peek(kLook)];
        if (e) {
                r.skip(e >> 8);
                return e & 0xff;
        }
        const uint32_t v16 = r.peek(16);
        for (int l = kLook + 1; l <= 16; ++l) {
                const int code = (int) (v16 >> (16 - l));
                if (code <= t->maxcode[tab][l]) {
                        r.skip(l);
                        return t->vals[tab][t->valoff[tab][l] + code];
                }
        }
        r.skip(16);
        return 0;  // corrupt stream
}
__device__ __forceinline__ int receive_extend(bit_reader &r, int n)  // F.2.2.1, n in 1..15
{
        const int v = (int) r.peek(n);
        r.skip(n);
        return v < (1 << (n - 1)) ? v - (1 << n) + 1 : v;
}

/// FULL: every block of the coefficient array is decoded by exactly one thread (the host checks: every component in a scan, the scans' MCU grids equal to the
/// padded planes) - the thread then builds its block in shared memory ([word][thread]: conflict-free, dynamically indexable) and writes all 128 bytes of it,
/// so the array needs no clearing beforehand (133 MB at 8K) and the scattered 2-byte stores become whole-line stores.  !FULL: sparse stores into a cleared array.
/// kHuffThreads: an 8K UYVY frame has 64 800 restart segments = threads, all resident at once; with 128-thread CTAs that is 3.4 CTAs per SM (some SMs run four, the
/// kernel lasts as long as those), with 64-thread CTAs 6.8 (seven against six)
constexpr int kHuffThreads = 64;
/// block-wide copy of `bytes` (a multiple of 4) between 4-byte aligned addresses
__device__ __forceinline__ void copy_words(void *dst, const void *src, int bytes)
{
        for (int i = threadIdx.x; i < bytes / 4; i += blockDim.x) {
                ((uint32_t *) dst)[i] = ((const uint32_t *) src)[i];
        }
}

template <bool FULL>
__global__ void __launch_bounds__(kHuffThreads) jpeg_decode_huffman_kernel(const uint8_t *__restrict__ stream, const uint32_t *__restrict__ seg_begin,
                                                                  const uint32_t *__restrict__ seg_end, const dec_tables *__restrict__ tables,
                                                                  dec_geom g, int16_t *__restrict__ coef, const uint32_t *__restrict__ dev_scans)
{
        extern __shared__ uint8_t smem_raw[];
        dec_tables *t = (dec_tables *) smem_raw;
        uint32_t *const col = (uint32_t *) (smem_raw + ((sizeof(dec_tables) + 15) & ~(size_t) 15)) + threadIdx.x;  // FULL: word w of my block at col[w * kHuffThreads]
        // what this kernel reads: the slots in use and the zig-zag order (not the dequantisation multipliers)
        copy_words(t->lut, tables->lut, g.ntables * (int) sizeof t->lut[0]);
        copy_words(t->maxcode, tables->maxcode, g.ntables * (int) sizeof t->maxcode[0]);
        copy_words(t->valoff, tables->valoff, g.ntables * (int) sizeof t->valoff[0]);
        copy_words(t->vals, tables->vals, g.ntables * (int) sizeof t->vals[0]);
        copy_words(t->zz, tables->zz, (int) sizeof t->zz);
        __syncthreads();
        const int s = blockIdx.x * blockDim.x + threadIdx.x;
        int sc = 0;
        while (sc < g.nscans && s >= g.s[sc].seg0 + g.s[sc].nseg) {
                ++sc;
        }
        if (sc >= g.nscans) {
                return;
        }
        dec_scan S = g.s[sc];
        if (dev_scans != nullptr && sc > 0) {  // multi-scan stream with the marker scan on the device: the SOS headers of the later scans were read there
                S.td[0] = (int) dev_scans[kMetaBounds + 6 * sc + 4], S.ta[0] = 2 + (int) dev_scans[kMetaBounds + 6 * sc + 5];  // no DHT between the scans
        }
        const int ls = s - S.seg0;
        const int m0 = g.ri ? ls * g.ri : 0, m1 = g.ri ? min(m0 + g.ri, S.nmcu) : S.nmcu;
        bit_reader r = { stream + seg_begin[s], stream + seg_end[s], 0, 0, nullptr, 0, 0 };
        r.prime();
        int pred[4] = { 0, 0, 0, 0 };
        for (int m = m0; m < m1; ++m) {
                const int mx = m % S.mcux, my = m / S.mcux;
                for (int k = 0; k < S.ns; ++k) {
                        const dec_comp &c = g.c[S.comp[k]];
                        const int nh = S.ns == 1 ? 1 : c.h, nv = S.ns == 1 ? 1 : c.v;
                        for (int by = 0; by < nv; ++by) {
                                for (int bx = 0; bx < nh; ++bx) {
                                        const int X = mx * nh + bx, Y = my * nv + by;
                                        const bool inside = X < c.bw && Y < c.bh;
                                        int16_t *blk = coef + ((long) c.blk_off + (long) Y * c.bw + X) * 64;
                                        if (FULL) {
#pragma unroll
                                                for (int w = 0; w < 32; ++w) {
                                                        col[w * kHuffThreads] = 0;
                                                }
                                        }
                                        r.refill();
                                        const int tt = decode_symbol(r, t, S.td[k]);
                                        r.refill();
                                        if (tt) {
                                                pred[k] += receive_extend(r, tt & 15);
                                        }
                                        if (FULL) {
                                                col[0] = (uint32_t) pred[k] & 0xffffu;
                                        } else if (inside && pred[k] != 0) {
                                                blk[0] = (int16_t) pred[k];
                                        }
                                        for (int i = 1; i < 64;) {
                                                r.refill();
                                                const int rs = decode_symbol(r, t, S.ta[k]), run = rs >> 4, sz = rs & 15;
                                                if (sz == 0) {
                                                        if (run != 15) {
                                                                break;  // EOB
                                                        }
                                                        i += 16;
                                                        continue;
                                                }
                                                i += run;
                                                const int v = receive_extend(r, sz);  // refill guarantees >= 33 bits: 16 + 15 fit
                                                if (FULL) {
                                                        if (i < 64) {
                                                                const int n = t->zz[i];
                                                                ((int16_t *) (col + (n >> 1) * kHuffThreads))[n & 1] = (int16_t) v;
                                                        }
                                                } else if (i < 64 && inside) {
                                                        blk[t->zz[i]] = (int16_t) v;
                                                }
                                                ++i;
                                        }
                                        if (FULL && inside) {
#pragma unroll
                                                for (int q = 0; q < 8; ++q) {
                                                        ((uint4 *) blk)[q] = make_uint4(col[(4 * q) * kHuffThreads], col[(4 * q + 1) * kHuffThreads], col[(4 * q + 2) * kHuffThreads], col[(4 * q + 3) * kHuffThreads]);
                                                }
                                        }
                                }
                        }
                }
        }
}

__device__ __forceinline__ void idct8(float &d0, float &d1, float &d2, float &d3, float &d4, float &d5, float &d6, float &d7)
{
        const float e0 = __fadd_rn(d0, d4), e1 = __fadd_rn(d0, -d4);
        const float e3 = __fadd_rn(d2, d6), e2 = __fadd_rn(__fmul_rn(__fadd_rn(d2, -d6), 1.414213562f), -e3);
        const float a0 = __fadd_rn(e0, e3), a3 = __fadd_rn(e0, -e3), a1 = __fadd_rn(e1, e2), a2 = __fadd_rn(e1, -e2);
        const float z13 = __fadd_rn(d5, d3), z10 = __fadd_rn(d5, -d3), z11 = __fadd_rn(d1, d7), z12 = __fadd_rn(d1, -d7);
        const float b7 = __fadd_rn(z11, z13);
        const float b11 = __fmul_rn(__fadd_rn(z11, -z13), 1.414213562f);
        const float z5 = __fmul_rn(__fadd_rn(z10, z12), 1.847759065f);
        const float b10 = __fmaf_rn(1.082392200f, z12, -z5);
        const float b12 = __fmaf_rn(-2.613125930f, z10, z5);
        const float b6 = __fadd_rn(b12, -b7), b5 = __fadd_rn(b11, -b6), b4 = __fadd_rn(b10, b5);
        d0 = __fadd_rn(a0, b7), d7 = __fadd_rn(a0, -b7);
        d1 = __fadd_rn(a1, b6), d6 = __fadd_rn(a1, -b6);
        d2 = __fadd_rn(a2, b5), d5 = __fadd_rn(a2, -b5);
        d4 = __fadd_rn(a3, b4), d3 = __fadd_rn(a3, -b4);
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const int16_t *__restrict__ coef, const dec_tables *__restrict__ tables, dec_geom g,
                                                        uint8_t *__restrict__ planes)
{
        __shared__ float s_m[4][64];
        for (int i = threadIdx.x; i < 256; i += blockDim.x) {
                s_m[i >> 6][i & 63] = tables->m[i >> 6][i & 63];
        }
        __syncthreads();
        const int b = blockIdx.x * blockDim.x + threadIdx.x;
        if (b >= g.nblocks) {
                return;
        }
        int ci = 0;
        while (ci + 1 < g.ncomp && b >= g.c[ci + 1].blk_off) {
                ++ci;
        }
        const dec_comp &c = g.c[ci];
        const int lb = b - c.blk_off, X = lb % c.bw, Y = lb / c.bw;
        const float *m = s_m[c.tq];
        float f[64];
        const uint4 *src = (const uint4 *) (coef + (long) b * 64);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
                const uint4 v = __ldg(src + q);
                const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (int j = 0; j < 4; ++j) {  // int16 -> float without I2F: 1.5 * 2^23 + c is exact
                        const int lo = (int) (short) (w[j] & 0xffffu), hi = (int) w[j] >> 16;
                        f[8 * q + 2 * j] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) lo), -12582912.0f), m[8 * q + 2 * j]);
                        f[8 * q + 2 * j + 1] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) hi), -12582912.0f), m[8 * q + 2 * j + 1]);
                }
        }
#pragma unroll
        for (int col = 0; col < 8; ++col) {
                idct8(f[col], f[8 + col], f[16 + col], f[24 + col], f[32 + col], f[40 + col], f[48 + col], f[56 + col]);
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
                idct8(f[8 * r], f[8 * r + 1], f[8 * r + 2], f[8 * r + 3], f[8 * r + 4], f[8 * r + 5], f[8 * r + 6], f[8 * r + 7]);
        }
        uint8_t *dst = planes + c.plane_off + ((long) Y * 8) * (c.bw * 8) + X * 8;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
                uint32_t o[8];
#pragma unroll
                for (int x = 0; x < 8; ++x) {  // rintf(v + 128) through the 1.5 * 2^23 magic, clamp 0..255
                        const int v = (int) __float_as_uint(__fadd_rn(__fadd_rn(f[8 * r + x], 128.0f), 12582912.0f)) - 0x4B400000;
                        o[x] = (uint32_t) min(max(v, 0), 255);
                }
                *(uint2 *) (dst + (long) r * (c.bw * 8)) = make_uint2(o[0] | o[1] << 8 | o[2] << 16 | o[3] << 24, o[4] | o[5] << 8 | o[6] << 16 | o[7] << 24);
        }
}

/// 4:2:2 streams: IDCT and UYVY packing in one kernel.  CTA = 32 MCUs x (Y0, Y1, Cb, Cr), warp k = block kind k (component-uniform
/// dequantisation), lane = MCU.  The 8 x 8 samples of each block go to a shared tile as 8-byte rows; then the 8 KB tile leaves as 512
/// 16-byte UYVY pieces, consecutive pieces consecutive in memory.  Same arithmetic as jpeg_idct_kernel.
__global__ void __launch_bounds__(128) jpeg_idct_uyvy_kernel(const int16_t *__restrict__ coef, const dec_tables *__restrict__ tables, dec_geom g,
                                                             uint8_t *__restrict__ out, long pitch, bool vec_ok)
{
        __shared__ float s_m[4][64];
        __shared__ uint2 s_tile[4][8][32];
        const int tid = threadIdx.x;
        for (int i = tid; i < 256; i += blockDim.x) {
                s_m[i >> 6][i & 63] = tables->m[i >> 6][i & 63];
        }
        __syncthreads();
        const int mcux = g.c[1].bw, nmcu = mcux * g.c[1].bh;
        const int k = tid >> 5, lane = tid & 31, m0 = blockIdx.x * 32, m = m0 + lane;
        if (m < nmcu) {
                const int mx = m % mcux, my = m / mcux;
                const dec_comp &c = g.c[k < 2 ? 0 : k - 1];
                const int X = k < 2 ? 2 * mx + k : mx;
                const long b = (long) c.blk_off + (long) my * c.bw + X;
                const float *mq = s_m[c.tq];
                float f[64];
                const uint4 *src = (const uint4 *) (coef + b * 64);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                        const uint4 v = __ldg(src + q);
                        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                                const int lo = (int) (short) (w[j] & 0xffffu), hi = (int) w[j] >> 16;
                                f[8 * q + 2 * j] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) lo), -12582912.0f), mq[8 * q + 2 * j]);
                                f[8 * q + 2 * j + 1] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) hi), -12582912.0f), mq[8 * q + 2 * j + 1]);
                        }
                }
#pragma unroll
                for (int col = 0; col < 8; ++col) {
                        idct8(f[col], f[8 + col], f[16 + col], f[24 + col], f[32 + col], f[40 + col], f[48 + col], f[56 + col]);
                }
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                        idct8(f[8 * r], f[8 * r + 1], f[8 * r + 2], f[8 * r + 3], f[8 * r + 4], f[8 * r + 5], f[8 * r + 6], f[8 * r + 7]);
                        uint32_t o[8];
#pragma unroll
                        for (int x = 0; x < 8; ++x) {
                                const int v = (int) __float_as_uint(__fadd_rn(__fadd_rn(f[8 * r + x], 128.0f), 12582912.0f)) - 0x4B400000;
                                o[x] = (uint32_t) min(max(v, 0), 255);
                        }
                        s_tile[k][r][lane] = make_uint2(o[0] | o[1] << 8 | o[2] << 16 | o[3] << 24, o[4] | o[5] << 8 | o[6] << 16 | o[7] << 24);
                }
        }
        __syncthreads();
        const int row_bytes = ((g.w + 1) / 2) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
                const int cidx = tid + 128 * i, row = cidx >> 6, within = cidx & 63, mcu = within >> 1, half = within & 1;
                const int mm = m0 + mcu;
                if (mm >= nmcu) {
                        continue;
                }
                const int mx = mm % mcux, y = (mm / mcux) * 8 + row, xoff = mx * 32 + half * 16;
                if (y >= g.h || xoff >= row_bytes) {
                        continue;
                }
                const uint2 Y = s_tile[half][row][mcu], CB = s_tile[2][row][mcu], CR = s_tile[3][row][mcu];
                const uint32_t C = half ? CB.y : CB.x, R = half ? CR.y : CR.x;
                const uint32_t w0 = __byte_perm(__byte_perm(C, R, 0x0040), Y.x, 0x5140), w1 = __byte_perm(__byte_perm(C, R, 0x0051), Y.x, 0x7160);
                const uint32_t w2 = __byte_perm(__byte_perm(C, R, 0x0062), Y.y, 0x5140), w3 = __byte_perm(__byte_perm(C, R, 0x0073), Y.y, 0x7160);
                uint8_t *d = out + (long) y * pitch + xoff;
                if (vec_ok && xoff + 16 <= row_bytes) {
                        *(uint4 *) d = make_uint4(w0, w1, w2, w3);
                } else {
                        const uint32_t w[4] = { w0, w1, w2, w3 };
                        for (int bq = 0; bq < 16 && xoff + bq < row_bytes; ++bq) {
                                d[bq] = (uint8_t) (w[bq >> 2] >> (8 * (bq & 3)));
                        }
                }
        }
}

// ---- marker scan on the device (streams with one interleaved scan: what UltraGrid sends for UYVY; or one scan per component: RGB) ---------------
// The host's part shrinks to the header segments in front of the SOS and a plain copy of the stream into pinned memory; the RSTn markers that
// split the entropy-coded data are found here: K-a counts the marker candidates of every 4 KB piece, K-b is a one-CTA exclusive scan, K-c writes
// their positions in stream order and notes the first one that is not an RSTn (it ends the scan), K-d turns the list into the segment table the
// Huffman kernel reads - the same rules as parse_stream (excess RSTn are ignored, missing segments decode as nothing).
constexpr int kMarkThreads = 256;  // x 16 bytes

/// bit k: byte base + k is 0xFF, its follower neither a stuffed 0x00 nor a fill 0xFF, and the pair lies inside [from, len)
__device__ __forceinline__ unsigned marker_mask16(const uint8_t *__restrict__ s, size_t len, size_t base, size_t from)
{
        if (base + 1 >= len) {
                return 0;
        }
        const uint4 v = *(const uint4 *) (s + base);       // the buffer is 16 bytes longer than the stream
        const uint32_t nxt = s[base + 16];
        const uint32_t w[5] = { v.x, v.y, v.z, v.w, nxt };
        unsigned mask = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
                const uint32_t follower = __funnelshift_r(w[i], w[i + 1], 8);
                const uint32_t cand = __vcmpeq4(w[i], 0xffffffffu) & ~(__vcmpeq4(follower, 0u) | __vcmpeq4(follower, 0xffffffffu));
                mask |= (((cand & 0x01010101u) * 0x01020408u) >> 24) << (4 * i);
        }
        const size_t last = len - 1;  // candidates need p + 1 < len
        if (base + 16 > last) {
                mask &= (1u << (unsigned) (last - base)) - 1u;
        }
        if (from > base) {
                mask &= from - base >= 16 ? 0u : ~((1u << (unsigned) (from - base)) - 1u);
        }
        return mask;
}

__global__ void __launch_bounds__(kMarkThreads) jpeg_marker_count_kernel(const uint8_t *__restrict__ s, size_t len, size_t from, uint32_t *__restrict__ cnt)
{
        __shared__ uint32_t s_w[kMarkThreads / 32];
        const size_t base = ((size_t) blockIdx.x * kMarkThreads + threadIdx.x) * 16;
        uint32_t n = __popc(marker_mask16(s, len, base, from));
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
                n += __shfl_xor_sync(0xffffffffu, n, d);
        }
        if ((threadIdx.x & 31) == 0) {
                s_w[threadIdx.x >> 5] = n;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
                uint32_t t = 0;
                for (int i = 0; i < kMarkThreads / 32; ++i) {
                        t += s_w[i];
                }
                cnt[blockIdx.x] = t;
        }
}

/// exclusive scan of cnt[0..n) in place; meta[0] = total, meta[1] = 0xFFFFFFFF (index of the first non-RSTn candidate, filled by K-c)
__global__ void __launch_bounds__(1024) jpeg_marker_scan_kernel(uint32_t *__restrict__ cnt, int n, uint32_t *__restrict__ meta)
{
        __shared__ uint32_t s_w[32];
        __shared__ uint32_t s_carry;
        if (threadIdx.x == 0) {
                s_carry = 0;
        }
        __syncthreads();
        for (int base = 0; base < n; base += 1024) {
                const int i = base + (int) threadIdx.x;
                const uint32_t v = i < n ? cnt[i] : 0;
                uint32_t incl = v;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                        if ((threadIdx.x & 31) >= (unsigned) d) {
                                incl += o;
                        }
                }
                if ((threadIdx.x & 31) == 31) {
                        s_w[threadIdx.x >> 5] = incl;
                }
                __syncthreads();
                uint32_t before = s_carry;
                for (int w = 0; w < (int) (threadIdx.x >> 5); ++w) {
                        before += s_w[w];
                }
                if (i < n) {
                        cnt[i] = before + incl - v;
                }
                __syncthreads();
                if (threadIdx.x == 1023) {
                        s_carry = before + incl;
                }
                __syncthreads();
        }
        if (threadIdx.x == 0) {
                meta[kMetaTotal] = s_carry, meta[kMetaFirstOther] = 0xffffffffu, meta[kMetaOtherCount] = 0, meta[kMetaError] = 0;
        }
}

__global__ void __launch_bounds__(kMarkThreads) jpeg_marker_write_kernel(const uint8_t *__restrict__ s, size_t len, size_t from, const uint32_t *__restrict__ off,
                                                                         uint32_t *__restrict__ list, uint32_t *__restrict__ meta)
{
        __shared__ uint32_t s_w[kMarkThreads / 32];
        const size_t base = ((size_t) blockIdx.x * kMarkThreads + threadIdx.x) * 16;
        unsigned mask = marker_mask16(s, len, base, from);
        const uint32_t n = __popc(mask);
        uint32_t incl = n;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                if ((threadIdx.x & 31) >= (unsigned) d) {
                        incl += o;
                }
        }
        if ((threadIdx.x & 31) == 31) {
                s_w[threadIdx.x >> 5] = incl;
        }
        __syncthreads();
        uint32_t idx = off[blockIdx.x] + incl - n;
        for (int w = 0; w < (int) (threadIdx.x >> 5); ++w) {
                idx += s_w[w];
        }
        while (mask) {
                const size_t p = base + (size_t) (__ffs((int) mask) - 1);
                mask &= mask - 1;
                list[idx] = (uint32_t) p;
                const int code = s[p + 1];
                if (code < 0xD0 || code > 0xD7) {
                        atomicMin(meta + kMetaFirstOther, idx);
                        const uint32_t k = atomicAdd(meta + kMetaOtherCount, 1u);  // the handful of markers that are not RSTn: SOS of later scans, EOI
                        if (k < (uint32_t) kMaxOther) {
                                meta[kMetaOther + k] = idx;
                        }
                }
                ++idx;
        }
}

/// segment table of ONE scan that starts at `begin0`: the rules of parse_stream's SOS branch
__global__ void __launch_bounds__(256) jpeg_marker_segments_kernel(const uint32_t *__restrict__ list, const uint32_t *__restrict__ meta, uint32_t begin0, uint32_t len,
                                                                   int nseg, uint32_t *__restrict__ seg_begin, uint32_t *__restrict__ seg_end)
{
        const int i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= nseg) {
                return;
        }
        const uint32_t total = meta[0], stop = min(meta[1], total);  // `stop` RSTn candidates precede the marker that ends the scan
        const uint32_t term = stop < total ? list[stop] : len;
        const uint32_t pushed = min(stop, (uint32_t) (nseg - 1));
        uint32_t b, e;
        if ((uint32_t) i < pushed) {
                b = i == 0 ? begin0 : list[i - 1] + 2, e = list[i];
        } else if ((uint32_t) i == pushed) {
                b = stop == 0 ? begin0 : list[stop - 1] + 2, e = term;
        } else {
                b = e = term;
        }
        seg_begin[i] = b, seg_end[i] = e;
}

/// multi-scan streams: see jpeg_marker_bounds.cuh (the same code is checked against the host parser on the CPU)
__global__ void jpeg_marker_bounds_kernel(const uint8_t *__restrict__ s, uint32_t len, const uint32_t *__restrict__ list, uint32_t *__restrict__ meta, uint32_t begin0,
                                          int nscans, uint32_t comp_ids)
{
        if (threadIdx.x == 0 && blockIdx.x == 0) {
                marker_bounds(s, len, list, meta, begin0, nscans, comp_ids);
        }
}

/// segment table of a multi-scan stream from the bounds above: the rules of jpeg_marker_segments_kernel per scan
__global__ void __launch_bounds__(256) jpeg_marker_segments_multi_kernel(const uint32_t *__restrict__ list, const uint32_t *__restrict__ meta, int nscans, int seg1, int seg2,
                                                                         int nseg, uint32_t *__restrict__ seg_begin, uint32_t *__restrict__ seg_end)
{
        const int i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i < nseg) {
                marker_segment_multi(list, meta, nscans, seg1, seg2, nseg, i, seg_begin + i, seg_end + i);
        }
}

}  // namespace ugb

using namespace ugb;

/// A handful of persistent host threads for the marker scan (creating threads per frame costs more than the scan of an 8K stream).
class scan_pool {
public:
        explicit scan_pool(int n)
        {
                for (int i = 0; i < n; ++i) {
                        workers.emplace_back([this, i] { run(i); });
                }
        }
        ~scan_pool()
        {
                {
                        std::lock_guard<std::mutex> lk(m);
                        quit = true;
                }
                cv.notify_all();
                for (auto &t : workers) {
                        t.join();
                }
        }
        int size() const { return (int) workers.size(); }
        /// runs job(i) for i in 0..n-1 on the workers (n <= size()) while the caller does its own share; returns when all are done
        void parallel(int n, const std::function<void(int)> &job_, const std::function<void()> &own)
        {
                {
                        std::lock_guard<std::mutex> lk(m);
                        job = &job_, todo = n, left = n, ++generation;
                }
                cv.notify_all();
                own();
                std::unique_lock<std::mutex> lk(m);
                done.wait(lk, [this] { return left == 0; });
                job = nullptr;
        }

private:
        void run(int i)
        {
                unsigned seen = 0;
                for (;;) {
                        const std::function<void(int)> *j;
                        {
                                std::unique_lock<std::mutex> lk(m);
                                cv.wait(lk, [&] { return quit || (generation != seen && i < todo); });
                                if (quit) {
                                        return;
                                }
                                seen = generation, j = job;
                        }
                        (*j)(i);
                        std::lock_guard<std::mutex> lk(m);
                        if (--left == 0) {
                                done.notify_one();
                        }
                }
        }
        std::vector<std::thread> workers;
        std::mutex m;
        std::condition_variable cv, done;
        const std::function<void(int)> *job = nullptr;
        int todo = 0, left = 0;
        unsigned generation = 0;
        bool quit = false;
};

struct ugb200_jpeg_decoder {
        cudaStream_t stream = nullptr;
        scan_pool pool{ 7 };
        cudaStream_t copy = nullptr;  // the stream upload of frame n + 1 runs here, under the kernels of frame n (its device copy is double-buffered with the host slots)
        uint8_t *planes = nullptr, *native = nullptr, *staging = nullptr;
        int16_t *coef = nullptr;
        uint32_t *d_seg = nullptr, *d_marks = nullptr, *d_mark_cnt = nullptr;  // d_mark_cnt: per-piece counts / offsets, then meta[kMetaWords]
        dec_tables *d_tables = nullptr;
        size_t planes_cap = 0, native_cap = 0, staging_cap = 0, coef_cap = 0, seg_cap = 0, marks_cap = 0, mark_cnt_cap = 0;
        int scan_mode = 0;      // 0: device scan for large streams (one interleaved scan, or one scan per component), 1: always the host scan, 2: device scan at any size
        bool host_once = false; // the device found a multi-scan stream irregular: this frame is repeated with the host parser
        uint32_t *h_flag = nullptr;  // pinned: the device's verdict on a multi-scan stream
        size_t last_nseg = 0;   // segments of the last decode (ugb200_jpeg_decoder_last_segments)
        // pinned staging (the caller's stream buffer is pageable and freed right after the call), two slots: the host side of frame
        // i + 1 (scan, parse, staging copy) runs while the device still works on frame i
        struct host_slot {
                uint8_t *stream = nullptr;
                uint32_t *seg = nullptr;
                dec_tables *tables = nullptr;
                uint8_t *d_stream = nullptr;  // this slot's copy of the stream on the device (16 bytes longer than the stream)
                size_t stream_cap = 0, seg_cap = 0, d_stream_cap = 0;
                cudaEvent_t uploaded = nullptr;   // segment table + Huffman / quantisation tables left the pinned slot (decoder's stream)
                cudaEvent_t stream_up = nullptr;  // the stream left the pinned slot and is on the device (copy stream)
                cudaEvent_t consumed = nullptr;   // the last kernel that reads d_stream is done (decoder's stream)
                bool pending = false, consumed_pending = false;
        } hs[2];
        unsigned frame_no = 0;
        int expect_w = 0, expect_h = 0;  // ugb200_jpeg_decoder_expect: the destination was sized for these; 0 = unchecked
        // host scratch that keeps its capacity from frame to frame
        std::vector<uint64_t> scan_part[8], markers;
        std::vector<uint32_t> seg_begin, seg_end;
};

namespace {

template <class T>
bool dgrow(T *&ptr, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        if (ptr) {
                cudaFree(ptr);
        }
        ptr = nullptr, cap = 0;
        if (cudaMalloc((void **) &ptr, need * sizeof(T)) != cudaSuccess) {
                return false;
        }
        cap = need;
        return true;
}
template <class T>
bool hgrow(T *&ptr, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        if (ptr) {
                cudaFreeHost(ptr);
        }
        ptr = nullptr, cap = 0;
        if (cudaMallocHost((void **) &ptr, need * sizeof(T)) != cudaSuccess) {
                return false;
        }
        cap = need;
        return true;
}

int be16(const uint8_t *p) { return p[0] << 8 | p[1]; }

constexpr long kMaxPixels = 16384L * 16384L;  // four 8K frames side by side; larger SOF dimensions are refused before anything is allocated

struct huff_defs {  // the current DHT definition of each table id, built into a slot of dec_tables when a scan first uses it
        uint8_t bits[4][16], vals[4][256];
        int n[4] = { 0, 0, 0, 0 };
        bool defined[4] = { false, false, false, false };
        int slot[4] = { -1, -1, -1, -1 };  // slot holding the current definition, -1 = not built yet
        bool taken[kTables] = {};          // built: a scan reads it
};

struct parsed {
        dec_geom g{};
        int adobe = -1, comp_id[4] = { 0, 0, 0, 0 };
        bool have_sof = false, have_q[4] = { false, false, false, false };
        huff_defs hd;
        uint8_t q[4][64];
        std::vector<uint32_t> seg_begin, seg_end;
};

/// @returns false for an over-subscribed code-length histogram (the Kraft check behind libjpeg's JERR_BAD_HUFF_TABLE): after the codes of
/// length l are assigned the next code must still fit in l bits, otherwise the look-up fill of build_table would run past the table
bool kraft_ok(const uint8_t *bits)
{
        for (int l = 1, code = 0; l <= 16; ++l) {
                code += bits[l - 1];
                if (code > (1 << l)) {
                        return false;
                }
                code <<= 1;
        }
        return true;
}

/// the bits / values have passed kraft_ok
void build_table(dec_tables &t, int tab, const uint8_t *bits, const uint8_t *vals, int n)
{
        memset(t.lut[tab], 0, sizeof t.lut[tab]);
        memcpy(t.vals[tab], vals, n);
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
                t.valoff[tab][l] = k - code;
                for (int i = 0; i < bits[l - 1]; ++i, ++k, ++code) {
                        if (l <= kLook) {
                                for (int fill = 0; fill < (1 << (kLook - l)); ++fill) {
                                        t.lut[tab][(code << (kLook - l)) | fill] = (uint16_t) (l << 8 | vals[k]);
                                }
                        }
                }
                t.maxcode[tab][l] = bits[l - 1] ? code - 1 : -1;
                code <<= 1;
        }
        t.maxcode[tab][17] = 0x7fffffff;
}

/// the table slot of the current definition of table id `id`, built on first use (see kTables); -1: the table is undefined or no slot is left
int table_slot(huff_defs &H, dec_tables *T, int id)
{
        if (!H.defined[id]) {
                return -1;
        }
        if (H.slot[id] < 0) {
                int k = id;
                if (H.taken[k]) {
                        for (k = 0; k < kTables && H.taken[k]; ++k) {
                        }
                        if (k == kTables) {
                                return -1;
                        }
                }
                H.taken[k] = true, H.slot[id] = k;
                if (T) {
                        build_table(*T, k, H.bits[id], H.vals[id], H.n[id]);
                }
        }
        return H.slot[id];
}

const bool g_stream_stores = [] {
        const char *e = getenv("UGB200_JPEG_STAGE");  // "plain": ordinary stores into the pinned staging buffer (A/B timing)
        return !(e && e[0] == 'p');
}();

const float kAan[8] = { 1.0f, 1.387039845f, 1.306562965f, 1.175875602f, 1.0f, 0.785694958f, 0.541196100f, 0.275899379f };

/// marker candidates of [lo, hi): positions p with s[p] == 0xFF and s[p + 1] neither a stuffed 0x00 nor a fill 0xFF.  One SSE2 compare per
/// 16 bytes, then only the 0xFF positions are looked at.  Optionally copies the range to `copy_to` in the same pass (staging for the upload).
void scan_markers(const uint8_t *s, size_t lo, size_t hi, size_t len, std::vector<uint64_t> &out, uint8_t *copy_to)
{
        const __m128i ff16 = _mm_set1_epi8((char) 0xFF), zero = _mm_setzero_si128();
        size_t i = lo;
        // the staging buffer is read next by the copy engine, not by a CPU: non-temporal stores keep it out of the caches (an upload of a stream
        // that several cores had just written through their caches was slow on an earlier machine)
        const bool stream_stores = copy_to != nullptr && g_stream_stores && ((uintptr_t) (copy_to + lo) & 15) == 0;
        // 0xFF is frequent in Huffman-coded data (runs of 1-bits), a marker is not: the follower byte is tested in the vector domain too
        for (; i + 17 <= len && i + 16 <= hi; i += 16) {
                const __m128i v = _mm_loadu_si128((const __m128i *) (s + i)), nx = _mm_loadu_si128((const __m128i *) (s + i + 1));
                if (copy_to) {
                        if (stream_stores) {
                                _mm_stream_si128((__m128i *) (copy_to + i), v);
                        } else {
                                _mm_storeu_si128((__m128i *) (copy_to + i), v);
                        }
                }
                const __m128i stuffed = _mm_or_si128(_mm_cmpeq_epi8(nx, zero), _mm_cmpeq_epi8(nx, ff16));
                unsigned mask = (unsigned) _mm_movemask_epi8(_mm_andnot_si128(stuffed, _mm_cmpeq_epi8(v, ff16)));
                while (mask) {  // entry = marker code << 32 | position: the parser never has to touch the stream again (one cache miss per marker)
                        const size_t p = i + (size_t) __builtin_ctz(mask);
                        out.push_back((uint64_t) s[p + 1] << 32 | p);
                        mask &= mask - 1;
                }
        }
        for (; i < hi; ++i) {
                if (copy_to) {
                        copy_to[i] = s[i];
                }
                if (s[i] == 0xFF && i + 1 < len && s[i + 1] != 0 && s[i + 1] != 0xFF) {
                        out.push_back((uint64_t) s[i + 1] << 32 | i);
                }
        }
        if (stream_stores) {
                _mm_sfence();
        }
}

/// plain staging copy (device marker scan): non-temporal stores when the destination allows it
void stage_copy(uint8_t *dst, const uint8_t *src, size_t n)
{
        if (!g_stream_stores || ((uintptr_t) dst & 15) != 0) {
                memcpy(dst, src, n);
                return;
        }
        size_t i = 0;
        for (; i + 64 <= n; i += 64) {
                const __m128i a = _mm_loadu_si128((const __m128i *) (src + i)), b = _mm_loadu_si128((const __m128i *) (src + i + 16));
                const __m128i c = _mm_loadu_si128((const __m128i *) (src + i + 32)), e = _mm_loadu_si128((const __m128i *) (src + i + 48));
                _mm_stream_si128((__m128i *) (dst + i), a), _mm_stream_si128((__m128i *) (dst + i + 16), b);
                _mm_stream_si128((__m128i *) (dst + i + 32), c), _mm_stream_si128((__m128i *) (dst + i + 48), e);
        }
        memcpy(dst + i, src + i, n - i);
        _mm_sfence();
}

/// header markers up to and including every SOS; `full` also finds the restart segments of the entropy-coded data, from the marker
/// candidates in `markers` (sorted; scanned here when the caller has none)
int parse_stream(const uint8_t *s, size_t len, parsed &P, dec_tables *T, bool full, const std::vector<uint64_t> *markers = nullptr,
                 size_t *first_scan_data = nullptr)
{
        std::vector<uint64_t> own;
        if (full && markers == nullptr) {
                scan_markers(s, 0, len, len, own, nullptr);
                markers = &own;
        }
        const uint8_t *p = s, *end = s + len;
        if (len < 4 || p[0] != 0xFF || p[1] != 0xD8) {
                return -1;
        }
        p += 2;
        dec_geom &g = P.g;
        while (p + 4 <= end) {
                if (p[0] != 0xFF) {
                        return -3;
                }
                const int mk = p[1];
                if (mk == 0xD9) {
                        break;
                }
                if (mk == 0xFF) {  // fill byte
                        ++p;
                        continue;
                }
                const int L = be16(p + 2);
                const uint8_t *d = p + 4, *dend = p + 2 + L;
                if (L < 2 || dend > end) {
                        return -3;
                }
                if (mk == 0xDB) {
                        while (d + 65 <= dend) {
                                const int pq = d[0] >> 4, tq = d[0] & 15;
                                if (pq != 0 || tq > 3) {
                                        return -4;
                                }
                                for (int k = 0; k < 64; ++k) {
                                        P.q[tq][kZigzag[k]] = d[1 + k];
                                }
                                P.have_q[tq] = true;
                                if (T) {
                                        for (int n = 0; n < 64; ++n) {
                                                T->m[tq][n] = ((float) P.q[tq][n] * kAan[n >> 3]) * kAan[n & 7] * 0.125f;
                                        }
                                }
                                d += 65;
                        }
                } else if (mk == 0xC4) {
                        while (d + 17 <= dend) {
                                const int tc = d[0] >> 4, th = d[0] & 15;
                                int n = 0;
                                for (int i = 0; i < 16; ++i) {
                                        n += d[1 + i];
                                }
                                if (tc > 1 || th > 1 || n > 256 || d + 17 + n > dend) {
                                        return -4;  // baseline: two tables per class
                                }
                                if (!kraft_ok(d + 1)) {
                                        return -4;  // over-subscribed Huffman table
                                }
                                const int id = tc * 2 + th;  // a new definition: the slot of the old one stays with the scans that used it
                                memcpy(P.hd.bits[id], d + 1, 16), memcpy(P.hd.vals[id], d + 17, n);
                                P.hd.n[id] = n, P.hd.defined[id] = true, P.hd.slot[id] = -1;
                                d += 17 + n;
                        }
                } else if (mk == 0xC0) {
                        if (L < 8 || L < 8 + 3 * d[5] || d[0] != 8) {  // L first: d[5] lies inside the segment only then
                                return -4;
                        }
                        g.h = be16(d + 1), g.w = be16(d + 3), g.ncomp = d[5];
                        if ((g.ncomp != 3 && g.ncomp != 4) || g.w == 0 || g.h == 0) {
                                return -4;
                        }
                        if ((long) g.w * g.h > kMaxPixels) {  // header fields are untrusted: they size every host and device allocation below
                                return -4;
                        }
                        g.hmax = g.vmax = 1;
                        for (int i = 0; i < g.ncomp; ++i) {
                                P.comp_id[i] = d[6 + 3 * i];
                                g.c[i].h = d[7 + 3 * i] >> 4, g.c[i].v = d[7 + 3 * i] & 15, g.c[i].tq = d[8 + 3 * i];
                                g.hmax = g.c[i].h > g.hmax ? g.c[i].h : g.hmax, g.vmax = g.c[i].v > g.vmax ? g.c[i].v : g.vmax;
                        }
                        int blk = 0;
                        long off = 0;
                        for (int i = 0; i < g.ncomp; ++i) {  // four components: every one sampled 1x1 (no subsampled alpha)
                                dec_comp &c = g.c[i];
                                if (c.h < 1 || c.h > 2 || c.v < 1 || c.v > 2 || ((i > 0 || g.ncomp == 4) && (c.h != 1 || c.v != 1)) || c.tq > 3) {
                                        return -4;
                                }
                                if (c.v > c.h) {  // luma 1x2 (4:4:0): no output layout packs it (UYVY and the 4:4:4 packers would read chroma rows that do not exist)
                                        return -4;
                                }
                                c.bw = (g.w + 8 * g.hmax - 1) / (8 * g.hmax) * c.h, c.bh = (g.h + 8 * g.vmax - 1) / (8 * g.vmax) * c.v;
                                c.blk_off = blk, c.plane_off = off;
                                blk += c.bw * c.bh, off += (long) c.bw * c.bh * 64;
                        }
                        g.nblocks = blk;
                        P.have_sof = true;
                } else if (mk >= 0xC1 && mk <= 0xCF && mk != 0xC4 && mk != 0xC8 && mk != 0xCC) {
                        return -4;  // not baseline sequential Huffman
                } else if (mk == 0xDD) {
                        if (L < 4) {
                                return -3;
                        }
                        g.ri = be16(d);
                } else if (mk == 0xEE && L >= 14 && memcmp(d, "Adobe", 5) == 0) {
                        P.adobe = d[11];
                } else if (mk == 0xDA) {
                        if (!P.have_sof || g.nscans >= g.ncomp) {
                                return -3;
                        }
                        if (g.ncomp == 4 && P.adobe != -1 && P.adobe != 0) {
                                return -4;  // Adobe transform 2 (YCCK) or 1: samples are not R G B A as stored
                        }
                        dec_scan &S = g.s[g.nscans];
                        if (L < 3) {
                                return -3;
                        }
                        S.ns = d[0];
                        if (S.ns < 1 || S.ns > g.ncomp || L < 6 + 2 * S.ns) {
                                return -4;
                        }
                        for (int i = 0; i < S.ns; ++i) {
                                S.comp[i] = -1;
                                for (int j = 0; j < g.ncomp; ++j) {
                                        if (P.comp_id[j] == d[1 + 2 * i]) {
                                                S.comp[i] = j;
                                        }
                                }
                                const int td = d[2 + 2 * i] >> 4, ta = d[2 + 2 * i] & 15;
                                if (S.comp[i] < 0 || td > 1 || ta > 1 || !P.have_q[g.c[S.comp[i]].tq]) {
                                        return -4;
                                }
                                S.td[i] = table_slot(P.hd, T, td), S.ta[i] = table_slot(P.hd, T, 2 + ta);
                                if (S.td[i] < 0 || S.ta[i] < 0) {
                                        return -4;  // an undefined table, or more table definitions in use than a valid stream has
                                }
                        }
                        int mcuy;
                        if (S.ns == 1) {
                                const dec_comp &c = g.c[S.comp[0]];
                                S.mcux = ((g.w * c.h + g.hmax - 1) / g.hmax + 7) / 8, mcuy = ((g.h * c.v + g.vmax - 1) / g.vmax + 7) / 8;
                        } else {
                                S.mcux = (g.w + 8 * g.hmax - 1) / (8 * g.hmax), mcuy = (g.h + 8 * g.vmax - 1) / (8 * g.vmax);
                        }
                        S.nmcu = S.mcux * mcuy;
                        S.seg0 = (int) P.seg_begin.size();
                        S.nseg = g.ri ? (S.nmcu + g.ri - 1) / g.ri : 1;
                        // every segment but the last ends in a 2-byte RSTn: a stream of `len` bytes cannot hold more than len / 2 + 1 of them (the
                        // rest of a truncated stream is filled in below, bounded by kMaxPixels)
                        P.seg_begin.reserve(P.seg_begin.size() + std::min((size_t) S.nseg, len / 2 + 1)), P.seg_end.reserve(P.seg_begin.capacity());
                        ++g.nscans;
                        p = dend;
                        if (!full) {
                                if (first_scan_data) {
                                        *first_scan_data = (size_t) (p - s);
                                }
                                return 0;  // enough for the image info
                        }
                        // entropy-coded segment(s): RSTn candidates split it, the first other marker ends it
                        uint32_t begin = (uint32_t) (p - s);
                        int found = 0;
                        auto it = std::lower_bound(markers->begin(), markers->end(), (uint64_t) begin,
                                                   [](uint64_t e, uint64_t pos) { return (uint32_t) e < pos; });
                        for (; it != markers->end(); ++it) {
                                const int c2 = (int) (*it >> 32);
                                const uint32_t pos = (uint32_t) *it;
                                if (c2 < 0xD0 || c2 > 0xD7) {
                                        break;
                                }
                                if (found + 1 < S.nseg) {
                                        P.seg_begin.push_back(begin), P.seg_end.push_back(pos);
                                        ++found;
                                }
                                begin = pos + 2;
                        }
                        p = it != markers->end() ? s + (uint32_t) *it : end;
                        P.seg_begin.push_back(begin), P.seg_end.push_back((uint32_t) (p - s));
                        ++found;
                        while (found < S.nseg) {  // truncated stream: the missing segments decode as nothing (zero coefficients)
                                P.seg_begin.push_back((uint32_t) (p - s)), P.seg_end.push_back((uint32_t) (p - s));
                                ++found;
                        }
                        continue;
                }
                p = dend;
        }
        return P.have_sof && g.nscans > 0 ? 0 : -3;
}

/// all marker candidates of the stream, in order; large streams are split over the pool (piece 0 on the calling thread)
constexpr int kMaxScanThreads = 8;
/// `scratch`: kMaxScanThreads vectors that keep their capacity between frames (a decoder's frames have the same ~65 000 markers each time:
/// growing eight fresh vectors and the merged list per frame was a visible share of the host time), or nullptr
void collect_markers(const uint8_t *stream, size_t len, scan_pool *pool, uint8_t *copy_to, std::vector<uint64_t> &markers, std::vector<uint64_t> *scratch = nullptr)
{
        constexpr int kMaxThreads = kMaxScanThreads;
        int nt = len > (4u << 20) ? kMaxThreads : len > (1u << 20) ? 4 : 1;
        if (pool == nullptr || pool->size() + 1 < nt) {
                nt = pool ? pool->size() + 1 : 1;
        }
        std::vector<uint64_t> own[kMaxThreads];
        std::vector<uint64_t> *part = scratch ? scratch : own;
        for (int i = 0; i < kMaxThreads; ++i) {
                part[i].clear();
        }
        const size_t chunk = (len / nt + 15) & ~(size_t) 15;
        auto range = [&](int i) {
                const size_t lo = std::min(len, chunk * i), hi = i == nt - 1 ? len : std::min(len, chunk * (i + 1));
                scan_markers(stream, lo, hi, len, part[i], copy_to);
        };
        if (nt == 1) {
                range(0);
        } else {
                pool->parallel(nt - 1, [&](int w) { range(w + 1); }, [&] { range(0); });
        }
        for (int i = 0; i < nt; ++i) {
                markers.insert(markers.end(), part[i].begin(), part[i].end());
        }
}

int native_codec(const parsed &P)
{
        const dec_geom &g = P.g;
        if (g.ncomp == 4) {
                return UGB_RGBA;  // R G B A as stored (the parser refuses subsampled and YCCK four-component streams)
        }
        if (g.c[0].h == 2) {
                return UGB_UYVY;  // 4:2:2 and 4:2:0 land in UYVY
        }
        const bool rgb = P.adobe == 0 || (P.comp_id[0] == 'R' && P.comp_id[1] == 'G' && P.comp_id[2] == 'B');
        return rgb ? UGB_RGB : UGB_VUYA;
}

}  // namespace

extern "C" {

UGB_API int ugb200_jpeg_get_image_info(const uint8_t *stream, size_t len, struct ugb200_jpeg_image_info *info)
{
        if (!stream || !info) {
                return -1;
        }
        parsed P;
        const int rc = parse_stream(stream, len, P, nullptr, false);
        if (rc != 0) {
                return rc;
        }
        info->width = P.g.w, info->height = P.g.h, info->components = P.g.ncomp;
        info->h_samp = P.g.c[0].h, info->v_samp = P.g.c[0].v;
        info->adobe_transform = P.adobe, info->restart_interval = P.g.ri;
        info->native_codec = native_codec(P);
        return 0;
}

UGB_API long ugb200_jpeg_debug_segments(const uint8_t *stream, size_t len, uint32_t *begin, uint32_t *end, long cap)
{
        if (!stream) {
                return -1;
        }
        parsed P;
        dec_tables T;
        std::vector<uint64_t> markers;
        if (len > (1u << 20)) {  // the same threaded scan the decoder uses
                scan_pool pool(7);
                collect_markers(stream, len, &pool, nullptr, markers);
        } else {
                collect_markers(stream, len, nullptr, nullptr, markers);
        }
        const int rc = parse_stream(stream, len, P, &T, true, &markers);
        if (rc != 0) {
                return rc;
        }
        const long n = (long) P.seg_begin.size();
        for (long i = 0; i < n && i < cap; ++i) {
                begin[i] = P.seg_begin[i], end[i] = P.seg_end[i];
        }
        return n;
}

UGB_API ugb200_jpeg_decoder *ugb200_jpeg_decoder_create(cuda_wrapper_stream_t stream)
{
        ugb200_jpeg_decoder *d = new (std::nothrow) ugb200_jpeg_decoder;
        if (!d) {
                return nullptr;
        }
        d->stream = (cudaStream_t) stream;
        if (cudaMalloc((void **) &d->d_tables, sizeof(dec_tables)) != cudaSuccess || cudaMallocHost((void **) &d->hs[0].tables, sizeof(dec_tables)) != cudaSuccess ||
            cudaMallocHost((void **) &d->hs[1].tables, sizeof(dec_tables)) != cudaSuccess || cudaMallocHost((void **) &d->h_flag, 64) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[0].uploaded, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[1].uploaded, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[0].stream_up, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[1].stream_up, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[0].consumed, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[1].consumed, cudaEventDisableTiming) != cudaSuccess ||
            cudaStreamCreateWithFlags(&d->copy, cudaStreamNonBlocking) != cudaSuccess) {
                ugb200_jpeg_decoder_destroy(d);
                return nullptr;
        }
        const char *m = getenv("UGB200_JPEG_MARKER_SCAN");  // "host" / "device": force one of the two marker scans (tests, A/B timing)
        d->scan_mode = !m ? 0 : m[0] == 'h' ? 1 : m[0] == 'd' ? 2 : 0;
        return d;
}

UGB_API void ugb200_jpeg_decoder_destroy(ugb200_jpeg_decoder *d)
{
        if (!d) {
                return;
        }
        cudaStreamSynchronize(d->stream);
        if (d->copy) {
                cudaStreamSynchronize(d->copy);
                cudaStreamDestroy(d->copy);
        }
        cudaFree(d->planes), cudaFree(d->native), cudaFree(d->staging), cudaFree(d->coef), cudaFree(d->d_seg), cudaFree(d->d_tables);
        cudaFree(d->d_marks), cudaFree(d->d_mark_cnt);
        cudaFreeHost(d->h_flag);
        for (auto &h : d->hs) {
                if (h.stream) {
                        cuda_wrapper_free_host(h.stream);
                }
                cudaFreeHost(h.seg), cudaFreeHost(h.tables);
                cudaFree(h.d_stream);
                for (cudaEvent_t e : { h.stream_up, h.consumed }) {
                        if (e) {
                                cudaEventDestroy(e);
                        }
                }
                if (h.uploaded) {
                        cudaEventDestroy(h.uploaded);
                }
        }
        delete d;
}

/// the segment table of the last decode as the device holds it (tests: the device marker scan against the host's)
UGB_API long ugb200_jpeg_decoder_last_segments(ugb200_jpeg_decoder *d, uint32_t *begin, uint32_t *end, long cap)
{
        if (!d || !begin || !end) {
                return -1;
        }
        const long n = (long) d->last_nseg;
        if (cudaStreamSynchronize(d->stream) != cudaSuccess) {
                return -2;
        }
        const long m = n < cap ? n : cap;
        if (m > 0 && (cudaMemcpy(begin, d->d_seg, (size_t) m * 4, cudaMemcpyDeviceToHost) != cudaSuccess ||
                      cudaMemcpy(end, d->d_seg + n, (size_t) m * 4, cudaMemcpyDeviceToHost) != cudaSuccess)) {
                return -2;
        }
        return n;
}

UGB_API int ugb200_jpeg_decoder_expect(ugb200_jpeg_decoder *d, int width, int height)
{
        if (!d || width < 0 || height < 0) {
                return -1;
        }
        d->expect_w = width, d->expect_h = height;
        return 0;
}

UGB_API int ugb200_jpeg_decode(ugb200_jpeg_decoder *d, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch, int out_codec,
                               int rshift, int gshift, int bshift)
{
        const long dst_pitch_arg = dst_pitch;
        if (!d || !stream || !dst || len > 0xFFFFFFF0u) {
                return -1;
        }
        if (out_codec != UGB_UYVY && out_codec != UGB_RGB && out_codec != UGB_RGBA && out_codec != UGB_VUYA && out_codec != UGB_I420) {
                return -4;
        }
        static const int timing = getenv("UGB200_JPEG_TIMING") ? atoi(getenv("UGB200_JPEG_TIMING")) : 0;  // 1: stage times of the host side on stderr; 2: + device stages
        const auto t_start = std::chrono::steady_clock::now();
        auto lap = [&](const char *what) {
                if (timing) {
                        if (what[0] == '+') {  // device stages: wait for the stream, so that the lap is the stage's own time (serialises the pipeline)
                                if (timing < 2) {
                                        return;
                                }
                                cudaStreamSynchronize(d->stream);
                        }
                        fprintf(stderr, "[jpeg decode] %-14s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count());
                }
        };
        if (d->expect_w > 0) {  // the SOF dimensions are untrusted input and decide how much is written to dst: check them before anything else
                parsed head;
                const int hrc = parse_stream(stream, len, head, nullptr, false);
                if (hrc != 0) {
                        return hrc;
                }
                if (head.g.w != d->expect_w || head.g.h != d->expect_h) {
                        return -3;
                }
        }
        ugb200_jpeg_decoder::host_slot &H = d->hs[d->frame_no++ & 1];
        if (H.pending) {
                cudaEventSynchronize(H.uploaded);  // the uploads of the frame before last left this slot long ago
                cudaEventSynchronize(H.stream_up);
                H.pending = false;
        }
        lap("slot free");
        parsed P;
        P.seg_begin.swap(d->seg_begin), P.seg_end.swap(d->seg_end);  // last frame's capacity
        P.seg_begin.clear(), P.seg_end.clear();
        memset(H.tables, 0, sizeof(dec_tables));
        memcpy(H.tables->zz, kZigzag, 64);
        if (len > H.stream_cap) {  // pinned pages on the GPU's NUMA node (cuda_wrapper_malloc_host_near falls back to cudaMallocHost)
                if (H.stream) {
                        cuda_wrapper_free_host(H.stream);
                }
                H.stream = nullptr, H.stream_cap = 0;
                int device = 0;
                cudaGetDevice(&device);
                const size_t want = len + len / 4 + 4096;
                if (cuda_wrapper_malloc_host_near((void **) &H.stream, want, device) != 0) {
                        return -2;
                }
                H.stream_cap = want;
        }
        // Streams with ONE scan holding all components (UltraGrid's UYVY streams, interleaved RGB): the host reads the headers in front of the SOS and
        // copies the stream to pinned memory; the restart markers are found on the device (jpeg_marker_*_kernel).  Everything else - several scans,
        // whose later SOS headers lie behind entropy-coded data - takes the host scan below.
        size_t scan_data = 0;
        bool device_scan = false, multi = false;
        int rc = 0;
        const bool host_only = d->host_once;
        d->host_once = false;
        if (d->scan_mode != 1 && !host_only && len <= (1u << 30) && (d->scan_mode == 2 || len >= (1u << 20))) {
                rc = parse_stream(stream, len, P, H.tables, false, nullptr, &scan_data);
                device_scan = rc == 0 && P.g.nscans == 1 && P.g.s[0].ns == P.g.ncomp && scan_data > 0;
                if (rc == 0 && !device_scan && P.g.nscans == 1 && P.g.s[0].ns == 1 && P.g.s[0].comp[0] == 0 && P.g.ncomp == 3 && scan_data > 0 && P.have_q[P.g.c[1].tq] &&
                    P.have_q[P.g.c[2].tq]) {
                        // one scan per component, in component order, is what the first SOS promises (GPUJPEG's RGB streams): scans 2 and 3 are laid out as the
                        // host parser would lay them out, their table selectors come from the device, and the device checks the promise
                        dec_geom &g = P.g;
                        for (int id = 0; id < 4; ++id) {  // the kernel reads table id k of scans 2 and 3 from slot k: the first scan took slots by id
                                table_slot(P.hd, H.tables, id);
                        }
                        for (int j = 1; j < 3; ++j) {
                                dec_scan &S = g.s[j];
                                const dec_comp &c = g.c[j];
                                S.ns = 1, S.comp[0] = j, S.td[0] = 0, S.ta[0] = 2;  // table slots: the kernel takes the selectors from the device
                                S.mcux = ((g.w * c.h + g.hmax - 1) / g.hmax + 7) / 8;
                                S.nmcu = S.mcux * (((g.h * c.v + g.vmax - 1) / g.vmax + 7) / 8);
                                S.seg0 = g.s[j - 1].seg0 + g.s[j - 1].nseg;
                                S.nseg = g.ri ? (S.nmcu + g.ri - 1) / g.ri : 1;
                        }
                        g.nscans = 3;
                        device_scan = multi = true;
                }
                if (!device_scan) {  // start over on the host path (tables and geometry are rebuilt there)
                        P.g = dec_geom{}, P.adobe = -1, P.have_sof = false;
                        memset(P.have_q, 0, sizeof P.have_q);
                        P.hd = huff_defs{};
                        memset(H.tables, 0, sizeof(dec_tables));
                        memcpy(H.tables->zz, kZigzag, 64);
                }
        }
        std::vector<uint64_t> &markers = d->markers;
        if (device_scan) {
                const int nt = len > (4u << 20) ? kMaxScanThreads : len > (1u << 20) ? 4 : 1;
                if (nt == 1) {
                        stage_copy(H.stream, stream, len);
                } else {
                        const size_t chunk = (len / nt + 63) & ~(size_t) 63;
                        auto piece = [&](int i) {
                                const size_t lo = std::min(len, chunk * i), hi = i == nt - 1 ? len : std::min(len, chunk * (i + 1));
                                stage_copy(H.stream + lo, stream + lo, hi - lo);
                        };
                        d->pool.parallel(nt - 1, [&](int w) { piece(w + 1); }, [&] { piece(0); });
                }
                lap("stage");
        } else {
                // one pass over the caller's (pageable) buffer: copy it to the pinned staging buffer and collect the marker candidates, split over a
                // few threads when the stream is large (an 8K frame is 5-50 MB)
                markers.clear();
                collect_markers(stream, len, &d->pool, H.stream, markers, d->scan_part);
                lap("scan+stage");
                rc = parse_stream(stream, len, P, H.tables, true, &markers);
        }
        struct give_back {  // the segment vectors return to the decoder on every path out of this function
                parsed &p;
                ugb200_jpeg_decoder *dec;
                ~give_back() { p.seg_begin.swap(dec->seg_begin), p.seg_end.swap(dec->seg_end); }
        } give_back_guard{ P, d };
        if (rc != 0) {
                return rc;
        }
        lap("parse");
        P.g.ntables = multi ? 4 : 0;  // multi: scans 2 and 3 take their selectors from the device, any of slots 0..3 (zeroed when undefined)
        for (int k = 0; k < kTables; ++k) {
                P.g.ntables = P.hd.taken[k] ? k + 1 : P.g.ntables;
        }
        const dec_geom &g = P.g;
        const size_t nseg = multi ? (size_t) (g.s[2].seg0 + g.s[2].nseg) : device_scan ? (size_t) g.s[0].nseg : P.seg_begin.size();
        d->last_nseg = nseg;
        const long plane_bytes = (long) g.nblocks * 64;
        // Four components (R G B A): packed to RGBA when RGBA is asked for - with other shifts than (0, 8, 16) the packed frame then goes through the
        // RGBA -> RGBA line converter, as vc_copylineRGBA re-shifts it (alpha becomes 0xFF) - and to RGB (the first three planes) for any other
        // output, which then takes the routes of an RGB stream
        const int stream_codec = native_codec(P);
        const bool alpha = stream_codec == UGB_RGBA;
        const bool reshift = alpha && out_codec == UGB_RGBA && !(rshift == 0 && gshift == 8 && bshift == 16);
        const int native = alpha && out_codec != UGB_RGBA ? UGB_RGB : stream_codec;
        const long npitch = native == UGB_UYVY ? (long) ((g.w + 1) / 2) * 4 : native == UGB_RGB ? (long) g.w * 3 : (long) g.w * 4;
        const long opitch = out_codec == UGB_UYVY ? (long) ((g.w + 1) / 2) * 4 : out_codec == UGB_RGB ? (long) g.w * 3 : (long) g.w * 4;
        if (dst_pitch == 0) {
                dst_pitch = opitch;
        }
        if (!dgrow(H.d_stream, H.d_stream_cap, len + 16) || !dgrow(d->planes, d->planes_cap, (size_t) plane_bytes) || !dgrow(d->coef, d->coef_cap, (size_t) g.nblocks * 64) ||
            !dgrow(d->d_seg, d->seg_cap, 2 * nseg) || !dgrow(d->native, d->native_cap, (size_t) npitch * g.h + 64) || !hgrow(H.seg, H.seg_cap, 2 * nseg)) {
                return -2;
        }
        cudaStream_t s = d->stream;
        const uint32_t *dev_scans = nullptr;
        // the upload goes over the copy stream: it may start as soon as the kernels of the frame before last have read this slot's device copy, i.e. it
        // runs under the kernels of the previous frame; this frame's kernels wait for it
        uint8_t *const d_stream = H.d_stream;
        if (H.consumed_pending) {
                cudaStreamWaitEvent(d->copy, H.consumed, 0);
        }
        cudaMemcpyAsync(d_stream, H.stream, len, cudaMemcpyHostToDevice, d->copy);
        cudaEventRecord(H.stream_up, d->copy);
        cudaStreamWaitEvent(s, H.stream_up, 0);
        lap("+stream on the device");
        if (device_scan) {
                const unsigned pieces = (unsigned) ((len + kMarkThreads * 16 - 1) / (kMarkThreads * 16));
                if (!dgrow(d->d_marks, d->marks_cap, len / 2 + 2) || !dgrow(d->d_mark_cnt, d->mark_cnt_cap, (size_t) pieces + kMetaWords)) {
                        return -2;
                }
                uint32_t *meta = d->d_mark_cnt + pieces;
                dev_scans = multi ? meta : nullptr;
                jpeg_marker_count_kernel<<<pieces, kMarkThreads, 0, s>>>(d_stream, len, scan_data, d->d_mark_cnt);
                jpeg_marker_scan_kernel<<<1, 1024, 0, s>>>(d->d_mark_cnt, (int) pieces, meta);
                jpeg_marker_write_kernel<<<pieces, kMarkThreads, 0, s>>>(d_stream, len, scan_data, d->d_mark_cnt, d->d_marks, meta);
                if (multi) {
                        jpeg_marker_bounds_kernel<<<1, 32, 0, s>>>(d_stream, (uint32_t) len, d->d_marks, meta, (uint32_t) scan_data, g.nscans,
                                                                   (uint32_t) P.comp_id[0] | (uint32_t) P.comp_id[1] << 8 | (uint32_t) P.comp_id[2] << 16);
                        jpeg_marker_segments_multi_kernel<<<(unsigned) ((nseg + 255) / 256), 256, 0, s>>>(d->d_marks, meta, g.nscans, g.s[1].seg0, g.s[2].seg0, (int) nseg, d->d_seg,
                                                                                                           d->d_seg + nseg);
                        // The verdict must be known before the Huffman kernel is queued (an irregular stream is decoded by the host parser's rules instead).
                        // The wait covers the upload and four small kernels of THIS frame - and whatever the stream still holds of the frame before, which
                        // the device works on anyway; the host side of the next frame still overlaps this frame's Huffman and IDCT kernels.
                        if (cudaMemcpyAsync(d->h_flag, meta + kMetaError, 4, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
                                return -2;
                        }
                        lap("verdict");
                        if (*d->h_flag != 0) {
                                d->host_once = true;
                                return ugb200_jpeg_decode(d, stream, len, dst, dst_is_device, dst_pitch_arg, out_codec, rshift, gshift, bshift);
                        }
                } else {
                        jpeg_marker_segments_kernel<<<(unsigned) ((nseg + 255) / 256), 256, 0, s>>>(d->d_marks, meta, (uint32_t) scan_data, (uint32_t) len, (int) nseg, d->d_seg,
                                                                                                     d->d_seg + nseg);
                }
        } else {
                memcpy(H.seg, P.seg_begin.data(), nseg * 4), memcpy(H.seg + nseg, P.seg_end.data(), nseg * 4);
                cudaMemcpyAsync(d->d_seg, H.seg, 2 * nseg * 4, cudaMemcpyHostToDevice, s);
        }
        cudaMemcpyAsync(d->d_tables, H.tables, sizeof(dec_tables), cudaMemcpyHostToDevice, s);
        cudaEventRecord(H.uploaded, s);
        H.pending = true;
        lap("uploads queued");
        lap("+segments on the device");
        // Does every block of the coefficient array belong to exactly one scan's MCU grid?  (Interleaved scans cover the padded planes by construction; a
        // one-component scan covers ceil(w_c / 8) x ceil(h_c / 8) blocks, which is the whole plane only without MCU padding; a component no scan names - a
        // truncated multi-scan stream - is covered by nobody.)  Then the Huffman kernel writes whole blocks and the array is not cleared.
        bool full = true;
        {
                int seen[4] = { 0, 0, 0, 0 };
                for (int j = 0; j < g.nscans; ++j) {
                        const dec_scan &S = g.s[j];
                        for (int k = 0; k < S.ns; ++k) {
                                ++seen[S.comp[k]];
                        }
                        if (S.ns == 1) {
                                const dec_comp &c = g.c[S.comp[0]];
                                full = full && S.mcux == c.bw && S.nmcu == c.bw * c.bh;
                        }
                }
                full = full && seen[0] == 1 && seen[1] == 1 && seen[2] == 1 && (g.ncomp == 3 || seen[3] == 1);
        }
        const unsigned hgrid = (unsigned) ((nseg + kHuffThreads - 1) / kHuffThreads);
        const size_t hsmem = ((sizeof(dec_tables) + 15) & ~(size_t) 15) + (size_t) kHuffThreads * 128;
        if (full) {
                jpeg_decode_huffman_kernel<true><<<hgrid, kHuffThreads, hsmem, s>>>(d_stream, d->d_seg, d->d_seg + nseg, d->d_tables, g, d->coef, dev_scans);
        } else {
                cudaMemsetAsync(d->coef, 0, (size_t) g.nblocks * 128, s);
                lap("+coefficients cleared");
                jpeg_decode_huffman_kernel<false><<<hgrid, kHuffThreads, hsmem, s>>>(d_stream, d->d_seg, d->d_seg + nseg, d->d_tables, g, d->coef, dev_scans);
        }
        cudaEventRecord(H.consumed, s);  // nothing behind this kernel reads the stream
        H.consumed_pending = true;
        const bool direct = native == out_codec && dst_is_device && !reshift;
        uint8_t *nat = direct ? (uint8_t *) dst : d->native;
        const bool fused_uyvy = native == UGB_UYVY && g.c[0].v == 1;  // 4:2:2: IDCT and packing in one kernel, no component planes
        if (fused_uyvy) {
                const long np = direct ? dst_pitch : npitch;
                jpeg_idct_uyvy_kernel<<<(g.c[1].bw * g.c[1].bh + 31) / 32, 128, 0, s>>>(d->coef, d->d_tables, g, nat, np, !(15 & (size_t) nat) && !(np & 15));
        } else {
                jpeg_idct_kernel<<<(g.nblocks + 127) / 128, 128, 0, s>>>(d->coef, d->d_tables, g, d->planes);
        }
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        lap("kernels queued");
        lap("+huffman + idct");
        // component planes -> the stream's native packed format
        struct ugb200_from_planar_data fp;
        memset(&fp, 0, sizeof fp);
        fp.width = native == UGB_UYVY ? (g.w + 1) & ~1 : g.w;  // the padded planes hold the second luma of an odd last pixel pair
        fp.height = g.h, fp.out_data = nat, fp.out_pitch = (unsigned) (direct ? dst_pitch : npitch);
        for (int i = 0; i < 3; ++i) {
                fp.in_data[i] = d->planes + g.c[i].plane_off, fp.in_linesize[i] = (unsigned) (g.c[i].bw * 8);
        }
        fp.in_depth = 8;
        if (alpha) {  // planes in G, B, R, A order (from_planar.c:335-366); all four have the same line size
                for (int i = 0; i < 4; ++i) {
                        const dec_comp &c = g.c[i == 3 ? 3 : (i + 1) % 3];
                        fp.in_data[i] = d->planes + c.plane_off, fp.in_linesize[i] = (unsigned) (c.bw * 8);
                }
        }
        if (fused_uyvy) {
                rc = 0;
        } else if (alpha) {
                rc = native == UGB_RGBA ? ugb200_gbrap_to_rgba(&fp, s) : ugb200_gbrap_to_rgb(&fp, s);
        } else if (native == UGB_UYVY) {
                rc = g.c[0].v == 2 ? ugb200_yuv420p_to_uyvy(&fp, s) : ugb200_yuv422p_to_uyvy(&fp, s);
        } else if (native == UGB_RGB) {
                rc = ugb200_rgbpXX_to_rgb(&fp, s);
        } else {
                rc = ugb200_yuv444p_to_vuya(&fp, s);
        }
        if (rc != 0) {
                return rc;
        }
        if (direct) {
                return 0;
        }
        if (out_codec == UGB_I420) {  // GPUJPEG_420_U8_P0P1P2 (gpujpeg.c:113-116): Y, then Cb, then Cr plane, tightly packed
                const size_t cw = (size_t) (g.w + 1) / 2, chh = (size_t) (g.h + 1) / 2, total = (size_t) g.w * g.h + 2 * cw * chh;
                uint8_t *uy = nat;
                long uy_pitch = npitch;
                if (native != UGB_UYVY) {
                        if (!ugb200_pixfmt_supported(native, UGB_UYVY) || !dgrow(d->staging, d->staging_cap, (size_t) ((g.w + 1) / 2) * 4 * g.h + total + 64)) {
                                return -4;
                        }
                        uy = d->staging, uy_pitch = (long) ((g.w + 1) / 2) * 4;
                        rc = ugb200_pixfmt_convert(native, UGB_UYVY, uy, uy_pitch, nat, npitch, (int) uy_pitch, g.h, (long) npitch * g.h, 0, 8, 16, s);
                        if (rc != 0) {
                                return rc;
                        }
                } else if (!dgrow(d->staging, d->staging_cap, total + 64)) {
                        return -2;
                }
                uint8_t *planes_out = dst_is_device ? (uint8_t *) dst : d->staging + (native != UGB_UYVY ? (size_t) uy_pitch * g.h : 0);
                struct ugb200_to_planar_data tp;
                memset(&tp, 0, sizeof tp);
                tp.width = g.w, tp.height = g.h, tp.in_data = uy;
                tp.out_data[0] = planes_out, tp.out_data[1] = planes_out + (size_t) g.w * g.h, tp.out_data[2] = tp.out_data[1] + cw * chh;
                tp.out_linesize[0] = (unsigned) g.w, tp.out_linesize[1] = tp.out_linesize[2] = (unsigned) cw;
                if (uy_pitch != (long) ((g.w + 1) / 2) * 4) {
                        return -4;
                }
                rc = ugb200_uyvy_to_i420(&tp, s);
                if (rc != 0 || dst_is_device) {
                        return rc;
                }
                return cudaMemcpyAsync(dst, planes_out, total, cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess ? 0 : -2;
        }
        // native -> requested codec (UltraGrid's own line converters), then to the caller
        uint8_t *result = nat;
        long rpitch = npitch;
        if (native != out_codec || reshift) {
                if (!ugb200_pixfmt_supported(native, out_codec)) {
                        return -4;
                }
                uint8_t *conv;
                if (dst_is_device) {
                        conv = (uint8_t *) dst, rpitch = dst_pitch;
                } else {
                        if (!dgrow(d->staging, d->staging_cap, (size_t) opitch * g.h + 64)) {
                                return -2;
                        }
                        conv = d->staging, rpitch = opitch;
                }
                const int len_out = out_codec == UGB_UYVY ? ((g.w + 1) / 2) * 4 : out_codec == UGB_RGB ? g.w * 3 : g.w * 4;
                rc = ugb200_pixfmt_convert(native, out_codec, conv, rpitch, nat, npitch, len_out, g.h, (long) npitch * g.h, rshift, gshift, bshift, s);
                if (rc != 0) {
                        return rc;
                }
                result = conv;
                if (dst_is_device) {
                        return 0;
                }
        }
        if (dst_is_device) {
                return cudaMemcpy2DAsync(dst, dst_pitch, result, rpitch, opitch, g.h, cudaMemcpyDeviceToDevice, s) == cudaSuccess ? 0 : -2;
        }
        if (cudaMemcpy2DAsync(dst, dst_pitch, result, rpitch, opitch, g.h, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
                return -2;
        }
        return 0;
}

}  // extern "C"
