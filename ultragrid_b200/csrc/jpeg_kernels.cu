// Baseline JPEG encoder (include/ugb200_jpeg.h): the DCT / quantisation / Huffman stage GPUJPEG performs for
// UltraGrid's src/video_compress/gpujpeg.cpp, re-designed for sm_90a (Hopper).
//
// Round-1 structure (correct first; fusion of the stages is the next optimisation step, see DESIGN.md):
//   K1 jpeg_dct_kernel      one thread per 8x8 block: 128-bit row loads straight from UYVY / packed RGB, level
//                           shift, separable AAN FDCT in registers, quantise (reciprocal multiply + rint),
//                           zig-zag, one 128-byte store of int16 coefficients          (HBM: 1 B in, 2 B out per sample)
//   K2 jpeg_huffman_kernel  one thread per restart segment: non-zero map per block, one loop turn per NON-ZERO coefficient,
//                           Annex K codes + byte stuffing into a private worst-case slot (32-bit stores), RSTn, byte count
//   K3 jpeg_scan_kernel     second level of the stream-offset prefix sum (first level: inside K2's CTAs); no host round trip
//   K4 jpeg_compact_kernel  eight lanes per segment: slot -> final position (aligned 32-bit stores); writes SOS headers of scans 2,3 and EOI
// Arithmetic is float with an explicit operation order so that oracle/jpeg_oracle.c reproduces the bytes exactly.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <vector>

#include "../../include/ugb200.h"
#include "../../include/ugb200_jpeg.h"
#include "color_space.h"
#include "jpeg_compact.cuh"
#include "f32x2.cuh"
#include "jpeg_tables.h"

namespace ugb {

// FMT_PLANAR: three 8-bit planes (I420 read in place, or the planes jpeg_prep_kernel writes), a YCbCr stream with luma sampled
// 1x1, 2x1 or 2x2 and chroma 1x1; it always takes the split path (an interleaved 4:2:0 MCU has 6 blocks)
enum { FMT_UYVY_422 = 0, FMT_RGB_444 = 1, FMT_PLANAR = 2 };
constexpr int kSlotBytesPerBlock = 416;  // worst case: 1658 bits/block = 208 B, every byte stuffed
constexpr int kSlotExtra = 8;            // final pad byte + RSTn

// Per-encoder tables, no module-level state (encoders with different quality may run concurrently on one device):
//   the quantiser multipliers travel BY VALUE as a kernel parameter - they sit in the constant bank of that launch and are read with
//   immediate offsets exactly like a __constant__ array;
//   the Huffman code tables live in a small per-encoder global buffer; a CTA copies them to shared memory with coalesced loads
//   (indexing a constant bank with the thread id would serialise into 32 replays per warp).
struct jpeg_qtab {
        float qmul[2][64];     // [luma|chroma][natural index]
};
struct jpeg_hufftab {
        uint32_t dc[2][16];    // (len << 16) | code, by category
        uint32_t ac[2][256];   // (len << 16) | code, by (run << 4 | size)
};

struct jpeg_geom {
        int fmt, w, h;
        int bw, bh;        // component-0 blocks per row / rows (RGB), or MCUs per row / rows (UYVY)
        int nblocks;       // total 8x8 blocks (all components)
        int ri;            // MCUs per restart segment
        int nseg;          // total restart segments (all scans)
        int seg_per_scan;  // segments in one scan
        int mcu_per_scan;  // MCUs in one scan
        int blocks_per_mcu;
        int slot;          // bytes reserved per segment
        int header_len;    // bytes before the first entropy-coded byte (including the first SOS)
        int sos_len;       // length of one later SOS header (RGB)
        int interleaved;   // RGB only: one scan, MCU = the R, G and B block of an 8x8 area (GPUJPEG's `interleaved` option, gpujpeg.cpp:303)
};

// Scan table of every stream (the offset scan and the compaction read it) and the geometry of FMT_PLANAR.  Kept out of jpeg_geom, which
// the fused kernel takes: its code stays exactly as it was.
struct jpeg_layout {
        int nscans;        // scans in the stream
        int scan_seg0[4];  // first segment of each scan; the entries from nscans on hold nseg
        // FMT_PLANAR only
        int hs, vs;                  // luma sampling factors (chroma is 1x1)
        int scan_mcus[3];            // MCUs of each scan
        int comp_bw[3], comp_blk0[3];  // non-interleaved: blocks per row of each component (T.81 A.2) and its first block in scan order
        int plane_w[3], plane_h[3];  // valid samples of each plane (edges replicate the last column / row)
        long plane_pitch[3];
        const uint8_t *plane[3];
};

// ---- K1 -------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fdct8(float &d0, float &d1, float &d2, float &d3, float &d4, float &d5, float &d6, float &d7)
{
        const float t0 = __fadd_rn(d0, d7), t7 = __fadd_rn(d0, -d7), t1 = __fadd_rn(d1, d6), t6 = __fadd_rn(d1, -d6);
        const float t2 = __fadd_rn(d2, d5), t5 = __fadd_rn(d2, -d5), t3 = __fadd_rn(d3, d4), t4 = __fadd_rn(d3, -d4);
        const float e0 = __fadd_rn(t0, t3), e3 = __fadd_rn(t0, -t3), e1 = __fadd_rn(t1, t2), e2 = __fadd_rn(t1, -t2);
        d0 = __fadd_rn(e0, e1);
        d4 = __fadd_rn(e0, -e1);
        const float s1 = __fadd_rn(e2, e3);  // every multiply-add is one explicit FMA: no product feeds a separate add, so this
        d2 = __fmaf_rn(s1, 0.707106781f, e3);  // function and its paired twin fdct8_2() compute the same operation tree
        d6 = __fmaf_rn(s1, -0.707106781f, e3);
        const float o0 = __fadd_rn(t4, t5), o1 = __fadd_rn(t5, t6), o2 = __fadd_rn(t6, t7);
        const float z5 = __fmul_rn(__fadd_rn(o0, -o2), 0.382683433f);
        const float z2 = __fmaf_rn(0.541196100f, o0, z5);
        const float z4 = __fmaf_rn(1.306562965f, o2, z5);
        const float z11 = __fmaf_rn(o1, 0.707106781f, t7), z13 = __fmaf_rn(o1, -0.707106781f, t7);
        d5 = __fadd_rn(z13, z2);
        d3 = __fadd_rn(z13, -z2);
        d1 = __fadd_rn(z11, z4);
        d7 = __fadd_rn(z11, -z4);
}

__device__ __forceinline__ int clampi(int v, int hi) { return min(max(v, 0), hi); }

/// level-shifted sample as float without the slow I2F pipe: as_float(0x4B000000 | b) = 2^23 + b, minus (2^23 + 128) is exact
__device__ __forceinline__ float shifted(uint32_t word, unsigned byte_sel)
{
        return __fadd_rn(__uint_as_float(__byte_perm(word, 0x4B000000u, 0x7540u | byte_sel)), -8388736.0f);
}

/// 8 samples of one row of the block into f[0..7] (already level-shifted)
__device__ __forceinline__ void load_row(const uint8_t *__restrict__ src, long pitch, const jpeg_geom &g, int comp, int bx, int y,
                                         bool interior, float *f)
{
        const uint8_t *row = src + (long) clampi(y, g.h - 1) * pitch;
        if (g.fmt == FMT_UYVY_422) {
                if (interior && comp == 0) {  // 8 luma samples = 16 bytes
                        const uint4 v = __ldg((const uint4 *) (row + (long) bx * 16));
                        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                                f[2 * i] = shifted(w[i], 1);
                                f[2 * i + 1] = shifted(w[i], 3);
                        }
                } else if (interior) {  // 8 chroma samples = 32 bytes
                        const uint4 a = __ldg((const uint4 *) (row + (long) bx * 32)), b = __ldg((const uint4 *) (row + (long) bx * 32) + 1);
                        const uint32_t w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
                        const unsigned sel = comp == 1 ? 0 : 2;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                f[i] = shifted(w[i], sel);
                        }
                } else {
#pragma unroll
                        for (int x = 0; x < 8; ++x) {
                                int s;
                                if (comp == 0) {
                                        s = row[2 * clampi(bx * 8 + x, g.w - 1) + 1];
                                } else {
                                        s = row[4 * clampi(bx * 8 + x, (g.w + 1) / 2 - 1) + (comp == 1 ? 0 : 2)];
                                }
                                f[x] = shifted((uint32_t) s, 0);
                        }
                }
        } else {
#pragma unroll
                for (int x = 0; x < 8; ++x) {
                        f[x] = shifted((uint32_t) __ldg(row + 3 * clampi(bx * 8 + x, g.w - 1) + comp), 0);
                }
        }
}

/// 8 samples of one row of a block of plane `comp` (FMT_PLANAR); interior: 8-byte aligned and inside the plane
__device__ __forceinline__ void load_row_planar(const jpeg_layout &L, int comp, int bx, int y, bool interior, float *f)
{
        const uint8_t *plane = comp == 0 ? L.plane[0] : comp == 1 ? L.plane[1] : L.plane[2];
        const long pitch = comp == 0 ? L.plane_pitch[0] : comp == 1 ? L.plane_pitch[1] : L.plane_pitch[2];
        const int pw = comp == 0 ? L.plane_w[0] : L.plane_w[1], ph = comp == 0 ? L.plane_h[0] : L.plane_h[1];
        const uint8_t *row = plane + (long) clampi(y, ph - 1) * pitch;
        if (interior) {
                const uint2 v = __ldg((const uint2 *) (row + (long) bx * 8));
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        f[i] = shifted(v.x, i);
                        f[4 + i] = shifted(v.y, i);
                }
        } else {
#pragma unroll
                for (int x = 0; x < 8; ++x) {
                        f[x] = shifted((uint32_t) __ldg(row + clampi(bx * 8 + x, pw - 1)), 0);
                }
        }
}

/// PLANAR: FMT_PLANAR geometry (a template flag, so that the UYVY / RGB instantiation keeps its code)
template <bool PLANAR>
__global__ void __launch_bounds__(128) jpeg_dct_kernel(const uint8_t *__restrict__ src, long pitch, jpeg_geom g, int16_t *__restrict__ coef,
                                                       bool vec_ok, const __grid_constant__ jpeg_qtab qt, const __grid_constant__ jpeg_layout L)
{
        int b = blockIdx.x * blockDim.x + threadIdx.x;
        int comp, bx, by;
        if (PLANAR) {
                if (b >= g.nblocks) {
                        return;
                }
                if (g.interleaved) {  // MCU = hs x vs luma blocks in raster order, then Cb, Cr (T.81 A.2.3)
                        const int nl = L.hs * L.vs, m = b / g.blocks_per_mcu, k = b - m * g.blocks_per_mcu;
                        const int mx = m % g.bw, my = m / g.bw;
                        comp = k < nl ? 0 : k - nl + 1;
                        bx = k < nl ? mx * L.hs + k % L.hs : mx;
                        by = k < nl ? my * L.vs + k / L.hs : my;
                } else {  // one scan per component, each in raster order of its own block grid
                        comp = b >= L.comp_blk0[2] ? 2 : b >= L.comp_blk0[1] ? 1 : 0;
                        const int r = b - (comp == 0 ? 0 : comp == 1 ? L.comp_blk0[1] : L.comp_blk0[2]);
                        const int cbw = comp == 0 ? L.comp_bw[0] : comp == 1 ? L.comp_bw[1] : L.comp_bw[2];
                        bx = r % cbw, by = r / cbw;
                }
        } else if (g.fmt == FMT_UYVY_422) {
                // a CTA of 4 warps owns 32 MCUs; warp k encodes block k (Y0, Y1, Cb, Cr) of each, so that a warp is
                // component-uniform: no luma/chroma divergence, uniform constant-bank reads of the quantiser table
                const int k = threadIdx.x >> 5, m = blockIdx.x * 32 + (threadIdx.x & 31);
                if (m >= g.mcu_per_scan) {
                        return;
                }
                b = m * 4 + k;
                const int mx = m % g.bw, my = m / g.bw;
                comp = k < 2 ? 0 : k - 1;
                bx = comp == 0 ? mx * 2 + k : mx;
                by = my;
        } else {
                if (b >= g.nblocks) {
                        return;
                }
                if (g.interleaved) {  // scan order: block b = component b % 3 of MCU b / 3
                        const int m = b / 3;
                        comp = b - 3 * m;
                        bx = m % g.bw, by = m / g.bw;
                } else {
                        const int per = g.bw * g.bh;
                        comp = b / per;
                        const int r = b - comp * per;
                        bx = r % g.bw, by = r / g.bw;
                }
        }
        // interior: the whole block lies inside the image (and vector loads are aligned)
        float f[64];
        if (PLANAR) {
                const int pw = comp == 0 ? L.plane_w[0] : L.plane_w[1], ph = comp == 0 ? L.plane_h[0] : L.plane_h[1];
                const bool interior = vec_ok && (bx + 1) * 8 <= pw && (by + 1) * 8 <= ph;
#pragma unroll
                for (int y = 0; y < 8; ++y) {
                        load_row_planar(L, comp, bx, by * 8 + y, interior, f + 8 * y);
                }
        } else {
                const int px_w = (g.fmt == FMT_UYVY_422 && comp != 0) ? 16 : 8;
                const bool interior = vec_ok && (bx + 1) * px_w <= g.w && (by + 1) * 8 <= g.h;
#pragma unroll
                for (int y = 0; y < 8; ++y) {
                        load_row(src, pitch, g, comp, bx, by * 8 + y, interior, f + 8 * y);
                }
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
                fdct8(f[8 * r], f[8 * r + 1], f[8 * r + 2], f[8 * r + 3], f[8 * r + 4], f[8 * r + 5], f[8 * r + 6], f[8 * r + 7]);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
                fdct8(f[c], f[8 + c], f[16 + c], f[24 + c], f[32 + c], f[40 + c], f[48 + c], f[56 + c]);
        }
        const float *qm = qt.qmul[comp == 0 ? 0 : 1];
        int q[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) {
                q[i] = (int) __float_as_uint(__fmaf_rn(f[i], qm[i], 12582912.0f)) - 0x4B400000;  // nearest-even of the exact product, no F2I
        }
        // zig-zag (Figure A.6) + AC clamp to the 10-bit category range, two int16 per word, 8 x 16-byte stores
        constexpr int zz[64] = { 0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };
        uint32_t o[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) {
                int a = q[zz[2 * k]], c2 = q[zz[2 * k + 1]];
                if (k > 0) {
                        a = min(max(a, -1023), 1023);
                }
                c2 = min(max(c2, -1023), 1023);
                o[k] = ((uint32_t) a & 0xffffu) | ((uint32_t) c2 << 16);
        }
        uint4 *dst = (uint4 *) (coef + (long) b * 64);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
                dst[k] = make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
        }
}

// ---- paired (float2) helpers of the fused kernel: two lanes per call (f32x2.cuh), same roundings as the scalar code ----------
__device__ __forceinline__ float2 neg2(float2 a) { return make_float2(-a.x, -a.y); }  // folds into the operand modifier
__device__ __forceinline__ void fdct8_2(float2 &d0, float2 &d1, float2 &d2, float2 &d3, float2 &d4, float2 &d5, float2 &d6, float2 &d7)
{
        const float2 t0 = __fadd2_rn(d0, d7), t7 = __fadd2_rn(d0, neg2(d7)), t1 = __fadd2_rn(d1, d6), t6 = __fadd2_rn(d1, neg2(d6));
        const float2 t2 = __fadd2_rn(d2, d5), t5 = __fadd2_rn(d2, neg2(d5)), t3 = __fadd2_rn(d3, d4), t4 = __fadd2_rn(d3, neg2(d4));
        const float2 e0 = __fadd2_rn(t0, t3), e3 = __fadd2_rn(t0, neg2(t3)), e1 = __fadd2_rn(t1, t2), e2 = __fadd2_rn(t1, neg2(t2));
        d0 = __fadd2_rn(e0, e1);
        d4 = __fadd2_rn(e0, neg2(e1));
        const float2 s1 = __fadd2_rn(e2, e3);
        d2 = __ffma2_rn(s1, make_float2(0.707106781f, 0.707106781f), e3);
        d6 = __ffma2_rn(s1, make_float2(-0.707106781f, -0.707106781f), e3);
        const float2 o0 = __fadd2_rn(t4, t5), o1 = __fadd2_rn(t5, t6), o2 = __fadd2_rn(t6, t7);
        const float2 z5 = __fmul2_rn(__fadd2_rn(o0, neg2(o2)), make_float2(0.382683433f, 0.382683433f));
        const float2 z2 = __ffma2_rn(make_float2(0.541196100f, 0.541196100f), o0, z5);
        const float2 z4 = __ffma2_rn(make_float2(1.306562965f, 1.306562965f), o2, z5);
        const float2 z11 = __ffma2_rn(o1, make_float2(0.707106781f, 0.707106781f), t7), z13 = __ffma2_rn(o1, make_float2(-0.707106781f, -0.707106781f), t7);
        d5 = __fadd2_rn(z13, z2);
        d3 = __fadd2_rn(z13, neg2(z2));
        d1 = __fadd2_rn(z11, z4);
        d7 = __fadd2_rn(z11, neg2(z4));
}
/// the 8 samples of one row of a block as 2^23 + sample (level shift and conversion happen in one packed add later)
/// TILE_ONLY: the caller guarantees the staged tile (the global-memory forms below are not instantiated: LEAN kernels)
template <bool TILE_ONLY = false>
__device__ __forceinline__ void load_row_magic(const uint8_t *__restrict__ src, long pitch, const jpeg_geom &g, int comp, int bx, int y, bool interior,
                                               float *m, const uint8_t *tile_row = nullptr, int tile_x = 0)
{
        if (TILE_ONLY || tile_row != nullptr) {  // the CTA's 8 x 1024-byte input tile is in shared memory (UYVY only): tile_x = my MCU within the tile
                if (comp == 0) {
                        const uint4 v = *(const uint4 *) (tile_row + tile_x * 32 + (bx & 1) * 16);
                        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                                m[2 * i] = __uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7541u));
                                m[2 * i + 1] = __uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7543u));
                        }
                } else {
                        const uint4 a = *(const uint4 *) (tile_row + tile_x * 32), b = *(const uint4 *) (tile_row + tile_x * 32 + 16);
                        const uint32_t w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
                        const unsigned sel = comp == 1 ? 0x7540u : 0x7542u;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                m[i] = __uint_as_float(__byte_perm(w[i], 0x4B000000u, sel));
                        }
                }
                return;
        }
        if (TILE_ONLY) {
                return;
        }
        const uint8_t *row = src + (long) clampi(y, g.h - 1) * pitch;
        if (g.fmt == FMT_UYVY_422) {
                if (interior && comp == 0) {
                        const uint4 v = __ldg((const uint4 *) (row + (long) bx * 16));
                        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                                m[2 * i] = __uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7541u));
                                m[2 * i + 1] = __uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7543u));
                        }
                } else if (interior) {
                        const uint4 a = __ldg((const uint4 *) (row + (long) bx * 32)), b = __ldg((const uint4 *) (row + (long) bx * 32) + 1);
                        const uint32_t w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
                        const unsigned sel = comp == 1 ? 0x7540u : 0x7542u;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                m[i] = __uint_as_float(__byte_perm(w[i], 0x4B000000u, sel));
                        }
                } else {
#pragma unroll
                        for (int x = 0; x < 8; ++x) {
                                uint32_t s;
                                if (comp == 0) {
                                        s = row[2 * clampi(bx * 8 + x, g.w - 1) + 1];
                                } else {
                                        s = row[4 * clampi(bx * 8 + x, (g.w + 1) / 2 - 1) + (comp == 1 ? 0 : 2)];
                                }
                                m[x] = __uint_as_float(0x4B000000u | s);
                        }
                }
        } else {
#pragma unroll
                for (int x = 0; x < 8; ++x) {
                        m[x] = __uint_as_float(0x4B000000u | (uint32_t) __ldg(row + 3 * clampi(bx * 8 + x, g.w - 1) + comp));
                }
        }
}

/// the 8 samples of component `comp` of one block row from the staged packed-RGB tile: 24 bytes at an 8-byte aligned shared address.  The row is
/// shifted down by `comp` bytes (funnel shifts), after which the samples sit at the fixed byte offsets 0, 3, 6 ... 21
__device__ __forceinline__ void load_row_rgb_tile(const uint8_t *p, int comp, float *m)
{
        const uint2 a = *(const uint2 *) p, b = *(const uint2 *) (p + 8), c = *(const uint2 *) (p + 16);
        const unsigned sh = 8u * (unsigned) comp;
        const uint32_t v0 = __funnelshift_r(a.x, a.y, sh), v1 = __funnelshift_r(a.y, b.x, sh), v2 = __funnelshift_r(b.x, b.y, sh);
        const uint32_t v3 = __funnelshift_r(b.y, c.x, sh), v4 = __funnelshift_r(c.x, c.y, sh), v5 = __funnelshift_r(c.y, 0u, sh);
        m[0] = __uint_as_float(__byte_perm(v0, 0x4B000000u, 0x7540u));  // byte 0
        m[1] = __uint_as_float(__byte_perm(v0, 0x4B000000u, 0x7543u));  // byte 3
        m[2] = __uint_as_float(__byte_perm(v1, 0x4B000000u, 0x7542u));  // byte 6
        m[3] = __uint_as_float(__byte_perm(v2, 0x4B000000u, 0x7541u));  // byte 9
        m[4] = __uint_as_float(__byte_perm(v3, 0x4B000000u, 0x7540u));  // byte 12
        m[5] = __uint_as_float(__byte_perm(v3, 0x4B000000u, 0x7543u));  // byte 15
        m[6] = __uint_as_float(__byte_perm(v4, 0x4B000000u, 0x7542u));  // byte 18
        m[7] = __uint_as_float(__byte_perm(v5, 0x4B000000u, 0x7541u));  // byte 21
}

// ---- fused path: DCT + quantise + per-block entropy coding + restart-segment assembly in ONE kernel ----------------------------
// No int16 coefficient round trip through HBM (2 B/sample written + read by the split path), and the unit of serial work is one
// 8x8 block instead of one restart segment.  CTA = 128 threads = 128 blocks in scan order:
//   1. every thread loads its block straight from the frame, DCT + quantise in registers, zig-zag coefficients to shared memory
//   2. DC prediction through shared memory, Huffman-codes its block into a private (shared-memory) bit string
//   3. threads are re-mapped to blocks in scan order; the blocks of a restart segment (4..32 threads) prefix-sum their bit lengths
//      and OR their bit strings into the segment buffer
//   4. the same threads byte-stuff the segment cooperatively (ballot of 0xFF bytes) into its slot, append RSTn, record the size
//   5. CTA-level prefix of its segment sizes (first level of the stream-offset scan, as in the split path)
//
// Shared memory is what bounds the occupancy of this kernel, and a block's worst case is 1658 bits (52 words) although a
// typical one needs well below 200.  The per-block bit strings are therefore CAPPED at `cap` words (16 by default = 35 KB per
// CTA, six CTAs per SM).  A CTA in which any block exceeds the cap (noise at high quality) takes the serial route instead:
// one thread per restart segment codes its blocks from the shared coefficients straight into the slot, exactly like the split
// path's jpeg_huffman_kernel.  The largest block seen is reported so that the host can raise the cap for the next frame.
constexpr int kBlkWords = 52;  // 1658 bits worst case per block
constexpr int kCapDefault = 16;

__device__ __forceinline__ int category(int v) { return 32 - __clz(abs(v)); }

/// Shared-memory column of scan-order block p (0..127).  The arrays indexed by block ([k][128] words) are touched in two patterns: phases 1-2
/// with p = 4 * lane + component (stride 4: a 4-way bank conflict on a plain layout) and phase 3 with p = tid (stride 1).  Rotating each
/// group of 32 columns by its group index makes both conflict-free: bank = (p + p / 32) mod 32.
__device__ __forceinline__ int blk_col(int p) { return (p & ~31) | ((p + (p >> 5)) & 31); }

/// MSB-first bit writer with byte stuffing; bytes are gathered into aligned 32-bit words before they go to memory
struct bit_writer {
        uint32_t *p;     // next aligned word of the slot
        uint32_t word;   // bytes gathered so far (little endian in memory)
        int nbytes;      // 0..3 bytes in `word`
        uint64_t acc;
        int nbits;
        __device__ __forceinline__ void emit_byte(uint32_t b)
        {
                word |= b << (8 * nbytes);
                if (++nbytes == 4) {
                        *p++ = word;
                        word = 0, nbytes = 0;
                }
        }
        __device__ __forceinline__ void put(uint32_t code, int len)
        {
                acc = (acc << len) | (code & ((1u << len) - 1u));
                nbits += len;
                while (nbits >= 8) {
                        const uint32_t b = (uint32_t) (acc >> (nbits - 8)) & 0xffu;
                        emit_byte(b);
                        if (b == 0xFF) {
                                emit_byte(0);  // T.81 B.1.1.5
                        }
                        nbits -= 8;
                }
        }
        __device__ __forceinline__ void flush_bits()
        {
                if (nbits > 0) {
                        put(0x7F, 8 - nbits);  // pad with ones, T.81 F.1.2.3
                }
                acc = 0, nbits = 0;
        }
        /// @returns total bytes written to the slot starting at `base`
        __device__ __forceinline__ uint32_t finish(uint32_t *base)
        {
                const uint32_t n = (uint32_t) (p - base) * 4 + nbytes;
                if (nbytes) {
                        *p = word;
                }
                return n;
        }
};


struct block_bits {  // MSB-first bit string of one block in shared memory, word w of block p at base[w * 128 + p]
        uint32_t *base;
        uint64_t acc;
        int nbits, nwords, cap;  // words beyond `cap` are counted but not stored
        __device__ __forceinline__ void put(uint32_t code, int len)  // code must not have bits above len
        {
                acc = (acc << len) | code;
                nbits += len;
                if (nbits >= 32) {
                        if (nwords < cap) {
                                base[nwords * 128] = (uint32_t) (acc >> (nbits - 32));
                        }
                        ++nwords;
                        nbits -= 32;
                }
        }
        __device__ __forceinline__ uint32_t finish()
        {
                if (nbits > 0 && nwords < cap) {
                        base[nwords * 128] = (uint32_t) ((acc & ((1ull << nbits) - 1ull)) << (32 - nbits));
                }
                return (uint32_t) (nwords * 32 + nbits);
        }
};

/// byte stuffing of one assembled restart segment (T bits in `seg`, MSB first) by the bps threads of its group; appends RSTn when rst >= 0.
/// @returns the number of bytes written (identical in every thread of the group)
__device__ __forceinline__ uint32_t stuff_segment(uint8_t *__restrict__ dst, const uint32_t *seg, uint32_t T, int bps, int gl, unsigned lane32, unsigned gmask,
                                                  int rst)
{
        uint32_t written = 0;
        const uint32_t n = (T + 7) >> 3;
        for (uint32_t base = 0; base < n; base += bps) {
                const uint32_t i = base + gl;
                const uint32_t b = i < n ? (seg[i >> 2] >> (24 - 8 * (i & 3))) & 0xffu : 0u;
                const unsigned ff = __ballot_sync(gmask, b == 0xFF) & gmask;
                const uint32_t before = __popc(ff & ((1u << lane32) - 1u));
                if (i < n) {
                        dst[written + gl + before] = (uint8_t) b;
                        if (b == 0xFF) {
                                dst[written + gl + before + 1] = 0;
                        }
                }
                written += min((uint32_t) bps, n - base) + __popc(ff);
        }
        if (rst >= 0) {
                if (gl == 0) {
                        dst[written] = 0xFF, dst[written + 1] = (uint8_t) rst;
                }
                written += 2;
        }
        return written;
}

/// The same stuffing a 32-bit word (four segment bytes) per lane and round instead of a byte: the stuffed segment is built in the CTA's shared
/// staging area `stage` (capacity `cap_bytes`; the dead per-block bit strings) with byte stores there, and leaves for its slot as aligned
/// 32-bit words.  A round handles 4 * bps bytes with one prefix scan - the byte-wise routine above needs four times as many rounds and
/// writes every byte to global memory by itself.  @returns the stuffed size, or 0xFFFFFFFF if it did not fit the staging area (nothing
/// written to the slot then: the caller falls back to stuff_segment()).
__device__ __forceinline__ uint32_t stuff_segment_words(uint8_t *__restrict__ slot, uint8_t *stage, uint32_t cap_bytes, const uint32_t *seg, uint32_t T, int bps,
                                                        int gl, unsigned gmask, int rst)
{
        const uint32_t n = (T + 7) >> 3, nw = (n + 3) >> 2;
        uint32_t written = 0;
        for (uint32_t base = 0; base < nw; base += bps) {
                const uint32_t wi = base + gl;
                const uint32_t w = wi < nw ? seg[wi] : 0u;                       // bytes beyond n are zero (the segment image starts cleared)
                const uint32_t nb = wi < nw ? min(4u, n - 4u * wi) : 0u;
                const uint32_t ff = __vcmpeq4(w, 0xFFFFFFFFu);                   // 0xFF in every byte that needs a stuffed zero behind it
                const uint32_t mine = nb + (__popc(ff) >> 3);
                uint32_t incl = mine;
                for (int d = 1; d < bps; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(gmask, incl, d, bps);
                        if (gl >= d) {
                                incl += o;
                        }
                }
                uint32_t pos = written + incl - mine;
                written += __shfl_sync(gmask, incl, bps - 1, bps);
                if (pos + mine <= cap_bytes) {
                        if (ff == 0) {
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                        if ((uint32_t) k < nb) {
                                                stage[pos + k] = (uint8_t) (w >> (24 - 8 * k));
                                        }
                                }
                        } else {
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                        if ((uint32_t) k < nb) {
                                                const uint32_t b = (w >> (24 - 8 * k)) & 0xffu;
                                                stage[pos++] = (uint8_t) b;
                                                if (b == 0xFF) {
                                                        stage[pos++] = 0;
                                                }
                                        }
                                }
                        }
                }
        }
        if (rst >= 0) {
                if (gl == 0 && written + 2 <= cap_bytes) {
                        stage[written] = 0xFF, stage[written + 1] = (uint8_t) rst;
                }
                written += 2;
        }
        if (written > cap_bytes) {
                return 0xFFFFFFFFu;
        }
        __syncwarp(gmask);
        const uint32_t *sw = (const uint32_t *) stage;  // stage and slot are both 8-byte aligned; the bytes behind `written` in the last word are
        uint32_t *dw = (uint32_t *) slot;               // don't-care (the compaction copies `written` bytes)
        for (uint32_t i = gl; i * 4 < written; i += bps) {
                dw[i] = sw[i];
        }
        return written;
}

/// Single-pass stream compaction (decoupled look-back): when `state` is set the kernel writes the stuffed segments straight to their final
/// position in the stream, so that neither the per-segment slots nor the scan / compact kernels are needed.  A CTA takes a ticket (its
/// logical index: every CTA with a smaller one has started), publishes the byte count of its segments, adds up the counts of its
/// predecessors until it meets one that already knows its own prefix, publishes its prefix, and writes.
struct jpeg_lookback {
        unsigned long long *state;  // per CTA: flag << 62 | bytes; flag 1 = own count, 2 = inclusive prefix (zeroed before the launch)
        uint32_t *ticket;           // zeroed before the launch
        uint8_t *out;
        uint32_t out_cap;
        uint32_t *total;
        int ctas_per_scan;
};

// ---- TMA (bulk async copy) staging of the input tile: one thread arms an mbarrier with the byte count and issues one cp.async.bulk per tile
//      row; the copy engine moves the rows while the CTA fetches its Huffman tables, and every thread waits on the mbarrier itself - no
//      per-thread LDGSTS, no commit / wait group (SASS: UBLKCP + SYNCS)
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t) __cvta_generic_to_shared(bar)), "r"(count) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes)
{
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t) __cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar)
{
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"((uint32_t) __cvta_generic_to_shared(dst)),
                     "l"(src), "r"(bytes), "r"((uint32_t) __cvta_generic_to_shared(bar))
                     : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity)
{
        asm volatile("{\n\t"
                     ".reg .pred p;\n\t"
                     "WAIT_%=:\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                     "@p bra DONE_%=;\n\t"
                     "bra WAIT_%=;\n\t"
                     "DONE_%=:\n\t"
                     "}" ::"r"((uint32_t) __cvta_generic_to_shared(bar)),
                     "r"(parity)
                     : "memory");
}

/// MINB = resident CTAs per SM the register allocation aims at: 6 (80 registers) for any cap, 7 (72 registers) when the bit buffers are
/// capped at 12 words or fewer (28 KB of dynamic shared memory per CTA)
/// BLOCKS_ONLY (round 2, the two-kernel form): the kernel stops behind the entropy phase.  The bit string of every block goes to global memory
/// (`gbits`, [CTA][word][128 blocks] - the layout of the shared array, so the stores of a warp are contiguous), its length to `glen`, and
/// jpeg_assemble_kernel builds the restart segments from them.  What that buys: this kernel has no barrier behind its unequal part (a CTA's chroma
/// warps finish their entropy coding long before its luma warps), needs 16 KB of
/// shared memory instead of 28, and the assembly runs as a light kernel of its own at full occupancy.  A block longer than `cap` words (noise) also
/// leaves its coefficients in `gcoef` (DC slot = the DC DIFFERENCE), from which the assembly kernel codes it again inside a serial segment.
/// LEAN (state j): an instantiation for frames in which EVERY CTA's tile is whole and goes through the copy engine (the host checks the geometry: 8K and other sizes whose
/// MCU rows are multiples of the tile) - the global-memory fall-back loads, the cp.async staging and the edge handling are not compiled in: about a fifth less code in
/// a kernel whose instruction fetch shows up in the stall list (`no_instruction`).  Same arithmetic, same bytes.
template <int FMT, int MINB, bool BLOCKS_ONLY = false, bool LEAN = false>
__global__ void __launch_bounds__(128, MINB) jpeg_fused_kernel(const uint8_t *__restrict__ src, long pitch, jpeg_geom g, uint8_t *__restrict__ slots,
                                                         uint32_t *__restrict__ sizes, uint32_t *__restrict__ local_off,
                                                         uint32_t *__restrict__ cta_total, bool vec_ok, int cap, uint32_t *__restrict__ stats,
                                                         jpeg_lookback lb, const __grid_constant__ jpeg_qtab qt, const uint32_t *__restrict__ huff,
                                                         uint32_t *__restrict__ gbits = nullptr, uint16_t *__restrict__ glen = nullptr,
                                                         int16_t *__restrict__ gcoef = nullptr)
{
        extern __shared__ __align__(128) uint32_t smem[];
        uint32_t *s_coef = smem;                // [32][128] zig-zag coefficients, two int16 per word
        uint32_t *s_bits = s_coef + 32 * 128;   // [cap][128]   (BLOCKS_ONLY: not allocated - the bit strings live in gbits)
        uint32_t *s_seg = s_bits + cap * 128;   // [segments of the CTA][bps * cap]
        __shared__ __align__(16) uint32_t s_huff[32 + 512];  // jpeg_hufftab as it lies in global memory: dc[2][16], ac[2][256]
        uint32_t(*const s_dctab)[16] = (uint32_t(*)[16]) s_huff;
        uint32_t(*const s_ac)[256] = (uint32_t(*)[256]) (s_huff + 32);
        __shared__ uint32_t s_len[128], s_warp[4], s_max[4];
        __shared__ int s_dc[128];
        __shared__ uint32_t s_ticket, s_tot, s_base;
        __shared__ __align__(8) unsigned long long s_bar;  // mbarrier of the input tile
        const int tid = threadIdx.x;
        asm volatile("griddepcontrol.launch_dependents;");  // the one-CTA offset scan behind this kernel may be set up now (it waits for this grid to finish)
        int cta_x = blockIdx.x, cta_y = blockIdx.y, ticket = 0;
        if (lb.state != nullptr) {
                if (tid == 0) {
                        s_ticket = atomicAdd(lb.ticket, 1u);
                }
                __syncthreads();
                ticket = (int) s_ticket;
                cta_x = FMT == FMT_UYVY_422 ? ticket : ticket % lb.ctas_per_scan, cta_y = FMT == FMT_UYVY_422 ? 0 : ticket / lb.ctas_per_scan;
        } else if (FMT == FMT_RGB_444) {
                // one-dimensional grid, component fastest: the three CTAs that read the same 24 KB of packed RGB run next to each other (L2 / L1 hits
                // instead of three passes over the frame)
                cta_x = blockIdx.x / 3, cta_y = blockIdx.x - 3 * cta_x;
        }
        // UYVY: the tile copy is issued before anything else - the copy engine moves the 8 KB while the CTA fetches its Huffman tables and works out its
        // block mapping (round 2, state i: the tables used to be fetched first and the copy waited behind their barrier: two global latencies in a row)
        bool early_tile = false;
        if (FMT == FMT_UYVY_422) {
                const int fm = cta_x * 32, mx0 = fm % g.bw, my0 = fm / g.bw;
                early_tile = LEAN || (vec_ok && cap >= 8 && mx0 + 32 <= g.bw && (mx0 + 32) * 16 <= g.w && (my0 + 1) * 8 <= g.h);
                if (early_tile && tid == 0) {
                        uint8_t *tile0 = (uint8_t *) (BLOCKS_ONLY ? s_coef : s_bits);
                        const uint8_t *gsrc = src + (long) (my0 * 8) * pitch + (long) mx0 * 32;
                        mbar_init(&s_bar, 1);
                        mbar_expect_tx(&s_bar, 8 * 1024 + (uint32_t) sizeof s_huff);
                        for (int r = 0; r < 8; ++r) {
                                bulk_g2s((void *) (tile0 + r * 1024), gsrc + (long) r * pitch, 1024, &s_bar);
                        }
                        bulk_g2s((void *) s_huff, huff, (uint32_t) sizeof s_huff, &s_bar);  // the Huffman tables ride the same barrier (cudaMalloc'ed: 256-byte aligned)
                }
        }
        if (FMT == FMT_RGB_444) {  // the same for the packed-RGB tile (8 rows x 3072 bytes, at most two runs per row) when whole runs can go through the copy engine
                const int fm = cta_x * 128;
                early_tile = LEAN || (vec_ok && cap >= 8 && fm + 128 <= g.mcu_per_scan && (g.w & 7) == 0 && (g.h & 7) == 0 && g.bw >= 128 && !(g.bw & 1) &&
                                      !(15 & (size_t) src) && !(pitch & 15));
                if (early_tile && tid == 0) {
                        uint8_t *tile0 = (uint8_t *) s_coef;
                        const int bx0 = fm % g.bw, by0 = fm / g.bw;
                        const int in_row = min(128, g.bw - bx0);  // blocks of the tile that lie in block row by0; the rest starts block row by0 + 1
                        mbar_init(&s_bar, 1);
                        mbar_expect_tx(&s_bar, 8 * 3072 + (uint32_t) sizeof s_huff);
                        const uint8_t *ga = src + (long) (by0 * 8) * pitch + (long) bx0 * 24, *gb = src + (long) (by0 * 8 + 8) * pitch;
                        for (int r = 0; r < 8; ++r, ga += pitch, gb += pitch) {
                                bulk_g2s((void *) (tile0 + r * 3072), ga, (uint32_t) in_row * 24, &s_bar);
                                if (in_row < 128) {
                                        bulk_g2s((void *) (tile0 + r * 3072 + in_row * 24), gb, (uint32_t) (128 - in_row) * 24, &s_bar);
                                }
                        }
                        bulk_g2s((void *) s_huff, huff, (uint32_t) sizeof s_huff, &s_bar);
                }
        }
        if (!early_tile) {
                for (int i = tid; i < 32 + 512; i += 128) {
                        s_huff[i] = __ldg(huff + i);
                }
        }
        // ---- which block is mine -------------------------------------------------------------------------------------------
        const int bps = g.ri * g.blocks_per_mcu;  // blocks per restart segment: 4, 8, 16 or 32 (checked by the host)
        int comp, bx, by, p;                      // p = position of my block in the CTA's scan order
        bool valid;
        int first_mcu;                            // scan-local index of the CTA's first MCU
        if (FMT == FMT_UYVY_422) {
                const int k = tid >> 5, lane = tid & 31;
                first_mcu = cta_x * 32;
                const int m = first_mcu + lane;
                valid = LEAN || m < g.mcu_per_scan;
                comp = k < 2 ? 0 : k - 1;
                const int mx = m % g.bw;
                bx = comp == 0 ? mx * 2 + k : mx, by = m / g.bw;
                p = lane * 4 + k;
        } else {
                first_mcu = cta_x * 128;
                const int b = first_mcu + tid;
                valid = LEAN || b < g.mcu_per_scan;
                comp = cta_y;
                bx = b % g.bw, by = b / g.bw;
                p = tid;
        }
        // ---- 0. stage the CTA's input tile (32 MCUs x 8 rows = 8 x 1024 bytes) through shared memory: coalesced, asynchronous, and the
        //         luma and chroma warps read every byte from there instead of fetching it twice.  The tile borrows s_bits and, for a cap below 16
        //         words, the start of s_seg behind it (both are free until phase 2; s_seg is cleared after the DCT).
        bool staged = false;
        const uint8_t *tile = FMT == FMT_UYVY_422 && !BLOCKS_ONLY ? (const uint8_t *) s_bits : (const uint8_t *) s_coef;
        if (FMT == FMT_RGB_444) {
                // The CTA's 128 blocks are consecutive in raster order of ONE component: 8 rows x 3072 bytes of packed RGB (the run may wrap into the
                // next block row; the tile keeps block order, not image order).  cp.async in 8-byte pieces - a block starts at a multiple of 24 bytes -
                // instead of 64 single-byte loads per thread.  24 KB: the tile lies over the coefficient array, the bit strings and the segment images,
                // all of which are written only after the last sample has been read (barrier below).
                staged = LEAN || (vec_ok && cap >= 8 && first_mcu + 128 <= g.mcu_per_scan && (g.w & 7) == 0 && (g.h & 7) == 0);
                // 16-byte aligned rows and an even number of blocks per row: the (at most two) runs of a tile row start and end on 48-byte
                // boundaries, so whole runs go through the copy engine
                // (a frame less than 128 blocks wide wraps more than once inside a tile: that goes the cp.async way below)
                const bool bulk = early_tile;  // issued at the top of the kernel
                if (bulk) {
                        __syncthreads();  // the mbarrier's initialisation (thread 0) is visible to the waiting threads
                        mbar_wait(&s_bar, 0);
                } else if (staged) {
#pragma unroll
                        for (int j = 0; j < 3; ++j) {
                                const int c = tid + 128 * j;            // 8-byte piece c of a 3072-byte tile row
                                const int blk = c / 3, part = c - 3 * blk;
                                const int b = first_mcu + blk;
                                const int bxx = b % g.bw, byy = b / g.bw;
                                const uint8_t *gp = src + (long) (byy * 8) * pitch + (long) bxx * 24 + part * 8;
                                uint32_t dst = (uint32_t) __cvta_generic_to_shared(tile + c * 8);
#pragma unroll
                                for (int r = 0; r < 8; ++r, gp += pitch, dst += 3072) {
                                        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(gp) : "memory");
                                }
                        }
                        asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
                        __syncthreads();
                }
        }
        if (FMT == FMT_UYVY_422) {
                const int mx0 = first_mcu % g.bw, my0 = first_mcu / g.bw;
                staged = early_tile;
                (void) mx0, (void) my0;
                if (staged) {  // vec_ok: 16-byte aligned frame and pitch - one bulk copy per 1024-byte tile row, issued at the top of the kernel
                        __syncthreads();  // the mbarrier's initialisation (thread 0) is visible to the waiting threads
                        mbar_wait(&s_bar, 0);
                }
        }
        // ---- 1. DCT + quantise, packed: lanes (x, y) of a float2 = rows (2r, 2r + 1) in the row pass, columns (2c, 2c + 1) in the column pass ----
        float2 g2[8][4];  // after the column pass: g2[r][cp] = coefficients (r, 2cp) and (r, 2cp + 1), still as 1.5 * 2^23 + q
        {
                const int px_w = (FMT == FMT_UYVY_422 && comp != 0) ? 16 : 8;
                const bool interior = LEAN || (vec_ok && valid && (bx + 1) * px_w <= g.w && (by + 1) * 8 <= g.h);
                float2 f2[4][8];
#pragma unroll
                for (int rp = 0; rp < 4; ++rp) {
                        float ma[8], mb[8];
                        if (FMT == FMT_RGB_444 && staged) {
                                load_row_rgb_tile(tile + (2 * rp) * 3072 + tid * 24, comp, ma);
                                load_row_rgb_tile(tile + (2 * rp + 1) * 3072 + tid * 24, comp, mb);
                        } else {
                                load_row_magic<LEAN>(src, pitch, g, comp, valid ? bx : 0, valid ? by * 8 + 2 * rp : 0, interior, ma,
                                                     staged ? tile + (2 * rp) * 1024 : nullptr, tid & 31);
                                load_row_magic<LEAN>(src, pitch, g, comp, valid ? bx : 0, valid ? by * 8 + 2 * rp + 1 : 0, interior, mb,
                                                     staged ? tile + (2 * rp + 1) * 1024 : nullptr, tid & 31);
                        }
#pragma unroll
                        for (int x = 0; x < 8; ++x) {  // (2^23 + s) - (2^23 + 128): level shift, exact
                                f2[rp][x] = __fadd2_rn(make_float2(ma[x], mb[x]), make_float2(-8388736.0f, -8388736.0f));
                        }
                        fdct8_2(f2[rp][0], f2[rp][1], f2[rp][2], f2[rp][3], f2[rp][4], f2[rp][5], f2[rp][6], f2[rp][7]);
                }
#pragma unroll
                for (int rp = 0; rp < 4; ++rp) {  // re-pair: rows apart, neighbouring columns together
#pragma unroll
                        for (int cp = 0; cp < 4; ++cp) {
                                g2[2 * rp][cp] = make_float2(f2[rp][2 * cp].x, f2[rp][2 * cp + 1].x);
                                g2[2 * rp + 1][cp] = make_float2(f2[rp][2 * cp].y, f2[rp][2 * cp + 1].y);
                        }
                }
                const float2 *qm = (const float2 *) qt.qmul[comp == 0 ? 0 : 1];
#pragma unroll
                for (int cp = 0; cp < 4; ++cp) {
                        fdct8_2(g2[0][cp], g2[1][cp], g2[2][cp], g2[3][cp], g2[4][cp], g2[5][cp], g2[6][cp], g2[7][cp]);
#pragma unroll
                        for (int r = 0; r < 8; ++r) {  // rint without F2I: low 16 bits of the result = the quantised value
                                g2[r][cp] = __ffma2_rn(g2[r][cp], qm[4 * r + cp], make_float2(12582912.0f, 12582912.0f));
                        }
                }
        }
        const int pc = blk_col(p);  // my block's column in the [k][128] arrays
        constexpr int zz[64] = { 0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };
        if ((FMT == FMT_RGB_444 || BLOCKS_ONLY) && staged) {
                __syncthreads();  // the tile lies over the coefficient array: every thread has its samples in registers before the first store
        }
        // word k of the block = zig-zag coefficients k (low half) and k + 32 (high half): the non-zero flags of 16 words then add up
        // into one register without touching each other (bit k and bit 16 + k), and two byte permutes assemble the 64-bit map
        uint32_t flags_a = 0, flags_b = 0;
        int dcv = 0;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
                const int na = zz[k], nb = zz[k + 32];
                const float2 pa = g2[na >> 3][(na & 7) >> 1], pb = g2[nb >> 3][(nb & 7) >> 1];
                const uint32_t ua = __float_as_uint((na & 1) ? pa.y : pa.x), ub = __float_as_uint((nb & 1) ? pb.y : pb.x);
                // No clamp to the 10-bit AC categories is needed: with samples in [-128, 127] the largest AC coefficient is F(4,4) (all |cos| =
                // 1/sqrt(2)) = 1/4 * 1/2 * 32 * (127 + 128) = 1020 before quantisation, as is F(4,0); every other one is below 930.  The oracle
                // keeps its clamp, which therefore never acts.  (DC: up to 1024 in magnitude, differences in category 11 of the DC table.)
                const uint32_t w = __byte_perm(ua, ub, 0x5410);
                s_coef[k * 128 + pc] = w;
                const uint32_t fl = __vminu2(w, 0x00010001u);
                if (k < 16) {
                        flags_a += fl << k;
                } else {
                        flags_b += fl << (k - 16);
                }
                if (k == 0) {
                        dcv = (int) (short) (w & 0xffffu);
                }
        }
        uint64_t nz = (uint64_t) __byte_perm(flags_a, flags_b, 0x5410) | (uint64_t) __byte_perm(flags_a, flags_b, 0x7632) << 32;
        nz &= ~1ull;
        s_dc[pc] = dcv;
        __syncthreads();
        if (!BLOCKS_ONLY) {
                for (int i = tid; i < cap * 128; i += 128) {  // the segment images start empty (the input tile, dead by now, may have reached into them)
                        s_seg[i] = 0;
                }
        }
        // linear index of this CTA (the order of cta_total / gbits / glen) and of my block in the frame's scan order
        const int cta_lin = FMT == FMT_UYVY_422 ? cta_x : cta_y * lb.ctas_per_scan + cta_x;
        // ---- 2. entropy-code my block --------------------------------------------------------------------------------------------
        uint32_t bits = 0;
        if (valid) {
                const int t = comp == 0 ? 0 : 1;
                int pred;
                if (FMT == FMT_UYVY_422) {  // MCU = Y0 Y1 Cb Cr; a segment starts every ri MCUs (ri divides the CTA's 32 MCUs)
                        const int k = tid >> 5;
                        const bool first = (p % bps) < 4;
                        pred = k == 1 ? s_dc[blk_col(p - 1)] : first ? 0 : k == 0 ? s_dc[blk_col(p - 3)] : s_dc[blk_col(p - 4)];
                } else {
                        pred = (p % bps) == 0 ? 0 : s_dc[blk_col(p - 1)];
                }
                block_bits bw = { (BLOCKS_ONLY ? gbits + (size_t) cta_lin * cap * 128 : s_bits) + pc, 0, 0, 0, cap };
                const int diff = dcv - pred;
                int sz = category(diff);
                bw.put(s_dctab[t][sz] & 0xffff, s_dctab[t][sz] >> 16);
                if (sz) {
                        bw.put((uint32_t) (diff < 0 ? diff - 1 : diff) & ((1u << sz) - 1u), sz);
                }
                // AC: one turn per non-zero coefficient.  The map is walked as two 32-bit halves: bit b of half h is zig-zag index b + 32 h,
                // stored in half h of word b
                int prev = 0;
                const uint32_t *cw = s_coef + pc;
                const uint32_t *act = s_ac[t];
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                        uint32_t m = half ? (uint32_t) (nz >> 32) : (uint32_t) nz;
                        while (m) {
                                const int b = __ffs((int) m) - 1;
                                m &= m - 1;
                                const int i = b + 32 * half;
                                int run = i - prev - 1;
                                prev = i;
                                while (run > 15) {
                                        bw.put(act[0xF0] & 0xffff, act[0xF0] >> 16);  // ZRL
                                        run -= 16;
                                }
                                const int v = half ? (int) cw[b * 128] >> 16 : (int) (short) (cw[b * 128] & 0xffffu);
                                sz = category(v);
                                const uint32_t e = act[(run << 4) | sz];
                                bw.put(((e & 0xffff) << sz) | ((uint32_t) (v < 0 ? v - 1 : v) & ((1u << sz) - 1u)), (int) (e >> 16) + sz);
                        }
                }
                if (prev != 63) {
                        bw.put(act[0] & 0xffff, act[0] >> 16);  // EOB
                }
                bits = bw.finish();
                if (BLOCKS_ONLY && bits > (uint32_t) cap * 32u) {
                        // longer than the cap: the assembly kernel codes this block again from its coefficients (natural order of the split path's
                        // coefficient buffer: 64 int16 per block in scan order); slot 0 carries the DC difference - the predictor is not known there
                        const long blk = FMT == FMT_UYVY_422 ? (long) first_mcu * 4 + p : (long) cta_y * g.mcu_per_scan + first_mcu + p;
                        uint32_t *dst = (uint32_t *) (gcoef + blk * 64);
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                                const uint32_t w0 = cw[(2 * j) * 128], w1 = cw[(2 * j + 1) * 128];
                                dst[j] = __byte_perm(w0, w1, 0x5410);       // coefficients 2j, 2j + 1
                                dst[16 + j] = __byte_perm(w0, w1, 0x7632);  // coefficients 32 + 2j, 33 + 2j
                        }
                        ((int16_t *) dst)[0] = (int16_t) diff;
                }
        }
        if (BLOCKS_ONLY) {
                glen[(size_t) cta_lin * 128 + pc] = (uint16_t) bits;
                uint32_t mx = bits;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) {
                        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
                }
                if ((tid & 31) == 0) {
                        atomicMax(stats, mx);
                        if (mx > (uint32_t) cap * 32u) {
                                atomicAdd(stats + 1, 1u);
                        }
                }
                return;
        }
        s_len[pc] = bits;
        const bool overflow = __syncthreads_or(bits > (uint32_t) cap * 32u) != 0;
        {  // largest block of the CTA (reported at the end: the host sizes the next frame's cap from the frame maximum)
                uint32_t mx = bits;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) {
                        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
                }
                if ((tid & 31) == 0) {
                        s_max[tid >> 5] = mx;
                }
        }
        const int sg = tid / bps, gl = tid % bps;          // segment within the CTA, my lane within the segment's group
        const unsigned lane32 = tid & 31;
        const int ls = first_mcu / g.ri + sg;              // index of the segment within its scan
        const int seg_global = FMT == FMT_UYVY_422 ? ls : cta_y * g.seg_per_scan + ls;
        const bool seg_valid = ls < g.seg_per_scan && (long) ls * g.ri < g.mcu_per_scan;
        uint32_t written = 0;
        const unsigned gmask = bps == 32 ? 0xffffffffu : (((1u << bps) - 1u) << (lane32 - gl));
        uint32_t T = 0;                                    // bits of my segment (fast route)
        uint32_t *seg = s_seg + sg * bps * cap;            // its assembled bit string
        if (overflow) {
                // ---- serial route: the segment's first thread codes all its blocks into the slot --------------------------------------
                if (gl == 0 && seg_valid) {
                        uint32_t *base = (uint32_t *) (slots + (long) seg_global * g.slot);
                        bit_writer bw = { base, 0, 0, 0, 0 };
                        int pred[3] = { 0, 0, 0 };
                        for (int q = tid; q < tid + bps; ++q) {
                                const int m = first_mcu + (FMT == FMT_UYVY_422 ? q >> 2 : q);
                                if (m >= g.mcu_per_scan) {
                                        break;
                                }
                                const int comp = FMT == FMT_UYVY_422 ? ((q & 3) < 2 ? 0 : (q & 3) - 1) : cta_y;
                                const int t = comp == 0 ? 0 : 1, qc = blk_col(q);
                                uint64_t map = 0;
                                for (int k = 0; k < 32; ++k) {
                                        const uint32_t w = s_coef[k * 128 + qc];
                                        map |= (uint64_t) ((w & 0xffffu) != 0) << k | (uint64_t) ((w >> 16) != 0) << (k + 32);
                                }
                                map &= ~1ull;
                                const int dc = s_dc[qc], diff = dc - pred[FMT == FMT_UYVY_422 ? comp : 0];
                                pred[FMT == FMT_UYVY_422 ? comp : 0] = dc;
                                int sz = category(diff);
                                bw.put(s_dctab[t][sz] & 0xffff, s_dctab[t][sz] >> 16);
                                if (sz) {
                                        bw.put((uint32_t) (diff < 0 ? diff - 1 : diff), sz);
                                }
                                int prev = 0;
                                while (map) {
                                        const int i = __ffsll((long long) map) - 1;
                                        map &= map - 1;
                                        int run = i - prev - 1;
                                        prev = i;
                                        while (run > 15) {
                                                bw.put(s_ac[t][0xF0] & 0xffff, s_ac[t][0xF0] >> 16);
                                                run -= 16;
                                        }
                                        const int v = (int) (short) (s_coef[(i & 31) * 128 + qc] >> (16 * (i >> 5)));
                                        sz = category(v);
                                        const uint32_t e = s_ac[t][(run << 4) | sz];
                                        bw.put(((e & 0xffff) << sz) | ((uint32_t) (v < 0 ? v - 1 : v) & ((1u << sz) - 1u)), (int) (e >> 16) + sz);
                                }
                                if (prev != 63) {
                                        bw.put(s_ac[t][0] & 0xffff, s_ac[t][0] >> 16);
                                }
                        }
                        bw.flush_bits();
                        if (ls != g.seg_per_scan - 1) {
                                bw.emit_byte(0xFF);
                                bw.emit_byte(0xD0 + (ls & 7));
                        }
                        written = bw.finish(base);
                        sizes[seg_global] = written;
                }
        } else {
                // ---- 3. assemble restart segments: thread tid now owns scan-order block tid ---------------------------------------------
                const int tc = blk_col(tid);
                const uint32_t L = s_len[tc];
                uint32_t incl = L;
                for (int d = 1; d < bps; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(gmask, incl, d, bps);
                        if (gl >= d) {
                                incl += o;
                        }
                }
                T = __shfl_sync(gmask, incl, bps - 1, bps);  // bits of the whole segment
                {
                        const uint32_t off = incl - L, sh = off & 31;
                        uint32_t *d = seg + (off >> 5);
                        for (uint32_t w = 0; w * 32 < L; ++w) {
                                const uint32_t v = s_bits[w * 128 + tc];
                                atomicOr(d + w, v >> sh);
                                if (sh && (v << (32 - sh))) {
                                        atomicOr(d + w + 1, v << (32 - sh));
                                }
                        }
                        if (gl == 0 && (T & 7)) {  // pad the last byte with ones (T.81 F.1.2.3)
                                const uint32_t pad = 8 - (T & 7);
                                atomicOr(seg + (T >> 5), ((1u << pad) - 1u) << (32 - (T & 31) - pad));
                        }
                }
                __syncthreads();
                // ---- 4. byte stuffing into the slot - or, with the single-pass compaction, only the SIZE of the stuffed segment for now -------
                if (seg_valid && lb.state != nullptr) {
                        const uint32_t n = (T + 7) >> 3;
                        uint32_t cnt = 0;
                        for (uint32_t wi = gl; wi * 4 < n; wi += bps) {  // bytes beyond n are zero: whole words can be tested
                                cnt += __popc(__vcmpeq4(seg[wi], 0xFFFFFFFFu)) >> 3;
                        }
                        for (int d = bps >> 1; d > 0; d >>= 1) {
                                cnt += __shfl_xor_sync(gmask, cnt, d, bps);
                        }
                        written = n + cnt + (ls != g.seg_per_scan - 1 ? 2u : 0u);
                } else if (seg_valid) {
                        const int rst = ls != g.seg_per_scan - 1 ? 0xD0 + (ls & 7) : -1;
                        uint8_t *slot = slots + (long) seg_global * g.slot;
                        // staging area of this segment: its share of the per-block bit strings, which nobody reads any more (barrier above)
                        written = stuff_segment_words(slot, (uint8_t *) s_bits + (size_t) sg * bps * cap * 4, (uint32_t) (bps * cap * 4), seg, T, bps, gl, gmask, rst);
                        if (written == 0xFFFFFFFFu) {  // more 0xFF bytes than the staging area has room for: byte-wise, straight to the slot
                                written = stuff_segment(slot, seg, T, bps, gl, lane32, gmask, rst);
                        }
                        if (gl == 0) {
                                sizes[seg_global] = written;
                        }
                }
        }
        // ---- 5. CTA prefix of the segment sizes ----------------------------------------------------------------------------------------
        const uint32_t mine = (gl == 0 && seg_valid) ? (written) : 0;  // one value per segment, carried by its first thread
        uint32_t inc2 = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, inc2, d);
                if (lane32 >= (unsigned) d) {
                        inc2 += o;
                }
        }
        if (lane32 == 31) {
                s_warp[tid >> 5] = inc2;
        }
        __syncthreads();
        uint32_t before = 0;
        for (int w = 0; w < (tid >> 5); ++w) {
                before += s_warp[w];
        }
        if (tid == 127) {
                atomicMax(stats, max(max(s_max[0], s_max[1]), max(s_max[2], s_max[3])));
                if (overflow) {
                        atomicAdd(stats + 1, 1u);
                }
        }
        if (lb.state == nullptr) {  // two-level scan + compaction kernels follow
                if (gl == 0 && seg_valid) {
                        local_off[seg_global] = before + inc2 - mine;
                }
                if (tid == 127) {
                        const int cta = FMT == FMT_UYVY_422 ? cta_x : cta_y * lb.ctas_per_scan + cta_x;
                        cta_total[cta] = before + inc2;
                }
                return;
        }
        // ---- 6. single-pass compaction: my CTA's offset in the stream by decoupled look-back, then the segments go to their final place -------
        if (tid == 127) {
                s_tot = before + inc2;
        }
        __syncthreads();
        if (tid < 32) {  // warp 0 looks back 32 predecessors at a time
                constexpr unsigned long long kAgg = 1ull << 62, kPfx = 2ull << 62, kMask = (1ull << 62) - 1;
                unsigned long long base = 0;
                if (ticket > 0) {
                        if (tid == 0) {
                                atomicExch(lb.state + ticket, kAgg | s_tot);
                        }
                        for (int j = ticket - 1;;) {
                                const int idx = j - tid;
                                const unsigned long long v = idx >= 0 ? *(volatile unsigned long long *) (lb.state + idx) : kPfx;  // nothing before CTA 0
                                const unsigned flag = (unsigned) (v >> 62);
                                const unsigned pfx = __ballot_sync(0xffffffffu, flag == 2), inv = __ballot_sync(0xffffffffu, flag == 0);
                                const int first = pfx ? __ffs((int) pfx) - 1 : 31;           // nearest predecessor that knows its prefix
                                const unsigned window = first == 31 ? 0xffffffffu : (2u << first) - 1u;
                                if (inv & window) {
                                        continue;  // one of them has not published yet (it has started: tickets are handed out in order)
                                }
                                unsigned long long part = (window >> tid) & 1u ? v & kMask : 0ull;
#pragma unroll
                                for (int d = 16; d > 0; d >>= 1) {
                                        part += __shfl_xor_sync(0xffffffffu, part, d);
                                }
                                base += part;
                                if (pfx) {
                                        break;
                                }
                                j -= 32;
                        }
                }
                if (tid == 0) {
                        atomicExch(lb.state + ticket, kPfx | (base + s_tot));
                        s_base = (uint32_t) base;
                }
        }
        __syncthreads();
        const uint32_t seg_off = __shfl_sync(gmask, before + inc2 - mine, 0, bps), seg_size = __shfl_sync(gmask, written, 0, bps);
        const unsigned long long pos0 = (unsigned long long) g.header_len + (unsigned long long) g.sos_len * cta_y + s_base;
        if (seg_valid && pos0 + seg_off + seg_size <= lb.out_cap) {  // a stream larger than the buffer is reported by the host, never written
                uint8_t *dstp = lb.out + pos0 + seg_off;
                if (overflow) {  // the serial route left the finished segment in its slot
                        const uint8_t *slot = slots + (long) seg_global * g.slot;
                        for (uint32_t i = gl; i < seg_size; i += bps) {
                                dstp[i] = slot[i];
                        }
                } else {
                        stuff_segment(dstp, seg, T, bps, gl, lane32, gmask, ls != g.seg_per_scan - 1 ? 0xD0 + (ls & 7) : -1);
                }
        }
        if (tid == 0) {
                if (FMT == FMT_RGB_444 && cta_x == 0 && cta_y > 0 && pos0 <= lb.out_cap) {  // SOS header of a later scan, right in front of its data
                        uint8_t *h = lb.out + pos0 - g.sos_len;
                        const uint8_t sos[10] = { 0xFF, 0xDA, 0, 8, 1, (uint8_t) (cta_y + 1), 0x11, 0, 63, 0 };
                        for (int i = 0; i < 10; ++i) {
                                h[i] = sos[i];
                        }
                }
                if (ticket == (int) gridDim.x - 1) {  // the last CTA of the stream: EOI and the total
                        const unsigned long long end = pos0 + s_tot;
                        if (end + 2 <= lb.out_cap) {
                                lb.out[end] = 0xFF, lb.out[end + 1] = 0xD9;
                        }
                        *lb.total = (uint32_t) (end + 2);
                }
        }
}

// ---- restart-segment assembly of the two-kernel form --------------------------------------------------------------------------------------------
/// Second kernel behind jpeg_fused_kernel<.., BLOCKS_ONLY>: thread t of a CTA owns scan-order block t of the CTA's 128 (same CTA numbering), the
/// threads of a restart segment sit in one warp.  Phases 3-5 of the one-kernel form: prefix of the bit lengths, the bit strings ORed into the
/// segment image, byte stuffing, slot + size, CTA prefix of the sizes - with warp-level synchronisation only (a segment never leaves its warp), 12 KB
/// of shared memory at the default cap and ~40 registers, i.e. at full occupancy.  A segment with a block beyond the cap is coded by its first
/// thread alone: stored bit strings are appended as they are, the long block is coded again from its coefficients in `gcoef`.
template <int FMT>
__global__ void __launch_bounds__(128) jpeg_assemble_kernel(jpeg_geom g, const uint32_t *__restrict__ gbits, const uint16_t *__restrict__ glen,
                                                            const int16_t *__restrict__ gcoef, uint8_t *__restrict__ slots, uint32_t *__restrict__ sizes,
                                                            uint32_t *__restrict__ local_off, uint32_t *__restrict__ cta_total, int cap, int ctas_per_scan,
                                                            const uint32_t *__restrict__ huff)
{
        extern __shared__ __align__(128) uint32_t smem[];
        uint32_t *s_seg = smem;                 // [segments of the CTA][bps * cap]
        uint32_t *s_stage = smem + cap * 128;   // stuffing area, same partition
        __shared__ uint32_t s_warp[4];
        const int tid = threadIdx.x;
        asm volatile("griddepcontrol.launch_dependents;");
        const int cta_x = FMT == FMT_UYVY_422 ? blockIdx.x : blockIdx.x % ctas_per_scan, cta_y = FMT == FMT_UYVY_422 ? 0 : blockIdx.x / ctas_per_scan;
        const int cta_lin = blockIdx.x;  // = cta_y * ctas_per_scan + cta_x
        const int bps = g.ri * g.blocks_per_mcu;
        const int first_mcu = cta_x * (FMT == FMT_UYVY_422 ? 32 : 128);
        for (int i = tid & 31; i < 32 * cap; i += 32) {  // every warp clears the images of its own segments
                s_seg[(tid >> 5) * 32 * cap + i] = 0;
        }
        __syncwarp();
        asm volatile("griddepcontrol.wait;" ::: "memory");  // bit strings and lengths of the kernel in front (programmatic dependent launch)
        const int sg = tid / bps, gl = tid % bps;
        const unsigned lane32 = tid & 31;
        const int ls = first_mcu / g.ri + sg;
        const int seg_global = FMT == FMT_UYVY_422 ? ls : cta_y * g.seg_per_scan + ls;
        const bool seg_valid = ls < g.seg_per_scan && (long) ls * g.ri < g.mcu_per_scan;
        const unsigned gmask = bps == 32 ? 0xffffffffu : (((1u << bps) - 1u) << (lane32 - gl));
        const int tc = blk_col(tid);
        const uint32_t L = glen[(size_t) cta_lin * 128 + tc];
        const uint32_t *myb = gbits + (size_t) cta_lin * cap * 128 + tc;
        const bool seg_over = (__ballot_sync(0xffffffffu, L > (uint32_t) cap * 32u) & gmask) != 0;
        uint32_t written = 0;
        if (seg_over) {
                if (gl == 0 && seg_valid) {  // serial: the segment's first thread appends the 16 strings one after the other
                        uint32_t *base = (uint32_t *) (slots + (long) seg_global * g.slot);
                        bit_writer bw = { base, 0, 0, 0, 0 };
                        for (int q = tid; q < tid + bps; ++q) {
                                const int m = first_mcu + (FMT == FMT_UYVY_422 ? q >> 2 : q);
                                if (m >= g.mcu_per_scan) {
                                        break;
                                }
                                const int qc = blk_col(q);
                                const uint32_t Lq = glen[(size_t) cta_lin * 128 + qc];
                                if (Lq <= (uint32_t) cap * 32u) {
                                        const uint32_t *qb = gbits + (size_t) cta_lin * cap * 128 + qc;
                                        for (uint32_t w = 0; w * 32 < Lq; ++w) {
                                                const uint32_t v = qb[w * 128];
                                                const int n = (int) min(32u, Lq - w * 32), first = min(n, 16);  // the top n bits of v, MSB first
                                                bw.put(v >> (32 - first), first);
                                                if (n > 16) {
                                                        bw.put(v >> (32 - n), n - 16);  // put() keeps the low n - 16 bits
                                                }
                                        }
                                        continue;
                                }
                                // the block's own coefficients (natural order; slot 0 = DC difference)
                                const int comp = FMT == FMT_UYVY_422 ? ((q & 3) < 2 ? 0 : (q & 3) - 1) : cta_y;
                                const int t = comp == 0 ? 0 : 1;
                                const long blk = FMT == FMT_UYVY_422 ? (long) first_mcu * 4 + q : (long) cta_y * g.mcu_per_scan + first_mcu + q;
                                const int16_t *zz = gcoef + blk * 64;
                                const uint32_t *dct = huff + 16 * t, *act = huff + 32 + 256 * t;
                                const int diff = zz[0];
                                int sz = category(diff);
                                bw.put(dct[sz] & 0xffff, dct[sz] >> 16);
                                if (sz) {
                                        bw.put((uint32_t) (diff < 0 ? diff - 1 : diff), sz);
                                }
                                int prev = 0;
                                for (int i = 1; i < 64; ++i) {
                                        const int v = zz[i];
                                        if (v == 0) {
                                                continue;
                                        }
                                        int run = i - prev - 1;
                                        prev = i;
                                        while (run > 15) {
                                                bw.put(act[0xF0] & 0xffff, act[0xF0] >> 16);
                                                run -= 16;
                                        }
                                        sz = category(v);
                                        const uint32_t e = act[(run << 4) | sz];
                                        bw.put(((e & 0xffff) << sz) | ((uint32_t) (v < 0 ? v - 1 : v) & ((1u << sz) - 1u)), (int) (e >> 16) + sz);
                                }
                                if (prev != 63) {
                                        bw.put(act[0] & 0xffff, act[0] >> 16);
                                }
                        }
                        bw.flush_bits();
                        if (ls != g.seg_per_scan - 1) {
                                bw.emit_byte(0xFF);
                                bw.emit_byte(0xD0 + (ls & 7));
                        }
                        written = bw.finish(base);
                        sizes[seg_global] = written;
                }
        } else {
                uint32_t incl = L;
                for (int d = 1; d < bps; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(gmask, incl, d, bps);
                        if (gl >= d) {
                                incl += o;
                        }
                }
                const uint32_t T = __shfl_sync(gmask, incl, bps - 1, bps);
                uint32_t *seg = s_seg + sg * bps * cap;
                {
                        const uint32_t off = incl - L, sh = off & 31;
                        uint32_t *d = seg + (off >> 5);
                        for (uint32_t w = 0; w * 32 < L; ++w) {
                                const uint32_t v = myb[w * 128];
                                atomicOr(d + w, v >> sh);
                                if (sh && (v << (32 - sh))) {
                                        atomicOr(d + w + 1, v << (32 - sh));
                                }
                        }
                        if (gl == 0 && (T & 7)) {  // pad the last byte with ones (T.81 F.1.2.3)
                                const uint32_t pad = 8 - (T & 7);
                                atomicOr(seg + (T >> 5), ((1u << pad) - 1u) << (32 - (T & 31) - pad));
                        }
                }
                __syncwarp(gmask);
                if (seg_valid) {
                        const int rst = ls != g.seg_per_scan - 1 ? 0xD0 + (ls & 7) : -1;
                        uint8_t *slot = slots + (long) seg_global * g.slot;
                        written = stuff_segment_words(slot, (uint8_t *) s_stage + (size_t) sg * bps * cap * 4, (uint32_t) (bps * cap * 4), seg, T, bps, gl, gmask, rst);
                        if (written == 0xFFFFFFFFu) {
                                written = stuff_segment(slot, seg, T, bps, gl, lane32, gmask, rst);
                        }
                        if (gl == 0) {
                                sizes[seg_global] = written;
                        }
                }
        }
        // CTA prefix of the segment sizes (first level of the stream-offset scan, as in the one-kernel form)
        const uint32_t mine = (gl == 0 && seg_valid) ? written : 0;
        uint32_t inc2 = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, inc2, d);
                if (lane32 >= (unsigned) d) {
                        inc2 += o;
                }
        }
        if (lane32 == 31) {
                s_warp[tid >> 5] = inc2;
        }
        __syncthreads();
        uint32_t before = 0;
        for (int w = 0; w < (tid >> 5); ++w) {
                before += s_warp[w];
        }
        if (gl == 0 && seg_valid) {
                local_off[seg_global] = before + inc2 - mine;
        }
        if (tid == 127) {
                cta_total[cta_lin] = before + inc2;
        }
}

// ---- K2 -------------------------------------------------------------------------------------------------------------
/// One thread per restart segment.  Per block: 8 x LDG.128 build a 64-bit non-zero map (uniform work), then the loop runs once
/// per NON-ZERO coefficient (ffs over the map) instead of once per coefficient — far less divergence inside a warp.
/// The CTA also produces the exclusive prefix of its 128 segment sizes and its total (first level of the stream scan).
/// PLANAR: FMT_PLANAR geometry (scans of different lengths; luma blocks per MCU from the sampling factors)
template <bool PLANAR>
__global__ void __launch_bounds__(128) jpeg_huffman_kernel(const int16_t *__restrict__ coef, jpeg_geom g, uint8_t *__restrict__ slots,
                                                           uint32_t *__restrict__ sizes, uint32_t *__restrict__ local_off,
                                                           uint32_t *__restrict__ cta_total, const uint32_t *__restrict__ huff,
                                                           const __grid_constant__ jpeg_layout L)
{
        __shared__ uint32_t s_dc[2][16], s_ac[2][256], s_warp[4];
        for (int i = threadIdx.x; i < 32; i += blockDim.x) {
                s_dc[i >> 4][i & 15] = __ldg(huff + i);
        }
        for (int i = threadIdx.x; i < 512; i += blockDim.x) {
                s_ac[i >> 8][i & 255] = __ldg(huff + 32 + i);
        }
        __syncthreads();
        const int s = blockIdx.x * blockDim.x + threadIdx.x;
        uint32_t nbytes = 0;
        if (s < g.nseg) {
                int scan, ls, segs, mcus;
                if (PLANAR) {
                        scan = (s >= L.scan_seg0[1]) + (s >= L.scan_seg0[2]);
                        const int s0 = scan == 0 ? 0 : scan == 1 ? L.scan_seg0[1] : L.scan_seg0[2];
                        ls = s - s0;
                        segs = (scan == 0 ? L.scan_seg0[1] : scan == 1 ? L.scan_seg0[2] : L.scan_seg0[3]) - s0;
                        mcus = scan == 0 ? L.scan_mcus[0] : scan == 1 ? L.scan_mcus[1] : L.scan_mcus[2];
                } else {
                        scan = s / g.seg_per_scan, ls = s - scan * g.seg_per_scan;
                        segs = g.seg_per_scan, mcus = g.mcu_per_scan;
                }
                const int m0 = ls * g.ri, m1 = min(m0 + g.ri, mcus);
                uint32_t *base = (uint32_t *) (slots + (long) s * g.slot);
                bit_writer bw = { base, 0, 0, 0, 0 };
                int pred[3] = { 0, 0, 0 };
                for (int m = m0; m < m1; ++m) {
                        for (int k = 0; k < g.blocks_per_mcu; ++k) {
                                int comp;
                                long blk;
                                if (PLANAR) {
                                        const int nl = g.blocks_per_mcu - 2;
                                        comp = !g.interleaved ? scan : k < nl ? 0 : k - nl + 1;
                                        blk = !g.interleaved ? (long) (scan == 0 ? 0 : scan == 1 ? L.comp_blk0[1] : L.comp_blk0[2]) + m
                                                             : (long) m * g.blocks_per_mcu + k;
                                } else if (g.fmt == FMT_UYVY_422) {
                                        comp = k < 2 ? 0 : k - 1;
                                        blk = (long) m * 4 + k;
                                } else if (g.interleaved) {
                                        comp = k;
                                        blk = (long) m * 3 + k;
                                } else {
                                        comp = scan;
                                        blk = (long) scan * g.mcu_per_scan + m;
                                }
                                const int t = comp == 0 ? 0 : 1;
                                const int16_t *zz = coef + blk * 64;
                                // non-zero map of the block
                                uint64_t nz = 0;
                                int dcv = 0;
#pragma unroll
                                for (int q = 0; q < 8; ++q) {
                                        const uint4 v = __ldg((const uint4 *) zz + q);
                                        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
                                        if (q == 0) {
                                                dcv = (int) (short) (v.x & 0xffff);
                                        }
#pragma unroll
                                        for (int j = 0; j < 4; ++j) {
                                                const uint64_t lo = (w[j] & 0xffffu) != 0, hi = (w[j] >> 16) != 0;
                                                nz |= (lo | hi << 1) << (8 * q + 2 * j);
                                        }
                                }
                                nz &= ~1ull;
                                // DC difference (T.81 F.1.2.1)
                                const int diff = dcv - pred[comp];
                                pred[comp] = dcv;
                                int sz = category(diff);
                                bw.put(s_dc[t][sz] & 0xffff, s_dc[t][sz] >> 16);
                                if (sz) {
                                        bw.put((uint32_t) (diff < 0 ? diff - 1 : diff), sz);
                                }
                                // AC run-lengths (F.1.2.2): one turn per non-zero coefficient
                                int prev = 0;
                                while (nz) {
                                        const int i = __ffsll((long long) nz) - 1;
                                        nz &= nz - 1;
                                        int run = i - prev - 1;
                                        prev = i;
                                        while (run > 15) {
                                                bw.put(s_ac[t][0xF0] & 0xffff, s_ac[t][0xF0] >> 16);  // ZRL
                                                run -= 16;
                                        }
                                        const int v = zz[i];  // L1 hit: the line was just read for the map
                                        sz = category(v);
                                        const uint32_t e = s_ac[t][(run << 4) | sz];
                                        // code and value bits in one put (<= 16 + 10 bits)
                                        bw.put(((e & 0xffff) << sz) | ((uint32_t) (v < 0 ? v - 1 : v) & ((1u << sz) - 1u)), (int) (e >> 16) + sz);
                                }
                                if (prev != 63) {
                                        bw.put(s_ac[t][0] & 0xffff, s_ac[t][0] >> 16);  // EOB
                                }
                        }
                }
                bw.flush_bits();
                if (ls != segs - 1) {  // RSTn between segments of a scan
                        bw.emit_byte(0xFF);
                        bw.emit_byte(0xD0 + (ls & 7));
                }
                nbytes = bw.finish(base);
                sizes[s] = nbytes;
        }
        // exclusive prefix of the CTA's 128 sizes
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t incl = nbytes;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) {
                        incl += o;
                }
        }
        if (lane == 31) {
                s_warp[warp] = incl;
        }
        __syncthreads();
        uint32_t before = 0;
        for (int w = 0; w < warp; ++w) {
                before += s_warp[w];
        }
        if (s < g.nseg) {
                local_off[s] = before + incl - nbytes;
        }
        if (threadIdx.x == blockDim.x - 1) {
                cta_total[blockIdx.x] = before + incl;
        }
}

// ---- K3: exclusive scan of the per-CTA totals (second level; a frame has 8 100 - 36 450 of them) ------------------------------------
// One CTA of 1024 threads, eight consecutive totals per thread and round (two 128-bit loads, thread-local prefix, one block scan of the
// thread sums): an 8K UYVY frame is ONE round.
__global__ void __launch_bounds__(1024) jpeg_scan_kernel(uint32_t *__restrict__ cta_total, int n, jpeg_geom g, uint32_t *__restrict__ total, int nscans)
{
        __shared__ uint32_t s_warp[32];
        __shared__ uint32_t s_carry;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t carry = 0;
        // programmatic dependent launch: this CTA may have been set up while the entropy kernel was still running; its totals are complete (and
        // visible) behind the wait.  The compaction kernel may be set up in turn.
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;");
        for (int base = 0; base < n; base += 8192) {  // the buffer is padded to a multiple of 8 entries (configure)
                const int i = base + threadIdx.x * 8;
                uint4 a = make_uint4(0, 0, 0, 0), b = a;
                if (i < n) {
                        a = *(const uint4 *) (cta_total + i), b = *(const uint4 *) (cta_total + i + 4);
                }
                uint32_t v[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
                uint32_t sum = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                        const uint32_t x = i + k < n ? v[k] : 0u;
                        v[k] = sum;  // exclusive within the thread
                        sum += x;
                }
                uint32_t incl = sum;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                        if (lane >= d) {
                                incl += o;
                        }
                }
                if (lane == 31) {
                        s_warp[warp] = incl;
                }
                __syncthreads();
                if (warp == 0) {
                        uint32_t w = s_warp[lane];
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                                const uint32_t o = __shfl_up_sync(0xffffffffu, w, d);
                                if (lane >= d) {
                                        w += o;
                                }
                        }
                        s_warp[lane] = w;  // inclusive over warps
                        if (lane == 31) {
                                s_carry = w;
                        }
                }
                __syncthreads();
                const uint32_t before = carry + (warp ? s_warp[warp - 1] : 0) + incl - sum;
                if (i < n) {  // exclusive prefixes in place (entries beyond n are padding)
                        *(uint4 *) (cta_total + i) = make_uint4(before + v[0], before + v[1], before + v[2], before + v[3]);
                        *(uint4 *) (cta_total + i + 4) = make_uint4(before + v[4], before + v[5], before + v[6], before + v[7]);
                }
                carry += s_carry;
                __syncthreads();
        }
        if (threadIdx.x == 0) {
                *total = g.header_len + carry + g.sos_len * (nscans - 1) + 2;  // + later SOS headers + EOI
        }
}

// ---- K4 -------------------------------------------------------------------------------------------------------------
// Eight lanes per segment (a typical segment is ~100 bytes); the per-segment routine, aligned 32-bit stores through a funnel shift, is
// compact_segment() in jpeg_compact.cuh, chosen over a warp per segment moving bytes with tools/exp_compact.cu on an earlier GPU
// (not re-measured on the H100); the same routine is checked on the CPU against memcpy (tests/test_device_identities.py).
constexpr int kCompactLanes = 8;

__global__ void __launch_bounds__(256) jpeg_compact_kernel(const uint8_t *__restrict__ slots, const uint32_t *__restrict__ sizes,
                                                           const uint32_t *__restrict__ local_off, const uint32_t *__restrict__ cta_base,
                                                           jpeg_geom g, int segs_per_cta, int ctas_per_scan, uint8_t *__restrict__ out,
                                                           const uint32_t *__restrict__ total, uint32_t out_cap, const __grid_constant__ jpeg_layout L)
{
        const int t = blockIdx.x * blockDim.x + threadIdx.x;
        const int s = t / kCompactLanes, lane = t % kCompactLanes;
        asm volatile("griddepcontrol.wait;" ::: "memory");  // offsets of the scan kernel (programmatic dependent launch)
        if (s >= g.nseg || *total > out_cap) {  // a stream larger than the output buffer is reported by the host, never written
                return;
        }
        const int scan = (s >= L.scan_seg0[1]) + (s >= L.scan_seg0[2]);  // scans may differ in length (4:2:0: the Y scan has 4x the blocks)
        const int seg0 = scan == 0 ? 0 : scan == 1 ? L.scan_seg0[1] : L.scan_seg0[2];
        // which CTA of the entropy kernel produced this segment: split path = 128 consecutive segments; fused path = per scan
        const int cta = ctas_per_scan ? scan * ctas_per_scan + (s - seg0) / segs_per_cta : s / segs_per_cta;
        const uint32_t n = sizes[s], off = g.header_len + cta_base[cta] + local_off[s] + g.sos_len * scan;
        compact_segment(lane, kCompactLanes, (const uint32_t *) (slots + (long) s * g.slot), n, out + off);  // g.slot is a multiple of 8
        if (lane == 0 && s > 0 && s == seg0) {  // SOS header of a later scan (one component per scan)
                uint8_t *h = out + off - g.sos_len;
                const uint8_t sos[10] = { 0xFF, 0xDA, 0, 8, 1, (uint8_t) (scan + 1), 0x11, 0, 63, 0 };
                for (int i = 0; i < 10; ++i) {
                        h[i] = sos[i];
                }
        }
        if (lane == 0 && s == g.nseg - 1) {
                out[off + n] = 0xFF, out[off + n + 1] = 0xD9;  // EOI
        }
}

// ---- pre-processing of the planar path: packed input -> the encoder's planes -------------------------------------------------
// Integer arithmetic only, restated by the test oracle byte for byte:
//   RGB:  Y = ((y_r R + y_g G + y_b B) >> 14) + off_y, Cb / Cr = (... >> 14) + 128 - the RGB_TO_* expressions of the reference's
//         rgb_to_yuv444p (to_lavc_vid_conv.c:1206-1214) at 8 bits; >> is a floor division.  Every result lies in 0..255 for the three
//         coefficient sets used (checked over the whole RGB cube by the tests), so nothing is clamped.  Subsampled chroma is the
//         rounded mean of the full-resolution values: (a + b + 1) >> 1 of a pair (4:2:2), (a + b + c + d + 2) >> 2 of a quad (4:2:0);
//         a missing last column or row takes its neighbour's value.
//   UYVY -> 4:2:0: uyvy_to_i420 (to_planar.c:343-378): Cb / Cr = (a + b + 1) / 2 of two rows, the last row paired with itself.
// what jpeg_prep_kernel does: nothing (I420 planes are read in place), UYVY -> 4:2:0, or RGB -> YCbCr with the coefficients of
// PREP_RGB + UGB200_JPEG_CS_{Y601,Y601FULL,Y709}
enum { PREP_NONE = 0, PREP_UYVY = 1, PREP_RGB = 2 };
struct jpeg_prep_args {
        const uint8_t *src;
        long pitch;
        int w, h;
        int rgb;       // 1 packed RGB, 0 UYVY (4:2:0 only)
        int hs, vs;    // luma samples per chroma sample
        int c[9];      // y_r y_g y_b cb_r cb_g cb_b cr_r cr_g cr_b (Q14)
        int off_y;
        int cw, ch;    // chroma plane size
        uint8_t *p[3];
        long pp[3];
};

__global__ void __launch_bounds__(256) jpeg_prep_kernel(const __grid_constant__ jpeg_prep_args a)
{
        const long i = (long) blockIdx.x * blockDim.x + threadIdx.x;  // one thread per chroma sample
        if (i >= (long) a.cw * a.ch) {
                return;
        }
        const int cx = (int) (i % a.cw), cy = (int) (i / a.cw);
        if (!a.rgb) {
                const int y0 = 2 * cy, y1 = min(y0 + 1, a.h - 1), x0 = 2 * cx;
                const uint8_t *r0 = a.src + (long) y0 * a.pitch + 4 * cx, *r1 = a.src + (long) y1 * a.pitch + 4 * cx;
                const uchar4 u = make_uchar4(r0[0], r0[1], r0[2], r0[3]), v = make_uchar4(r1[0], r1[1], r1[2], r1[3]);  // any pitch
                a.p[1][(long) cy * a.pp[1] + cx] = (uint8_t) ((u.x + v.x + 1) / 2);
                a.p[2][(long) cy * a.pp[2] + cx] = (uint8_t) ((u.z + v.z + 1) / 2);
                uint8_t *o0 = a.p[0] + (long) y0 * a.pp[0] + x0, *o1 = a.p[0] + (long) y1 * a.pp[0] + x0;
                o0[0] = u.y, o1[0] = v.y;
                if (x0 + 1 < a.w) {
                        o0[1] = u.w, o1[1] = v.w;
                }
                return;
        }
        int sb = 0, sr = 0;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                        if (j < a.vs && k < a.hs) {
                                const int x = cx * a.hs + k, y = cy * a.vs + j;
                                const uint8_t *px = a.src + (long) min(y, a.h - 1) * a.pitch + 3 * (long) min(x, a.w - 1);
                                const int R = px[0], G = px[1], B = px[2];
                                if (x < a.w && y < a.h) {
                                        a.p[0][(long) y * a.pp[0] + x] = (uint8_t) (((a.c[0] * R + a.c[1] * G + a.c[2] * B) >> 14) + a.off_y);
                                }
                                sb += ((a.c[3] * R + a.c[4] * G + a.c[5] * B) >> 14) + 128;
                                sr += ((a.c[6] * R + a.c[7] * G + a.c[8] * B) >> 14) + 128;
                        }
                }
        }
        const int n = a.hs * a.vs, sh = n == 1 ? 0 : n == 2 ? 1 : 2;  // n = 1, 2 or 4
        a.p[1][(long) cy * a.pp[1] + cx] = (uint8_t) ((sb + (n >> 1)) >> sh);
        a.p[2][(long) cy * a.pp[2] + cx] = (uint8_t) ((sr + (n >> 1)) >> sh);
}

}  // namespace ugb

// =====================================================================================================================
// host side
// =====================================================================================================================
using namespace ugb;

struct ugb200_jpeg_encoder {
        cudaStream_t stream = nullptr;
        // cached configuration
        int fmt = -1, w = 0, h = 0, quality = -1, ri = -1, interleaved = -1, hs = 0, vs = 0, prep = -1;
        jpeg_geom g{};
        jpeg_layout lay{};
        uint8_t *planes = nullptr;  // FMT_PLANAR from packed input: jpeg_prep_kernel's output
        size_t planes_cap = 0;
        std::vector<uint8_t> header;
        // device buffers
        int16_t *coef = nullptr;
        uint8_t *slots = nullptr, *out = nullptr, *staging = nullptr;
        uint32_t *sizes = nullptr, *offsets = nullptr, *cta_total = nullptr, *total = nullptr;
        jpeg_qtab qt{};                  // quantiser multipliers of the current quality (kernel parameter)
        uint32_t *d_huff = nullptr;      // jpeg_hufftab on the device
        unsigned long long *lb_state = nullptr;  // look-back state of the single-pass compaction ([0] = ticket counter)
        size_t lb_cap = 0;
        uint32_t *gbits = nullptr;               // two-kernel form: bit strings [CTA][cap][128] and lengths [CTA][128] of all blocks
        uint16_t *glen = nullptr;
        size_t gbits_cap = 0, glen_cap = 0;
        size_t coef_cap = 0, slots_cap = 0, out_cap = 0, seg_cap = 0, staging_cap = 0, cta_cap = 0;
        // pinned host buffers
        uint8_t *h_out = nullptr, *h_in = nullptr;
        uint32_t *h_total = nullptr;  // [0] stream bytes, [1] largest block (bits) if above half the cap, [2] CTAs on the serial route
        int cap_words = kCapDefault;  // shared-memory words per block of the fused kernel (adapted from the previous frame)
        size_t h_out_cap = 0, h_in_cap = 0;
        bool pending = false;
        const void *last_src = nullptr;  // for ugb200_jpeg_debug_coefficients (the fused path keeps coefficients on chip)
        long last_pitch = 0;
        bool last_vec_ok = false, last_fused = false;
        cudaEvent_t stats_ev = nullptr;  // recorded behind the copy of h_total: lets an asynchronous caller adapt the cap too
        bool stats_pending = false;
        int form = 0;  // 0: one fused kernel (default), 1 / 2: block kernel + assembly kernel
        bool attr_set[3] = { false, false, false };  // cudaFuncSetAttribute done for the fused / assembly kernels on this encoder's device
        bool stage_timing = false;       // ugb200_jpeg_encoder_stage_timing: events between the kernels of an encode
        cudaEvent_t stage_ev[5] = { nullptr, nullptr, nullptr, nullptr, nullptr };
};

namespace {

template <class T>
bool grow(T *&ptr, size_t &cap, size_t need)
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
bool grow_host(uint8_t *&ptr, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        if (ptr) {
                cudaFreeHost(ptr);
        }
        ptr = nullptr, cap = 0;
        if (cudaMallocHost((void **) &ptr, need) != cudaSuccess) {
                return false;
        }
        cap = need;
        return true;
}

void put16(std::vector<uint8_t> &v, unsigned x) { v.push_back((uint8_t) (x >> 8)), v.push_back((uint8_t) x); }
void put_dht(std::vector<uint8_t> &v, int tc_th, const uint8_t bits[16], const uint8_t *vals, int n)
{
        v.push_back(0xFF), v.push_back(0xC4);
        put16(v, 2 + 1 + 16 + n);
        v.push_back((uint8_t) tc_th);
        v.insert(v.end(), bits, bits + 16);
        v.insert(v.end(), vals, vals + n);
}

/// header layout as the reference's RFC 2435 writer (src/utils/jpeg_writer.c:215-382): SOI, APPn, DQT x2, SOF0, DHT x4, DRI, SOS
void build_header(ugb200_jpeg_encoder *e, const uint8_t ql[64], const uint8_t qc[64])
{
        std::vector<uint8_t> &v = e->header;
        v.clear();
        v.push_back(0xFF), v.push_back(0xD8);
        if (e->fmt == FMT_RGB_444) {
                static const uint8_t adobe[] = { 0xFF, 0xEE, 0, 14, 'A', 'd', 'o', 'b', 'e', 0, 100, 0, 0, 0, 0, 0 };
                v.insert(v.end(), adobe, adobe + sizeof adobe);
        } else {
                static const uint8_t jfif[] = { 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0 };
                v.insert(v.end(), jfif, jfif + sizeof jfif);
        }
        for (int t = 0; t < 2; ++t) {
                v.push_back(0xFF), v.push_back(0xDB);
                put16(v, 67);
                v.push_back((uint8_t) t);
                for (int k = 0; k < 64; ++k) {
                        v.push_back((t ? qc : ql)[ugb_jpeg_zigzag[k]]);
                }
        }
        v.push_back(0xFF), v.push_back(0xC0);
        put16(v, 17);
        v.push_back(8);
        put16(v, e->h), put16(v, e->w);
        v.push_back(3);
        for (int c = 0; c < 3; ++c) {
                v.push_back((uint8_t) (c + 1));
                v.push_back(c != 0 ? 0x11 : e->fmt == FMT_UYVY_422 ? 0x21 : e->fmt == FMT_PLANAR ? (uint8_t) (e->hs << 4 | e->vs) : 0x11);
                v.push_back(c == 0 ? 0 : 1);
        }
        put_dht(v, 0x00, ugb_jpeg_dc_luma_bits, ugb_jpeg_dc_vals, 12);
        put_dht(v, 0x10, ugb_jpeg_ac_luma_bits, ugb_jpeg_ac_luma_vals, 162);
        put_dht(v, 0x01, ugb_jpeg_dc_chroma_bits, ugb_jpeg_dc_vals, 12);
        put_dht(v, 0x11, ugb_jpeg_ac_chroma_bits, ugb_jpeg_ac_chroma_vals, 162);
        v.push_back(0xFF), v.push_back(0xDD);
        put16(v, 4), put16(v, e->ri);
        const int ncomp = e->fmt == FMT_UYVY_422 || e->g.interleaved ? 3 : 1;
        v.push_back(0xFF), v.push_back(0xDA);
        put16(v, 6 + 2 * ncomp);
        v.push_back((uint8_t) ncomp);
        for (int c = 0; c < ncomp; ++c) {
                v.push_back((uint8_t) (c + 1));
                v.push_back(c == 0 ? 0x00 : 0x11);
        }
        v.push_back(0), v.push_back(63), v.push_back(0);
}

/// FMT_PLANAR: hs x vs luma sampling, the caller resolves `interleaved` and the restart interval; `prep` = what jpeg_prep_kernel does
/// (PREP_*), part of the cache key like the geometry
int configure(ugb200_jpeg_encoder *e, int fmt, int w, int h, int quality, int ri, int interleaved, int hs = 1, int vs = 1, int prep = PREP_NONE)
{
        if (fmt != FMT_PLANAR) {
                interleaved = fmt == FMT_RGB_444 && interleaved ? 1 : 0;  // a UYVY stream is one interleaved scan anyway
                hs = vs = 1, prep = PREP_NONE;
        }
        if (ri <= 0) {
                ri = fmt == FMT_RGB_444 ? 8 : 4;  // src/video_compress/gpujpeg.cpp:351
        }
        if (ri > 65535) {
                return -1;
        }
        quality = quality < 1 ? 1 : quality > 100 ? 100 : quality;
        const bool same = e->fmt == fmt && e->w == w && e->h == h && e->quality == quality && e->ri == ri && e->interleaved == interleaved &&
                          e->hs == hs && e->vs == vs && e->prep == prep;
        if (same) {
                return 0;
        }
        e->fmt = fmt, e->w = w, e->h = h, e->quality = quality, e->ri = ri, e->interleaved = interleaved, e->hs = hs, e->vs = vs, e->prep = prep;
        jpeg_geom &g = e->g;
        jpeg_layout &L = e->lay;
        g = jpeg_geom{}, L = jpeg_layout{};
        g.fmt = fmt, g.w = w, g.h = h, g.ri = ri, g.interleaved = interleaved;
        L.hs = hs, L.vs = vs;
        if (fmt == FMT_PLANAR) {
                const int cw = (w + hs - 1) / hs, ch = (h + vs - 1) / vs;  // T.81 A.1.1: chroma is ceil(w * 1 / hs) x ceil(h * 1 / vs)
                L.plane_w[0] = w, L.plane_h[0] = h;
                for (int c = 1; c < 3; ++c) {
                        L.plane_w[c] = cw, L.plane_h[c] = ch;
                }
                if (interleaved) {  // one scan; MCU = hs x vs luma blocks + Cb + Cr over an (8 hs) x (8 vs) area
                        g.bw = (w + 8 * hs - 1) / (8 * hs), g.bh = (h + 8 * vs - 1) / (8 * vs);
                        g.mcu_per_scan = g.bw * g.bh, g.blocks_per_mcu = hs * vs + 2;
                        g.nblocks = g.mcu_per_scan * g.blocks_per_mcu;
                        g.seg_per_scan = (g.mcu_per_scan + ri - 1) / ri;
                        g.nseg = g.seg_per_scan, L.nscans = 1, g.sos_len = 0;
                        L.scan_mcus[0] = g.mcu_per_scan;
                } else {  // one scan per component; MCU = one block; each component's block grid is not padded to whole MCUs (T.81 A.2.2)
                        g.blocks_per_mcu = 1, L.nscans = 3, g.sos_len = 10, g.nblocks = 0, g.nseg = 0;
                        for (int c = 0; c < 3; ++c) {
                                L.comp_bw[c] = (L.plane_w[c] + 7) / 8;
                                L.comp_blk0[c] = g.nblocks;
                                L.scan_mcus[c] = L.comp_bw[c] * ((L.plane_h[c] + 7) / 8);
                                L.scan_seg0[c] = g.nseg;
                                g.nblocks += L.scan_mcus[c];
                                g.nseg += (L.scan_mcus[c] + ri - 1) / ri;
                        }
                        g.bw = L.comp_bw[0], g.bh = (h + 7) / 8, g.mcu_per_scan = L.scan_mcus[0];
                        g.seg_per_scan = (g.mcu_per_scan + ri - 1) / ri;
                }
                for (int c = L.nscans; c < 4; ++c) {
                        L.scan_seg0[c] = g.nseg;
                }
                if (prep != PREP_NONE) {  // planes written by jpeg_prep_kernel: 16-byte aligned rows, 256-byte aligned planes
                        const long py = (w + 15) & ~15, pc = (cw + 15) & ~15;
                        const size_t oc = ((size_t) py * h + 255) & ~(size_t) 255, oc2 = oc + (((size_t) pc * ch + 255) & ~(size_t) 255);
                        if (!grow(e->planes, e->planes_cap, oc2 + (size_t) pc * ch)) {
                                return -2;
                        }
                        L.plane[0] = e->planes, L.plane[1] = e->planes + oc, L.plane[2] = e->planes + oc2;
                        L.plane_pitch[0] = py, L.plane_pitch[1] = L.plane_pitch[2] = pc;
                }
        } else if (fmt == FMT_UYVY_422) {
                g.bw = (w + 15) / 16, g.bh = (h + 7) / 8;
                g.mcu_per_scan = g.bw * g.bh, g.blocks_per_mcu = 4;
                g.nblocks = g.mcu_per_scan * 4;
                g.seg_per_scan = (g.mcu_per_scan + ri - 1) / ri;
                g.nseg = g.seg_per_scan;
                g.sos_len = 0;
        } else {
                g.bw = (w + 7) / 8, g.bh = (h + 7) / 8;
                g.mcu_per_scan = g.bw * g.bh, g.blocks_per_mcu = 1;
                g.nblocks = g.mcu_per_scan * 3;
                g.seg_per_scan = (g.mcu_per_scan + ri - 1) / ri;
                g.nseg = g.seg_per_scan * 3;
                g.sos_len = 10;
                if (interleaved) {  // one scan of R G B MCUs
                        g.blocks_per_mcu = 3;
                        g.nseg = g.seg_per_scan, g.sos_len = 0;
                }
        }
        if (fmt != FMT_PLANAR) {  // scans of equal length
                L.nscans = g.nseg / g.seg_per_scan;
                for (int c = 0; c < 4; ++c) {
                        L.scan_seg0[c] = min(c, L.nscans) * g.seg_per_scan;
                }
        }
        g.slot = ri * g.blocks_per_mcu * kSlotBytesPerBlock + kSlotExtra;

        uint8_t ql[64], qc[64];
        ugb_jpeg_scaled_qtable(ugb_jpeg_q_luma, quality, ql);
        ugb_jpeg_scaled_qtable(ugb_jpeg_q_chroma, quality, qc);
        jpeg_hufftab t;
        ugb_jpeg_quant_multipliers(ql, e->qt.qmul[0]);
        ugb_jpeg_quant_multipliers(qc, e->qt.qmul[1]);
        uint16_t code[256];
        uint8_t len[256];
        for (int k = 0; k < 2; ++k) {
                ugb_jpeg_build_codes(k ? ugb_jpeg_dc_chroma_bits : ugb_jpeg_dc_luma_bits, ugb_jpeg_dc_vals, 12, code, len);
                for (int i = 0; i < 16; ++i) {
                        t.dc[k][i] = ((uint32_t) len[i] << 16) | code[i];
                }
                ugb_jpeg_build_codes(k ? ugb_jpeg_ac_chroma_bits : ugb_jpeg_ac_luma_bits, k ? ugb_jpeg_ac_chroma_vals : ugb_jpeg_ac_luma_vals,
                                     162, code, len);
                for (int i = 0; i < 256; ++i) {
                        t.ac[k][i] = ((uint32_t) len[i] << 16) | code[i];
                }
        }
        if ((e->d_huff == nullptr && cudaMalloc((void **) &e->d_huff, sizeof t) != cudaSuccess) ||
            cudaMemcpyAsync(e->d_huff, &t, sizeof t, cudaMemcpyHostToDevice, e->stream) != cudaSuccess) {
                return -2;
        }
        build_header(e, ql, qc);
        g.header_len = (int) e->header.size();

        const size_t out_need = (size_t) w * h * 3 + 4096;  // gpujpeg.cpp:355
        if (!grow(e->coef, e->coef_cap, (size_t) g.nblocks * 64) || !grow(e->slots, e->slots_cap, (size_t) g.nseg * g.slot) ||
            !grow(e->out, e->out_cap, out_need)) {
                return -2;
        }
        size_t cap2 = e->seg_cap;
        if (!grow(e->sizes, e->seg_cap, (size_t) g.nseg) || !grow(e->offsets, cap2, (size_t) g.nseg) ||
            !grow(e->cta_total, e->cta_cap, (size_t) g.nseg + 8)) {
                return -2;
        }
        if (e->total == nullptr && cudaMalloc((void **) &e->total, 16) != cudaSuccess) {
                return -2;
        }
        if (e->h_total == nullptr && cudaMallocHost((void **) &e->h_total, 16) != cudaSuccess) {
                return -2;
        }
        if (cudaMemcpyAsync(e->out, e->header.data(), e->header.size(), cudaMemcpyHostToDevice, e->stream) != cudaSuccess) {
                return -2;
        }
        cudaStreamSynchronize(e->stream);  // header vector / table struct are host temporaries
        return 0;
}

}  // namespace

extern "C" {

void ugb200_jpeg_default_params(struct ugb200_jpeg_params *p)
{
        p->quality = 75;  // gpujpeg_set_default_parameters
        p->restart_interval = 0;
        p->interleaved = 0;
}

ugb200_jpeg_encoder *ugb200_jpeg_encoder_create(cuda_wrapper_stream_t stream)
{
        ugb200_jpeg_encoder *e = new (std::nothrow) ugb200_jpeg_encoder;
        if (e) {
                e->stream = (cudaStream_t) stream;
                const char *f = getenv("UGB200_JPEG_TWO_KERNELS");  // "1": two-kernel form, "8": the same with the 64-register block kernel
                e->form = !f ? 0 : f[0] == '8' ? 2 : 1;
        }
        return e;
}

void ugb200_jpeg_encoder_destroy(ugb200_jpeg_encoder *e)
{
        if (!e) {
                return;
        }
        cudaStreamSynchronize(e->stream);
        cudaFree(e->coef), cudaFree(e->slots), cudaFree(e->out), cudaFree(e->staging);
        cudaFree(e->sizes), cudaFree(e->offsets), cudaFree(e->cta_total), cudaFree(e->total), cudaFree(e->lb_state), cudaFree(e->d_huff);
        cudaFree(e->gbits), cudaFree(e->glen), cudaFree(e->planes);
        cudaFreeHost(e->h_out), cudaFreeHost(e->h_in), cudaFreeHost(e->h_total);
        if (e->stats_ev) {
                cudaEventDestroy(e->stats_ev);
        }
        for (cudaEvent_t ev : e->stage_ev) {
                if (ev) {
                        cudaEventDestroy(ev);
                }
        }
        delete e;
}

/// size the fused kernel's per-block bit buffer for the next frame: the last finished frame's largest block + 25 %
static void adapt_cap(ugb200_jpeg_encoder *e)
{
        if (e->last_fused && e->stats_pending) {
                const int want = (int) ((e->h_total[1] + e->h_total[1] / 4 + 31) / 32);
                e->cap_words = want <= 12 ? 12 : want <= 16 ? 16 : want <= 24 ? 24 : want <= 32 ? 32 : kBlkWords;
        }
        e->stats_pending = false;
}

static int launch_tail(ugb200_jpeg_encoder *e, int nctas, int segs_per_cta, int ctas_per_scan, bool single_pass, bool two_kernels);

int ugb200_jpeg_encode_device(ugb200_jpeg_encoder *e, const void *src, long pitch, int width, int height, int codec,
                              const struct ugb200_jpeg_params *params)
{
        if (!e || !src || width <= 0 || height <= 0 || width > 65535 || height > 65535 || !params) {
                return -1;
        }
        int fmt;
        if (codec == UGB_UYVY) {
                fmt = FMT_UYVY_422;
        } else if (codec == UGB_RGB) {
                fmt = FMT_RGB_444;
        } else {
                return -4;
        }
        if (pitch == 0) {
                pitch = (long) width * (fmt == FMT_UYVY_422 ? 2 : 3);
        }
        const int rc = configure(e, fmt, width, height, params->quality, params->restart_interval, params->interleaved);
        if (rc != 0) {
                return rc;
        }
        const jpeg_geom &g = e->g;
        // UYVY: 128-bit loads and 16-byte cp.async; RGB: 8-byte cp.async pieces of the staged tile
        const bool vec_ok = fmt == FMT_UYVY_422 ? !(15 & (size_t) src) && !(pitch & 15) : !(7 & (size_t) src) && !(pitch & 7);
        e->last_src = src, e->last_pitch = pitch, e->last_vec_ok = vec_ok;
        if (e->stats_pending && cudaEventQuery(e->stats_ev) == cudaSuccess) {
                adapt_cap(e);  // the previous frame has finished although nobody fetched its result yet
        }
        const int bps = g.ri * g.blocks_per_mcu;
        static const bool force_split = getenv("UGB200_JPEG_SPLIT") != nullptr;
        const bool fused = !force_split && !g.interleaved && (bps == 4 || bps == 8 || bps == 16 || bps == 32);
        e->last_fused = fused;
        int nctas, segs_per_cta, ctas_per_scan;
        bool single_pass = false, two_kernels = false;
        if (e->stage_timing) {
                cudaEventRecord(e->stage_ev[0], e->stream);
        }
        if (fused) {  // one kernel: DCT + entropy coding + segment assembly
                static const char *cap_env = getenv("UGB200_JPEG_CAP");
                const int cap = cap_env ? atoi(cap_env) : e->cap_words;
                const size_t smem = (size_t) (32 * 128 + 2 * cap * 128) * sizeof(uint32_t);
                segs_per_cta = 128 / bps;
                cudaMemsetAsync(e->total + 1, 0, 8, e->stream);
                ctas_per_scan = fmt == FMT_UYVY_422 ? (g.mcu_per_scan + 31) / 32 : (g.mcu_per_scan + 127) / 128;
                nctas = fmt == FMT_UYVY_422 ? ctas_per_scan : ctas_per_scan * 3;
                // Single-pass compaction (decoupled look-back inside the fused kernel) is implemented and byte-exact, was no faster than
                // slots + scan + compact on an earlier GPU (the ticket, the size pre-pass and two more barriers cost what the two small kernels
                // cost; not re-measured on the H100) - it stays behind a switch.
                static const bool want_single_pass = getenv("UGB200_JPEG_SINGLE_PASS") != nullptr;
                single_pass = want_single_pass;
                jpeg_lookback lb = { nullptr, nullptr, e->out, (uint32_t) e->out_cap, e->total, ctas_per_scan };
                if (single_pass) {
                        if (!grow(e->lb_state, e->lb_cap, (size_t) nctas + 1)) {
                                return -2;
                        }
                        cudaMemsetAsync(e->lb_state, 0, ((size_t) nctas + 1) * sizeof(unsigned long long), e->stream);
                        lb.state = e->lb_state + 1, lb.ticket = (uint32_t *) e->lb_state;  // word 0 of the array = the ticket counter
                }
                const bool seven = cap <= 12;  // 28 KB per CTA: seven CTAs (28 warps) fit an SM
                const int max_smem = (int) ((32 * 128 + 2 * kBlkWords * 128) * sizeof(uint32_t));
                if (!e->attr_set[fmt == FMT_UYVY_422 ? 0 : 1]) {  // per encoder = per device context: the attribute does not carry over to another GPU
                        if (fmt == FMT_UYVY_422) {
                                cudaFuncSetAttribute(jpeg_fused_kernel<FMT_UYVY_422, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
                        } else {
                                cudaFuncSetAttribute(jpeg_fused_kernel<FMT_RGB_444, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
                        }
                        e->attr_set[fmt == FMT_UYVY_422 ? 0 : 1] = true;
                }
                const dim3 grid(nctas);  // RGB: component fastest (two-pass) or tickets running over the three scans (single pass)
                // two-kernel form (UGB200_JPEG_TWO_KERNELS at encoder creation): blocks -> bit strings in global memory, then the segment assembly as a
                // kernel of its own.  Not the default: on an earlier GPU it was no faster on one stream and only slightly faster with two encoders alternating.
                const bool eight = e->form == 2;  // 64 registers / 8 CTAs per SM for the block kernel
                two_kernels = !single_pass && e->form != 0;
                if (two_kernels) {
                        if (!grow(e->gbits, e->gbits_cap, (size_t) nctas * cap * 128) || !grow(e->glen, e->glen_cap, (size_t) nctas * 128)) {
                                return -2;
                        }
                        const size_t smem_a = fmt == FMT_UYVY_422 ? 32 * 128 * 4 : 8 * 3072;  // the coefficient array; the RGB tile over it is 24 KB
#define UGB_BLOCKS(FMT, MINB)                                                                                                                                  \
        jpeg_fused_kernel<FMT, MINB, true><<<grid, 128, smem_a, e->stream>>>((const uint8_t *) src, pitch, g, e->slots, e->sizes, e->offsets, e->cta_total, vec_ok, \
                                                                             cap, e->total + 1, lb, e->qt, e->d_huff, e->gbits, e->glen, e->coef)
                        if (fmt == FMT_UYVY_422) {
                                if (eight) {
                                        UGB_BLOCKS(FMT_UYVY_422, 8);
                                } else {
                                        UGB_BLOCKS(FMT_UYVY_422, 7);
                                }
                        } else {
                                if (eight) {
                                        UGB_BLOCKS(FMT_RGB_444, 8);
                                } else {
                                        UGB_BLOCKS(FMT_RGB_444, 7);
                                }
                        }
#undef UGB_BLOCKS
                        if (e->stage_timing) {
                                cudaEventRecord(e->stage_ev[1], e->stream);
                        }
                        cudaLaunchAttribute pdl[1];
                        pdl[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
                        pdl[0].val.programmaticStreamSerializationAllowed = 1;
                        cudaLaunchConfig_t cfg{};
                        cfg.stream = e->stream, cfg.attrs = pdl, cfg.numAttrs = e->stage_timing ? 0 : 1;
                        cfg.gridDim = dim3((unsigned) nctas), cfg.blockDim = dim3(128), cfg.dynamicSmemBytes = (size_t) cap * 1024;
                        if (cfg.dynamicSmemBytes > 48 * 1024 && !e->attr_set[2]) {
                                cudaFuncSetAttribute(jpeg_assemble_kernel<FMT_UYVY_422>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBlkWords * 1024);
                                cudaFuncSetAttribute(jpeg_assemble_kernel<FMT_RGB_444>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBlkWords * 1024);
                                e->attr_set[2] = true;
                        }
                        if (fmt == FMT_UYVY_422) {
                                cudaLaunchKernelEx(&cfg, jpeg_assemble_kernel<FMT_UYVY_422>, g, (const uint32_t *) e->gbits, (const uint16_t *) e->glen, (const int16_t *) e->coef,
                                                   e->slots, e->sizes, e->offsets, e->cta_total, cap, ctas_per_scan, (const uint32_t *) e->d_huff);
                        } else {
                                cudaLaunchKernelEx(&cfg, jpeg_assemble_kernel<FMT_RGB_444>, g, (const uint32_t *) e->gbits, (const uint16_t *) e->glen, (const int16_t *) e->coef,
                                                   e->slots, e->sizes, e->offsets, e->cta_total, cap, ctas_per_scan, (const uint32_t *) e->d_huff);
                        }
                } else {
#define UGB_FUSED(FMT, MINB, LEAN)                                                                                                                        \
        jpeg_fused_kernel<FMT, MINB, false, LEAN><<<grid, 128, smem, e->stream>>>((const uint8_t *) src, pitch, g, e->slots, e->sizes, e->offsets, e->cta_total, vec_ok, \
                                                                                  cap, e->total + 1, lb, e->qt, e->d_huff)
                // every CTA's tile whole and bulk-copyable?  (the conditions of the kernel's `early_tile`, for all CTAs at once; UGB200_JPEG_LEAN=0 keeps the general kernel)
                static const bool allow_lean = getenv("UGB200_JPEG_LEAN") == nullptr || atoi(getenv("UGB200_JPEG_LEAN")) != 0;
                const bool lean = allow_lean && vec_ok && cap >= 8 && (g.h & 7) == 0 &&
                                  (fmt == FMT_UYVY_422 ? g.bw % 32 == 0 && g.bw * 16 == g.w
                                                       : g.mcu_per_scan % 128 == 0 && (g.w & 7) == 0 && g.bw >= 128 && !(g.bw & 1) && !(15 & (size_t) src) && !(pitch & 15));
                if (fmt == FMT_UYVY_422) {
                        if (seven) {
                                lean ? UGB_FUSED(FMT_UYVY_422, 7, true) : UGB_FUSED(FMT_UYVY_422, 7, false);
                        } else {
                                lean ? UGB_FUSED(FMT_UYVY_422, 6, true) : UGB_FUSED(FMT_UYVY_422, 6, false);
                        }
                } else {
                        if (seven) {
                                lean ? UGB_FUSED(FMT_RGB_444, 7, true) : UGB_FUSED(FMT_RGB_444, 7, false);
                        } else {
                                lean ? UGB_FUSED(FMT_RGB_444, 6, true) : UGB_FUSED(FMT_RGB_444, 6, false);
                        }
                }
#undef UGB_FUSED
                }
        } else {  // split path: any restart interval
                const int dct_ctas = fmt == FMT_UYVY_422 ? (g.mcu_per_scan + 31) / 32 : (g.nblocks + 127) / 128;
                jpeg_dct_kernel<false><<<dct_ctas, 128, 0, e->stream>>>((const uint8_t *) src, pitch, g, e->coef, vec_ok, e->qt, e->lay);
                nctas = (g.nseg + 127) / 128, segs_per_cta = 128, ctas_per_scan = 0;
                jpeg_huffman_kernel<false><<<nctas, 128, 0, e->stream>>>(e->coef, g, e->slots, e->sizes, e->offsets, e->cta_total, e->d_huff, e->lay);
        }
        return launch_tail(e, nctas, segs_per_cta, ctas_per_scan, single_pass, two_kernels);
}

/// the common end of an encode: offset scan + compaction (nothing behind the single-pass form), the copy of the stream size and statistics
static int launch_tail(ugb200_jpeg_encoder *e, int nctas, int segs_per_cta, int ctas_per_scan, bool single_pass, bool two_kernels)
{
        const jpeg_geom &g = e->g;
        if (e->stage_timing) {
                if (!two_kernels) {
                        cudaEventRecord(e->stage_ev[1], e->stream);
                }
                cudaEventRecord(e->stage_ev[2], e->stream);  // behind the assembly kernel (= behind the one-kernel form when there is none)
        }
        if (!single_pass) {
                // programmatic dependent launch: the scan and the compaction are set up while their predecessor drains (they wait for its results
                // with griddepcontrol.wait), which takes the launch latencies of two tiny kernels out of the frame time.  Stage timing records
                // events between the kernels, which serialises them again: timing mode launches the plain way.
                cudaLaunchAttribute pdl[1];
                pdl[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
                pdl[0].val.programmaticStreamSerializationAllowed = 1;
                cudaLaunchConfig_t cfg{};
                cfg.stream = e->stream;
                cfg.attrs = pdl, cfg.numAttrs = e->stage_timing ? 0 : 1;
                cfg.gridDim = dim3(1), cfg.blockDim = dim3(1024);
                cudaLaunchKernelEx(&cfg, jpeg_scan_kernel, e->cta_total, nctas, g, e->total, e->lay.nscans);
                if (e->stage_timing) {
                        cudaEventRecord(e->stage_ev[3], e->stream);
                }
                cfg.gridDim = dim3((unsigned) (((long) g.nseg * kCompactLanes + 255) / 256)), cfg.blockDim = dim3(256);
                cudaLaunchKernelEx(&cfg, jpeg_compact_kernel, (const uint8_t *) e->slots, (const uint32_t *) e->sizes, (const uint32_t *) e->offsets,
                                   (const uint32_t *) e->cta_total, g, segs_per_cta, ctas_per_scan, e->out, (const uint32_t *) e->total, (uint32_t) e->out_cap, e->lay);
        }
        if (e->stage_timing) {
                if (single_pass) {
                        cudaEventRecord(e->stage_ev[3], e->stream);
                }
                cudaEventRecord(e->stage_ev[4], e->stream);
        }
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        cudaMemcpyAsync(e->h_total, e->total, 12, cudaMemcpyDeviceToHost, e->stream);
        if (e->stats_ev != nullptr || cudaEventCreateWithFlags(&e->stats_ev, cudaEventDisableTiming) == cudaSuccess) {
                cudaEventRecord(e->stats_ev, e->stream);
                e->stats_pending = true;
        }
        e->pending = true;
        return 0;
}

void ugb200_jpeg_default_params_ex(struct ugb200_jpeg_params_ex *p)
{
        ugb200_jpeg_default_params(&p->base);
        p->subsampling = 0;
        p->color_space = UGB200_JPEG_CS_NATIVE;
}

/// the supported matrix of ugb200_jpeg.h: @returns 0 for the stream of ugb200_jpeg_encode_device (UYVY 4:2:2, RGB 4:4:4), 1 for
/// FMT_PLANAR with hs x vs luma sampling and pre-processing `prep`, -4 for anything else (chroma upsampling, YCbCr -> RGB, one YCbCr
/// matrix -> another, subsampled RGB)
static int resolve_layout(int codec, int sub, int cs, int *hs, int *vs, int *prep)
{
        if ((sub != 0 && sub != 444 && sub != 422 && sub != 420) || cs < UGB200_JPEG_CS_NATIVE || cs > UGB200_JPEG_CS_RGB) {
                return -4;
        }
        const bool yuv_cs = cs == UGB200_JPEG_CS_NATIVE || cs == UGB200_JPEG_CS_Y709;  // UYVY and I420 frames are BT.709 YCbCr
        if (codec == UGB_UYVY && yuv_cs) {
                if (sub == 0 || sub == 422) {
                        return 0;
                }
                *hs = *vs = 2, *prep = PREP_UYVY;
                return sub == 420 ? 1 : -4;
        }
        if (codec == UGB_I420 && yuv_cs) {
                *hs = *vs = 2, *prep = PREP_NONE;
                return sub == 0 || sub == 420 ? 1 : -4;
        }
        if (codec == UGB_RGB) {
                if (cs == UGB200_JPEG_CS_NATIVE || cs == UGB200_JPEG_CS_RGB) {
                        return sub == 0 || sub == 444 ? 0 : -4;
                }
                *hs = sub == 422 || sub == 420 ? 2 : 1, *vs = sub == 420 ? 2 : 1, *prep = PREP_RGB + cs;
                return 1;
        }
        return -4;
}

/// FMT_PLANAR: pre-processing (unless the I420 frame is read in place), then the split path
static int encode_planar(ugb200_jpeg_encoder *e, const void *src, long pitch, int width, int height, int codec, const struct ugb200_jpeg_params *params,
                         int hs, int vs, int prep)
{
        if (codec == UGB_I420 && pitch != 0) {
                return -1;  // I420 is three tight planes (vc_get_datalen)
        }
        const bool rgb = codec == UGB_RGB;
        if (pitch == 0) {
                pitch = (long) width * (rgb ? 3 : 2);  // as ugb200_jpeg_encode_device
        }
        const int ri = params->restart_interval > 0 ? params->restart_interval : rgb ? 8 : 4;  // gpujpeg.cpp:351: by the input format
        const int interleaved = rgb ? (params->interleaved ? 1 : 0) : 1;                       // gpujpeg.cpp:303: UYVY / I420 one scan
        int rc = configure(e, FMT_PLANAR, width, height, params->quality, ri, interleaved, hs, vs, prep);
        if (rc != 0) {
                return rc;
        }
        const jpeg_geom &g = e->g;
        jpeg_layout &L = e->lay;
        if (prep == PREP_NONE) {  // UltraGrid's I420 frame: Y w x h, then Cb and Cr of ceil(w / 2) x ceil(h / 2) each, tightly packed
                const uint8_t *y = (const uint8_t *) src;
                const size_t cn = (size_t) L.plane_w[1] * L.plane_h[1];
                L.plane[0] = y, L.plane[1] = y + (size_t) width * height, L.plane[2] = y + (size_t) width * height + cn;
                L.plane_pitch[0] = width, L.plane_pitch[1] = L.plane_pitch[2] = L.plane_w[1];
        }
        if (e->stats_pending && cudaEventQuery(e->stats_ev) == cudaSuccess) {
                adapt_cap(e);
        }
        if (prep != PREP_NONE) {
                jpeg_prep_args a{};
                a.src = (const uint8_t *) src, a.pitch = pitch, a.w = width, a.h = height, a.rgb = rgb, a.hs = hs, a.vs = vs;
                a.cw = L.plane_w[1], a.ch = L.plane_h[1];
                if (rgb) {
                        const color_coeffs c = prep == PREP_RGB + UGB200_JPEG_CS_Y709 ? coeffs_709(8) : prep == PREP_RGB + UGB200_JPEG_CS_Y601 ? coeffs_601(8) : coeffs_601(0);
                        const int k[9] = { c.y_r, c.y_g, c.y_b, c.cb_r, c.cb_g, c.cb_b, c.cr_r, c.cr_g, c.cr_b };
                        memcpy(a.c, k, sizeof k);
                        a.off_y = prep == PREP_RGB + UGB200_JPEG_CS_Y601FULL ? 0 : 16;
                }
                for (int c = 0; c < 3; ++c) {
                        a.p[c] = (uint8_t *) L.plane[c], a.pp[c] = L.plane_pitch[c];
                }
                const long n = (long) a.cw * a.ch;
                jpeg_prep_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, e->stream>>>(a);
        }
        bool vec_ok = true;  // 8-byte row loads
        for (int c = 0; c < 3; ++c) {
                vec_ok = vec_ok && !(7 & (size_t) L.plane[c]) && !(7 & L.plane_pitch[c]);
        }
        e->last_src = src, e->last_pitch = pitch, e->last_vec_ok = vec_ok, e->last_fused = false;
        if (e->stage_timing) {
                cudaEventRecord(e->stage_ev[0], e->stream);
        }
        jpeg_dct_kernel<true><<<(g.nblocks + 127) / 128, 128, 0, e->stream>>>(nullptr, 0, g, e->coef, vec_ok, e->qt, L);
        const int nctas = (g.nseg + 127) / 128;
        jpeg_huffman_kernel<true><<<nctas, 128, 0, e->stream>>>(e->coef, g, e->slots, e->sizes, e->offsets, e->cta_total, e->d_huff, L);
        return launch_tail(e, nctas, 128, 0, false, false);
}

int ugb200_jpeg_encode_device_ex(ugb200_jpeg_encoder *e, const void *src, long pitch, int width, int height, int codec,
                                 const struct ugb200_jpeg_params_ex *params)
{
        if (!e || !src || width <= 0 || height <= 0 || width > 65535 || height > 65535 || !params) {
                return -1;
        }
        int hs = 1, vs = 1, prep = PREP_NONE;
        const int layout = resolve_layout(codec, params->subsampling, params->color_space, &hs, &vs, &prep);
        if (layout < 0) {
                return layout;
        }
        if (layout == 0) {
                return ugb200_jpeg_encode_device(e, src, pitch, width, height, codec, &params->base);
        }
        return encode_planar(e, src, pitch, width, height, codec, &params->base, hs, vs, prep);
}

int ugb200_jpeg_encoder_stage_timing(ugb200_jpeg_encoder *e, int enable)
{
        if (!e) {
                return -1;
        }
        if (enable) {
                for (cudaEvent_t &ev : e->stage_ev) {
                        if (ev == nullptr && cudaEventCreate(&ev) != cudaSuccess) {
                                return -2;
                        }
                }
        }
        e->stage_timing = enable != 0;
        return 0;
}

int ugb200_jpeg_encoder_stage_times(ugb200_jpeg_encoder *e, float us[4])
{
        if (!e || !us || !e->stage_timing || !e->pending) {
                return -1;
        }
        if (cudaEventSynchronize(e->stage_ev[4]) != cudaSuccess) {
                return -2;
        }
        for (int i = 0; i < 4; ++i) {
                float ms = 0;
                if (cudaEventElapsedTime(&ms, e->stage_ev[i], e->stage_ev[i + 1]) != cudaSuccess) {
                        return -2;
                }
                us[i] = ms * 1000.0f;
        }
        return 0;
}

int ugb200_jpeg_result_device(ugb200_jpeg_encoder *e, const void **dev_ptr, size_t *size)
{
        if (!e || !e->pending) {
                return -1;
        }
        if (cudaStreamSynchronize(e->stream) != cudaSuccess) {
                return -2;
        }
        if (*e->h_total > e->out_cap) {
                return -5;  // the stream does not fit w * h * 3 bytes (the capacity the reference gives libgpujpeg, gpujpeg.cpp:355)
        }
        if (dev_ptr) {
                *dev_ptr = e->out;
        }
        adapt_cap(e);
        if (size) {
                *size = *e->h_total;
        }
        return 0;
}

/// shared body of ugb200_jpeg_encode(_into)(_ex): upload (host source), encode, wait, stream to `dst` (host).  I420 only through the _ex calls
static int encode_to_host(ugb200_jpeg_encoder *e, const void *src, int src_is_device, long pitch, int width, int height, int codec,
                          const struct ugb200_jpeg_params_ex *params, bool ex, uint8_t *dst, size_t dst_cap, uint8_t **out, size_t *out_size)
{
        if (!e || !src || !out_size || width <= 0 || height <= 0) {
                return -1;
        }
        const int bpp = codec == UGB_UYVY ? 2 : codec == UGB_RGB ? 3 : codec == UGB_I420 && ex ? 1 : 0;
        if (bpp == 0) {
                return -4;
        }
        const void *dsrc = src;
        if (!src_is_device) {
                size_t n;
                if (codec == UGB_I420) {  // vc_get_datalen (host/video_codec.cpp:56-58); three tight planes, no pitch
                        if (pitch != 0) {
                                return -1;
                        }
                        n = (size_t) width * height + 2 * (size_t) ((width + 1) / 2) * ((height + 1) / 2);
                } else {
                        if (pitch == 0) {
                                pitch = (long) width * bpp;
                        }
                        n = (size_t) pitch * height;
                }
                if (!grow(e->staging, e->staging_cap, n)) {
                        return -2;
                }
                if (cudaMemcpyAsync(e->staging, src, n, cudaMemcpyHostToDevice, e->stream) != cudaSuccess) {
                        return -2;
                }
                dsrc = e->staging;
        }
        int rc = ex ? ugb200_jpeg_encode_device_ex(e, dsrc, pitch, width, height, codec, params)
                    : ugb200_jpeg_encode_device(e, dsrc, pitch, width, height, codec, params ? &params->base : nullptr);
        if (rc != 0) {
                return rc;
        }
        size_t n = 0;
        rc = ugb200_jpeg_result_device(e, nullptr, &n);
        if (rc != 0) {
                return rc;
        }
        if (dst == nullptr) {  // encoder-owned pinned buffer
                if (!grow_host(e->h_out, e->h_out_cap, e->out_cap)) {
                        return -2;
                }
                dst = e->h_out;
        } else if (n > dst_cap) {
                return -5;
        }
        if (cudaMemcpyAsync(dst, e->out, n, cudaMemcpyDeviceToHost, e->stream) != cudaSuccess ||
            cudaStreamSynchronize(e->stream) != cudaSuccess) {
                return -2;
        }
        if (out) {
                *out = dst;
        }
        *out_size = n;
        return 0;
}

int ugb200_jpeg_encode(ugb200_jpeg_encoder *e, const void *src, int src_is_device, long pitch, int width, int height, int codec,
                       const struct ugb200_jpeg_params *params, uint8_t **out, size_t *out_size)
{
        if (!out) {
                return -1;
        }
        ugb200_jpeg_params_ex px{};
        if (params) {
                px.base = *params;
        }
        return encode_to_host(e, src, src_is_device, pitch, width, height, codec, params ? &px : nullptr, false, nullptr, 0, out, out_size);
}

int ugb200_jpeg_encode_into(ugb200_jpeg_encoder *e, const void *src, int src_is_device, long pitch, int width, int height, int codec,
                            const struct ugb200_jpeg_params *params, uint8_t *dst, size_t dst_cap, size_t *out_size)
{
        if (!dst) {
                return -1;
        }
        ugb200_jpeg_params_ex px{};
        if (params) {
                px.base = *params;
        }
        return encode_to_host(e, src, src_is_device, pitch, width, height, codec, params ? &px : nullptr, false, dst, dst_cap, nullptr, out_size);
}

int ugb200_jpeg_encode_into_ex(ugb200_jpeg_encoder *e, const void *src, int src_is_device, long pitch, int width, int height, int codec,
                               const struct ugb200_jpeg_params_ex *params, uint8_t *dst, size_t dst_cap, size_t *out_size)
{
        if (!dst) {
                return -1;
        }
        return encode_to_host(e, src, src_is_device, pitch, width, height, codec, params, true, dst, dst_cap, nullptr, out_size);
}

int ugb200_jpeg_debug_coefficients(ugb200_jpeg_encoder *e, const int16_t **dev_ptr, size_t *count)
{
        if (!e || !e->coef || !e->last_src) {
                return -1;
        }
        {  // recompute them with the stand-alone DCT kernel from the last source frame (which must still be alive)
                const jpeg_geom &g = e->g;
                const int dct_ctas = g.fmt == FMT_UYVY_422 ? (g.mcu_per_scan + 31) / 32 : (g.nblocks + 127) / 128;
                if (g.fmt == FMT_PLANAR) {  // the planes of the last encode (I420: its source frame)
                        jpeg_dct_kernel<true><<<dct_ctas, 128, 0, e->stream>>>(nullptr, 0, g, e->coef, e->last_vec_ok, e->qt, e->lay);
                } else {
                        jpeg_dct_kernel<false><<<dct_ctas, 128, 0, e->stream>>>((const uint8_t *) e->last_src, e->last_pitch, g, e->coef, e->last_vec_ok, e->qt, e->lay);
                }
        }
        cudaStreamSynchronize(e->stream);
        *dev_ptr = e->coef;
        *count = (size_t) e->g.nblocks * 64;
        return 0;
}

}  // extern "C"
