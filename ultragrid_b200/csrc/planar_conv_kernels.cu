// Whole-buffer packed <-> planar converters: device form of the rest of UltraGrid's src/to_planar.c and of src/from_planar.c
// (v210_to_p010le lives in planar_kernels.cu).  Same function names and the same by-value argument structs as the reference
// (include/ugb200.h); every routine states the reference lines it follows.
//
// All of them are pure HBM streaming (1-8 B/px in, 1-8 B/px out, a handful of byte permutes per word).  One scheme serves all:
// a thread owns one UNIT (4 or 8 pixels, or one 36-byte R12L group) of one row (or row pair for 4:2:0), lanes walk along the
// row so that every plane is read/written as consecutive 4-16 byte pieces; the vector path is taken when the host has verified
// the alignment of every pointer and stride and the unit lies wholly inside the row, otherwise the same unit goes sample by
// sample with the reference's edge rules.  Grid = (units / 128, rows).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ugb200.h"
#include "host/video_codec.h"

namespace ugb {

template <class T>
__device__ __forceinline__ T ldv(const void *p)
{
        return __ldg((const T *) p);
}
template <class T>
__device__ __forceinline__ void stv(void *p, T v)
{
        *(T *) p = v;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) { return __byte_perm(a, b, s); }

template <class Op>
__global__ void __launch_bounds__(128) planar_kernel(const Op op)
{
        const int u = blockIdx.x * blockDim.x + threadIdx.x;
        if (u >= op.units) {
                return;
        }
        for (int r = blockIdx.y; r < op.rows; r += gridDim.y) {
                op.run(u, r);
        }
}

template <class Op>
static int launch_planar(const Op &op, cudaStream_t s)
{
        if (op.units <= 0 || op.rows <= 0) {
                return 0;
        }
        dim3 grid((op.units + 127) / 128, op.rows > 65535 ? 65535 : op.rows);
        planar_kernel<Op><<<grid, 128, 0, s>>>(op);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

static bool al16(const void *p) { return (15 & (size_t) p) == 0; }
static bool al16(unsigned v) { return (15 & v) == 0; }

// =====================================================================================================================
// to_planar
// =====================================================================================================================

/// y216_to_p010le, to_planar.c:164-200.  Y216 = Y0 Cb Y1 Cr as 16-bit words, copied verbatim; chroma from the even rows only.
/// Odd width: the even row still emits Cb AND Cr of the last pixel (so the chroma row holds width + 1 samples).
/// The reference never re-seeks its luma pointer for the odd row of a pair (:187-197): that row lands directly behind the even
/// row's `width` samples, not at the next out_linesize[0] - identical for a tight plane, reproduced for a padded one.
struct op_y216_p010 {
        const uint8_t *in;
        long in_ls;
        uint8_t *oy, *oc;
        long ls_y, ls_c;
        int width, height, units, rows;
        bool vec;
        __device__ __forceinline__ void run(int u, int pr) const
        {
                const int x0 = 4 * u;
                const bool second = 2 * pr + 1 < height;
                const uint16_t *s0 = (const uint16_t *) (in + (long) 2 * pr * in_ls) + 2 * x0;
                const uint16_t *s1 = (const uint16_t *) (in + (long) (2 * pr + 1) * in_ls) + 2 * x0;
                uint16_t *y0 = (uint16_t *) (oy + (long) 2 * pr * ls_y) + x0, *y1 = y0 + width;
                uint16_t *c = (uint16_t *) (oc + (long) pr * ls_c) + x0;
                const bool full = vec && x0 + 4 <= width;
                if (full) {
                        const uint4 a = ldv<uint4>(s0);
                        stv(y0, make_uint2(prmt(a.x, a.y, 0x5410), prmt(a.z, a.w, 0x5410)));
                        stv(c, make_uint2(prmt(a.x, a.y, 0x7632), prmt(a.z, a.w, 0x7632)));
                }
                if (full && second && !(width & 3)) {
                        const uint4 b = ldv<uint4>(s1);
                        stv(y1, make_uint2(prmt(b.x, b.y, 0x5410), prmt(b.z, b.w, 0x5410)));
                }
                const int cw = (width + 1) & ~1;
                for (int k = 0; k < 4; ++k) {
                        const int x = x0 + k;
                        if (x < width && !full) {
                                y0[k] = s0[2 * k];
                        }
                        if (x < width && second && !(full && !(width & 3))) {
                                y1[k] = s1[2 * k];
                        }
                        if (x < cw && !full) {
                                c[k] = s0[2 * k + 1];
                        }
                }
        }
};

/// uyvy_to_nv12 (to_planar.c:207-302) and uyvy_to_i420 (:343-378).  Chroma = mean of the two rows.  nv12: the reference's SSE3 loop
/// (x < width - 15, _mm_avg_epu8 = round half up) and its scalar tail ((a + b) / 2, truncation) DISAGREE; the build that is the
/// contract (-msse4.1) therefore rounds up for x < 16 * (width / 16) and truncates beyond.  i420 rounds up everywhere.
template <bool I420>
struct op_uyvy_420 {
        const uint8_t *in;
        long in_ls;
        uint8_t *oy, *o1, *o2;
        long ls_y, ls_1, ls_2;
        int width, height, units, rows, sse_end;
        bool vec;
        __device__ __forceinline__ void run(int u, int pr) const
        {
                const int x0 = 8 * u, y = 2 * pr;
                const bool single = y == height - 1;  // :226-229 / :358-361: the last row pairs with itself
                const uint8_t *s0 = in + (long) y * in_ls + 2 * x0, *s1 = single ? s0 : s0 + in_ls;
                uint8_t *y0 = oy + (long) y * ls_y + x0, *y1 = y0 + ls_y;
                const bool up = I420 || x0 < sse_end;
                if (vec && x0 + 8 <= width) {
                        const uint4 a = ldv<uint4>(s0), b = single ? a : ldv<uint4>(s1);
                        stv(y0, make_uint2(prmt(a.x, a.y, 0x7531), prmt(a.z, a.w, 0x7531)));
                        if (!single) {
                                stv(y1, make_uint2(prmt(b.x, b.y, 0x7531), prmt(b.z, b.w, 0x7531)));
                        }
                        const uint32_t ca0 = prmt(a.x, a.y, 0x6420), ca1 = prmt(a.z, a.w, 0x6420);  // Cb Cr Cb Cr
                        const uint32_t cb0 = prmt(b.x, b.y, 0x6420), cb1 = prmt(b.z, b.w, 0x6420);
                        const uint32_t m0 = up ? __vavgu4(ca0, cb0) : __vhaddu4(ca0, cb0), m1 = up ? __vavgu4(ca1, cb1) : __vhaddu4(ca1, cb1);
                        if (I420) {
                                stv(o1 + (long) pr * ls_1 + x0 / 2, prmt(m0, m1, 0x6420));
                                stv(o2 + (long) pr * ls_2 + x0 / 2, prmt(m0, m1, 0x7531));
                        } else {
                                stv(o1 + (long) pr * ls_1 + x0, make_uint2(m0, m1));
                        }
                        return;
                }
                for (int k = 0; k < 8; k += 2) {
                        const int x = x0 + k;
                        if (x >= width) {
                                break;
                        }
                        const int r = up ? 1 : 0;
                        const uint8_t cb = (uint8_t) ((s0[2 * k] + s1[2 * k] + r) / 2), cr = (uint8_t) ((s0[2 * k + 2] + s1[2 * k + 2] + r) / 2);
                        if (I420) {
                                o1[(long) pr * ls_1 + x / 2] = cb, o2[(long) pr * ls_2 + x / 2] = cr;
                        } else {
                                o1[(long) pr * ls_1 + x] = cb, o1[(long) pr * ls_1 + x + 1] = cr;
                        }
                        y0[k] = s0[2 * k + 1];
                        if (!single) {
                                y1[k] = s1[2 * k + 1];
                        }
                        if (x + 1 < width) {  // the odd-width tail drops the second luma (:295-300 / :371-376)
                                y0[k + 1] = s0[2 * k + 3];
                                if (!single) {
                                        y1[k + 1] = s1[2 * k + 3];
                                }
                        }
                }
        }
};

/// rgba_to_bgra, to_planar.c:304-319
struct op_rgba_bgra {
        const uint8_t *in;
        long in_ls;
        uint8_t *out;
        long ls;
        int width, height, units, rows;
        bool vec;
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u;
                const uint8_t *s = in + (long) row * in_ls + 4 * x0;
                uint8_t *d = out + (long) row * ls + 4 * x0;
                if (vec && x0 + 4 <= width) {
                        const uint4 a = ldv<uint4>(s);
                        stv(d, make_uint4(prmt(a.x, 0, 0x3012), prmt(a.y, 0, 0x3012), prmt(a.z, 0, 0x3012), prmt(a.w, 0, 0x3012)));
                        return;
                }
                for (int k = 0; k < 4 && x0 + k < width; ++k) {
                        d[4 * k] = s[4 * k + 2], d[4 * k + 1] = s[4 * k + 1], d[4 * k + 2] = s[4 * k], d[4 * k + 3] = s[4 * k + 3];
                }
        }
};

/// vuya_to_i444, to_planar.c:321-337
struct op_vuya_i444 {
        const uint8_t *in;
        long in_ls;
        uint8_t *o[3];  // y, u, v
        long ls[3];
        int width, height, units, rows;
        bool vec;
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u;
                const uint8_t *s = in + (long) row * in_ls + 4 * x0;
                if (vec && x0 + 4 <= width) {
                        const uint4 a = ldv<uint4>(s);
                        const uint32_t lo = prmt(a.x, a.y, 0x6240), hi = prmt(a.z, a.w, 0x6240);  // V0 V1 Y0 Y1
                        stv(o[2] + (long) row * ls[2] + x0, prmt(lo, hi, 0x5410));
                        stv(o[0] + (long) row * ls[0] + x0, prmt(lo, hi, 0x7632));
                        stv(o[1] + (long) row * ls[1] + x0, prmt(prmt(a.x, a.y, 0x0051), prmt(a.z, a.w, 0x0051), 0x5410));
                        return;
                }
                for (int k = 0; k < 4 && x0 + k < width; ++k) {
                        o[2][(long) row * ls[2] + x0 + k] = s[4 * k], o[1][(long) row * ls[1] + x0 + k] = s[4 * k + 1], o[0][(long) row * ls[0] + x0 + k] = s[4 * k + 2];
                }
        }
};

// R12L: 8 px x 3 x 12 bit = 36 bytes; component k of a group sits at bit 12k (little endian)
__device__ __forceinline__ uint32_t r12_get(const uint32_t *w, int k)
{
        const int off = 12 * k, wi = off >> 5, sh = off & 31;
        return sh <= 20 ? (w[wi] >> sh) & 0xfffu : ((w[wi] >> sh) | (w[wi + 1] << (32 - sh))) & 0xfffu;
}

/// r12l_to_gbrpXXle, to_planar.c:381-481 (gbrp12le / gbrp16le / rgbp12le = plane order + depth).  The reference converts whole
/// groups, i.e. writes up to 7 samples past `width`; rows run concurrently here, so every row but the last stops at its linesize
/// (the next row would overwrite the spill anyway), the last row spills exactly like the reference.
struct op_r12l_gbrp {
        const uint8_t *in;
        long in_ls;
        uint8_t *o[3];  // r, g, b
        long ls[3];
        int width, height, units, rows, shift;
        bool vec, in4;
        __device__ __forceinline__ void run(int u, int row) const
        {
                uint32_t w[9];
                const uint8_t *s = in + (long) row * in_ls + 36L * u;
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                        w[i] = in4 ? ldv<uint32_t>(s + 4 * i) : (uint32_t) s[4 * i] | (uint32_t) s[4 * i + 1] << 8 | (uint32_t) s[4 * i + 2] << 16 | (uint32_t) s[4 * i + 3] << 24;
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        uint32_t v[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                v[i] = (r12_get(w, 3 * i + c) << shift) & 0xffffu;
                        }
                        uint16_t *d = (uint16_t *) (o[c] + (long) row * ls[c]) + 8 * u;
                        const int lim = row == height - 1 ? 8 * units : min(8 * units, (int) (ls[c] / 2));
                        if (vec && 8 * u + 8 <= lim) {
                                stv(d, make_uint4(v[0] | v[1] << 16, v[2] | v[3] << 16, v[4] | v[5] << 16, v[6] | v[7] << 16));
                        } else {
#pragma unroll
                                for (int i = 0; i < 8; ++i) {
                                        if (8 * u + i < lim) {
                                                d[i] = (uint16_t) v[i];
                                        }
                                }
                        }
                }
        }
};

// =====================================================================================================================
// from_planar
// =====================================================================================================================
struct fp_args {
        uint8_t *out;
        long pitch;
        const uint8_t *in[4];
        long ls[4];
        int width, height, units, rows, depth;
        int rs, gs, bs;
        bool vec;
};

/// 4 consecutive 16-bit samples of a plane row starting at sample x0 (zero beyond `width`)
__device__ __forceinline__ void load4x16(const uint8_t *row, int x0, int width, bool vec, uint32_t *v)
{
        const uint16_t *p = (const uint16_t *) row + x0;
        if (vec && x0 + 4 <= width) {
                const uint2 a = ldv<uint2>(p);
                v[0] = a.x & 0xffffu, v[1] = a.x >> 16, v[2] = a.y & 0xffffu, v[3] = a.y >> 16;
        } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        v[k] = x0 + k < width ? ldv<uint16_t>(p + k) : 0u;
                }
        }
}
/// 4 consecutive 8-bit samples
__device__ __forceinline__ void load4x8(const uint8_t *row, int x0, int width, bool vec, uint32_t *v)
{
        if (vec && x0 + 4 <= width) {
                const uint32_t a = ldv<uint32_t>(row + x0);
                v[0] = a & 0xffu, v[1] = (a >> 8) & 0xffu, v[2] = (a >> 16) & 0xffu, v[3] = a >> 24;
        } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        v[k] = x0 + k < width ? ldv<uint8_t>(row + x0 + k) : 0u;
                }
        }
}
/// store n <= N bytes of words[] (vector store when whole and aligned)
template <int NW>
__device__ __forceinline__ void store_bytes(uint8_t *d, const uint32_t *w, int nbytes, bool vec)
{
        if (vec && nbytes == 4 * NW) {
                if constexpr (NW % 4 == 0) {
#pragma unroll
                        for (int i = 0; i < NW / 4; ++i) {
                                stv(d + 16 * i, make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]));
                        }
                } else if constexpr (NW % 2 == 0) {
#pragma unroll
                        for (int i = 0; i < NW / 2; ++i) {
                                stv(d + 8 * i, make_uint2(w[2 * i], w[2 * i + 1]));
                        }
                } else {
#pragma unroll
                        for (int i = 0; i < NW; ++i) {
                                stv(d + 4 * i, w[i]);
                        }
                }
                return;
        }
#pragma unroll
        for (int i = 0; i < 4 * NW; ++i) {
                if (i < nbytes) {
                        d[i] = (uint8_t) (w[i >> 2] >> (8 * (i & 3)));
                }
        }
}

/// gbrpXXle_to_r12l, from_planar.c:61-129 (R, G, B = planes in[0..2] after the caller's index mapping).  The reference stages a
/// partial last group through an UNINITIALISED temporary (:78-86): bytes that depend on samples beyond `width` are indeterminate
/// there; here those samples read as zero.
struct op_gbrp_r12l : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                uint32_t f[24];  // r0 g0 b0 r1 ...
                const int x0 = 8 * u, sh = depth - 12;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        uint32_t v[8];
                        const uint8_t *r = in[c] + (long) row * ls[c];
                        load4x16(r, x0, width, vec, v), load4x16(r, x0 + 4, width, vec, v + 4);
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                f[3 * i + c] = v[i] >> sh;
                        }
                }
                uint32_t w[9] = { 0, 0, 0, 0, 0, 0, 0, 0, 0 };
#pragma unroll
                for (int p = 0; p < 12; ++p) {  // fields 2p (byte aligned) and 2p + 1 make 3 bytes, each truncated like the reference's stores
                        const uint32_t e = f[2 * p], o = f[2 * p + 1];
                        const uint32_t t = (e & 0xffu) | ((((o & 0xfu) << 4) | (e >> 8)) & 0xffu) << 8 | ((o >> 4) & 0xffu) << 16;
                        const int bo = 3 * p, wi = bo >> 2, bs8 = 8 * (bo & 3);
                        w[wi] |= t << bs8;
                        if (bs8 > 8) {
                                w[wi + 1] |= t >> (32 - bs8);
                        }
                }
                store_bytes<9>(out + (long) row * pitch + 36L * u, w, 36, vec);
        }
};

/// rgbpXXle_to_rg48_int, from_planar.c:157-177
struct op_rgbp_rg48 : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u, sh = 16 - depth;
                uint32_t v[3][4];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        load4x16(in[c] + (long) row * ls[c], x0, width, vec, v[c]);
                }
                uint32_t s[12], w[6];
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        s[i] = (v[i % 3][i / 3] << sh) & 0xffffu;
                }
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                        w[i] = s[2 * i] | s[2 * i + 1] << 16;
                }
                store_bytes<6>(out + (long) row * pitch + 6L * x0, w, 6 * min(4, width - x0), vec);
        }
};

/// gbrpXXle_to_r10k, from_planar.c:203-226 (each byte truncated like the reference's uint8 stores)
struct op_gbrp_r10k : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u, d = depth;
                uint32_t v[3][4], w[4];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        load4x16(in[c] + (long) row * ls[c], x0, width, vec, v[c]);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        const uint32_t r = v[0][k], g = v[1][k], b = v[2][k];
                        w[k] = ((r >> (d - 8)) & 0xffu) | (((((r >> (d - 10)) & 0x3u) << 6) | (g >> (d - 6))) & 0xffu) << 8 |
                               (((((g >> (d - 10)) & 0xfu) << 4) | (b >> (d - 4))) & 0xffu) << 16 | (((((b >> (d - 10)) & 0x3fu) << 2) | 0x3u) & 0xffu) << 24;
                }
                store_bytes<4>(out + (long) row * pitch + 4L * x0, w, 4 * min(4, width - x0), vec);
        }
};

/// yuv422p10le_to_v210, from_planar.c:295-333: whole 6-pixel groups only (x < width / 6); samples are OR-ed unmasked
struct op_yuv422p10_v210 : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const uint16_t *y = (const uint16_t *) (in[0] + (long) row * ls[0]) + 6 * u;
                const uint16_t *cb = (const uint16_t *) (in[1] + (long) row * ls[1]) + 3 * u, *cr = (const uint16_t *) (in[2] + (long) row * ls[2]) + 3 * u;
                uint32_t Y[6], B[3], R[3];
                if (vec) {  // 12 luma bytes of a group start 4-byte aligned
                        const uint32_t a = ldv<uint32_t>(y), b = ldv<uint32_t>(y + 2), c = ldv<uint32_t>(y + 4);
                        Y[0] = a & 0xffffu, Y[1] = a >> 16, Y[2] = b & 0xffffu, Y[3] = b >> 16, Y[4] = c & 0xffffu, Y[5] = c >> 16;
                } else {
#pragma unroll
                        for (int i = 0; i < 6; ++i) {
                                Y[i] = ldv<uint16_t>(y + i);
                        }
                }
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                        B[i] = ldv<uint16_t>(cb + i), R[i] = ldv<uint16_t>(cr + i);
                }
                uint32_t w[4] = { B[0] | Y[0] << 10 | R[0] << 20, Y[1] | B[1] << 10 | Y[2] << 20, R[1] | Y[3] << 10 | B[2] << 20, Y[4] | R[2] << 10 | Y[5] << 20 };
                store_bytes<4>(out + (long) row * pitch + 16L * u, w, 16, vec);
        }
};

/// gbrap_to_rgb_rgba, from_planar.c:335-354: 8-bit planes; every plane is indexed with in_linesize[0] (:347); A = 3 or 4 bytes out
template <int A>
struct op_gbrap_rgbx : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u;
                uint32_t v[4][4];
#pragma unroll
                for (int c = 0; c < A; ++c) {
                        load4x8(in[c] + (long) row * ls[0], x0, width, vec, v[c]);
                }
                uint32_t b[4 * A], w[A];
#pragma unroll
                for (int i = 0; i < 4 * A; ++i) {
                        b[i] = v[i % A][i / A];
                }
#pragma unroll
                for (int i = 0; i < A; ++i) {
                        w[i] = b[4 * i] | b[4 * i + 1] << 8 | b[4 * i + 2] << 16 | b[4 * i + 3] << 24;
                }
                store_bytes<A>(out + (long) row * pitch + (long) A * x0, w, A * min(4, width - x0), vec);
        }
};

/// yuv422p_to_uyvy_yuyv, from_planar.c:392-417 (8 bit, width / 2 pairs) and yuv422pXXle_to_uyvy_int, :425-441 (16-bit samples >> depth - 8)
template <bool YUYV, bool WIDE>
struct op_yuv422p_packed : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u, w2 = width & ~1;  // an odd last pixel is not converted
                if (x0 >= w2) {  // the unit holds only the odd last pixel: nothing to write.  (Clamping the byte count at 0 instead, as
                        return;      // max(0, min(4, w2 - x0)), made ptxas 12.9 for sm_90a take the 8-byte vector store for a partial unit.)
                }
                uint32_t y[4], cb[4], cr[4];
                if (WIDE) {
                        load4x16(in[0] + (long) row * ls[0], x0, w2, vec, y);
                        const uint16_t *b = (const uint16_t *) (in[1] + (long) row * ls[1]) + x0 / 2, *r = (const uint16_t *) (in[2] + (long) row * ls[2]) + x0 / 2;
#pragma unroll
                        for (int k = 0; k < 2; ++k) {
                                const bool ok = x0 + 2 * k < w2;
                                cb[k] = ok ? ldv<uint16_t>(b + k) >> (depth - 8) : 0u, cr[k] = ok ? ldv<uint16_t>(r + k) >> (depth - 8) : 0u;
                                y[2 * k] >>= depth - 8, y[2 * k + 1] >>= depth - 8;
                        }
                } else {
                        load4x8(in[0] + (long) row * ls[0], x0, w2, vec, y);
#pragma unroll
                        for (int k = 0; k < 2; ++k) {
                                const bool ok = x0 + 2 * k < w2;
                                cb[k] = ok ? ldv<uint8_t>(in[1] + (long) row * ls[1] + x0 / 2 + k) : 0u, cr[k] = ok ? ldv<uint8_t>(in[2] + (long) row * ls[2] + x0 / 2 + k) : 0u;
                        }
                }
                uint32_t w[2];
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                        const uint32_t a = y[2 * k] & 0xffu, c = y[2 * k + 1] & 0xffu, bb = cb[k] & 0xffu, rr = cr[k] & 0xffu;
                        w[k] = YUYV ? (a | bb << 8 | c << 16 | rr << 24) : (bb | a << 8 | rr << 16 | c << 24);
                }
                store_bytes<2>(out + (long) row * pitch + 2L * x0, w, 2 * min(4, w2 - x0), vec);
        }
};

/// gbrpXXle_to_rgb, from_planar.c:465-484 (planes in[] = R, G, B after mapping)
struct op_gbrp_rgb : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u;
                uint32_t v[3][4];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        load4x16(in[c] + (long) row * ls[c], x0, width, vec, v[c]);
                }
                uint32_t b[12], w[3];
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        b[i] = (v[i % 3][i / 3] >> (depth - 8)) & 0xffu;
                }
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                        w[i] = b[4 * i] | b[4 * i + 1] << 8 | b[4 * i + 2] << 16 | b[4 * i + 3] << 24;
                }
                store_bytes<3>(out + (long) row * pitch + 3L * x0, w, 3 * min(4, width - x0), vec);
        }
};

/// gbrpXXle_to_rgba, from_planar.c:486-517: planes are G, B, R (:500-502); components are shifted unmasked
struct op_gbrp_rgba : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u;
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << rs) ^ (0xFFu << gs) ^ (0xFFu << bs);
                uint32_t v[3][4], w[4];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        load4x16(in[c] + (long) row * ls[c], x0, width, vec, v[c]);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        w[k] = amask | (v[2][k] >> (depth - 8)) << rs | (v[0][k] >> (depth - 8)) << gs | (v[1][k] >> (depth - 8)) << bs;
                }
                store_bytes<4>(out + (long) row * pitch + 4L * x0, w, 4 * min(4, width - x0), vec);
        }
};

/// yuv444p_to_vuya, from_planar.c:565-580
struct op_yuv444p_vuya : fp_args {
        __device__ __forceinline__ void run(int u, int row) const
        {
                const int x0 = 4 * u;
                uint32_t v[3][4], w[4];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                        load4x8(in[c] + (long) row * ls[c], x0, width, vec, v[c]);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        w[k] = v[2][k] | v[1][k] << 8 | v[0][k] << 16 | 0xFF000000u;
                }
                store_bytes<4>(out + (long) row * pitch + 4L * x0, w, 4 * min(4, width - x0), vec);
        }
};

/// yuv420p_to_uyvy, from_planar.c:582-683: a chroma row serves two luma rows; odd width: the last pixel is Cb Y Cr 0 (:670-680);
/// odd height: the last row pairs with itself.  (The reference's SSE3 loop bound `width - 15` is unsigned: widths below 15 are
/// undefined there.)
struct op_yuv420p_uyvy : fp_args {
        __device__ __forceinline__ void run(int u, int pr) const
        {
                const int x0 = 4 * u;
                const int r0 = 2 * pr, r1 = min(2 * pr + 1, height - 1);
                uint32_t ya[4], yb[4], cb[2], cr[2];
                load4x8(in[0] + (long) r0 * ls[0], x0, width, vec, ya);
                load4x8(in[0] + (long) r1 * ls[0], x0, width, vec, yb);
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                        const bool ok = x0 + 2 * k < width;
                        cb[k] = ok ? ldv<uint8_t>(in[1] + (long) pr * ls[1] + x0 / 2 + k) : 0u, cr[k] = ok ? ldv<uint8_t>(in[2] + (long) pr * ls[2] + x0 / 2 + k) : 0u;
                }
                uint32_t wa[2], wb[2];
#pragma unroll
                for (int k = 0; k < 2; ++k) {  // load4x8 returns 0 beyond width = the reference's explicit 0 for the missing luma
                        wa[k] = cb[k] | ya[2 * k] << 8 | cr[k] << 16 | ya[2 * k + 1] << 24;
                        wb[k] = cb[k] | yb[2 * k] << 8 | cr[k] << 16 | yb[2 * k + 1] << 24;
                }
                const int nb = 2 * min(4, ((width + 1) & ~1) - x0);
                store_bytes<2>(out + (long) r0 * pitch + 2L * x0, wa, nb, vec);
                if (r1 != r0) {
                        store_bytes<2>(out + (long) r1 * pitch + 2L * x0, wb, nb, vec);
                }
        }
};

static bool fp_fill(fp_args &a, const struct ugb200_from_planar_data *d, int nplanes, const int *map, int px_per_unit, int rows)
{
        if (d == nullptr || d->out_data == nullptr || d->width <= 0 || d->height <= 0) {
                return false;
        }
        a.out = d->out_data, a.pitch = d->out_pitch;
        bool vec = al16(d->out_data) && al16(d->out_pitch);
        for (int i = 0; i < 4; ++i) {
                a.in[i] = nullptr, a.ls[i] = 0;
        }
        for (int i = 0; i < nplanes; ++i) {
                a.in[i] = d->in_data[map[i]], a.ls[i] = d->in_linesize[map[i]];
                if (a.in[i] == nullptr) {
                        return false;
                }
                vec = vec && al16(a.in[i]) && al16((unsigned) a.ls[i]);
        }
        a.width = d->width, a.height = d->height, a.units = (d->width + px_per_unit - 1) / px_per_unit, a.rows = rows;
        a.depth = d->in_depth, a.rs = d->rgb_shift[0], a.gs = d->rgb_shift[1], a.bs = d->rgb_shift[2];
        a.vec = vec;
        return true;
}

static const int kGBR[3] = { 2, 0, 1 };  // R, G, B planes of a GBR(A) frame
static const int kRGB[3] = { 0, 1, 2 };
static const int kGBRA[4] = { 2, 0, 1, 3 };
static const int kIdent[4] = { 0, 1, 2, 3 };

template <class Op>
static int run_fp(const struct ugb200_from_planar_data *d, int nplanes, const int *map, int px, int depth, bool pairs, cudaStream_t s)
{
        Op op;
        if (!fp_fill(op, d, nplanes, map, px, pairs ? (d ? (d->height + 1) / 2 : 0) : (d ? d->height : 0))) {
                return -1;
        }
        if (depth != 0) {
                op.depth = depth;
        }
        return launch_planar(op, s);
}

}  // namespace ugb

using namespace ugb;

// ---- to_planar entry points ----------------------------------------------------------------------------------------------
static bool tp_ok(const struct ugb200_to_planar_data *d, int planes)
{
        if (d == nullptr || d->in_data == nullptr || d->width <= 0 || d->height <= 0) {
                return false;
        }
        for (int i = 0; i < planes; ++i) {
                if (d->out_data[i] == nullptr) {
                        return false;
                }
        }
        return true;
}
static bool tp_vec(const struct ugb200_to_planar_data *d, int planes, long in_ls)
{
        bool v = al16(d->in_data) && !(in_ls & 15);
        for (int i = 0; i < planes; ++i) {
                v = v && al16(d->out_data[i]) && al16(d->out_linesize[i]);
        }
        return v;
}

extern "C" UGB_API int ugb200_y216_to_p010le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream)
{
        if (!tp_ok(d, 2)) {
                return -1;
        }
        const long in_ls = vc_linesize64(d->width, Y216);
        const op_y216_p010 op = { d->in_data, in_ls, d->out_data[0], d->out_data[1], d->out_linesize[0], d->out_linesize[1], d->width, d->height,
                                  (d->width + 1 + 3) / 4, (d->height + 1) / 2, tp_vec(d, 2, in_ls) };
        return launch_planar(op, (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_uyvy_to_nv12(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream)
{
        if (!tp_ok(d, 2)) {
                return -1;
        }
        const long in_ls = (long) d->width * 2;  // to_planar.c:215 (not vc_get_linesize)
        const op_uyvy_420<false> op = { d->in_data, in_ls, d->out_data[0], d->out_data[1], nullptr, d->out_linesize[0], d->out_linesize[1], 0, d->width, d->height,
                                        (d->width + 7) / 8, (d->height + 1) / 2, d->width / 16 * 16, tp_vec(d, 2, in_ls) };
        return launch_planar(op, (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_uyvy_to_i420(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream)
{
        if (!tp_ok(d, 3)) {
                return -1;
        }
        const long in_ls = vc_linesize64(d->width, UYVY);
        const op_uyvy_420<true> op = { d->in_data, in_ls, d->out_data[0], d->out_data[1], d->out_data[2], d->out_linesize[0], d->out_linesize[1], d->out_linesize[2],
                                       d->width, d->height, (d->width + 7) / 8, (d->height + 1) / 2, 0, tp_vec(d, 3, in_ls) };
        return launch_planar(op, (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_rgba_to_bgra(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream)
{
        if (!tp_ok(d, 1)) {
                return -1;
        }
        const long in_ls = (long) d->width * 4;
        const op_rgba_bgra op = { d->in_data, in_ls, d->out_data[0], d->out_linesize[0], d->width, d->height, (d->width + 3) / 4, d->height, tp_vec(d, 1, in_ls) };
        return launch_planar(op, (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_vuya_to_i444(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream)
{
        if (!tp_ok(d, 3)) {
                return -1;
        }
        const long in_ls = (long) d->width * 4;
        const op_vuya_i444 op = { d->in_data, in_ls, { d->out_data[0], d->out_data[1], d->out_data[2] }, { d->out_linesize[0], d->out_linesize[1], d->out_linesize[2] },
                                  d->width, d->height, (d->width + 3) / 4, d->height, tp_vec(d, 3, in_ls) };
        return launch_planar(op, (cudaStream_t) stream);
}

static int r12l_to_planes(const struct ugb200_to_planar_data *d, int depth, int rind, int gind, int bind, cuda_wrapper_stream_t stream)
{
        if (!tp_ok(d, 3) || (d->out_linesize[0] & 1) || (d->out_linesize[1] & 1) || (d->out_linesize[2] & 1)) {
                return -1;  // asserts of to_planar.c:385-388
        }
        const long in_ls = vc_linesize64(d->width, R12L);
        const op_r12l_gbrp op = { d->in_data, in_ls, { d->out_data[rind], d->out_data[gind], d->out_data[bind] },
                                  { d->out_linesize[rind], d->out_linesize[gind], d->out_linesize[bind] }, d->width, d->height, (d->width + 7) / 8, d->height, depth - 12,
                                  tp_vec(d, 3, 16), (3 & (size_t) d->in_data) == 0 };
        return launch_planar(op, (cudaStream_t) stream);
}
extern "C" UGB_API int ugb200_r12l_to_gbrp12le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t s) { return r12l_to_planes(d, 12, 2, 0, 1, s); }
extern "C" UGB_API int ugb200_r12l_to_gbrp16le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t s) { return r12l_to_planes(d, 16, 2, 0, 1, s); }
extern "C" UGB_API int ugb200_r12l_to_rgbp12le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t s) { return r12l_to_planes(d, 12, 0, 1, 2, s); }

// ---- from_planar entry points ----------------------------------------------------------------------------------------------
#define UGB_FP(name, OP, NPL, MAP, PX, DEPTH, PAIRS)                                                                                          \
        extern "C" UGB_API int ugb200_##name(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)                               \
        {                                                                                                                                    \
                return run_fp<OP>(d, NPL, MAP, PX, DEPTH, PAIRS, (cudaStream_t) s);                                                          \
        }
static bool depth_ok(const struct ugb200_from_planar_data *d, int lo) { return d != nullptr && d->in_depth >= lo && d->in_depth <= 16; }

UGB_FP(gbrap_to_rgb, op_gbrap_rgbx<3>, 3, kGBR, 4, 0, false)
UGB_FP(gbrap_to_rgba, op_gbrap_rgbx<4>, 4, kGBRA, 4, 0, false)
UGB_FP(gbrp10le_to_rgb, op_gbrp_rgb, 3, kGBR, 4, 10, false)
UGB_FP(gbrp12le_to_rgb, op_gbrp_rgb, 3, kGBR, 4, 12, false)
UGB_FP(gbrp16le_to_rgb, op_gbrp_rgb, 3, kGBR, 4, 16, false)
extern "C" UGB_API int ugb200_rgbpXX_to_rgb(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)  // from_planar.c:555-563
{
        if (d != nullptr && d->in_depth == 8) {
                return run_fp<op_gbrap_rgbx<3>>(d, 3, kRGB, 4, 0, false, (cudaStream_t) s);
        }
        return depth_ok(d, 9) ? run_fp<op_gbrp_rgb>(d, 3, kRGB, 4, 0, false, (cudaStream_t) s) : -1;
}
UGB_FP(gbrp10le_to_rgba, op_gbrp_rgba, 3, kIdent, 4, 10, false)
UGB_FP(gbrp12le_to_rgba, op_gbrp_rgba, 3, kIdent, 4, 12, false)
UGB_FP(gbrp16le_to_rgba, op_gbrp_rgba, 3, kIdent, 4, 16, false)
UGB_FP(gbrp10le_to_rg48, op_rgbp_rg48, 3, kGBR, 4, 10, false)
UGB_FP(gbrp12le_to_rg48, op_rgbp_rg48, 3, kGBR, 4, 12, false)
UGB_FP(gbrp16le_to_rg48, op_rgbp_rg48, 3, kGBR, 4, 16, false)
extern "C" UGB_API int ugb200_rgbpXXle_to_rg48(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)
{
        return depth_ok(d, 1) ? run_fp<op_rgbp_rg48>(d, 3, kRGB, 4, 0, false, (cudaStream_t) s) : -1;
}
UGB_FP(gbrp10le_to_r10k, op_gbrp_r10k, 3, kGBR, 4, 10, false)
UGB_FP(gbrp12le_to_r10k, op_gbrp_r10k, 3, kGBR, 4, 12, false)
UGB_FP(gbrp16le_to_r10k, op_gbrp_r10k, 3, kGBR, 4, 16, false)
extern "C" UGB_API int ugb200_rgbpXXle_to_r10k(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)
{
        return depth_ok(d, 10) ? run_fp<op_gbrp_r10k>(d, 3, kRGB, 4, 0, false, (cudaStream_t) s) : -1;
}
UGB_FP(gbrp12le_to_r12l, op_gbrp_r12l, 3, kGBR, 8, 12, false)
UGB_FP(gbrp16le_to_r12l, op_gbrp_r12l, 3, kGBR, 8, 16, false)
extern "C" UGB_API int ugb200_rgbpXXle_to_r12l(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)
{
        return depth_ok(d, 12) ? run_fp<op_gbrp_r12l>(d, 3, kRGB, 8, 0, false, (cudaStream_t) s) : -1;
}
UGB_FP(yuv444p_to_vuya, op_yuv444p_vuya, 3, kIdent, 4, 0, false)
UGB_FP(yuv420p_to_uyvy, op_yuv420p_uyvy, 3, kIdent, 4, 0, true)
using op_422p8_uyvy = op_yuv422p_packed<false, false>;
using op_422p8_yuyv = op_yuv422p_packed<true, false>;
using op_422p16_uyvy = op_yuv422p_packed<false, true>;
UGB_FP(yuv422p_to_uyvy, op_422p8_uyvy, 3, kIdent, 4, 0, false)
UGB_FP(yuv422p_to_yuyv, op_422p8_yuyv, 3, kIdent, 4, 0, false)
UGB_FP(yuv422p10le_to_uyvy, op_422p16_uyvy, 3, kIdent, 4, 10, false)
extern "C" UGB_API int ugb200_yuv422pXX_to_uyvy(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)  // from_planar.c:447-455
{
        if (d != nullptr && d->in_depth == 8) {
                return run_fp<op_422p8_uyvy>(d, 3, kIdent, 4, 0, false, (cudaStream_t) s);
        }
        return depth_ok(d, 9) ? run_fp<op_422p16_uyvy>(d, 3, kIdent, 4, 0, false, (cudaStream_t) s) : -1;
}
extern "C" UGB_API int ugb200_yuv422p10le_to_v210(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t s)
{
        op_yuv422p10_v210 op;
        if (!fp_fill(op, d, 3, kIdent, 6, d ? d->height : 0)) {
                return -1;
        }
        op.units = d->width / 6;  // from_planar.c:308: whole groups only
        op.vec = op.vec && !(3 & (size_t) d->out_data);
        return launch_planar(op, (cudaStream_t) s);
}

/// yuv420_to_i420, from_planar.c:368-390: three plane copies into one contiguous I420 buffer (out_pitch ignored)
extern "C" UGB_API int ugb200_yuv420_to_i420(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream)
{
        if (d == nullptr || d->out_data == nullptr || d->width <= 0 || d->height <= 0 || (d->width & 1) || (d->height & 1) || d->in_data[0] == nullptr ||
            d->in_data[1] == nullptr || d->in_data[2] == nullptr) {
                return -1;  // asserts at :371-372
        }
        cudaStream_t s = (cudaStream_t) stream;
        const size_t w = d->width, h = d->height;
        unsigned char *y = d->out_data, *u = y + w * h, *v = u + (w / 2) * (h / 2);
        if (cudaMemcpy2DAsync(y, w, d->in_data[0], d->in_linesize[0], w, h, cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
            cudaMemcpy2DAsync(u, w / 2, d->in_data[1], d->in_linesize[1], w / 2, h / 2, cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
            cudaMemcpy2DAsync(v, w / 2, d->in_data[2], d->in_linesize[2], w / 2, h / 2, cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
                return -2;
        }
        return 0;
}
