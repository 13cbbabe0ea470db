// The resize capture filter / postprocessor on the device (src/capture_filter/resize.c).  The reference resamples with
// OpenCV (resize_utils.cpp: cvtColor to RGB, then cv::resize), which is not in the reference tree and whose bytes
// depend on how it was built, so the resampling here follows an exact contract modelled on OpenCV's generic path
// (DESIGN.md §2 "Resize"; differences §8):
//
//   colour (8-bit YUV routes only), BT.601 limited range in Q20 as cvtColor applies it:
//     Yq = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128
//     R = sat8((Yq + 1673527 v + 2^19) >> 20), G = sat8((Yq - 852492 v - 409993 u + 2^19) >> 20),
//     B = sat8((Yq + 2116026 u + 2^19) >> 20)             (arithmetic shifts)
//     UYVY / YUYV: one chroma pair per two pixels; I420: chroma of (x / 2, y / 2).  RGBA drops alpha; RGB, RG48 as is.
//     Every source tap is converted, then filtered.
//   nearest: s = min(floor(d * (1 / inv_scale)), n - 1) in double, per axis.
//   linear, 8-bit: per column f = (float) ((dx + 0.5) * scale - 0.5), sx = floor(f), f -= sx; sx < 0 -> sx = 0, f = 0;
//     sx >= sw - 1 -> sx = sw - 1, f = 0; a0 = cvRound((1.0f - f) * 2048), a1 = cvRound(f * 2048).  Rows the same,
//     but f is kept and sy, sy + 1 are clamped into [0, sh - 1] (b0, b1).  H = a0 S[sx] + a1 S[sx + 1] (source column
//     clamped), result sat8((b0 H0 + b1 H1 + 2^21) >> 22).
//   linear, RG48: float weights 1.0f - f, f; H = fl(fl(S0 a0) + fl(S1 a1)), V = fl(fl(H0 b0) + fl(H1 b1)), no FMA;
//     result sat16(round-half-even(V)).
//   area, integer k x l downscale: the box [dx k, dx k + k) x [dy l, dy l + l), floor((sum + k l / 2) / (k l)).
// Handles from ugb200_cf_resize_create2 also build (the tables' formulas in host/resize_tables.h):
//   cubic (K = 4), lanczos4 (K = 8): taps clamp(sx - K / 2 + 1 + j), f as linear but never zeroed.  8-bit: Q11 weights,
//     H = sum a_j S_j, V = sum b_k H_k exact, sat8((V + 2^21) >> 22).  RG48: float weights, H and V summed left to
//     right, each product and sum one float operation; sat16(round-half-even(V)).
//   area, other downscales (both scales >= 1): computeResizeAreaTab's entries per axis; per channel in float,
//     buf = sum over x entries of fl(S alpha) in order, sum = beta_0 buf_0 + beta_1 buf_1 ..., sat(round-half-even(sum)).
//   area, either scale < 1: linear with area-mode positions (linear_area_table).
//
// The column and row tables (host/resize_tables.cpp) are computed once per input descriptor and cached in the handle.
// One fused kernel per (source layout, algorithm) reads the taps, converts them in registers, resamples, and writes
// the letterbox margins as zeros: every output byte is written by exactly one thread of one launch.  A thread stores a
// run of 24 output bytes along x (8 RGB or 4 RG48 pixels), as 8-byte words where the row allows.  Codecs
// outside the resize set are converted to their route codec first (ugb200_pixfmt_convert into the handle's staging
// frame, same stream), as resize.c's parallel_pix_conv does.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "../../include/ugb200.h"
#include "filter_args.h"
#include "host/resize_tables.h"
#include "host/video_codec.h"

namespace ugb_resize {

constexpr int kThreads = 128;

enum Layout { L_RGB, L_RGBA, L_UYVY, L_YUYV, L_I420, L_RG48 };
// cv::INTER_* values, then the two area forms that handles from ugb200_cf_resize_create2 add
enum Algo { A_NEAREST = 0, A_LINEAR = 1, A_CUBIC = 2, A_AREA = 3, A_LANCZOS4 = 4, A_AREA_ANY = 5, A_AREA_UP = 6 };

struct Args {
        const uint8_t *src;    // packed rows, or the I420 Y plane
        const uint8_t *u, *v;  // I420 chroma planes
        long src_pitch;        // bytes per source row (Y plane for I420)
        int cpitch;            // I420 chroma bytes per row
        uint8_t *dst;
        long dst_pitch;
        int dw, dh;            // output frame
        int rx, ry, rw, rh;    // resampled rectangle; the rest of the frame is 0
        const Tap2 *xt, *yt;   // rw column and rh row entries (nearest, linear)
        int kx, ky;            // area box
        bool div32;            // area: every box sum plus kx * ky / 2 fits in 32 bits (kx * ky <= 65535)
        double inv_n;          // area: 1 / (kx * ky)
};

// the algorithms of ugb200_cf_resize_create2 handles (a struct of their own, so the kernels above keep their code)
struct ArgsX : Args {
        int sw, sh;              // source frame
        const int32_t *xk, *yk;  // cubic, lanczos4: K + 1 int32 per column / row (first tap, K weights)
        bool v32;                // cubic, lanczos4, 8-bit: every V + 2^21 fits in an int (bound from the tables)
        int ty;                  // cubic, lanczos4: output rows per tile
        const int32_t *axh, *ayh, *axe, *aye;  // other area: (offset, count) per column / row; (index, alpha) entries
};

__device__ __forceinline__ int sat8(int v) { return min(max(v, 0), 255); }

__device__ __forceinline__ void yuv_to_rgb(int Y, int U, int V, int *c)
{
        const int yq = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128;
        c[0] = sat8((yq + 1673527 * v + (1 << 19)) >> 20);
        c[1] = sat8((yq - 852492 * v - 409993 * u + (1 << 19)) >> 20);
        c[2] = sat8((yq + 2116026 * u + (1 << 19)) >> 20);
}

struct Row {
        const uint8_t *p, *u, *v;
};

template <int L>
__device__ __forceinline__ Row row(const Args &a, int sy)
{
        Row r{ a.src + sy * a.src_pitch, nullptr, nullptr };
        if constexpr (L == L_I420) {
                r.u = a.u + (long) (sy >> 1) * a.cpitch;
                r.v = a.v + (long) (sy >> 1) * a.cpitch;
        }
        return r;
}

// source pixel x of a row, as RGB (8 or 16 bits per channel)
template <int L>
__device__ __forceinline__ void tap(const Row &r, int x, int *c)
{
        if constexpr (L == L_RGB || L == L_RGBA) {
                const uint8_t *p = r.p + (L == L_RGB ? 3 : 4) * (long) x;
                c[0] = __ldg(p), c[1] = __ldg(p + 1), c[2] = __ldg(p + 2);
        } else if constexpr (L == L_UYVY) {  // U Y0 V Y1
                const uint8_t *q = r.p + 4 * (long) (x >> 1);
                yuv_to_rgb(__ldg(q + 1 + 2 * (x & 1)), __ldg(q), __ldg(q + 2), c);
        } else if constexpr (L == L_YUYV) {  // Y0 U Y1 V
                const uint8_t *q = r.p + 4 * (long) (x >> 1);
                yuv_to_rgb(__ldg(q + 2 * (x & 1)), __ldg(q + 1), __ldg(q + 3), c);
        } else if constexpr (L == L_I420) {
                yuv_to_rgb(__ldg(r.p + x), __ldg(r.u + (x >> 1)), __ldg(r.v + (x >> 1)), c);
        } else {  // RG48, little-endian 16-bit R, G, B
                const uint8_t *p = r.p + 6 * (long) x;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                        c[k] = __ldg(p + 2 * k) | __ldg(p + 2 * k + 1) << 8;
                }
        }
}

// one output pixel of the rectangle at (x, y) relative to it
template <int L, int A, typename Params>
__device__ __forceinline__ void pixel(const Params &a, int x, int y, int *out)
{
        constexpr bool W16 = L == L_RG48;
        if constexpr (A == A_NEAREST) {
                tap<L>(row<L>(a, a.yt[y].s0), a.xt[x].s0, out);
        } else if constexpr (A == A_LINEAR) {
                const Tap2 tx = a.xt[x], ty = a.yt[y];
                int t[4][3];
                const Row r0 = row<L>(a, ty.s0), r1 = row<L>(a, ty.s1);
                tap<L>(r0, tx.s0, t[0]);
                tap<L>(r0, tx.s1, t[1]);
                tap<L>(r1, tx.s0, t[2]);
                tap<L>(r1, tx.s1, t[3]);
                if constexpr (W16) {
                        const float a0 = __int_as_float(tx.w0), a1 = __int_as_float(tx.w1);
                        const float b0 = __int_as_float(ty.w0), b1 = __int_as_float(ty.w1);
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                                const float h0 = __fadd_rn(__fmul_rn((float) t[0][k], a0), __fmul_rn((float) t[1][k], a1));
                                const float h1 = __fadd_rn(__fmul_rn((float) t[2][k], a0), __fmul_rn((float) t[3][k], a1));
                                const float v = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
                                out[k] = min(max(__float2int_rn(v), 0), 65535);
                        }
                } else {
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                                const int h0 = tx.w0 * t[0][k] + tx.w1 * t[1][k], h1 = tx.w0 * t[2][k] + tx.w1 * t[3][k];
                                out[k] = sat8((ty.w0 * h0 + ty.w1 * h1 + (1 << 21)) >> 22);
                        }
                }
        } else if constexpr (A == A_AREA_ANY) {  // computeResizeAreaTab entries, float, in the contract's order
                const int2 hx = reinterpret_cast<const int2 *>(a.axh)[x], hy = reinterpret_cast<const int2 *>(a.ayh)[y];
                const int2 *ex = reinterpret_cast<const int2 *>(a.axe) + hx.x, *ey = reinterpret_cast<const int2 *>(a.aye) + hy.x;
                float sum[3];
                for (int j = 0; j < hy.y; ++j) {
                        const int2 e = ey[j];
                        const Row r = row<L>(a, e.x);
                        float buf[3] = { 0.f, 0.f, 0.f };
                        for (int i = 0; i < hx.y; ++i) {
                                const int2 t = ex[i];
                                int c[3];
                                tap<L>(r, t.x, c);
#pragma unroll
                                for (int k = 0; k < 3; ++k) {
                                        buf[k] = __fadd_rn(buf[k], __fmul_rn((float) c[k], __int_as_float(t.y)));
                                }
                        }
                        const float beta = __int_as_float(e.y);
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                                sum[k] = j == 0 ? __fmul_rn(beta, buf[k]) : __fadd_rn(sum[k], __fmul_rn(beta, buf[k]));
                        }
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                        out[k] = min(max(__float2int_rn(sum[k]), 0), W16 ? 65535 : 255);
                }
        } else if (a.div32) {  // area, every box sum below 2^32 (so every box row too): 32-bit sums and division
                unsigned s[3] = { 0, 0, 0 };
                for (int j = 0; j < a.ky; ++j) {
                        const Row r = row<L>(a, y * a.ky + j);
                        for (int i = 0; i < a.kx; ++i) {
                                int c[3];
                                tap<L>(r, x * a.kx + i, c);
                                s[0] += c[0], s[1] += c[1], s[2] += c[2];
                        }
                }
                const unsigned n = (unsigned) a.kx * a.ky;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                        out[k] = (int) ((s[k] + n / 2) / n);
                }
        } else {  // area, larger boxes: 64-bit sums (below 2^16 * kx * ky < 2^53)
                unsigned long long s[3] = { 0, 0, 0 };
                for (int j = 0; j < a.ky; ++j) {
                        const Row r = row<L>(a, y * a.ky + j);
                        for (int i = 0; i < a.kx; ++i) {
                                int c[3];
                                tap<L>(r, x * a.kx + i, c);
                                s[0] += (unsigned) c[0], s[1] += (unsigned) c[1], s[2] += (unsigned) c[2];
                        }
                }
                const unsigned long long n = (unsigned long long) a.kx * a.ky;
#pragma unroll
                for (int k = 0; k < 3; ++k) {  // S / n < 2^16: the double quotient is q or q - 1 (S < 2^53), then made exact
                        const unsigned long long S = s[k] + n / 2;
                        unsigned long long q = (unsigned long long) ((double) S * a.inv_n);
                        q -= q * n > S;
                        q += (q + 1) * n <= S;
                        out[k] = (int) q;
                }
        }
}

// A block makes kThreads * P consecutive pixels of a row.  Lane-interleaved pixels (pixel i of a thread is
// i * kThreads + threadIdx.x), so that the lanes of a warp read neighbouring taps in each load; the bytes go through
// shared memory, and each thread then stores 24 consecutive bytes.  At least 8 blocks per SM: a 64-register budget,
// under which no instance spills (ptxas picks 48 without the hint, and the 8-bit area kernels then spill).
template <int L, int A, typename Params = Args>
__global__ void __launch_bounds__(kThreads, 8) resize_kernel(Params a)
{
        constexpr bool W16 = L == L_RG48;
        constexpr int B = W16 ? 6 : 3, P = 24 / B;  // bytes per output pixel, pixels per thread
        __shared__ uint32_t seg[kThreads * 6];      // the block's kThreads * 24 output bytes of one row
        uint8_t *sb = reinterpret_cast<uint8_t *>(seg);
        const int bx0 = blockIdx.x * kThreads * P, x0 = bx0 + threadIdx.x * P;
        const int valid = min(24, (a.dw - x0) * B);  // this thread's bytes to store (<= 0: none)
        for (int y = blockIdx.y; y < a.dh; y += gridDim.y) {
                const bool yin = y >= a.ry && y < a.ry + a.rh;
#pragma unroll
                for (int i = 0; i < P; ++i) {
                        const int j = i * kThreads + threadIdx.x, x = bx0 + j - a.rx;
                        int c[3] = { 0, 0, 0 };
                        if (yin && x >= 0 && x < a.rw && bx0 + j < a.dw) {
                                pixel<L, A, Params>(a, x, y - a.ry, c);
                        }
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                                if constexpr (W16) {
                                        sb[B * j + 2 * k] = (uint8_t) c[k];
                                        sb[B * j + 2 * k + 1] = (uint8_t) (c[k] >> 8);
                                } else {
                                        sb[B * j + k] = (uint8_t) c[k];
                                }
                        }
                }
                __syncthreads();
                uint32_t w[6];
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                        w[i] = seg[6 * threadIdx.x + i];
                }
                __syncthreads();
                uint8_t *d = a.dst + y * a.dst_pitch + (long) x0 * B;
                if (valid == 24 && (uintptr_t) d % 8 == 0) {
#pragma unroll
                        for (int i = 0; i < 3; ++i) {
                                reinterpret_cast<uint2 *>(d)[i] = make_uint2(w[2 * i], w[2 * i + 1]);
                        }
                } else if (valid == 24 && (uintptr_t) d % 4 == 0) {
#pragma unroll
                        for (int i = 0; i < 6; ++i) {
                                reinterpret_cast<uint32_t *>(d)[i] = w[i];
                        }
                } else {
#pragma unroll
                        for (int i = 0; i < 24; ++i) {
                                if (i < valid) {
                                        d[i] = (uint8_t) (w[i >> 2] >> (8 * (i & 3)));
                                }
                        }
                }
        }
}

// cubic (K = 4) and lanczos4 (K = 8), separable.  A block owns a tile of kThreads output columns (one per thread) by
// a.ty output rows of the frame, and writes the tile's letterbox margins as zeros.  It walks the source rows its rows
// tap, in order.  For each one:
//   1. the pixels the tile's columns tap are read and converted to RGB once, into shared memory.  Dense: the span
//      from the first column's first tap to the last column's last, when it fits in kThreads * K slots (about when
//      scale_x < K, where neighbouring columns share taps); sparse: K slots per column, in tap order.
//   2. each thread forms H of its column into a ring of K rows (slot r % K);
//   3. every output row whose last tap row is r takes its K rows of H.
// Rows that no remaining output row of the tile taps (scale_y > K) are skipped.  A thread's column of the ring is its
// own, so only the staging buffer needs barriers.
template <int L, int K>
__global__ void __launch_bounds__(kThreads, 8) multitap_kernel(ArgsX a)
{
        constexpr bool W16 = L == L_RG48;
        constexpr int B = W16 ? 6 : 3, S = kThreads * K;
        __shared__ uint32_t stage[W16 ? 2 : 1][S];  // R | G << 8 | B << 16, or R | G << 16 and B
        __shared__ uint32_t ring[K][3][kThreads];   // H of source row r (int, or float bits) at r % K
        const int bx = blockIdx.x * kThreads, x = bx + threadIdx.x, xr = x - a.rx;
        const bool xin = x < a.dw, col = xin && xr >= 0 && xr < a.rw;
        const int c0 = max(bx, a.rx) - a.rx, c1 = min(min(bx + kThreads, a.dw), a.rx + a.rw) - a.rx;  // columns in the rectangle
        int first = 0, w[K];
#pragma unroll
        for (int j = 0; j < K; ++j) {
                w[j] = col ? a.xk[(long) xr * (K + 1) + 1 + j] : 0;
        }
        if (col) {
                first = a.xk[(long) xr * (K + 1)];
        }
        const int base = c0 < c1 ? a.xk[(long) c0 * (K + 1)] : 0;
        const int span = c0 < c1 ? a.xk[(long) (c1 - 1) * (K + 1)] + K - base : 0;
        const bool dense = span <= S;
        const int nslot = dense ? span : (c1 - c0) * K, slot0 = dense ? first - base : (xr - c0) * K;
        const int tiles = (a.dh + a.ty - 1) / a.ty;
        for (int tile = blockIdx.y; tile < tiles; tile += gridDim.y) {
                const int fy0 = tile * a.ty, fy1 = min(a.dh, fy0 + a.ty);
                for (int y = fy0; y < fy1; ++y) {
                        if (xin && (!col || y < a.ry || y >= a.ry + a.rh)) {
                                uint8_t *d = a.dst + y * a.dst_pitch + (long) x * B;
#pragma unroll
                                for (int i = 0; i < B; ++i) {
                                        d[i] = 0;
                                }
                        }
                }
                const int y0 = max(fy0, a.ry) - a.ry, y1 = min(fy1, a.ry + a.rh) - a.ry;  // rows in the rectangle
                if (c0 >= c1 || y0 >= y1) {
                        continue;
                }
                int ye = y0;  // the next output row to make
                const int rend = min(max(a.yk[(long) (y1 - 1) * (K + 1)] + K - 1, 0), a.sh - 1);
                for (int r = min(max(a.yk[(long) y0 * (K + 1)], 0), a.sh - 1); r <= rend && ye < y1; ++r) {
                        if (r < a.yk[(long) ye * (K + 1)]) {
                                continue;  // no remaining row taps it
                        }
                        const Row src = row<L>(a, r);
                        for (int s = threadIdx.x; s < nslot; s += kThreads) {
                                const int sx = dense ? base + s : a.xk[(long) (c0 + s / K) * (K + 1)] + s % K;
                                int c[3];
                                tap<L>(src, min(max(sx, 0), a.sw - 1), c);
                                if constexpr (W16) {
                                        stage[0][s] = (uint32_t) c[0] | (uint32_t) c[1] << 16;
                                        stage[1][s] = (uint32_t) c[2];
                                } else {
                                        stage[0][s] = (uint32_t) c[0] | (uint32_t) c[1] << 8 | (uint32_t) c[2] << 16;
                                }
                        }
                        __syncthreads();
                        if (col) {
                                uint32_t *h = &ring[r & (K - 1)][0][threadIdx.x];
                                if constexpr (W16) {
                                        float hs[3];
#pragma unroll
                                        for (int j = 0; j < K; ++j) {
                                                const uint32_t p = stage[0][slot0 + j], q = stage[1][slot0 + j];
                                                const float aj = __int_as_float(w[j]);
                                                const float t[3] = { __fmul_rn((float) (p & 65535), aj), __fmul_rn((float) (p >> 16), aj),
                                                                     __fmul_rn((float) q, aj) };
#pragma unroll
                                                for (int k = 0; k < 3; ++k) {
                                                        hs[k] = j == 0 ? t[k] : __fadd_rn(hs[k], t[k]);
                                                }
                                        }
#pragma unroll
                                        for (int k = 0; k < 3; ++k) {
                                                h[k * kThreads] = __float_as_uint(hs[k]);
                                        }
                                } else {
                                        int hs[3] = { 0, 0, 0 };
#pragma unroll
                                        for (int j = 0; j < K; ++j) {
                                                const uint32_t p = stage[0][slot0 + j];
                                                hs[0] += w[j] * (int) (p & 255), hs[1] += w[j] * (int) (p >> 8 & 255), hs[2] += w[j] * (int) (p >> 16);
                                        }
#pragma unroll
                                        for (int k = 0; k < 3; ++k) {
                                                h[k * kThreads] = (uint32_t) hs[k];
                                        }
                                }
                        }
                        __syncthreads();
                        for (; ye < y1 && min(a.yk[(long) ye * (K + 1)] + K - 1, a.sh - 1) <= r; ++ye) {
                                if (!col) {
                                        continue;
                                }
                                const int32_t *t = a.yk + (long) ye * (K + 1);
                                int out[3];
                                if constexpr (W16) {
                                        float v[3];
#pragma unroll
                                        for (int k = 0; k < K; ++k) {
                                                const int sr = min(max(t[0] + k, 0), a.sh - 1) & (K - 1);
                                                const float b = __int_as_float(t[1 + k]);
#pragma unroll
                                                for (int c = 0; c < 3; ++c) {
                                                        const float p = __fmul_rn(__uint_as_float(ring[sr][c][threadIdx.x]), b);
                                                        v[c] = k == 0 ? p : __fadd_rn(v[c], p);
                                                }
                                        }
#pragma unroll
                                        for (int c = 0; c < 3; ++c) {
                                                out[c] = min(max(__float2int_rn(v[c]), 0), 65535);
                                        }
                                } else if (a.v32) {
                                        int v[3] = { 1 << 21, 1 << 21, 1 << 21 };
#pragma unroll
                                        for (int k = 0; k < K; ++k) {
                                                const int sr = min(max(t[0] + k, 0), a.sh - 1) & (K - 1), b = t[1 + k];
#pragma unroll
                                                for (int c = 0; c < 3; ++c) {
                                                        v[c] += b * (int) ring[sr][c][threadIdx.x];
                                                }
                                        }
#pragma unroll
                                        for (int c = 0; c < 3; ++c) {
                                                out[c] = sat8(v[c] >> 22);
                                        }
                                } else {  // V may pass 2^31 (lanczos4): exact 64-bit sums
                                        long long v[3] = { 1 << 21, 1 << 21, 1 << 21 };
#pragma unroll
                                        for (int k = 0; k < K; ++k) {
                                                const int sr = min(max(t[0] + k, 0), a.sh - 1) & (K - 1), b = t[1 + k];
#pragma unroll
                                                for (int c = 0; c < 3; ++c) {
                                                        v[c] += (long long) b * (int) ring[sr][c][threadIdx.x];
                                                }
                                        }
#pragma unroll
                                        for (int c = 0; c < 3; ++c) {
                                                out[c] = (int) min(max(v[c] >> 22, 0ll), 255ll);
                                        }
                                }
                                uint8_t *d = a.dst + (a.ry + ye) * a.dst_pitch + (long) x * B;
#pragma unroll
                                for (int c = 0; c < 3; ++c) {
                                        if constexpr (W16) {
                                                d[2 * c] = (uint8_t) out[c];
                                                d[2 * c + 1] = (uint8_t) (out[c] >> 8);
                                        } else {
                                                d[c] = (uint8_t) out[c];
                                        }
                                }
                        }
                }
        }
}

template <int L>
static void launch_layout(int algo, const ArgsX &a, dim3 grid, dim3 tgrid, cudaStream_t st)
{
        const Args &b = a;
        switch (algo) {
        case A_NEAREST: resize_kernel<L, A_NEAREST><<<grid, kThreads, 0, st>>>(b); break;
        case A_LINEAR:
        case A_AREA_UP: resize_kernel<L, A_LINEAR><<<grid, kThreads, 0, st>>>(b); break;
        case A_AREA: resize_kernel<L, A_AREA><<<grid, kThreads, 0, st>>>(b); break;
        case A_AREA_ANY: resize_kernel<L, A_AREA_ANY, ArgsX><<<grid, kThreads, 0, st>>>(a); break;
        case A_CUBIC: multitap_kernel<L, 4><<<tgrid, kThreads, 0, st>>>(a); break;
        default: multitap_kernel<L, 8><<<tgrid, kThreads, 0, st>>>(a); break;
        }
}

static int layout_of(codec_t c)
{
        switch (c) {
        case RGB: return L_RGB;
        case RGBA: return L_RGBA;
        case UYVY: return L_UYVY;
        case YUYV: return L_YUYV;
        case I420: return L_I420;
        default: return L_RG48;
        }
}

// what reconfigure_if_needed and resize_frame decide for one input descriptor
struct Geometry {
        int out[8];  // route, out codec, out_w, out_h, rect x, y, w, h
        int algo;    // Algo
        int kx, ky;  // area box (A_AREA)
};

}  // namespace ugb_resize

using namespace ugb_resize;

struct ugb200_cf_resize {
        int mode;
        double factor;
        int tw, th, algo;
        bool all_algos;  // from ugb200_cf_resize_create2: cubic, lanczos4 and area at any ratio too
        // the input descriptor of the cached state
        int codec, width, height;
        Geometry g;
        int32_t *tables;  // the column table, then the row table (area other than A_AREA: heads, then entries)
        size_t toff[4];   // int32 offsets of the column and row tables (and of the column and row area entries)
        bool v32;         // cubic, lanczos4, 8-bit: every V + 2^21 fits in an int
        void *stage;   // the route codec's frame, for codecs outside the resize set
        size_t stage_bytes;
};
using ResizeState = struct ugb200_cf_resize;  // the struct shares its name with the entry point

static int resize_geometry(const ResizeState *r, int codec, int width, int height, Geometry *g)
{
        if (r == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        // reconfigure_if_needed (resize.c:181-210)
        static const codec_t set[] = { RGB, RGBA, I420, UYVY, YUYV, RG48, VIDEO_CODEC_NONE };  // RESIZE_SUPPORTED_PIXFMT_INIT
        codec_t route = VIDEO_CODEC_NONE;
        for (const codec_t *c = set; *c != VIDEO_CODEC_NONE; ++c) {
                if (*c == (codec_t) codec) {
                        route = *c;
                }
        }
        if (route == VIDEO_CODEC_NONE && (codec <= VIDEO_CODEC_NONE || codec >= VIDEO_CODEC_END ||
                                          !get_best_decoder_from((codec_t) codec, set, &route))) {
                return -4;  // the reference logs and drops the frame
        }
        const bool w16 = get_bits_per_component(route) != 8;
        long ow, oh;
        if (r->mode == 2) {
                ow = r->tw, oh = r->th;
        } else {
                const double fw = width * r->factor, fh = height * r->factor;
                if (!(fw < 2147483648.0 && fh < 2147483648.0)) {
                        return -1;
                }
                ow = (long) fw, oh = (long) fh;  // resize.c:219-220, truncation
        }
        if (ow <= 0 || oh <= 0 || ow * oh > (long) INT32_MAX / 6) {
                return -1;
        }
        if (((route == UYVY || route == YUYV || route == I420) && width % 2) || (route == I420 && height % 2)) {
                return -1;  // OpenCV takes even sizes only there (DESIGN.md §8)
        }
        // resize_frame / resize_frame_dimensions (resize_utils.cpp:141-173)
        int rx = 0, ry = 0, rw = (int) ow, rh = (int) oh;
        double isx = r->factor, isy = r->factor;
        if (r->mode == 2) {
                const double in_aspect = (double) width / height, out_aspect = (double) r->tw / r->th;
                if (in_aspect == out_aspect) {
                } else if (in_aspect > out_aspect) {
                        rh = (int) (r->tw / in_aspect);
                        ry = (r->th - rh) / 2;
                } else {
                        rw = (int) (r->th * in_aspect);
                        rx = (r->tw - rw) / 2;
                }
                if (rw <= 0 || rh <= 0) {
                        return -1;  // cv::resize asserts on an empty destination
                }
                isx = (double) rw / width, isy = (double) rh / height;  // cv::resize with dsize and fx = fy = 0
        }
        g->algo = r->algo == -1 ? A_LINEAR : r->algo;
        g->kx = g->ky = 0;
        bool every_handle = true;  // nearest, linear and integer area: built for handles from either constructor
        if (g->algo == A_AREA) {
                g->kx = area_factor(width, rw, isx);
                g->ky = area_factor(height, rh, isy);
                if (g->kx == 0 || g->ky == 0) {  // cv::resize: INTER_AREA with both scales >= 1, else area-mode linear
                        g->algo = 1. / isx >= 1 && 1. / isy >= 1 ? A_AREA_ANY : A_AREA_UP;
                        every_handle = false;
                }
        } else if (g->algo == A_CUBIC || g->algo == A_LANCZOS4) {
                every_handle = false;
        }
        if (!every_handle && !r->all_algos) {
                return -4;  // ugb200_cf_resize_create handles: cubic, lanczos4, fractional area and area upscaling
        }
        const int out[8] = { route, w16 ? RG48 : RGB, (int) ow, (int) oh, rx, ry, rw, rh };
        for (int i = 0; i < 8; ++i) {
                g->out[i] = out[i];
        }
        return 0;
}

template <typename T>
static void append(std::vector<int32_t> &t, const std::vector<T> &v)
{
        const size_t n = t.size();
        t.resize(n + v.size() * sizeof(T) / sizeof(int32_t));
        std::memcpy(t.data() + n, v.data(), v.size() * sizeof(T));
}

// the largest sums of positive and of negative weights over a table's entries
static void weight_bounds(const std::vector<int32_t> &k, int K, long long *pos, long long *neg)
{
        *pos = *neg = 0;
        for (size_t i = 0; i < k.size(); i += K + 1) {
                long long p = 0, n = 0;
                for (int j = 1; j <= K; ++j) {
                        (k[i + j] > 0 ? p : n) += std::llabs(k[i + j]);
                }
                *pos = std::max(*pos, p), *neg = std::max(*neg, n);
        }
}

// the tables of an input descriptor, scales as cv::resize receives them (DESIGN.md §2 "Resize"); off as toff
static void build_tables(const ResizeState *r, int width, int height, const Geometry &g, std::vector<int32_t> &t, size_t off[4], bool *v32)
{
        const int rw = g.out[6], rh = g.out[7];
        const double isx = r->mode == 2 ? (double) rw / width : r->factor, isy = r->mode == 2 ? (double) rh / height : r->factor;
        const bool w16 = g.out[1] == RG48;
        t.clear();
        *v32 = true;
        off[0] = off[2] = off[3] = 0;
        if (g.algo == A_NEAREST || g.algo == A_LINEAR || g.algo == A_AREA_UP) {
                std::vector<Tap2> p((size_t) rw + rh);
                if (g.algo == A_NEAREST) {
                        nearest_table(width, rw, isx, p.data());
                        nearest_table(height, rh, isy, p.data() + rw);
                } else if (g.algo == A_LINEAR) {
                        linear_table(width, rw, isx, true, w16, p.data());
                        linear_table(height, rh, isy, false, w16, p.data() + rw);
                } else {
                        linear_area_table(width, rw, isx, true, w16, p.data());
                        linear_area_table(height, rh, isy, false, w16, p.data() + rw);
                }
                append(t, p);
                off[1] = 4 * (size_t) rw;
        } else if (g.algo == A_CUBIC || g.algo == A_LANCZOS4) {
                const int K = g.algo == A_CUBIC ? 4 : 8;
                std::vector<int32_t> kx((size_t) rw * (K + 1)), ky((size_t) rh * (K + 1));
                (K == 4 ? cubic_table : lanczos4_table)(rw, isx, w16, kx.data());
                (K == 4 ? cubic_table : lanczos4_table)(rh, isy, w16, ky.data());
                if (!w16) {  // |V| <= 255 * (the largest sum of same-sign weight products)
                        long long px, nx, py, ny;
                        weight_bounds(kx, K, &px, &nx);
                        weight_bounds(ky, K, &py, &ny);
                        *v32 = 255 * (px * py + nx * ny) + (1 << 21) <= INT32_MAX && 255 * (px * ny + nx * py) <= (1ll << 31) + (1 << 21);
                }
                append(t, kx);
                off[1] = t.size();
                append(t, ky);
        } else {  // A_AREA_ANY
                std::vector<int32_t> hx, ex, hy, ey;
                area_tab(width, rw, 1. / isx, hx, ex);
                area_tab(height, rh, 1. / isy, hy, ey);
                append(t, hx);
                off[1] = t.size();
                append(t, hy);
                off[2] = t.size();
                append(t, ex);
                off[3] = t.size();
                append(t, ey);
        }
}

static ugb200_cf_resize_t create(int mode, double factor, int tw, int th, int algo, bool all_algos)
{
        if (!((mode == 1 && factor > 0 && factor < HUGE_VAL) || (mode == 2 && tw > 0 && th > 0)) || algo < -1 || algo > 4) {
                return nullptr;
        }
        return new (std::nothrow) ResizeState{ mode, mode == 1 ? factor : 0., mode == 2 ? tw : 0, mode == 2 ? th : 0, algo, all_algos, -1, 0, 0, {}, nullptr, {}, true, nullptr, 0 };
}

extern "C" UGB_API ugb200_cf_resize_t ugb200_cf_resize_create(int mode, double factor, int tw, int th, int algo)
{
        return create(mode, factor, tw, th, algo, false);
}

extern "C" UGB_API ugb200_cf_resize_t ugb200_cf_resize_create2(int mode, double factor, int tw, int th, int algo)
{
        return create(mode, factor, tw, th, algo, true);
}

extern "C" UGB_API void ugb200_cf_resize_destroy(ugb200_cf_resize_t r)
{
        if (r != nullptr) {
                cudaFree(r->tables);
                cudaFree(r->stage);
                delete r;
        }
}

extern "C" UGB_API int ugb200_cf_resize_geometry(ugb200_cf_resize_t r, int codec, int width, int height, int out[8])
{
        Geometry g;
        const int rc = resize_geometry(r, codec, width, height, &g);
        if (rc == 0 && out != nullptr) {
                for (int i = 0; i < 8; ++i) {
                        out[i] = g.out[i];
                }
        }
        return rc;
}

// Slack after the staging frame.  A line converter writes whole output groups, so on the last row it may write up to
// one group past vc_get_linesize (v210 -> RG48 rounds to 36-byte groups, R12L -> RG48 to 48); the reference allocates
// every frame with MAX_PADDING (64) bytes after it (video_frame.c:146, video_codec.h:61) for the same reason.
constexpr size_t kStageSlack = 64;

// reconfigure_if_needed: tables and staging frame for a new input descriptor.  The old buffers are freed first
// (cudaFree waits for the device), so no launch still reading them sees them change.  The tables are copied on the
// caller's stream, which is then synchronised: the launch that reads them is ordered after the copy on any stream,
// and the host vector outlives the copy.
static int reconfigure(ResizeState *r, int codec, int width, int height, const Geometry &g, cudaStream_t st)
{
        if (r->codec == codec && r->width == width && r->height == height) {
                return 0;
        }
        r->codec = -1;
        cudaFree(r->tables);
        r->tables = nullptr;
        if (g.algo != A_AREA) {
                std::vector<int32_t> t;
                build_tables(r, width, height, g, t, r->toff, &r->v32);
                if (cudaMalloc(&r->tables, t.size() * sizeof(int32_t)) != cudaSuccess ||
                    cudaMemcpyAsync(r->tables, t.data(), t.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st) != cudaSuccess ||
                    cudaStreamSynchronize(st) != cudaSuccess) {
                        return -2;
                }
        }
        const size_t stage = g.out[0] == codec ? 0 : vc_get_datalen(width, height, (codec_t) g.out[0]) + kStageSlack;
        if (stage != r->stage_bytes) {
                cudaFree(r->stage);
                r->stage = nullptr;
                r->stage_bytes = 0;
                if (stage != 0 && cudaMalloc(&r->stage, stage) != cudaSuccess) {
                        return -2;
                }
                r->stage_bytes = stage;
        }
        r->codec = codec, r->width = width, r->height = height;
        r->g = g;
        return 0;
}

extern "C" UGB_API int ugb200_cf_resize(ugb200_cf_resize_t r, int codec, int width, int height, const void *src, void *dst,
                                        cuda_wrapper_stream_t stream)
{
        if (r == nullptr || src == nullptr || dst == nullptr) {
                return -1;
        }
        Geometry g;
        int rc = resize_geometry(r, codec, width, height, &g);
        if (rc != 0) {
                return rc;
        }
        const codec_t route = (codec_t) g.out[0];
        const int ow = g.out[2], oh = g.out[3];
        const long out_ls = vc_get_linesize(ow, (codec_t) g.out[1]);
        if (overlap(src, vc_get_datalen(width, height, (codec_t) codec), dst, (size_t) out_ls * oh)) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        if ((rc = reconfigure(r, codec, width, height, g, st)) != 0) {
                return rc;
        }
        const uint8_t *in = (const uint8_t *) src;
        if (route != (codec_t) codec) {  // parallel_pix_conv with the route's decoder, default shifts (resize.c:254-259)
                const long ls = vc_get_linesize(width, route);
                rc = ugb200_pixfmt_convert(codec, route, r->stage, ls, src, vc_get_linesize(width, (codec_t) codec), (int) ls, height, 0,
                                           0, 8, 16, stream);
                if (rc != 0) {
                        return rc;
                }
                in = (const uint8_t *) r->stage;
        }
        ArgsX a{};
        a.src = in;
        a.src_pitch = route == I420 ? width : vc_get_linesize(width, route);
        a.cpitch = width / 2;
        a.u = in + (size_t) width * height;
        a.v = a.u + (size_t) a.cpitch * (height / 2);
        a.dst = (uint8_t *) dst;
        a.dst_pitch = out_ls;
        a.dw = ow, a.dh = oh;
        a.rx = g.out[4], a.ry = g.out[5], a.rw = g.out[6], a.rh = g.out[7];
        a.xt = reinterpret_cast<const Tap2 *>(r->tables);
        a.yt = a.xt + (r->tables ? a.rw : 0);
        a.sw = width, a.sh = height;
        if (r->tables != nullptr) {
                a.xk = a.axh = r->tables + r->toff[0];
                a.yk = a.ayh = r->tables + r->toff[1];
                a.axe = r->tables + r->toff[2];
                a.aye = r->tables + r->toff[3];
        }
        a.v32 = r->v32;
        a.kx = g.kx, a.ky = g.ky;
        a.div32 = (unsigned long long) g.kx * g.ky * 65536ull < (1ull << 32);
        a.inv_n = g.algo == A_AREA ? 1. / ((double) g.kx * g.ky) : 0.;
        const int per = g.out[1] == RG48 ? 4 : 8;
        const dim3 grid((unsigned) (((ow + per - 1) / per + kThreads - 1) / kThreads), oh < 65535 ? oh : 65535);
        // cubic, lanczos4: tiles of kThreads columns by 32, 16 or 8 rows, the tallest that still gives about 8 blocks
        // per SM of an H100 (132 SMs): taller tiles read fewer halo rows, and more blocks fill the GPU
        const unsigned tx = (unsigned) ((ow + kThreads - 1) / kThreads);
        a.ty = 32;
        while (a.ty > 8 && (long) tx * ((oh + a.ty - 1) / a.ty) < 8 * 132) {
                a.ty /= 2;
        }
        const long tiles = (oh + a.ty - 1) / a.ty;
        const dim3 tgrid(tx, (unsigned) (tiles < 65535 ? tiles : 65535));
        switch (layout_of(route)) {
        case L_RGB: launch_layout<L_RGB>(g.algo, a, grid, tgrid, st); break;
        case L_RGBA: launch_layout<L_RGBA>(g.algo, a, grid, tgrid, st); break;
        case L_UYVY: launch_layout<L_UYVY>(g.algo, a, grid, tgrid, st); break;
        case L_YUYV: launch_layout<L_YUYV>(g.algo, a, grid, tgrid, st); break;
        case L_I420: launch_layout<L_I420>(g.algo, a, grid, tgrid, st); break;
        default: launch_layout<L_RG48>(g.algo, a, grid, tgrid, st); break;
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
