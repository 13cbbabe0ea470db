// The UYVY -> RGB / RGBA line converters of pixfmt_kernels.cu as device functors, shared with the JPEG decoder, whose fused IDCT kernel
// (jpeg_decode_kernels.cu) hands them the UYVY words of its tile instead of writing UYVY to memory and converting it in a second pass.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "color_space.h"
#include "f32x2.cuh"

namespace ugb {

struct conv_params {
        int rshift, gshift, bshift;
        int aux;  // converter-specific, computed on the host from dst_len (see conv_rgba_rgb)
};
/// where a chunk sits, for the rare converter whose result depends on more than its own chunk
struct row_ctx {
        const uint8_t *src;  // buffer start
        long row_abs;        // byte offset of this row in src
        long src_total;      // readable bytes
        int cx;              // chunk index within the row
};

/// YCbCr colour spaces of the integer YCbCr -> RGB conversion (UltraGrid's YCBCR_TO_R/G/B, color_space.h:106-109, at 8 bits): the
/// coefficient set and the luma offset subtracted before scaling
struct ycbcr_709 {  // BT.709 limited range: what vc_copylineUYVYtoRGB assumes
        static constexpr color_coeffs coeffs() { return coeffs_709(8); }
        static constexpr int y_off = 16;
};
struct ycbcr_601 {  // BT.601 limited range
        static constexpr color_coeffs coeffs() { return coeffs_601(8); }
        static constexpr int y_off = 16;
};
struct ycbcr_601_full {  // BT.601 full range (JFIF, T.871)
        static constexpr color_coeffs coeffs() { return coeffs_601(0); }
        static constexpr int y_off = 0;
};

/// copylineYUVtoRGB (pixfmt_conv.c:1065-1094) via vc_copylineUYVYtoRGB (:1102-1108) / YUYVtoRGB (:1116-1122), generalised over the colour
/// space CS; RGBA packs R, G and B at the shifts of conv_params and sets every other bit (alpha 0xFF).  ycbcr_709 without RGBA is the
/// reference's converter.  The reference computes (y_scale * (Y - 16) + c * (C - 128)) >> 14 in int32.  Every intermediate is an integer
/// below 2^24, so the same values are formed exactly in fp32 (FFMA2 issues two lanes per slot where the integer pipe is half rate); the
/// arithmetic shift is a round-down FMA onto the 1.5 * 2^23 magic (mantissa = floor(x / 2^14)), the clamp one VIMNMX.S16x2.RELU per two values.
template <int Y1, int Y2, int U, int V, class CS = ycbcr_709, bool RGBA = false>
struct conv_yuv422_rgb {
        static constexpr int IN = 32, OUT = RGBA ? 64 : 48;
        static __host__ int out_len(int dst_len) { return dst_len < OUT / 8 ? 0 : dst_len / (OUT / 8) * (OUT / 8); }
        static __device__ __forceinline__ float2 magic2(uint32_t w0, uint32_t w1, int byte)
        {
                return make_float2(__uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7540u | byte)), __uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7540u | byte)));
        }
        static __device__ __forceinline__ uint32_t floor_clamp2(float2 x)  // {clamp(x.x >> 14), clamp(x.y >> 14)} as two 16-bit lanes
        {
                const float2 f = __ffma2_rd(x, make_float2(0x1p-14f, 0x1p-14f), make_float2(12582912.0f, 12582912.0f));
                return __vimin_s16x2_relu(__byte_perm(__float_as_uint(f.x), __float_as_uint(f.y), 0x5410), 0x00ff00ffu);
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                constexpr color_coeffs c = CS::coeffs();
                static_assert((255L - CS::y_off) * c.y_scale + 128L * c.b_cb < (1L << 24) && (255L - CS::y_off) * c.y_scale + 128L * c.r_cr < (1L << 24) &&
                                      CS::y_off * (long) c.y_scale + 128L * c.b_cb < (1L << 24) && CS::y_off * (long) c.y_scale + 128L * c.r_cr < (1L << 24),
                              "fp32 must hold the sums exactly");
                constexpr float ybias = -(8388608.0f + CS::y_off);  // magic2 gives 2^23 + byte
                const float2 ys = make_float2((float) c.y_scale, (float) c.y_scale);
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
#pragma unroll
                for (int i = 0; i < 8; i += 2) {  // lanes = the same sample of words i and i + 1 (four pixels)
                        const float2 ya = __fadd2_rn(magic2(in[i], in[i + 1], Y1), make_float2(ybias, ybias));  // Y - y_off
                        const float2 yb = __fadd2_rn(magic2(in[i], in[i + 1], Y2), make_float2(ybias, ybias));
                        const float2 u = __fadd2_rn(magic2(in[i], in[i + 1], U), make_float2(-8388736.0f, -8388736.0f));    // Cb - 128
                        const float2 v = __fadd2_rn(magic2(in[i], in[i + 1], V), make_float2(-8388736.0f, -8388736.0f));
                        const float2 rc = __fmul2_rn(v, make_float2((float) c.r_cr, (float) c.r_cr));
                        const float2 gc = __ffma2_rn(u, make_float2((float) c.g_cb, (float) c.g_cb), __fmul2_rn(v, make_float2((float) c.g_cr, (float) c.g_cr)));
                        const float2 bc = __fmul2_rn(u, make_float2((float) c.b_cb, (float) c.b_cb));
                        // lanes of each: {word i, word i + 1}
                        const uint32_t r1 = floor_clamp2(__ffma2_rn(ya, ys, rc)), g1 = floor_clamp2(__ffma2_rn(ya, ys, gc)), b1 = floor_clamp2(__ffma2_rn(ya, ys, bc));
                        const uint32_t r2 = floor_clamp2(__ffma2_rn(yb, ys, rc)), g2 = floor_clamp2(__ffma2_rn(yb, ys, gc)), b2 = floor_clamp2(__ffma2_rn(yb, ys, bc));
                        if constexpr (RGBA) {  // pixels 2i, 2i + 1 (word i, low lanes) and 2i + 2, 2i + 3 (word i + 1, high lanes)
                                out[2 * i + 0] = amask | (r1 & 0xffu) << p.rshift | (g1 & 0xffu) << p.gshift | (b1 & 0xffu) << p.bshift;
                                out[2 * i + 1] = amask | (r2 & 0xffu) << p.rshift | (g2 & 0xffu) << p.gshift | (b2 & 0xffu) << p.bshift;
                                out[2 * i + 2] = amask | (r1 >> 16) << p.rshift | (g1 >> 16) << p.gshift | (b1 >> 16) << p.bshift;
                                out[2 * i + 3] = amask | (r2 >> 16) << p.rshift | (g2 >> 16) << p.gshift | (b2 >> 16) << p.bshift;
                        } else {
                                // bytes of the 12 output bytes: word i -> r1 g1 b1 r2 g2 b2 (low lanes), word i + 1 -> the high lanes
                                const uint32_t rg1 = __byte_perm(r1, g1, 0x6240), br = __byte_perm(b1, r2, 0x6240), gb2 = __byte_perm(g2, b2, 0x6240);  // {lo.a, lo.b, hi.a, hi.b}
                                out[3 * (i / 2) + 0] = __byte_perm(rg1, br, 0x5410);   // r1 g1 b1 r2   (word i)
                                out[3 * (i / 2) + 1] = __byte_perm(gb2, rg1, 0x7610);  // g2 b2 | r1' g1' (word i + 1)
                                out[3 * (i / 2) + 2] = __byte_perm(br, gb2, 0x7632);   // b1' r2' g2' b2'
                        }
                }
        }
};

/// vc_copylineUYVYtoRGBA, pixfmt_conv.c:1137-1163 — the one double-precision matrix on the CPU path:
/// products and sums in IEEE double (no contraction: the reference is built without -mfma), truncation
/// toward zero, clamp 0..255, packed with runtime shifts + alpha mask.
struct conv_uyvy_rgba {
        static constexpr int IN = 16, OUT = 32;
        static __host__ int out_len(int dst_len) { return dst_len < 8 ? 0 : dst_len / 8 * 8; }
        // The conversions are the slow FP64 instructions on this part (I2F / F2I: 16 lanes/clk/SM against 63 for DADD/DMUL), so both go
        // through the 2^52 magic: 2^52 + byte is exact, and x + 1.5 * 2^52 rounded toward zero leaves floor(x) in the low word - equal to
        // the reference's truncation for x >= 0, and below zero both end at 0 after the clamp.
        static __device__ __forceinline__ double byte_minus(uint32_t b, double bias) { return __dadd_rn(__hiloint2double(0x43300000, (int) b), bias); }
        static __device__ __forceinline__ int trunc_int(double x) { return __double2loint(__dadd_rz(x, 6755399441055744.0)); }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
                // byte-aligned shifts (every caller in the tree): one permute places the three clamped components, selector built once per thread
                const bool aligned = !((p.rshift | p.gshift | p.bshift) & 7);
                uint32_t sel = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                        sel |= (8 * j == p.rshift ? 0u : 8 * j == p.gshift ? 2u : 8 * j == p.bshift ? 4u : 5u) << (4 * j);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint32_t w = in[i];
                        const double du = byte_minus(w & 0xff, -4503599627370624.0), dv = byte_minus((w >> 16) & 0xff, -4503599627370624.0);  // - (2^52 + 128)
                        const double rv = __dmul_rn(1.793, dv), gv = __dmul_rn(0.534, dv), gu = __dmul_rn(0.213, du), bu = __dmul_rn(2.115, du);
#pragma unroll
                        for (int k = 0; k < 2; ++k) {
                                const double yy = __dmul_rn(1.164, byte_minus((w >> (8 + 16 * k)) & 0xff, -4503599627370512.0));  // - (2^52 + 16)
                                const int r = trunc_int(__dadd_rn(yy, rv)), g = trunc_int(__dadd_rn(__dadd_rn(yy, -gv), -gu)), b = trunc_int(__dadd_rn(yy, bu));
                                // clamp 0..255 two at a time (the values fit 16 bits): VIMNMX.S16x2.RELU
                                const uint32_t rg = __vimin_s16x2_relu(__byte_perm((uint32_t) r, (uint32_t) g, 0x5410), 0x00ff00ffu);
                                const uint32_t bb = __vimin_s16x2_relu((uint32_t) b & 0xffffu, 0x00ff00ffu);
                                out[2 * i + k] = aligned ? amask | __byte_perm(rg, bb, sel) : amask | (rg & 0xff) << p.rshift | (rg >> 16) << p.gshift | bb << p.bshift;
                        }
                }
        }
};

}  // namespace ugb
