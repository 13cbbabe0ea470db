// Whole-buffer pixel-format line converters: the device form of UltraGrid's decoder_t line functions
// (src/pixfmt_conv.c, table :3041-3103) looped over rows as tools/convert.cpp:148-152 does.
//
// Every converter is a pure streaming kernel (HBM-bound): a thread owns one "chunk" of a row whose
// input and output sizes are both multiples of 16 bytes, reads it with 128-bit loads, converts in
// registers, writes 128-bit stores.  Chunks that straddle the end of a row (or unaligned buffers)
// take a byte-granular guarded path inside the same kernel, so edge semantics (how many bytes of
// dst_len each reference loop really writes) are preserved exactly.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/ugb200.h"
#include "color_space.h"
#include "f32x2.cuh"
#include "rgb_line_conv.cuh"
#include "rgb_to_uyvy.cuh"
#include "yuv_rgb_conv.cuh"

namespace ugb {

__device__ __forceinline__ int clamp255(int v) { return min(max(v, 0), 255); }

// ---- converters ----------------------------------------------------------------------------------
// Each declares IN/OUT bytes per chunk, out_len(dst_len) = number of bytes the reference loop writes
// for a given dst_len, and run().  A converter that reads colour coefficients takes their set as the template parameter CS
// (bt709 / bt601, color_space.h); ugb200_pixfmt_convert_cs picks the instantiation.

/// vc_copylinev210, pixfmt_conv.c:86-130: drop the 2 LSBs of each 10-bit sample; 16 B (6 px) -> 12 B
struct conv_v210_uyvy {
        static constexpr int IN = 64, OUT = 48;
        static __host__ int out_len(int dst_len)
        {
                const int rem = dst_len % 12;
                return dst_len - rem + (rem >= 4 ? 4 : 0) + (rem >= 8 ? 4 : 0);  // :118-129
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                        const uint32_t w0 = in[4 * g], w1 = in[4 * g + 1], w2 = in[4 * g + 2], w3 = in[4 * g + 3];
#define S8(w, sh) (((w) >> ((sh) + 2)) & 0xffu)
                        out[3 * g + 0] = pack4(S8(w0, 0), S8(w0, 10), S8(w0, 20), S8(w1, 0));
                        out[3 * g + 1] = pack4(S8(w1, 10), S8(w1, 20), S8(w2, 0), S8(w2, 10));
                        out[3 * g + 2] = pack4(S8(w2, 20), S8(w3, 0), S8(w3, 10), S8(w3, 20));
#undef S8
                }
        }
};

/// vc_copylineYUYV, pixfmt_conv.c:136-198 (same byte swap both directions)
struct conv_yuyv_uyvy {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int dst_len) { return dst_len / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        out[i] = __byte_perm(in[i], 0, 0x2301);
                }
        }
};

/// vc_copylineToRGBA_inplace, pixfmt_conv.c:907-921: pick R, G, B out of a 32-bit pixel by SOURCE shifts; the fourth byte becomes 0.
/// dst may be src (a thread reads its whole chunk before it writes it).
struct conv_to_rgba_inplace {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int dst_len) { return dst_len < 4 ? 0 : dst_len / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        out[i] = ((in[i] >> p.rshift) & 0xff) | ((in[i] >> p.gshift) & 0xff) << 8 | ((in[i] >> p.bshift) & 0xff) << 16;
                }
        }
};

/// vc_copylineRGBA, pixfmt_conv.c:538-589: re-shift an RGBA word, alpha forced to 0xFF in the unused byte.
/// (With default shifts the reference does a memcpy of `len` bytes; the launcher handles that case.)
struct conv_rgba_rgba {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int dst_len) { return dst_len < 4 ? 0 : dst_len / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint32_t t = in[i];
                        out[i] = amask | (t & 0xff) << p.rshift | ((t >> 8) & 0xff) << p.gshift | ((t >> 16) & 0xff) << p.bshift;
                }
        }
};

/// vc_copylineRGB, pixfmt_conv.c:732-753 (colour order change through shifts; default shifts = memcpy)
/// and vc_copylineBGRtoRGB (rshift 16, gshift 8, bshift 0).
struct conv_rgb_rgb {
        static constexpr int IN = 48, OUT = 48;
        static __host__ int out_len(int dst_len) { return dst_len < 3 ? 0 : dst_len / 3 * 3; }
        template <int K>
        static __device__ __forceinline__ void px(const uint32_t *in, uint32_t *o, const conv_params &p)
        {
                if constexpr (K < 16) {
                        const uint32_t w = gb<3 * K>(in) << p.rshift | gb<3 * K + 1>(in) << p.gshift | gb<3 * K + 2>(in) << p.bshift;
                        o[3 * K] = w & 0xff, o[3 * K + 1] = (w >> 8) & 0xff, o[3 * K + 2] = (w >> 16) & 0xff;
                        px<K + 1>(in, o, p);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                uint32_t o[48];
                px<0>(in, o, p);
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        out[i] = pack4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                }
        }
};

// ---- v210 family (A8) ---------------------------------------------------------------------------------------------
#define UGB_S10(w, sh) (((w) >> (sh)) & 0x3ffu)

/// vc_copylineUYVYtoV210, pixfmt_conv.c:2581-2607: every 3 consecutive source BYTES (u, y, v in the loop's naming) become one
/// v210 word with each byte << 2; one word per 4 bytes of dst_len
struct conv_uyvy_v210 {
        static constexpr int IN = 48, OUT = 64;
        static __host__ int out_len(int dst_len) { return dst_len < 4 ? 0 : dst_len / 4 * 4; }
        template <int K>
        static __device__ __forceinline__ void word(const uint32_t *in, uint32_t *out)
        {
                if constexpr (K < 16) {
                        out[K] = (gb<3 * K>(in) << 2) | (gb<3 * K + 1>(in) << 12) | (gb<3 * K + 2>(in) << 22);
                        word<K + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { word<0>(in, out); }
};

/// vc_copylineY216toV210, pixfmt_conv.c:2761-2790: 12 16-bit samples (Y U Y V ...) >> 6 into four v210 words; ceil(dst_len/16) groups
struct conv_y216_v210 {
        static constexpr int IN = 48, OUT = 32;
        static __host__ int out_len(int dst_len) { return (dst_len + 15) / 16 * 16; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int g = 0; g < 2; ++g) {
                        uint32_t s[12];
#pragma unroll
                        for (int i = 0; i < 6; ++i) {
                                s[2 * i] = (in[6 * g + i] & 0xffffu) >> 6, s[2 * i + 1] = in[6 * g + i] >> 22;
                        }
                        // s = y1 u y2 v | y1 u y2 v | y1 u y2 v
                        out[4 * g + 0] = s[1] | s[0] << 10 | s[3] << 20;
                        out[4 * g + 1] = s[2] | s[5] << 10 | s[4] << 20;
                        out[4 * g + 2] = s[7] | s[6] << 10 | s[9] << 20;
                        out[4 * g + 3] = s[8] | s[11] << 10 | s[10] << 20;
                }
        }
};

/// vc_copylineV210toY216, pixfmt_conv.c:2792-2832: 10-bit samples << 6 into Y U Y V 16-bit words; floor(dst_len/24) groups
struct conv_v210_y216 {
        static constexpr int IN = 32, OUT = 48;
        static __host__ int out_len(int dst_len) { return dst_len / 24 * 24; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int g = 0; g < 2; ++g) {
                        const uint32_t w0 = in[4 * g], w1 = in[4 * g + 1], w2 = in[4 * g + 2], w3 = in[4 * g + 3];
#define UGB_P(a, b) ((a) << 6 | (b) << 22)
                        out[6 * g + 0] = UGB_P(UGB_S10(w0, 10), UGB_S10(w0, 0));   // Y0 U0
                        out[6 * g + 1] = UGB_P(UGB_S10(w1, 0), UGB_S10(w0, 20));   // Y1 V0
                        out[6 * g + 2] = UGB_P(UGB_S10(w1, 20), UGB_S10(w1, 10));  // Y2 U1
                        out[6 * g + 3] = UGB_P(UGB_S10(w2, 10), UGB_S10(w2, 0));   // Y3 V1
                        out[6 * g + 4] = UGB_P(UGB_S10(w3, 0), UGB_S10(w2, 20));   // Y4 U2
                        out[6 * g + 5] = UGB_P(UGB_S10(w3, 20), UGB_S10(w3, 10));  // Y5 V2
#undef UGB_P
                }
        }
};

/// vc_copylineV210toY416, pixfmt_conv.c:2834-2882: U Y V A per pixel (chroma replicated, alpha 0xFFFF); floor(dst_len/48) groups
struct conv_v210_y416 {
        static constexpr int IN = 16, OUT = 48;
        static __host__ int out_len(int dst_len) { return dst_len / 48 * 48; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                const uint32_t w0 = in[0], w1 = in[1], w2 = in[2], w3 = in[3];
                const uint32_t y[6] = { UGB_S10(w0, 10), UGB_S10(w1, 0), UGB_S10(w1, 20), UGB_S10(w2, 10), UGB_S10(w3, 0), UGB_S10(w3, 20) };
                const uint32_t u[3] = { UGB_S10(w0, 0), UGB_S10(w1, 10), UGB_S10(w2, 20) };
                const uint32_t v[3] = { UGB_S10(w0, 20), UGB_S10(w2, 0), UGB_S10(w3, 10) };
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                        out[2 * i] = u[i / 2] << 6 | y[i] << 22;
                        out[2 * i + 1] = v[i / 2] << 6 | 0xFFFF0000u;
                }
        }
};

/// vc_copylineV210toRGB, pixfmt_conv.c:2884-2940: top 8 bits of each sample, depth-8 coefficients, CLAMP_FULL (1..254);
/// the loop runs while x < dst_len in steps of 18 bytes, i.e. it may write past dst_len up to the end of the last group
template <class CS = bt709>
struct conv_v210_rgb {  // fp32 like conv_yuv422_rgb: the sums stay below 2^24 (8-bit samples, depth-8 coefficients), >> 14 = round-down FMA
        static constexpr int IN = 128, OUT = 144;
        static __host__ int out_len(int dst_len) { return (dst_len + 17) / 18 * 18; }
        static __device__ __forceinline__ float magic8(uint32_t w, int sh) { return __uint_as_float(((w >> (sh + 2)) & 0xffu) | 0x4B000000u); }  // top 8 of 10 bits
        static __device__ __forceinline__ uint32_t floor_clamp2(float2 x)  // {CLAMP_FULL(x.x >> 14), CLAMP_FULL(x.y >> 14)}: 1..254 (color_space.h:96-98)
        {
                const float2 f = __ffma2_rd(x, make_float2(0x1p-14f, 0x1p-14f), make_float2(12582912.0f, 12582912.0f));
                return __vmaxs2(__vmins2(__byte_perm(__float_as_uint(f.x), __float_as_uint(f.y), 0x5410), 0x00FE00FEu), 0x00010001u);
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(8);
                static_assert(239L * c.y_scale + 128L * c.b_cb < (1L << 24) && 239L * c.y_scale + 128L * c.r_cr < (1L << 24) &&
                                      16L * c.y_scale + 128L * c.b_cb < (1L << 24) && 16L * c.y_scale + 128L * c.r_cr < (1L << 24) &&
                                      239L * c.y_scale - 128L * (c.g_cb + c.g_cr) < (1L << 24),
                              "fp32 must hold the sums exactly");
                const float2 ys = make_float2((float) c.y_scale, (float) c.y_scale), ybias = make_float2(-8388624.0f, -8388624.0f),
                             cbias = make_float2(-8388736.0f, -8388736.0f);
#pragma unroll
                for (int gp = 0; gp < 4; ++gp) {  // lanes of every float2 = the same sample of groups 2 gp and 2 gp + 1 (2 x 6 pixels)
                        const uint32_t *a = in + 8 * gp, *b = a + 4;
                        // sample positions inside a v210 group: word, bit shift (pixfmt_conv.c:2907-2925)
                        constexpr int yw[6] = { 0, 1, 1, 2, 3, 3 }, ysh[6] = { 10, 0, 20, 10, 0, 20 };
                        constexpr int uw[3] = { 0, 1, 2 }, ush[3] = { 0, 10, 20 }, vw[3] = { 0, 2, 3 }, vsh[3] = { 20, 0, 10 };
                        float2 rc[3], gc[3], bc[3];
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                                const float2 u = __fadd2_rn(make_float2(magic8(a[uw[k]], ush[k]), magic8(b[uw[k]], ush[k])), cbias);
                                const float2 v = __fadd2_rn(make_float2(magic8(a[vw[k]], vsh[k]), magic8(b[vw[k]], vsh[k])), cbias);
                                rc[k] = __fmul2_rn(v, make_float2((float) c.r_cr, (float) c.r_cr));
                                gc[k] = __ffma2_rn(u, make_float2((float) c.g_cb, (float) c.g_cb), __fmul2_rn(v, make_float2((float) c.g_cr, (float) c.g_cr)));
                                bc[k] = __fmul2_rn(u, make_float2((float) c.b_cb, (float) c.b_cb));
                        }
                        uint32_t val[18];  // R G B of the six pixels; low half-word = group 2 gp, high = group 2 gp + 1
#pragma unroll
                        for (int i = 0; i < 6; ++i) {
                                const float2 y = __fadd2_rn(make_float2(magic8(a[yw[i]], ysh[i]), magic8(b[yw[i]], ysh[i])), ybias);
                                val[3 * i] = floor_clamp2(__ffma2_rn(y, ys, rc[i / 2]));
                                val[3 * i + 1] = floor_clamp2(__ffma2_rn(y, ys, gc[i / 2]));
                                val[3 * i + 2] = floor_clamp2(__ffma2_rn(y, ys, bc[i / 2]));
                        }
#pragma unroll
                        for (int j = 0; j < 9; ++j) {  // byte n of the 36 output bytes: n < 18 -> val[n] byte 0, else val[n - 18] byte 2
                                uint32_t t[2];
#pragma unroll
                                for (int h = 0; h < 2; ++h) {
                                        const int n0 = 4 * j + 2 * h, n1 = n0 + 1;
                                        const uint32_t A = val[n0 < 18 ? n0 : n0 - 18], B = val[n1 < 18 ? n1 : n1 - 18];
                                        t[h] = __byte_perm(A, B, (n0 < 18 ? 0u : 2u) | (n1 < 18 ? 4u : 6u) << 4);
                                }
                                out[9 * gp + j] = __byte_perm(t[0], t[1], 0x5410);
                        }
                }
        }
};
/// vc_copylineV210toRG48, pixfmt_conv.c:2942-3002: all 10 bits, depth-10 coefficients, >> (COMP_BASE - 6), CLAMP_FULL at 16 bit
template <class CS = bt709>
struct conv_v210_rg48 {
        static constexpr int IN = 64, OUT = 144;
        static __host__ int out_len(int dst_len) { return (dst_len + 35) / 36 * 36; }
        static __device__ __forceinline__ uint32_t cf(int v) { return (uint32_t) min(max(v, 256), 65279); }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(10);
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                        const uint32_t w0 = in[4 * g], w1 = in[4 * g + 1], w2 = in[4 * g + 2], w3 = in[4 * g + 3];
#define UGB_T10(w, sh) ((int) (((w) >> (sh)) & 0x3ffu))
                        const int y[6] = { UGB_T10(w0, 10), UGB_T10(w1, 0), UGB_T10(w1, 20), UGB_T10(w2, 10), UGB_T10(w3, 0), UGB_T10(w3, 20) };
                        const int u[3] = { UGB_T10(w0, 0) - 512, UGB_T10(w1, 10) - 512, UGB_T10(w2, 20) - 512 };
                        const int v[3] = { UGB_T10(w0, 20) - 512, UGB_T10(w2, 0) - 512, UGB_T10(w3, 10) - 512 };
#undef UGB_T10
                        uint32_t o[18];
#pragma unroll
                        for (int i = 0; i < 6; ++i) {
                                const int ys = c.y_scale * (y[i] - 64), uu = u[i / 2], vv = v[i / 2];
                                o[3 * i + 0] = cf((ys + vv * c.r_cr) >> (COMP_BASE - 6));
                                o[3 * i + 1] = cf((ys + uu * c.g_cb + vv * c.g_cr) >> (COMP_BASE - 6));
                                o[3 * i + 2] = cf((ys + uu * c.b_cb) >> (COMP_BASE - 6));
                        }
#pragma unroll
                        for (int i = 0; i < 9; ++i) {
                                out[9 * g + i] = o[2 * i] | o[2 * i + 1] << 16;
                        }
                }
        }
};

// ---- pure byte-permutation converters (A9): out byte j = in byte M::src(j), or 0x00 (-1) / 0xFF (-2) -------------------
struct map_uyvy_gray {  // vc_copylineUYVYtoGrayscale, pixfmt_conv.c:927-938: the luma bytes
        static constexpr int IN = 32, OUT = 16;
        static __host__ int out_len(int n) { return n / 2 * 2; }
        static constexpr int src(int j) { return 2 * j + 1; }
};
struct map_dvs10_uyvy {  // vc_copylineDVS10 (C variant, pixfmt_conv.c:690-720): bytes 0..2 of every 32-bit word; src_len = dst_len / 1.5
        static constexpr int IN = 64, OUT = 48;
        static __host__ int out_len(int n) { return (int) (2 * (long long) n / 3) / 16 * 24; }
        static constexpr int src(int j) { return 4 * (j / 3) + j % 3; }
};
struct map_rgba_rg48 {  // vc_copylineRGBAtoRG48, :1336-1351
        static constexpr int IN = 32, OUT = 48;
        static __host__ int out_len(int n) { return n < 6 ? 0 : n / 6 * 6; }
        static constexpr int src(int j) { return (j % 2) ? 4 * (j / 6) + (j % 6) / 2 : -1; }
};
struct map_uyvy_y216 {  // vc_copylineUYVYtoY216, :2609-2627: Y0 U Y1 V, value in the high byte
        static constexpr int IN = 16, OUT = 32;
        static __host__ int out_len(int n) { return n / 8 * 8; }
        static constexpr int src(int j)
        {
                const int k = j % 8, g = j / 8;
                return k == 1 ? 4 * g + 1 : k == 3 ? 4 * g : k == 5 ? 4 * g + 3 : k == 7 ? 4 * g + 2 : -1;
        }
};
struct map_uyvy_y416 {  // vc_copylineUYVYtoY416, :2629-2665.  QUIRK: the loop tests dst_len >= 12 but consumes 16 per turn
        static constexpr int IN = 16, OUT = 64;
        static __host__ int out_len(int n)
        {
                if (n < 8) {
                        return 0;
                }
                const int turns = (n + 4) / 16, rem = n - 16 * turns;
                return 16 * turns + (rem >= 8 ? 8 : 0);
        }
        static constexpr int src(int j)
        {
                const int k = j % 16, g = j / 16;
                return k == 1 || k == 9 ? 4 * g : k == 3 ? 4 * g + 1 : k == 11 ? 4 * g + 3 : k == 5 || k == 13 ? 4 * g + 2 : k == 6 || k == 7 || k == 14 || k == 15 ? -2 : -1;
        }
};
struct map_y216_uyvy {  // vc_copylineY216toUYVY, :2728-2743
        static constexpr int IN = 32, OUT = 16;
        static __host__ int out_len(int n) { return n / 4 * 4; }
        static constexpr int src(int j)
        {
                const int k = j % 4, g = j / 4;
                return 8 * g + (k == 0 ? 3 : k == 1 ? 1 : k == 2 ? 7 : 5);
        }
};
struct map_vuya_y416 {  // vc_copylineVUYAtoY416, :2667-2686
        static constexpr int IN = 16, OUT = 32;
        static __host__ int out_len(int n) { return n / 8 * 8; }
        static constexpr int src(int j)
        {
                const int k = j % 8, g = j / 8;
                return k == 1 ? 4 * g + 1 : k == 3 ? 4 * g + 2 : k == 5 ? 4 * g : k == 7 ? 4 * g + 3 : -1;
        }
};

// ---- R10k (10-bit RGB, 4 B/px: R9..2 | R1..0 G9..4 | G3..0 B9..6 | B5..0 xx) --------------------------------------------
/// vc_copyliner10k, pixfmt_conv.c:211-272: top 8 bits of each component into an RGBA word with runtime shifts
struct conv_r10k_rgba {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int n) { return n / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint32_t w = in[i];
                        const uint32_t r = w & 0xff, g = ((w >> 8) & 0x3f) << 2 | ((w >> 22) & 3), b = ((w >> 16) & 0xf) << 4 | (w >> 28);
                        out[i] = amask | r << p.rshift | g << p.gshift | b << p.bshift;
                }
        }
};
/// vc_copyliner10ktoRGB, :331-340 (runs while x < dstlen in steps of 3)
struct conv_r10k_rgb {
        static constexpr int IN = 64, OUT = 48;
        static __host__ int out_len(int n) { return (n + 2) / 3 * 3; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                uint32_t o[48];
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                        const uint32_t b0 = in[i] & 0xff, b1 = (in[i] >> 8) & 0xff, b2 = (in[i] >> 16) & 0xff, b3 = in[i] >> 24;
                        o[3 * i] = b0, o[3 * i + 1] = (b1 << 2 | b2 >> 6) & 0xff, o[3 * i + 2] = (b2 << 4 | b3 >> 4) & 0xff;
                }
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        out[i] = pack4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                }
        }
};
/// vc_copyliner10ktoRG48, :274-292 (runs while dstlen > 0 in steps of 6)
struct conv_r10k_rg48 {
        static constexpr int IN = 32, OUT = 48;
        static __host__ int out_len(int n) { return (n + 5) / 6 * 6; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                uint32_t h[24];  // 16-bit samples
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        const uint32_t b1 = in[i] & 0xff, b2 = (in[i] >> 8) & 0xff, b3 = (in[i] >> 16) & 0xff, b4 = in[i] >> 24;
                        h[3 * i] = b1 << 8 | (b2 & 0xC0);
                        h[3 * i + 1] = ((b2 << 2 | b3 >> 6) & 0xff) << 8 | ((b3 & 0x30) << 2);
                        h[3 * i + 2] = (((b3 & 0xf) << 4 | b4 >> 4) & 0xff) << 8 | ((b4 & 0xC) << 4);
                }
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        out[i] = h[2 * i] | h[2 * i + 1] << 16;
                }
        }
};
/// vc_copylineRGBAtoR10k, :2538-2577
struct conv_rgba_r10k {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int n) { return n / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint32_t r = in[i] & 0xff, g = (in[i] >> 8) & 0xff, b = (in[i] >> 16) & 0xff;
                        out[i] = r | (g >> 2) << 8 | (b >> 4) << 16 | (g & 3) << 22 | 3u << 24 | (b & 0xf) << 28;
                }
        }
};
/// vc_copylineRG48toR10k, :2008-2028
struct conv_rg48_r10k {
        static constexpr int IN = 48, OUT = 32;
        static __host__ int out_len(int n) { return n < 4 ? 0 : n / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        const uint32_t s0 = 3 * i, s1 = 3 * i + 1, s2 = 3 * i + 2;
                        const uint32_t r = ((in[s0 / 2] >> (16 * (s0 & 1))) & 0xffff) >> 6, g = ((in[s1 / 2] >> (16 * (s1 & 1))) & 0xffff) >> 6,
                                       b = ((in[s2 / 2] >> (16 * (s2 & 1))) & 0xffff) >> 6;
                        out[i] = (b & 0x3F) << 26 | 0x3000000u | (g & 0xF) << 20 | (b >> 6) << 16 | (r & 0x3) << 14 | (g >> 4) << 8 | r >> 2;
                }
        }
};
/// vc_copylineRG48toRGBA, :2044-2055
struct conv_rg48_rgba {
        static constexpr int IN = 48, OUT = 32;
        static __host__ int out_len(int n) { return n < 4 ? 0 : n / 4 * 4; }
        template <int K>
        static __device__ __forceinline__ void px(const uint32_t *in, uint32_t *out, const conv_params &p, uint32_t amask)
        {
                if constexpr (K < 8) {
                        out[K] = amask | gb<6 * K + 1>(in) << p.rshift | gb<6 * K + 3>(in) << p.gshift | gb<6 * K + 5>(in) << p.bshift;
                        px<K + 1>(in, out, p, amask);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                px<0>(in, out, p, 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift));
        }
};

// ---- 4:4:4 <-> 4:2:2 with chroma averaging, VUYA colour conversions ----------------------------------------------------
/// vc_copylineVUYAtoUYVY (:2688-2703) and vc_copylineY416toUYVY (:2745-2759): chroma = (c0 + c1) / 2, luma copied.
/// OFF_Y1 is relative to the start of the pixel PAIR.  QUIRK kept: VUYAtoUYVY takes src[7] — the second pixel's ALPHA — as Y1.
template <int PIX, int OFF_U, int OFF_Y, int OFF_V, int OFF_Y1>
struct conv_444_uyvy {
        static constexpr int IN = 8 * PIX, OUT = 16;
        static __host__ int out_len(int n) { return n / 4 * 4; }
        template <int K>
        static __device__ __forceinline__ void pair(const uint32_t *in, uint32_t *out)
        {
                if constexpr (K < 4) {
                        constexpr int A = 2 * K * PIX, B = A + PIX;
                        out[K] = pack4((gb<A + OFF_U>(in) + gb<B + OFF_U>(in)) / 2, gb<A + OFF_Y>(in), (gb<A + OFF_V>(in) + gb<B + OFF_V>(in)) / 2,
                                       gb<A + OFF_Y1>(in));
                        pair<K + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { pair<0>(in, out); }
};
using conv_vuya_uyvy = conv_444_uyvy<4, 1, 2, 0, 7>;
using conv_y416_uyvy = conv_444_uyvy<8, 1, 3, 5, 11>;
/// vc_copylineVUYAtoRGB, :2705-2726 (depth-8 coefficients, CLAMP_FULL 1..254, runs while x < dst_len in steps of 3)
template <class CS = bt709>
struct conv_vuya_rgb {
        static constexpr int IN = 64, OUT = 48;
        static __host__ int out_len(int n) { return (n + 2) / 3 * 3; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(8);
                uint32_t o[48];
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                        const int v = (int) (in[i] & 0xff) - 128, u = (int) ((in[i] >> 8) & 0xff) - 128, y = c.y_scale * ((int) ((in[i] >> 16) & 0xff) - 16);
                        o[3 * i] = min(max((y + v * c.r_cr) >> COMP_BASE, 1), 254);
                        o[3 * i + 1] = min(max((y + u * c.g_cb + v * c.g_cr) >> COMP_BASE, 1), 254);
                        o[3 * i + 2] = min(max((y + u * c.b_cb) >> COMP_BASE, 1), 254);
                }
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        out[i] = pack4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                }
        }
};
/// vc_copylineRGBAtoVUYA, :2280-2302 (V U Y A; no clamp, bytes wrap)
template <class CS = bt709>
struct conv_rgba_vuya {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int n) { return n / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(8);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const int r = in[i] & 0xff, g = (in[i] >> 8) & 0xff, b = (in[i] >> 16) & 0xff;
                        const int v = ((r * c.cr_r + g * c.cr_g + b * c.cr_b) >> COMP_BASE) + 128, u = ((r * c.cb_r + g * c.cb_g + b * c.cb_b) >> COMP_BASE) + 128;
                        const int y = ((r * c.y_r + g * c.y_g + b * c.y_b) >> COMP_BASE) + 16;
                        out[i] = pack4(v & 0xff, u & 0xff, y & 0xff, in[i] >> 24);
                }
        }
};

// ---- 16-bit colour-space converters (Y416 / RG48 / R10k), depth-10/16 coefficients ------------------------------------------
// 16-bit sample K of a packed word array
template <int K>
__device__ __forceinline__ int gh(const uint32_t *a)
{
        return (int) ((a[K >> 1] >> (16 * (K & 1))) & 0xffffu);
}

/// Y416 (U Y V A, 16 bit) -> RGB-like.  MODE 0: RG48 (vc_copylineY416toRG48, pixfmt_conv.c:2485-2514), 1: RGB (:1948-1976),
/// 2: RGBA (:1978-2006), 3: R10k (:1917-1946).  int32 arithmetic wraps exactly like the reference's comp_type_t.
template <int MODE, class CS = bt709>
struct conv_y416_rgbx {
        static constexpr int NPX = MODE == 0 ? 8 : MODE == 1 ? 16 : 4;
        static constexpr int IN = NPX * 8, OUT = NPX * (MODE == 0 ? 6 : MODE == 1 ? 3 : 4);
        static __host__ int out_len(int n) { return MODE == 0 ? (n + 5) / 6 * 6 : MODE == 1 ? (n + 2) / 3 * 3 : (n + 3) / 4 * 4; }
        template <int K>
        static __device__ __forceinline__ void px(const uint32_t *in, uint32_t *o, const conv_params &p)
        {
                if constexpr (K < NPX) {
                        constexpr color_coeffs c = CS::at(16);
                        constexpr int SH = COMP_BASE + (MODE == 0 ? 0 : MODE == 3 ? 6 : 8);
                        constexpr int LO = MODE == 0 ? 256 : MODE == 3 ? 4 : 1, HI = MODE == 0 ? 65279 : MODE == 3 ? 1019 : 254;  // CLAMP_FULL
                        const int u = gh<4 * K>(in) - 32768, y = c.y_scale * (gh<4 * K + 1>(in) - 4096), v = gh<4 * K + 2>(in) - 32768;
                        const uint32_t r = clampr((y + v * c.r_cr) >> SH, LO, HI), g = clampr((y + u * c.g_cb + v * c.g_cr) >> SH, LO, HI),
                                       b = clampr((y + u * c.b_cb) >> SH, LO, HI);
                        if constexpr (MODE == 0 || MODE == 1) {
                                o[3 * K] = r, o[3 * K + 1] = g, o[3 * K + 2] = b;
                        } else if constexpr (MODE == 2) {
                                o[K] = (0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift)) | r << p.rshift | g << p.gshift |
                                       b << p.bshift;
                        } else {
                                o[K] = (r >> 2) | (((r & 3) << 6 | g >> 4) & 0xff) << 8 | (((g & 0xf) << 4 | b >> 6) & 0xff) << 16 | ((b & 0x3f) << 2) << 24;
                        }
                        px<K + 1>(in, o, p);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                if constexpr (MODE == 0) {
                        uint32_t o[24];
                        px<0>(in, o, p);
#pragma unroll
                        for (int i = 0; i < 12; ++i) {
                                out[i] = o[2 * i] | o[2 * i + 1] << 16;
                        }
                } else if constexpr (MODE == 1) {
                        uint32_t o[48];
                        px<0>(in, o, p);
#pragma unroll
                        for (int i = 0; i < 12; ++i) {
                                out[i] = pack4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                        }
                } else {
                        px<0>(in, out, p);
                }
        }
};

/// vc_copylineY416toV210, pixfmt_conv.c:3004-3033: chroma of a pixel pair averaged as uint16, every sample >> 6
struct conv_y416_v210 {
        static constexpr int IN = 96, OUT = 32;
        static __host__ int out_len(int n) { return n / 16 * 16; }
        template <int G>
        static __device__ __forceinline__ void group(const uint32_t *in, uint32_t *out)
        {
                if constexpr (G < 2) {
                        constexpr int S = 24 * G;  // 16-bit sample index of the group's first pixel (U Y V A per pixel)
#define UGB_AVG(a, b) ((uint32_t) ((gh<S + (a)>(in) + gh<S + (b)>(in)) / 2) >> 6)
#define UGB_Y(a) ((uint32_t) gh<S + (a)>(in) >> 6)
                        out[4 * G + 0] = UGB_AVG(0, 4) | UGB_Y(1) << 10 | UGB_AVG(2, 6) << 20;
                        out[4 * G + 1] = UGB_Y(5) | UGB_AVG(8, 12) << 10 | UGB_Y(9) << 20;
                        out[4 * G + 2] = UGB_AVG(10, 14) | UGB_Y(13) << 10 | UGB_AVG(16, 20) << 20;
                        out[4 * G + 3] = UGB_Y(17) | UGB_AVG(18, 22) << 10 | UGB_Y(21) << 20;
#undef UGB_AVG
#undef UGB_Y
                        group<G + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { group<0>(in, out); }
};

/// RG48 -> Y416 (vc_copylineRG48toY416, :2451-2483) / Y216 (:2410-2449) with depth-16 coefficients; results stored as uint16 (wrap)
template <class CS = bt709>
struct conv_rg48_y416 {
        static constexpr int IN = 48, OUT = 64;
        static __host__ int out_len(int n) { return (n + 7) / 8 * 8; }
        template <int K>
        static __device__ __forceinline__ void px(const uint32_t *in, uint32_t *out)
        {
                if constexpr (K < 8) {
                        constexpr color_coeffs c = CS::at(16);
                        const int r = gh<3 * K>(in), g = gh<3 * K + 1>(in), b = gh<3 * K + 2>(in);
                        const uint32_t u = ((r * c.cb_r + g * c.cb_g + b * c.cb_b) >> COMP_BASE) + 32768, y = ((r * c.y_r + g * c.y_g + b * c.y_b) >> COMP_BASE) + 4096,
                                       v = ((r * c.cr_r + g * c.cr_g + b * c.cr_b) >> COMP_BASE) + 32768;
                        out[2 * K] = (u & 0xffff) | (y & 0xffff) << 16;
                        out[2 * K + 1] = (v & 0xffff) | 0xFFFF0000u;
                        px<K + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { px<0>(in, out); }
};
template <class CS = bt709>
struct conv_rg48_y216 {
        static constexpr int IN = 48, OUT = 32;
        static __host__ int out_len(int n) { return (n + 7) / 8 * 8; }
        template <int K>
        static __device__ __forceinline__ void pair(const uint32_t *in, uint32_t *out)
        {
                if constexpr (K < 4) {
                        constexpr color_coeffs c = CS::at(16);
                        const int r0 = gh<6 * K>(in), g0 = gh<6 * K + 1>(in), b0 = gh<6 * K + 2>(in), r1 = gh<6 * K + 3>(in), g1 = gh<6 * K + 4>(in),
                                  b1 = gh<6 * K + 5>(in);
                        const int y0 = ((r0 * c.y_r + g0 * c.y_g + b0 * c.y_b) >> COMP_BASE) + 4096, y1 = ((r1 * c.y_r + g1 * c.y_g + b1 * c.y_b) >> COMP_BASE) + 4096;
                        const int u = (((r0 * c.cb_r + g0 * c.cb_g + b0 * c.cb_b) >> COMP_BASE) + ((r1 * c.cb_r + g1 * c.cb_g + b1 * c.cb_b) >> COMP_BASE)) / 2 + 32768;
                        const int v = (((r0 * c.cr_r + g0 * c.cr_g + b0 * c.cr_b) >> COMP_BASE) + ((r1 * c.cr_r + g1 * c.cr_g + b1 * c.cr_b) >> COMP_BASE)) / 2 + 32768;
                        out[2 * K] = ((uint32_t) y0 & 0xffff) | ((uint32_t) u & 0xffff) << 16;
                        out[2 * K + 1] = ((uint32_t) y1 & 0xffff) | ((uint32_t) v & 0xffff) << 16;
                        pair<K + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { pair<0>(in, out); }
};
/// vc_copylineRG48toV210, :2354-2407: depth-10 coefficients, shift COMP_BASE + 6; chroma shifted per pixel, summed, C '/ 2'
template <class CS = bt709>
struct conv_rg48_v210 {
        static constexpr int IN = 144, OUT = 64;
        static __host__ int out_len(int n) { return n < 16 ? 0 : n / 16 * 16; }
        template <int P>  // pixel pair P of the chunk (12 pairs): y1, y2, u, v
        static __device__ __forceinline__ void fetch(const uint32_t *in, uint32_t &y1, uint32_t &y2, uint32_t &u, uint32_t &v)
        {
                constexpr color_coeffs c = CS::at(10);
                constexpr int OFF = COMP_BASE + 6;
                const int r0 = gh<6 * P>(in), g0 = gh<6 * P + 1>(in), b0 = gh<6 * P + 2>(in), r1 = gh<6 * P + 3>(in), g1 = gh<6 * P + 4>(in), b1 = gh<6 * P + 5>(in);
                y1 = (uint32_t) (((r0 * c.y_r + g0 * c.y_g + b0 * c.y_b) >> OFF) + 64);
                y2 = (uint32_t) (((r1 * c.y_r + g1 * c.y_g + b1 * c.y_b) >> OFF) + 64);
                u = (uint32_t) ((((r0 * c.cb_r + g0 * c.cb_g + b0 * c.cb_b) >> OFF) + ((r1 * c.cb_r + g1 * c.cb_g + b1 * c.cb_b) >> OFF)) / 2 + 512);
                v = (uint32_t) ((((r0 * c.cr_r + g0 * c.cr_g + b0 * c.cr_b) >> OFF) + ((r1 * c.cr_r + g1 * c.cr_g + b1 * c.cr_b) >> OFF)) / 2 + 512);
        }
        template <int G>
        static __device__ __forceinline__ void group(const uint32_t *in, uint32_t *out)
        {
                if constexpr (G < 4) {
                        uint32_t ya, yb, u0, v0, yc, yd, u1, v1, ye, yf, u2, v2;
                        fetch<3 * G>(in, ya, yb, u0, v0);
                        fetch<3 * G + 1>(in, yc, yd, u1, v1);
                        fetch<3 * G + 2>(in, ye, yf, u2, v2);
                        out[4 * G + 0] = u0 | ya << 10 | v0 << 20;
                        out[4 * G + 1] = yb | u1 << 10 | yc << 20;
                        out[4 * G + 2] = v1 | yd << 10 | u2 << 20;
                        out[4 * G + 3] = ye | v2 << 10 | yf << 20;
                        group<G + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { group<0>(in, out); }
};
/// vc_copylineUYVYtoRG48, :1124-1130 = copylineYUVtoRGB with rgb16: each 8-bit result in the HIGH byte of a 16-bit sample
template <class CS = bt709>
struct conv_uyvy_rg48 {
        static constexpr int IN = 16, OUT = 48;
        static __host__ int out_len(int n) { return n < 12 ? 0 : n / 12 * 12; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(8);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint32_t w = in[i];
                        const int y1 = c.y_scale * ((int) ((w >> 8) & 0xff) - 16), y2 = c.y_scale * ((int) (w >> 24) - 16);
                        const int u = (int) (w & 0xff) - 128, v = (int) ((w >> 16) & 0xff) - 128;
                        const int rc = v * c.r_cr, gc = u * c.g_cb + v * c.g_cr, bc = u * c.b_cb;
                        const uint32_t r1 = clamp255((y1 + rc) >> COMP_BASE), g1 = clamp255((y1 + gc) >> COMP_BASE), b1 = clamp255((y1 + bc) >> COMP_BASE);
                        const uint32_t r2 = clamp255((y2 + rc) >> COMP_BASE), g2 = clamp255((y2 + gc) >> COMP_BASE), b2 = clamp255((y2 + bc) >> COMP_BASE);
                        out[3 * i] = r1 << 8 | g1 << 24, out[3 * i + 1] = b1 << 8 | r2 << 24, out[3 * i + 2] = g2 << 8 | b2 << 24;
                }
        }
};
/// vc_copyliner10ktoY416, :294-329 (components widened to 16 bit, depth-16 coefficients) and vc_copylineR10ktoUYVY, :2318-2334
/// (8-bit truncation, then the RGB -> UYVY body)
template <class CS = bt709>
struct conv_r10k_y416 {
        static constexpr int IN = 32, OUT = 64;
        static __host__ int out_len(int n) { return (n + 7) / 8 * 8; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(16);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        const int b1 = in[i] & 0xff, b2 = (in[i] >> 8) & 0xff, b3 = (in[i] >> 16) & 0xff, b4 = in[i] >> 24;
                        const int r = b1 << 8 | (b2 & 0xC0), g = (b2 & 0x3F) << 10 | (b3 & 0xF0) << 2, b = (b3 & 0xF) << 12 | (b4 & 0xFC) << 4;
                        const uint32_t u = ((r * c.cb_r + g * c.cb_g + b * c.cb_b) >> COMP_BASE) + 32768, y = ((r * c.y_r + g * c.y_g + b * c.y_b) >> COMP_BASE) + 4096,
                                       v = ((r * c.cr_r + g * c.cr_g + b * c.cr_b) >> COMP_BASE) + 32768;
                        out[2 * i] = (u & 0xffff) | (y & 0xffff) << 16;
                        out[2 * i + 1] = (v & 0xffff) | 0xFFFF0000u;
                }
        }
};
template <class CS = bt709>
struct conv_r10k_uyvy {
        static constexpr int IN = 32, OUT = 16;
        static __host__ int out_len(int n) { return (n + 3) / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(8);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        int r[2], g[2], b[2];
#pragma unroll
                        for (int k = 0; k < 2; ++k) {
                                const uint32_t w = in[2 * i + k];
                                r[k] = w & 0xff, g[k] = (((w >> 8) & 0xff) << 2 | ((w >> 16) & 0xff) >> 6) & 0xff, b[k] = (((w >> 16) & 0xff) << 4 | (w >> 24) >> 4) & 0xff;
                        }
                        const int y1 = ((r[0] * c.y_r + g[0] * c.y_g + b[0] * c.y_b) >> COMP_BASE) + 16, y2 = ((r[1] * c.y_r + g[1] * c.y_g + b[1] * c.y_b) >> COMP_BASE) + 16;
                        int u = (r[0] * c.cb_r + g[0] * c.cb_g + b[0] * c.cb_b) + (r[1] * c.cb_r + g[1] * c.cb_g + b[1] * c.cb_b);
                        int v = (r[0] * c.cr_r + g[0] * c.cr_g + b[0] * c.cr_b) + (r[1] * c.cr_r + g[1] * c.cr_g + b[1] * c.cr_b);
                        u = ((u / 2) >> COMP_BASE) + 128, v = ((v / 2) >> COMP_BASE) + 128;
                        out[i] = pack4(u & 0xff, y1 & 0xff, v & 0xff, y2 & 0xff);
                }
        }
};

/// R12L -> Y416 (vc_copylineR12LtoY416, :1478-1542; components << 4, depth-16 coefficients) and
/// R12L -> UYVY (vc_copylineR12LtoUYVY, :1544-1638; depth-8 coefficients on 16-bit components, one shift of COMP_BASE + 8 (+1 for chroma))
template <class CS = bt709>
struct conv_r12l_y416 {
        static constexpr int IN = 144, OUT = 256;
        static __host__ int out_len(int n) { return (n + 63) / 64 * 64; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(16);
#pragma unroll
                for (int g = 0; g < 4; ++g) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                const int r = r12_get(in + 9 * g, 3 * i) << 4, gg = r12_get(in + 9 * g, 3 * i + 1) << 4, b = r12_get(in + 9 * g, 3 * i + 2) << 4;
                                const uint32_t u = ((r * c.cb_r + gg * c.cb_g + b * c.cb_b) >> COMP_BASE) + 32768, y = ((r * c.y_r + gg * c.y_g + b * c.y_b) >> COMP_BASE) + 4096,
                                               v = ((r * c.cr_r + gg * c.cr_g + b * c.cr_b) >> COMP_BASE) + 32768;
                                out[2 * (8 * g + i)] = (u & 0xffff) | (y & 0xffff) << 16;
                                out[2 * (8 * g + i) + 1] = (v & 0xffff) | 0xFFFF0000u;
                        }
                }
        }
};
template <class CS = bt709>
struct conv_r12l_uyvy {
        static constexpr int IN = 144, OUT = 64;
        static __host__ int out_len(int n) { return (n + 15) / 16 * 16; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
                constexpr color_coeffs c = CS::at(8);
#pragma unroll
                for (int g = 0; g < 4; ++g) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                                int r[2], gg[2], b[2];
#pragma unroll
                                for (int k = 0; k < 2; ++k) {
                                        r[k] = r12_get(in + 9 * g, 6 * i + 3 * k) << 4, gg[k] = r12_get(in + 9 * g, 6 * i + 3 * k + 1) << 4,
                                        b[k] = r12_get(in + 9 * g, 6 * i + 3 * k + 2) << 4;
                                }
                                const int u = (((r[0] * c.cb_r + gg[0] * c.cb_g + b[0] * c.cb_b) + (r[1] * c.cb_r + gg[1] * c.cb_g + b[1] * c.cb_b)) >> (COMP_BASE + 9)) + 128;
                                const int v = (((r[0] * c.cr_r + gg[0] * c.cr_g + b[0] * c.cr_b) + (r[1] * c.cr_r + gg[1] * c.cr_g + b[1] * c.cr_b)) >> (COMP_BASE + 9)) + 128;
                                const int y0 = ((r[0] * c.y_r + gg[0] * c.y_g + b[0] * c.y_b) >> (COMP_BASE + 8)) + 16;
                                const int y1 = ((r[1] * c.y_r + gg[1] * c.y_g + b[1] * c.y_b) >> (COMP_BASE + 8)) + 16;
                                out[4 * g + i] = pack4(u & 0xff, y0 & 0xff, v & 0xff, y1 & 0xff);
                        }
                }
        }
};

/// DVS10 -> v210 (vc_copylineDVS10toV210, pixfmt_conv.c:595-618): the 2 LSBs of the three samples live in byte 3 of each word
struct conv_dvs10_v210 {
        static constexpr int IN = 16, OUT = 16;
        static __host__ int out_len(int n) { return n / 4 * 4; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint32_t a = in[i];
                        out[i] = (((a >> 24) * 0x00010101u) & 0x00300c03u) | ((a << 2) & (0xffu << 2)) | ((a << 4) & (0xff00u << 4)) | ((a << 6) & (0xff0000u << 6));
                }
        }
};

// ---- generic kernel ------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(256) line_conv_kernel(uint8_t *__restrict__ dst, long dst_pitch, const uint8_t *__restrict__ src,
                                                        long src_pitch, int wlen, int height, long src_total, bool vec_ok,
                                                        conv_params p)
{
        constexpr int NI = C::IN / 4, NO = C::OUT / 4;
        const int cx = blockIdx.x * blockDim.x + threadIdx.x;
        const long out_off = (long) cx * C::OUT;
        if (out_off >= wlen) {
                return;
        }
        const long in_off = (long) cx * C::IN;
        // Some reference loops write a whole pixel group past dst_len.  In the CPU row loop the next row then overwrites the
        // spill; rows run concurrently here, so every row but the last stops at the pitch (same final bytes, no race).
        const int wlen_last = wlen;
        for (int row = blockIdx.y; row < height; row += gridDim.y) {
                const int wlen = (row == height - 1 || wlen_last <= dst_pitch) ? wlen_last : (int) dst_pitch;
                if (out_off >= wlen) {
                        continue;
                }
                const long in_abs = row * src_pitch + in_off;
                uint32_t in[NI], out[NO];
                if (vec_ok && in_abs + C::IN <= src_total) {
                        const uint4 *s = (const uint4 *) (src + in_abs);
#pragma unroll
                        for (int i = 0; i < NI / 4; ++i) {
                                uint4 v;
                                if (NI >= 16) {  // four or more 16-byte pieces per thread: neighbouring lanes are 64+ bytes apart and every piece touches a
                                                 // fresh part of lines the previous one already pulled in - let L1 keep them (chosen on an earlier GPU,
                                                 // not re-measured on the H100; with two or three pieces per thread the streaming load is used)
                                        v = __ldg(s + i);
                                } else {
                                        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                                                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                                                     : "l"(s + i));
                                }
                                in[4 * i] = v.x, in[4 * i + 1] = v.y, in[4 * i + 2] = v.z, in[4 * i + 3] = v.w;
                        }
                } else {
#pragma unroll
                        for (int i = 0; i < NI; ++i) {
                                uint32_t w = 0;
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                        const long a = in_abs + 4 * i + k;
                                        if (a < src_total) {
                                                w |= (uint32_t) src[a] << (8 * k);
                                        }
                                }
                                in[i] = w;
                        }
                }
                const row_ctx rc = { src, row * src_pitch, src_total, cx };
                C::run(in, out, p, rc);
                uint8_t *d = dst + row * dst_pitch + out_off;
                const bool full = vec_ok && out_off + C::OUT <= wlen;
                if (full) {
#pragma unroll
                        for (int i = 0; i < NO / 4; ++i) {
                                ((uint4 *) d)[i] = make_uint4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
                        }
                } else {
#pragma unroll
                        for (int i = 0; i < NO; ++i) {
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                        if (out_off + 4 * i + k < wlen) {
                                                d[4 * i + k] = (uint8_t) (out[i] >> (8 * k));
                                        }
                                }
                        }
                }
        }
}

// ---- staged kernel: the same converter structs behind coalesced global accesses --------------------------------------------
// A thread of line_conv_kernel owns C::IN input bytes and C::OUT output bytes; with chunks of 64 bytes and more, the lanes of a warp sit 64-256 bytes
// apart and every 16-byte access of a warp touches 32 different cache lines (each line several times over the unrolled accesses): the L1 tag stage, one
// line per clock, becomes the limiter (R12L family, v210 -> RG48).  Here a CTA of T threads moves the T chunks
// of a row span as ONE contiguous byte run - 16 bytes per lane, 512 contiguous bytes per warp access - through shared memory: global -> shared
// (chunk c at 16-byte unit c * SI, SI = units per chunk made odd so that the per-thread 128-bit shared accesses of a quarter warp fall into distinct
// banks), C::run on registers exactly as in line_conv_kernel, registers -> shared (stride SO) -> global.  Used when pointers and pitches are 16-byte
// aligned (vec_ok) and the converter is marked staged (staged_default below); results are identical by construction.
template <class C, int T, bool SIN, bool SOUT>
__global__ void __launch_bounds__(T) line_conv_staged_kernel(uint8_t *__restrict__ dst, long dst_pitch, const uint8_t *__restrict__ src, long src_pitch,
                                                             int wlen_last, int height, long src_total, conv_params p)
{
        constexpr int NI = C::IN / 4, NO = C::OUT / 4, UI = C::IN / 16, UO = C::OUT / 16, SI = UI | 1, SO = UO | 1;
        static_assert(C::IN % 16 == 0 && C::OUT % 16 == 0, "chunks are whole 16-byte units");
        static_assert(SIN || SOUT, "the unstaged form is line_conv_kernel");
        __shared__ uint4 sm[T * ((SIN ? SI : 0) > (SOUT ? SO : 0) ? SI : SO)];
        const int tid = threadIdx.x, chunk0 = blockIdx.x * T;
        const long out_base = (long) chunk0 * C::OUT, in_base_row = (long) chunk0 * C::IN;
        for (int row = blockIdx.y; row < height; row += gridDim.y) {
                const int wlen = (row == height - 1 || wlen_last <= dst_pitch) ? wlen_last : (int) dst_pitch;  // see line_conv_kernel
                if (out_base >= wlen) {
                        continue;  // uniform for the CTA
                }
                const long left = wlen - out_base;
                const bool whole = left >= (long) T * C::OUT;  // all T chunks of the CTA are whole
                const int nchunks = whole ? T : (int) ((left + C::OUT - 1) / C::OUT);
                const long in_abs0 = row * src_pitch + in_base_row;
                uint32_t in[NI], out[NO];
                if (SIN) {  // global -> shared, linear in the byte run
                        if (whole && in_abs0 + (long) T * C::IN <= src_total) {
                                uint4 v[UI];
#pragma unroll
                                for (int i = 0; i < UI; ++i) {  // all loads of the thread in flight before the first shared store
                                        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                                                     : "=r"(v[i].x), "=r"(v[i].y), "=r"(v[i].z), "=r"(v[i].w)
                                                     : "l"(src + in_abs0 + 16l * (tid + i * T)));
                                }
#pragma unroll
                                for (int i = 0; i < UI; ++i) {
                                        const int j = tid + i * T, c = j / UI, k = j - c * UI;
                                        sm[c * SI + k] = v[i];
                                }
                        } else {
                                for (int j = tid; j < nchunks * UI; j += T) {
                                        const int c = j / UI, k = j - c * UI;
                                        const long a = in_abs0 + 16l * j;
                                        uint32_t w[4] = { 0, 0, 0, 0 };
                                        for (int b = 0; b < 16; ++b) {  // reads past src_size give 0 (include/ugb200.h)
                                                if (a + b < src_total) {
                                                        w[b >> 2] |= (uint32_t) src[a + b] << (8 * (b & 3));
                                                }
                                        }
                                        sm[c * SI + k] = make_uint4(w[0], w[1], w[2], w[3]);
                                }
                        }
                        __syncthreads();
                        if (tid < nchunks) {
#pragma unroll
                                for (int i = 0; i < UI; ++i) {
                                        const uint4 v = sm[tid * SI + i];
                                        in[4 * i] = v.x, in[4 * i + 1] = v.y, in[4 * i + 2] = v.z, in[4 * i + 3] = v.w;
                                }
                        }
                        if (SOUT) {
                                __syncthreads();  // the output image reuses the staging buffer
                        }
                } else if (tid < nchunks) {  // own chunk straight from global memory, as line_conv_kernel
                        const long in_abs = in_abs0 + (long) tid * C::IN;
                        if (in_abs + C::IN <= src_total) {
                                const uint4 *s4 = (const uint4 *) (src + in_abs);
#pragma unroll
                                for (int i = 0; i < UI; ++i) {
                                        uint4 v;
                                        if (NI >= 16) {
                                                v = __ldg(s4 + i);
                                        } else {
                                                asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(s4 + i));
                                        }
                                        in[4 * i] = v.x, in[4 * i + 1] = v.y, in[4 * i + 2] = v.z, in[4 * i + 3] = v.w;
                                }
                        } else {
#pragma unroll
                                for (int i = 0; i < NI; ++i) {
                                        uint32_t w = 0;
#pragma unroll
                                        for (int k = 0; k < 4; ++k) {
                                                const long a = in_abs + 4 * i + k;
                                                if (a < src_total) {
                                                        w |= (uint32_t) src[a] << (8 * k);
                                                }
                                        }
                                        in[i] = w;
                                }
                        }
                }
                if (tid < nchunks) {
                        const row_ctx rc = { src, row * src_pitch, src_total, chunk0 + tid };
                        C::run(in, out, p, rc);
                }
                uint8_t *d = dst + row * dst_pitch + out_base;
                if (SOUT) {
                        if (tid < nchunks) {
#pragma unroll
                                for (int i = 0; i < UO; ++i) {
                                        sm[tid * SO + i] = make_uint4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
                                }
                        }
                        __syncthreads();
                        // shared -> global: whole 16-byte units, then the bytes of a last partial unit (wlen need not be a multiple of 16)
                        if (whole) {
#pragma unroll
                                for (int i = 0; i < UO; ++i) {
                                        const int j = tid + i * T, c = j / UO, k = j - c * UO;
                                        ((uint4 *) d)[j] = sm[c * SO + k];
                                }
                        } else {
                                const long nbytes = left < (long) nchunks * C::OUT ? left : (long) nchunks * C::OUT;
                                const int nfull = (int) (nbytes >> 4);
                                for (int j = tid; j < nfull; j += T) {
                                        const int c = j / UO, k = j - c * UO;
                                        ((uint4 *) d)[j] = sm[c * SO + k];
                                }
                                if (tid < (int) (nbytes & 15)) {
                                        const int j = nfull, c = j / UO, k = j - c * UO;
                                        d[16l * j + tid] = ((const uint8_t *) &sm[c * SO + k])[tid];
                                }
                        }
                        __syncthreads();  // before the next row touches the buffer
                } else if (tid < nchunks) {  // own chunk straight to global memory
                        const long out_off = (long) tid * C::OUT;
                        if (out_base + out_off + C::OUT <= wlen) {
#pragma unroll
                                for (int i = 0; i < UO; ++i) {
                                        ((uint4 *) (d + out_off))[i] = make_uint4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
                                }
                        } else {
#pragma unroll
                                for (int i = 0; i < NO; ++i) {
#pragma unroll
                                        for (int k = 0; k < 4; ++k) {
                                                if (out_base + out_off + 4 * i + k < wlen) {
                                                        d[out_off + 4 * i + k] = (uint8_t) (out[i] >> (8 * k));
                                                }
                                        }
                                }
                        }
                }
                if (SIN && !SOUT) {
                        __syncthreads();  // the next row's fill must not overtake this row's reads (the row loop only repeats for height > 65535)
                }
        }
}

/// which converters take the staged kernel by default; UGB200_LINE_STAGED=0 / 1 forces none / all (experiments)
template <class C>
struct staged_default {
        static constexpr int value = 0;  // 0 direct, 1 input and output staged, 2 output only, 3 input only
};
// chosen by timing all four forms of every converter at 7680x4320 on an earlier GPU (gains of 5 % and more); carried over, not re-measured on the H100
// (tools/pixfmt_sweep.py repeats the sweep).  The pattern: staging
// the OUTPUT pays wherever a thread's output chunk is large or oddly sized (36-byte R12L groups, 48-byte RG48 / Y416 runs): the direct form stores 16 bytes
// per lane at a stride of the whole chunk.  Staging the input almost never pays - strided 16-byte loads of a warp hit L1 lines the previous load brought in.
#define UGB_STAGED(CONV, MODE)                                                                                                                \
        template <>                                                                                                                           \
        struct staged_default<CONV> {                                                                                                         \
                static constexpr int value = MODE;                                                                                            \
        };
// converters that read colour coefficients: one form for every coefficient set (the sets differ in immediates only)
#define UGB_STAGED_CS(MODE, ...)                                                                                                              \
        template <class CS>                                                                                                                   \
        struct staged_default<__VA_ARGS__> {                                                                                                  \
                static constexpr int value = MODE;                                                                                            \
        };
UGB_STAGED_CS(2, conv_v210_rg48<CS>)
UGB_STAGED(conv_r12l_rgbx<0>, 2)     // R12L -> RGB
UGB_STAGED(conv_r12l_rgbx<1>, 2)     // R12L -> RGBA
UGB_STAGED(conv_r12l_rgbx<2>, 2)     // R12L -> RG48
UGB_STAGED(conv_r12l_rgbx<3>, 2)     // R12L -> R10k
UGB_STAGED_CS(2, conv_r12l_y416<CS>)
UGB_STAGED(conv_x_r12l<0>, 2)        // RGB  -> R12L
UGB_STAGED(conv_x_r12l<1>, 2)        // RGBA -> R12L
UGB_STAGED(conv_x_r12l<2>, 2)        // RG48 -> R12L
UGB_STAGED_CS(2, conv_x_r12l<3, CS>)  // Y416 -> R12L
UGB_STAGED(conv_rgb_rgba, 2)
UGB_STAGED(conv_bytemap<map_uyvy_y416>, 1)
UGB_STAGED_CS(2, conv_r10k_y416<CS>)
UGB_STAGED(conv_uyvy_v210, 2)
UGB_STAGED_CS(2, conv_vuya_rgb<CS>)
UGB_STAGED_CS(2, conv_rg48_y416<CS>)
UGB_STAGED(conv_r10k_rg48, 2)
UGB_STAGED(conv_v210_y416, 2)
UGB_STAGED_CS(2, conv_rg48_v210<CS>)
UGB_STAGED_CS(3, conv_rg48_y216<CS>)
UGB_STAGED(conv_v210_uyvy, 2)
UGB_STAGED(conv_rg48_r10k, 2)
#undef UGB_STAGED_CS
#undef UGB_STAGED

static int &staged_mode()
{
        static int v = [] {
                const char *e = getenv("UGB200_LINE_STAGED");
                return e == nullptr || e[0] == '\0' ? -1 : atoi(e);
        }();
        return v;
}
static int staged_override() { return staged_mode(); }

/// LEAN form of line_conv_kernel for the common case the host can guarantee up front: 16-byte aligned pointers and pitches, every chunk of every row whole, inside the
/// readable source and inside the destination pitch.  Nothing but the vector loads, C::run and the vector stores is compiled in - the byte-wise paths of the general
/// kernel cost registers (v210 -> RG48: 170) and instruction-cache footprint even when they never run (the lesson of the JPEG encoder's lean instantiation).
template <class C>
__global__ void __launch_bounds__(256) line_conv_lean_kernel(uint8_t *__restrict__ dst, long dst_pitch, const uint8_t *__restrict__ src, long src_pitch, int wlen, int height,
                                                             long src_total, conv_params p)
{
        constexpr int NI = C::IN / 4, NO = C::OUT / 4;
        const int cx = blockIdx.x * blockDim.x + threadIdx.x;
        const long out_off = (long) cx * C::OUT;
        if (out_off >= wlen) {
                return;
        }
        const long in_off = (long) cx * C::IN;
        for (int row = blockIdx.y; row < height; row += gridDim.y) {
                uint32_t in[NI], out[NO];
                const uint4 *s4 = (const uint4 *) (src + row * src_pitch + in_off);
#pragma unroll
                for (int i = 0; i < NI / 4; ++i) {
                        uint4 v;
                        if (NI >= 16) {
                                v = __ldg(s4 + i);
                        } else {
                                asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(s4 + i));
                        }
                        in[4 * i] = v.x, in[4 * i + 1] = v.y, in[4 * i + 2] = v.z, in[4 * i + 3] = v.w;
                }
                const row_ctx rc = { src, row * src_pitch, src_total, cx };
                C::run(in, out, p, rc);
                uint4 *d4 = (uint4 *) (dst + row * dst_pitch + out_off);
#pragma unroll
                for (int i = 0; i < NO / 4; ++i) {
                        d4[i] = make_uint4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
                }
        }
}

/// which converters take the lean kernel by default: the ones it timed at least 5 % faster for at 8K on an earlier GPU, carried over and not re-measured on the
/// H100 (it was slower for a few, v210 -> RGB among them: with fewer registers ptxas schedules the long arithmetic chains with less overlap).  UGB200_LINE_LEAN=0 / 1: none / all.
template <class C>
struct lean_default {
        static constexpr bool value = false;
};
#define UGB_LEAN(...)                                                                                                                         \
        template <>                                                                                                                           \
        struct lean_default<__VA_ARGS__> {                                                                                                    \
                static constexpr bool value = true;                                                                                           \
        };
#define UGB_LEAN_CS(...)                                                                                                                      \
        template <class CS>                                                                                                                   \
        struct lean_default<__VA_ARGS__> {                                                                                                    \
                static constexpr bool value = true;                                                                                           \
        };
UGB_LEAN(conv_uyvy_rgba)
UGB_LEAN(conv_r10k_rgba)
UGB_LEAN_CS(conv_uyvy_rg48<CS>)
UGB_LEAN_CS(conv_rgba_vuya<CS>)
UGB_LEAN_CS(conv_to_uyvy<2, 1, 0, 3, CS>)  // BGR  -> UYVY
UGB_LEAN_CS(conv_to_uyvy<0, 1, 2, 4, CS>)  // RGBA -> UYVY
UGB_LEAN(conv_rgba_r10k)
UGB_LEAN_CS(conv_y416_rgbx<3, CS>)         // Y416 -> R10k
UGB_LEAN_CS(conv_y416_rgbx<2, CS>)         // Y416 -> RGBA
UGB_LEAN(conv_vuya_uyvy)
#undef UGB_LEAN_CS
#undef UGB_LEAN

template <class C>
static int launch_line(void *dst, long dst_pitch, const void *src, long src_pitch, int dst_len, int height, long src_size,
                       conv_params p, cudaStream_t s)
{
        const int wlen = C::out_len(dst_len);
        if (wlen <= 0 || height <= 0) {
                return 0;
        }
        if (src_size <= 0) {
                src_size = src_pitch * height;
        }
        const bool vec_ok = !(15 & (size_t) dst) && !(15 & (size_t) src) && !(dst_pitch & 15) && !(src_pitch & 15);
        const int chunks = (wlen + C::OUT - 1) / C::OUT;
        const int threads = 128;
        dim3 grid((chunks + threads - 1) / threads, height > 65535 ? 65535 : height);
        if constexpr (C::IN % 16 == 0 && C::OUT % 16 == 0) {
                const int ov = staged_override();
                const int mode = !vec_ok ? 0 : ov < 0 ? staged_default<C>::value : ov;
                if (mode == 1) {
                        line_conv_staged_kernel<C, threads, true, true><<<grid, threads, 0, s>>>((uint8_t *) dst, dst_pitch, (const uint8_t *) src, src_pitch, wlen, height, src_size, p);
                } else if (mode == 2) {
                        line_conv_staged_kernel<C, threads, false, true><<<grid, threads, 0, s>>>((uint8_t *) dst, dst_pitch, (const uint8_t *) src, src_pitch, wlen, height, src_size, p);
                } else if (mode == 3) {
                        line_conv_staged_kernel<C, threads, true, false><<<grid, threads, 0, s>>>((uint8_t *) dst, dst_pitch, (const uint8_t *) src, src_pitch, wlen, height, src_size, p);
                }
                if (mode != 0) {
                        return cudaGetLastError() == cudaSuccess ? 0 : -2;
                }
        }
        if constexpr (C::IN % 16 == 0 && C::OUT % 16 == 0) {
                static const int lean_env = getenv("UGB200_LINE_LEAN") == nullptr ? -1 : atoi(getenv("UGB200_LINE_LEAN"));
                const bool allow_lean = lean_env < 0 ? lean_default<C>::value : lean_env != 0;
                if (allow_lean && vec_ok && wlen % C::OUT == 0 && wlen <= dst_pitch && (long) (height - 1) * src_pitch + (long) chunks * C::IN <= src_size) {
                        line_conv_lean_kernel<C><<<grid, threads, 0, s>>>((uint8_t *) dst, dst_pitch, (const uint8_t *) src, src_pitch, wlen, height, src_size, p);
                        return cudaGetLastError() == cudaSuccess ? 0 : -2;
                }
        }
        line_conv_kernel<C><<<grid, threads, 0, s>>>((uint8_t *) dst, dst_pitch, (const uint8_t *) src, src_pitch, wlen, height,
                                                     src_size, vec_ok, p);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

/// rows [row0, height) of copy_rows, byte by byte: reads past src_total give 0 (include/ugb200.h)
__global__ void __launch_bounds__(256) copy_rows_tail_kernel(uint8_t *__restrict__ dst, long dst_pitch, const uint8_t *__restrict__ src, long src_pitch, int len,
                                                             int row0, int height, long src_total)
{
        const long n = (long) (height - row0) * len;
        for (long i = blockIdx.x * (long) blockDim.x + threadIdx.x; i < n; i += (long) gridDim.x * blockDim.x) {
                const long row = row0 + i / len, x = i % len, a = row * src_pitch + x;
                dst[row * dst_pitch + x] = a < src_total ? src[a] : 0;
        }
}

/// vc_memcpy over the rows: the rows that lie inside src_size in one cudaMemcpy2DAsync, the rest (where the source ends) by copy_rows_tail_kernel
static int copy_rows(void *dst, long dst_pitch, const void *src, long src_pitch, int len, int height, long src_size, cudaStream_t s)
{
        if (len <= 0 || height <= 0) {
                return 0;
        }
        if (src_size <= 0) {
                src_size = src_pitch * height;
        }
        const long whole = src_size < len ? 0 : (src_size - len) / src_pitch + 1 < height ? (src_size - len) / src_pitch + 1 : height;
        if (whole > 0 && cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, len, whole, cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
                return -2;
        }
        if (whole == height) {
                return 0;
        }
        const long n = (height - whole) * (long) len, blocks = (n + 255) / 256;
        copy_rows_tail_kernel<<<(int) (blocks < 4096 ? blocks : 4096), 256, 0, s>>>((uint8_t *) dst, dst_pitch, (const uint8_t *) src, src_pitch, len, (int) whole,
                                                                                  height, src_size);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace ugb

using namespace ugb;

extern "C" UGB_API int ugb200_vc_copyline(int func, void *dst, long dst_pitch, const void *src, long src_pitch, int dst_len, int height, long src_size,
                                          int rshift, int gshift, int bshift, cuda_wrapper_stream_t stream)
{
        if (dst == nullptr || src == nullptr || dst_len < 0 || height < 0 || dst_pitch <= 0 || src_pitch <= 0) {
                return -1;
        }
        cudaStream_t s = (cudaStream_t) stream;
        switch (func) {
        case UGB_LINE_ABGR_TO_RGB:
                return launch_line<conv_abgr_rgb>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, conv_params{ 0, 8, 16, conv_abgr_rgb::aux(dst_len) }, s);
        case UGB_LINE_BGRA_TO_RGB:
                return launch_line<conv_bgra_rgb>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, conv_params{ 0, 8, 16, conv_bgra_rgb::aux(dst_len) }, s);
        case UGB_LINE_TO_RGBA_INPLACE:
                if ((unsigned) rshift > 24 || (unsigned) gshift > 24 || (unsigned) bshift > 24) {
                        return -1;
                }
                return launch_line<conv_to_rgba_inplace>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, conv_params{ rshift, gshift, bshift, 0 }, s);
        case UGB_LINE_UYVY_TO_GRAYSCALE:
                return launch_line<conv_bytemap<map_uyvy_gray>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, conv_params{ 0, 8, 16, 0 }, s);
        default:
                return -4;
        }
}

extern "C" UGB_API int ugb200_pixfmt_staged_mode(int mode)
{
        const int prev = staged_mode();
        staged_mode() = mode < 0 || mode > 3 ? -1 : mode;
        return prev;
}

extern "C" UGB_API int ugb200_pixfmt_supported(int in_codec, int out_codec)
{
        if (in_codec == out_codec && out_codec != UGB_RGBA && out_codec != UGB_RGB) {
                return in_codec > UGB_VIDEO_CODEC_NONE && in_codec < UGB_VIDEO_CODEC_COUNT;  // vc_memcpy, pixfmt_conv.c:3111-3114
        }
        switch (in_codec * 256 + out_codec) {
        case UGB_v210 * 256 + UGB_UYVY:
        case UGB_YUYV * 256 + UGB_UYVY:
        case UGB_UYVY * 256 + UGB_YUYV:
        case UGB_UYVY * 256 + UGB_RGB:
        case UGB_YUYV * 256 + UGB_RGB:
        case UGB_UYVY * 256 + UGB_RGBA:
        case UGB_RGB * 256 + UGB_UYVY:
        case UGB_BGR * 256 + UGB_UYVY:
        case UGB_RGBA * 256 + UGB_UYVY:
        case UGB_RG48 * 256 + UGB_UYVY:
        case UGB_RGB * 256 + UGB_RGBA:
        case UGB_RGBA * 256 + UGB_RGB:
        case UGB_RGBA * 256 + UGB_RGBA:
        case UGB_RGB * 256 + UGB_RGB:
        case UGB_BGR * 256 + UGB_RGB:
        case UGB_UYVY * 256 + UGB_v210:
        case UGB_Y216 * 256 + UGB_v210:
        case UGB_v210 * 256 + UGB_Y216:
        case UGB_v210 * 256 + UGB_Y416:
        case UGB_v210 * 256 + UGB_RGB:
        case UGB_v210 * 256 + UGB_RG48:
        case UGB_RG48 * 256 + UGB_RGB:
        case UGB_RGBA * 256 + UGB_RG48:
        case UGB_RGB * 256 + UGB_RG48:
        case UGB_UYVY * 256 + UGB_Y216:
        case UGB_UYVY * 256 + UGB_Y416:
        case UGB_Y216 * 256 + UGB_UYVY:
        case UGB_VUYA * 256 + UGB_Y416:
        case UGB_R10k * 256 + UGB_RGBA:
        case UGB_R10k * 256 + UGB_RGB:
        case UGB_R10k * 256 + UGB_RG48:
        case UGB_RGBA * 256 + UGB_R10k:
        case UGB_RG48 * 256 + UGB_R10k:
        case UGB_RG48 * 256 + UGB_RGBA:
        case UGB_VUYA * 256 + UGB_UYVY:
        case UGB_Y416 * 256 + UGB_UYVY:
        case UGB_VUYA * 256 + UGB_RGB:
        case UGB_RGBA * 256 + UGB_VUYA:
        case UGB_Y416 * 256 + UGB_RG48:
        case UGB_Y416 * 256 + UGB_RGB:
        case UGB_Y416 * 256 + UGB_RGBA:
        case UGB_Y416 * 256 + UGB_R10k:
        case UGB_Y416 * 256 + UGB_v210:
        case UGB_RG48 * 256 + UGB_Y416:
        case UGB_RG48 * 256 + UGB_Y216:
        case UGB_RG48 * 256 + UGB_v210:
        case UGB_UYVY * 256 + UGB_RG48:
        case UGB_R10k * 256 + UGB_Y416:
        case UGB_R10k * 256 + UGB_UYVY:
        case UGB_DVS10 * 256 + UGB_UYVY:
        case UGB_DVS10 * 256 + UGB_v210:
        case UGB_R12L * 256 + UGB_RGB:
        case UGB_R12L * 256 + UGB_RGBA:
        case UGB_R12L * 256 + UGB_RG48:
        case UGB_R12L * 256 + UGB_R10k:
        case UGB_R12L * 256 + UGB_Y416:
        case UGB_R12L * 256 + UGB_UYVY:
        case UGB_RGB * 256 + UGB_R12L:
        case UGB_RGBA * 256 + UGB_R12L:
        case UGB_RG48 * 256 + UGB_R12L:
        case UGB_Y416 * 256 + UGB_R12L:
                return 1;
        }
        return 0;
}

/// the 8-bit limited-range YCbCr space of conv_yuv422_rgb for a coefficient set
template <class CS>
struct ycbcr8;
template <>
struct ycbcr8<bt709> {
        using type = ycbcr_709;
};
template <>
struct ycbcr8<bt601> {
        using type = ycbcr_601;
};

/// ugb200_pixfmt_convert_cs with the coefficient set CS; converters that read no coefficients are the same instantiation for every CS
template <class CS>
static int pixfmt_convert(int in_codec, int out_codec, void *dst, long dst_pitch, const void *src, long src_pitch, int dst_len, int height, long src_size,
                          int rshift, int gshift, int bshift, cudaStream_t s)
{
        const conv_params p = { rshift, gshift, bshift, 0 };
        if (in_codec == out_codec && out_codec != UGB_RGBA && out_codec != UGB_RGB) {
                return copy_rows(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, s);  // vc_memcpy (pixfmt_conv.c:2529-2536)
        }
        const bool dfl_shift = rshift == 0 && gshift == 8 && bshift == 16;
        switch (in_codec * 256 + out_codec) {
        case UGB_v210 * 256 + UGB_UYVY:
                return launch_line<conv_v210_uyvy>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_YUYV * 256 + UGB_UYVY:
        case UGB_UYVY * 256 + UGB_YUYV:
                return launch_line<conv_yuyv_uyvy>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_UYVY * 256 + UGB_RGB:
                return launch_line<conv_yuv422_rgb<1, 3, 0, 2, typename ycbcr8<CS>::type>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_YUYV * 256 + UGB_RGB:
                return launch_line<conv_yuv422_rgb<0, 2, 1, 3, typename ycbcr8<CS>::type>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_UYVY * 256 + UGB_RGBA:
                return launch_line<conv_uyvy_rgba>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_RGB * 256 + UGB_UYVY:
                return launch_line<conv_to_uyvy<0, 1, 2, 3, CS>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_BGR * 256 + UGB_UYVY:
                return launch_line<conv_to_uyvy<2, 1, 0, 3, CS>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_RGBA * 256 + UGB_UYVY:
                return launch_line<conv_to_uyvy<0, 1, 2, 4, CS>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_RG48 * 256 + UGB_UYVY:
                return launch_line<conv_to_uyvy<1, 3, 5, 6, CS>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_RGB * 256 + UGB_RGBA:
                return launch_line<conv_rgb_rgba>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_RGBA * 256 + UGB_RGB:
                return launch_line<conv_rgba_rgb>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, conv_params{ 0, 8, 16, conv_rgba_rgb::aux(dst_len) }, s);
        case UGB_RGBA * 256 + UGB_RGBA:
                if (dfl_shift) {
                        return copy_rows(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, s);  // pixfmt_conv.c:546-547
                }
                return launch_line<conv_rgba_rgba>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_RGB * 256 + UGB_RGB:
                if (dfl_shift) {
                        return copy_rows(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, s);  // pixfmt_conv.c:740-741
                }
                return launch_line<conv_rgb_rgb>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_UYVY * 256 + UGB_v210:
                return launch_line<conv_uyvy_v210>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_Y216 * 256 + UGB_v210:
                return launch_line<conv_y216_v210>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_v210 * 256 + UGB_Y216:
                return launch_line<conv_v210_y216>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_v210 * 256 + UGB_Y416:
                return launch_line<conv_v210_y416>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
        case UGB_v210 * 256 + UGB_RGB:
                return launch_line<conv_v210_rgb<CS>>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
#define UGB_CASE(IN_C, OUT_C, ...)                                                                                                          \
        case IN_C * 256 + OUT_C:                                                                                                            \
                return launch_line<__VA_ARGS__>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, p, s);
                UGB_CASE(UGB_RG48, UGB_RGB, conv_bytemap<map_rg48_rgb>)
                UGB_CASE(UGB_RGBA, UGB_RG48, conv_bytemap<map_rgba_rg48>)
                UGB_CASE(UGB_RGB, UGB_RG48, conv_bytemap<map_rgb_rg48>)
                UGB_CASE(UGB_UYVY, UGB_Y216, conv_bytemap<map_uyvy_y216>)
                UGB_CASE(UGB_UYVY, UGB_Y416, conv_bytemap<map_uyvy_y416>)
                UGB_CASE(UGB_Y216, UGB_UYVY, conv_bytemap<map_y216_uyvy>)
                UGB_CASE(UGB_VUYA, UGB_Y416, conv_bytemap<map_vuya_y416>)
                UGB_CASE(UGB_R10k, UGB_RGBA, conv_r10k_rgba)
                UGB_CASE(UGB_R10k, UGB_RGB, conv_r10k_rgb)
                UGB_CASE(UGB_R10k, UGB_RG48, conv_r10k_rg48)
                UGB_CASE(UGB_RGBA, UGB_R10k, conv_rgba_r10k)
                UGB_CASE(UGB_RG48, UGB_R10k, conv_rg48_r10k)
                UGB_CASE(UGB_RG48, UGB_RGBA, conv_rg48_rgba)
                UGB_CASE(UGB_VUYA, UGB_UYVY, conv_vuya_uyvy)
                UGB_CASE(UGB_Y416, UGB_UYVY, conv_y416_uyvy)
                UGB_CASE(UGB_VUYA, UGB_RGB, conv_vuya_rgb<CS>)
                UGB_CASE(UGB_RGBA, UGB_VUYA, conv_rgba_vuya<CS>)
                UGB_CASE(UGB_Y416, UGB_RG48, conv_y416_rgbx<0, CS>)
                UGB_CASE(UGB_Y416, UGB_RGB, conv_y416_rgbx<1, CS>)
                UGB_CASE(UGB_Y416, UGB_RGBA, conv_y416_rgbx<2, CS>)
                UGB_CASE(UGB_Y416, UGB_R10k, conv_y416_rgbx<3, CS>)
                UGB_CASE(UGB_Y416, UGB_v210, conv_y416_v210)
                UGB_CASE(UGB_RG48, UGB_Y416, conv_rg48_y416<CS>)
                UGB_CASE(UGB_RG48, UGB_Y216, conv_rg48_y216<CS>)
                UGB_CASE(UGB_RG48, UGB_v210, conv_rg48_v210<CS>)
                UGB_CASE(UGB_UYVY, UGB_RG48, conv_uyvy_rg48<CS>)
                UGB_CASE(UGB_R10k, UGB_Y416, conv_r10k_y416<CS>)
                UGB_CASE(UGB_R10k, UGB_UYVY, conv_r10k_uyvy<CS>)
                UGB_CASE(UGB_v210, UGB_RG48, conv_v210_rg48<CS>)
                UGB_CASE(UGB_DVS10, UGB_UYVY, conv_bytemap<map_dvs10_uyvy>)
                UGB_CASE(UGB_DVS10, UGB_v210, conv_dvs10_v210)
                UGB_CASE(UGB_R12L, UGB_RGB, conv_r12l_rgbx<0>)
                UGB_CASE(UGB_R12L, UGB_RGBA, conv_r12l_rgbx<1>)
                UGB_CASE(UGB_R12L, UGB_RG48, conv_r12l_rgbx<2>)
                UGB_CASE(UGB_R12L, UGB_R10k, conv_r12l_rgbx<3>)
                UGB_CASE(UGB_R12L, UGB_Y416, conv_r12l_y416<CS>)
                UGB_CASE(UGB_R12L, UGB_UYVY, conv_r12l_uyvy<CS>)
                UGB_CASE(UGB_RGB, UGB_R12L, conv_x_r12l<0>)
                UGB_CASE(UGB_RGBA, UGB_R12L, conv_x_r12l<1>)
                UGB_CASE(UGB_RG48, UGB_R12L, conv_x_r12l<2>)
                UGB_CASE(UGB_Y416, UGB_R12L, conv_x_r12l<3, CS>)
#undef UGB_CASE
        case UGB_BGR * 256 + UGB_RGB: {
                const conv_params q = { 16, 8, 0, 0 };  // vc_copylineBGRtoRGB
                return launch_line<conv_rgb_rgb>(dst, dst_pitch, src, src_pitch, dst_len, height, src_size, q, s);
        }
        }
        return -4;  // no decoder (get_decoder_from_to() == NULL, pixfmt_conv.c:3122-3124)
}

extern "C" UGB_API int ugb200_pixfmt_convert_cs(int in_codec, int out_codec, void *dst, long dst_pitch, const void *src, long src_pitch, int dst_len,
                                                int height, long src_size, int rshift, int gshift, int bshift, int cs, cuda_wrapper_stream_t stream)
{
        if (dst == nullptr || src == nullptr || dst_len < 0 || height < 0) {
                return -1;
        }
        switch (cs) {
        case UGB_CS_DFL:
        case UGB_CS_709:
                return pixfmt_convert<bt709>(in_codec, out_codec, dst, dst_pitch, src, src_pitch, dst_len, height, src_size, rshift, gshift, bshift,
                                             (cudaStream_t) stream);
        case UGB_CS_601:
                return pixfmt_convert<bt601>(in_codec, out_codec, dst, dst_pitch, src, src_pitch, dst_len, height, src_size, rshift, gshift, bshift,
                                             (cudaStream_t) stream);
        default:
                return -1;
        }
}

extern "C" UGB_API int ugb200_pixfmt_convert(int in_codec, int out_codec, void *dst, long dst_pitch, const void *src, long src_pitch,
                                     int dst_len, int height, long src_size, int rshift, int gshift, int bshift,
                                     cuda_wrapper_stream_t stream)
{
        return ugb200_pixfmt_convert_cs(in_codec, out_codec, dst, dst_pitch, src, src_pitch, dst_len, height, src_size, rshift, gshift, bshift, UGB_CS_709,
                                        stream);
}

// ---- src/cuda_wrapper/kernels.cu under its own names (include/cuda_wrapper_kernels.hpp) ------------------------------------------------
// The reference's two callbacks are vc_copylineRG48toR12L / vc_copylineR12LtoRG48 run over tightly packed rows (kernels.cu:72-74,312 say so):
// the same converter structs, launched with the reference's row geometry.
#include "../../include/cuda_wrapper_kernels.hpp"

int postprocess_rg48_to_r12l(void *, void *, size_t, int size_x, int size_y, struct cmpto_j2k_dec_comp_format *, int, void *input_samples, size_t, void *, size_t,
                             void *output_buffer, size_t, void *stream)
{
        if (size_x <= 0 || size_y <= 0) {
                return (int) cudaSuccess;  // the reference launches an empty grid
        }
        const long r12_pitch = (long) ((size_x + 7) / 8) * 36, rg48_pitch = (long) size_x * 6;
        // dst_len = the whole R12L row: the last (partial) group is written too, as kernel_rg48_to_r12l does (kernels.cu:238-257)
        launch_line<conv_x_r12l<2>>(output_buffer, r12_pitch, input_samples, rg48_pitch, (int) r12_pitch, size_y, rg48_pitch * size_y, conv_params{ 0, 8, 16, 0 },
                                    (cudaStream_t) stream);
        return (int) cudaGetLastError();
}

int preprocess_r12l_to_rg48(void *, void *, size_t, int size_x, int size_y, struct cmpto_j2k_enc_comp_format *, int, void *input_samples, size_t, void *output_samples,
                            size_t, void *stream)
{
        if (size_x <= 0 || size_y <= 0) {
                return (int) cudaSuccess;
        }
        const long r12_pitch = (long) ((size_x + 7) / 8) * 36, rg48_pitch = (long) size_x * 6;
        launch_line<conv_r12l_rgbx<2>>(output_samples, rg48_pitch, input_samples, r12_pitch, (int) rg48_pitch, size_y, r12_pitch * size_y, conv_params{ 0, 8, 16, 0 },
                                       (cudaStream_t) stream);
        return (int) cudaGetLastError();
}
