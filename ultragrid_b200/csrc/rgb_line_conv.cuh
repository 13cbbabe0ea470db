// The RGB <-> RGBA, RG48 -> RGB, RGB -> RG48 and R12L <-> RGB-like line converters of pixfmt_kernels.cu as device
// functors, shared with the logo capture filter (logo_kernels.cu), whose fused kernel decodes a frame's pixels to RGB,
// blends them and encodes them back in registers, and with the R12L <-> Y416 pass-through filters (r12_get / r12_put).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "color_space.h"
#include "rgb_to_uyvy.cuh"
#include "yuv_rgb_conv.cuh"

namespace ugb {

__device__ __forceinline__ int clampr(int v, int lo, int hi) { return min(max(v, lo), hi); }

/// vc_copylineRGBtoRGBA, pixfmt_conv.c:944-990
struct conv_rgb_rgba {
        static constexpr int IN = 48, OUT = 64;
        static __host__ int out_len(int dst_len) { return dst_len < 4 ? 0 : dst_len / 4 * 4; }
        template <int K>
        static __device__ __forceinline__ void px(const uint32_t *in, uint32_t *out, const conv_params &p, uint32_t amask)
        {
                if constexpr (K < 16) {
                        out[K] = amask | gb<3 * K>(in) << p.rshift | gb<3 * K + 1>(in) << p.gshift | gb<3 * K + 2>(in) << p.bshift;
                        px<K + 1>(in, out, p, amask);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
                px<0>(in, out, p, amask);
        }
};

/// 32-bit pixel -> RGB with source shifts RS/GS/BS:
///   vc_copylineRGBAtoRGB (pixfmt_conv.c:866-900, shifts 0/8/16) and vc_copylineABGRtoRGB (:809-843, 24/16/8) in the SSSE3 build that is the
///   contract: QUIRK reproduced for bit-exactness - the scalar tail loop (:889-895, :834-839) never advances `src`, so every pixel from the end
///   of the pshufb loop (x <= dst_len - 24) on repeats the first tail pixel.  p.aux = first tail pixel.
///   vc_copylineBGRAtoRGB (:845-860, 16/8/0) goes through the plain C loop vc_copylineRGBAtoRGBwithShift (:769-801): no quirk.
template <int RS, int GS, int BS, bool QUIRK>
struct conv_x32_rgb {
        static constexpr int IN = 64, OUT = 48;
        static __host__ int out_len(int dst_len) { return dst_len < 3 ? 0 : dst_len / 3 * 3; }
        static __host__ int aux(int dst_len) { return !QUIRK ? 0x7fffffff : dst_len >= 24 ? ((dst_len - 24) / 12 + 1) * 4 : 0; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &rc)
        {
                uint32_t tail = 0;
                if (QUIRK && (rc.cx + 1) * 16 > p.aux) {  // this chunk reaches into the tail
                        const long a = rc.row_abs + 4L * p.aux;
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                                if (a + k < rc.src_total) {
                                        tail |= (uint32_t) rc.src[a + k] << (8 * k);
                                }
                        }
                }
                uint32_t o[48];
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                        const uint32_t w = QUIRK && rc.cx * 16 + i >= p.aux ? tail : in[i];
                        o[3 * i] = (w >> RS) & 0xff;
                        o[3 * i + 1] = (w >> GS) & 0xff;
                        o[3 * i + 2] = (w >> BS) & 0xff;
                }
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        out[i] = pack4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
                }
        }
};
using conv_rgba_rgb = conv_x32_rgb<0, 8, 16, true>;
using conv_abgr_rgb = conv_x32_rgb<24, 16, 8, true>;
using conv_bgra_rgb = conv_x32_rgb<16, 8, 0, false>;

// ---- pure byte-permutation converters: out byte j = in byte M::src(j), or 0x00 (-1) / 0xFF (-2) ---------------------------
template <class M>
struct conv_bytemap {
        static constexpr int IN = M::IN, OUT = M::OUT;
        static __host__ int out_len(int dst_len) { return M::out_len(dst_len); }
        template <int J>
        static __device__ __forceinline__ uint32_t byte(const uint32_t *in)
        {
                constexpr int sidx = M::src(J);
                if constexpr (sidx == -1) {
                        return 0u;
                } else if constexpr (sidx == -2) {
                        return 0xffu;
                } else {
                        return gb<sidx>(in);
                }
        }
        template <int W>
        static __device__ __forceinline__ void word(const uint32_t *in, uint32_t *out)
        {
                if constexpr (W < OUT / 4) {
                        out[W] = byte<4 * W>(in) | byte<4 * W + 1>(in) << 8 | byte<4 * W + 2>(in) << 16 | byte<4 * W + 3>(in) << 24;
                        word<W + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { word<0>(in, out); }
};
struct map_rg48_rgb {  // vc_copylineRG48toRGB, pixfmt_conv.c:2030-2042: the high byte of each 16-bit sample
        static constexpr int IN = 96, OUT = 48;
        static __host__ int out_len(int n) { return n < 3 ? 0 : n / 3 * 3; }
        static constexpr int src(int j) { return 6 * (j / 3) + 2 * (j % 3) + 1; }
};
struct map_rgb_rg48 {  // vc_copylineRGBtoRG48, :1353-1363
        static constexpr int IN = 16, OUT = 32;
        static __host__ int out_len(int n) { return n < 2 ? 0 : n / 2 * 2; }
        static constexpr int src(int j) { return (j % 2) ? j / 2 : -1; }
};

// ---- R12L: 8 pixels x 3 components x 12 bits = 36 bytes, component k of a group at bit 12k (little endian) --------------------
__device__ __forceinline__ uint32_t r12_get(const uint32_t *w, int k)  // k folds to a constant once the loops are unrolled
{
        const int off = 12 * k, wi = off >> 5, sh = off & 31;
        return sh <= 20 ? (w[wi] >> sh) & 0xfffu : ((w[wi] >> sh) | (w[wi + 1] << (32 - sh))) & 0xfffu;
}
__device__ __forceinline__ void r12_put(uint32_t *w, int k, uint32_t v)
{
        const int off = 12 * k, wi = off >> 5, sh = off & 31;
        w[wi] |= v << sh;
        if (sh > 20) {
                w[wi + 1] |= v >> (32 - sh);
        }
}

/// R12L -> 8/10/16-bit RGB layouts.  MODE 0: RGB (vc_copylineR12LtoRGB, pixfmt_conv.c:353-430), 1: RGBA (vc_copylineR12L, :438-523),
/// 2: RG48 (:1371-1476), 3: R10k (:1640-1699)
template <int MODE>
struct conv_r12l_rgbx {
        static constexpr int IN = 144, OUT = MODE == 0 ? 96 : MODE == 2 ? 192 : 128;
        static __host__ int out_len(int n) { return MODE == 0 ? n / 24 * 24 : MODE == 3 ? n / 32 * 32 : n; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &p, const row_ctx &)
        {
                const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
                uint32_t o8[MODE == 0 ? 96 : 1];
                uint32_t o16[MODE == 2 ? 96 : 1];
#pragma unroll
                for (int g = 0; g < 4; ++g) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                const uint32_t r = r12_get(in + 9 * g, 3 * i), gg = r12_get(in + 9 * g, 3 * i + 1), b = r12_get(in + 9 * g, 3 * i + 2);
                                const int px = 8 * g + i;
                                if (MODE == 0) {
                                        o8[3 * px] = r >> 4, o8[3 * px + 1] = gg >> 4, o8[3 * px + 2] = b >> 4;
                                } else if (MODE == 1) {
                                        out[px] = amask | (r >> 4) << p.rshift | (gg >> 4) << p.gshift | (b >> 4) << p.bshift;
                                } else if (MODE == 2) {
                                        o16[3 * px] = r << 4, o16[3 * px + 1] = gg << 4, o16[3 * px + 2] = b << 4;
                                } else {  // not a clean R10k: byte 3 keeps B[7:0]; pixel 1 of a group gets R[3:0] in its low nibble (pixfmt_conv.c:1661)
                                        out[px] = (r >> 4) | ((r & 0xC) << 4 | gg >> 6) << 8 | (((gg >> 2) & 0xF) << 4 | b >> 8) << 16 |
                                                  (i == 1 ? (b & 0xF0) | (r & 0xF) : b & 0xFF) << 24;
                                }
                        }
                }
                if (MODE == 0) {
#pragma unroll
                        for (int i = 0; i < 24; ++i) {
                                out[i] = pack4(o8[4 * i], o8[4 * i + 1], o8[4 * i + 2], o8[4 * i + 3]);
                        }
                }
                if (MODE == 2) {
#pragma unroll
                        for (int i = 0; i < 48; ++i) {
                                out[i] = o16[2 * i] | o16[2 * i + 1] << 16;
                        }
                }
        }
};

/// X -> R12L.  SRC 0: RGB, 1: RGBA (vc_copylineRGB_AtoR12L, :1258-1334: 8-bit << 4), 2: RG48 (vc_copylineRG48toR12L, :1701-1826: 16-bit >> 4),
/// 3: Y416 (vc_copylineY416toR12L, :1828-1915: depth-16 coefficients of CS, >> COMP_BASE + 4, CLAMP_FULL 12 bit)
template <int SRC, class CS = bt709>
struct conv_x_r12l {
        static constexpr int IN = SRC == 0 ? 96 : SRC == 1 ? 128 : SRC == 2 ? 192 : 256, OUT = 144;
        static __host__ int out_len(int n) { return SRC == 3 ? (n + 35) / 36 * 36 : n / 36 * 36; }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 36; ++i) {
                        out[i] = 0;
                }
#pragma unroll
                for (int px = 0; px < 32; ++px) {
                        uint32_t r, g, b;
                        if (SRC == 0 || SRC == 1) {
                                const int o = px * (SRC == 0 ? 3 : 4);
                                r = ((in[o >> 2] >> (8 * (o & 3))) & 0xff) << 4, g = ((in[(o + 1) >> 2] >> (8 * ((o + 1) & 3))) & 0xff) << 4,
                                b = ((in[(o + 2) >> 2] >> (8 * ((o + 2) & 3))) & 0xff) << 4;
                        } else if (SRC == 2) {
                                const int o = 3 * px;
                                r = ((in[o >> 1] >> (16 * (o & 1))) & 0xffff) >> 4, g = ((in[(o + 1) >> 1] >> (16 * ((o + 1) & 1))) & 0xffff) >> 4,
                                b = ((in[(o + 2) >> 1] >> (16 * ((o + 2) & 1))) & 0xffff) >> 4;
                        } else {
                                constexpr color_coeffs c = CS::at(16);
                                const int u = (int) (in[2 * px] & 0xffff) - 32768, y = c.y_scale * ((int) (in[2 * px] >> 16) - 4096), v = (int) (in[2 * px + 1] & 0xffff) - 32768;
                                r = clampr((y + v * c.r_cr) >> (COMP_BASE + 4), 16, 4079), g = clampr((y + u * c.g_cb + v * c.g_cr) >> (COMP_BASE + 4), 16, 4079),
                                b = clampr((y + u * c.b_cb) >> (COMP_BASE + 4), 16, 4079);
                        }
                        uint32_t *w = out + 9 * (px >> 3);
                        r12_put(w, 3 * (px & 7), r), r12_put(w, 3 * (px & 7) + 1, g), r12_put(w, 3 * (px & 7) + 2, b);
                }
        }
};

}  // namespace ugb
