// The RGB-like -> UYVY line converter of pixfmt_kernels.cu as a device functor, shared with the border postprocessor
// (geometry_kernels.cu), whose UYVY fill is this converter's output for two pixels of the border colour.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "color_space.h"
#include "yuv_rgb_conv.cuh"

namespace ugb {

// byte k (compile-time) of a packed word array
template <int K>
__device__ __forceinline__ uint32_t gb(const uint32_t *a)
{
        return (a[K >> 2] >> (8 * (K & 3))) & 0xffu;
}
__device__ __forceinline__ uint32_t pack4(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3)
{
        return b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
}

/// vc_copylineToUYVY, pixfmt_conv.c:1008-1053: RGB-like (ROFF/GOFF/BOFF within PIX bytes) -> UYVY.
/// y = (RGB_TO_Y >> 14) + 16 unclamped; chroma = ((cb0 + cb1) / 2 >> 14) + 128 with C '/' truncation;
/// bytes stored & 0xFF.  Used by RGB (:2061), BGR (:2271), RGBA (:2316), RG48 (:2343, high bytes).  CS: coefficient set (color_space.h).
template <int ROFF, int GOFF, int BOFF, int PIX, class CS = bt709>
struct conv_to_uyvy {
        static constexpr int NPX = 16 / (PIX == 3 ? 1 : PIX == 4 ? 2 : 2);  // 16, 8 (RGBA), 8 (RG48)
        static constexpr int IN = NPX * PIX, OUT = NPX * 2;
        static __host__ int out_len(int dst_len) { return (dst_len + 3) / 4 * 4; }  // count = (dst_len+3)/4 words, :1045
        template <int K>
        static __device__ __forceinline__ void pair(const uint32_t *in, uint32_t *out)
        {
                constexpr color_coeffs c = CS::at(8);
                constexpr int P0 = 2 * K * PIX, P1 = P0 + PIX;
                const int r0 = gb<P0 + ROFF>(in), g0 = gb<P0 + GOFF>(in), b0 = gb<P0 + BOFF>(in);
                const int r1 = gb<P1 + ROFF>(in), g1 = gb<P1 + GOFF>(in), b1 = gb<P1 + BOFF>(in);
                const int y1 = ((r0 * c.y_r + g0 * c.y_g + b0 * c.y_b) >> COMP_BASE) + 16;
                const int y2 = ((r1 * c.y_r + g1 * c.y_g + b1 * c.y_b) >> COMP_BASE) + 16;
                int u = (r0 * c.cb_r + g0 * c.cb_g + b0 * c.cb_b) + (r1 * c.cb_r + g1 * c.cb_g + b1 * c.cb_b);
                int v = (r0 * c.cr_r + g0 * c.cr_g + b0 * c.cr_b) + (r1 * c.cr_r + g1 * c.cr_g + b1 * c.cr_b);
                u = ((u / 2) >> COMP_BASE) + 128;
                v = ((v / 2) >> COMP_BASE) + 128;
                out[K] = pack4(u & 0xff, y1 & 0xff, v & 0xff, y2 & 0xff);
        }
        template <int K>
        static __device__ __forceinline__ void pairs(const uint32_t *in, uint32_t *out)
        {
                if constexpr (K < NPX / 2) {
                        pair<K>(in, out);
                        pairs<K + 1>(in, out);
                }
        }
        static __device__ __forceinline__ void run(const uint32_t *in, uint32_t *out, const conv_params &, const row_ctx &) { pairs<0>(in, out); }
};

}  // namespace ugb
