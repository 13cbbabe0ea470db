// DXT1 / DXT5-YCoCg 4x4 block encoders — device side.
//
// Arithmetic contract: bit-exact with UltraGrid's cuda_dxt/cuda_dxt.cu *as built by nvcc 12.9 for
// sm_90a with default flags (--fmad=true)*.  ptxas contracts the reference's float expressions into
// a specific FMA tree; that tree was read out of the reference cubin's SASS and is restated here with
// explicit-rounding intrinsics (__fmaf_rn/__fmul_rn/__fadd_rn never re-contract), so the result does
// not depend on what the optimiser does with *this* file.  Reference source lines are cited per step.
//
// What is new here (not in the reference): byte->float through a 2^23 "magic" word folded into the
// first FMA (no I2F), float->int through magic adds (no F2I/FRND on the slow conversion pipe), a
// fused UYVY loader (no 4:4:4 intermediate), 128-bit loads/stores, right-sized grids.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "f32x2.cuh"

namespace ugb {

// ---- constants -------------------------------------------------------------------------------
// 0.00392156862745f == 0x3B808081 == 8421505 * 2^-31          (cuda_dxt.cu:666-683)
__device__ constexpr float kInv255 = 0.00392156862745f;
// 2^23 + b  (b < 256) is exactly representable; fma(2^23 + b, kInv255, -(2^23*kInv255) - k) is
// the single-rounded value of b*kInv255 - k, i.e. identical to fma(float(b), kInv255, -k).
// 2^23*kInv255 = 8421505/256 exactly; the three biases below are all exactly representable.
__device__ constexpr float kBiasRGB = -32896.50390625f;  // k = 0       -> fl(b * kInv255)
__device__ constexpr float kBiasY   = -32896.56640625f;  // k = 0.0625  -> fma(b, kInv255, -0.0625)
__device__ constexpr float kBiasC   = -32897.00390625f;  // k = 0.5     -> fma(b, kInv255, -0.5)

__device__ constexpr float kRoundMagic = 12582912.0f;    // 1.5 * 2^23: x + M rounds x to nearest-even int
__device__ constexpr float kFloorMagic = 8388608.0f;     // 2^23: (x + M) toward -inf == floor(x), x >= 0

__device__ constexpr float kInv31 = 0.0322580645161f;    // cuda_dxt.cu:434
__device__ constexpr float kInv63 = 0.015873015873f;     // cuda_dxt.cu:435

/// 0x4B0000bb where bb is byte @p sel of @p w, i.e. the float 2^23 + bb.
__device__ __forceinline__ float magic_byte(uint32_t w, unsigned sel)
{
        return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540u | sel));
}

/// saturate(a + b) in one instruction, never contracted with neighbours
__device__ __forceinline__ float add_sat_rn(float a, float b)
{
        float d;
        asm("add.rn.sat.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
        return d;
}

// ---- pixel loaders ---------------------------------------------------------------------------

/// byte (already as 2^23+b magic float) -> unit-range sample, cuda_dxt.cu:666-683
__device__ __forceinline__ float unit_from_magic(float m)
{
        return __fmaf_rn(m, kInv255, kBiasRGB);
}

/// YCbCr -> RGB of cuda_dxt.cu:444-451 as contracted by ptxas:
///   Yf = fma(Y, 1/255, -0.0625); y = Yf * 1.1643
///   u  = fma(U, 1/255, -0.5);    v = fma(V, 1/255, -0.5)
///   R  = fma(v, 1.7926, y);  G = fma(v, -0.5328, fma(u, -0.2132, y));  B = fma(u, 2.1124, y)
struct chroma_t {
        float u, v;
};
__device__ __forceinline__ chroma_t chroma_from_magic(float mu, float mv)
{
        chroma_t c;
        c.u = __fmaf_rn(mu, kInv255, kBiasC);
        c.v = __fmaf_rn(mv, kInv255, kBiasC);
        return c;
}
__device__ __forceinline__ void yuv_px_to_rgb(float my, chroma_t c, float &r, float &g, float &b)
{
        const float y = __fmul_rn(__fmaf_rn(my, kInv255, kBiasY), 1.1643f);
        r = __fmaf_rn(c.v, 1.7926f, y);
        g = __fmaf_rn(c.v, -0.5328f, __fmaf_rn(c.u, -0.2132f, y));
        b = __fmaf_rn(c.u, 2.1124f, y);
}

/// One row (4 px) of a block from packed 3-byte pixels: three 32-bit words p0,p1,p2 (cuda_dxt.cu:661-683).
template <bool YUV>
__device__ __forceinline__ void load_row_packed3(uint32_t p0, uint32_t p1, uint32_t p2, float *r, float *g,
                                                 float *b)
{
        const float m[12] = { magic_byte(p0, 0), magic_byte(p0, 1), magic_byte(p0, 2), magic_byte(p0, 3),
                              magic_byte(p1, 0), magic_byte(p1, 1), magic_byte(p1, 2), magic_byte(p1, 3),
                              magic_byte(p2, 0), magic_byte(p2, 1), magic_byte(p2, 2), magic_byte(p2, 3) };
#pragma unroll
        for (int i = 0; i < 4; ++i) {
                if (YUV) {
                        yuv_px_to_rgb(m[3 * i], chroma_from_magic(m[3 * i + 1], m[3 * i + 2]), r[i], g[i], b[i]);
                } else {
                        r[i] = unit_from_magic(m[3 * i]);
                        g[i] = unit_from_magic(m[3 * i + 1]);
                        b[i] = unit_from_magic(m[3 * i + 2]);
                }
        }
}

/// One row (4 px) of a block straight from UYVY: w0 = U0 Y0 V0 Y1, w1 = U1 Y2 V1 Y3.  Equals
/// cuda_yuv422_to_yuv444 (chroma replication, cuda_dxt.cu:709-727) followed by the YUV loader above.
__device__ __forceinline__ void load_row_uyvy(uint32_t w0, uint32_t w1, float *r, float *g, float *b)
{
        const chroma_t c0 = chroma_from_magic(magic_byte(w0, 0), magic_byte(w0, 2));
        const chroma_t c1 = chroma_from_magic(magic_byte(w1, 0), magic_byte(w1, 2));
        yuv_px_to_rgb(magic_byte(w0, 1), c0, r[0], g[0], b[0]);
        yuv_px_to_rgb(magic_byte(w0, 3), c0, r[1], g[1], b[1]);
        yuv_px_to_rgb(magic_byte(w1, 1), c1, r[2], g[2], b[2]);
        yuv_px_to_rgb(magic_byte(w1, 3), c1, r[3], g[3], b[3]);
}

// ---- DXT1 --------------------------------------------------------------------------------------

/// 5:6:5 endpoint quantiser of cuda_dxt.cu:424-440.  @returns the magic-biased integer
/// (float bits 0x4B400000 + q) so that both the integer code and float(q) come out of full-rate adds.
__device__ __forceinline__ float quant_magic(float v, float levels)
{
        return __fadd_rn(__fmul_rn(__saturatef(v), levels), kRoundMagic);
}

/// dxt_encode<1>, cuda_dxt.cu:512-617.
__device__ __forceinline__ uint2 dxt1_encode(const float (&r)[16], const float (&g)[16], const float (&b)[16])
{
        // bounding box (:516-529) — min/max are order-independent
        float mnr = r[0], mng = g[0], mnb = b[0], mxr = r[0], mxg = g[0], mxb = b[0];
#pragma unroll
        for (int i = 1; i < 16; ++i) {
                mnr = fminf(mnr, r[i]);
                mng = fminf(mng, g[i]);
                mnb = fminf(mnb, b[i]);
                mxr = fmaxf(mxr, r[i]);
                mxg = fmaxf(mxg, g[i]);
                mxb = fmaxf(mxb, b[i]);
        }
        // inset (:532-540): d = max - min; min' = fma(d, 1/16, min); max' = fma(d, -1/16, max)
        const float dr = __fadd_rn(mxr, -mnr), dg = __fadd_rn(mxg, -mng), db = __fadd_rn(mxb, -mnb);
        const float lor = __fmaf_rn(dr, 0.0625f, mnr), hir = __fmaf_rn(dr, -0.0625f, mxr);
        const float log_ = __fmaf_rn(dg, 0.0625f, mng), hig = __fmaf_rn(dg, -0.0625f, mxg);
        const float lob = __fmaf_rn(db, 0.0625f, mnb), hib = __fmaf_rn(db, -0.0625f, mxb);

        // diagonal select (:543-560): (x - (lo+hi)*0.5) is fma(lo+hi, -0.5, x); cov accumulates
        // sequentially i = 0..15 from +0 through FMAs
        const float sr = __fadd_rn(lor, hir), sg = __fadd_rn(log_, hig), sb = __fadd_rn(lob, hib);
        float covx = 0.0f, covy = 0.0f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
                const float er = __fmaf_rn(sr, -0.5f, r[i]);
                const float eg = __fmaf_rn(sg, -0.5f, g[i]);
                const float eb = __fmaf_rn(sb, -0.5f, b[i]);
                covx = __fmaf_rn(er, eb, covx);
                covy = __fmaf_rn(eg, eb, covy);
        }
        const bool swr = covx < 0.0f, swg = covy < 0.0f;
        const float maxr = swr ? lor : hir, minr = swr ? hir : lor;
        const float maxg = swg ? log_ : hig, ming = swg ? hig : log_;

        // endpoints (:563-572, :424-431)
        const float qxr = quant_magic(maxr, 31.0f), qxg = quant_magic(maxg, 63.0f), qxb = quant_magic(hib, 31.0f);
        const float qnr = quant_magic(minr, 31.0f), qng = quant_magic(ming, 63.0f), qnb = quant_magic(lob, 31.0f);
        constexpr uint32_t kCodeBias = 0x4B400000u * 2081u;  // (1<<11) + (1<<5) + 1, mod 2^32
        const uint32_t max_code = (__float_as_uint(qxr) << 11) + (__float_as_uint(qxg) << 5) + __float_as_uint(qxb) - kCodeBias;
        const uint32_t min_code = (__float_as_uint(qnr) << 11) + (__float_as_uint(qng) << 5) + __float_as_uint(qnb) - kCodeBias;

        uint32_t indices = 0;
        if (max_code != min_code) {  // :576-602
                // quantised endpoints back in unit range (:434-436); dir = min - max is contracted into
                // fma(q_min, 1/31, -(q_max * 1/31))
                const float ex_r = __fmul_rn(__fadd_rn(qxr, -kRoundMagic), kInv31);
                const float ex_g = __fmul_rn(__fadd_rn(qxg, -kRoundMagic), kInv63);
                const float ex_b = __fmul_rn(__fadd_rn(qxb, -kRoundMagic), kInv31);
                const float dir_r = __fmaf_rn(__fadd_rn(qnr, -kRoundMagic), kInv31, -ex_r);
                const float dir_g = __fmaf_rn(__fadd_rn(qng, -kRoundMagic), kInv63, -ex_g);
                const float dir_b = __fmaf_rn(__fadd_rn(qnb, -kRoundMagic), kInv31, -ex_b);
                const float len2 = __fmaf_rn(dir_b, dir_b, __fmaf_rn(dir_r, dir_r, __fmul_rn(dir_g, dir_g)));
                const float inv = __fdividef(1.0f, len2);  // :584 — MUFU.RCP
                const float tr = __fmul_rn(dir_r, inv), tg = __fmul_rn(dir_g, inv), tb = __fmul_rn(dir_b, inv);
                const float nbias = -__fmaf_rn(ex_b, tb, __fmaf_rn(ex_r, tr, __fmul_rn(ex_g, tg)));
                uint32_t acc = 0;
#pragma unroll
                for (int i = 0; i < 16; ++i) {  // :591-601
                        const float t = __fmaf_rn(b[i], tb, __fmaf_rn(r[i], tr, __fmul_rn(g[i], tg)));
                        const float x = __fmaf_rn(add_sat_rn(t, nbias), 3.0f, 0.5f);
                        // (u32)x truncates; x is in [0.5, 3.5] so floor == trunc
                        acc += __float_as_uint(__fadd_rd(x, kFloorMagic)) << (2 * i);
                }
                constexpr uint32_t kIdxBias = 0x4B000000u * 0x55555555u;  // sum of (bias << 2i), mod 2^32
                indices = acc - kIdxBias;
        }
        const bool swap_end = max_code < min_code;  // :568-572
        if (swap_end) {
                indices = ~indices;  // :605-607
        }
        const uint32_t lsbs = indices & 0x55555555u, msbs = indices & 0xaaaaaaaau;  // :611-613
        indices = msbs ^ (2 * lsbs + (msbs >> 1));
        const uint32_t palette = swap_end ? min_code + (max_code << 16) : max_code + (min_code << 16);
        return make_uint2(palette, indices);
}

}  // namespace ugb

// ================================================================================================
// Paired (float2) formulation of the fused UYVY -> DXT1 block encode.
//
// Same operation tree, hence the same bits, as load_row_uyvy() + dxt1_encode(); the work is written two pixels at a time
// (f32x2.cuh: two scalar instructions per pair on sm_90).
// Pairing: pixels x and x+2 of a row share an instruction, because their chroma (U0,U1)/(V0,V1) is itself a natural
// pair; element [2y + (x&1)].{x,y}[x>>1] of an array holds pixel (x, y).
// ================================================================================================
namespace ugb {

__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 dup(float a) { return make_float2(a, a); }
/// load_row_uyvy() with the operations of pixels x and x + 2 paired (same operation tree)
__device__ __forceinline__ void load_row_uyvy_packed(uint32_t w0, uint32_t w1, float *r, float *g, float *b)
{
        const float2 c2 = dup(kInv255);
        const float2 u = __ffma2_rn(f2(magic_byte(w0, 0), magic_byte(w1, 0)), c2, dup(kBiasC));
        const float2 v = __ffma2_rn(f2(magic_byte(w0, 2), magic_byte(w1, 2)), c2, dup(kBiasC));
#pragma unroll
        for (int k = 0; k < 2; ++k) {  // k = 0: pixels 0, 2;  k = 1: pixels 1, 3
                const float2 yy = __fmul2_rn(__ffma2_rn(f2(magic_byte(w0, 1 + 2 * k), magic_byte(w1, 1 + 2 * k)), c2, dup(kBiasY)), dup(1.1643f));
                const float2 R = __ffma2_rn(v, dup(1.7926f), yy);
                const float2 G = __ffma2_rn(v, dup(-0.5328f), __ffma2_rn(u, dup(-0.2132f), yy));
                const float2 B = __ffma2_rn(u, dup(2.1124f), yy);
                r[k] = R.x, r[k + 2] = R.y, g[k] = G.x, g[k + 2] = G.y, b[k] = B.x, b[k + 2] = B.y;
        }
}

__device__ __forceinline__ float px(const float2 (&v)[8], int i) { return ((i & 3) >> 1) ? v[2 * (i >> 2) + (i & 1)].y : v[2 * (i >> 2) + (i & 1)].x; }

/// BRANCH = false computes the indices of a flat block (max_code == min_code) too and discards them: straight-line code, so that
/// the scheduler may interleave the two blocks of a thread.  Colour values come packed: element [2y + (x&1)].{x,y}[x>>1] = pixel (x, y).
template <bool BRANCH = true>
__device__ __forceinline__ uint2 dxt1_encode_packed_core(const float2 (&R)[8], const float2 (&G)[8], const float2 (&B)[8])
{
        // bounding box, seeded with the first pixel pair (15 FMNMX per chain)
        float mnr = fminf(R[0].x, R[0].y), mxr = fmaxf(R[0].x, R[0].y);
        float mng = fminf(G[0].x, G[0].y), mxg = fmaxf(G[0].x, G[0].y);
        float mnb = fminf(B[0].x, B[0].y), mxb = fmaxf(B[0].x, B[0].y);
#pragma unroll
        for (int j = 1; j < 8; ++j) {
                mnr = fminf(mnr, fminf(R[j].x, R[j].y)), mxr = fmaxf(mxr, fmaxf(R[j].x, R[j].y));
                mng = fminf(mng, fminf(G[j].x, G[j].y)), mxg = fmaxf(mxg, fmaxf(G[j].x, G[j].y));
                mnb = fminf(mnb, fminf(B[j].x, B[j].y)), mxb = fmaxf(mxb, fmaxf(B[j].x, B[j].y));
        }
        const float dr = __fadd_rn(mxr, -mnr), dg = __fadd_rn(mxg, -mng), db = __fadd_rn(mxb, -mnb);
        const float lor = __fmaf_rn(dr, 0.0625f, mnr), hir = __fmaf_rn(dr, -0.0625f, mxr);
        const float log_ = __fmaf_rn(dg, 0.0625f, mng), hig = __fmaf_rn(dg, -0.0625f, mxg);
        const float lob = __fmaf_rn(db, 0.0625f, mnb), hib = __fmaf_rn(db, -0.0625f, mxb);
        // deviations from the box centre, packed; covariance chains stay scalar and sequential (i = 0..15)
        const float2 sr2 = dup(__fadd_rn(lor, hir)), sg2 = dup(__fadd_rn(log_, hig)), sb2 = dup(__fadd_rn(lob, hib)), mh = dup(-0.5f);
        float2 ER[8], EG[8], EB[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
                ER[j] = __ffma2_rn(sr2, mh, R[j]);
                EG[j] = __ffma2_rn(sg2, mh, G[j]);
                EB[j] = __ffma2_rn(sb2, mh, B[j]);
        }
        float covx = 0.0f, covy = 0.0f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
                covx = __fmaf_rn(px(ER, i), px(EB, i), covx);
                covy = __fmaf_rn(px(EG, i), px(EB, i), covy);
        }
        const bool swr = covx < 0.0f, swg = covy < 0.0f;
        const float maxr = swr ? lor : hir, minr = swr ? hir : lor;
        const float maxg = swg ? log_ : hig, ming = swg ? hig : log_;
        const float qxr = quant_magic(maxr, 31.0f), qxg = quant_magic(maxg, 63.0f), qxb = quant_magic(hib, 31.0f);
        const float qnr = quant_magic(minr, 31.0f), qng = quant_magic(ming, 63.0f), qnb = quant_magic(lob, 31.0f);
        constexpr uint32_t kCodeBias = 0x4B400000u * 2081u;
        const uint32_t max_code = (__float_as_uint(qxr) << 11) + (__float_as_uint(qxg) << 5) + __float_as_uint(qxb) - kCodeBias;
        const uint32_t min_code = (__float_as_uint(qnr) << 11) + (__float_as_uint(qng) << 5) + __float_as_uint(qnb) - kCodeBias;

        uint32_t indices = 0;
        if (!BRANCH || max_code != min_code) {
                const float ex_r = __fmul_rn(__fadd_rn(qxr, -kRoundMagic), kInv31);
                const float ex_g = __fmul_rn(__fadd_rn(qxg, -kRoundMagic), kInv63);
                const float ex_b = __fmul_rn(__fadd_rn(qxb, -kRoundMagic), kInv31);
                const float dir_r = __fmaf_rn(__fadd_rn(qnr, -kRoundMagic), kInv31, -ex_r);
                const float dir_g = __fmaf_rn(__fadd_rn(qng, -kRoundMagic), kInv63, -ex_g);
                const float dir_b = __fmaf_rn(__fadd_rn(qnb, -kRoundMagic), kInv31, -ex_b);
                const float len2 = __fmaf_rn(dir_b, dir_b, __fmaf_rn(dir_r, dir_r, __fmul_rn(dir_g, dir_g)));
                const float inv = __fdividef(1.0f, len2);
                const float tr = __fmul_rn(dir_r, inv), tg = __fmul_rn(dir_g, inv), tb = __fmul_rn(dir_b, inv);
                const float nbias = -__fmaf_rn(ex_b, tb, __fmaf_rn(ex_r, tr, __fmul_rn(ex_g, tg)));
                const float2 tr2 = dup(tr), tg2 = dup(tg), tb2 = dup(tb);
                uint32_t acc0 = 0, acc1 = 0;  // two independent chains; integer adds are associative, the bits are the same
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                        const float2 t = __ffma2_rn(B[j], tb2, __ffma2_rn(R[j], tr2, __fmul2_rn(G[j], tg2)));
                        const float2 x = __ffma2_rn(f2(add_sat_rn(t.x, nbias), add_sat_rn(t.y, nbias)), dup(3.0f), dup(0.5f));
                        const float2 m = __fadd2_rd(x, dup(kFloorMagic));
                        const int i0 = 4 * (j >> 1) + (j & 1);  // pixel of .x; .y is pixel i0 + 2
                        acc0 += __float_as_uint(m.x) << (2 * i0);
                        acc1 += __float_as_uint(m.y) << (2 * (i0 + 2));
                }
                constexpr uint32_t kIdxBias = 0x4B000000u * 0x55555555u;
                indices = acc0 + acc1 - kIdxBias;
                if (!BRANCH) {
                        indices = max_code != min_code ? indices : 0u;
                }
        }
        const bool swap_end = max_code < min_code;
        if (swap_end) {
                indices = ~indices;
        }
        const uint32_t lsbs = indices & 0x55555555u, msbs = indices & 0xaaaaaaaau;
        indices = msbs ^ (2 * lsbs + (msbs >> 1));
        const uint32_t palette = swap_end ? min_code + (max_code << 16) : max_code + (min_code << 16);
        return make_uint2(palette, indices);
}

/// fused UYVY loader (chroma shared by a pixel pair) + the packed core
template <bool BRANCH = true>
__device__ __forceinline__ uint2 dxt1_encode_uyvy_packed(const uint32_t (&w)[4][2])
{
        float2 R[8], G[8], B[8];
        const float2 c2 = dup(kInv255), ky2 = dup(kBiasY), kc2 = dup(kBiasC);
#pragma unroll
        for (int y = 0; y < 4; ++y) {
                const uint32_t w0 = w[y][0], w1 = w[y][1];
                const float2 u = __ffma2_rn(f2(magic_byte(w0, 0), magic_byte(w1, 0)), c2, kc2);
                const float2 v = __ffma2_rn(f2(magic_byte(w0, 2), magic_byte(w1, 2)), c2, kc2);
#pragma unroll
                for (int k = 0; k < 2; ++k) {  // k = 0: pixels x = 0, 2;  k = 1: pixels x = 1, 3
                        const float2 yy = __fmul2_rn(__ffma2_rn(f2(magic_byte(w0, 1 + 2 * k), magic_byte(w1, 1 + 2 * k)), c2, ky2), dup(1.1643f));
                        R[2 * y + k] = __ffma2_rn(v, dup(1.7926f), yy);
                        G[2 * y + k] = __ffma2_rn(v, dup(-0.5328f), __ffma2_rn(u, dup(-0.2132f), yy));
                        B[2 * y + k] = __ffma2_rn(u, dup(2.1124f), yy);
                }
        }
        return dxt1_encode_packed_core<BRANCH>(R, G, B);
}

/// packed 3-byte source (cuda_rgb_to_dxt1 / cuda_yuv_to_dxt1, cuda_dxt.cu:661-683 + :444-451): w[y] = the three words (4 pixels) of row y.  Same
/// per-sample operations as load_row_packed3(), pixels x and x + 2 paired.
template <bool YUV>
__device__ __forceinline__ uint2 dxt1_encode_packed3(const uint32_t (&w)[4][3])
{
        float2 R[8], G[8], B[8];
        const float2 c2 = dup(kInv255);
#pragma unroll
        for (int y = 0; y < 4; ++y) {
                const uint32_t p0 = w[y][0], p1 = w[y][1], p2 = w[y][2];
                // pixel 0 = p0.b0 p0.b1 p0.b2, pixel 1 = p0.b3 p1.b0 p1.b1, pixel 2 = p1.b2 p1.b3 p2.b0, pixel 3 = p2.b1 p2.b2 p2.b3
                const float2 a0 = f2(magic_byte(p0, 0), magic_byte(p1, 2)), a1 = f2(magic_byte(p0, 1), magic_byte(p1, 3)), a2 = f2(magic_byte(p0, 2), magic_byte(p2, 0));
                const float2 b0 = f2(magic_byte(p0, 3), magic_byte(p2, 1)), b1 = f2(magic_byte(p1, 0), magic_byte(p2, 2)), b2 = f2(magic_byte(p1, 1), magic_byte(p2, 3));
                if (YUV) {
#pragma unroll
                        for (int k = 0; k < 2; ++k) {
                                const float2 my = k ? b0 : a0, mu = k ? b1 : a1, mv = k ? b2 : a2;
                                const float2 yy = __fmul2_rn(__ffma2_rn(my, c2, dup(kBiasY)), dup(1.1643f));
                                const float2 u = __ffma2_rn(mu, c2, dup(kBiasC)), v = __ffma2_rn(mv, c2, dup(kBiasC));
                                R[2 * y + k] = __ffma2_rn(v, dup(1.7926f), yy);
                                G[2 * y + k] = __ffma2_rn(v, dup(-0.5328f), __ffma2_rn(u, dup(-0.2132f), yy));
                                B[2 * y + k] = __ffma2_rn(u, dup(2.1124f), yy);
                        }
                } else {
                        R[2 * y] = __ffma2_rn(a0, c2, dup(kBiasRGB)), G[2 * y] = __ffma2_rn(a1, c2, dup(kBiasRGB)), B[2 * y] = __ffma2_rn(a2, c2, dup(kBiasRGB));
                        R[2 * y + 1] = __ffma2_rn(b0, c2, dup(kBiasRGB)), G[2 * y + 1] = __ffma2_rn(b1, c2, dup(kBiasRGB)), B[2 * y + 1] = __ffma2_rn(b2, c2, dup(kBiasRGB));
                }
        }
        return dxt1_encode_packed_core<true>(R, G, B);
}

}  // namespace ugb

// ================================================================================================
// Two blocks per thread, phases SKEWED by hand (round 2).
//
// The encode of one block alternates long FMA-pipe-only stretches (deviations + covariance chains, index projection) with ALU-pipe-only
// stretches (bounding box, index packing): a warp inside a one-pipe stretch cannot use the other pipe, and the SM only keeps both busy
// when other warps happen to be in the complementary stretch.  Here the two blocks of a thread are one phase apart, statement by statement:
//     A: unpack+RGB | bbox        | dev + cov   | endpoints + indices | pack
//     B:            | unpack+RGB  | bbox        | dev + cov           | endpoints + indices | pack
// so that the ALU-only bounding box of one block sits between the FMA-only instructions of the other.  Same operation tree per block as
// dxt1_encode_uyvy_packed(), hence the same bits.
// ================================================================================================
namespace ugb {

struct dxt1_blk {
        float2 R[8], G[8], B[8];
        float mnr, mng, mnb, mxr, mxg, mxb;
        float lor, hir, log_, hig, lob, hib;
        float2 sr2, sg2, sb2;
        float covx, covy;
        float qxr, qxg, qxb, qnr, qng, qnb;
        uint32_t max_code, min_code;
        float2 tr2, tg2, tb2;
        float nbias;
        uint32_t acc0, acc1;
};

__device__ __forceinline__ void d1_rgb_row(dxt1_blk &s, uint32_t w0, uint32_t w1, int y)
{
        const float2 c2 = dup(kInv255), ky2 = dup(kBiasY), kc2 = dup(kBiasC);
        const float2 u = __ffma2_rn(f2(magic_byte(w0, 0), magic_byte(w1, 0)), c2, kc2);
        const float2 v = __ffma2_rn(f2(magic_byte(w0, 2), magic_byte(w1, 2)), c2, kc2);
#pragma unroll
        for (int k = 0; k < 2; ++k) {
                const float2 yy = __fmul2_rn(__ffma2_rn(f2(magic_byte(w0, 1 + 2 * k), magic_byte(w1, 1 + 2 * k)), c2, ky2), dup(1.1643f));
                s.R[2 * y + k] = __ffma2_rn(v, dup(1.7926f), yy);
                s.G[2 * y + k] = __ffma2_rn(v, dup(-0.5328f), __ffma2_rn(u, dup(-0.2132f), yy));
                s.B[2 * y + k] = __ffma2_rn(u, dup(2.1124f), yy);
        }
}
/// bounding box seeded with the first pixel pair; d1_bbox_step() then takes pairs 1..7
__device__ __forceinline__ void d1_bbox_init(dxt1_blk &s)
{
        s.mnr = fminf(s.R[0].x, s.R[0].y), s.mxr = fmaxf(s.R[0].x, s.R[0].y);
        s.mng = fminf(s.G[0].x, s.G[0].y), s.mxg = fmaxf(s.G[0].x, s.G[0].y);
        s.mnb = fminf(s.B[0].x, s.B[0].y), s.mxb = fmaxf(s.B[0].x, s.B[0].y);
}
__device__ __forceinline__ void d1_bbox_step(dxt1_blk &s, int j)
{
        s.mnr = fminf(s.mnr, fminf(s.R[j].x, s.R[j].y)), s.mxr = fmaxf(s.mxr, fmaxf(s.R[j].x, s.R[j].y));
        s.mng = fminf(s.mng, fminf(s.G[j].x, s.G[j].y)), s.mxg = fmaxf(s.mxg, fmaxf(s.G[j].x, s.G[j].y));
        s.mnb = fminf(s.mnb, fminf(s.B[j].x, s.B[j].y)), s.mxb = fmaxf(s.mxb, fmaxf(s.B[j].x, s.B[j].y));
}
__device__ __forceinline__ void d1_inset(dxt1_blk &s)
{
        const float dr = __fadd_rn(s.mxr, -s.mnr), dg = __fadd_rn(s.mxg, -s.mng), db = __fadd_rn(s.mxb, -s.mnb);
        s.lor = __fmaf_rn(dr, 0.0625f, s.mnr), s.hir = __fmaf_rn(dr, -0.0625f, s.mxr);
        s.log_ = __fmaf_rn(dg, 0.0625f, s.mng), s.hig = __fmaf_rn(dg, -0.0625f, s.mxg);
        s.lob = __fmaf_rn(db, 0.0625f, s.mnb), s.hib = __fmaf_rn(db, -0.0625f, s.mxb);
        s.sr2 = dup(__fadd_rn(s.lor, s.hir)), s.sg2 = dup(__fadd_rn(s.log_, s.hig)), s.sb2 = dup(__fadd_rn(s.lob, s.hib));
        s.covx = 0.0f, s.covy = 0.0f;
}
/// deviations of pixel pair j and their four covariance terms.  The chain order i = 0..15 is pixel order: element j holds pixels
/// 4 (j >> 1) + (j & 1) (.x) and that + 2 (.y), so the pairs are consumed as j = 0, 1 (pixels 0, 1 then 2, 3 of row 0), 2, 3, ...
__device__ __forceinline__ void d1_cov_row(dxt1_blk &s, int y)
{
        const float2 mh = dup(-0.5f);
        const float2 er0 = __ffma2_rn(s.sr2, mh, s.R[2 * y]), er1 = __ffma2_rn(s.sr2, mh, s.R[2 * y + 1]);
        const float2 eg0 = __ffma2_rn(s.sg2, mh, s.G[2 * y]), eg1 = __ffma2_rn(s.sg2, mh, s.G[2 * y + 1]);
        const float2 eb0 = __ffma2_rn(s.sb2, mh, s.B[2 * y]), eb1 = __ffma2_rn(s.sb2, mh, s.B[2 * y + 1]);
        // pixels 4y, 4y+1, 4y+2, 4y+3 = (j0.x, j1.x, j0.y, j1.y)
        s.covx = __fmaf_rn(er0.x, eb0.x, s.covx), s.covy = __fmaf_rn(eg0.x, eb0.x, s.covy);
        s.covx = __fmaf_rn(er1.x, eb1.x, s.covx), s.covy = __fmaf_rn(eg1.x, eb1.x, s.covy);
        s.covx = __fmaf_rn(er0.y, eb0.y, s.covx), s.covy = __fmaf_rn(eg0.y, eb0.y, s.covy);
        s.covx = __fmaf_rn(er1.y, eb1.y, s.covx), s.covy = __fmaf_rn(eg1.y, eb1.y, s.covy);
}
__device__ __forceinline__ void d1_endpoints(dxt1_blk &s)
{
        const bool swr = s.covx < 0.0f, swg = s.covy < 0.0f;
        const float maxr = swr ? s.lor : s.hir, minr = swr ? s.hir : s.lor;
        const float maxg = swg ? s.log_ : s.hig, ming = swg ? s.hig : s.log_;
        s.qxr = quant_magic(maxr, 31.0f), s.qxg = quant_magic(maxg, 63.0f), s.qxb = quant_magic(s.hib, 31.0f);
        s.qnr = quant_magic(minr, 31.0f), s.qng = quant_magic(ming, 63.0f), s.qnb = quant_magic(s.lob, 31.0f);
        constexpr uint32_t kCodeBias = 0x4B400000u * 2081u;
        s.max_code = (__float_as_uint(s.qxr) << 11) + (__float_as_uint(s.qxg) << 5) + __float_as_uint(s.qxb) - kCodeBias;
        s.min_code = (__float_as_uint(s.qnr) << 11) + (__float_as_uint(s.qng) << 5) + __float_as_uint(s.qnb) - kCodeBias;
        const float ex_r = __fmul_rn(__fadd_rn(s.qxr, -kRoundMagic), kInv31);
        const float ex_g = __fmul_rn(__fadd_rn(s.qxg, -kRoundMagic), kInv63);
        const float ex_b = __fmul_rn(__fadd_rn(s.qxb, -kRoundMagic), kInv31);
        const float dir_r = __fmaf_rn(__fadd_rn(s.qnr, -kRoundMagic), kInv31, -ex_r);
        const float dir_g = __fmaf_rn(__fadd_rn(s.qng, -kRoundMagic), kInv63, -ex_g);
        const float dir_b = __fmaf_rn(__fadd_rn(s.qnb, -kRoundMagic), kInv31, -ex_b);
        const float len2 = __fmaf_rn(dir_b, dir_b, __fmaf_rn(dir_r, dir_r, __fmul_rn(dir_g, dir_g)));
        const float inv = __fdividef(1.0f, len2);
        const float tr = __fmul_rn(dir_r, inv), tg = __fmul_rn(dir_g, inv), tb = __fmul_rn(dir_b, inv);
        s.nbias = -__fmaf_rn(ex_b, tb, __fmaf_rn(ex_r, tr, __fmul_rn(ex_g, tg)));
        s.tr2 = dup(tr), s.tg2 = dup(tg), s.tb2 = dup(tb);
        s.acc0 = 0, s.acc1 = 0;
}
__device__ __forceinline__ void d1_index_step(dxt1_blk &s, int j)
{
        const float2 t = __ffma2_rn(s.B[j], s.tb2, __ffma2_rn(s.R[j], s.tr2, __fmul2_rn(s.G[j], s.tg2)));
        const float2 x = __ffma2_rn(f2(add_sat_rn(t.x, s.nbias), add_sat_rn(t.y, s.nbias)), dup(3.0f), dup(0.5f));
        const float2 m = __fadd2_rd(x, dup(kFloorMagic));
        const int i0 = 4 * (j >> 1) + (j & 1);
        s.acc0 += __float_as_uint(m.x) << (2 * i0);
        s.acc1 += __float_as_uint(m.y) << (2 * (i0 + 2));
}
__device__ __forceinline__ uint2 d1_pack(const dxt1_blk &s)
{
        constexpr uint32_t kIdxBias = 0x4B000000u * 0x55555555u;
        uint32_t indices = s.acc0 + s.acc1 - kIdxBias;
        indices = s.max_code != s.min_code ? indices : 0u;  // a flat block's indices are computed too (inf / NaN arithmetic has no side effect) and dropped
        const bool swap_end = s.max_code < s.min_code;
        if (swap_end) {
                indices = ~indices;
        }
        const uint32_t lsbs = indices & 0x55555555u, msbs = indices & 0xaaaaaaaau;
        indices = msbs ^ (2 * lsbs + (msbs >> 1));
        const uint32_t palette = swap_end ? s.min_code + (s.max_code << 16) : s.max_code + (s.min_code << 16);
        return make_uint2(palette, indices);
}

/// two horizontally adjacent blocks: v[y] = the 16 bytes (8 pixels) of row y
__device__ __forceinline__ uint4 dxt1_encode_uyvy_pair_skewed(const uint4 (&v)[4])
{
        dxt1_blk a, b;
#pragma unroll
        for (int y = 0; y < 4; ++y) {
                d1_rgb_row(a, v[y].x, v[y].y, y);
        }
        d1_bbox_init(a);
#pragma unroll
        for (int y = 0; y < 4; ++y) {  // B: unpack + RGB (FMA pipe, PRMT)   A: bounding box (ALU pipe)
                d1_rgb_row(b, v[y].z, v[y].w, y);
                if (y > 0) {
                        d1_bbox_step(a, 2 * y);
                }
                d1_bbox_step(a, 2 * y + 1);
        }
        d1_inset(a);
        d1_bbox_init(b);
#pragma unroll
        for (int y = 0; y < 4; ++y) {  // A: deviations + covariance chains (FMA pipe)   B: bounding box (ALU pipe)
                d1_cov_row(a, y);
                if (y > 0) {
                        d1_bbox_step(b, 2 * y);
                }
                d1_bbox_step(b, 2 * y + 1);
        }
        d1_endpoints(a);
        d1_inset(b);
#pragma unroll
        for (int y = 0; y < 4; ++y) {  // A: indices   B: deviations + covariance
                d1_index_step(a, 2 * y);
                d1_cov_row(b, y);
                d1_index_step(a, 2 * y + 1);
        }
        d1_endpoints(b);
        const uint2 ra = d1_pack(a);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
                d1_index_step(b, j);
        }
        const uint2 rb = d1_pack(b);
        return make_uint4(ra.x, ra.y, rb.x, rb.y);
}

}  // namespace ugb
