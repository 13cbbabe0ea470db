// Q14 integer RGB<->YCbCr coefficients — the contract of UltraGrid's src/color_space.{h,c}.
//
// The reference derives the coefficients in double at compile time (color_space.c:46-131) and rounds
// with +-0.5 before truncating to int (C_EPS, color_space.c:55).  The same formulas are evaluated here
// as constexpr and pinned with static_asserts to the values probed from the reference build
// (SURVEY.md section 8 A3), so a transcription error cannot compile.
#pragma once
#include <stdint.h>

namespace ugb {

constexpr int COMP_BASE = 14;  // color_space.h:70 (comp_type_t is int32_t)

constexpr double KR_709 = .212639, KB_709 = .072192;  // color_space.h:75-76
constexpr double KR_601 = .299, KB_601 = .114;        // color_space.h:73-74

struct color_coeffs {  // field meaning as color_space.h:135-149 (all widened to int here)
        int y_r, y_g, y_b;
        int cb_r, cb_g, cb_b;
        int cr_r, cr_g, cr_b;
        int y_scale;
        int r_cr, g_cb, g_cr;
        int b_cb;
};

namespace detail {
constexpr double kg(double kr, double kb) { return 1. - kr - kb; }
constexpr double dd(double kr, double kb) { return 2. * (kr + kg(kr, kb)); }  // D(), color_space.c:47
constexpr double ee(double kr) { return 2. * (1. - kr); }                     // E(), color_space.c:48
// limited-range scale factors, color_space.c:56-63; depth 0 = full range
constexpr double y_limit(int d) { return d == 0 ? 1.0 : (219. * (1 << (d - 8)) / ((1 << d) - 1)); }
constexpr double c_limit(int d) { return d == 0 ? 1.0 : (224. * (1 << (d - 8)) / ((1 << d) - 1)); }
constexpr int    to_i(double v) { return (int) v; }  // C cast: truncation toward zero
constexpr int    scaled(double x) { return to_i(x * (1 << COMP_BASE) + (x > 0 ? 1. : -1.) * 0.5); }  // color_space.c:104-105
}  // namespace detail

/// compute_color_coeffs(), color_space.c:192-196 / COEFFS(), color_space.c:116-128
constexpr color_coeffs compute_color_coeffs(double kr, double kb, int depth)
{
        using namespace detail;
        const double B = 1 << COMP_BASE;
        return color_coeffs{
                to_i(kr * y_limit(depth) * B + 0.5),
                to_i(kg(kr, kb) * y_limit(depth) * B + 0.5),
                to_i(kb * y_limit(depth) * B + 0.5),
                to_i(-kr / dd(kr, kb) * c_limit(depth) * B - 0.5),
                to_i(-kg(kr, kb) / dd(kr, kb) * c_limit(depth) * B - 0.5),
                to_i((1 - kb) / dd(kr, kb) * c_limit(depth) * B + 0.5),
                to_i((1 - kr) / ee(kr) * c_limit(depth) * B - 0.5),
                to_i(-kg(kr, kb) / ee(kr) * c_limit(depth) * B - 0.5),
                to_i(-kb / ee(kr) * c_limit(depth) * B + 0.5),
                scaled(1. / y_limit(depth)),
                scaled((2. * (1. - kr)) / c_limit(depth)),
                scaled((-kb * (2. * (kr + kg(kr, kb))) / kg(kr, kb)) / c_limit(depth)),
                scaled((-kr * (2. * (1. - kr)) / kg(kr, kb)) / c_limit(depth)),
                scaled((2. * (kr + kg(kr, kb))) / c_limit(depth)),
        };
}

/// get_color_coeffs(CS_DFL, depth) with the default (BT.709) colour space, color_space.c:149-183.
/// depth 0 = full range.
constexpr color_coeffs coeffs_709(int depth) { return compute_color_coeffs(KR_709, KB_709, depth); }
constexpr color_coeffs coeffs_601(int depth) { return compute_color_coeffs(KR_601, KB_601, depth); }

/// The coefficient set of get_color_coeffs(CS_DFL, depth) as a compile-time parameter of the converters that read it: bt709 under UltraGrid's
/// default, bt601 under `--param color-601` (get_default_cs(), color_space.c:186-191).  A converter takes one as a template argument, so its
/// coefficients stay immediates in each instantiation; the launcher picks the instantiation from the caller's colour space.
struct bt709 {
        static constexpr color_coeffs at(int depth) { return coeffs_709(depth); }
};
struct bt601 {
        static constexpr color_coeffs at(int depth) { return coeffs_601(depth); }
};

// ---- pinned to the reference build (SURVEY.md 8a A3) --------------------------------------------
namespace pin {
constexpr color_coeffs c8 = coeffs_709(8), c10 = coeffs_709(10), c16 = coeffs_709(16), c0 = coeffs_709(0);
static_assert(c8.y_r == 2992 && c8.y_g == 10063 && c8.y_b == 1016, "709/8 Y row");
static_assert(c8.cb_r == -1649 && c8.cb_g == -5547 && c8.cb_b == 7196, "709/8 Cb row");
static_assert(c8.cr_r == 7195 && c8.cr_g == -6536 && c8.cr_b == -659, "709/8 Cr row");
static_assert(c8.y_scale == 19077 && c8.r_cr == 29371 && c8.g_cb == -3494 && c8.g_cr == -8733 && c8.b_cb == 34610, "709/8 inverse");
static_assert(c10.y_r == 2983 && c10.y_g == 10034 && c10.y_b == 1013, "709/10 Y row");
static_assert(c10.cb_r == -1644 && c10.cb_g == -5531 && c10.cb_b == 7175, "709/10 Cb row");
static_assert(c10.cr_r == 7174 && c10.cr_g == -6517 && c10.cr_b == -657, "709/10 Cr row");
static_assert(c10.y_scale == 19133 && c10.r_cr == 29457 && c10.g_cb == -3504 && c10.g_cr == -8758 && c10.b_cb == 34712, "709/10 inverse");
static_assert(c16.y_r == 2980 && c16.y_g == 10024 && c16.y_b == 1012, "709/16 Y row");
static_assert(c16.cb_r == -1643 && c16.cb_g == -5525 && c16.cb_b == 7168, "709/16 Cb row");
static_assert(c16.cr_r == 7167 && c16.cr_g == -6511 && c16.cr_b == -656, "709/16 Cr row");
static_assert(c16.y_scale == 19152 && c16.r_cr == 29486 && c16.g_cb == -3507 && c16.g_cr == -8767 && c16.b_cb == 34745, "709/16 inverse");
static_assert(c0.y_r == 3484 && c0.y_g == 11717 && c0.y_b == 1183, "709/full Y row");
static_assert(c0.cb_r == -1877 && c0.cb_g == -6315 && c0.cb_b == 8192, "709/full Cb row");
static_assert(c0.cr_r == 8191 && c0.cr_g == -7441 && c0.cr_b == -750, "709/full Cr row");
static_assert(c0.y_scale == 16384 && c0.r_cr == 25800 && c0.g_cb == -3069 && c0.g_cr == -7671 && c0.b_cb == 30402, "709/full inverse");
// BT.601, as the reference built with color-601 returns them for CS_DFL (tests/test_color601.py probes every depth)
constexpr color_coeffs s8 = coeffs_601(8), s10 = coeffs_601(10), s16 = coeffs_601(16);
static_assert(s8.y_r == 4207 && s8.y_g == 8260 && s8.y_b == 1604, "601/8 Y row");
static_assert(s8.cb_r == -2428 && s8.cb_g == -4768 && s8.cb_b == 7196, "601/8 Cb row");
static_assert(s8.cr_r == 7195 && s8.cr_g == -6026 && s8.cr_b == -1169, "601/8 Cr row");
static_assert(s8.y_scale == 19077 && s8.r_cr == 26149 && s8.g_cb == -6419 && s8.g_cr == -13320 && s8.b_cb == 33050, "601/8 inverse");
static_assert(s10.y_r == 4195 && s10.y_g == 8235 && s10.y_b == 1599 && s10.cb_r == -2421 && s10.cb_g == -4754 && s10.cb_b == 7175, "601/10 Y, Cb");
static_assert(s10.cr_r == 7174 && s10.cr_g == -6008 && s10.cr_b == -1166, "601/10 Cr row");
static_assert(s10.y_scale == 19133 && s10.r_cr == 26226 && s10.g_cb == -6438 && s10.g_cr == -13359 && s10.b_cb == 33148, "601/10 inverse");
static_assert(s16.y_r == 4191 && s16.y_g == 8228 && s16.y_b == 1598 && s16.cb_r == -2419 && s16.cb_g == -4749 && s16.cb_b == 7168, "601/16 Y, Cb");
static_assert(s16.cr_r == 7167 && s16.cr_g == -6002 && s16.cr_b == -1165, "601/16 Cr row");
static_assert(s16.y_scale == 19152 && s16.r_cr == 26251 && s16.g_cb == -6444 && s16.g_cr == -13372 && s16.b_cb == 33179, "601/16 inverse");
}  // namespace pin

// ---- YCbCr -> YCbCr between two colour spaces (ugb200_jpeg_decode_to) ------------------------------------------------------------
//   Y'  = clamp(((yy * (Y - o_in) + yb * (Cb - 128) + yr * (Cr - 128) + 8192) >> 14) + o_out, 0, 255)
//   Cb' = clamp(((bb * (Cb - 128) + br * (Cr - 128) + 8192) >> 14) + 128, 0, 255)
//   Cr' = clamp(((rb * (Cb - 128) + rr * (Cr - 128) + 8192) >> 14) + 128, 0, 255)
// The coefficients are round(2^14 * M), M = (RGB -> YCbCr of the target) * (YCbCr -> RGB of the source), formed in double from kr, kb and
// the range scales above and rounded once (not the product of the rounded Q14 tables).  The target's chroma does not depend on the
// source's luma: both are scaled B - Y and R - Y, and a grey source pixel (Cb = Cr = 128) has R = G = B.
struct ycc_matrix {
        int yy, yb, yr;
        int bb, br;
        int rb, rr;
        int o_in, o_out;
};

constexpr ycc_matrix compute_ycc_matrix(double kr_s, double kb_s, int depth_s, double kr_t, double kb_t, int depth_t)
{
        using namespace detail;
        const double ys = 1. / y_limit(depth_s), cs = 1. / c_limit(depth_s), kg_s = kg(kr_s, kb_s);
        // R, G, B of the source as rows over (Y - o_in, Cb - 128, Cr - 128)
        const double r[3] = { ys, 0., ee(kr_s) * cs };
        const double g[3] = { ys, -kb_s * dd(kr_s, kb_s) / kg_s * cs, -kr_s * ee(kr_s) / kg_s * cs };
        const double b[3] = { ys, dd(kr_s, kb_s) * cs, 0. };
        const double l[3] = { kr_t * r[0] + kg(kr_t, kb_t) * g[0] + kb_t * b[0], kr_t * r[1] + kg(kr_t, kb_t) * g[1] + kb_t * b[1],
                              kr_t * r[2] + kg(kr_t, kb_t) * g[2] + kb_t * b[2] };  // full-range luma of the target
        const double yt = y_limit(depth_t), cb = c_limit(depth_t) / dd(kr_t, kb_t), cr = c_limit(depth_t) / ee(kr_t);
        return ycc_matrix{ scaled(yt * l[0]),          scaled(yt * l[1]),          scaled(yt * l[2]),
                           scaled(cb * (b[1] - l[1])), scaled(cb * (b[2] - l[2])), scaled(cr * (r[1] - l[1])), scaled(cr * (r[2] - l[2])),
                           depth_s == 0 ? 0 : 16,      depth_t == 0 ? 0 : 16 };
}

/// the spaces in the order of UGB200_JPEG_CS_Y601, _Y601FULL, _Y709 (values 1, 2, 3 of include/ugb200_jpeg.h)
constexpr ycc_matrix ycc_matrix_between(int cs_in, int cs_out)
{
        return compute_ycc_matrix(cs_in == 3 ? KR_709 : KR_601, cs_in == 3 ? KB_709 : KB_601, cs_in == 2 ? 0 : 8, cs_out == 3 ? KR_709 : KR_601,
                                  cs_out == 3 ? KB_709 : KB_601, cs_out == 2 ? 0 : 8);
}

namespace pin {
constexpr bool ycc_is(const ycc_matrix &m, int yy, int yb, int yr, int bb, int br, int rb, int rr, int o_in, int o_out)
{
        return m.yy == yy && m.yb == yb && m.yr == yr && m.bb == bb && m.br == br && m.rb == rb && m.rr == rr && m.o_in == o_in && m.o_out == o_out;
}
static_assert(ycc_is(ycc_matrix_between(1, 1), 16384, 0, 0, 16384, 0, 0, 16384, 16, 16), "Y601 -> Y601 is the identity");
static_assert(ycc_is(ycc_matrix_between(2, 2), 16384, 0, 0, 16384, 0, 0, 16384, 0, 0), "Y601FULL -> Y601FULL is the identity");
static_assert(ycc_is(ycc_matrix_between(3, 3), 16384, 0, 0, 16384, 0, 0, 16384, 16, 16), "Y709 -> Y709 is the identity");
static_assert(ycc_is(ycc_matrix_between(2, 3), 14071, -1663, -2992, 14660, 1649, 1080, 14757, 0, 16), "JFIF -> BT.709: what a camera's MJPEG needs");
static_assert(ycc_is(ycc_matrix_between(3, 2), 19077, 1895, 3656, 18462, -2063, -1351, 18342, 16, 0), "Y709 -> Y601FULL");
static_assert(ycc_is(ycc_matrix_between(1, 3), 16384, -1893, -3406, 16689, 1877, 1230, 16799, 16, 16), "Y601 -> Y709");
static_assert(ycc_is(ycc_matrix_between(2, 1), 14071, 0, 0, 14392, 0, 0, 14392, 0, 16), "Y601FULL -> Y601: a range change only");
}  // namespace pin

}  // namespace ugb
