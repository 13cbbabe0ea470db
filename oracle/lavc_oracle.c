/* TEST INFRASTRUCTURE - CPU restatement of the libavcodec bridge conversions of src/libavcodec/to_lavc_vid_conv.c that
 * ultragrid_b200/csrc/lavc_conv_kernels.cu implements (SURVEY.md section 8f rank 3).
 *
 * PARITY UNPINNED against the reference object: to_lavc_vid_conv.c needs libavutil / libavcodec headers (AVFrame, AV_PIX_FMT_*, pixdesc), which
 * are not in this image, so the file itself cannot be compiled here.  What pins this restatement instead: (1) each function cites the lines it
 * follows; (2) the colour coefficients come from the UNMODIFIED src/color_space.c (oracle/_ref: ref_get_color_coeffs) in the tests;
 * (3) identities against functions that ARE pinned: v210 -> yuv422p10le -> v210 round trip through the reference's yuv422p10le_to_v210
 * (from_planar.c:295-333, the idea of test/ff_codec_conversions_test.cpp:346-401), v210 -> yuv420p10le == v210_to_p010le >> 6
 * (to_planar.c:64-155), UYVY -> yuv422p == the inverse of yuv422p_to_uyvy.  A frame is plane pointers + line sizes (the AVFrame fields the
 * reference touches). */
#include <stdint.h>
#include <string.h>

#define API __attribute__((visibility("default")))

struct coeffs { /* struct color_coeffs, src/color_space.h:135-149 (first nine members) */
        int y_r, y_g, y_b, cb_r, cb_g, cb_b, cr_r, cr_g, cr_b;
};
enum { LAVC_COMP_BASE = 14 };

static long v210_linesize(int w) { return (long) ((w + 47) / 48) * 128; }
static uint32_t s10(uint32_t w, int sh) { return (w >> sh) & 0x3ff; }

/* mode 0: v210_to_yuv420p10le (:197-262), 1: v210_to_yuv422p10le (:264-301), 2: v210_to_yuv444p10le (:303-346), 3: v210_to_yuv444p16le (:348-385) */
API void orc_lavc_v210(int mode, const uint8_t *in, int width, int height, uint8_t *const p[3], const int ls[3])
{
        const int sh = mode == 3 ? 6 : 0;
        for (int y = 0; y < height; y += mode == 0 ? 2 : 1) {
                if (mode == 0 && y + 1 >= height) {
                        break; /* the reference would read and write one row beyond the frame here */
                }
                const uint32_t *s0 = (const uint32_t *) (in + y * v210_linesize(width)), *s1 = (const uint32_t *) (in + (y + 1) * v210_linesize(width));
                uint16_t *dy = (uint16_t *) (p[0] + (long) ls[0] * y), *dy2 = (uint16_t *) (p[0] + (long) ls[0] * (y + 1));
                uint16_t *dcb = (uint16_t *) (p[1] + (long) ls[1] * (mode == 0 ? y / 2 : y)), *dcr = (uint16_t *) (p[2] + (long) ls[2] * (mode == 0 ? y / 2 : y));
                for (int x = 0; x < width / 6; ++x) {
                        const uint32_t *a = s0 + 4 * x, *b = s1 + 4 * x;
                        *dy++ = s10(a[0], 10) << sh, *dy++ = s10(a[1], 0) << sh, *dy++ = s10(a[1], 20) << sh;
                        *dy++ = s10(a[2], 10) << sh, *dy++ = s10(a[3], 0) << sh, *dy++ = s10(a[3], 20) << sh;
                        uint32_t u[3] = { s10(a[0], 0), s10(a[1], 10), s10(a[2], 20) }, v[3] = { s10(a[0], 20), s10(a[2], 0), s10(a[3], 10) };
                        if (mode == 0) {
                                *dy2++ = s10(b[0], 10), *dy2++ = s10(b[1], 0), *dy2++ = s10(b[1], 20);
                                *dy2++ = s10(b[2], 10), *dy2++ = s10(b[3], 0), *dy2++ = s10(b[3], 20);
                                u[0] = (u[0] + s10(b[0], 0)) / 2, u[1] = (u[1] + s10(b[1], 10)) / 2, u[2] = (u[2] + s10(b[2], 20)) / 2;
                                v[0] = (v[0] + s10(b[0], 20)) / 2, v[1] = (v[1] + s10(b[2], 0)) / 2, v[2] = (v[2] + s10(b[3], 10)) / 2;
                        }
                        for (int j = 0; j < 3; ++j) {
                                *dcb++ = u[j] << sh, *dcr++ = v[j] << sh;
                                if (mode >= 2) {
                                        *dcb++ = u[j] << sh, *dcr++ = v[j] << sh;
                                }
                        }
                }
        }
}

/* uyvy_to_yuv422p (:137-151), uyvy_to_yuv444p (:172-184) */
API void orc_lavc_uyvy(int to444, const uint8_t *in, int width, int height, uint8_t *const p[3], const int ls[3])
{
        for (int y = 0; y < height; ++y) {
                const uint8_t *src = in + (long) y * ((width + 1) / 2) * 4; /* the source pointer runs on over (width + 1) / 2 pairs per row */
                uint8_t *dy = p[0] + (long) ls[0] * y, *dcb = p[1] + (long) ls[1] * y, *dcr = p[2] + (long) ls[2] * y;
                for (int x = 0; x < width; x += 2) {
                        *dcb++ = src[0];
                        *dy++ = src[1];
                        *dcr++ = src[2];
                        *dy++ = src[3];
                        if (to444) {
                                *dcb++ = src[0], *dcr++ = src[2];
                        }
                        src += 4;
                }
        }
}

static void put3(const struct coeffs *c, int in_depth, int depth, int r, int g, int b, int *y, int *cb, int *cr)
{ /* the RGB_TO_* expressions of :722-733 (R10k), :1155-1163 (RG48), :1206-1214 (RGB), WRITE_RES :768-787 (R12L) */
        const int sh = LAVC_COMP_BASE + in_depth - depth;
        *y = ((r * c->y_r + g * c->y_g + b * c->y_b) >> sh) + (1 << (depth - 4));
        *cb = ((r * c->cb_r + g * c->cb_g + b * c->cb_b) >> sh) + (1 << (depth - 1));
        *cr = ((r * c->cr_r + g * c->cr_g + b * c->cr_b) >> sh) + (1 << (depth - 1));
}

/* src 0: r10k_to_yuv444pXXle (:702-755), 1: rg48_to_yuv444pXXle (:1132-1183), 2: r12l_to_yuv4XXpYYle (:757-895; sub422 = out_422),
 * 3: rgb_to_yuv444p (:1185-1227; 8-bit planes).  CLAMP_LIMITED_* are identities (color_space.h:93-94): the stores wrap. */
API void orc_lavc_rgb(int src_kind, int depth, int sub422, const struct coeffs *c, const uint8_t *in, int width, int height, uint8_t *const p[3],
                      const int ls[3])
{
        for (int y = 0; y < height; ++y) {
                int Y, CB, CR;
                if (src_kind == 3) {
                        const uint8_t *s = in + (long) y * width * 3;
                        uint8_t *dy = p[0] + (long) ls[0] * y, *dcb = p[1] + (long) ls[1] * y, *dcr = p[2] + (long) ls[2] * y;
                        for (int x = 0; x < width; ++x, s += 3) {
                                put3(c, 8, 8, s[0], s[1], s[2], &Y, &CB, &CR);
                                *dy++ = (uint8_t) Y, *dcb++ = (uint8_t) CB, *dcr++ = (uint8_t) CR;
                        }
                        continue;
                }
                uint16_t *dy = (uint16_t *) (p[0] + (long) ls[0] * y), *dcb = (uint16_t *) (p[1] + (long) ls[1] * y), *dcr = (uint16_t *) (p[2] + (long) ls[2] * y);
                if (src_kind == 0) {
                        const uint8_t *s = in + (long) y * ((width + 63) / 64) * 256; /* vc_get_linesize(width, R10k): 64-pixel rows (:712) */
                        for (int x = 0; x < width; ++x, s += 4) {
                                put3(c, 10, depth, s[0] << 2 | s[1] >> 6, (s[1] & 0x3F) << 4 | s[2] >> 4, (s[2] & 0x0F) << 6 | s[3] >> 2, &Y, &CB, &CR);
                                *dy++ = (uint16_t) Y, *dcb++ = (uint16_t) CB, *dcr++ = (uint16_t) CR;
                        }
                } else if (src_kind == 1) {
                        const uint16_t *s = (const uint16_t *) (in + (long) y * width * 6);
                        for (int x = 0; x < width; ++x, s += 3) {
                                put3(c, 16, depth, s[0], s[1], s[2], &Y, &CB, &CR);
                                *dy++ = (uint16_t) Y, *dcb++ = (uint16_t) CB, *dcr++ = (uint16_t) CR;
                        }
                } else {
                        const uint8_t *s = in + (long) y * ((width + 7) / 8) * 36;
                        const long cap_y = ls[0] / 2, cap_c = ls[1] / 2;
                        for (int x = 0; x < width; x += 8, s += 36) { /* whole groups, like the reference; clipped to the plane row */
                                int r[8], g[8], b[8];
                                /* the byte picking of :790-870 */
                                r[0] = s[0] | (s[1] & 0xF) << 8, g[0] = s[2] << 4 | s[1] >> 4, b[0] = s[3] | (s[4] & 0xF) << 8;
                                r[1] = s[5] << 4 | s[4] >> 4, g[1] = s[6] | (s[7] & 0xF) << 8, b[1] = s[7] >> 4 | s[8] << 4;
                                r[2] = s[9] | (s[10] & 0xF) << 8, g[2] = s[11] << 4 | s[10] >> 4, b[2] = s[12] | (s[13] & 0xF) << 8;
                                r[3] = s[14] << 4 | s[13] >> 4, g[3] = s[15] | (s[16] & 0xF) << 8, b[3] = s[17] << 4 | s[16] >> 4;
                                r[4] = s[18] | (s[19] & 0xF) << 8, g[4] = s[19] >> 4 | s[20] << 4, b[4] = s[21] | (s[22] & 0xF) << 8;
                                r[5] = s[23] << 4 | s[22] >> 4, g[5] = s[24] | (s[25] & 0xF) << 8, b[5] = s[26] << 4 | s[25] >> 4;
                                r[6] = s[27] | (s[28] & 0xF) << 8, g[6] = s[29] << 4 | s[28] >> 4, b[6] = s[30] | (s[31] & 0xF) << 8;
                                r[7] = s[31] >> 4 | s[32] << 4, g[7] = s[33] | (s[34] & 0xF) << 8, b[7] = s[35] << 4 | s[34] >> 4;
                                for (int i = 0; i < 8; ++i) {
                                        put3(c, 12, depth, r[i], g[i], b[i], &Y, &CB, &CR);
                                        if (x + i < cap_y) {
                                                dy[x + i] = (uint16_t) Y;
                                        }
                                        if (!sub422 && x + i < cap_c) {
                                                dcb[x + i] = (uint16_t) CB, dcr[x + i] = (uint16_t) CR;
                                        } else if (sub422 && i % 2 == 0 && (x + i) / 2 < cap_c) {
                                                dcb[(x + i) / 2] = (uint16_t) CB, dcr[(x + i) / 2] = (uint16_t) CR;
                                        }
                                }
                        }
                }
        }
}

/* rgb_rgba_to_gbrp (:1315-1333): planes G, B, R */
API void orc_lavc_gbrp(int bpp, const uint8_t *in, int width, int height, uint8_t *const p[3], const int ls[3])
{
        for (int y = 0; y < height; ++y) {
                const uint8_t *s = in + (long) y * width * bpp;
                for (int x = 0; x < width; ++x, s += bpp) {
                        p[0][(long) ls[0] * y + x] = s[1], p[1][(long) ls[1] * y + x] = s[2], p[2][(long) ls[2] * y + x] = s[0];
                }
        }
}
