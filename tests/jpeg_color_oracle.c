/* TEST INFRASTRUCTURE - not part of the product.
 * CPU restatement of JPEG decode in a colour space (ugb200_jpeg_decode_cs, include/ugb200_jpeg.h): the decode oracle's own samples
 * (oracle/jpeg_decode_oracle.c, included), then UltraGrid's integer YCbCr -> RGB (YCBCR_TO_R/G/B, src/color_space.h:106-109) at 8 bits
 * with the coefficients of the declared space and its luma offset, `>>` a floor:
 *   cs 1 = Y601 (coeffs_601(8), o = 16), 2 = Y601FULL (coeffs_601(0), o = 0), 3 = Y709 (coeffs_709(8), o = 16)   (UGB200_JPEG_CS_*)
 * Chroma is replicated: a 4:2:2 / 4:2:0 stream is decoded to UYVY (both rows of a 4:2:0 pair take the same chroma row) and each word's
 * Cb / Cr serve both of its pixels; only whole pixel pairs are written (an odd width leaves the last pixel of each row as it was).
 * A 4:4:4 stream is converted pixel by pixel. */
#include "../oracle/jpeg_decode_oracle.c"

struct cs_coeffs {
        int y_scale, r_cr, g_cb, g_cr, b_cb, y_off;
};

/* compute_color_coeffs (UltraGrid's color_space.c:116-128, 192-196): the inverse row, rounded as scaled() rounds */
static int scaled(double x) { return (int) (x * (1 << 14) + (x > 0 ? 1. : -1.) * 0.5); }
static struct cs_coeffs coeffs(int cs)
{
        const double kr = cs == 3 ? .212639 : .299, kb = cs == 3 ? .072192 : .114, kg = 1. - kr - kb;
        const int depth = cs == 2 ? 0 : 8;
        const double yl = depth == 0 ? 1.0 : 219. / 255., cl = depth == 0 ? 1.0 : 224. / 255.;
        struct cs_coeffs c;
        c.y_scale = scaled(1. / yl);
        c.r_cr = scaled((2. * (1. - kr)) / cl);
        c.g_cb = scaled((-kb * (2. * (kr + kg))) / kg / cl);
        c.g_cr = scaled((-kr * (2. * (1. - kr))) / kg / cl);
        c.b_cb = scaled((2. * (kr + kg)) / cl);
        c.y_off = depth == 0 ? 0 : 16;
        return c;
}

static uint8_t clamp8(int v) { return (uint8_t) (v < 0 ? 0 : v > 255 ? 255 : v); }

static void convert(const struct cs_coeffs *c, int y, int cb, int cr, uint8_t rgb[3])
{
        const int ys = c->y_scale * (y - c->y_off);
        rgb[0] = clamp8((ys + c->r_cr * (cr - 128)) >> 14);
        rgb[1] = clamp8((ys + c->g_cb * (cb - 128) + c->g_cr * (cr - 128)) >> 14);
        rgb[2] = clamp8((ys + c->b_cb * (cb - 128)) >> 14);
}

/* the coefficient row (y_scale, r_cr, g_cb, g_cr, b_cb, y_off) of colour space cs */
API void orc_cs_coeffs(int cs, int *out)
{
        const struct cs_coeffs c = coeffs(cs);
        out[0] = c.y_scale, out[1] = c.r_cr, out[2] = c.g_cb, out[3] = c.g_cr, out[4] = c.b_cb, out[5] = c.y_off;
}

/* n (Y, Cb, Cr) triples -> n (R, G, B) triples */
API void orc_ycbcr_to_rgb(int cs, const uint8_t *ycc, uint8_t *rgb, long n)
{
        const struct cs_coeffs c = coeffs(cs);
        for (long i = 0; i < n; ++i) {
                convert(&c, ycc[3 * i], ycc[3 * i + 1], ycc[3 * i + 2], rgb + 3 * i);
        }
}

static void store(uint8_t *d, const uint8_t rgb[3], int rgba, int rs, int gs, int bs)
{
        if (!rgba) {
                d[0] = rgb[0], d[1] = rgb[1], d[2] = rgb[2];
                return;
        }
        const uint32_t v = (0xFFFFFFFFu ^ (0xFFu << rs) ^ (0xFFu << gs) ^ (0xFFu << bs)) | (uint32_t) rgb[0] << rs | (uint32_t) rgb[1] << gs | (uint32_t) rgb[2] << bs;
        d[0] = (uint8_t) v, d[1] = (uint8_t) (v >> 8), d[2] = (uint8_t) (v >> 16), d[3] = (uint8_t) (v >> 24);
}

/* UYVY rows (pitch upitch) -> RGB (rgba 0) or RGBA with shifts, whole pixel pairs only */
API void orc_uyvy_to_rgb_cs(int cs, const uint8_t *uyvy, long upitch, int w, int h, int rgba, int rs, int gs, int bs, uint8_t *out, long pitch)
{
        const struct cs_coeffs c = coeffs(cs);
        const int bpp = rgba ? 4 : 3;
        for (int y = 0; y < h; ++y) {
                for (int p = 0; p < w / 2; ++p) {
                        const uint8_t *u = uyvy + (long) y * upitch + 4 * p;
                        uint8_t rgb[3];
                        convert(&c, u[1], u[0], u[2], rgb);
                        store(out + (long) y * pitch + (long) (2 * p) * bpp, rgb, rgba, rs, gs, bs);
                        convert(&c, u[3], u[0], u[2], rgb);
                        store(out + (long) y * pitch + (long) (2 * p + 1) * bpp, rgb, rgba, rs, gs, bs);
                }
        }
}

/* decode `s` and convert its samples from colour space cs to RGB / RGBA (rgba, shifts) in `out` (pitch bytes per row); returns the decode's code */
API int orc_jpeg_decode_cs(const uint8_t *s, size_t len, int cs, int rgba, int rs, int gs, int bs, uint8_t *out, long pitch)
{
        int info[6], rc;
        const uint8_t *p = s + 2;  /* SOF0: the size of the scratch frame the samples are decoded into */
        int w = 0, h = 0, hs = 1;
        while (p + 4 <= s + len && p[0] == 0xFF) {
                const int mk = p[1], L = be16(p + 2);
                if (mk == 0xC0) {
                        h = be16(p + 5), w = be16(p + 7), hs = p[11] >> 4;
                        break;
                }
                p += 2 + L;
        }
        if (w == 0 || h == 0) {
                return -3;
        }
        const long upitch = hs == 2 ? (long) (w + 1) / 2 * 4 : (long) w * 3;
        uint8_t *tmp = malloc((size_t) upitch * h + 64);
        if (!tmp) {
                return -2;
        }
        rc = orc_jpeg_decode(s, len, hs == 2 ? 0 : 1, tmp, upitch, info);
        if (rc == 0) {
                if (hs == 2) {
                        orc_uyvy_to_rgb_cs(cs, tmp, upitch, w, h, rgba, rs, gs, bs, out, pitch);
                } else {
                        const struct cs_coeffs c = coeffs(cs);
                        for (int y = 0; y < h; ++y) {
                                for (int x = 0; x < w; ++x) {
                                        const uint8_t *q = tmp + (long) y * upitch + 3L * x;
                                        uint8_t rgb[3];
                                        convert(&c, q[0], q[1], q[2], rgb);
                                        store(out + (long) y * pitch + (long) x * (rgba ? 4 : 3), rgb, rgba, rs, gs, bs);
                                }
                        }
                }
        }
        free(tmp);
        return rc;
}
