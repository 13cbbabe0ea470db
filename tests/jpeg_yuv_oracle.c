/* TEST INFRASTRUCTURE - not part of the product.
 * CPU restatement of JPEG decode to a YCbCr colour space (ugb200_jpeg_decode_to, include/ugb200_jpeg.h), written from the header's contract:
 * the decode oracle's own samples (oracle/jpeg_decode_oracle.c, included), each converted between two of
 *   cs 1 = Y601 (BT.601, 16-235/240), 2 = Y601FULL (BT.601, JFIF full range), 3 = Y709 (BT.709, 16-235/240)   (UGB200_JPEG_CS_*)
 * with the seven coefficients round(2^14 * M), M = F(target) * I(source): F the 3 x 3 RGB -> YCbCr matrix of a space and I the 3 x 3
 * YCbCr -> RGB matrix, both built in double from kr, kb and the range scales 219 / 255 and 224 / 255, multiplied in double and rounded once.
 * "Convert, then pack": the conversion is applied to the samples at the stream's sampling, and packing to UYVY only permutes and
 * replicates samples, so it is applied here to the UYVY words of the decode oracle (a word's Cb / Cr once, its two lumas with that source
 * chroma), to the Y Cb Cr triples of a 4:4:4 stream, and to the luma of a grayscale stream (chroma stays 128). */
#include "../oracle/jpeg_decode_oracle.c"

struct space {
        double kr, kb, yl, cl;
        int off;
};
static struct space space_of(int cs)
{
        struct space s;
        s.kr = cs == 3 ? .212639 : .299, s.kb = cs == 3 ? .072192 : .114;
        s.yl = cs == 2 ? 1. : 219. / 255., s.cl = cs == 2 ? 1. : 224. / 255.;
        s.off = cs == 2 ? 0 : 16;
        return s;
}
/* rows Y, Cb, Cr over columns R, G, B */
static void forward(const struct space *s, double m[3][3])
{
        const double kg = 1. - s->kr - s->kb;
        m[0][0] = s->kr * s->yl, m[0][1] = kg * s->yl, m[0][2] = s->kb * s->yl;
        m[1][0] = -s->kr / (2. * (1. - s->kb)) * s->cl, m[1][1] = -kg / (2. * (1. - s->kb)) * s->cl, m[1][2] = .5 * s->cl;
        m[2][0] = .5 * s->cl, m[2][1] = -kg / (2. * (1. - s->kr)) * s->cl, m[2][2] = -s->kb / (2. * (1. - s->kr)) * s->cl;
}
/* rows R, G, B over columns Y - off, Cb - 128, Cr - 128 */
static void inverse(const struct space *s, double m[3][3])
{
        const double kg = 1. - s->kr - s->kb;
        m[0][0] = m[1][0] = m[2][0] = 1. / s->yl;
        m[0][1] = 0., m[0][2] = 2. * (1. - s->kr) / s->cl;
        m[1][1] = -s->kb * 2. * (1. - s->kb) / kg / s->cl, m[1][2] = -s->kr * 2. * (1. - s->kr) / kg / s->cl;
        m[2][1] = 2. * (1. - s->kb) / s->cl, m[2][2] = 0.;
}
static int q14(double x) { return (int) floor(fabs(x) * 16384. + .5) * (x < 0 ? -1 : 1); }

struct ycc {
        int yy, yb, yr, bb, br, rb, rr, o_in, o_out;
};
static struct ycc ycc_of(int cs_in, int cs_out)
{
        const struct space a = space_of(cs_in), b = space_of(cs_out);
        double f[3][3], inv[3][3], m[3][3];
        forward(&b, f), inverse(&a, inv);
        for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) {
                        m[i][j] = f[i][0] * inv[0][j] + f[i][1] * inv[1][j] + f[i][2] * inv[2][j];
                }
        }
        const struct ycc c = { q14(m[0][0]), q14(m[0][1]), q14(m[0][2]), q14(m[1][1]), q14(m[1][2]), q14(m[2][1]), q14(m[2][2]), a.off, b.off };
        return c;
}
static uint8_t clamp8(int v) { return (uint8_t) (v < 0 ? 0 : v > 255 ? 255 : v); }
static uint8_t conv_y(const struct ycc *c, int y, int cb, int cr)
{
        return clamp8(((c->yy * (y - c->o_in) + c->yb * (cb - 128) + c->yr * (cr - 128) + 8192) >> 14) + c->o_out);
}
static uint8_t conv_cb(const struct ycc *c, int cb, int cr) { return clamp8(((c->bb * (cb - 128) + c->br * (cr - 128) + 8192) >> 14) + 128); }
static uint8_t conv_cr(const struct ycc *c, int cb, int cr) { return clamp8(((c->rb * (cb - 128) + c->rr * (cr - 128) + 8192) >> 14) + 128); }

/* yy, yb, yr, bb, br, rb, rr, o_in, o_out; also the Y <- Cb / Cr column that must vanish, as out[9], out[10] (unrounded, times 2^14) */
API void orc_ycc_coeffs(int cs_in, int cs_out, int *out, double *chroma_from_luma)
{
        const struct ycc c = ycc_of(cs_in, cs_out);
        out[0] = c.yy, out[1] = c.yb, out[2] = c.yr, out[3] = c.bb, out[4] = c.br, out[5] = c.rb, out[6] = c.rr, out[7] = c.o_in, out[8] = c.o_out;
        const struct space a = space_of(cs_in), b = space_of(cs_out);
        double f[3][3], inv[3][3];
        forward(&b, f), inverse(&a, inv);
        for (int i = 1; i < 3; ++i) {
                chroma_from_luma[i - 1] = (f[i][0] * inv[0][0] + f[i][1] * inv[1][0] + f[i][2] * inv[2][0]) * 16384.;
        }
}

/* n (Y, Cb, Cr) triples -> n triples of the other space */
API void orc_ycc_convert(int cs_in, int cs_out, const uint8_t *in, uint8_t *out, long n)
{
        const struct ycc c = ycc_of(cs_in, cs_out);
        for (long i = 0; i < n; ++i) {
                const int y = in[3 * i], cb = in[3 * i + 1], cr = in[3 * i + 2];
                out[3 * i] = conv_y(&c, y, cb, cr), out[3 * i + 1] = conv_cb(&c, cb, cr), out[3 * i + 2] = conv_cr(&c, cb, cr);
        }
}

/* decode `s` and convert its samples from cs_in to cs_out (either 0: no conversion).  4:2:2, 4:2:0 and grayscale streams give UYVY rows of
 * ((w + 1) / 2) * 4 bytes (grayscale: Cb = Cr = 128; the last pair of an odd width takes the padded plane's luma), 4:4:4 streams rows of w
 * (Y, Cb, Cr) triples.  `out` holds h rows of `pitch` bytes.  Returns the decode's code. */
API int orc_jpeg_decode_yuv(const uint8_t *s, size_t len, int cs_in, int cs_out, uint8_t *out, long pitch)
{
        const int conv = cs_in != 0 && cs_out != 0 && cs_in != cs_out;
        const struct ycc c = conv ? ycc_of(cs_in, cs_out) : ycc_of(1, 1);
        size_t sof = 0;
        for (size_t p = 2; p + 4 <= len && s[p] == 0xFF;) {
                if (s[p + 1] == 0xC0) {
                        sof = p;
                        break;
                }
                p += 2 + (size_t) be16(s + p + 2);
        }
        if (!sof || sof + 12 > len) {
                return -3;
        }
        const int h = be16(s + sof + 5), w = be16(s + sof + 7), ncomp = s[sof + 9], hs = s[sof + 11] >> 4;
        if (ncomp == 1) {  /* the luma plane at an even width: the column past an odd width is the padded plane's, which the block grid still covers */
                const int we = (w + 1) / 2 * 2;
                uint8_t *copy = malloc(len), *tmp = malloc((size_t) we * 3 * h);
                if (!copy || !tmp) {
                        free(copy), free(tmp);
                        return -2;
                }
                memcpy(copy, s, len);
                copy[sof + 7] = (uint8_t) (we >> 8), copy[sof + 8] = (uint8_t) we;
                const int rc = orc_jpeg_decode(copy, len, 1, tmp, (long) we * 3, NULL);
                for (int y = 0; rc == 0 && y < h; ++y) {
                        for (int x = 0; x < we; ++x) {
                                const int v = tmp[((size_t) y * we + x) * 3];
                                out[(size_t) y * pitch + 2 * x] = 128;
                                out[(size_t) y * pitch + 2 * x + 1] = conv ? conv_y(&c, v, 128, 128) : (uint8_t) v;
                        }
                }
                free(copy), free(tmp);
                return rc;
        }
        const int rc = orc_jpeg_decode(s, len, hs == 2 ? 0 : 1, out, pitch, NULL);
        if (rc != 0 || !conv) {
                return rc;
        }
        for (int y = 0; y < h; ++y) {
                uint8_t *o = out + (size_t) y * pitch;
                if (hs == 2) {
                        for (int p = 0; p < (w + 1) / 2; ++p, o += 4) {
                                const int cb = o[0], y0 = o[1], cr = o[2], y1 = o[3];
                                o[0] = conv_cb(&c, cb, cr), o[1] = conv_y(&c, y0, cb, cr), o[2] = conv_cr(&c, cb, cr), o[3] = conv_y(&c, y1, cb, cr);
                        }
                } else {
                        orc_ycc_convert(cs_in, cs_out, o, o, w);
                }
        }
        return rc;
}
