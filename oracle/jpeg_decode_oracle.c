/* TEST INFRASTRUCTURE - not part of the product.
 * CPU restatement of the baseline-JPEG DECODE stage (SURVEY.md section 8f rank 1: what libgpujpeg does for UltraGrid's
 * src/video_decompress/gpujpeg.c:74-145,268 and gpujpeg_to_dxt.cpp:117-166).  PARITY UNPINNED against GPUJPEG (absent, see
 * jpeg_oracle.c); pinned instead against an independent decoder (libjpeg via PIL: every sample within 1 of its output, most
 * equal - libjpeg's default IDCT is the integer "islow", this one is the float AAN inverse with a fixed operation order so that
 * the CUDA decoder reproduces the bytes exactly) and by the encode -> decode round trip of the reference's own test
 * (test/gpujpeg_test.cpp:68-106: flat grey, max |diff| <= 1).
 *
 * Scope (ITU-T T.81 baseline sequential DCT, Huffman, 8 bit): 1 or 3 components, luma sampling 1x1, 2x1 or 2x2 with 1x1 chroma,
 * interleaved or one-scan-per-component, restart intervals, byte stuffing, tables from the stream (DQT 8-bit, DHT).  Output
 * is the stream's own colour space, like the reference's default configuration stores it (gpujpeg.cpp:304-305): no transform.
 *   out_fmt 0: UYVY  (3 components, 2x1 or 2x2 luma)         out_fmt 1: packed 3 bytes/pixel, component order of the frame
 *   header: SOF0 only (as src/utils/jpeg_reader.c:860-1003 accepts), APPn/COM skipped. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

static const uint8_t zigzag[64] = { 0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

struct dhuff {  /* T.81 F.2.2.3 decoding tables */
        int mincode[17], maxcode[18], valptr[17];
        uint8_t vals[256];
        int present;
};
static void build_dhuff(struct dhuff *h, const uint8_t bits[16], const uint8_t *vals, int nvals)
{
        int code = 0, k = 0;
        memcpy(h->vals, vals, nvals);
        for (int l = 1; l <= 16; ++l) {
                h->valptr[l] = k;
                h->mincode[l] = code;
                code += bits[l - 1];
                k += bits[l - 1];
                h->maxcode[l] = bits[l - 1] ? code - 1 : -1;
                code <<= 1;
        }
        h->maxcode[17] = 0x7fffffff;
        h->present = 1;
}

struct bitr {
        const uint8_t *p, *end;
        uint32_t acc;
        int nbits;
};
static int get_bit(struct bitr *r)
{
        if (r->nbits == 0) {
                uint8_t b = 0;
                if (r->p < r->end) {
                        b = *r->p++;
                        if (b == 0xFF && r->p < r->end && *r->p == 0) {
                                ++r->p; /* stuffed zero */
                        }
                }
                r->acc = b, r->nbits = 8;
        }
        return (r->acc >> --r->nbits) & 1;
}
static int get_bits(struct bitr *r, int n)
{
        int v = 0;
        while (n--) {
                v = (v << 1) | get_bit(r);
        }
        return v;
}
static int decode_sym(struct bitr *r, const struct dhuff *h)
{
        int code = 0;
        for (int l = 1; l <= 16; ++l) {
                code = (code << 1) | get_bit(r);
                if (h->maxcode[l] >= 0 && code <= h->maxcode[l] && code >= h->mincode[l]) {
                        return h->vals[h->valptr[l] + code - h->mincode[l]];
                }
        }
        return 0;
}
static int extend(int v, int t) { return t == 0 ? 0 : v < (1 << (t - 1)) ? v - (1 << t) + 1 : v; } /* F.2.2.1 */

/* 8-point AAN inverse DCT, explicit operation order (mirror of the encoder's fdct8: the dequantisation multipliers carry the
 * AAN scale factors, idct_multipliers) */
static void idct8(float *d, int stride)
{
        const float t0 = d[0 * stride], t1 = d[2 * stride], t2 = d[4 * stride], t3 = d[6 * stride];
        const float e0 = t0 + t2, e1 = t0 - t2;
        const float e3 = t1 + t3, e2 = (t1 - t3) * 1.414213562f - e3;
        const float a0 = e0 + e3, a3 = e0 - e3, a1 = e1 + e2, a2 = e1 - e2;
        const float o4 = d[1 * stride], o5 = d[3 * stride], o6 = d[5 * stride], o7 = d[7 * stride];
        const float z13 = o6 + o5, z10 = o6 - o5, z11 = o4 + o7, z12 = o4 - o7;
        const float b7 = z11 + z13;
        const float b11 = (z11 - z13) * 1.414213562f;
        const float z5 = (z10 + z12) * 1.847759065f;
        const float b10 = fmaf(1.082392200f, z12, -z5);
        const float b12 = fmaf(-2.613125930f, z10, z5);
        const float b6 = b12 - b7, b5 = b11 - b6, b4 = b10 + b5;
        d[0 * stride] = a0 + b7, d[7 * stride] = a0 - b7;
        d[1 * stride] = a1 + b6, d[6 * stride] = a1 - b6;
        d[2 * stride] = a2 + b5, d[5 * stride] = a2 - b5;
        d[4 * stride] = a3 + b4, d[3 * stride] = a3 - b4;
}
/* dequantisation multiplier of natural index n: q[n] * aan[row] * aan[col] / 8 (float products in this order) */
static const float aan_scale[8] = { 1.0f, 1.387039845f, 1.306562965f, 1.175875602f, 1.0f, 0.785694958f, 0.541196100f, 0.275899379f };
API void orc_jpeg_idct_multipliers(const uint8_t q_natural[64], float m[64])
{
        for (int n = 0; n < 64; ++n) {
                m[n] = ((float) q_natural[n] * aan_scale[n >> 3]) * aan_scale[n & 7] * 0.125f;
        }
}
static void coeffs_to_block(const int16_t nat[64], const float m[64], uint8_t px[64])
{
        float f[64];
        for (int i = 0; i < 64; ++i) {
                f[i] = (float) nat[i] * m[i];
        }
        for (int c = 0; c < 8; ++c) {
                idct8(f + c, 8);
        }
        for (int r = 0; r < 8; ++r) {
                idct8(f + 8 * r, 1);
        }
        for (int i = 0; i < 64; ++i) {
                const float v = rintf(f[i] + 128.0f);
                px[i] = v < 0.0f ? 0 : v > 255.0f ? 255 : (uint8_t) v;
        }
}

struct comp {
        int id, h, v, tq, td, ta;
        int bw, bh;      /* blocks per row / rows in the padded component */
        uint8_t *plane;  /* bw*8 x bh*8 samples */
};
struct frame {
        int w, h, ncomp, hmax, vmax, ri;
        struct comp c[3];
        uint8_t q[4][64]; /* natural order */
        float m[4][64];
        struct dhuff dc[4], ac[4];
        int adobe_transform; /* -1 = no Adobe marker */
};

static int be16(const uint8_t *p) { return p[0] << 8 | p[1]; }

/* decodes one scan's entropy-coded data starting at *pp; returns 0 on success and leaves *pp at the next marker */
static int decode_scan(struct frame *f, const int *scomp, int ns, const uint8_t **pp, const uint8_t *end)
{
        const uint8_t *p = *pp;
        int mcux, mcuy;
        if (ns == 1) {  /* non-interleaved: MCU = one block, only the blocks covering the component's real size (A.2.3) */
                const struct comp *c = &f->c[scomp[0]];
                const int cw = (f->w * c->h + f->hmax - 1) / f->hmax, ch = (f->h * c->v + f->vmax - 1) / f->vmax;
                mcux = (cw + 7) / 8, mcuy = (ch + 7) / 8;
        } else {
                mcux = (f->w + 8 * f->hmax - 1) / (8 * f->hmax), mcuy = (f->h + 8 * f->vmax - 1) / (8 * f->vmax);
        }
        const int nmcu = mcux * mcuy;
        int pred[3] = { 0, 0, 0 };
        struct bitr r = { p, end, 0, 0 };
        for (int m = 0; m < nmcu; ++m) {
                if (f->ri && m && m % f->ri == 0) {  /* expect RSTn: byte align, skip the marker, reset predictions (F.2.1.3.1, E.2.4) */
                        r.nbits = 0;
                        while (r.p + 1 < end && !(r.p[0] == 0xFF && r.p[1] >= 0xD0 && r.p[1] <= 0xD7)) {
                                ++r.p;
                        }
                        r.p += 2;
                        pred[0] = pred[1] = pred[2] = 0;
                }
                for (int s = 0; s < ns; ++s) {
                        struct comp *c = &f->c[scomp[s]];
                        const int nh = ns == 1 ? 1 : c->h, nv = ns == 1 ? 1 : c->v;
                        for (int by = 0; by < nv; ++by) {
                                for (int bx = 0; bx < nh; ++bx) {
                                        int16_t nat[64] = { 0 };
                                        const int t = decode_sym(&r, &f->dc[c->td]);
                                        pred[s] += extend(get_bits(&r, t), t);
                                        nat[0] = (int16_t) pred[s];
                                        for (int k = 1; k < 64;) {
                                                const int rs = decode_sym(&r, &f->ac[c->ta]), run = rs >> 4, sz = rs & 15;
                                                if (sz == 0) {
                                                        if (run != 15) {
                                                                break; /* EOB */
                                                        }
                                                        k += 16;
                                                        continue;
                                                }
                                                k += run;
                                                if (k > 63) {
                                                        return -2;
                                                }
                                                nat[zigzag[k]] = (int16_t) extend(get_bits(&r, sz), sz);
                                                ++k;
                                        }
                                        uint8_t px[64];
                                        coeffs_to_block(nat, f->m[c->tq], px);
                                        const int X = (ns == 1 ? m % mcux : (m % mcux) * c->h + bx), Y = (ns == 1 ? m / mcux : (m / mcux) * c->v + by);
                                        if (X < c->bw && Y < c->bh) {
                                                for (int y = 0; y < 8; ++y) {
                                                        memcpy(c->plane + (size_t) (Y * 8 + y) * c->bw * 8 + X * 8, px + 8 * y, 8);
                                                }
                                        }
                                }
                        }
                }
        }
        /* to the next marker */
        p = r.p;
        while (p + 1 < end && !(p[0] == 0xFF && p[1] != 0 && !(p[1] >= 0xD0 && p[1] <= 0xD7))) {
                ++p;
        }
        *pp = p;
        return 0;
}

/* @returns 0 ok; <0 error.  info[0..4] = width, height, components, luma h sampling, luma v sampling, info[5] = Adobe transform or -1 */
API int orc_jpeg_decode(const uint8_t *s, size_t len, int out_fmt, uint8_t *out, long pitch, int *info)
{
        struct frame f;
        memset(&f, 0, sizeof f);
        f.adobe_transform = -1;
        const uint8_t *p = s, *end = s + len;
        if (len < 4 || p[0] != 0xFF || p[1] != 0xD8) {
                return -1;
        }
        p += 2;
        int rc = 0, have_sof = 0, done = 0;
        while (!done && p + 4 <= end) {
                if (p[0] != 0xFF) {
                        rc = -3;
                        break;
                }
                const int mk = p[1];
                if (mk == 0xD9) {
                        break;
                }
                const int L = be16(p + 2);
                const uint8_t *d = p + 4, *dend = p + 2 + L;
                if (dend > end) {
                        rc = -3;
                        break;
                }
                if (mk == 0xDB) {  /* DQT, B.2.4.1 */
                        while (d < dend) {
                                const int pq = d[0] >> 4, tq = d[0] & 15;
                                if (pq != 0 || tq > 3) {
                                        rc = -4;
                                        break;
                                }
                                for (int k = 0; k < 64; ++k) {
                                        f.q[tq][zigzag[k]] = d[1 + k];
                                }
                                orc_jpeg_idct_multipliers(f.q[tq], f.m[tq]);
                                d += 65;
                        }
                } else if (mk == 0xC4) {  /* DHT, B.2.4.2 */
                        while (d < dend) {
                                const int tc = d[0] >> 4, th = d[0] & 15;
                                int n = 0;
                                for (int i = 0; i < 16; ++i) {
                                        n += d[1 + i];
                                }
                                if (th > 3 || n > 256) {
                                        rc = -4;
                                        break;
                                }
                                build_dhuff(tc ? &f.ac[th] : &f.dc[th], d + 1, d + 17, n);
                                d += 17 + n;
                        }
                } else if (mk == 0xC0) {  /* SOF0, B.2.2 */
                        if (d[0] != 8) {
                                rc = -4;
                                break;
                        }
                        f.h = be16(d + 1), f.w = be16(d + 3), f.ncomp = d[5];
                        if ((f.ncomp != 1 && f.ncomp != 3) || f.w == 0 || f.h == 0) {
                                rc = -4;
                                break;
                        }
                        for (int i = 0; i < f.ncomp; ++i) {
                                f.c[i].id = d[6 + 3 * i], f.c[i].h = d[7 + 3 * i] >> 4, f.c[i].v = d[7 + 3 * i] & 15, f.c[i].tq = d[8 + 3 * i];
                                if (f.c[i].h > f.hmax) {
                                        f.hmax = f.c[i].h;
                                }
                                if (f.c[i].v > f.vmax) {
                                        f.vmax = f.c[i].v;
                                }
                        }
                        for (int i = 0; i < f.ncomp; ++i) {
                                struct comp *c = &f.c[i];
                                if (c->h < 1 || c->h > 2 || c->v < 1 || c->v > 2 || (i > 0 && (c->h != 1 || c->v != 1)) || c->v > c->h) { /* no luma 1x2 */
                                        rc = -4;
                                        break;
                                }
                                c->bw = (f.w + 8 * f.hmax - 1) / (8 * f.hmax) * c->h, c->bh = (f.h + 8 * f.vmax - 1) / (8 * f.vmax) * c->v;
                                c->plane = calloc((size_t) c->bw * c->bh, 64);
                        }
                        have_sof = 1;
                } else if (mk >= 0xC1 && mk <= 0xCF && mk != 0xC4 && mk != 0xC8 && mk != 0xCC) {
                        rc = -4; /* not baseline */
                } else if (mk == 0xDD) {
                        f.ri = be16(d);
                } else if (mk == 0xEE && L >= 14 && memcmp(d, "Adobe", 5) == 0) {
                        f.adobe_transform = d[11];
                } else if (mk == 0xDA) {  /* SOS, B.2.3 */
                        if (!have_sof) {
                                rc = -3;
                                break;
                        }
                        const int ns = d[0];
                        int scomp[3];
                        if (ns < 1 || ns > f.ncomp) {
                                rc = -4;
                                break;
                        }
                        for (int i = 0; i < ns; ++i) {
                                scomp[i] = -1;
                                for (int j = 0; j < f.ncomp; ++j) {
                                        if (f.c[j].id == d[1 + 2 * i]) {
                                                scomp[i] = j;
                                                f.c[j].td = d[2 + 2 * i] >> 4, f.c[j].ta = d[2 + 2 * i] & 15;
                                        }
                                }
                                if (scomp[i] < 0) {
                                        rc = -4;
                                }
                        }
                        if (rc) {
                                break;
                        }
                        p = dend;
                        rc = decode_scan(&f, scomp, ns, &p, end);
                        if (rc) {
                                break;
                        }
                        continue;
                }
                if (rc) {
                        break;
                }
                p = dend;
        }
        if (rc == 0 && have_sof) {
                if (info) {
                        info[0] = f.w, info[1] = f.h, info[2] = f.ncomp, info[3] = f.c[0].h, info[4] = f.c[0].v, info[5] = f.adobe_transform;
                }
                if (out) {
                        if (out_fmt == 0) {
                                if (f.ncomp != 3 || f.c[0].h != 2) {
                                        rc = -5;
                                } else {
                                        for (int y = 0; y < f.h; ++y) {
                                                const int cy = y / f.c[0].v; /* 4:2:0: a chroma row serves two luma rows (nearest) */
                                                const uint8_t *Y = f.c[0].plane + (size_t) y * f.c[0].bw * 8, *B = f.c[1].plane + (size_t) cy * f.c[1].bw * 8,
                                                              *R = f.c[2].plane + (size_t) cy * f.c[2].bw * 8;
                                                uint8_t *o = out + (size_t) y * pitch;
                                                for (int x = 0; x < f.w; x += 2) {
                                                        o[2 * x] = B[x / 2], o[2 * x + 1] = Y[x], o[2 * x + 2] = R[x / 2];
                                                        o[2 * x + 3] = Y[x + 1]; /* the padded plane always holds it */
                                                }
                                        }
                                }
                        } else {
                                for (int y = 0; y < f.h; ++y) {
                                        uint8_t *o = out + (size_t) y * pitch;
                                        for (int x = 0; x < f.w; ++x) {
                                                for (int i = 0; i < 3; ++i) {
                                                        const struct comp *c = &f.c[f.ncomp == 1 ? 0 : i];
                                                        const int sx = x * c->h / f.hmax, sy = y * c->v / f.vmax; /* nearest (replicating) upsampling */
                                                        o[3 * x + i] = c->plane[(size_t) sy * c->bw * 8 + sx];
                                                }
                                        }
                                }
                        }
                }
        } else if (rc == 0) {
                rc = -3;
        }
        for (int i = 0; i < 3; ++i) {
                free(f.c[i].plane);
        }
        return rc;
}
