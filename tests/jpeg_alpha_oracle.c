/* TEST INFRASTRUCTURE — CPU restatement of the RGBA layout of ugb200_jpeg_encode_device_ex (include/ugb200_jpeg.h: UGB_RGBA with
 * subsampling 4444, the GPUJPEG module's `alpha` stream) and of the decoder's four-component path:
 *   orc_jpeg_encode_rgba   packed RGBA -> SOI, Adobe APP14 (transform 0), DQT, SOF0 with components 1..4 sampled 1x1 and tables 0 1 1 1,
 *                          DHT, DRI, then one scan per component (R G B A) or one interleaved scan of 4-block MCUs
 *   orc_jpeg_decode_rgba   a four-component baseline stream -> packed R G B A (samples as stored, no colour transform)
 * The DCT, the quantiser, the entropy coder, the Huffman decoder and the IDCT are those of oracle/jpeg_oracle.c and
 * oracle/jpeg_decode_oracle.c, included here so that they stay single-sourced.  tests/test_jpeg_alpha.py compiles this file on its own. */
#include "../oracle/jpeg_oracle.c"
#include "../oracle/jpeg_decode_oracle.c"

/* one 8x8 block of component `comp` of packed RGBA at block coordinates (bx, by); edges replicate the last column / row */
static void gather_rgba(const uint8_t *src, long pitch, int w, int h, int comp, int bx, int by, uint8_t px[64])
{
        for (int y = 0; y < 8; ++y) {
                const uint8_t *row = src + (long) clampi(by * 8 + y, h - 1) * pitch;
                for (int x = 0; x < 8; ++x) {
                        px[8 * y + x] = row[4 * clampi(bx * 8 + x, w - 1) + comp];
                }
        }
}

/* @returns the stream length (0 on error); ri <= 0: the default 8 */
API size_t orc_jpeg_encode_rgba(const uint8_t *src, long pitch, int w, int h, int quality, int ri, int interleaved, uint8_t *out, size_t cap)
{
        const size_t nblk = (size_t) ((w + 7) / 8) * ((h + 7) / 8) * 4;
        if (w <= 0 || h <= 0 || cap < 2048 + nblk * 418) {
                return 0;
        }
        if (ri <= 0) {
                ri = 8;
        }
        uint8_t ql[64], qc[64];
        float ml[64], mc[64];
        ugb_jpeg_scaled_qtable(ugb_jpeg_q_luma, quality, ql);
        ugb_jpeg_scaled_qtable(ugb_jpeg_q_chroma, quality, qc);
        ugb_jpeg_quant_multipliers(ql, ml);
        ugb_jpeg_quant_multipliers(qc, mc);
        struct huff dcl, acl, dcc, acc;
        ugb_jpeg_build_codes(ugb_jpeg_dc_luma_bits, ugb_jpeg_dc_vals, 12, dcl.code, dcl.len);
        ugb_jpeg_build_codes(ugb_jpeg_ac_luma_bits, ugb_jpeg_ac_luma_vals, 162, acl.code, acl.len);
        ugb_jpeg_build_codes(ugb_jpeg_dc_chroma_bits, ugb_jpeg_dc_vals, 12, dcc.code, dcc.len);
        ugb_jpeg_build_codes(ugb_jpeg_ac_chroma_bits, ugb_jpeg_ac_chroma_vals, 162, acc.code, acc.len);

        /* the RGB headers with a fourth component in SOF0: FF C0 Lf(2) P Y(2) X(2) Nf, then 3 bytes per component */
        uint8_t hdr[2048];
        const uint8_t *he = write_headers(hdr, w, h, FMT_RGB_444, ql, qc, ri);
        const uint8_t *sof = hdr;
        while (!(sof[0] == 0xFF && sof[1] == 0xC0)) {
                ++sof;
        }
        uint8_t *p = out;
        memcpy(p, hdr, (size_t) (sof - hdr)), p += sof - hdr;
        *p++ = 0xFF, *p++ = 0xC0;
        p = put16(p, 8 + 3 * 4);
        memcpy(p, sof + 4, 5), p += 5; /* P, Y, X */
        *p++ = 4;
        for (int c = 0; c < 4; ++c) {
                *p++ = (uint8_t) (c + 1), *p++ = 0x11, *p++ = c == 0 ? 0 : 1;
        }
        const uint8_t *rest = sof + 2 + 17;
        memcpy(p, rest, (size_t) (he - rest)), p += he - rest;

        const int bwid = (w + 7) / 8, nm = bwid * ((h + 7) / 8);
        uint8_t px[64];
        int16_t zz[64];
        if (interleaved) { /* one scan; MCU = the R, G, B and A block of an 8x8 area */
                p = write_sos(p, 0, 4);
                struct bitw bw = { p, 0, 0 };
                int pred[4] = { 0, 0, 0, 0 };
                for (int m = 0; m < nm; ++m) {
                        if (m > 0 && m % ri == 0) {
                                flush_bits(&bw);
                                *bw.p++ = 0xFF, *bw.p++ = (uint8_t) (0xD0 + ((m / ri - 1) & 7));
                                pred[0] = pred[1] = pred[2] = pred[3] = 0;
                        }
                        for (int comp = 0; comp < 4; ++comp) {
                                gather_rgba(src, pitch, w, h, comp, m % bwid, m / bwid, px);
                                block_to_coeffs(px, comp == 0 ? ml : mc, zz);
                                encode_block(&bw, zz, &pred[comp], comp == 0 ? &dcl : &dcc, comp == 0 ? &acl : &acc);
                        }
                }
                flush_bits(&bw);
                p = bw.p;
        } else { /* four scans, one component each; MCU = one 8x8 block */
                for (int comp = 0; comp < 4; ++comp) {
                        p = write_sos(p, comp, 1);
                        struct bitw bw = { p, 0, 0 };
                        int pred = 0;
                        for (int b = 0; b < nm; ++b) {
                                if (b > 0 && b % ri == 0) {
                                        flush_bits(&bw);
                                        *bw.p++ = 0xFF, *bw.p++ = (uint8_t) (0xD0 + ((b / ri - 1) & 7));
                                        pred = 0;
                                }
                                gather_rgba(src, pitch, w, h, comp, b % bwid, b / bwid, px);
                                block_to_coeffs(px, comp == 0 ? ml : mc, zz);
                                encode_block(&bw, zz, &pred, comp == 0 ? &dcl : &dcc, comp == 0 ? &acl : &acc);
                        }
                        flush_bits(&bw);
                        p = bw.p;
                }
        }
        *p++ = 0xFF, *p++ = 0xD9;
        return (size_t) (p - out);
}

/* @returns 0, -1 not a JPEG, -3 malformed, -4 not a baseline stream of four components sampled 1x1 with Adobe transform 0 or no Adobe
 * marker.  out: packed R G B A (components 1..4 in SOF order) with `pitch` bytes per row; info[0..1] = width, height (either may be NULL) */
API int orc_jpeg_decode_rgba(const uint8_t *s, size_t len, uint8_t *out, long pitch, int *info)
{
        struct frame f; /* tables and geometry; the four component planes live here */
        memset(&f, 0, sizeof f);
        int ids[4] = { 0 }, tq[4] = { 0 }, ncomp = 0, adobe = -1, rc = 0, have_sof = 0;
        uint8_t *plane[4] = { NULL, NULL, NULL, NULL };
        int bwid = 0, bh = 0;
        const uint8_t *p = s, *end = s + len;
        if (len < 4 || p[0] != 0xFF || p[1] != 0xD8) {
                return -1;
        }
        p += 2;
        while (rc == 0 && p + 4 <= end) {
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
                if (mk == 0xDB) {
                        for (; d + 65 <= dend; d += 65) {
                                const int t = d[0] & 15;
                                if (d[0] >> 4 || t > 3) {
                                        rc = -4;
                                        break;
                                }
                                for (int k = 0; k < 64; ++k) {
                                        f.q[t][zigzag[k]] = d[1 + k];
                                }
                                orc_jpeg_idct_multipliers(f.q[t], f.m[t]);
                        }
                } else if (mk == 0xC4) {
                        while (d + 17 <= dend) {
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
                } else if (mk == 0xC0) {
                        f.h = be16(d + 1), f.w = be16(d + 3), ncomp = d[5];
                        if (d[0] != 8 || ncomp != 4 || f.w == 0 || f.h == 0) {
                                rc = -4;
                                break;
                        }
                        for (int i = 0; i < 4; ++i) {
                                ids[i] = d[6 + 3 * i], tq[i] = d[8 + 3 * i] & 3;
                                if (d[7 + 3 * i] != 0x11) {
                                        rc = -4;
                                }
                        }
                        bwid = (f.w + 7) / 8, bh = (f.h + 7) / 8;
                        for (int i = 0; i < 4 && rc == 0; ++i) {
                                plane[i] = calloc((size_t) bwid * bh, 64);
                        }
                        have_sof = 1;
                } else if (mk >= 0xC1 && mk <= 0xCF && mk != 0xC4 && mk != 0xC8 && mk != 0xCC) {
                        rc = -4;
                } else if (mk == 0xDD) {
                        f.ri = be16(d);
                } else if (mk == 0xEE && L >= 14 && memcmp(d, "Adobe", 5) == 0) {
                        adobe = d[11];
                } else if (mk == 0xDA) {
                        if (!have_sof) {
                                rc = -3;
                                break;
                        }
                        if (adobe > 0) {
                                rc = -4; /* YCCK */
                                break;
                        }
                        const int ns = d[0];
                        int sc[4], td[4], ta[4];
                        if (ns < 1 || ns > 4) {
                                rc = -4;
                                break;
                        }
                        for (int i = 0; i < ns; ++i) {
                                sc[i] = -1;
                                for (int j = 0; j < 4; ++j) {
                                        if (ids[j] == d[1 + 2 * i]) {
                                                sc[i] = j;
                                        }
                                }
                                td[i] = d[2 + 2 * i] >> 4, ta[i] = d[2 + 2 * i] & 15;
                                if (sc[i] < 0) {
                                        rc = -4;
                                }
                        }
                        if (rc) {
                                break;
                        }
                        /* every component is 1x1: MCU = one block of each scan component, the same block grid for both layouts */
                        const int nmcu = bwid * bh;
                        int pred[4] = { 0, 0, 0, 0 };
                        struct bitr r = { dend, end, 0, 0 };
                        for (int m = 0; m < nmcu; ++m) {
                                if (f.ri && m && m % f.ri == 0) {
                                        r.nbits = 0;
                                        while (r.p + 1 < end && !(r.p[0] == 0xFF && r.p[1] >= 0xD0 && r.p[1] <= 0xD7)) {
                                                ++r.p;
                                        }
                                        r.p += 2;
                                        pred[0] = pred[1] = pred[2] = pred[3] = 0;
                                }
                                for (int k = 0; k < ns; ++k) {
                                        int16_t nat[64] = { 0 };
                                        const int t = decode_sym(&r, &f.dc[td[k]]);
                                        pred[k] += extend(get_bits(&r, t), t);
                                        nat[0] = (int16_t) pred[k];
                                        for (int i = 1; i < 64;) {
                                                const int rs = decode_sym(&r, &f.ac[ta[k]]), run = rs >> 4, sz = rs & 15;
                                                if (sz == 0) {
                                                        if (run != 15) {
                                                                break;
                                                        }
                                                        i += 16;
                                                        continue;
                                                }
                                                i += run;
                                                if (i > 63) {
                                                        rc = -3;
                                                        break;
                                                }
                                                nat[zigzag[i]] = (int16_t) extend(get_bits(&r, sz), sz);
                                                ++i;
                                        }
                                        uint8_t px[64];
                                        coeffs_to_block(nat, f.m[tq[sc[k]]], px);
                                        const int X = m % bwid, Y = m / bwid;
                                        for (int y = 0; y < 8; ++y) {
                                                memcpy(plane[sc[k]] + (size_t) (Y * 8 + y) * bwid * 8 + X * 8, px + 8 * y, 8);
                                        }
                                }
                        }
                        p = r.p;
                        while (p + 1 < end && !(p[0] == 0xFF && p[1] != 0 && !(p[1] >= 0xD0 && p[1] <= 0xD7))) {
                                ++p;
                        }
                        continue;
                }
                p = dend;
        }
        if (rc == 0 && !have_sof) {
                rc = -3;
        }
        if (rc == 0) {
                if (info) {
                        info[0] = f.w, info[1] = f.h;
                }
                if (out) {
                        for (int y = 0; y < f.h; ++y) {
                                for (int x = 0; x < f.w; ++x) {
                                        for (int c = 0; c < 4; ++c) {
                                                out[(size_t) y * pitch + 4 * x + c] = plane[c][(size_t) y * bwid * 8 + x];
                                        }
                                }
                        }
                }
        }
        for (int i = 0; i < 4; ++i) {
                free(plane[i]);
        }
        return rc;
}
