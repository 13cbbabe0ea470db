/* TEST INFRASTRUCTURE — CPU restatement of the planar JPEG layouts of ugb200_jpeg_encode_device_ex (include/ugb200_jpeg.h):
 *   orc_jpeg_prep           packed input -> three 8-bit planes (the arithmetic of jpeg_prep_kernel)
 *   orc_jpeg_encode_planar  three planes -> YCbCr stream with luma sampling hs x vs (1x1, 2x1, 2x2), chroma 1x1
 * The two compose: the GPU stream of every planar layout equals orc_jpeg_encode_planar(orc_jpeg_prep(src)).
 * The DCT, the quantiser, the entropy coder and the header writer are those of oracle/jpeg_oracle.c, included here so that they stay
 * single-sourced.  tests/test_jpeg_planar.py compiles this file on its own. */
#include "../oracle/jpeg_oracle.c"

enum { C_UYVY = 2, C_RGB = 12, C_I420 = 29 };            /* codec_t */
enum { CS_NATIVE = 0, CS_Y601, CS_Y601FULL, CS_Y709 };  /* UGB200_JPEG_CS_* */

/* Q14 RGB -> YCbCr rows of compute_color_coeffs (ultragrid_b200/csrc/color_space.h, color_space.c:116-128); depth 0 = full range */
API void orc_jpeg_prep_coeffs(int color_space, int c[9])
{
        const double kr = color_space == CS_Y709 ? .212639 : .299, kb = color_space == CS_Y709 ? .072192 : .114, kg = 1. - kr - kb;
        const int depth = color_space == CS_Y601FULL ? 0 : 8;
        const double yl = depth ? 219. / 255. : 1., cl = depth ? 224. / 255. : 1., B = 1 << 14, d = 2. * (kr + kg), e = 2. * (1. - kr);
        c[0] = (int) (kr * yl * B + .5), c[1] = (int) (kg * yl * B + .5), c[2] = (int) (kb * yl * B + .5);
        c[3] = (int) (-kr / d * cl * B - .5), c[4] = (int) (-kg / d * cl * B - .5), c[5] = (int) ((1 - kb) / d * cl * B + .5);
        c[6] = (int) ((1 - kr) / e * cl * B - .5), c[7] = (int) (-kg / e * cl * B - .5), c[8] = (int) (-kb / e * cl * B + .5);
}

static int floor_shift14(int v) { return v >= 0 ? v >> 14 : -((-v + (1 << 14) - 1) >> 14); } /* floor(v / 2^14), written out */

/* planes p[0] (w x h), p[1], p[2] (ceil(w / hs) x ceil(h / vs)) with row pitches ls[]; subsampling 0 = native for the codec.
 * @returns 0, or -4 for a combination the encoder refuses */
API int orc_jpeg_prep(const uint8_t *src, long pitch, int w, int h, int codec, int subsampling, int color_space, uint8_t *const p[3], const int ls[3])
{
        const int cw = (w + 1) / 2, ch = (h + 1) / 2;
        if (codec == C_I420) { /* vc_get_datalen layout, copied */
                if (subsampling != 0 && subsampling != 420) {
                        return -4;
                }
                const uint8_t *cb = src + (size_t) w * h, *cr = cb + (size_t) cw * ch;
                for (int y = 0; y < h; ++y) {
                        memcpy(p[0] + (size_t) y * ls[0], src + (size_t) y * w, w);
                }
                for (int y = 0; y < ch; ++y) {
                        memcpy(p[1] + (size_t) y * ls[1], cb + (size_t) y * cw, cw);
                        memcpy(p[2] + (size_t) y * ls[2], cr + (size_t) y * cw, cw);
                }
                return 0;
        }
        if (codec == C_UYVY) { /* uyvy_to_i420, to_planar.c:343-378: (a + b + 1) / 2 of two rows, the last row paired with itself */
                if (subsampling != 420) {
                        return -4;
                }
                for (int y = 0; y < h; y += 2) {
                        const int y2 = y + 1 < h ? y + 1 : y;
                        const uint8_t *a = src + y * pitch, *b = src + y2 * pitch;
                        for (int x = 0; x < w; x += 2) {
                                p[1][(size_t) (y / 2) * ls[1] + x / 2] = (uint8_t) ((a[2 * x] + b[2 * x] + 1) / 2);
                                p[2][(size_t) (y / 2) * ls[2] + x / 2] = (uint8_t) ((a[2 * x + 2] + b[2 * x + 2] + 1) / 2);
                                for (int k = 0; k < 2 && x + k < w; ++k) {
                                        p[0][(size_t) y * ls[0] + x + k] = a[2 * x + 1 + 2 * k];
                                        p[0][(size_t) y2 * ls[0] + x + k] = b[2 * x + 1 + 2 * k];
                                }
                        }
                }
                return 0;
        }
        if (codec != C_RGB || color_space < CS_Y601 || color_space > CS_Y709) {
                return -4;
        }
        /* RGB_TO_Y/CB/CR at 8 bits (rgb_to_yuv444p, to_lavc_vid_conv.c:1206-1214); chroma mean of the pair / quad, rounded half up;
         * a missing last column / row takes its neighbour's value */
        const int hs = subsampling == 422 || subsampling == 420 ? 2 : 1, vs = subsampling == 420 ? 2 : 1, off_y = color_space == CS_Y601FULL ? 0 : 16;
        int c[9];
        orc_jpeg_prep_coeffs(color_space, c);
        const int pcw = (w + hs - 1) / hs, pch = (h + vs - 1) / vs;
        for (int cy = 0; cy < pch; ++cy) {
                for (int cx = 0; cx < pcw; ++cx) {
                        int sb = 0, sr = 0;
                        for (int j = 0; j < vs; ++j) {
                                for (int k = 0; k < hs; ++k) {
                                        const int x = cx * hs + k, y = cy * vs + j;
                                        const uint8_t *px = src + (long) (y < h ? y : h - 1) * pitch + 3 * (x < w ? x : w - 1);
                                        if (x < w && y < h) {
                                                p[0][(size_t) y * ls[0] + x] = (uint8_t) (floor_shift14(c[0] * px[0] + c[1] * px[1] + c[2] * px[2]) + off_y);
                                        }
                                        sb += floor_shift14(c[3] * px[0] + c[4] * px[1] + c[5] * px[2]) + 128;
                                        sr += floor_shift14(c[6] * px[0] + c[7] * px[1] + c[8] * px[2]) + 128;
                                }
                        }
                        const int n = hs * vs;
                        p[1][(size_t) cy * ls[1] + cx] = (uint8_t) ((sb + n / 2) / n);
                        p[2][(size_t) cy * ls[2] + cx] = (uint8_t) ((sr + n / 2) / n);
                }
        }
        return 0;
}

/* one 8x8 block of a plane of pw x ph valid samples at block coordinates (bx, by); edges replicate the plane's last column / row */
static void gather_plane(const uint8_t *plane, int pitch, int pw, int ph, int bx, int by, uint8_t px[64])
{
        for (int y = 0; y < 8; ++y) {
                for (int x = 0; x < 8; ++x) {
                        px[8 * y + x] = plane[(long) clampi(by * 8 + y, ph - 1) * pitch + clampi(bx * 8 + x, pw - 1)];
                }
        }
}

/* @returns the stream length (0 on error).  interleaved: one scan, MCU = hs x vs luma blocks in raster order, Cb, Cr (T.81 A.2.3);
 * otherwise one scan per component over its own block grid, not padded to whole MCUs (T.81 A.2.2).  ri > 0 MCUs per restart segment. */
API size_t orc_jpeg_encode_planar(const uint8_t *const p[3], const int ls[3], int w, int h, int hs, int vs, int quality, int ri, int interleaved, uint8_t *out,
                                  size_t cap)
{
        const int pw[3] = { w, (w + hs - 1) / hs, (w + hs - 1) / hs }, ph[3] = { h, (h + vs - 1) / vs, (h + vs - 1) / vs };
        const int mw = (w + 8 * hs - 1) / (8 * hs), mh = (h + 8 * vs - 1) / (8 * vs);
        const size_t nblk = (size_t) mw * mh * (hs * vs + 2);
        if (w <= 0 || h <= 0 || ri <= 0 || cap < 2048 + nblk * 418) {
                return 0;
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

        uint8_t *q = write_headers(out, w, h, FMT_UYVY_422, ql, qc, ri); /* JFIF; SOF0 component 0 sampling set below */
        for (uint8_t *s = out; s + 11 < q; ++s) {
                if (s[0] == 0xFF && s[1] == 0xC0) { /* FF C0 Lf(2) P Y(2) X(2) Nf C1 H1V1 */
                        s[11] = (uint8_t) (hs << 4 | vs);
                        break;
                }
        }
        uint8_t px[64];
        int16_t zz[64];
        if (interleaved) {
                q = write_sos(q, 0, 3);
                struct bitw bw = { q, 0, 0 };
                int pred[3] = { 0, 0, 0 };
                for (int m = 0; m < mw * mh; ++m) {
                        if (m > 0 && m % ri == 0) {
                                flush_bits(&bw);
                                *bw.p++ = 0xFF, *bw.p++ = (uint8_t) (0xD0 + ((m / ri - 1) & 7));
                                pred[0] = pred[1] = pred[2] = 0;
                        }
                        const int mx = m % mw, my = m / mw;
                        for (int k = 0; k < hs * vs + 2; ++k) {
                                const int comp = k < hs * vs ? 0 : k - hs * vs + 1;
                                const int bx = comp ? mx : mx * hs + k % hs, by = comp ? my : my * vs + k / hs;
                                gather_plane(p[comp], ls[comp], pw[comp], ph[comp], bx, by, px);
                                block_to_coeffs(px, comp == 0 ? ml : mc, zz);
                                encode_block(&bw, zz, &pred[comp], comp == 0 ? &dcl : &dcc, comp == 0 ? &acl : &acc);
                        }
                }
                flush_bits(&bw);
                q = bw.p;
        } else {
                for (int comp = 0; comp < 3; ++comp) {
                        q = write_sos(q, comp, 1);
                        const int bwid = (pw[comp] + 7) / 8, nb = bwid * ((ph[comp] + 7) / 8);
                        struct bitw bw = { q, 0, 0 };
                        int pred = 0;
                        for (int b = 0; b < nb; ++b) {
                                if (b > 0 && b % ri == 0) {
                                        flush_bits(&bw);
                                        *bw.p++ = 0xFF, *bw.p++ = (uint8_t) (0xD0 + ((b / ri - 1) & 7));
                                        pred = 0;
                                }
                                gather_plane(p[comp], ls[comp], pw[comp], ph[comp], b % bwid, b / bwid, px);
                                block_to_coeffs(px, comp == 0 ? ml : mc, zz);
                                encode_block(&bw, zz, &pred, comp == 0 ? &dcl : &dcc, comp == 0 ? &acl : &acc);
                        }
                        flush_bits(&bw);
                        q = bw.p;
                }
        }
        *q++ = 0xFF, *q++ = 0xD9;
        return (size_t) (q - out);
}
