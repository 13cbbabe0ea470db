// Packed -> planar whole-buffer converters: device form of UltraGrid's src/to_planar.c.
//
//   v210_to_p010le (to_planar.c:64-155): 10-bit 4:2:2 packed -> P010 (Y plane + interleaved CbCr plane,
//   4:2:0, samples in the 10 MSBs of a 16-bit word).  Y: sample << 6.  CbCr: ((row0 + row1) / 2) << 6.
//
// HBM-bound: 16/6 B/px in, 3 B/px out.  A thread owns 4 v210 groups (24 px) of a row PAIR: 2 x 4 LDG.128,
// 3 + 3 + 3 STG.128.  Edge rules of the reference are kept (odd height: last row pairs with itself; width%6:
// middle rows write whole groups past `width`, the last 1-2 rows stop at full groups and copy the tail from
// two rows above, to_planar.c:83-92,141-151 — note the reference's pointer arithmetic there is in uint16
// elements, i.e. out_linesize *elements* = two rows up).
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include "../../include/ugb200.h"

namespace ugb {

__device__ __forceinline__ uint32_t s10(uint32_t w, int sh) { return (w >> sh) & 0x3ffu; }
__device__ __forceinline__ uint32_t y2(uint32_t a, uint32_t b) { return (a << 6) | (b << 22); }
__device__ __forceinline__ uint32_t c2(uint32_t a0, uint32_t a1, uint32_t b0, uint32_t b1)
{
        return (((a0 + a1) / 2) << 6) | (((b0 + b1) / 2) << 22);
}

template <int G, bool SPILL>  // groups per thread; SPILL: a pair before the last writes whole groups past a row's end (see below)
__global__ void __launch_bounds__(128) v210_to_p010_kernel(const uint8_t *__restrict__ in, long in_pitch, uint8_t *__restrict__ out_y,
                                                           long ls_y, uint8_t *__restrict__ out_c, long ls_c, int height,
                                                           int groups_mid, int groups_last, bool vec_ok)
{
        const int cx = blockIdx.x * blockDim.x + threadIdx.x;
        const int g0 = cx * G;
        for (int pr = blockIdx.y; pr < (height + 1) / 2; pr += gridDim.y) {
                const int y = pr * 2;
                const bool single = height - y == 1;                 // to_planar.c:84-87
                const bool last = single || height - y == 2;         // :90-92
                const int groups = last ? groups_last : groups_mid;
                if (g0 >= groups) {
                        continue;
                }
                const uint8_t *s0 = in + (long) y * in_pitch + (long) g0 * 16;
                const uint8_t *s1 = single ? s0 : s0 + in_pitch;
                uint32_t a[4 * G], b[4 * G];
                const bool full = g0 + G <= groups;
                if (full && vec_ok) {
#pragma unroll
                        for (int i = 0; i < G; ++i) {
                                const uint4 va = __ldg((const uint4 *) s0 + i), vb = __ldg((const uint4 *) s1 + i);
                                a[4 * i] = va.x, a[4 * i + 1] = va.y, a[4 * i + 2] = va.z, a[4 * i + 3] = va.w;
                                b[4 * i] = vb.x, b[4 * i + 1] = vb.y, b[4 * i + 2] = vb.z, b[4 * i + 3] = vb.w;
                        }
                } else {
#pragma unroll
                        for (int i = 0; i < 4 * G; ++i) {
                                const bool ok = g0 + i / 4 < groups;
                                a[i] = ok ? ((const uint32_t *) s0)[i] : 0;
                                b[i] = ok ? ((const uint32_t *) s1)[i] : 0;
                        }
                }
                uint32_t oy0[3 * G], oy1[3 * G], oc[3 * G];
#pragma unroll
                for (int i = 0; i < G; ++i) {
                        const uint32_t *w = a + 4 * i, *v = b + 4 * i;
                        // sample positions: to_planar.c:95-106
                        oy0[3 * i + 0] = y2(s10(w[0], 10), s10(w[1], 0));
                        oy0[3 * i + 1] = y2(s10(w[1], 20), s10(w[2], 10));
                        oy0[3 * i + 2] = y2(s10(w[3], 0), s10(w[3], 20));
                        oy1[3 * i + 0] = y2(s10(v[0], 10), s10(v[1], 0));
                        oy1[3 * i + 1] = y2(s10(v[1], 20), s10(v[2], 10));
                        oy1[3 * i + 2] = y2(s10(v[3], 0), s10(v[3], 20));
                        oc[3 * i + 0] = c2(s10(w[0], 0), s10(v[0], 0), s10(w[0], 20), s10(v[0], 20));    // Cb0 Cr0
                        oc[3 * i + 1] = c2(s10(w[1], 10), s10(v[1], 10), s10(w[2], 0), s10(v[2], 0));    // Cb1 Cr1
                        oc[3 * i + 2] = c2(s10(w[2], 20), s10(v[2], 20), s10(w[3], 10), s10(v[3], 10));  // Cb2 Cr2
                }
                uint8_t *dy0 = out_y + (long) y * ls_y + (long) g0 * 12;
                uint8_t *dy1 = dy0 + ls_y;
                uint8_t *dc = out_c + (long) pr * ls_c + (long) g0 * 12;  // out_linesize[1] * y / 2, :79
                if (!SPILL) {  // every sample lands inside its own row
                        if (full && vec_ok && G == 4) {
#pragma unroll
                                for (int i = 0; i < 3; ++i) {
                                        ((uint4 *) dy0)[i] = make_uint4(oy0[4 * i], oy0[4 * i + 1], oy0[4 * i + 2], oy0[4 * i + 3]);
                                        if (!single) {
                                                ((uint4 *) dy1)[i] = make_uint4(oy1[4 * i], oy1[4 * i + 1], oy1[4 * i + 2], oy1[4 * i + 3]);
                                        }
                                        ((uint4 *) dc)[i] = make_uint4(oc[4 * i], oc[4 * i + 1], oc[4 * i + 2], oc[4 * i + 3]);
                                }
                        } else {
#pragma unroll
                                for (int i = 0; i < 3 * G; ++i) {
                                        if (g0 + i / 3 < groups) {
                                                // 2-byte granularity keeps this correct for any (even) out_linesize
                                                ((uint16_t *) dy0)[2 * i] = (uint16_t) oy0[i], ((uint16_t *) dy0)[2 * i + 1] = (uint16_t) (oy0[i] >> 16);
                                                if (!single) {
                                                        ((uint16_t *) dy1)[2 * i] = (uint16_t) oy1[i], ((uint16_t *) dy1)[2 * i + 1] = (uint16_t) (oy1[i] >> 16);
                                                }
                                                ((uint16_t *) dc)[2 * i] = (uint16_t) oc[i], ((uint16_t *) dc)[2 * i + 1] = (uint16_t) (oc[i] >> 16);
                                        }
                                }
                        }
                        continue;
                }
                // A pair before the last converts (width + 5) / 6 groups (:89) and writes both rows group by group.  Past a tight row's end the
                // first row's last samples land at the start of the second row after that row's own samples - they stay there - and the second
                // row's land on the next pair's first row, which overwrites them later.  Pairs run concurrently here, so that order is made
                // explicit: the first row keeps its whole groups, the second skips the samples the first row's spill owns and stops at its linesize.
                // This holds when a row holds the width and the width at least one group (the spill, under 6 samples, then stays in the next
                // row and comes from a later group than that row's own group 0); the host sends every other geometry to the serial kernel.
                const long row = ls_y / 2, pos = (long) g0 * 6;  // samples per luma row; this thread's first sample
                const long lim0 = last ? row : LONG_MAX, skip1 = last ? 0 : (long) groups * 6 - row;
                const long lim1 = row, lim_c = ls_c / 2;
                if (full && vec_ok && G == 4 && pos + 6 * G <= min(row, lim_c) && pos >= skip1) {
#pragma unroll
                        for (int i = 0; i < 3; ++i) {
                                ((uint4 *) dy0)[i] = make_uint4(oy0[4 * i], oy0[4 * i + 1], oy0[4 * i + 2], oy0[4 * i + 3]);
                                if (!single) {
                                        ((uint4 *) dy1)[i] = make_uint4(oy1[4 * i], oy1[4 * i + 1], oy1[4 * i + 2], oy1[4 * i + 3]);
                                }
                                ((uint4 *) dc)[i] = make_uint4(oc[4 * i], oc[4 * i + 1], oc[4 * i + 2], oc[4 * i + 3]);
                        }
                } else {
#pragma unroll
                        for (int i = 0; i < 3 * G; ++i) {
                                if (g0 + i / 3 < groups) {
                                        // 2-byte granularity keeps this correct for any (even) out_linesize
                                        for (int k = 0; k < 2; ++k) {
                                                const long x = pos + 2 * i + k;
                                                if (x < lim0) {
                                                        ((uint16_t *) dy0)[2 * i + k] = (uint16_t) (oy0[i] >> (16 * k));
                                                }
                                                if (!single && x < lim1 && x >= skip1) {
                                                        ((uint16_t *) dy1)[2 * i + k] = (uint16_t) (oy1[i] >> (16 * k));
                                                }
                                                if (x < lim_c) {
                                                        ((uint16_t *) dc)[2 * i + k] = (uint16_t) (oc[i] >> (16 * k));
                                                }
                                        }
                                }
                        }
                }
        }
}

/// width % 6 tail of the last 1-2 rows (to_planar.c:141-151): copy pix_cnt samples from two rows above
__global__ void v210_to_p010_tail_kernel(uint8_t *out_y, long ls_y, uint8_t *out_c, long ls_c, int height, int full_px, int pix_cnt)
{
        const int i = threadIdx.x;
        if (i >= pix_cnt) {
                return;
        }
        const int y = (height - 1) / 2 * 2;  // first row of the last pair
        uint16_t *dy = (uint16_t *) (out_y + (long) y * ls_y) + full_px;
        uint16_t *dc = (uint16_t *) (out_c + (long) (y / 2) * ls_c) + full_px;
        // reference: dst_y - d.out_linesize[0] on a uint16_t* => out_linesize ELEMENTS = 2 * out_linesize bytes
        // rows that would be read from before the buffer (reference UB) are left untouched
        if (y >= 2) {
                const uint16_t vy = *(dy + i - ls_y);
                dy[i] = vy;
                if (height - y == 2) {
                        ((uint16_t *) ((uint8_t *) dy + ls_y))[i] = vy;
                }
        }
        if (y / 2 >= 2) {
                dc[i] = *(dc + i - ls_c);
        }
}

/// The reference's loop itself (to_planar.c:73-152), in one thread, for the geometries the parallel kernel's ordering rule does not cover: a
/// width below one group, where a pair's single group spills over several rows, or a plane row shorter than the width.  The final bytes are
/// those of the reference's sequential writes; writes past the end of a plane (the reference's own overflow there) are dropped, and the tail
/// copy that would read before the plane is skipped, as in v210_to_p010_tail_kernel.
__global__ void v210_to_p010_serial_kernel(const uint8_t *__restrict__ in, long in_pitch, uint16_t *out_y, long ls_y, uint16_t *out_c, long ls_c,
                                           int width, int height)
{
        const long ry = ls_y / 2, rc = ls_c / 2, ny = ry * height, nc = rc * ((height + 1) / 2);  // samples per row and per plane
        for (int y = 0; y < height; y += 2) {
                const bool single = height - y == 1, last = single || height - y == 2;  // :84-92
                const uint32_t *a = (const uint32_t *) (in + (long) y * in_pitch), *b = single ? a : (const uint32_t *) (in + (long) (y + 1) * in_pitch);
                long dy = (long) y * ry, dy2 = (long) (y + 1) * ry, dc = (long) (y / 2) * rc;
                const int groups = last ? width / 6 : (width + 5) / 6;
                for (int x = 0; x < groups; ++x, a += 4, b += 4) {
                        const uint32_t ya[6] = { s10(a[0], 10), s10(a[1], 0), s10(a[1], 20), s10(a[2], 10), s10(a[3], 0), s10(a[3], 20) };
                        const uint32_t yb[6] = { s10(b[0], 10), s10(b[1], 0), s10(b[1], 20), s10(b[2], 10), s10(b[3], 0), s10(b[3], 20) };
                        const uint32_t c[6] = { (s10(a[0], 0) + s10(b[0], 0)) / 2,   (s10(a[0], 20) + s10(b[0], 20)) / 2, (s10(a[1], 10) + s10(b[1], 10)) / 2,
                                                (s10(a[2], 0) + s10(b[2], 0)) / 2,   (s10(a[2], 20) + s10(b[2], 20)) / 2, (s10(a[3], 10) + s10(b[3], 10)) / 2 };
                        for (int k = 0; k < 6; ++k, ++dy) {
                                if (dy < ny) {
                                        out_y[dy] = (uint16_t) (ya[k] << 6);
                                }
                        }
                        for (int k = 0; k < 6 && !single; ++k, ++dy2) {  // a single last row writes its partner into a scratch row (:84-87)
                                if (dy2 < ny) {
                                        out_y[dy2] = (uint16_t) (yb[k] << 6);
                                }
                        }
                        for (int k = 0; k < 6; ++k, ++dc) {
                                if (dc < nc) {
                                        out_c[dc] = (uint16_t) (c[k] << 6);
                                }
                        }
                }
                if (last && width % 6 != 0) {  // :141-151: pix_cnt samples from out_linesize ELEMENTS back, i.e. two rows up
                        for (int i = 0; i < width % 6; ++i) {
                                if (y >= 2 && dy + i < ny) {
                                        out_y[dy + i] = out_y[dy - 2 * ry + i];
                                }
                                if (y >= 2 && height - y == 2 && dy2 + i < ny) {
                                        out_y[dy2 + i] = out_y[dy - 2 * ry + i];
                                }
                                if (y / 2 >= 2 && dc + i < nc) {
                                        out_c[dc + i] = out_c[dc - 2 * rc + i];
                                }
                        }
                }
        }
}

}  // namespace ugb

extern "C" int ugb200_v210_to_p010le(const struct ugb200_to_planar_data *d, long in_linesize, cuda_wrapper_stream_t stream)
{
        using namespace ugb;
        if (d == nullptr || d->in_data == nullptr || d->out_data[0] == nullptr || d->out_data[1] == nullptr || d->width <= 0 ||
            d->height <= 0 || (d->out_linesize[0] & 1) || (d->out_linesize[1] & 1) || (3 & (size_t) d->in_data)) {
                return -1;  // asserts of to_planar.c:66-68
        }
        if (in_linesize == 0) {
                in_linesize = (d->width + 47) / 48 * 128;  // vc_get_linesize(width, v210), video_codec.c:507-521
        }
        const int groups_mid = (d->width + 5) / 6, groups_last = d->width / 6;  // :89-92
        cudaStream_t s = (cudaStream_t) stream;
        if (d->width < 6 || d->out_linesize[0] / 2 < (unsigned) d->width || d->out_linesize[1] / 2 < (unsigned) d->width) {
                v210_to_p010_serial_kernel<<<1, 1, 0, s>>>((const uint8_t *) d->in_data, in_linesize, (uint16_t *) d->out_data[0], d->out_linesize[0],
                                                           (uint16_t *) d->out_data[1], d->out_linesize[1], d->width, d->height);
                return cudaGetLastError() == cudaSuccess ? 0 : -2;
        }
        const bool vec_ok = !(15 & (size_t) d->in_data) && !(in_linesize & 15) && !(15 & (size_t) d->out_data[0]) &&
                            !(15 & (size_t) d->out_data[1]) && !(d->out_linesize[0] & 15) && !(d->out_linesize[1] & 15);
        const int chunks = (groups_mid + 3) / 4, threads = 128;
        const int pairs = (d->height + 1) / 2;
        dim3 grid((chunks + threads - 1) / threads, pairs > 65535 ? 65535 : pairs);
        // whole groups of a pair before the last reach past a row only when they are wider than it
        const bool spill = d->height > 2 && (6L * groups_mid > d->out_linesize[0] / 2 || 6L * groups_mid > d->out_linesize[1] / 2);
        if (spill) {
                v210_to_p010_kernel<4, true><<<grid, threads, 0, s>>>((const uint8_t *) d->in_data, in_linesize, (uint8_t *) d->out_data[0],
                                                                      d->out_linesize[0], (uint8_t *) d->out_data[1], d->out_linesize[1], d->height,
                                                                      groups_mid, groups_last, vec_ok);
        } else {
                v210_to_p010_kernel<4, false><<<grid, threads, 0, s>>>((const uint8_t *) d->in_data, in_linesize, (uint8_t *) d->out_data[0],
                                                                       d->out_linesize[0], (uint8_t *) d->out_data[1], d->out_linesize[1], d->height,
                                                                       groups_mid, groups_last, vec_ok);
        }
        const int pix_cnt = d->width % 6;
        if (pix_cnt != 0 && d->height > 2) {
                v210_to_p010_tail_kernel<<<1, 32, 0, s>>>((uint8_t *) d->out_data[0], d->out_linesize[0], (uint8_t *) d->out_data[1],
                                                         d->out_linesize[1], d->height, groups_last * 6, pix_cnt);
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
