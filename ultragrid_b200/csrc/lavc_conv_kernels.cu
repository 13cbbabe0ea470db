// libavcodec bridge conversions on the device (include/ugb200_lavc.h): UltraGrid packed formats -> libavcodec planar formats and back.
// Device form of src/libavcodec/to_lavc_vid_conv.c (the functions of uv_to_av_conversions[], :1458-1531); fills the CUDA hooks the reference
// ships empty (to_lavc_vid_conv_cuda.cu:55-79, from_lavc_vid_conv_cuda.cu:54-72).
//
// All of it is HBM-streaming integer work: a thread owns one pixel group of the packed format (v210: two groups of 6 px = 32 bytes; R10k / RG48 /
// R12L / RGB: 8 px), reads it with 32- or 128-bit loads and writes 8 or 12 consecutive samples per plane with the widest store the plane's
// alignment allows.  Colour matrix: the Q14 integer coefficients of src/color_space.c at the OUTPUT depth (color_space.h constexpr, pinned).
#include <cuda_runtime.h>
#include <stdint.h>

#include <new>

#include "../../include/ugb200.h"
#include "../../include/ugb200_lavc.h"
#include "color_space.h"
#include "host/video_codec.h"  // vc_get_linesize (src/video_codec.c:507-521)

namespace ugb {

struct lavc_planes {
        uint8_t *p[3];
        long ls[3];
};

__device__ __forceinline__ uint32_t v10(uint32_t w, int sh) { return (w >> sh) & 0x3ffu; }

/// n consecutive 16-bit samples to a plane row; `vec`: the row start + element offset is 4-byte aligned (host-checked) and n is even
template <int N>
__device__ __forceinline__ void store16(uint8_t *row, long elem, const uint32_t (&v)[N], int count, bool vec)
{
        uint16_t *d = (uint16_t *) row + elem;
        if (vec && count == N) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) {
                        ((uint32_t *) d)[i] = (v[2 * i] & 0xffffu) | (v[2 * i + 1] << 16);
                }
        } else {
#pragma unroll
                for (int i = 0; i < N; ++i) {
                        if (i < count) {
                                d[i] = (uint16_t) v[i];
                        }
                }
        }
}

// ---- v210 -> yuv420p10le / yuv422p10le / yuv444p10le / yuv444p16le (to_lavc_vid_conv.c:197-385) ------------------------------------
// MODE 0: 4:2:0 10-bit (chroma = (row0 + row1) / 2, :253-259), 1: 4:2:2 10-bit, 2: 4:4:4 10-bit (chroma replicated), 3: 4:4:4 16-bit (<< 6)
template <int MODE>
__global__ void __launch_bounds__(128) lavc_v210_kernel(const uint8_t *__restrict__ in, long in_pitch, lavc_planes o, int groups, int height, bool vec)
{
        const int pair = blockIdx.x * blockDim.x + threadIdx.x;  // two v210 groups = 12 pixels
        const int g0 = pair * 2;
        if (g0 >= groups) {
                return;
        }
        const int ng = min(2, groups - g0);
        const int rows = MODE == 0 ? (height + 1) / 2 : height;
        for (int ry = blockIdx.y; ry < rows; ry += gridDim.y) {
                const int y = MODE == 0 ? ry * 2 : ry;
                if (MODE == 0 && y + 1 >= height) {
                        break;  // the reference reads row y + 1 unconditionally (:207); an odd last row has no partner - it is left alone
                }
                const uint32_t *s0 = (const uint32_t *) (in + (long) y * in_pitch) + g0 * 4;
                uint32_t w[8], x[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        w[i] = i < 4 * ng ? __ldg(s0 + i) : 0u;
                }
                if (MODE == 0) {
                        const uint32_t *s1 = (const uint32_t *) (in + (long) (y + 1) * in_pitch) + g0 * 4;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                x[i] = i < 4 * ng ? __ldg(s1 + i) : 0u;
                        }
                }
                constexpr int SH = MODE == 3 ? 6 : 0;
                uint32_t ya[12], yb[12], cb[12], cr[12];
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                        const uint32_t *a = w + 4 * k, *b = x + 4 * k;
                        ya[6 * k + 0] = v10(a[0], 10) << SH, ya[6 * k + 1] = v10(a[1], 0) << SH, ya[6 * k + 2] = v10(a[1], 20) << SH;
                        ya[6 * k + 3] = v10(a[2], 10) << SH, ya[6 * k + 4] = v10(a[3], 0) << SH, ya[6 * k + 5] = v10(a[3], 20) << SH;
                        uint32_t u[3] = { v10(a[0], 0), v10(a[1], 10), v10(a[2], 20) }, v[3] = { v10(a[0], 20), v10(a[2], 0), v10(a[3], 10) };
                        if (MODE == 0) {
                                yb[6 * k + 0] = v10(b[0], 10), yb[6 * k + 1] = v10(b[1], 0), yb[6 * k + 2] = v10(b[1], 20);
                                yb[6 * k + 3] = v10(b[2], 10), yb[6 * k + 4] = v10(b[3], 0), yb[6 * k + 5] = v10(b[3], 20);
                                u[0] = (u[0] + v10(b[0], 0)) / 2, u[1] = (u[1] + v10(b[1], 10)) / 2, u[2] = (u[2] + v10(b[2], 20)) / 2;
                                v[0] = (v[0] + v10(b[0], 20)) / 2, v[1] = (v[1] + v10(b[2], 0)) / 2, v[2] = (v[2] + v10(b[3], 10)) / 2;
                        }
                        if (MODE >= 2) {
#pragma unroll
                                for (int j = 0; j < 3; ++j) {
                                        cb[6 * k + 2 * j] = cb[6 * k + 2 * j + 1] = u[j] << SH;
                                        cr[6 * k + 2 * j] = cr[6 * k + 2 * j + 1] = v[j] << SH;
                                }
                        } else {
#pragma unroll
                                for (int j = 0; j < 3; ++j) {
                                        cb[3 * k + j] = u[j], cr[3 * k + j] = v[j];
                                }
                        }
                }
                store16<12>(o.p[0] + (long) y * o.ls[0], (long) g0 * 6, ya, ng * 6, vec);
                if (MODE == 0) {
                        store16<12>(o.p[0] + (long) (y + 1) * o.ls[0], (long) g0 * 6, yb, ng * 6, vec);
                }
                const long crow = MODE == 0 ? ry : y;  // out_frame->linesize[1] * y / 2 (:212)
                if (MODE >= 2) {
                        store16<12>(o.p[1] + crow * o.ls[1], (long) g0 * 6, cb, ng * 6, vec);
                        store16<12>(o.p[2] + crow * o.ls[2], (long) g0 * 6, cr, ng * 6, vec);
                } else {
                        const uint32_t cb6[6] = { cb[0], cb[1], cb[2], cb[3], cb[4], cb[5] }, cr6[6] = { cr[0], cr[1], cr[2], cr[3], cr[4], cr[5] };
                        store16<6>(o.p[1] + crow * o.ls[1], (long) g0 * 3, cb6, ng * 3, vec);
                        store16<6>(o.p[2] + crow * o.ls[2], (long) g0 * 3, cr6, ng * 3, vec);
                }
        }
}

// ---- UYVY -> yuv422p / yuv444p (to_lavc_vid_conv.c:137-184): byte moves, 8 pixels (16 bytes) per thread ------------------------------------
template <bool TO444>
__global__ void __launch_bounds__(128) lavc_uyvy_kernel(const uint8_t *__restrict__ in, long in_pitch, lavc_planes o, int width, int height, bool vec)
{
        const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
        if (x0 >= width) {
                return;
        }
        for (int y = blockIdx.y; y < height; y += gridDim.y) {
                const uint8_t *s = in + (long) y * in_pitch + (long) x0 * 2;
                uint8_t *dy = o.p[0] + (long) y * o.ls[0] + x0, *dcb = o.p[1] + (long) y * o.ls[1], *dcr = o.p[2] + (long) y * o.ls[2];
                if (vec && x0 + 8 <= width) {
                        const uint4 q = __ldg((const uint4 *) s);
                        const uint32_t w[4] = { q.x, q.y, q.z, q.w };  // U Y0 V Y1 per word
                        const uint32_t y01 = __byte_perm(w[0], w[1], 0x7531), y23 = __byte_perm(w[2], w[3], 0x7531);
                        const uint32_t u = __byte_perm(__byte_perm(w[0], w[1], 0x0040), __byte_perm(w[2], w[3], 0x0040), 0x5410);
                        const uint32_t v = __byte_perm(__byte_perm(w[0], w[1], 0x0062), __byte_perm(w[2], w[3], 0x0062), 0x5410);
                        *(uint2 *) dy = make_uint2(y01, y23);
                        if (TO444) {  // every chroma sample twice (:170-176)
                                *(uint2 *) (dcb + x0) = make_uint2(__byte_perm(u, 0, 0x1100), __byte_perm(u, 0, 0x3322));
                                *(uint2 *) (dcr + x0) = make_uint2(__byte_perm(v, 0, 0x1100), __byte_perm(v, 0, 0x3322));
                        } else {
                                *(uint32_t *) (dcb + x0 / 2) = u;
                                *(uint32_t *) (dcr + x0 / 2) = v;
                        }
                } else {
                        // the reference steps two pixels at a time and writes both (:145-150): an odd width writes one luma (4:4:4: and chroma)
                        // sample more, kept only where the plane row has room for it
                        for (int x = x0; x < min(x0 + 8, width); x += 2) {
                                const uint8_t *p = in + (long) y * in_pitch + (long) x * 2;
                                dy[x - x0] = p[1];
                                if (x + 1 < o.ls[0]) {
                                        dy[x - x0 + 1] = p[3];
                                }
                                if (TO444) {
                                        dcb[x] = p[0], dcr[x] = p[2];
                                        if (x + 1 < o.ls[1]) {
                                                dcb[x + 1] = p[0];
                                        }
                                        if (x + 1 < o.ls[2]) {
                                                dcr[x + 1] = p[2];
                                        }
                                } else {
                                        dcb[x / 2] = p[0], dcr[x / 2] = p[2];
                                }
                        }
                }
        }
}

// ---- RGB sources -> YCbCr planes at DEPTH (to_lavc_vid_conv.c:702-755 R10k, :757-895 R12L, :1132-1183 RG48, :1185-1227 RGB) ------------------
enum { SRC_R10K = 0, SRC_RG48 = 1, SRC_R12L = 2, SRC_RGB8 = 3 };
template <int SRC>
struct rgb_src;
template <>
struct rgb_src<SRC_R10K> {  // big-endian 10:10:10:2 words
        static constexpr int kDepth = 10, kBytes = 32;
        static __device__ __forceinline__ void load(const uint8_t *p, int (&r)[8], int (&g)[8], int (&b)[8])
        {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        const uint32_t w = __byte_perm(__ldg((const uint32_t *) p + i), 0, 0x0123);
                        r[i] = (int) (w >> 22), g[i] = (int) ((w >> 12) & 0x3ffu), b[i] = (int) ((w >> 2) & 0x3ffu);
                }
        }
};
template <>
struct rgb_src<SRC_RG48> {
        static constexpr int kDepth = 16, kBytes = 48;
        static __device__ __forceinline__ void load(const uint8_t *p, int (&r)[8], int (&g)[8], int (&b)[8])
        {
                uint32_t w[12];
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        w[i] = __ldg((const uint32_t *) p + i);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {  // sample k of the group = 16-bit element k of the 24
                        const int k = 3 * i;
                        r[i] = (int) ((w[k >> 1] >> (16 * (k & 1))) & 0xffffu);
                        g[i] = (int) ((w[(k + 1) >> 1] >> (16 * ((k + 1) & 1))) & 0xffffu);
                        b[i] = (int) ((w[(k + 2) >> 1] >> (16 * ((k + 2) & 1))) & 0xffffu);
                }
        }
};
template <>
struct rgb_src<SRC_R12L> {  // 8 pixels in 36 bytes: a little-endian string of 12-bit fields r0 g0 b0 r1 ... (the byte picking of :790-870)
        static constexpr int kDepth = 12, kBytes = 36;
        static __device__ __forceinline__ void load(const uint8_t *p, int (&r)[8], int (&g)[8], int (&b)[8])
        {
                uint32_t w[10];
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                        w[i] = __ldg((const uint32_t *) p + i);
                }
                w[9] = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                                const int bit = 12 * (3 * i + c);
                                const int val = (int) (__funnelshift_r(w[bit >> 5], w[(bit >> 5) + 1], bit & 31) & 0xfffu);
                                (c == 0 ? r[i] : c == 1 ? g[i] : b[i]) = val;
                        }
                }
        }
};
template <>
struct rgb_src<SRC_RGB8> {
        static constexpr int kDepth = 8, kBytes = 24;
        static __device__ __forceinline__ void load(const uint8_t *p, int (&r)[8], int (&g)[8], int (&b)[8])
        {
                uint32_t w[6];
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                        w[i] = __ldg((const uint32_t *) p + i);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        const int k = 3 * i;
                        r[i] = (int) ((w[k >> 2] >> (8 * (k & 3))) & 0xffu);
                        g[i] = (int) ((w[(k + 1) >> 2] >> (8 * ((k + 1) & 3))) & 0xffu);
                        b[i] = (int) ((w[(k + 2) >> 2] >> (8 * ((k + 2) & 3))) & 0xffu);
                }
        }
};

/// DEPTH: output depth (coefficients of get_color_coeffs(CS_DFL, DEPTH), from the set CS of color_space.h); SUB422: chroma of the even pixels only
/// (r12l_to_yuv422pXXle, :776-787)
template <int SRC, int DEPTH, bool SUB422, class CS = bt709>
__global__ void __launch_bounds__(128) lavc_rgb_kernel(const uint8_t *__restrict__ in, long in_pitch, lavc_planes o, int width, int height, int groups,
                                                       bool vec, bool in_vec)
{
        typedef rgb_src<SRC> S;
        constexpr color_coeffs cf = CS::at(DEPTH);
        constexpr int SHIFT = COMP_BASE + S::kDepth - DEPTH;
        const int gidx = blockIdx.x * blockDim.x + threadIdx.x;
        if (gidx >= groups) {
                return;
        }
        const int x0 = gidx * 8;
        for (int y = blockIdx.y; y < height; y += gridDim.y) {
                int r[8], g[8], b[8];
                const uint8_t *src = in + (long) y * in_pitch + (long) gidx * S::kBytes;
                if (in_vec && (SRC == SRC_R12L || x0 + 8 <= width)) {
                        S::load(src, r, g, b);
                } else {  // a partial last group of a byte-granular format: never read beyond the row's pixels
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                                r[i] = g[i] = b[i] = 0;
                        }
                        if (SRC == SRC_R10K) {
                                for (int i = 0; i < 8 && x0 + i < width; ++i) {
                                        const uint8_t *q = src + 4 * i;
                                        r[i] = q[0] << 2 | q[1] >> 6, g[i] = (q[1] & 0x3f) << 4 | q[2] >> 4, b[i] = (q[2] & 0x0f) << 6 | q[3] >> 2;
                                }
                        } else if (SRC == SRC_RG48) {
                                for (int i = 0; i < 8 && x0 + i < width; ++i) {
                                        const uint16_t *q = (const uint16_t *) src + 3 * i;
                                        r[i] = q[0], g[i] = q[1], b[i] = q[2];
                                }
                        } else if (SRC == SRC_RGB8) {
                                for (int i = 0; i < 8 && x0 + i < width; ++i) {
                                        r[i] = src[3 * i], g[i] = src[3 * i + 1], b[i] = src[3 * i + 2];
                                }
                        } else {
                                uint8_t tmp[40];
                                for (int i = 0; i < 36; ++i) {
                                        tmp[i] = src[i];
                                }
                                for (int i = 0; i < 8; ++i) {
                                        for (int c = 0; c < 3; ++c) {
                                                const int bit = 12 * (3 * i + c), by = bit >> 3;
                                                const int val = ((tmp[by] | tmp[by + 1] << 8) >> (bit & 7)) & 0xfff;
                                                (c == 0 ? r[i] : c == 1 ? g[i] : b[i]) = val;
                                        }
                                }
                        }
                }
                uint32_t oy[8], ocb[8], ocr[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                        oy[i] = (uint32_t) (((r[i] * cf.y_r + g[i] * cf.y_g + b[i] * cf.y_b) >> SHIFT) + (1 << (DEPTH - 4)));
                        ocb[i] = (uint32_t) (((r[i] * cf.cb_r + g[i] * cf.cb_g + b[i] * cf.cb_b) >> SHIFT) + (1 << (DEPTH - 1)));
                        ocr[i] = (uint32_t) (((r[i] * cf.cr_r + g[i] * cf.cr_g + b[i] * cf.cr_b) >> SHIFT) + (1 << (DEPTH - 1)));
                }
                // whole groups are written like the reference does (R12L: x += 8), clipped to what the plane row can hold
                if (DEPTH == 8) {
                        uint8_t *dy = o.p[0] + (long) y * o.ls[0] + x0, *dcb = o.p[1] + (long) y * o.ls[1] + x0, *dcr = o.p[2] + (long) y * o.ls[2] + x0;
                        const int n = min(8, width - x0);
                        if (vec && n == 8) {
                                *(uint2 *) dy = make_uint2(oy[0] & 0xff | (oy[1] & 0xff) << 8 | (oy[2] & 0xff) << 16 | oy[3] << 24,
                                                           oy[4] & 0xff | (oy[5] & 0xff) << 8 | (oy[6] & 0xff) << 16 | oy[7] << 24);
                                *(uint2 *) dcb = make_uint2(ocb[0] & 0xff | (ocb[1] & 0xff) << 8 | (ocb[2] & 0xff) << 16 | ocb[3] << 24,
                                                            ocb[4] & 0xff | (ocb[5] & 0xff) << 8 | (ocb[6] & 0xff) << 16 | ocb[7] << 24);
                                *(uint2 *) dcr = make_uint2(ocr[0] & 0xff | (ocr[1] & 0xff) << 8 | (ocr[2] & 0xff) << 16 | ocr[3] << 24,
                                                            ocr[4] & 0xff | (ocr[5] & 0xff) << 8 | (ocr[6] & 0xff) << 16 | ocr[7] << 24);
                        } else {
                                for (int i = 0; i < n; ++i) {
                                        dy[i] = (uint8_t) oy[i], dcb[i] = (uint8_t) ocb[i], dcr[i] = (uint8_t) ocr[i];
                                }
                        }
                } else {
                        const int cap_y = (int) min((long) 8, o.ls[0] / 2 - x0);
                        const int ny = SRC == SRC_R12L ? cap_y : min(8, width - x0);
                        store16<8>(o.p[0] + (long) y * o.ls[0], x0, oy, ny, vec);
                        if (SUB422) {
                                const uint32_t cb4[4] = { ocb[0], ocb[2], ocb[4], ocb[6] }, cr4[4] = { ocr[0], ocr[2], ocr[4], ocr[6] };
                                const int nc = (int) min((long) 4, o.ls[1] / 2 - x0 / 2);
                                store16<4>(o.p[1] + (long) y * o.ls[1], x0 / 2, cb4, nc, vec);
                                store16<4>(o.p[2] + (long) y * o.ls[2], x0 / 2, cr4, nc, vec);
                        } else {
                                const int nc = SRC == SRC_R12L ? (int) min((long) 8, o.ls[1] / 2 - x0) : ny;
                                store16<8>(o.p[1] + (long) y * o.ls[1], x0, ocb, nc, vec);
                                store16<8>(o.p[2] + (long) y * o.ls[2], x0, ocr, nc, vec);
                        }
                }
        }
}

// ---- RGB / RGBA -> GBRP (to_lavc_vid_conv.c:1315-1360): planes G, B, R -------------------------------------------------------------------
template <int BPP>
__global__ void __launch_bounds__(256) lavc_gbrp_kernel(const uint8_t *__restrict__ in, long in_pitch, lavc_planes o, int width, int height)
{
        const int x = blockIdx.x * blockDim.x + threadIdx.x;
        if (x >= width) {
                return;
        }
        for (int y = blockIdx.y; y < height; y += gridDim.y) {
                const uint8_t *s = in + (long) y * in_pitch + (long) x * BPP;
                o.p[0][(long) y * o.ls[0] + x] = s[1];
                o.p[1][(long) y * o.ls[1] + x] = s[2];
                o.p[2][(long) y * o.ls[2] + x] = s[0];
        }
}

// ---- from_lavc YUV444P -> UYVY (from_lavc_vid_conv.c:663-685): width / 2 pixel pairs, chroma = (c[2x] + c[2x + 1]) / 2 (C truncation) ------------
__global__ void __launch_bounds__(128) lavc_yuv444p_uyvy_kernel(const uint8_t *__restrict__ py, const uint8_t *__restrict__ pb,
                                                                 const uint8_t *__restrict__ pr, long ls_y, long ls_b, long ls_r, uint8_t *out,
                                                                 long pitch, int pairs, int height, bool al4)
{
        const int x = blockIdx.x * blockDim.x + threadIdx.x;
        if (x >= pairs) {
                return;
        }
        for (int y = blockIdx.y; y < height; y += gridDim.y) {
                const uint8_t *sy = py + (long) y * ls_y + 2 * x, *sb = pb + (long) y * ls_b + 2 * x, *sr = pr + (long) y * ls_r + 2 * x;
                const uint32_t u = ((uint32_t) __ldg(sb) + __ldg(sb + 1)) / 2, v = ((uint32_t) __ldg(sr) + __ldg(sr + 1)) / 2;
                const uint32_t w = u | (uint32_t) __ldg(sy) << 8 | v << 16 | (uint32_t) __ldg(sy + 1) << 24;
                uint8_t *d = out + (long) y * pitch + 4L * x;
                if (al4) {
                        *(uint32_t *) d = w;
                } else {
                        d[0] = (uint8_t) w, d[1] = (uint8_t) (w >> 8), d[2] = (uint8_t) (w >> 16), d[3] = (uint8_t) (w >> 24);
                }
        }
}

// ---- from_lavc YUV422P10LE -> v210 intermediate: the partial last 6-pixel group of each row, which yuv422p10le_to_v210 leaves out (from_planar.c:308)
// and the line converter after it reads; samples beyond the width are 0 --------------------------------------------------------------------------
__global__ void __launch_bounds__(128) lavc_v210_partial_kernel(const uint8_t *py, const uint8_t *pb, const uint8_t *pr, long ls_y, long ls_b,
                                                                long ls_r, uint8_t *mid, long mid_pitch, int width, int height)
{
        const int y = blockIdx.x * blockDim.x + threadIdx.x;
        if (y >= height) {
                return;
        }
        const int g = width / 6, ny = width - 6 * g, nc = (width + 1) / 2 - 3 * g;
        const uint16_t *sy = (const uint16_t *) (py + (long) y * ls_y) + 6 * g, *sb = (const uint16_t *) (pb + (long) y * ls_b) + 3 * g,
                       *sr = (const uint16_t *) (pr + (long) y * ls_r) + 3 * g;
        uint32_t Y[6], B[3], R[3];
#pragma unroll
        for (int i = 0; i < 6; ++i) {
                Y[i] = i < ny ? sy[i] : 0u;
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
                B[i] = i < nc ? sb[i] : 0u, R[i] = i < nc ? sr[i] : 0u;
        }
        *(uint4 *) (mid + (long) y * mid_pitch + 16L * g) =
                make_uint4(B[0] | Y[0] << 10 | R[0] << 20, Y[1] | B[1] << 10 | Y[2] << 20, R[1] | Y[3] << 10 | B[2] << 20, Y[4] | R[2] << 10 | Y[5] << 20);
}

struct lavc_fmt_info {
        int planes, depth_bytes, hsub, vsub;  // chroma subsampling shifts
        bool semi;                            // two-plane (NV12 / P010)
};
inline lavc_fmt_info fmt_info(int f)
{
        switch (f) {
        case UGB_AV_YUV420P: return { 3, 1, 1, 1, false };
        case UGB_AV_YUV422P: return { 3, 1, 1, 0, false };
        case UGB_AV_YUV444P: return { 3, 1, 0, 0, false };
        case UGB_AV_GBRP: return { 3, 1, 0, 0, false };
        case UGB_AV_NV12: return { 2, 1, 1, 1, true };
        case UGB_AV_P010LE: return { 2, 2, 1, 1, true };
        case UGB_AV_YUV420P10LE: return { 3, 2, 1, 1, false };
        case UGB_AV_YUV422P10LE:
        case UGB_AV_YUV422P12LE:
        case UGB_AV_YUV422P16LE: return { 3, 2, 1, 0, false };
        case UGB_AV_YUV444P10LE:
        case UGB_AV_YUV444P12LE:
        case UGB_AV_YUV444P16LE: return { 3, 2, 0, 0, false };
        default: return { 0, 0, 0, 0, false };
        }
}

inline long linesize_of(int w, int codec)
{
        switch (codec) {
        case UGB_v210: return (long) ((w + 47) / 48) * 128;
        case UGB_UYVY: return (long) ((w + 1) / 2) * 4;  // uyvy_to_yuv422p's source pointer runs on over (w + 1) / 2 pairs per row (:144)
        case UGB_R10k: return (long) ((w + 63) / 64) * 256;  // vc_get_linesize: R10k rows are padded to 64 pixels (r10k_to_yuv444pXXle, :712)
        case UGB_RG48: return (long) w * 6;
        case UGB_R12L: return (long) ((w + 7) / 8) * 36;
        case UGB_RGB: return (long) w * 3;
        case UGB_RGBA: return (long) w * 4;
        case UGB_Y216: return (long) ((w + 1) / 2) * 8;
        default: return 0;
        }
}

}  // namespace ugb

using namespace ugb;

extern "C" {

int ugb200_to_lavc_supported(int in, int f)
{
        switch (in) {
        case UGB_v210: return f == UGB_AV_YUV420P10LE || f == UGB_AV_YUV422P10LE || f == UGB_AV_YUV444P10LE || f == UGB_AV_YUV444P16LE || f == UGB_AV_P010LE;
        case UGB_UYVY: return f == UGB_AV_YUV422P || f == UGB_AV_YUV444P || f == UGB_AV_YUV420P || f == UGB_AV_NV12;
        case UGB_R10k:
        case UGB_RG48: return f == UGB_AV_YUV444P10LE || f == UGB_AV_YUV444P12LE || f == UGB_AV_YUV444P16LE;
        case UGB_R12L:
                return f == UGB_AV_YUV444P10LE || f == UGB_AV_YUV444P12LE || f == UGB_AV_YUV444P16LE || f == UGB_AV_YUV422P10LE || f == UGB_AV_YUV422P12LE ||
                       f == UGB_AV_YUV422P16LE;
        case UGB_RGB: return f == UGB_AV_YUV444P || f == UGB_AV_GBRP;
        case UGB_RGBA: return f == UGB_AV_GBRP;
        case UGB_Y216: return f == UGB_AV_P010LE;
        default: return 0;
        }
}

}  // extern "C"

template <class CS>
static int to_lavc_convert(int in, int f, const struct ugb200_av_planes *out, const void *in_data, int width, int height, cuda_wrapper_stream_t stream)
{
        cudaStream_t st = (cudaStream_t) stream;
        const lavc_fmt_info fi = fmt_info(f);
        lavc_planes o{};
        bool vec = true;
        for (int i = 0; i < fi.planes; ++i) {
                if (!out->data[i] || out->linesize[i] <= 0) {
                        return -1;
                }
                if (fi.depth_bytes == 2 && (((size_t) out->data[i] & 1) || (out->linesize[i] & 1))) {
                        return -1;  // 16-bit samples: the reference asserts even line sizes (:200-202, :708-710, :763-765)
                }
                o.p[i] = out->data[i], o.ls[i] = out->linesize[i];
                vec = vec && !((size_t) out->data[i] & 15) && !(out->linesize[i] & 15);
        }
        const uint8_t *src = (const uint8_t *) in_data;
        const long pitch = linesize_of(width, in);
        const bool in_vec = !((size_t) src & 3) && !(pitch & 3);
        // conversions that the reference delegates to src/to_planar.c (:132-135,186-189 and to_lavc_v210_to_p010le / to_lavc_y216_to_p010le)
        if ((in == UGB_UYVY && (f == UGB_AV_YUV420P || f == UGB_AV_NV12)) || f == UGB_AV_P010LE) {
                struct ugb200_to_planar_data d{};
                d.width = width, d.height = height, d.in_data = src;
                for (int i = 0; i < fi.planes; ++i) {
                        d.out_data[i] = out->data[i], d.out_linesize[i] = (unsigned) out->linesize[i];
                }
                if (in == UGB_v210) {
                        return ugb200_v210_to_p010le(&d, 0, stream);
                }
                if (in == UGB_Y216) {
                        return ugb200_y216_to_p010le(&d, stream);
                }
                return f == UGB_AV_NV12 ? ugb200_uyvy_to_nv12(&d, stream) : ugb200_uyvy_to_i420(&d, stream);
        }
        const int gy = min(height, 16384);
        if (in == UGB_v210) {
                if (!in_vec) {
                        return -1;  // the reference asserts 4-byte alignment too (:199)
                }
                const int groups = width / 6;  // whole groups only (:215)
                if (groups == 0) {
                        return 0;
                }
                const dim3 grid(((groups + 1) / 2 + 127) / 128, f == UGB_AV_YUV420P10LE ? min((height + 1) / 2, 16384) : gy);
                switch (f) {
                case UGB_AV_YUV420P10LE: lavc_v210_kernel<0><<<grid, 128, 0, st>>>(src, pitch, o, groups, height, vec); break;
                case UGB_AV_YUV422P10LE: lavc_v210_kernel<1><<<grid, 128, 0, st>>>(src, pitch, o, groups, height, vec); break;
                case UGB_AV_YUV444P10LE: lavc_v210_kernel<2><<<grid, 128, 0, st>>>(src, pitch, o, groups, height, vec); break;
                default: lavc_v210_kernel<3><<<grid, 128, 0, st>>>(src, pitch, o, groups, height, vec); break;
                }
        } else if (in == UGB_UYVY) {
                const dim3 grid(((width + 7) / 8 + 127) / 128, gy);
                const bool v16 = vec && !((size_t) src & 15) && !(pitch & 15);
                if (f == UGB_AV_YUV444P) {
                        lavc_uyvy_kernel<true><<<grid, 128, 0, st>>>(src, pitch, o, width, height, v16);
                } else {
                        lavc_uyvy_kernel<false><<<grid, 128, 0, st>>>(src, pitch, o, width, height, v16);
                }
        } else if (f == UGB_AV_GBRP) {
                const dim3 grid((width + 255) / 256, gy);
                if (in == UGB_RGB) {
                        lavc_gbrp_kernel<3><<<grid, 256, 0, st>>>(src, pitch, o, width, height);
                } else {
                        lavc_gbrp_kernel<4><<<grid, 256, 0, st>>>(src, pitch, o, width, height);
                }
        } else {
                const int groups = (width + 7) / 8;
                const dim3 grid((groups + 127) / 128, gy);
#define UGB_RGB_LAUNCH(SRC, DEPTH, SUB) lavc_rgb_kernel<SRC, DEPTH, SUB, CS><<<grid, 128, 0, st>>>(src, pitch, o, width, height, groups, vec, in_vec)
#define UGB_RGB_DEPTHS(SRC)                                                                       \
        switch (f) {                                                                              \
        case UGB_AV_YUV444P10LE: UGB_RGB_LAUNCH(SRC, 10, false); break;                           \
        case UGB_AV_YUV444P12LE: UGB_RGB_LAUNCH(SRC, 12, false); break;                           \
        default: UGB_RGB_LAUNCH(SRC, 16, false); break;                                           \
        }
                if (in == UGB_R10k) {
                        UGB_RGB_DEPTHS(SRC_R10K)
                } else if (in == UGB_RG48) {
                        UGB_RGB_DEPTHS(SRC_RG48)
                } else if (in == UGB_RGB) {
                        UGB_RGB_LAUNCH(SRC_RGB8, 8, false);
                } else {
                        switch (f) {
                        case UGB_AV_YUV444P10LE: UGB_RGB_LAUNCH(SRC_R12L, 10, false); break;
                        case UGB_AV_YUV444P12LE: UGB_RGB_LAUNCH(SRC_R12L, 12, false); break;
                        case UGB_AV_YUV444P16LE: UGB_RGB_LAUNCH(SRC_R12L, 16, false); break;
                        case UGB_AV_YUV422P10LE: UGB_RGB_LAUNCH(SRC_R12L, 10, true); break;
                        case UGB_AV_YUV422P12LE: UGB_RGB_LAUNCH(SRC_R12L, 12, true); break;
                        default: UGB_RGB_LAUNCH(SRC_R12L, 16, true); break;
                        }
                }
#undef UGB_RGB_DEPTHS
#undef UGB_RGB_LAUNCH
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" {

int ugb200_to_lavc_convert_cs(int in, int f, const struct ugb200_av_planes *out, const void *in_data, int width, int height, int cs,
                              cuda_wrapper_stream_t stream)
{
        if (!out || !in_data || width <= 0 || height <= 0 || !ugb200_to_lavc_supported(in, f)) {
                return -1;
        }
        switch (cs) {
        case UGB_CS_DFL:
        case UGB_CS_709: return to_lavc_convert<bt709>(in, f, out, in_data, width, height, stream);
        case UGB_CS_601: return to_lavc_convert<bt601>(in, f, out, in_data, width, height, stream);
        default: return -1;
        }
}

int ugb200_to_lavc_convert(int in, int f, const struct ugb200_av_planes *out, const void *in_data, int width, int height, cuda_wrapper_stream_t stream)
{
        return ugb200_to_lavc_convert_cs(in, f, out, in_data, width, height, UGB_CS_709, stream);
}

// ---- hook shape: to_lavc_vid_conv_cuda_init / to_lavc_vid_conv_cuda / _destroy (to_lavc_vid_conv_cuda.h:60-65) -------------------------------
struct ugb200_to_lavc_conv {
        int in_codec, width, height, av_pixfmt, cs;
        struct ugb200_av_planes planes;  // device memory, owned
        void *d_in;                      // staging of a host input frame
        size_t in_bytes;
        cudaStream_t stream;
};

struct ugb200_to_lavc_conv *ugb200_to_lavc_vid_conv_init_cs(int in_codec, int width, int height, int av_pixfmt, int cs)
{
        if (width <= 0 || height <= 0 || !ugb200_to_lavc_supported(in_codec, av_pixfmt) || (cs != UGB_CS_DFL && cs != UGB_CS_601 && cs != UGB_CS_709)) {
                return nullptr;
        }
        auto *s = new (std::nothrow) ugb200_to_lavc_conv();
        if (!s) {
                return nullptr;
        }
        s->in_codec = in_codec, s->width = width, s->height = height, s->av_pixfmt = av_pixfmt, s->cs = cs;
        const lavc_fmt_info fi = fmt_info(av_pixfmt);
        bool ok = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) == cudaSuccess;
        for (int i = 0; i < fi.planes && ok; ++i) {
                const bool chroma = i > 0 && av_pixfmt != UGB_AV_GBRP;
                int w = chroma ? (width + (1 << fi.hsub) - 1) >> fi.hsub : width, h = chroma ? (height + (1 << fi.vsub) - 1) >> fi.vsub : height;
                if (chroma && fi.semi) {
                        w *= 2;  // interleaved CbCr
                }
                // rows padded like av_frame_get_buffer() pads them (64-byte multiples), one spare group for the whole-group writers
                s->planes.linesize[i] = ((w + 8) * fi.depth_bytes + 63) & ~63;
                ok = cudaMalloc((void **) &s->planes.data[i], (size_t) s->planes.linesize[i] * h) == cudaSuccess;
        }
        s->in_bytes = (size_t) linesize_of(width, in_codec) * height;
        ok = ok && cudaMalloc(&s->d_in, s->in_bytes + 64) == cudaSuccess;
        if (!ok) {
                ugb200_to_lavc_vid_conv_destroy(&s);
                return nullptr;
        }
        return s;
}

struct ugb200_to_lavc_conv *ugb200_to_lavc_vid_conv_init(int in_codec, int width, int height, int av_pixfmt)
{
        return ugb200_to_lavc_vid_conv_init_cs(in_codec, width, height, av_pixfmt, UGB_CS_709);
}

const struct ugb200_av_planes *ugb200_to_lavc_vid_conv(struct ugb200_to_lavc_conv *s, const char *in_data, int in_is_device)
{
        if (!s || !in_data) {
                return nullptr;
        }
        const void *src = in_data;
        if (!in_is_device) {
                if (cudaMemcpyAsync(s->d_in, in_data, s->in_bytes, cudaMemcpyHostToDevice, s->stream) != cudaSuccess) {
                        return nullptr;
                }
                src = s->d_in;
        }
        if (ugb200_to_lavc_convert_cs(s->in_codec, s->av_pixfmt, &s->planes, src, s->width, s->height, s->cs, s->stream) != 0 ||
            cudaStreamSynchronize(s->stream) != cudaSuccess) {
                return nullptr;
        }
        return &s->planes;
}

void ugb200_to_lavc_vid_conv_destroy(struct ugb200_to_lavc_conv **state)
{
        if (!state || !*state) {
                return;
        }
        ugb200_to_lavc_conv *s = *state;
        for (auto &p : s->planes.data) {
                cudaFree(p);
        }
        cudaFree(s->d_in);
        if (s->stream) {
                cudaStreamDestroy(s->stream);
        }
        delete s;
        *state = nullptr;
}

// ---- from_lavc: get_av_to_uv_cuda_conversion / av_to_uv_convert_cuda / av_to_uv_conversion_cuda_destroy (from_lavc_vid_conv_cuda.h:61-69) ----
struct ugb200_av_to_uv_conv {
        int av_pixfmt, out_codec, mid_codec;  // planar stage produces mid_codec; a line converter follows when it differs from out_codec
        void *d_mid, *d_out;  // intermediate frame; line-converter output when it writes whole groups past the destination's line
        size_t mid_cap, out_cap;
};

static bool grow(void **p, size_t *cap, size_t need)
{
        if (need <= *cap) {
                return true;
        }
        cudaFree(*p);
        *p = nullptr, *cap = 0;
        if (cudaMalloc(p, need) != cudaSuccess) {
                *p = nullptr;
                return false;
        }
        *cap = need;
        return true;
}

static int planar_mid_codec(int av_pixfmt)
{
        switch (av_pixfmt) {
        case UGB_AV_YUV420P:
        case UGB_AV_YUV422P: return UGB_UYVY;
        case UGB_AV_YUV444P: return UGB_VUYA;
        case UGB_AV_YUV422P10LE: return UGB_v210;
        case UGB_AV_GBRP: return UGB_RGB;
        default: return UGB_VIDEO_CODEC_NONE;
        }
}

struct ugb200_av_to_uv_conv *ugb200_get_av_to_uv_conversion(int av_pixfmt, int out_codec)
{
        const int mid = planar_mid_codec(av_pixfmt);
        if (mid == UGB_VIDEO_CODEC_NONE || (mid != out_codec && !ugb200_pixfmt_supported(mid, out_codec))) {
                return nullptr;
        }
        auto *s = new (std::nothrow) ugb200_av_to_uv_conv();
        if (s) {
                s->av_pixfmt = av_pixfmt, s->out_codec = out_codec, s->mid_codec = mid, s->d_mid = s->d_out = nullptr, s->mid_cap = s->out_cap = 0;
        }
        return s;
}

int ugb200_av_to_uv_convert(struct ugb200_av_to_uv_conv *s, char *dst_buffer, const struct ugb200_av_planes *in, int width, int height, int pitch,
                            const int *rgb_shift, cuda_wrapper_stream_t stream)
{
        if (!s || !dst_buffer || !in || width <= 0 || height <= 0) {
                return -1;
        }
        // the reference's own entries for YUV444P -> UYVY (yuv444p_to_uyvy, from_lavc_vid_conv.c:2100) and YUV422P10LE -> UYVY
        // (yuv422p10le_to_uyvy, :2057) convert in one step; the VUYA / v210 intermediate would lose the second luma (vc_copylineVUYAtoUYVY takes
        // it from the alpha byte, pixfmt_conv.c:2699) or the pixels of a partial 6-pixel group
        if (s->out_codec == UGB_UYVY && (s->av_pixfmt == UGB_AV_YUV444P || s->av_pixfmt == UGB_AV_YUV422P10LE)) {
                if (!in->data[0] || !in->data[1] || !in->data[2]) {
                        return -1;
                }
                if (s->av_pixfmt == UGB_AV_YUV422P10LE) {
                        struct ugb200_from_planar_data d{};
                        d.width = width, d.height = height, d.out_data = (unsigned char *) dst_buffer, d.out_pitch = (unsigned) pitch, d.in_depth = 10;
                        for (int i = 0; i < 3; ++i) {
                                d.in_data[i] = in->data[i], d.in_linesize[i] = (unsigned) in->linesize[i];
                        }
                        return ugb200_yuv422p10le_to_uyvy(&d, stream);
                }
                const int pairs = width / 2;
                if (pairs == 0) {
                        return 0;
                }
                const dim3 grid((pairs + 127) / 128, min(height, 16384));
                lavc_yuv444p_uyvy_kernel<<<grid, 128, 0, (cudaStream_t) stream>>>(in->data[0], in->data[1], in->data[2], in->linesize[0], in->linesize[1],
                                                                                  in->linesize[2], (uint8_t *) dst_buffer, pitch, pairs, height,
                                                                                  !((size_t) dst_buffer & 3) && !(pitch & 3));
                return cudaGetLastError() == cudaSuccess ? 0 : -2;
        }
        const bool direct = s->mid_codec == s->out_codec;
        const long mid_pitch = direct ? pitch : (long) vc_get_linesize((unsigned) width, (codec_t) s->mid_codec);
        unsigned char *mid = (unsigned char *) dst_buffer;
        if (!direct) {
                if (!grow(&s->d_mid, &s->mid_cap, (size_t) mid_pitch * height + 64)) {
                        return -2;
                }
                mid = (unsigned char *) s->d_mid;
        }
        struct ugb200_from_planar_data d{};
        d.width = width, d.height = height, d.out_data = mid, d.out_pitch = (unsigned) mid_pitch;
        for (int i = 0; i < 3; ++i) {
                d.in_data[i] = in->data[i], d.in_linesize[i] = (unsigned) in->linesize[i];
        }
        d.in_depth = s->av_pixfmt == UGB_AV_YUV422P10LE ? 10 : 8;
        d.rgb_shift[0] = rgb_shift ? rgb_shift[0] : 0, d.rgb_shift[1] = rgb_shift ? rgb_shift[1] : 8, d.rgb_shift[2] = rgb_shift ? rgb_shift[2] : 16;
        int rc;
        switch (s->av_pixfmt) {
        case UGB_AV_YUV420P: rc = ugb200_yuv420p_to_uyvy(&d, stream); break;
        case UGB_AV_YUV422P: rc = ugb200_yuv422p_to_uyvy(&d, stream); break;
        case UGB_AV_YUV444P: rc = ugb200_yuv444p_to_vuya(&d, stream); break;
        case UGB_AV_YUV422P10LE: rc = ugb200_yuv422p10le_to_v210(&d, stream); break;
        default: rc = ugb200_gbrap_to_rgb(&d, stream); break;  // 8-bit planes G, B, R
        }
        if (rc != 0 || direct) {
                return rc;
        }
        // A v210 intermediate: its partial last group is converted too, and the line converters after it write whole 6-pixel groups
        // (vc_copylineV210toRGB, pixfmt_conv.c:2884-2940), past the destination's line when the width is not a multiple of 6.  They write into
        // a frame of the rounded-up width, and the destination receives the lines.
        const int wc = s->mid_codec == UGB_v210 ? (width + 5) / 6 * 6 : width;
        const long ls = vc_get_linesize((unsigned) width, (codec_t) s->out_codec), lsc = vc_get_linesize((unsigned) wc, (codec_t) s->out_codec);
        cudaStream_t st = (cudaStream_t) stream;
        if (wc != width) {
                lavc_v210_partial_kernel<<<(height + 127) / 128, 128, 0, st>>>(in->data[0], in->data[1], in->data[2], in->linesize[0], in->linesize[1],
                                                                               in->linesize[2], mid, mid_pitch, width, height);
        }
        if (lsc == ls) {
                return ugb200_pixfmt_convert(s->mid_codec, s->out_codec, dst_buffer, pitch, mid, mid_pitch, (int) ls, height, (long) mid_pitch * height,
                                             d.rgb_shift[0], d.rgb_shift[1], d.rgb_shift[2], stream);
        }
        if (!grow(&s->d_out, &s->out_cap, (size_t) lsc * height + 64)) {
                return -2;
        }
        rc = ugb200_pixfmt_convert(s->mid_codec, s->out_codec, s->d_out, lsc, mid, mid_pitch, (int) lsc, height, (long) mid_pitch * height, d.rgb_shift[0],
                                   d.rgb_shift[1], d.rgb_shift[2], stream);
        if (rc != 0) {
                return rc;
        }
        return cudaMemcpy2DAsync(dst_buffer, pitch, s->d_out, lsc, ls, height, cudaMemcpyDeviceToDevice, st) == cudaSuccess ? 0 : -2;
}

void ugb200_av_to_uv_conversion_destroy(struct ugb200_av_to_uv_conv **state)
{
        if (state && *state) {
                cudaFree((*state)->d_mid);
                cudaFree((*state)->d_out);
                delete *state;
                *state = nullptr;
        }
}

}  // extern "C"
