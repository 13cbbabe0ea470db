// Geometry capture filters and postprocessors on the device: flip, mirror, crop, split, border and interlaced_3d
// (src/capture_filter/flip.c, mirror.c, src/vo_postprocess/crop.c, src/utils/vf_split.cpp, src/vo_postprocess/border.c,
// 3d-interlaced.c).  Contract: DESIGN.md §2 "Geometry filters"; differences: §8.
//
//   flip, crop, split and border are one row kernel: each block takes one output row segment, which a small
//   per-filter descriptor computes (where it lies, how many bytes, where its source is, which bytes are border fill).
//   Stores are 16-byte aligned; when source and destination differ in alignment mod 16, each chunk is funnel-shifted
//   out of two aligned 16-byte loads.  Bytes are handled singly only where a row starts or ends inside a chunk, and
//   where a funnel load would reach outside the segment's source bytes.
//
//   mirror maps four UYVY groups per thread; interlaced_3d maps one 16-byte output chunk per thread, at the drifted
//   position the reference's SSE2 loop writes it to.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/ugb200.h"
#include "filter_args.h"
#include "host/video_codec.h"
#include "rgb_to_uyvy.cuh"

namespace ugb_geo {

constexpr int kThreads = 256;

// a packed pixel format: crop and split take it (get_pf_block_bytes is meaningful)
bool packed(codec_t c) { return get_pf_block_bytes(c) > 0 && !is_codec_opaque(c) && !codec_is_planar(c); }

// ---- the row kernel ------------------------------------------------------------------------------------------------
// Bytes [0, n) of the row at d: byte b is s[b] for b in [c0, c1), else pat[b % period] (border fill).
struct Seg {
        uint8_t *d;
        const uint8_t *s;
        long n, c0, c1;
};

template <int Q> __device__ __forceinline__ uint4 funnel(const uint4 a, const uint4 b, unsigned r)
{
        const uint32_t w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
        return make_uint4(__funnelshift_r(w[Q], w[Q + 1], r), __funnelshift_r(w[Q + 1], w[Q + 2], r), __funnelshift_r(w[Q + 2], w[Q + 3], r),
                          __funnelshift_r(w[Q + 3], w[Q + 4], r));
}

// 16 bytes from p, which is misaligned by `sh` (uniform across the row): two aligned loads, funnel-shifted
__device__ __forceinline__ uint4 load_shifted(const uint8_t *p, unsigned sh)
{
        const uint4 *a = reinterpret_cast<const uint4 *>(p - sh);
        const uint4 lo = a[0], hi = a[1];
        const unsigned r = 8 * (sh & 3);
        switch (sh >> 2) {
        case 0: return funnel<0>(lo, hi, r);
        case 1: return funnel<1>(lo, hi, r);
        case 2: return funnel<2>(lo, hi, r);
        default: return funnel<3>(lo, hi, r);
        }
}

struct Fill {
        uint32_t pat;  // bytes of the fill pattern, low byte first
        int period;    // 3 or 4; unused when no row has fill
        __device__ __forceinline__ uint32_t byte(long b) const { return (pat >> (8 * (b % period))) & 0xffu; }
};

__device__ __forceinline__ uint32_t seg_byte(const Seg &g, const Fill &f, long b)
{
        return b >= g.c0 && b < g.c1 ? uint32_t(g.s[b]) : f.byte(b);
}

template <class Desc> __global__ void __launch_bounds__(kThreads) row_kernel(const Desc desc)
{
        const Fill fill = desc.fill();
        const Seg g = desc.row(blockIdx.x);
        if (g.n <= 0) {
                return;
        }
        const uintptr_t d0 = (uintptr_t) g.d, a0 = d0 & ~uintptr_t(15);
        const long chunks = long((d0 + g.n - a0 + 15) / 16);
        const unsigned sh = unsigned((uintptr_t) g.s - d0) & 15u;  // source misalignment relative to the destination
        for (long k = threadIdx.x; k < chunks; k += blockDim.x) {
                const long b = long(a0 + 16 * k) - long(d0);  // row byte at the chunk's first address (negative in the head)
                if (b >= 0 && b + 16 <= g.n) {
                        uint4 v;
                        const uint8_t *p = g.s + b;
                        const long lo = sh ? b - sh : b, hi = sh ? b - sh + 32 : b + 16;  // the aligned source bytes loaded
                        if (b >= g.c0 && b + 16 <= g.c1 && lo >= g.c0 && hi <= g.c1) {
                                v = sh ? load_shifted(p, sh) : *reinterpret_cast<const uint4 *>(p);
                        } else {
                                uint32_t w[4] = { 0, 0, 0, 0 };
#pragma unroll
                                for (int j = 0; j < 16; ++j) {
                                        w[j >> 2] |= seg_byte(g, fill, b + j) << (8 * (j & 3));
                                }
                                v = make_uint4(w[0], w[1], w[2], w[3]);
                        }
                        *reinterpret_cast<uint4 *>(g.d + b) = v;
                } else {
                        const long e = min(b + 16, g.n);
                        for (long j = max(b, 0L); j < e; ++j) {
                                g.d[j] = uint8_t(seg_byte(g, fill, j));
                        }
                }
        }
}

struct NoFill {
        __device__ __forceinline__ Fill fill() const { return Fill{ 0, 4 }; }
};

// flip.c:77-80: out row h-1-y = in row y
struct FlipDesc : NoFill {
        const uint8_t *s;
        uint8_t *d;
        long L, h;
        __device__ Seg row(long r) const { return Seg{ d + r * L, s + (h - 1 - r) * L, L, 0, L }; }
};

// crop.c:178-182: out row y (at y * pitch) = `pitch` bytes from (yoff + y) * src_linesize + xoff_bytes, clipped to the
// source frame
struct CropDesc : NoFill {
        const uint8_t *s;
        uint8_t *d;
        long pitch, src_ls, first, src_len;  // first = yoff * src_linesize + xoff_bytes >= 0
        __device__ Seg row(long r) const
        {
                const long o = first + r * src_ls, n = min(pitch, src_len - o);
                return Seg{ d + r * pitch, s + o, n, 0, n };
        }
};

// vf_split.cpp:71-82: source row `line`, tile column i -> tile (line / tile_h) * x + i, its row line % tile_h
struct SplitDesc : NoFill {
        const uint8_t *s;
        const uintptr_t *table;  // count tile pointers, then x source byte offsets
        long L, tile_ls, tile_h, n, count;
        int x;
        __device__ Seg row(long r) const
        {
                const long line = r / x, i = r % x;
                uint8_t *t = reinterpret_cast<uint8_t *>(table[(line / tile_h) * x + i]);
                return Seg{ t + (line % tile_h) * tile_ls, s + line * L + long(table[count + i]), n, 0, n };
        }
};

// border.c:132-190, one pass: rows [bh, h - bh) are copied outside the side bands [0, left) and [L - right, L), every
// other byte is the fill
struct BorderDesc {
        const uint8_t *s;
        uint8_t *d;
        long L, h, bh, left, right;
        uint32_t rgba;  // s->color as it lies in memory
        int codec;
        __device__ Fill fill() const
        {
                if (codec == UGB_UYVY) {
                        // vc_copylineRGBAtoUYVY over two pixels of the colour, as border.c:136-140 calls it
                        const uint32_t in[2] = { rgba, rgba };
                        uint32_t out[1];
                        ugb::conv_to_uyvy<0, 1, 2, 4>::pair<0>(in, out);
                        return Fill{ out[0], 4 };
                }
                return Fill{ rgba, codec == UGB_RGB ? 3 : 4 };
        }
        __device__ Seg row(long r) const
        {
                const bool band = r < bh || r >= h - bh;
                return Seg{ d + r * L, s + r * L, L, band ? 0 : left, band ? 0 : L - right };
        }
};

template <class Desc> int launch_rows(const Desc &desc, long rows, cudaStream_t st)
{
        if (rows <= 0) {
                return 0;
        }
        row_kernel<Desc><<<unsigned(rows), kThreads, 0, st>>>(desc);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// ---- mirror --------------------------------------------------------------------------------------------------------
// mirror.c:61-79: group k of a row (U Y0 V Y1) lands at byte L - 4 - 4k as (U Y1 V Y0).  A thread takes four output
// groups: with 16-byte aligned rows one 16-byte load and store, otherwise a word or bytes per group.
__device__ __forceinline__ uint32_t swap_lumas(uint32_t w) { return __byte_perm(w, 0, 0x1230); }

__global__ void __launch_bounds__(kThreads) mirror_kernel(const uint8_t *__restrict__ s, uint8_t *__restrict__ d, long G, long groups, bool vec,
                                                          bool words)
{
        const long t = long(blockIdx.x) * blockDim.x + threadIdx.x, g0 = 4 * t;
        if (g0 >= groups) {
                return;
        }
        if (vec && g0 + 4 <= groups) {
                // rows of a multiple of 4 groups: the four groups share a row, their sources are one aligned 16 bytes
                const long row = g0 / G, k = g0 % G;
                const uint4 v = *reinterpret_cast<const uint4 *>(s + 4 * (row * G + G - 4 - k));
                *reinterpret_cast<uint4 *>(d + 4 * g0) = make_uint4(swap_lumas(v.w), swap_lumas(v.z), swap_lumas(v.y), swap_lumas(v.x));
                return;
        }
        const long e = min(g0 + 4, groups);
        for (long g = g0; g < e; ++g) {
                const long row = g / G, k = g % G;
                const uint8_t *p = s + 4 * (row * G + G - 1 - k);
                uint8_t *q = d + 4 * g;
                if (words) {
                        *reinterpret_cast<uint32_t *>(q) = swap_lumas(*reinterpret_cast<const uint32_t *>(p));
                } else {
                        q[0] = p[0], q[1] = p[3], q[2] = p[2], q[3] = p[1];
                }
        }
}

// ---- interlaced_3d -------------------------------------------------------------------------------------------------
// 3d-interlaced.c:142-163: out row x is written from x * Lc (Lc = L rounded up to 16) in 16-byte chunks, chunk c the
// pavgb of bytes [16c, 16c + 16) of rows x/2*2 and x/2*2+1 of tile x % 2.  Bytes whose sources lie past a tile, and
// bytes past the output frame, are not written.
__device__ __forceinline__ uint4 load16(const uint8_t *base, long o, long len)
{
        const uint8_t *p = base + o;
        const unsigned sh = unsigned((uintptr_t) p & 15u);
        if (sh == 0) {
                return *reinterpret_cast<const uint4 *>(p);
        }
        if (o - long(sh) >= 0 && o - long(sh) + 32 <= len) {
                return load_shifted(p, sh);
        }
        uint32_t w[4] = { 0, 0, 0, 0 };
#pragma unroll
        for (int j = 0; j < 16; ++j) {
                w[j >> 2] |= uint32_t(p[j]) << (8 * (j & 3));
        }
        return make_uint4(w[0], w[1], w[2], w[3]);
}

__global__ void __launch_bounds__(kThreads) interlaced_3d_kernel(const uint8_t *__restrict__ left, const uint8_t *__restrict__ right,
                                                                 uint8_t *__restrict__ d, long L, long cpr, long rows, long len)
{
        const long t = long(blockIdx.x) * blockDim.x + threadIdx.x;
        if (t >= rows * cpr) {
                return;
        }
        const long x = t / cpr, c = t % cpr;
        const long o = x * cpr * 16 + c * 16;  // the drifted output position
        const long a1 = (x / 2 * 2) * L + 16 * c, a2 = a1 + L;
        const long n = min(min(16L, len - o), len - a2);  // bytes of the chunk inside the frame whose sources lie in the tile
        if (n <= 0) {
                return;
        }
        const uint8_t *tile = x % 2 ? right : left;
        if (n == 16 && ((uintptr_t) (d + o) & 15u) == 0) {
                const uint4 p = load16(tile, a1, len), q = load16(tile, a2, len);
                *reinterpret_cast<uint4 *>(d + o) = make_uint4(__vavgu4(p.x, q.x), __vavgu4(p.y, q.y), __vavgu4(p.z, q.z), __vavgu4(p.w, q.w));
                return;
        }
        for (long j = 0; j < n; ++j) {
                d[o + j] = uint8_t((uint32_t(tile[a1 + j]) + tile[a2 + j] + 1) >> 1);
        }
}

// ---- crop arithmetic (crop.c:118-136, :165-172) ------------------------------------------------------------------
struct CropGeom {
        int out_w, out_h, xoff, yoff, xoff_bytes;
};

int crop_geometry(codec_t c, int in_w, int in_h, int width, int height, int xoff, int yoff, CropGeom *g)
{
        // crop_postprocess_reconfigure: MIN in int, then the width rounded to whole blocks in the reference's double arithmetic
        int ow = width ? (width < in_w ? width : in_w) : in_w;
        const int oh = height ? (height < in_h ? height : in_h) : in_h;
        const double bpp = get_bpp(c);
        const int bytes = get_pf_block_bytes(c);
        const int ls = (int) (ow * bpp) / bytes * bytes;
        ow = (int) (unsigned) (ls / bpp);
        // crop_postprocess: unsigned comparison, so a negative offset is clamped only when the sum wraps
        g->out_w = ow;
        g->out_h = oh;
        g->xoff = (unsigned) xoff + (unsigned) ow > (unsigned) in_w ? in_w - ow : (int) (unsigned) xoff;
        g->yoff = (unsigned) yoff + (unsigned) oh > (unsigned) in_h ? in_h - oh : (int) (unsigned) yoff;
        g->xoff_bytes = (int) (g->xoff * bpp) / bytes * bytes;
        return 0;
}

}  // namespace ugb_geo

using namespace ugb_geo;

extern "C" UGB_API int ugb200_cf_flip(int codec, int width, int height, const void *src, void *dst, cuda_wrapper_stream_t stream)
{
        if (src == nullptr || dst == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        const long L = vc_linesize64(width, (codec_t) codec);
        if (L == 0) {
                return -4;
        }
        const size_t n = (size_t) L * height;
        if (overlap(src, n, dst, n)) {
                return -1;
        }
        return launch_rows(FlipDesc{ {}, (const uint8_t *) src, (uint8_t *) dst, L, height }, height, (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_cf_mirror(int codec, int width, int height, const void *src, void *dst, cuda_wrapper_stream_t stream)
{
        if (src == nullptr || dst == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        if (codec != UGB_UYVY) {
                return -4;
        }
        const long G = vc_linesize64(width, (codec_t) codec) / 4, groups = G * height;
        if (overlap(src, 4 * groups, dst, 4 * groups)) {
                return -1;
        }
        const bool vec = G % 4 == 0 && (uintptr_t) src % 16 == 0 && (uintptr_t) dst % 16 == 0;
        const bool words = (uintptr_t) src % 4 == 0 && (uintptr_t) dst % 4 == 0;
        const long threads = (groups + 3) / 4;
        mirror_kernel<<<unsigned((threads + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t) stream>>>(
            (const uint8_t *) src, (uint8_t *) dst, G, groups, vec, words);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" UGB_API int ugb200_cf_crop_geometry(int codec, int in_width, int in_height, int width, int height, int xoff, int yoff,
                                               int out[4])
{
        if (out == nullptr || in_width <= 0 || in_height <= 0 || width < 0 || height < 0) {
                return -1;
        }
        const codec_t c = (codec_t) codec;
        if (!packed(c)) {
                return -4;
        }
        CropGeom g;
        crop_geometry(c, in_width, in_height, width, height, xoff, yoff, &g);
        out[0] = g.out_w, out[1] = g.out_h, out[2] = g.xoff, out[3] = g.yoff;
        return 0;
}

extern "C" UGB_API int ugb200_cf_crop(int codec, int in_width, int in_height, int width, int height, int xoff, int yoff, const void *src,
                                      void *dst, size_t pitch, cuda_wrapper_stream_t stream)
{
        if (src == nullptr || in_width <= 0 || in_height <= 0 || width < 0 || height < 0) {
                return -1;
        }
        const codec_t c = (codec_t) codec;
        if (!packed(c)) {
                return -4;
        }
        CropGeom g;
        crop_geometry(c, in_width, in_height, width, height, xoff, yoff, &g);
        const long src_ls = vc_linesize64(in_width, c), src_len = src_ls * in_height;
        if (pitch == 0) {
                pitch = (size_t) vc_linesize64(g.out_w, c);  // the capture filter's vc_get_linesize(out width)
        }
        const long first = (long) g.yoff * src_ls + g.xoff_bytes;
        // an unclamped negative offset makes the first row start before the source
        if (first < 0) {
                return -1;
        }
        // a window narrower than one pixel block has an empty output frame (which may come without a buffer)
        if (pitch == 0 || g.out_h == 0) {
                return 0;
        }
        if (dst == nullptr || overlap(src, src_len, dst, pitch * g.out_h)) {
                return -1;
        }
        return launch_rows(CropDesc{ {}, (const uint8_t *) src, (uint8_t *) dst, (long) pitch, src_ls, first, src_len }, g.out_h,
                           (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_cf_split(int codec, int width, int height, int x, int y, const void *src, void *const *tiles,
                                       cuda_wrapper_stream_t stream)
{
        if (src == nullptr || tiles == nullptr || width <= 0 || height <= 0 || x <= 0 || y <= 0 || width % x || height % y) {
                return -1;
        }
        const codec_t c = (codec_t) codec;
        if (!packed(c)) {
                return -4;
        }
        const long count = (long) x * y, tw = width / x, th = height / y, L = vc_linesize64(width, c), tile_ls = vc_linesize64(tw, c);
        // vf_split.cpp:74-81 in the reference's arithmetic: (size_t) (tile_w * bpp) bytes per tile row, the source offset
        // accumulated as `unsigned byte += tile_w * bpp`, truncating at every step
        const size_t n = (size_t) (tw * get_bpp(c));
        std::vector<uintptr_t> table(count + x);
        unsigned byte = 0u;
        for (long i = 0; i < x; ++i) {
                table[count + i] = byte;
                byte += tw * get_bpp(c);
        }
        for (long t = 0; t < count; ++t) {
                if (tiles[t] == nullptr || overlap(src, (size_t) L * height, tiles[t], (size_t) tile_ls * th)) {
                        return -1;
                }
                table[t] = (uintptr_t) tiles[t];
        }
        const cudaStream_t st = (cudaStream_t) stream;
        void *dev = nullptr;
        const size_t bytes = table.size() * sizeof(uintptr_t);
        if (ugb_il::scratch_alloc(&dev, bytes, st) != 0) {
                return -2;
        }
        if (cudaMemcpyAsync(dev, table.data(), bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
                cudaFreeAsync(dev, st);
                return -2;
        }
        const SplitDesc desc{ {}, (const uint8_t *) src, (const uintptr_t *) dev, L, tile_ls, th, (long) n, count, x };
        const int rc = launch_rows(desc, (long) height * x, st);
        cudaFreeAsync(dev, st);
        return rc;
}

extern "C" UGB_API int ugb200_pp_border(int codec, int width, int height, const unsigned char color[4], unsigned border_width,
                                        unsigned border_height, const void *src, void *dst, cuda_wrapper_stream_t stream)
{
        if (src == nullptr || dst == nullptr || color == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        if (codec != UGB_UYVY && codec != UGB_RGB && codec != UGB_RGBA) {
                return -4;
        }
        const long L = vc_linesize64(width, (codec_t) codec), bh = border_height;
        long band;  // bytes of each side band
        if (codec == UGB_UYVY) {
                band = ((long) border_width + 1) / 2 * 4;  // a group at i / 2 * 4 for every even i < width
        } else {
                band = (long) border_width * (codec == UGB_RGB ? 3 : 4);
        }
        // the reference's memcpy length goes negative, or a side band starts before its row
        if (2 * bh > height || band > L) {
                return -1;
        }
        const size_t n = (size_t) L * height;
        if (overlap(src, n, dst, n)) {
                return -1;
        }
        uint32_t rgba;
        memcpy(&rgba, color, 4);
        return launch_rows(BorderDesc{ (const uint8_t *) src, (uint8_t *) dst, L, height, bh, band, band, rgba, codec }, height,
                           (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_pp_interlaced_3d(int codec, int width, int height, const void *left, const void *right, void *dst,
                                               cuda_wrapper_stream_t stream)
{
        if (left == nullptr || right == nullptr || dst == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        const long L = vc_linesize64(width, (codec_t) codec);
        if (L == 0) {
                return -4;
        }
        const long len = L * height, cpr = (L + 15) / 16;
        if (overlap(left, len, dst, len) || overlap(right, len, dst, len)) {
                return -1;
        }
        const long threads = cpr * height;
        interlaced_3d_kernel<<<unsigned((threads + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t) stream>>>(
            (const uint8_t *) left, (const uint8_t *) right, (uint8_t *) dst, L, cpr, height, len);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
