// The logo capture filter and the R12L <-> Y416 pass-through filters on the device (src/capture_filter/logo.c,
// r12l_to_y416_fake.c, src/vo_postprocess/y416_to_r12l_fake.c).  Contract: DESIGN.md §2 "Logo and the R12L <-> Y416
// pass-through filters"; differences: §8.
//
//   logo is one fused launch over the logo rectangle: a thread takes one chunk of a rectangle row (16 pixels, 32 for
//   R12L), decodes it to RGB with the line converter of pixfmt_kernels.cu that the reference's decoder_t is, blends
//   the logo pixels over it, encodes it back with the reference's coder and stores the bytes of the written span.
//   There is no RGB segment in memory, and nothing outside the rectangle's span is read or written.
//
//   r12l_to_y416_fake and y416_to_r12l_fake are streaming kernels, one thread per 8-pixel group: 36 bytes of R12L,
//   64 of Y416.
#include <cuda_runtime.h>
#include <stdint.h>

#include <new>

#include "../../include/ugb200.h"
#include "filter_args.h"
#include "host/video_codec.h"
#include "rgb_line_conv.cuh"
#include "rgb_to_uyvy.cuh"
#include "yuv_rgb_conv.cuh"

namespace ugb_logo {

using namespace ugb;

constexpr int kThreads = 128;

long c_div(long a, long b) { return a / b; }  // C truncation toward zero, as logo.c rounds rect_x

// ---- per-codec chunk: codec bytes <-> RGB of P pixels, with the reference's converters ------------------------------
template <int CODEC> struct Chunk;
template <> struct Chunk<UGB_RGB> {  // vc_copylineRGB with the default shifts is memcpy, both ways
        static constexpr int P = 16, IN = 48;
        static __device__ __forceinline__ void decode(const uint32_t *in, uint32_t *rgb, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        rgb[i] = in[i];
                }
        }
        static __device__ __forceinline__ void encode(const uint32_t *rgb, uint32_t *out, const conv_params &, const row_ctx &)
        {
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                        out[i] = rgb[i];
                }
        }
};
template <> struct Chunk<UGB_RGBA> {  // vc_copylineRGBAtoRGB (SSSE3 tail quirk, p.aux) / vc_copylineRGBtoRGBA (alpha 0xFF)
        static constexpr int P = 16, IN = 64;
        static __device__ __forceinline__ void decode(const uint32_t *in, uint32_t *rgb, const conv_params &p, const row_ctx &rc) { conv_rgba_rgb::run(in, rgb, p, rc); }
        static __device__ __forceinline__ void encode(const uint32_t *rgb, uint32_t *out, const conv_params &p, const row_ctx &rc) { conv_rgb_rgba::run(rgb, out, p, rc); }
};
template <> struct Chunk<UGB_UYVY> {  // vc_copylineUYVYtoRGB / vc_copylineRGBtoUYVY
        static constexpr int P = 16, IN = 32;
        static __device__ __forceinline__ void decode(const uint32_t *in, uint32_t *rgb, const conv_params &p, const row_ctx &rc)
        {
                conv_yuv422_rgb<1, 3, 0, 2>::run(in, rgb, p, rc);
        }
        static __device__ __forceinline__ void encode(const uint32_t *rgb, uint32_t *out, const conv_params &p, const row_ctx &rc)
        {
                conv_to_uyvy<0, 1, 2, 3>::run(rgb, out, p, rc);
        }
};
template <> struct Chunk<UGB_RG48> {  // vc_copylineRG48toRGB (high bytes) / vc_copylineRGBtoRG48 (low bytes 0)
        static constexpr int P = 16, IN = 96;
        static __device__ __forceinline__ void decode(const uint32_t *in, uint32_t *rgb, const conv_params &p, const row_ctx &rc)
        {
                conv_bytemap<map_rg48_rgb>::run(in, rgb, p, rc);
        }
        static __device__ __forceinline__ void encode(const uint32_t *rgb, uint32_t *out, const conv_params &p, const row_ctx &rc)
        {
#pragma unroll
                for (int k = 0; k < 3; ++k) {  // the map takes 16 bytes of RGB at a time
                        conv_bytemap<map_rgb_rg48>::run(rgb + 4 * k, out + 8 * k, p, rc);
                }
        }
};
template <> struct Chunk<UGB_R12L> {  // vc_copylineR12LtoRGB / vc_copylineRGBtoR12L (12 -> 8 -> 12 bits)
        static constexpr int P = 32, IN = 144;
        static __device__ __forceinline__ void decode(const uint32_t *in, uint32_t *rgb, const conv_params &p, const row_ctx &rc)
        {
                conv_r12l_rgbx<0>::run(in, rgb, p, rc);
        }
        static __device__ __forceinline__ void encode(const uint32_t *rgb, uint32_t *out, const conv_params &p, const row_ctx &rc)
        {
                conv_x_r12l<0>::run(rgb, out, p, rc);
        }
};

struct LogoArgs {
        uint8_t *frame;     // first byte of the span in the rectangle's first row
        long pitch;         // vc_get_linesize(frame width)
        const uint32_t *logo;  // RGBA, w * h pixels
        int w, h;
        int span;           // vc_get_linesize(w): bytes written per row
        int chunks;         // chunks per row
        conv_params p;      // default shifts; p.aux = the RGBA decoder's first tail pixel
};

template <int NB>
__device__ __forceinline__ void load_bytes(uint32_t *w, const uint8_t *s, int valid, bool vec)
{
        if (vec && valid >= NB) {
#pragma unroll
                for (int i = 0; i < NB / 4; ++i) {
                        w[i] = reinterpret_cast<const uint32_t *>(s)[i];
                }
                return;
        }
#pragma unroll
        for (int i = 0; i < NB / 4; ++i) {
                uint32_t v = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        if (4 * i + k < valid) {
                                v |= (uint32_t) s[4 * i + k] << (8 * k);
                        }
                }
                w[i] = v;
        }
}

template <int NB>
__device__ __forceinline__ void store_bytes(uint8_t *d, const uint32_t *w, int valid, bool vec)
{
        if (vec && valid >= NB) {
#pragma unroll
                for (int i = 0; i < NB / 4; ++i) {
                        reinterpret_cast<uint32_t *>(d)[i] = w[i];
                }
                return;
        }
#pragma unroll
        for (int i = 0; i < NB / 4; ++i) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        if (4 * i + k < valid) {
                                d[4 * i + k] = (uint8_t) (w[i] >> (8 * k));
                        }
                }
        }
}

// byte K of a packed word array, replaced
template <int K> __device__ __forceinline__ void sb(uint32_t *a, uint32_t v)
{
        a[K >> 2] = (a[K >> 2] & ~(0xffu << (8 * (K & 3)))) | (v << (8 * (K & 3)));
}

// logo.c:208-219: (p * (255 - a) + l * a) / 255 in int, over the first w pixels of the row
template <int I, int P>
__device__ __forceinline__ void blend(uint32_t *rgb, const uint32_t *lrow, int px0, int w)
{
        if constexpr (I < P) {
                if (px0 + I < w) {
                        const uint32_t l = __ldg(lrow + px0 + I), a = l >> 24;
                        sb<3 * I>(rgb, (gb<3 * I>(rgb) * (255 - a) + (l & 0xff) * a) / 255);
                        sb<3 * I + 1>(rgb, (gb<3 * I + 1>(rgb) * (255 - a) + ((l >> 8) & 0xff) * a) / 255);
                        sb<3 * I + 2>(rgb, (gb<3 * I + 2>(rgb) * (255 - a) + ((l >> 16) & 0xff) * a) / 255);
                }
                blend<I + 1, P>(rgb, lrow, px0, w);
        }
}

template <int CODEC>
__global__ void __launch_bounds__(kThreads) logo_kernel(LogoArgs a, bool vec)
{
        using C = Chunk<CODEC>;
        constexpr int OUT = C::IN;  // the chunk's codec bytes, read and written back
        const int cx = blockIdx.x * blockDim.x + threadIdx.x;
        if (cx >= a.chunks) {
                return;
        }
        const int b0 = cx * OUT, valid = a.span - b0;
        for (int y = blockIdx.y; y < a.h; y += gridDim.y) {
                uint8_t *row = a.frame + y * a.pitch;
                uint32_t in[OUT / 4], rgb[3 * C::P / 4], out[OUT / 4];
                load_bytes<OUT>(in, row + b0, valid, vec);
                const row_ctx rc = { row, 0, a.span, cx };
                C::decode(in, rgb, a.p, rc);
                blend<0, C::P>(rgb, a.logo + (long) y * a.w, cx * C::P, a.w);
                C::encode(rgb, out, a.p, rc);
                store_bytes<OUT>(row + b0, out, valid, vec);
        }
}

// ---- r12l_to_y416_fake / y416_to_r12l_fake ---------------------------------------------------------------------------
// r12l_to_y416_fake.c:100-113, y416_to_r12l_fake.c:139-158 (full range: << 4 / >> 4; limited: 14 * c + 4096 for R and
// B, 13 * g + 4096 for G, and back with max(v, 4096) - 4096 over 14 / 13, clamped to 4095)
template <bool FULL>
__device__ __forceinline__ uint32_t to16(uint32_t v, int scale)
{
        return FULL ? v << 4 : scale * v + 4096;
}
template <bool FULL>
__device__ __forceinline__ uint32_t to12(uint32_t v, int scale)
{
        return min(FULL ? v >> 4 : (max(v, 4096u) - 4096u) / scale, 4095u);
}

template <bool FULL>
__global__ void __launch_bounds__(256) r12l_to_y416_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, long groups, bool vec)
{
        const long g = (long) blockIdx.x * blockDim.x + threadIdx.x;
        if (g >= groups) {
                return;
        }
        uint32_t in[9], out[16];
        const uint32_t *s = reinterpret_cast<const uint32_t *>(src + 36 * g);
#pragma unroll
        for (int i = 0; i < 9; ++i) {
                in[i] = __ldg(s + i);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
                out[2 * i] = to16<FULL>(r12_get(in, 3 * i), 14) | to16<FULL>(r12_get(in, 3 * i + 1), 13) << 16;
                out[2 * i + 1] = to16<FULL>(r12_get(in, 3 * i + 2), 14) | 0xFFFF0000u;
        }
        uint8_t *d = dst + 64 * g;
        if (vec) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        reinterpret_cast<uint4 *>(d)[i] = make_uint4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
                }
        } else {
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                        reinterpret_cast<uint16_t *>(d)[i] = (uint16_t) (out[i / 2] >> (16 * (i & 1)));
                }
        }
}

template <bool FULL>
__global__ void __launch_bounds__(256) y416_to_r12l_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, long pitch, int row_groups,
                                                           long groups, bool vec_in, bool vec_out)
{
        const long g = (long) blockIdx.x * blockDim.x + threadIdx.x;
        if (g >= groups) {
                return;
        }
        uint32_t in[16], out[9];
        const uint8_t *s = src + 64 * g;
        if (vec_in) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(s) + i);
                        in[4 * i] = v.x, in[4 * i + 1] = v.y, in[4 * i + 2] = v.z, in[4 * i + 3] = v.w;
                }
        } else {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                        in[i] = (uint32_t) __ldg(reinterpret_cast<const uint16_t *>(s) + 2 * i) | (uint32_t) __ldg(reinterpret_cast<const uint16_t *>(s) + 2 * i + 1) << 16;
                }
        }
#pragma unroll
        for (int i = 0; i < 9; ++i) {
                out[i] = 0;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {  // alpha (the high half of word 2i + 1) is dropped
                r12_put(out, 3 * i, to12<FULL>(in[2 * i] & 0xffff, 14));
                r12_put(out, 3 * i + 1, to12<FULL>(in[2 * i] >> 16, 13));
                r12_put(out, 3 * i + 2, to12<FULL>(in[2 * i + 1] & 0xffff, 14));
        }
        const long y = g / row_groups, x = g - y * row_groups;
        uint8_t *d = dst + y * pitch + 36 * x;
        if (vec_out) {
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                        reinterpret_cast<uint32_t *>(d)[i] = out[i];
                }
        } else {
#pragma unroll
                for (int i = 0; i < 36; ++i) {
                        d[i] = (uint8_t) (out[i / 4] >> (8 * (i & 3)));
                }
        }
}

}  // namespace ugb_logo

using namespace ugb_logo;

struct ugb200_cf_logo {
        uint32_t *dev;  // RGBA, width * height pixels
        int width, height;
};
using LogoImage = struct ugb200_cf_logo;  // the struct shares its name with the entry point

extern "C" UGB_API ugb200_cf_logo_t ugb200_cf_logo_create(const unsigned char *rgba, unsigned width, unsigned height)
{
        if (rgba == nullptr || width == 0 || height == 0 || width > INT32_MAX || height > INT32_MAX) {
                return nullptr;
        }
        const size_t bytes = (size_t) width * height * 4;
        auto *l = new (std::nothrow) LogoImage{ nullptr, (int) width, (int) height };
        if (l == nullptr || cudaMalloc(&l->dev, bytes) != cudaSuccess || cudaMemcpy(l->dev, rgba, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
                if (l != nullptr) {
                        cudaFree(l->dev);
                }
                delete l;
                return nullptr;
        }
        return l;
}

extern "C" UGB_API void ugb200_cf_logo_destroy(ugb200_cf_logo_t l)
{
        if (l != nullptr) {
                cudaFree(l->dev);
                delete l;
        }
}

template <int CODEC>
static int launch_logo(const LogoArgs &a, cudaStream_t st)
{
        // 4-byte accesses when every row's span start is 4-byte aligned (chunk sizes are multiples of 4)
        const bool vec = (uintptr_t) a.frame % 4 == 0 && a.pitch % 4 == 0;
        const dim3 grid((a.chunks + kThreads - 1) / kThreads, a.h < 65535 ? a.h : 65535);
        logo_kernel<CODEC><<<grid, kThreads, 0, st>>>(a, vec);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" UGB_API int ugb200_cf_logo(ugb200_cf_logo_t l, int codec, int width, int height, int x, int y, void *frame,
                                      cuda_wrapper_stream_t stream)
{
        if (l == nullptr || frame == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        switch (codec) {
        case UGB_RGB: case UGB_RGBA: case UGB_UYVY: case UGB_RG48: case UGB_R12L: break;
        default: return -4;  // no decoder to or from RGB (get_decoder_from_to() == NULL): logo.c returns its input
        }
        const codec_t c = (codec_t) codec;
        const long bytes = get_pf_block_bytes(c);
        if ((codec == UGB_RG48 && (uintptr_t) frame % 2) || (codec == UGB_R12L && (uintptr_t) frame % 4)) {
                return -1;
        }
        const long w = l->width, h = l->height;
        // logo.c:184-197
        long rect_x = x, rect_y = y;
        if (rect_x < 0 || rect_x + w > width) {
                rect_x = width - w;
        }
        rect_x = c_div(rect_x, bytes) * bytes;  // whole blocks of bytes, counted in pixels
        if (rect_y < 0 || rect_y + h > height) {
                rect_y = height - h;
        }
        if (rect_x < 0 || rect_y < 0) {
                return 0;  // the reference returns its input untouched
        }
        const long pitch = vc_linesize64(width, c), off = vc_linesize64(rect_x, c), span = vc_linesize64(w, c);
        if (off + span > pitch) {
                return -1;  // the reference writes past the row (into the next one, or past the frame)
        }
        LogoArgs a{};
        a.frame = (uint8_t *) frame + rect_y * pitch + off;
        a.pitch = pitch;
        a.logo = l->dev;
        a.w = (int) w;
        a.h = (int) h;
        a.span = (int) span;
        a.p = conv_params{ 0, 8, 16, 0 };
        const cudaStream_t st = (cudaStream_t) stream;
        switch (codec) {
        case UGB_RGB:
                a.chunks = (int) ((w + 15) / 16);
                return launch_logo<UGB_RGB>(a, st);
        case UGB_RGBA:
                // the decoder runs over the padded row, rounded up to whole blocks (DESIGN.md §8): its SSSE3 tail
                // repeats pixel aux for every pixel from aux on
                a.p.aux = conv_rgba_rgb::aux((int) (3 * ((w + 3) / 4 * 4)));
                a.chunks = (int) ((w + 15) / 16);
                return launch_logo<UGB_RGBA>(a, st);
        case UGB_UYVY:
                a.chunks = (int) ((w + 15) / 16);
                return launch_logo<UGB_UYVY>(a, st);
        case UGB_RG48:
                a.chunks = (int) ((w + 15) / 16);
                return launch_logo<UGB_RG48>(a, st);
        default:
                a.chunks = (int) ((w + 31) / 32);
                return launch_logo<UGB_R12L>(a, st);
        }
}

extern "C" UGB_API int ugb200_cf_r12l_to_y416_fake(int width, int height, int full_range, const void *src, void *dst, cuda_wrapper_stream_t stream)
{
        if (src == nullptr || dst == nullptr || width <= 0 || height <= 0 || width % 8 || (uintptr_t) src % 4 || (uintptr_t) dst % 2) {
                return -1;
        }
        const long groups = (long) width / 8 * height;
        if (overlap(src, 36 * groups, dst, 64 * groups)) {
                return -1;
        }
        const bool vec = (uintptr_t) dst % 16 == 0;
        const unsigned blocks = (unsigned) ((groups + 255) / 256);
        if (full_range) {
                r12l_to_y416_kernel<true><<<blocks, 256, 0, (cudaStream_t) stream>>>((const uint8_t *) src, (uint8_t *) dst, groups, vec);
        } else {
                r12l_to_y416_kernel<false><<<blocks, 256, 0, (cudaStream_t) stream>>>((const uint8_t *) src, (uint8_t *) dst, groups, vec);
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" UGB_API int ugb200_pp_y416_to_r12l_fake(int width, int height, int full_range, const void *src, void *dst, size_t pitch,
                                                   cuda_wrapper_stream_t stream)
{
        if (src == nullptr || dst == nullptr || width <= 0 || height <= 0 || width % 8 || (uintptr_t) src % 2 || (uintptr_t) dst % 4) {
                return -1;
        }
        const long row_groups = width / 8, groups = row_groups * height, L = 36 * row_groups;
        if (pitch < (size_t) L || pitch > (size_t) INT32_MAX || overlap(src, 64 * groups, dst, (height - 1) * pitch + L)) {
                return -1;
        }
        const bool vec_in = (uintptr_t) src % 16 == 0, vec_out = pitch % 4 == 0;
        const unsigned blocks = (unsigned) ((groups + 255) / 256);
        if (full_range) {
                y416_to_r12l_kernel<true><<<blocks, 256, 0, (cudaStream_t) stream>>>((const uint8_t *) src, (uint8_t *) dst, (long) pitch, (int) row_groups,
                                                                                      groups, vec_in, vec_out);
        } else {
                y416_to_r12l_kernel<false><<<blocks, 256, 0, (cudaStream_t) stream>>>((const uint8_t *) src, (uint8_t *) dst, (long) pitch, (int) row_groups,
                                                                                       groups, vec_in, vec_out);
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
