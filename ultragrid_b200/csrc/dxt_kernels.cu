// DXT block-compression kernels + their C ABI (drop-in for UltraGrid's cuda_dxt/cuda_dxt.{h,cu}).
//
// Layout in HBM
//   packed-3 sources (RGB / YUV 4:4:4):  w*3 bytes per row, no padding      (cuda_dxt.h:20-29)
//   UYVY source (fused path):           U Y0 V Y1 per pixel pair, `pitch` bytes per row
//   DXT1 output: one uint2 {palette, indices} per 4x4 block, raster block order (cuda_dxt.cu:616,633)
//   DXT5-YCoCg output: one uint4 per block                                   (cuda_dxt.cu:507)
//
// Kernels (one thread encodes one 4x4 block; all HBM-streaming, no tensor cores):
//   dxt_uyvy_kernel<1,2>  thread = two horizontally adjacent blocks, encoded one phase apart: 4 x LDG.128, 1 x STG.128
//   dxt_uyvy_kernel<1,1>  fallback for (w/4) odd or 8-byte-only aligned buffers; dxt_uyvy_kernel<6,1> DXT5-YCoCg
//   dxt_packed3_kernel    cuda_{rgb,yuv}_to_dxt{1,6}: 3 x LDG.32 per row like the reference, but the grid
//                         is sized in blocks (the reference launches 16x more threads, cuda_dxt.cu:750-751)
//   yuv422_to_yuv444_kernel  ABI-compat only; the fused kernels never materialise 4:4:4
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/cuda_dxt.h"
#include "../../include/ugb200.h"
#include "dxt6_device.cuh"
#include "dxt_device.cuh"

namespace ugb {

__device__ __forceinline__ uint4 ld_stream_v4(const void *p)
{
        uint4 r;
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                     : "l"(p));
        return r;
}
__device__ __forceinline__ uint2 ld_stream_v2(const void *p)
{
        uint2 r;
        asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
        return r;
}

template <int DXT_TYPE>
struct block_out;
template <>
struct block_out<1> {
        typedef uint2 type;
};
template <>
struct block_out<6> {
        typedef uint4 type;
};

template <int DXT_TYPE>
__device__ __forceinline__ typename block_out<DXT_TYPE>::type encode_block(const float (&r)[16], const float (&g)[16],
                                                                           const float (&b)[16]);
template <>
__device__ __forceinline__ uint2 encode_block<1>(const float (&r)[16], const float (&g)[16], const float (&b)[16])
{
        return dxt1_encode(r, g, b);
}
template <>
__device__ __forceinline__ uint4 encode_block<6>(const float (&r)[16], const float (&g)[16], const float (&b)[16])
{
        return dxt6_encode(r, g, b);
}

// ------------------------------------------------------------------------------------------------
// fused UYVY -> DXT.  One thread = BPT horizontally adjacent blocks.
// ------------------------------------------------------------------------------------------------
/// CTA shape.  DXT1: 64-thread CTAs, 12 per SM (80 registers, no spill; a block row of an 8K frame is 960 threads, i.e. 15 CTAs of 64 but 7.5
/// of 128).  Measured with tools/exp_dxt.cu on an H100 80GB HBM3 at a 400 W power limit, 8K frames, median of 100 interleaved rounds: the
/// two-block kernel with the skewed encode 56.4 us; the same with (64, 10) 56.6, with (128, 5) 58.0; the unskewed encode 58.4 at (64, 12),
/// 57.4 at (64, 10), 58.9 at (128, 5); one block per thread 61.2; a persistent grid with the next item's rows loaded ahead 62.4 (128 registers
/// leave 16 warps per SM, and the item loop adds integer instructions to an issue-bound kernel).  DXT5-YCoCg: 128-thread CTAs, 7 per SM,
/// chosen on an earlier GPU and not re-measured on the H100.
template <int DXT_TYPE>
struct uyvy_cta {
        static constexpr int threads = DXT_TYPE == 1 ? 64 : 128, min_ctas = DXT_TYPE == 1 ? 12 : 7;
};

template <int DXT_TYPE, int BPT, bool MIRROR>
__global__ void __launch_bounds__(uyvy_cta<DXT_TYPE>::threads, uyvy_cta<DXT_TYPE>::min_ctas) dxt_uyvy_kernel(const uint8_t *__restrict__ src, void *__restrict__ out,
                                                        int wb /* blocks per row */, int h, long pitch)
{
        typedef typename block_out<DXT_TYPE>::type out_t;
        // grid: x over groups of BPT blocks in a block-row, y = block-row (no division, 32-bit index math)
        const int gx = blockIdx.x * blockDim.x + threadIdx.x;
        const int by = blockIdx.y;
        if (gx >= wb / BPT) {
                return;
        }
        const int row0 = MIRROR ? h - 1 - by * 4 : by * 4;  // cuda_dxt.cu:653-655
        const uint8_t *p = src + (long) row0 * pitch + gx * (8 * BPT);
        const long step = MIRROR ? -pitch : pitch;

        uint32_t w[4][2 * BPT];
#pragma unroll
        for (int y = 0; y < 4; ++y, p += step) {
                if (BPT == 2) {
                        const uint4 v = ld_stream_v4(p);
                        w[y][0] = v.x, w[y][1] = v.y, w[y][2] = v.z, w[y][3] = v.w;
                } else {
                        const uint2 v = ld_stream_v2(p);
                        w[y][0] = v.x, w[y][1] = v.y;
                }
        }
        out_t *o = (out_t *) out + ((long) by * wb + gx * BPT);
        if constexpr (DXT_TYPE == 1 && BPT == 2) {  // the two blocks one phase apart (same operation tree per block)
                const uint4 v[4] = { make_uint4(w[0][0], w[0][1], w[0][2], w[0][3]), make_uint4(w[1][0], w[1][1], w[1][2], w[1][3]),
                                     make_uint4(w[2][0], w[2][1], w[2][2], w[2][3]), make_uint4(w[3][0], w[3][1], w[3][2], w[3][3]) };
                *(uint4 *) o = dxt1_encode_uyvy_pair_skewed(v);
        } else {
#pragma unroll
                for (int k = 0; k < BPT; ++k) {
                        if constexpr (DXT_TYPE == 1) {  // paired formulation (same operation tree)
                                const uint32_t wk[4][2] = { { w[0][2 * k], w[0][2 * k + 1] }, { w[1][2 * k], w[1][2 * k + 1] },
                                                            { w[2][2 * k], w[2][2 * k + 1] }, { w[3][2 * k], w[3][2 * k + 1] } };
                                o[k] = dxt1_encode_uyvy_packed(wk);
                        } else {
                                float r[16], g[16], b[16];
#pragma unroll
                                for (int y = 0; y < 4; ++y) {
                                        load_row_uyvy_packed(w[y][2 * k], w[y][2 * k + 1], r + 4 * y, g + 4 * y, b + 4 * y);
                                }
                                o[k] = encode_block<DXT_TYPE>(r, g, b);
                        }
                }
        }
}

// ------------------------------------------------------------------------------------------------
// packed 3-byte source (RGB or YUV 4:4:4), ABI of cuda_dxt.h
// ------------------------------------------------------------------------------------------------
template <bool YUV, bool MIRROR, int DXT_TYPE>
__global__ void __launch_bounds__(128) dxt_packed3_kernel(const uint32_t *__restrict__ src, void *__restrict__ out,
                                                           int wb, int h)
{
        typedef typename block_out<DXT_TYPE>::type out_t;
        const int bx = blockIdx.x * blockDim.x + threadIdx.x;
        const int by = blockIdx.y;
        if (bx >= wb) {
                return;
        }
        const int stride_w = wb * 3;  // 32-bit words per row (cuda_dxt.cu:646)
        const int row0 = MIRROR ? h - 1 - by * 4 : by * 4;
        const uint32_t *p = src + ((long) stride_w * row0 + bx * 3);
        const int step = MIRROR ? -stride_w : stride_w;
        float r[16], g[16], b[16];
#pragma unroll
        for (int y = 0; y < 4; ++y, p += step) {
                load_row_packed3<YUV>(__ldg(p), __ldg(p + 1), __ldg(p + 2), r + 4 * y, g + 4 * y, b + 4 * y);
        }
        ((out_t *) out)[(long) by * wb + bx] = encode_block<DXT_TYPE>(r, g, b);
}

/// DXT1 from a packed 3-byte source, two horizontally adjacent blocks per thread: 3 x LDG.64 per row (24 contiguous bytes, 8-byte aligned when
/// the block row starts 16-byte aligned and the thread's first block index is even) instead of 2 x 3 LDG.32 at a 12-byte stride, the packed
/// (paired) encode, one 16-byte store.
template <bool YUV, bool MIRROR>
__global__ void __launch_bounds__(64, 12) dxt1_packed3_pair_kernel(const uint8_t *__restrict__ src, void *__restrict__ out, int wb, int h)
{
        const int gx = blockIdx.x * blockDim.x + threadIdx.x;  // pair index within the block row
        const int by = blockIdx.y;
        if (gx >= wb / 2) {
                return;
        }
        const long pitch = (long) wb * 12;
        const int row0 = MIRROR ? h - 1 - by * 4 : by * 4;
        const uint8_t *p = src + (long) row0 * pitch + (long) gx * 24;
        const long step = MIRROR ? -pitch : pitch;
        uint32_t wa[4][3], wb2[4][3];
#pragma unroll
        for (int y = 0; y < 4; ++y, p += step) {
                const uint2 q0 = ld_stream_v2(p), q1 = ld_stream_v2(p + 8), q2 = ld_stream_v2(p + 16);
                wa[y][0] = q0.x, wa[y][1] = q0.y, wa[y][2] = q1.x;
                wb2[y][0] = q1.y, wb2[y][1] = q2.x, wb2[y][2] = q2.y;
        }
        const uint2 ra = dxt1_encode_packed3<YUV>(wa), rb = dxt1_encode_packed3<YUV>(wb2);
        *((uint4 *) out + ((long) by * (wb / 2) + gx)) = make_uint4(ra.x, ra.y, rb.x, rb.y);
}

/// UYVY -> packed Y,U,V 4:4:4 with chroma replication (cuda_dxt.cu:697-732). 16 px per thread:
/// 2 x LDG.128 in, 3 x STG.128 out.
__global__ void __launch_bounds__(256) yuv422_to_yuv444_kernel(const uint4 *__restrict__ src, uint4 *__restrict__ out,
                                                                long groups16)
{
        const long gid = (long) blockIdx.x * blockDim.x + threadIdx.x;
        if (gid >= groups16) {
                return;
        }
        const uint4 a = ld_stream_v4(src + 2 * gid), c = ld_stream_v4(src + 2 * gid + 1);
        const uint32_t in[8] = { a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w };
        uint32_t o[12];
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // two words (4 px: U0 Y0 V0 Y1 | U1 Y2 V1 Y3) -> three words
                const uint32_t p = in[2 * k], q = in[2 * k + 1];
                o[3 * k + 0] = __byte_perm(p, 0, 0x3201);  // Y0 U0 V0 Y1
                o[3 * k + 1] = __byte_perm(p, q, 0x4520);  // U0 V0 Y2 U1
                o[3 * k + 2] = __byte_perm(q, 0, 0x2032);  // V1 Y3 U1 V1
        }
        out[3 * gid + 0] = make_uint4(o[0], o[1], o[2], o[3]);
        out[3 * gid + 1] = make_uint4(o[4], o[5], o[6], o[7]);
        out[3 * gid + 2] = make_uint4(o[8], o[9], o[10], o[11]);
}

/// scalar tail / unaligned fallback: 4 px per thread exactly like the reference
__global__ void yuv422_to_yuv444_tail_kernel(const uint32_t *__restrict__ src, uint32_t *__restrict__ out, long first4,
                                             long groups4)
{
        const long gid = first4 + (long) blockIdx.x * blockDim.x + threadIdx.x;
        if (gid >= groups4) {
                return;
        }
        const uint32_t p = src[2 * gid], q = src[2 * gid + 1];
        out[3 * gid + 0] = __byte_perm(p, 0, 0x3201);
        out[3 * gid + 1] = __byte_perm(p, q, 0x4520);
        out[3 * gid + 2] = __byte_perm(q, 0, 0x2032);
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
template <bool YUV, int DXT_TYPE>
static int launch_packed3(const void *src, void *out, int sx, int sy, cudaStream_t str, bool sync)
{
        bool mirrored = false;
        if (sy < 0) {  // cuda_dxt.cu:739-742
                mirrored = true;
                sy = -sy;
        }
        if ((sx & 3) || (sy & 3) || (15 & (size_t) src) || (7 & (size_t) out) || (DXT_TYPE == 6 && (15 & (size_t) out))) {
                return -1;  // cuda_dxt.cu:745-747 (a uint4 store additionally needs 16-B alignment)
        }
        const int wb = sx / 4, hb = sy / 4;
        if (hb > 65535) {
                return -1;
        }
        if (DXT_TYPE == 1 && wb > 0 && hb > 0 && !(wb & 1) && !(15 & (size_t) out)) {  // pairs of blocks: 8-byte aligned rows of 24-byte pieces
                const dim3 grid((wb / 2 + 63) / 64, hb);
                if (mirrored) {
                        dxt1_packed3_pair_kernel<YUV, true><<<grid, 64, 0, str>>>((const uint8_t *) src, out, wb, sy);
                } else {
                        dxt1_packed3_pair_kernel<YUV, false><<<grid, 64, 0, str>>>((const uint8_t *) src, out, wb, sy);
                }
                if (cudaGetLastError() != cudaSuccess) {
                        return -2;
                }
        } else if (wb > 0 && hb > 0) {
                const int threads = 128;
                const dim3 grid((wb + threads - 1) / threads, hb);
                if (mirrored) {
                        dxt_packed3_kernel<YUV, true, DXT_TYPE><<<grid, threads, 0, str>>>((const uint32_t *) src, out, wb, sy);
                } else {
                        dxt_packed3_kernel<YUV, false, DXT_TYPE><<<grid, threads, 0, str>>>((const uint32_t *) src, out, wb, sy);
                }
                if (cudaGetLastError() != cudaSuccess) {
                        return -2;
                }
        }
        if (sync) {
                return cudaSuccess != cudaStreamSynchronize(str) ? -3 : 0;  // cuda_dxt.cu:759
        }
        return 0;
}

template <int DXT_TYPE>
static int launch_uyvy(const void *src, void *out, int sx, int sy, long pitch, cudaStream_t str)
{
        bool mirrored = false;
        if (sy < 0) {
                mirrored = true;
                sy = -sy;
        }
        if (pitch == 0) {
                pitch = (long) sx * 2;
        }
        const size_t out_align = DXT_TYPE == 6 ? 15 : 7;
        if ((sx & 3) || (sy & 3) || (7 & (size_t) src) || (out_align & (size_t) out) || (pitch & 7) || pitch < (long) sx * 2) {
                return -1;
        }
        const int wb = sx / 4, hb = sy / 4;
        if (wb == 0 || hb == 0) {
                return 0;
        }
        const int threads = uyvy_cta<DXT_TYPE>::threads;
        // DXT5-YCoCg: one block per thread — two unrolled blocks (~50 KB of SASS) overflow the instruction cache (ncu: the top stall
        // was no_instruction); DXT1: two blocks per thread for 128-bit loads/stores
        const bool pair = DXT_TYPE == 1 && !(wb & 1) && !(15 & (size_t) src) && !(pitch & 15) && !(15 & (size_t) out);
        if (hb > 65535) {
                return -1;
        }
        const int groups = pair ? wb / 2 : wb;
        const dim3 grid((groups + threads - 1) / threads, hb);
        const uint8_t *s = (const uint8_t *) src;
#define UGB_LAUNCH(BPT, MIR) dxt_uyvy_kernel<DXT_TYPE, BPT, MIR><<<grid, threads, 0, str>>>(s, out, wb, sy, pitch)
        if (DXT_TYPE == 1 && pair) {
                if constexpr (DXT_TYPE == 1) {  // (the two-block variant is not even instantiated for DXT5-YCoCg)
                        if (mirrored) {
                                UGB_LAUNCH(2, true);
                        } else {
                                UGB_LAUNCH(2, false);
                        }
                }
        } else {
                if (mirrored) {
                        UGB_LAUNCH(1, true);
                } else {
                        UGB_LAUNCH(1, false);
                }
        }
#undef UGB_LAUNCH
        return cudaGetLastError() != cudaSuccess ? -2 : 0;
}

}  // namespace ugb

// ------------------------------------------------------------------------------------------------
// C ABI — same symbols, argument meaning and return codes as cuda_dxt/cuda_dxt.h:30-89
// ------------------------------------------------------------------------------------------------
extern "C" {

int cuda_rgb_to_dxt1(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<false, 1>(src, out, size_x, size_y, (cudaStream_t) stream, true);
}
int cuda_yuv_to_dxt1(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<true, 1>(src, out, size_x, size_y, (cudaStream_t) stream, true);
}
int cuda_rgb_to_dxt6(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<false, 6>(src, out, size_x, size_y, (cudaStream_t) stream, true);
}
int cuda_yuv_to_dxt6(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<true, 6>(src, out, size_x, size_y, (cudaStream_t) stream, true);
}

int cuda_yuv422_to_yuv444(const void *src, void *out, int pix_count, cuda_wrapper_stream_t str)
{
        cudaStream_t s = (cudaStream_t) str;
        if (pix_count < 0 || (3 & (size_t) src) || (3 & (size_t) out)) {
                return -1;
        }
        const long groups4 = pix_count / 4;  // cuda_dxt.cu:766 — 4 px per unit of work
        long done4 = 0;
        if (!(15 & (size_t) src) && !(15 & (size_t) out)) {
                const long groups16 = groups4 / 4;
                if (groups16 > 0) {
                        ugb::yuv422_to_yuv444_kernel<<<(unsigned) ((groups16 + 255) / 256), 256, 0, s>>>(
                            (const uint4 *) src, (uint4 *) out, groups16);
                }
                done4 = groups16 * 4;
        }
        if (done4 < groups4) {
                const long rest = groups4 - done4;
                ugb::yuv422_to_yuv444_tail_kernel<<<(unsigned) ((rest + 255) / 256), 256, 0, s>>>(
                    (const uint32_t *) src, (uint32_t *) out, done4, groups4);
        }
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        return cudaSuccess != cudaStreamSynchronize(s) ? -3 : 0;  // cuda_dxt.cu:769
}

// ---- additions of this library: asynchronous (no stream sync) and fused entry points ------------------------
int ugb200_rgb_to_dxt1_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<false, 1>(src, out, size_x, size_y, (cudaStream_t) stream, false);
}
int ugb200_yuv_to_dxt1_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<true, 1>(src, out, size_x, size_y, (cudaStream_t) stream, false);
}
int ugb200_rgb_to_dxt6_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<false, 6>(src, out, size_x, size_y, (cudaStream_t) stream, false);
}
int ugb200_yuv_to_dxt6_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream)
{
        return ugb::launch_packed3<true, 6>(src, out, size_x, size_y, (cudaStream_t) stream, false);
}
int ugb200_uyvy_to_dxt1_async(const void *src, void *out, int size_x, int size_y, long src_pitch,
                              cuda_wrapper_stream_t stream)
{
        return ugb::launch_uyvy<1>(src, out, size_x, size_y, src_pitch, (cudaStream_t) stream);
}
int ugb200_uyvy_to_dxt6_async(const void *src, void *out, int size_x, int size_y, long src_pitch,
                              cuda_wrapper_stream_t stream)
{
        return ugb::launch_uyvy<6>(src, out, size_x, size_y, src_pitch, (cudaStream_t) stream);
}

}  // extern "C"
