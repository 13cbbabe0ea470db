// Colour capture filters on the device: gamma, matrix, matrix2 and grayscale (src/capture_filter/gamma.cpp,
// matrix.c, matrix2.c, grayscale.c).  Arithmetic contract: DESIGN.md §2 "Colour filters"; differences: §8.
//
//   Every filter treats the frame as one flat stream, as the reference does, so each is a map from fixed-size input
//   chunks to fixed-size output chunks.  One thread takes one chunk: 16-byte (or 8-byte) vector loads and stores
//   when both buffers are aligned for them, byte loads and stores otherwise and for the partial chunk at the end.
//
//   double -> integer follows x86's cvttsd2si with a 32-bit destination, which is what the reference's conversions
//   compile to: truncation toward zero, INT_MIN for NaN and anything outside int32, then the low 8 or 16 bits.
//   FP64 sums are __dmul_rn / __dadd_rn in the reference's left-to-right order, so nothing is contracted to an FMA.
//
//   gamma's four tables are built on the host with the C library's pow (the device pow is not glibc's) and the same
//   conversion, then gathered through L1 (the 64 KB 16->8 table from shared memory by a persistent grid; DESIGN.md §4.4).
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <new>

#include "../../include/ugb200.h"

namespace ugb_cf {

constexpr int kThreads = 256;

// ---- chunk words: loads, stores and sample access ---------------------------------------------------------------
template <int NB> constexpr int vec_bytes() { return NB % 16 == 0 ? 16 : NB % 8 == 0 ? 8 : 4; }

template <int NB> __device__ __forceinline__ void load_vec(const uint8_t *p, uint32_t *w)
{
        if constexpr (vec_bytes<NB>() == 16) {
#pragma unroll
                for (int i = 0; i < NB / 16; ++i) {
                        const uint4 v = reinterpret_cast<const uint4 *>(p)[i];
                        w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
                }
        } else if constexpr (vec_bytes<NB>() == 8) {
#pragma unroll
                for (int i = 0; i < NB / 8; ++i) {
                        const uint2 v = reinterpret_cast<const uint2 *>(p)[i];
                        w[2 * i] = v.x, w[2 * i + 1] = v.y;
                }
        } else {
#pragma unroll
                for (int i = 0; i < NB / 4; ++i) {
                        w[i] = reinterpret_cast<const uint32_t *>(p)[i];
                }
        }
}

template <int NB> __device__ __forceinline__ void store_vec(uint8_t *p, const uint32_t *w)
{
        if constexpr (vec_bytes<NB>() == 16) {
#pragma unroll
                for (int i = 0; i < NB / 16; ++i) {
                        reinterpret_cast<uint4 *>(p)[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
                }
        } else if constexpr (vec_bytes<NB>() == 8) {
#pragma unroll
                for (int i = 0; i < NB / 8; ++i) {
                        reinterpret_cast<uint2 *>(p)[i] = make_uint2(w[2 * i], w[2 * i + 1]);
                }
        } else {
#pragma unroll
                for (int i = 0; i < NB / 4; ++i) {
                        reinterpret_cast<uint32_t *>(p)[i] = w[i];
                }
        }
}

// bytes [0, n) of the chunk; the rest of w stays 0 (w is zeroed by the caller)
template <int NB> __device__ __forceinline__ void load_bytes(const uint8_t *p, long n, uint32_t *w)
{
#pragma unroll
        for (int j = 0; j < NB; ++j) {
                if (j < n) {
                        w[j >> 2] |= uint32_t(p[j]) << (8 * (j & 3));
                }
        }
}

template <int NB> __device__ __forceinline__ void store_bytes(uint8_t *p, long n, const uint32_t *w)
{
#pragma unroll
        for (int j = 0; j < NB; ++j) {
                if (j < n) {
                        p[j] = uint8_t(w[j >> 2] >> (8 * (j & 3)));
                }
        }
}

__device__ __forceinline__ uint32_t b8(const uint32_t *w, int j) { return (w[j >> 2] >> (8 * (j & 3))) & 0xffu; }
__device__ __forceinline__ uint32_t h16(const uint32_t *w, int j) { return (w[j >> 1] >> (16 * (j & 1))) & 0xffffu; }
__device__ __forceinline__ void put8(uint32_t *w, int j, uint32_t v) { w[j >> 2] |= (v & 0xffu) << (8 * (j & 3)); }
__device__ __forceinline__ void put16(uint32_t *w, int j, uint32_t v) { w[j >> 1] |= (v & 0xffffu) << (16 * (j & 1)); }

// ---- the reference's double -> integer conversion ----------------------------------------------------------------
// cvttsd2si into a 32-bit register: truncation toward zero; NaN and values outside int32 give INT_MIN.
// (__double2int_rz saturates instead, so the out-of-range path is explicit.)
__device__ __forceinline__ int x86_i32(double v)
{
        return (v > -2147483649.0 && v < 2147483648.0) ? __double2int_rz(v) : INT_MIN;
}

template <bool BOUND> __device__ __forceinline__ uint32_t conv(double v)
{
        const int i = x86_i32(v);
        return BOUND ? uint32_t(min(max(i, 0), 255)) : uint32_t(i);  // put8 / put16 keep the low bits
}

struct Mat {
        double m[9];
};

// (m[r] * a0 + m[r+1] * a1) + m[r+2] * a2, no contraction
__device__ __forceinline__ double dot3(const Mat &M, int r, double a0, double a1, double a2)
{
        return __dadd_rn(__dadd_rn(__dmul_rn(M.m[r], a0), __dmul_rn(M.m[r + 1], a1)), __dmul_rn(M.m[r + 2], a2));
}

// ((off + m[r] * a0) + m[r+1] * a1) + m[r+2] * a2: matrix2's rows
__device__ __forceinline__ double off_dot3(const Mat &M, int r, double off, double a0, double a1, double a2)
{
        return __dadd_rn(__dadd_rn(__dadd_rn(off, __dmul_rn(M.m[r], a0)), __dmul_rn(M.m[r + 1], a1)), __dmul_rn(M.m[r + 2], a2));
}

// ---- the filters as chunk maps -----------------------------------------------------------------------------------
// matrix.c:137-168 / 228-253: UYVY (U Y0 V Y1) -> two RGB pixels from (Y0 - 16, U - 128, V - 128), (Y1 - 16, ...)
template <bool BOUND> struct MatrixUYVY {
        static constexpr int IN = 16, OUT = 24;
        Mat M;
        __device__ void operator()(const uint32_t *in, uint32_t *out) const
        {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        const double u = int(b8(in, 4 * k)) - 128, v = int(b8(in, 4 * k + 2)) - 128;
#pragma unroll
                        for (int p = 0; p < 2; ++p) {
                                const double y = int(b8(in, 4 * k + 1 + 2 * p)) - 16;
#pragma unroll
                                for (int r = 0; r < 3; ++r) {
                                        put8(out, 6 * k + 3 * p + r, conv<BOUND>(dot3(M, 3 * r, y, u, v)));
                                }
                        }
                }
        }
};

// matrix.c:169-186 / 254-270 (8-bit) and :187-204 / 271-287 (RG48, clamped at 255 with bounds checking)
template <bool BOUND, bool WIDE> struct MatrixRGB {
        static constexpr int IN = 48, OUT = 48, N = WIDE ? 8 : 16;
        Mat M;
        __device__ void operator()(const uint32_t *in, uint32_t *out) const
        {
#pragma unroll
                for (int k = 0; k < N; ++k) {
                        double a[3];
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                                a[c] = WIDE ? h16(in, 3 * k + c) : b8(in, 3 * k + c);
                        }
#pragma unroll
                        for (int r = 0; r < 3; ++r) {
                                const uint32_t o = conv<BOUND>(dot3(M, 3 * r, a[0], a[1], a[2]));
                                if (WIDE) {
                                        put16(out, 3 * k + r, o);
                                } else {
                                        put8(out, 3 * k + r, o);
                                }
                        }
                }
        }
};

// matrix2.c:162-191 (apply_to_uyvy): chroma rows take y = (y1 + y2) / 2
struct Matrix2UYVY {
        static constexpr int IN = 16, OUT = 16;
        Mat M;
        __device__ void operator()(const uint32_t *in, uint32_t *out) const
        {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                        const double u = int(b8(in, 4 * k)) - 128, y1 = int(b8(in, 4 * k + 1)) - 16;
                        const double v = int(b8(in, 4 * k + 2)) - 128, y2 = int(b8(in, 4 * k + 3)) - 16;
                        const double y = __dmul_rn(__dadd_rn(y1, y2), 0.5);
                        put8(out, 4 * k, conv<false>(off_dot3(M, 3, 128., y, u, v)));
                        put8(out, 4 * k + 1, conv<false>(off_dot3(M, 0, 16., y1, u, v)));
                        put8(out, 4 * k + 2, conv<false>(off_dot3(M, 6, 128., y, u, v)));
                        put8(out, 4 * k + 3, conv<false>(off_dot3(M, 0, 16., y2, u, v)));
                }
        }
};

// matrix2.c:209-230 on one Y416 pixel (U Y V A): returns U', Y', V' as 16-bit values
__device__ __forceinline__ void y416_pixel(const Mat &M, uint32_t U, uint32_t Y, uint32_t V, uint32_t &u_, uint32_t &y_, uint32_t &v_)
{
        const double u = int(U) - (1 << 15), y = int(Y) - (1 << 12), v = int(V) - (1 << 15);
        u_ = conv<false>(off_dot3(M, 3, 32768., y, u, v)) & 0xffffu;
        y_ = conv<false>(off_dot3(M, 0, 4096., y, u, v)) & 0xffffu;
        v_ = conv<false>(off_dot3(M, 6, 32768., y, u, v)) & 0xffffu;
}

// matrix2 on Y416 (vc_memcpy in and out): per pixel, A = 0xFFFF
struct Matrix2Y416 {
        static constexpr int IN = 16, OUT = 16;
        Mat M;
        __device__ void operator()(const uint32_t *in, uint32_t *out) const
        {
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                        uint32_t u, y, v;
                        y416_pixel(M, h16(in, 4 * k), h16(in, 4 * k + 1), h16(in, 4 * k + 2), u, y, v);
                        out[2 * k] = u | y << 16;
                        out[2 * k + 1] = v | 0xffff0000u;
                }
        }
};

// matrix2 on v210, fused: vc_copylineV210toY416 (pixfmt_conv.c:2834-2882) -> the Y416 matrix ->
// vc_copylineY416toV210 (:3004-3031: chroma of a pixel pair averaged, then >> 6).  Group x of the output is a
// function of group x of the input only.
struct Matrix2V210 {
        static constexpr int IN = 16, OUT = 16;
        Mat M;
        __device__ void operator()(const uint32_t *in, uint32_t *out) const
        {
                const uint32_t f[12] = { in[0] & 0x3ffu, in[0] >> 10 & 0x3ffu, in[0] >> 20 & 0x3ffu,
                                         in[1] & 0x3ffu, in[1] >> 10 & 0x3ffu, in[1] >> 20 & 0x3ffu,
                                         in[2] & 0x3ffu, in[2] >> 10 & 0x3ffu, in[2] >> 20 & 0x3ffu,
                                         in[3] & 0x3ffu, in[3] >> 10 & 0x3ffu, in[3] >> 20 & 0x3ffu };
                // pixel pairs (0,1), (2,3), (4,5): chroma (Cb, Cr) and the two lumas, as field indices of f
                const int cb[3] = { 0, 4, 8 }, cr[3] = { 2, 6, 10 }, ya[3] = { 1, 5, 9 }, yb[3] = { 3, 7, 11 };
                uint32_t U[3], V[3], Y[6];
#pragma unroll
                for (int p = 0; p < 3; ++p) {
                        uint32_t u0, v0, u1, v1;
                        y416_pixel(M, f[cb[p]] << 6, f[ya[p]] << 6, f[cr[p]] << 6, u0, Y[2 * p], v0);
                        y416_pixel(M, f[cb[p]] << 6, f[yb[p]] << 6, f[cr[p]] << 6, u1, Y[2 * p + 1], v1);
                        U[p] = (u0 + u1) / 2;
                        V[p] = (v0 + v1) / 2;
                }
                out[0] = U[0] >> 6 | Y[0] >> 6 << 10 | V[0] >> 6 << 20;
                out[1] = Y[1] >> 6 | U[1] >> 6 << 10 | Y[2] >> 6 << 20;
                out[2] = V[1] >> 6 | Y[3] >> 6 << 10 | U[2] >> 6 << 20;
                out[3] = Y[4] >> 6 | V[2] >> 6 << 10 | Y[5] >> 6 << 20;
        }
};

// grayscale.c:86-90: U and V become 127, Y is copied
struct Grayscale {
        static constexpr int IN = 16, OUT = 16;
        __device__ void operator()(const uint32_t *in, uint32_t *out) const
        {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                        out[i] = (in[i] & 0xff00ff00u) | 0x007f007fu;
                }
        }
};

// one thread per chunk: bytes [i0, i0 + IN) of src -> bytes [o0, o0 + OUT) of dst, clipped to in_len / out_len
template <class Op>
__global__ void __launch_bounds__(kThreads) stream_kernel(Op op, const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, long in_len,
                                                          long out_len, long chunks, bool vec)
{
        const long c = long(blockIdx.x) * blockDim.x + threadIdx.x;
        if (c >= chunks) {
                return;
        }
        const long i0 = c * Op::IN, o0 = c * Op::OUT;
        uint32_t in[Op::IN / 4] = {}, out[Op::OUT / 4] = {};
        const bool full = vec && i0 + Op::IN <= in_len && o0 + Op::OUT <= out_len;
        if (full) {
                load_vec<Op::IN>(src + i0, in);
        } else {
                load_bytes<Op::IN>(src + i0, in_len - i0, in);
        }
        op(in, out);
        if (full) {
                store_vec<Op::OUT>(dst + o0, out);
        } else if (o0 < out_len) {
                store_bytes<Op::OUT>(dst + o0, out_len - o0, out);
        }
}

bool overlap(const void *a, size_t na, const void *b, size_t nb)
{
        const uintptr_t x = (uintptr_t) a, y = (uintptr_t) b;
        return x < y + nb && y < x + na;
}

template <class Op> int launch(const Op &op, const void *src, size_t in_len, void *dst, size_t out_len, cudaStream_t st)
{
        const long chunks = long((in_len + Op::IN - 1) / Op::IN);
        const bool vec = (uintptr_t) src % vec_bytes<Op::IN>() == 0 && (uintptr_t) dst % vec_bytes<Op::OUT>() == 0;
        stream_kernel<Op><<<unsigned((chunks + kThreads - 1) / kThreads), kThreads, 0, st>>>(op, (const uint8_t *) src, (uint8_t *) dst,
                                                                                           long(in_len), long(out_len), chunks, vec);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

size_t frame_len(int codec, int width, int height)
{
        const size_t w = (size_t) width, h = (size_t) height;
        switch (codec) {
        case UGB_UYVY: return (w + 1) / 2 * 4 * h;
        case UGB_RGB: return w * 3 * h;
        case UGB_RG48: return w * 6 * h;
        case UGB_Y416: return w * 8 * h;
        case UGB_v210: return (w + 47) / 48 * 128 * h;
        default: return 0;
        }
}

// ---- gamma -------------------------------------------------------------------------------------------------------
// gamma.cpp:96-104: one chunk is 16 bytes of input; the table is staged in shared memory (SMEM) or read through L1
template <typename InT, typename OutT, bool SMEM>
__global__ void __launch_bounds__(1024) gamma_kernel(const OutT *__restrict__ lut, const uint8_t *__restrict__ src, uint8_t *__restrict__ dst,
                                                         long in_len, long out_len, long chunks, bool vec)
{
        constexpr int S = 16 / sizeof(InT), IN = 16, OUT = S * sizeof(OutT);
        constexpr int ENTRIES = 1 << (8 * sizeof(InT));
        extern __shared__ uint4 smem[];
        const OutT *t = lut;
        if (SMEM) {
                constexpr int V = ENTRIES * sizeof(OutT) / 16;
                for (int i = threadIdx.x; i < V; i += blockDim.x) {
                        smem[i] = reinterpret_cast<const uint4 *>(lut)[i];
                }
                __syncthreads();
                t = reinterpret_cast<const OutT *>(smem);
        }
        for (long c = long(blockIdx.x) * blockDim.x + threadIdx.x; c < chunks; c += long(gridDim.x) * blockDim.x) {
                const long i0 = c * IN, o0 = c * OUT;
                uint32_t in[IN / 4] = {}, out[OUT / 4] = {};
                const bool full = vec && i0 + IN <= in_len && o0 + OUT <= out_len;
                if (full) {
                        load_vec<IN>(src + i0, in);
                } else {
                        load_bytes<IN>(src + i0, in_len - i0, in);
                }
#pragma unroll
                for (int k = 0; k < S; ++k) {
                        const uint32_t idx = sizeof(InT) == 1 ? b8(in, k) : h16(in, k);
                        const uint32_t v = SMEM ? t[idx] : __ldg(t + idx);
                        if (sizeof(OutT) == 1) {
                                put8(out, k, v);
                        } else {
                                put16(out, k, v);
                        }
                }
                if (full) {
                        store_vec<OUT>(dst + o0, out);
                } else if (o0 < out_len) {
                        store_bytes<OUT>(dst + o0, out_len - o0, out);
                }
        }
}

template <typename InT, typename OutT, bool SMEM>
int launch_gamma(const OutT *lut, const void *src, size_t in_len, void *dst, size_t out_len, cudaStream_t st)
{
        constexpr int IN = 16, OUT = 16 / sizeof(InT) * sizeof(OutT);
        const long chunks = long((in_len + IN - 1) / IN);
        const bool vec = (uintptr_t) src % 16 == 0 && (uintptr_t) dst % vec_bytes<OUT>() == 0;
        auto *k = gamma_kernel<InT, OutT, SMEM>;
        long grid = (chunks + kThreads - 1) / kThreads;
        size_t smem = 0;
        if (SMEM) {
                // a persistent grid: each CTA stages the table once and strides over the frame
                smem = (size_t(1) << (8 * sizeof(InT))) * sizeof(OutT);
                int dev = 0, sms = 0, per_sm = 0;
                if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
                    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess ||
                    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kThreads, smem) != cudaSuccess || per_sm == 0) {
                        return -2;
                }
                grid = grid < long(sms) * per_sm ? grid : long(sms) * per_sm;
        }
        k<<<unsigned(grid > 0 ? grid : 1), kThreads, smem, st>>>(lut, (const uint8_t *) src, (uint8_t *) dst, long(in_len), long(out_len), chunks, vec);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// gamma.cpp:71-91: pow(i / max_in, g) * max_out into vector<uint8_t / uint16_t>, i.e. x86's conversion, low bits
int host_x86_i32(double v)
{
        return (v > -2147483649.0 && v < 2147483648.0) ? (int) v : INT_MIN;
}

template <typename T> void build_table(T *t, int entries, double max_in, double max_out, double g)
{
        for (int i = 0; i < entries; ++i) {
                t[i] = (T) (unsigned) host_x86_i32(pow((double) i / max_in, g) * max_out);
        }
}

}  // namespace ugb_cf

using namespace ugb_cf;

// one device allocation: lut16 (64K x u16), lut16_8 (64K x u8), lut8_16 (256 x u16), lut8 (256 x u8), 16-byte aligned
struct ugb200_cf_gamma {
        uint8_t *dev;
        const uint16_t *lut16() const { return (const uint16_t *) dev; }
        const uint8_t *lut16_8() const { return dev + 131072; }
        const uint16_t *lut8_16() const { return (const uint16_t *) (dev + 131072 + 65536); }
        const uint8_t *lut8() const { return dev + 131072 + 65536 + 512; }
};

using GammaTables = struct ugb200_cf_gamma;  // the struct shares its name with the entry point
static constexpr size_t kGammaBytes = 131072 + 65536 + 512 + 256;

extern "C" UGB_API ugb200_cf_gamma_t ugb200_cf_gamma_create(double gamma)
{
        static_assert(kGammaBytes % 16 == 0, "tables stay 16-byte aligned");
        uint8_t *host = new (std::nothrow) uint8_t[kGammaBytes];
        if (host == nullptr) {
                return nullptr;
        }
        build_table((uint16_t *) host, 65536, 65535., 65535., gamma);
        build_table(host + 131072, 65536, 65535., 255., gamma);
        build_table((uint16_t *) (host + 131072 + 65536), 256, 255., 65535., gamma);
        build_table(host + 131072 + 65536 + 512, 256, 255., 255., gamma);
        auto *g = new (std::nothrow) GammaTables{ nullptr };
        if (g == nullptr || cudaMalloc(&g->dev, kGammaBytes) != cudaSuccess || cudaMemcpy(g->dev, host, kGammaBytes, cudaMemcpyHostToDevice) != cudaSuccess) {
                if (g != nullptr) {
                        cudaFree(g->dev);
                }
                delete g;
                delete[] host;
                return nullptr;
        }
        delete[] host;
        return g;
}

extern "C" UGB_API void ugb200_cf_gamma_destroy(ugb200_cf_gamma_t g)
{
        if (g != nullptr) {
                cudaFree(g->dev);
                delete g;
        }
}

extern "C" UGB_API int ugb200_cf_gamma(ugb200_cf_gamma_t g, int codec, int out_depth, int width, int height, const void *src, void *dst,
                                       cuda_wrapper_stream_t stream)
{
        if (g == nullptr || src == nullptr || dst == nullptr || width <= 0 || height <= 0 || (out_depth != 0 && out_depth != 8 && out_depth != 16)) {
                return -1;
        }
        if (codec != UGB_RGB && codec != UGB_RG48) {
                return -4;
        }
        const int in_bits = codec == UGB_RGB ? 8 : 16, out_bits = out_depth == 0 ? in_bits : out_depth;
        const size_t in_len = frame_len(codec, width, height), samples = in_len / (in_bits / 8), out_len = samples * (out_bits / 8);
        if ((in_bits == 16 && (uintptr_t) src % 2) || (out_bits == 16 && (uintptr_t) dst % 2) || overlap(src, in_len, dst, out_len)) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        // where each table lives was measured (DESIGN.md §4.4): L1-cached global loads, except 16->8 from shared memory
        if (in_bits == 8) {
                return out_bits == 8 ? launch_gamma<uint8_t, uint8_t, false>(g->lut8(), src, in_len, dst, out_len, st)
                                     : launch_gamma<uint8_t, uint16_t, false>(g->lut8_16(), src, in_len, dst, out_len, st);
        }
        return out_bits == 8 ? launch_gamma<uint16_t, uint8_t, true>(g->lut16_8(), src, in_len, dst, out_len, st)
                             : launch_gamma<uint16_t, uint16_t, false>(g->lut16(), src, in_len, dst, out_len, st);
}

extern "C" UGB_API int ugb200_cf_matrix(int codec, int width, int height, const double m[9], int check_bounds, const void *src, void *dst,
                                        cuda_wrapper_stream_t stream)
{
        if (m == nullptr || src == nullptr || dst == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        if (codec != UGB_UYVY && codec != UGB_RGB && codec != UGB_RG48) {
                return -4;
        }
        Mat M;
        memcpy(M.m, m, sizeof M.m);
        const size_t in_len = frame_len(codec, width, height);
        // UYVY -> RGB: the reference writes 6 bytes per 4 over the whole UYVY frame; here output stops at 3 * w * h
        const size_t out_len = codec == UGB_UYVY ? frame_len(UGB_RGB, width, height) : in_len;
        if ((codec == UGB_RG48 && ((uintptr_t) src % 2 || (uintptr_t) dst % 2)) || overlap(src, in_len, dst, out_len)) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        const bool b = check_bounds != 0;
        switch (codec) {
        case UGB_UYVY: return b ? launch(MatrixUYVY<true>{ M }, src, in_len, dst, out_len, st) : launch(MatrixUYVY<false>{ M }, src, in_len, dst, out_len, st);
        case UGB_RGB:
                return b ? launch(MatrixRGB<true, false>{ M }, src, in_len, dst, out_len, st)
                         : launch(MatrixRGB<false, false>{ M }, src, in_len, dst, out_len, st);
        default:
                return b ? launch(MatrixRGB<true, true>{ M }, src, in_len, dst, out_len, st)
                         : launch(MatrixRGB<false, true>{ M }, src, in_len, dst, out_len, st);
        }
}

extern "C" UGB_API int ugb200_cf_matrix2(int codec, int width, int height, const double m[9], const void *src, void *dst,
                                         cuda_wrapper_stream_t stream)
{
        if (m == nullptr || src == nullptr || dst == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        if (codec != UGB_UYVY && codec != UGB_v210 && codec != UGB_Y416) {
                return -4;
        }
        Mat M;
        memcpy(M.m, m, sizeof M.m);
        const size_t len = frame_len(codec, width, height);
        const unsigned align = codec == UGB_UYVY ? 1 : codec == UGB_Y416 ? 2 : 4;
        if ((uintptr_t) src % align || (uintptr_t) dst % align || overlap(src, len, dst, len)) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        switch (codec) {
        case UGB_UYVY: return launch(Matrix2UYVY{ M }, src, len, dst, len, st);
        case UGB_Y416: return launch(Matrix2Y416{ M }, src, len, dst, len, st);
        default: return launch(Matrix2V210{ M }, src, len, dst, len, st);
        }
}

extern "C" UGB_API int ugb200_cf_grayscale(int width, int height, const void *src, void *dst, cuda_wrapper_stream_t stream)
{
        if (src == nullptr || dst == nullptr || width <= 0 || height <= 0) {
                return -1;
        }
        // grayscale.c:86: w * h pixels, 2 bytes each; at odd widths the last 2 * h bytes of the frame are not touched
        const size_t n = (size_t) width * height * 2;
        if (overlap(src, n, dst, n)) {
                return -1;
        }
        return launch(Grayscale{}, src, n, dst, n, (cudaStream_t) stream);
}
