// Interlaced video: device form of UltraGrid's linear-blend deinterlacers (src/video_codec.c) and field-order
// converters (src/video_frame.c).  Arithmetic contract and quirks: DESIGN.md §2 "Interlaced video".
//
//   vc_deinterlace_ex (video_codec.c:722-854): out row y = (row y + row y+1 + 1) >> 1 per sample, last row = out
//   row lines-2.  CTAs walk bands of rows down a strip of columns with the previous row in registers, so every
//   input row is read once.  In place, row y1 (the first row of the next band) is overwritten by that band, so a
//   pre-pass copies each band's first row to stream-ordered scratch and the band above reads it from there.
//
//   vc_deinterlace (video_codec.c:597-711, SSE2 form): an in-place recursive filter down each byte column.  One
//   thread per 4-byte column (__vavgu4 == pavgb) walks all rows with 2*G rows of loads in flight; a second tiny
//   pass redoes the k head bytes the reference's last 16-byte column re-filters one row down.
//
//   il_upper_to_merged / il_merged_to_upper (video_frame.c:332-379): row permutations; in place through
//   stream-ordered scratch (cudaMallocFromPoolAsync), so the host never waits.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <mutex>

#include "../../include/ugb200.h"

namespace ugb_il {

// ---- per-unit rounded average (pavgb / pavgw / the reference's scalar (a + b + 1) >> 1) ------------------
enum Kind { K8 = 0, K16 = 1, KV210 = 2, KR10K = 3 };

template <int K> __device__ __forceinline__ uint32_t avg32(uint32_t a, uint32_t b);
template <> __device__ __forceinline__ uint32_t avg32<K8>(uint32_t a, uint32_t b) { return __vavgu4(a, b); }
template <> __device__ __forceinline__ uint32_t avg32<K16>(uint32_t a, uint32_t b) { return __vavgu2(a, b); }
// v210 (video_codec.c:790-806): the field at 20 is taken as v >> 20, so padding bits 30-31 are averaged with it
template <> __device__ __forceinline__ uint32_t avg32<KV210>(uint32_t a, uint32_t b)
{
        return (((a >> 20) + (b >> 20) + 1) >> 1) << 20 | (((a >> 10 & 0x3ffu) + (b >> 10 & 0x3ffu) + 1) >> 1) << 10 |
               (((a & 0x3ffu) + (b & 0x3ffu) + 1) >> 1);
}
// R10k (:807-823): big-endian words, fields at 22, 12, 2; bits 0-1 of the output are zero
template <> __device__ __forceinline__ uint32_t avg32<KR10K>(uint32_t a, uint32_t b)
{
        a = __byte_perm(a, 0, 0x0123);
        b = __byte_perm(b, 0, 0x0123);
        const uint32_t o = (((a >> 22) + (b >> 22) + 1) >> 1) << 22 | (((a >> 12 & 0x3ffu) + (b >> 12 & 0x3ffu) + 1) >> 1) << 12 |
                           (((a >> 2 & 0x3ffu) + (b >> 2 & 0x3ffu) + 1) >> 1) << 2;
        return __byte_perm(o, 0, 0x0123);
}

// a unit is V bytes: uint4 / uint32_t of 32-bit lanes, or one uint16_t / uint8_t sample
template <int K, typename V> struct Avg;
template <int K> struct Avg<K, uint4> {
        static __device__ __forceinline__ uint4 f(uint4 a, uint4 b)
        {
                return make_uint4(avg32<K>(a.x, b.x), avg32<K>(a.y, b.y), avg32<K>(a.z, b.z), avg32<K>(a.w, b.w));
        }
};
template <int K> struct Avg<K, uint32_t> {
        static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return avg32<K>(a, b); }
};
template <int K> struct Avg<K, uint16_t> {
        static __device__ __forceinline__ uint16_t f(uint16_t a, uint16_t b) { return (uint16_t) ((a + b + 1) >> 1); }
};
template <int K> struct Avg<K, uint8_t> {
        static __device__ __forceinline__ uint8_t f(uint8_t a, uint8_t b) { return (uint8_t) ((a + b + 1) >> 1); }
};

// R12L (:824-848): a 36-byte group is 24 12-bit samples, little-endian bit stream; blended per sample
struct R12 {
        uint32_t w[9];
};
template <int K> struct Avg<K, R12> {
        static __device__ __forceinline__ R12 f(const R12 &a, const R12 &b)
        {
                R12 o;
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                        o.w[i] = 0;
                }
#pragma unroll
                for (int s = 0; s < 24; ++s) {
                        const int bit = s * 12, wi = bit / 32, sh = bit % 32;
                        uint32_t x = a.w[wi] >> sh, y = b.w[wi] >> sh;
                        if (sh > 20) {
                                x |= a.w[wi + 1] << (32 - sh);
                                y |= b.w[wi + 1] << (32 - sh);
                        }
                        const uint32_t r = ((x & 0xfffu) + (y & 0xfffu) + 1) >> 1;
                        o.w[wi] |= r << sh;
                        if (sh > 20) {
                                o.w[wi + 1] |= r >> (32 - sh);
                        }
                }
                return o;
        }
};

template <typename V> __device__ __forceinline__ V ld(const uint8_t *p) { return *reinterpret_cast<const V *>(p); }
template <typename V> __device__ __forceinline__ void st(uint8_t *p, const V &v) { *reinterpret_cast<V *>(p) = v; }
template <> __device__ __forceinline__ R12 ld<R12>(const uint8_t *p)
{
        R12 r;
        const uint32_t *q = reinterpret_cast<const uint32_t *>(p);
#pragma unroll
        for (int i = 0; i < 9; ++i) {
                r.w[i] = q[i];
        }
        return r;
}
template <> __device__ __forceinline__ void st<R12>(uint8_t *p, const R12 &v)
{
        uint32_t *q = reinterpret_cast<uint32_t *>(p);
#pragma unroll
        for (int i = 0; i < 9; ++i) {
                q[i] = v.w[i];
        }
}

// Stream-ordered scratch from a pool of this library's own, one per device.  The pool keeps up to kPoolKeep bytes
// across synchronisations, so a steady stream of in-place calls does not map and unmap memory every frame (the
// device's default pool returns everything at each synchronisation).
constexpr uint64_t kPoolKeep = 256ull << 20;

int scratch_alloc(void **p, size_t n, cudaStream_t st)
{
        static std::mutex mu;
        static cudaMemPool_t pools[64];
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
                return -2;
        }
        cudaMemPool_t pool;
        {
                std::lock_guard<std::mutex> lk(mu);
                if (!pools[dev]) {
                        cudaMemPoolProps props = {};
                        props.allocType = cudaMemAllocationTypePinned;
                        props.location.type = cudaMemLocationTypeDevice;
                        props.location.id = dev;
                        if (cudaMemPoolCreate(&pools[dev], &props) != cudaSuccess) {
                                pools[dev] = nullptr;
                                return -2;
                        }
                        uint64_t keep = kPoolKeep;
                        cudaMemPoolSetAttribute(pools[dev], cudaMemPoolAttrReleaseThreshold, &keep);
                }
                pool = pools[dev];
        }
        return cudaMallocFromPoolAsync(p, n, pool, st) == cudaSuccess ? 0 : -2;
}

constexpr int kThreads = 128;
constexpr int kPrefetch = 8;

// band pre-pass (in place only): scratch row b = source row (b + 1) * band, for every band but the last
template <typename V>
__global__ void __launch_bounds__(kThreads) band_heads_kernel(const uint8_t *src, size_t ls, size_t band, long units, uint8_t *scratch)
{
        const long u = (long) blockIdx.x * kThreads + threadIdx.x;
        if (u >= units) {
                return;
        }
        const size_t b = blockIdx.y;
        st<V>(scratch + b * units * sizeof(V) + u * sizeof(V), ld<V>(src + (b + 1) * band * ls + u * sizeof(V)));
}

// one thread per unit and band: out rows [y0, y1) = avg(row y, row y+1); the last band also writes row lines-1
template <int K, typename V>
__global__ void __launch_bounds__(kThreads) blend_kernel(const uint8_t *src, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t band,
                                                         long units, const uint8_t *scratch)
{
        const long u = (long) blockIdx.x * kThreads + threadIdx.x;
        if (u >= units) {
                return;
        }
        const size_t off = u * sizeof(V);
        const size_t b = blockIdx.y;
        const size_t y0 = b * band;
        const size_t last = lines - 1;  // rows written by blending: [0, last)
        const size_t y1 = y0 + band < last ? y0 + band : last;
        const uint8_t *s = src + off;
        uint8_t *d = dst + off;
        V prev = ld<V>(s + y0 * ls);
        size_t y = y0;
        for (; y + kPrefetch < y1; y += kPrefetch) {  // rows y+1 .. y+kPrefetch, all below y1: this band's own rows
                V nx[kPrefetch];
#pragma unroll
                for (int i = 0; i < kPrefetch; ++i) {
                        nx[i] = ld<V>(s + (y + 1 + i) * ls);
                }
#pragma unroll
                for (int i = 0; i < kPrefetch; ++i) {
                        st<V>(d + (y + i) * pitch, Avg<K, V>::f(prev, nx[i]));
                        prev = nx[i];
                }
        }
        V out = prev;
        for (; y < y1; ++y) {
                const V nx = (y + 1 == y1 && y1 != last && scratch) ? ld<V>(scratch + (b * units) * sizeof(V) + off)
                                                                    : ld<V>(s + (y + 1) * ls);
                out = Avg<K, V>::f(prev, nx);
                st<V>(d + y * pitch, out);
                prev = nx;
        }
        if (y1 == last) {
                st<V>(d + last * pitch, out);  // memcpy of row lines-2 (:851), for the bytes blended here
        }
}

// bytes of row lines-2 no blend covers (partial v210 / R10k / R12L groups) go to row lines-1 as they are (:851)
__global__ void tail_copy_kernel(uint8_t *dst, size_t pitch, size_t lines, size_t from, size_t to)
{
        const size_t x = from + (size_t) blockIdx.x * blockDim.x + threadIdx.x;
        if (x < to) {
                dst[(lines - 1) * pitch + x] = dst[(lines - 2) * pitch + x];
        }
}

template <int K, typename V>
int run_blend(const uint8_t *src, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t blend_bytes, cudaStream_t st)
{
        const long units = (long) (blend_bytes / sizeof(V));
        if (units == 0) {
                return 0;
        }
        const size_t rows = lines - 1;
        // bands short enough to fill the GPU, long enough that re-reading each band's boundary row stays cheap
        size_t band = 32;
        while (band > 4 && (size_t) units * ((rows + band - 1) / band) < 132u * 1024u) {
                band /= 2;
        }
        const size_t nbands = (rows + band - 1) / band;
        if (nbands > 65535) {
                band = (rows + 65534) / 65535;
        }
        const unsigned gy = (unsigned) ((rows + band - 1) / band);
        const dim3 grid((unsigned) ((units + kThreads - 1) / kThreads), gy);
        uint8_t *scratch = nullptr;
        if (src == dst && gy > 1) {
                if (scratch_alloc((void **) &scratch, (size_t) (gy - 1) * units * sizeof(V), st) != 0) {
                        return -2;
                }
                band_heads_kernel<V><<<dim3(grid.x, gy - 1), kThreads, 0, st>>>(src, ls, band, units, scratch);
        }
        blend_kernel<K, V><<<grid, kThreads, 0, st>>>(src, ls, dst, pitch, lines, band, units, scratch);
        const bool ok = cudaGetLastError() == cudaSuccess;
        if (scratch && cudaFreeAsync(scratch, st) != cudaSuccess) {
                return -2;
        }
        return ok ? 0 : -2;
}

// widest unit the addresses and pitches allow (8-bit: 16/4/1 bytes, 16-bit: 16/4/2)
template <int K>
int blend_lanes(const uint8_t *src, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t blend_bytes, cudaStream_t st)
{
        const uintptr_t a = (uintptr_t) src | (uintptr_t) dst | ls | pitch | blend_bytes;
        if (a % 16 == 0) {
                return run_blend<K, uint4>(src, ls, dst, pitch, lines, blend_bytes, st);
        }
        if (a % 4 == 0) {
                return run_blend<K, uint32_t>(src, ls, dst, pitch, lines, blend_bytes, st);
        }
        if (K == K16) {
                return run_blend<K, uint16_t>(src, ls, dst, pitch, lines, blend_bytes, st);
        }
        return run_blend<K, uint8_t>(src, ls, dst, pitch, lines, blend_bytes, st);
}

// ---- vc_deinterlace ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t vavg(uint32_t a, uint32_t b) { return __vavgu4(a, b); }
__device__ __forceinline__ uint8_t vavg(uint8_t a, uint8_t b) { return (uint8_t) ((a + b + 1) >> 1); }

constexpr int kLegacyG = 8;  // filter steps (2 rows each) whose loads are issued together

// the SSE2 loop body of :650-666 on one column of T: row 0 kept; step t writes rows 2t+1 and 2t+2
template <typename T>
__global__ void __launch_bounds__(kThreads) legacy_kernel(uint8_t *buf, long ls, int steps, long cols)
{
        const long c = (long) blockIdx.x * kThreads + threadIdx.x;
        if (c >= cols) {
                return;
        }
        uint8_t *p = buf + c * (long) sizeof(T);
        T a = *reinterpret_cast<const T *>(p), b = *reinterpret_cast<const T *>(p + ls);
        int t = 0;
        for (; t + kLegacyG <= steps; t += kLegacyG) {
                T cc[kLegacyG], dd[kLegacyG];
#pragma unroll
                for (int i = 0; i < kLegacyG; ++i) {
                        cc[i] = *reinterpret_cast<const T *>(p + (2L * (t + i) + 2) * ls);
                        dd[i] = *reinterpret_cast<const T *>(p + (2L * (t + i) + 3) * ls);
                }
#pragma unroll
                for (int i = 0; i < kLegacyG; ++i) {
                        const T n1 = vavg(vavg(a, cc[i]), b);
                        *reinterpret_cast<T *>(p + (2L * (t + i) + 1) * ls) = n1;
                        const T n2 = vavg(vavg(n1, dd[i]), cc[i]);
                        *reinterpret_cast<T *>(p + (2L * (t + i) + 2) * ls) = n2;
                        a = n2;
                        b = dd[i];
                }
        }
        for (; t < steps; ++t) {
                const T cc = *reinterpret_cast<const T *>(p + (2L * t + 2) * ls);
                const T dd = *reinterpret_cast<const T *>(p + (2L * t + 3) * ls);
                const T n1 = vavg(vavg(a, cc), b);
                *reinterpret_cast<T *>(p + (2L * t + 1) * ls) = n1;
                const T n2 = vavg(vavg(n1, dd), cc);
                *reinterpret_cast<T *>(p + (2L * t + 2) * ls) = n2;
                a = n2;
                b = dd;
        }
}

// ---- il_* --------------------------------------------------------------------------------------------------
template <typename V, bool TO_MERGED>
__global__ void __launch_bounds__(kThreads) permute_kernel(uint8_t *dst, const uint8_t *src, long ls, int height, long units)
{
        const long u = (long) blockIdx.x * kThreads + threadIdx.x;
        if (u >= units) {
                return;
        }
        const int half = (height + 1) / 2;  // upper-field rows
        for (int r = blockIdx.y; r < height; r += gridDim.y) {
                const int sr = TO_MERGED ? ((r & 1) ? half + r / 2 : r / 2) : (r < half ? 2 * r : 2 * (r - half) + 1);
                st<V>(dst + r * ls + u * (long) sizeof(V), ld<V>(src + sr * ls + u * (long) sizeof(V)));
        }
}

template <bool TO_MERGED, typename V> void launch_permute(uint8_t *dst, const uint8_t *src, long ls, int height, cudaStream_t st)
{
        const long units = ls / (long) sizeof(V);
        const dim3 grid((unsigned) ((units + kThreads - 1) / kThreads), (unsigned) (height < 65535 ? height : 65535));
        permute_kernel<V, TO_MERGED><<<grid, kThreads, 0, st>>>(dst, src, ls, height, units);
}

template <bool TO_MERGED> int il_permute(void *dst_, void *src_, int linesize, int height, cuda_wrapper_stream_t stream)
{
        if (linesize < 0 || height < 0 || !dst_ || !src_) {
                return -1;
        }
        if (linesize == 0 || height == 0) {
                return 0;
        }
        uint8_t *dst = (uint8_t *) dst_;
        const uint8_t *src = (const uint8_t *) src_;
        const size_t n = (size_t) linesize * height;
        const bool overlap = dst < src + n && src < dst + n;
        if (overlap && dst != src) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        const uint8_t *from = src;
        uint8_t *scratch = nullptr;
        if (dst == src) {
                if (scratch_alloc((void **) &scratch, n, st) != 0) {
                        return -2;
                }
                if (cudaMemcpyAsync(scratch, src, n, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
                        cudaFreeAsync(scratch, st);
                        return -2;
                }
                from = scratch;
        }
        const uintptr_t a = (uintptr_t) dst | (uintptr_t) from | (uintptr_t) linesize;
        if (a % 16 == 0) {
                launch_permute<TO_MERGED, uint4>(dst, from, linesize, height, st);
        } else if (a % 4 == 0) {
                launch_permute<TO_MERGED, uint32_t>(dst, from, linesize, height, st);
        } else {
                launch_permute<TO_MERGED, uint8_t>(dst, from, linesize, height, st);
        }
        const bool ok = cudaGetLastError() == cudaSuccess;
        if (scratch && cudaFreeAsync(scratch, st) != cudaSuccess) {
                return -2;
        }
        return ok ? 0 : -2;
}

// codec_info[] (video_codec.c:120-206): VCF_OPAQUE and the bits-per-component column
bool codec_opaque(int c)
{
        switch (c) {
        case UGB_RGBA: case UGB_UYVY: case UGB_YUYV: case UGB_VUYA: case UGB_R10k: case UGB_R12L: case UGB_v210: case UGB_DVS10:
        case UGB_RGB: case UGB_BGR: case UGB_RG48: case UGB_I420: case UGB_Y216: case UGB_Y416:
                return false;
        default:
                return true;
        }
}
int codec_bpc(int c)
{
        switch (c) {
        case UGB_R10k: case UGB_v210: case UGB_DVS10: return 10;
        case UGB_R12L: return 12;
        case UGB_RG48: case UGB_Y216: case UGB_Y416: return 16;
        default: return 8;
        }
}

}  // namespace ugb_il

using namespace ugb_il;

extern "C" UGB_API int ugb200_vc_deinterlace_ex(int codec, const void *src_, size_t src_linesize, void *dst_, size_t dst_pitch, size_t lines,
                                                cuda_wrapper_stream_t stream)
{
        if (codec <= UGB_VIDEO_CODEC_NONE || codec >= UGB_VIDEO_CODEC_COUNT || codec_opaque(codec)) {
                return -4;
        }
        const uint8_t *src = (const uint8_t *) src_;
        uint8_t *dst = (uint8_t *) dst_;
        if (!src || !dst || lines == 0 || dst_pitch < src_linesize) {
                return -1;
        }
        const int bpc = codec_bpc(codec);
        const bool word = codec == UGB_v210 || codec == UGB_R10k || codec == UGB_R12L;
        const uintptr_t align = word ? 4 : bpc == 16 ? 2 : 1;
        if (((uintptr_t) src | (uintptr_t) dst | src_linesize | dst_pitch) % align != 0) {
                return -1;
        }
        const bool in_place = dst == src && dst_pitch == src_linesize;
        const size_t src_end = src_linesize * lines, dst_end = dst_pitch * (lines - 1) + src_linesize;
        if (!in_place && src_linesize > 0 && dst < src + src_end && src < dst + dst_end) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        if (lines == 1) {  // :733-736, before the codec is looked at
                if (!in_place && src_linesize > 0 && cudaMemcpyAsync(dst, src, src_linesize, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
                        return -2;
                }
                return 0;
        }
        size_t blend = 0;  // leading bytes of each row that are blended; the rest of the row stays unwritten
        int rc;
        if (bpc == 8) {
                blend = src_linesize;
                rc = blend_lanes<K8>(src, src_linesize, dst, dst_pitch, lines, blend, st);
        } else if (bpc == 16) {
                blend = src_linesize;  // even: checked above
                rc = blend_lanes<K16>(src, src_linesize, dst, dst_pitch, lines, blend, st);
        } else if (codec == UGB_v210 || codec == UGB_R10k) {
                blend = src_linesize / 16 * 16;
                const uintptr_t a = (uintptr_t) src | (uintptr_t) dst | src_linesize | dst_pitch;
                if (codec == UGB_v210) {
                        rc = a % 16 == 0 ? run_blend<KV210, uint4>(src, src_linesize, dst, dst_pitch, lines, blend, st)
                                         : run_blend<KV210, uint32_t>(src, src_linesize, dst, dst_pitch, lines, blend, st);
                } else {
                        rc = a % 16 == 0 ? run_blend<KR10K, uint4>(src, src_linesize, dst, dst_pitch, lines, blend, st)
                                         : run_blend<KR10K, uint32_t>(src, src_linesize, dst, dst_pitch, lines, blend, st);
                }
        } else if (codec == UGB_R12L) {
                blend = src_linesize / 36 * 36;
                rc = run_blend<K8, R12>(src, src_linesize, dst, dst_pitch, lines, blend, st);
        } else {
                return -4;  // DVS10: neither 8 nor 16 bits and no packed-word branch (:849-851)
        }
        if (rc != 0) {
                return rc;
        }
        if (blend < src_linesize) {
                const size_t n = src_linesize - blend;
                tail_copy_kernel<<<(unsigned) ((n + 127) / 128), 128, 0, st>>>(dst, dst_pitch, lines, blend, src_linesize);
                if (cudaGetLastError() != cudaSuccess) {
                        return -2;
                }
        }
        return 0;
}

extern "C" UGB_API int ugb200_vc_deinterlace(void *buf_, long linesize, int lines, cuda_wrapper_stream_t stream)
{
        uint8_t *buf = (uint8_t *) buf_;
        if (!buf || linesize < 16 || lines < 0) {
                return -1;
        }
        if (lines <= 4) {
                return 0;  // the loop j < lines - 4 never runs
        }
        const cudaStream_t st = (cudaStream_t) stream;
        const int steps = (lines - 3) / 2;
        if ((uintptr_t) buf % 4 == 0 && linesize % 4 == 0) {
                const long cols = linesize / 4;
                legacy_kernel<uint32_t><<<(unsigned) ((cols + kThreads - 1) / kThreads), kThreads, 0, st>>>(buf, linesize, steps, cols);
        } else {
                legacy_kernel<uint8_t><<<(unsigned) ((linesize + kThreads - 1) / kThreads), kThreads, 0, st>>>(buf, linesize, steps, linesize);
        }
        // the last 16-byte column starts at i_L < linesize and runs k bytes into the next row, which column 0 has
        // already filtered: those k head bytes get the same filter again, one row down
        const long k = linesize % 16 ? 16 - linesize % 16 : 0;
        if (k > 0) {
                legacy_kernel<uint8_t><<<1, kThreads, 0, st>>>(buf + linesize, linesize, steps, k);
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" UGB_API int ugb200_il_upper_to_merged(void *dst, void *src, int linesize, int height, cuda_wrapper_stream_t stream)
{
        return il_permute<true>(dst, src, linesize, height, stream);
}

extern "C" UGB_API int ugb200_il_merged_to_upper(void *dst, void *src, int linesize, int height, cuda_wrapper_stream_t stream)
{
        return il_permute<false>(dst, src, linesize, height, stream);
}
