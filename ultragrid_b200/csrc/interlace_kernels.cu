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
#include <type_traits>

#include "../../include/ugb200.h"
#include "filter_args.h"
#include "host/video_codec.h"

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

// rows of the blend's input: the source frame itself (vc_deinterlace_ex), or the weave of double_framerate call 0
// read from where its rows live (the fused `:d`)
struct PlainRows {
        const uint8_t *src;
        size_t ls;
        __device__ __forceinline__ const uint8_t *row(size_t y) const { return src + y * ls; }
};

// one thread per unit and band: out rows [y0, y1) = avg(row y, row y+1); the last band also writes row lines-1
template <int K, typename V, typename Rows = PlainRows>
__global__ void __launch_bounds__(kThreads) blend_kernel(Rows rows, uint8_t *dst, size_t pitch, size_t lines, size_t band, long units,
                                                         const uint8_t *scratch)
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
        uint8_t *d = dst + off;
        V prev = ld<V>(rows.row(y0) + off);
        size_t y = y0;
        for (; y + kPrefetch < y1; y += kPrefetch) {  // rows y+1 .. y+kPrefetch, all below y1: this band's own rows
                V nx[kPrefetch];
#pragma unroll
                for (int i = 0; i < kPrefetch; ++i) {
                        nx[i] = ld<V>(rows.row(y + 1 + i) + off);
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
                                                                    : ld<V>(rows.row(y + 1) + off);
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

template <int K, typename V, typename Rows = PlainRows>
int run_blend_rows(const Rows &rows, bool in_place, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t blend_bytes, cudaStream_t st)
{
        const long units = (long) (blend_bytes / sizeof(V));
        if (units == 0) {
                return 0;
        }
        const size_t rows_n = lines - 1;
        // bands short enough to fill the GPU, long enough that re-reading each band's boundary row stays cheap
        size_t band = 32;
        while (band > 4 && (size_t) units * ((rows_n + band - 1) / band) < 132u * 1024u) {
                band /= 2;
        }
        const size_t nbands = (rows_n + band - 1) / band;
        if (nbands > 65535) {
                band = (rows_n + 65534) / 65535;
        }
        const unsigned gy = (unsigned) ((rows_n + band - 1) / band);
        const dim3 grid((unsigned) ((units + kThreads - 1) / kThreads), gy);
        uint8_t *scratch = nullptr;
        if (in_place && gy > 1) {
                if (scratch_alloc((void **) &scratch, (size_t) (gy - 1) * units * sizeof(V), st) != 0) {
                        return -2;
                }
                band_heads_kernel<V><<<dim3(grid.x, gy - 1), kThreads, 0, st>>>(dst, ls, band, units, scratch);
        }
        blend_kernel<K, V, Rows><<<grid, kThreads, 0, st>>>(rows, dst, pitch, lines, band, units, scratch);
        const bool ok = cudaGetLastError() == cudaSuccess;
        if (scratch && cudaFreeAsync(scratch, st) != cudaSuccess) {
                return -2;
        }
        return ok ? 0 : -2;
}

template <int K, typename V>
int run_blend(const uint8_t *src, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t blend_bytes, cudaStream_t st)
{
        return run_blend_rows<K, V>(PlainRows{src, ls}, src == dst, ls, dst, pitch, lines, blend_bytes, st);
}

// widest unit the addresses and pitches allow (8-bit: 16/4/1 bytes, 16-bit: 16/4/2); `addr` ORs every row base
template <int K, typename Rows>
int blend_lanes(const Rows &rows, bool in_place, uintptr_t addr, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t blend_bytes,
                cudaStream_t st)
{
        const uintptr_t a = addr | ls | pitch | blend_bytes;
        if (a % 16 == 0) {
                return run_blend_rows<K, uint4>(rows, in_place, ls, dst, pitch, lines, blend_bytes, st);
        }
        if (a % 4 == 0) {
                return run_blend_rows<K, uint32_t>(rows, in_place, ls, dst, pitch, lines, blend_bytes, st);
        }
        if (K == K16) {
                return run_blend_rows<K, uint16_t>(rows, in_place, ls, dst, pitch, lines, blend_bytes, st);
        }
        return run_blend_rows<K, uint8_t>(rows, in_place, ls, dst, pitch, lines, blend_bytes, st);
}

// vc_deinterlace_ex's blend of rows [0, lines-1) and the copy of row lines-2 to lines-1, for the bytes each codec
// blends (*blend of every row); the caller copies the rest of row lines-2 (tail_copy_kernel).  -4: DVS10.
template <typename Rows>
int blend_codec(int codec, const Rows &rows, bool in_place, uintptr_t addr, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t *blend,
                cudaStream_t st);

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

template <typename Rows>
int blend_codec(int codec, const Rows &rows, bool in_place, uintptr_t addr, size_t ls, uint8_t *dst, size_t pitch, size_t lines, size_t *blend,
                cudaStream_t st)
{
        const int bpc = get_bits_per_component((codec_t) codec);
        if (bpc == 8) {
                *blend = ls;
                return blend_lanes<K8>(rows, in_place, addr, ls, dst, pitch, lines, *blend, st);
        }
        if (bpc == 16) {
                *blend = ls;  // even: checked by the caller
                return blend_lanes<K16>(rows, in_place, addr, ls, dst, pitch, lines, *blend, st);
        }
        if (codec == UGB_v210 || codec == UGB_R10k) {
                *blend = ls / 16 * 16;
                const bool v4 = (addr | ls | pitch) % 16 == 0;
                if (codec == UGB_v210) {
                        return v4 ? run_blend_rows<KV210, uint4>(rows, in_place, ls, dst, pitch, lines, *blend, st)
                                  : run_blend_rows<KV210, uint32_t>(rows, in_place, ls, dst, pitch, lines, *blend, st);
                }
                return v4 ? run_blend_rows<KR10K, uint4>(rows, in_place, ls, dst, pitch, lines, *blend, st)
                          : run_blend_rows<KR10K, uint32_t>(rows, in_place, ls, dst, pitch, lines, *blend, st);
        }
        if (codec == UGB_R12L) {
                *blend = ls / 36 * 36;
                return run_blend_rows<K8, R12>(rows, in_place, ls, dst, pitch, lines, *blend, st);
        }
        return -4;  // DVS10: neither 8 nor 16 bits and no packed-word branch (:849-851)
}

}  // namespace ugb_il

using namespace ugb_il;

extern "C" UGB_API int ugb200_vc_deinterlace_ex(int codec, const void *src_, size_t src_linesize, void *dst_, size_t dst_pitch, size_t lines,
                                                cuda_wrapper_stream_t stream)
{
        if (codec <= UGB_VIDEO_CODEC_NONE || codec >= UGB_VIDEO_CODEC_COUNT || is_codec_opaque((codec_t) codec)) {
                return -4;
        }
        const uint8_t *src = (const uint8_t *) src_;
        uint8_t *dst = (uint8_t *) dst_;
        if (!src || !dst || lines == 0 || dst_pitch < src_linesize) {
                return -1;
        }
        const int bpc = get_bits_per_component((codec_t) codec);
        const bool word = codec == UGB_v210 || codec == UGB_R10k || codec == UGB_R12L;
        const uintptr_t align = word ? 4 : bpc == 16 ? 2 : 1;
        if (((uintptr_t) src | (uintptr_t) dst | src_linesize | dst_pitch) % align != 0) {
                return -1;
        }
        const bool in_place = dst == src && dst_pitch == src_linesize;
        const size_t src_end = src_linesize * lines, dst_end = dst_pitch * (lines - 1) + src_linesize;
        if (!in_place && overlap(src, src_end, dst, dst_end)) {
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
        const int rc = blend_codec(codec, PlainRows{src, src_linesize}, in_place, (uintptr_t) src | (uintptr_t) dst, src_linesize, dst, dst_pitch,
                                   lines, &blend, st);
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

// ---- field-rate postprocessors (src/vo_postprocess/temporal-deint.c, interlace.c) ----------------------------
//   weave_kernel: out row r = a source row chosen by the mode (double_framerate, bob, interlace); a thread walks a
//   band of rows down one unit column and loads a source row once when two out rows in a row take it.
//   linear_kernel: walks the rows of the call's parity; each is stored once as a copy and blended with the next one
//   for the row between them (avg_lines, :307-440), so every source row is read once.
//   The fused double_framerate:d runs blend_kernel on the rows where they lie: call 0 on WeaveRows (the weave read from
//   prev / cur), call 1 on cur; the partial group at the end of a row gets the copy, then row h-1 takes row h-2.
namespace ugb_il {

enum WeaveMode { W_DF0 = 0, W_COPY = 1, W_BOB0 = 2, W_BOB1 = 3, W_IL = 4 };

// source row of out row r (a: cur / even rows, b: prev / odd rows), or nullptr where the reference leaves the row
template <int M>
__device__ __forceinline__ const uint8_t *weave_src(int r, int h, const uint8_t *a, const uint8_t *b, size_t ls)
{
        if (M == W_DF0) {  // :244-258: odd rows from prev; the even loop stops at row h-2 (odd h: row h-1 stays)
                return (r & 1) ? b + (size_t) r * ls : r + 1 < h ? a + (size_t) r * ls : nullptr;
        }
        if (M == W_COPY) {  // :259-266
                return a + (size_t) r * ls;
        }
        if (M == W_IL) {  // interlace.c:173-180
                return ((r & 1) ? b : a) + (size_t) r * ls;
        }
        // bob (:279-300): a left-over last row copies the out row above it
        const int call = M == W_BOB1;
        const int rr = (r == h - 1 && ((h + call) & 1)) ? h - 2 : r;
        const int s = call == 0 ? (rr & ~1) : rr == 0 ? 1 : ((rr - 1) | 1);
        return a + (size_t) s * ls;
}

template <int M, typename V>
__global__ void __launch_bounds__(kThreads) weave_kernel(const uint8_t *__restrict__ a, const uint8_t *__restrict__ b, size_t ls,
                                                         uint8_t *__restrict__ dst, size_t pitch, int h, int band, long units)
{
        const long u = (long) blockIdx.x * kThreads + threadIdx.x;
        if (u >= units) {
                return;
        }
        const size_t off = u * sizeof(V);
        const int r0 = blockIdx.y * band;
        const int r1 = r0 + band < h ? r0 + band : h;
        const uint8_t *last = nullptr;  // the source row held in v
        V v{};
#pragma unroll 4
        for (int r = r0; r < r1; ++r) {
                const uint8_t *p = weave_src<M>(r, h, a, b, ls);
                if (p) {
                        if (p != last) {
                                v = ld<V>(p + off);
                        }
                        st<V>(dst + (size_t) r * pitch + off, v);
                }
                last = p;
        }
}

// rows per CTA: short enough that twice the threads the GPU holds are in flight (the walk keeps one load each)
inline int pick_band(long units, int rows)
{
        int band = 32;
        while (band > 4 && units * ((rows + band - 1) / band) < 132L * 4096) {
                band /= 2;
        }
        while ((rows + band - 1) / band > 65535) {
                band *= 2;
        }
        return band;
}

template <int M, typename V>
int launch_weave(const uint8_t *a, const uint8_t *b, size_t ls, uint8_t *dst, size_t pitch, int h, size_t bytes, cudaStream_t st)
{
        const long units = (long) (bytes / sizeof(V));
        if (units == 0) {
                return 0;
        }
        const int band = pick_band(units, h);
        const dim3 grid((unsigned) ((units + kThreads - 1) / kThreads), (unsigned) ((h + band - 1) / band));
        weave_kernel<M, V><<<grid, kThreads, 0, st>>>(a, b, ls, dst, pitch, h, band, units);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

// bytes [0, bytes) of every row; a and b (b may be null) are the row bases at the first byte
template <int M>
int weave(const uint8_t *a, const uint8_t *b, size_t ls, uint8_t *dst, size_t pitch, int h, size_t bytes, cudaStream_t st)
{
        const uintptr_t al = (uintptr_t) a | (uintptr_t) b | (uintptr_t) dst | ls | pitch | bytes;
        if (al % 16 == 0) {
                return launch_weave<M, uint4>(a, b, ls, dst, pitch, h, bytes, st);
        }
        if (al % 4 == 0) {
                return launch_weave<M, uint32_t>(a, b, ls, dst, pitch, h, bytes, st);
        }
        return launch_weave<M, uint8_t>(a, b, ls, dst, pitch, h, bytes, st);
}

// ---- avg_lines (:307-440) ------------------------------------------------------------------------------------
enum LinearKind { KH8 = 8, KH16 = 9, KR10K_LE = 10, KCOPY = 11 };

// c1/2 + c2/2 + (c1%2 + c1%2)/2 per lane (:318-319, :334-335): the upper row's low bit rounds; no lane carries
template <> __device__ __forceinline__ uint32_t avg32<KH8>(uint32_t a, uint32_t b)
{
        return ((a >> 1) & 0x7f7f7f7fu) + ((b >> 1) & 0x7f7f7f7fu) + (a & 0x01010101u);
}
template <> __device__ __forceinline__ uint32_t avg32<KH16>(uint32_t a, uint32_t b)
{
        return ((a >> 1) & 0x7fff7fffu) + ((b >> 1) & 0x7fff7fffu) + (a & 0x00010001u);
}
// R10k (:381-395): words read through ntohl, averaged, stored without htonl
template <> __device__ __forceinline__ uint32_t avg32<KR10K_LE>(uint32_t a, uint32_t b)
{
        a = __byte_perm(a, 0, 0x0123);
        b = __byte_perm(b, 0, 0x0123);
        return (((a >> 22) + (b >> 22) + 1) >> 1) << 22 | (((a >> 12 & 0x3ffu) + (b >> 12 & 0x3ffu) + 1) >> 1) << 12 |
               (((a >> 2 & 0x3ffu) + (b >> 2 & 0x3ffu) + 1) >> 1) << 2;
}
template <> __device__ __forceinline__ uint32_t avg32<KCOPY>(uint32_t a, uint32_t) { return a; }
template <> struct Avg<KH8, uint8_t> {
        static __device__ __forceinline__ uint8_t f(uint8_t a, uint8_t b) { return (uint8_t) (a / 2 + b / 2 + (a & 1)); }
};
template <> struct Avg<KH16, uint16_t> {
        static __device__ __forceinline__ uint16_t f(uint16_t a, uint16_t b) { return (uint16_t) (a / 2 + b / 2 + (a & 1)); }
};
template <> struct Avg<KCOPY, uint8_t> {
        static __device__ __forceinline__ uint8_t f(uint8_t a, uint8_t) { return a; }
};

// a unit of V at byte u * sizeof(V) of a row; lim (a byte count) bounds what is loaded and stored
template <typename V> struct Unit {
        static __device__ __forceinline__ V load(const uint8_t *row, long u, size_t) { return ld<V>(row + u * sizeof(V)); }
        static __device__ __forceinline__ void store(uint8_t *row, long u, const V &v, size_t lim)
        {
                if ((size_t) u * sizeof(V) < lim) {
                        st<V>(row + u * sizeof(V), v);
                }
        }
};
// R12L: a 36-byte group of 24 samples; the row's last group may be partial (words past lim are not touched)
template <> struct Unit<R12> {
        static __device__ __forceinline__ R12 load(const uint8_t *row, long u, size_t lim)
        {
                const uint32_t *q = reinterpret_cast<const uint32_t *>(row + u * 36);
                const long nw = ((long) lim - u * 36) / 4;
                R12 r;
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                        r.w[i] = i < nw ? q[i] : 0u;
                }
                return r;
        }
        static __device__ __forceinline__ void store(uint8_t *row, long u, const R12 &v, size_t lim)
        {
                uint32_t *q = reinterpret_cast<uint32_t *>(row + u * 36);
                const long nw = ((long) lim - u * 36) / 4;
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                        if (i < nw) {
                                q[i] = v.w[i];
                        }
                }
        }
};

// source rows s_k = call + 2k, k in [0, kend]; band [k0, k1) stores out row call+2k = s_k and out row call+2k+1 =
// avg(s_k, s_k+1) (its first n bytes); the band that ends at kend stores s_kend to rows call+2*kend .. h-1; call 1
// also puts s_0 (row 1) in out row 0
template <int K, typename V>
__global__ void __launch_bounds__(kThreads) linear_kernel(const uint8_t *__restrict__ cur, size_t ls, uint8_t *__restrict__ dst, size_t pitch, int h,
                                                          int call, int kend, int band, long units, size_t n)
{
        const long u = (long) blockIdx.x * kThreads + threadIdx.x;
        if (u >= units) {
                return;
        }
        const int k0 = blockIdx.y * band;
        const int k1 = k0 + band < kend ? k0 + band : kend;
        const uint8_t *s = cur + (size_t) call * ls;
        uint8_t *d = dst + (size_t) call * pitch;
        V a = Unit<V>::load(s + (size_t) (2 * k0) * ls, u, ls);
        if (call == 1 && k0 == 0) {
                Unit<V>::store(dst, u, a, ls);
        }
        int k = k0;
        for (; k + kPrefetch <= k1; k += kPrefetch) {
                V nx[kPrefetch];
#pragma unroll
                for (int i = 0; i < kPrefetch; ++i) {
                        nx[i] = Unit<V>::load(s + (size_t) (2 * (k + i + 1)) * ls, u, ls);
                }
#pragma unroll
                for (int i = 0; i < kPrefetch; ++i) {
                        Unit<V>::store(d + (size_t) (2 * (k + i)) * pitch, u, a, ls);
                        Unit<V>::store(d + (size_t) (2 * (k + i) + 1) * pitch, u, Avg<K, V>::f(a, nx[i]), n);
                        a = nx[i];
                }
        }
        for (; k < k1; ++k) {
                const V b = Unit<V>::load(s + (size_t) (2 * (k + 1)) * ls, u, ls);
                Unit<V>::store(d + (size_t) (2 * k) * pitch, u, a, ls);
                Unit<V>::store(d + (size_t) (2 * k + 1) * pitch, u, Avg<K, V>::f(a, b), n);
                a = b;
        }
        if (k1 == kend) {  // :462-465: the remaining rows repeat the last source row
                for (int r = call + 2 * kend; r < h; ++r) {
                        Unit<V>::store(dst + (size_t) r * pitch, u, a, ls);
                }
        }
}

template <int K, typename V>
int launch_linear(const uint8_t *cur, size_t ls, uint8_t *dst, size_t pitch, int h, int call, size_t n, cudaStream_t st)
{
        const long units = std::is_same<V, R12>::value ? (long) ((ls + 35) / 36) : (long) (ls / sizeof(V));
        const int yend = call + 2 * ((h - 2 - call > 0 ? h - 2 - call + 1 : 0) / 2);  // first y of the call's parity >= h-2
        const int kend = (yend - call) / 2;
        const int band = pick_band(units, kend > 0 ? kend : 1);
        const unsigned gy = kend > 0 ? (unsigned) ((kend + band - 1) / band) : 1u;
        const dim3 grid((unsigned) ((units + kThreads - 1) / kThreads), gy);
        linear_kernel<K, V><<<grid, kThreads, 0, st>>>(cur, ls, dst, pitch, h, call, kend, band, units, n);
        return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

template <int K>
int linear_lanes(const uint8_t *cur, size_t ls, uint8_t *dst, size_t pitch, int h, int call, size_t n, cudaStream_t st)
{
        const uintptr_t a = (uintptr_t) cur | (uintptr_t) dst | ls | pitch | n;
        if (a % 16 == 0) {
                return launch_linear<K, uint4>(cur, ls, dst, pitch, h, call, n, st);
        }
        if (a % 4 == 0) {
                return launch_linear<K, uint32_t>(cur, ls, dst, pitch, h, call, n, st);
        }
        if (K == KH16) {
                return launch_linear<K, uint16_t>(cur, ls, dst, pitch, h, call, n, st);
        }
        return launch_linear<K == KCOPY ? KCOPY : KH8, uint8_t>(cur, ls, dst, pitch, h, call, n, st);
}

// double_framerate call 0's weave, read in place: odd rows from prev, even rows from cur but the last at odd h,
// which is dst's own (the reference leaves it unwritten and then blends it)
struct WeaveRows {
        const uint8_t *prev, *cur, *dst;
        size_t ls;
        size_t h;
        __device__ __forceinline__ const uint8_t *row(size_t y) const
        {
                return ((y & 1) ? prev : y + 1 < h ? cur : dst) + y * ls;
        }
};

// the checks every ugb200_pp_* shares: -1 or 0
int pp_args(const void *a, const void *b, size_t ls, int h, int call, const void *dst, size_t pitch)
{
        if (!a || !dst || ls == 0 || h < 2 || pitch < ls || (call != 0 && call != 1)) {
                return -1;
        }
        const size_t dst_n = pitch * (size_t) (h - 1) + ls, src_n = ls * (size_t) h;
        return overlap(dst, dst_n, a, src_n) || (b && overlap(dst, dst_n, b, src_n)) ? -1 : 0;
}

// address alignment a codec's samples need (16-bit: 2, packed words: 4)
size_t codec_align(int codec)
{
        return codec == UGB_v210 || codec == UGB_R10k || codec == UGB_R12L ? 4 : get_bits_per_component((codec_t) codec) == 16 ? 2 : 1;
}

}  // namespace ugb_il

extern "C" UGB_API int ugb200_pp_double_framerate(int codec, const void *prev_, const void *cur_, size_t linesize, int height, int call,
                                                  int deinterlace, void *dst_, size_t pitch, cuda_wrapper_stream_t stream)
{
        const uint8_t *prev = (const uint8_t *) prev_, *cur = (const uint8_t *) cur_;
        uint8_t *dst = (uint8_t *) dst_;
        if (!prev || pp_args(cur, prev, linesize, height, call, dst, pitch) != 0) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        if (!deinterlace) {
                return call == 0 ? weave<W_DF0>(cur, prev, linesize, dst, pitch, height, linesize, st)
                                 : weave<W_COPY>(cur, nullptr, linesize, dst, pitch, height, linesize, st);
        }
        if (codec <= UGB_VIDEO_CODEC_NONE || codec >= UGB_VIDEO_CODEC_COUNT || is_codec_opaque((codec_t) codec) || codec == UGB_DVS10) {
                return -4;  // what ugb200_vc_deinterlace_ex refuses
        }
        const size_t al = codec_align(codec);
        if (((uintptr_t) prev | (uintptr_t) cur | (uintptr_t) dst | linesize | pitch) % al != 0) {
                return -1;
        }
        if (pitch != linesize) {
                // the reference blends the first linesize * height bytes as rows of linesize, whatever the weave's
                // pitch: weave, then the blend in place
                const int rc = call == 0 ? weave<W_DF0>(cur, prev, linesize, dst, pitch, height, linesize, st)
                                         : weave<W_COPY>(cur, nullptr, linesize, dst, pitch, height, linesize, st);
                return rc != 0 ? rc : ugb200_vc_deinterlace_ex(codec, dst, linesize, dst, linesize, (size_t) height, stream);
        }
        // one pass: blend the weave (call 0) or cur (call 1) where it lies
        const size_t h = (size_t) height;
        const uintptr_t addr = (uintptr_t) prev | (uintptr_t) cur | (uintptr_t) dst;
        size_t blend = 0;
        int rc = call == 0 ? blend_codec(codec, WeaveRows{prev, cur, dst, linesize, h}, false, addr, linesize, dst, linesize, h, &blend, st)
                           : blend_codec(codec, PlainRows{cur, linesize}, false, addr, linesize, dst, linesize, h, &blend, st);
        if (rc == 0 && blend < linesize) {
                // bytes no blend covers (partial v210 / R10k / R12L groups) keep what the copy put there, and row h-1
                // takes row h-2's
                const size_t n = linesize - blend;
                rc = call == 0 ? weave<W_DF0>(cur + blend, prev + blend, linesize, dst + blend, linesize, height, n, st)
                               : weave<W_COPY>(cur + blend, nullptr, linesize, dst + blend, linesize, height, n, st);
                if (rc == 0) {
                        tail_copy_kernel<<<(unsigned) ((n + 127) / 128), 128, 0, st>>>(dst, linesize, h, blend, linesize);
                        rc = cudaGetLastError() == cudaSuccess ? 0 : -2;
                }
        }
        return rc;
}

extern "C" UGB_API int ugb200_pp_bob(const void *cur, size_t linesize, int height, int call, void *dst, size_t pitch, cuda_wrapper_stream_t stream)
{
        if (pp_args(cur, nullptr, linesize, height, call, dst, pitch) != 0) {
                return -1;
        }
        const uint8_t *c = (const uint8_t *) cur;
        return call == 0 ? weave<W_BOB0>(c, nullptr, linesize, (uint8_t *) dst, pitch, height, linesize, (cudaStream_t) stream)
                         : weave<W_BOB1>(c, nullptr, linesize, (uint8_t *) dst, pitch, height, linesize, (cudaStream_t) stream);
}

extern "C" UGB_API int ugb200_pp_linear(int codec, const void *cur_, size_t linesize, int height, int call, void *dst_, size_t pitch,
                                        cuda_wrapper_stream_t stream)
{
        const uint8_t *cur = (const uint8_t *) cur_;
        uint8_t *dst = (uint8_t *) dst_;
        if (pp_args(cur, nullptr, linesize, height, call, dst, pitch) != 0) {
                return -1;
        }
        if (codec <= UGB_VIDEO_CODEC_NONE || codec >= UGB_VIDEO_CODEC_COUNT || is_codec_opaque((codec_t) codec)) {
                return -4;
        }
        if (((uintptr_t) cur | (uintptr_t) dst | linesize | pitch) % codec_align(codec) != 0) {
                return -1;
        }
        const cudaStream_t st = (cudaStream_t) stream;
        const size_t L = linesize;
        const int bpc = get_bits_per_component((codec_t) codec);
        if (bpc == 8) {
                return linear_lanes<KH8>(cur, L, dst, pitch, height, call, L, st);
        }
        if (bpc == 16) {
                return linear_lanes<KH16>(cur, L, dst, pitch, height, call, L, st);
        }
        const bool v4 = ((uintptr_t) cur | (uintptr_t) dst | L | pitch) % 16 == 0;
        if (codec == UGB_v210) {  // whole 16-byte groups are blended; the bytes after them stay
                const size_t n = L / 16 * 16;
                return v4 ? launch_linear<KV210, uint4>(cur, L, dst, pitch, height, call, n, st)
                          : launch_linear<KV210, uint32_t>(cur, L, dst, pitch, height, call, n, st);
        }
        if (codec == UGB_R10k) {
                return v4 ? launch_linear<KR10K_LE, uint4>(cur, L, dst, pitch, height, call, L, st)
                          : launch_linear<KR10K_LE, uint32_t>(cur, L, dst, pitch, height, call, L, st);
        }
        if (codec == UGB_R12L) {  // L/16 groups of 4 words; the last word is stored only if 3 divides L/16
                const size_t g = L / 16;
                const size_t n = g % 3 == 0 ? 16 * g : g > 0 ? 16 * g - 4 : 0;
                return launch_linear<K8, R12>(cur, L, dst, pitch, height, call, n, st);
        }
        return linear_lanes<KCOPY>(cur, L, dst, pitch, height, call, L, st);  // DVS10: avg_lines refuses, the row is copied
}

extern "C" UGB_API int ugb200_pp_interlace(const void *even_rows, const void *odd_rows, size_t linesize, int height, void *dst, size_t pitch,
                                           cuda_wrapper_stream_t stream)
{
        if (!odd_rows || pp_args(even_rows, odd_rows, linesize, height, 0, dst, pitch) != 0) {
                return -1;
        }
        return weave<W_IL>((const uint8_t *) even_rows, (const uint8_t *) odd_rows, linesize, (uint8_t *) dst, pitch, height, linesize,
                           (cudaStream_t) stream);
}
