// Measures where gamma's tables should live: shared memory with a persistent grid (what ugb200_cf_gamma runs) against
// L1-cached global loads (__ldg), on 8K frames of random samples, for all four tables.  It compiles the library's own
// kernels (colour_filter_kernels.cu) into this program and times each with CUDA events over 64 launches after warm-up.
//   nvcc -O3 -std=c++17 --expt-relaxed-constexpr -gencode arch=compute_90a,code=sm_90a -o tools/gamma_lut_exp tools/gamma_lut_exp.cu && tools/gamma_lut_exp
#include <stdio.h>
#include <stdlib.h>

#include "../ultragrid_b200/csrc/colour_filter_kernels.cu"

template <typename InT, typename OutT, bool SMEM>
static float time_us(const OutT *lut, const uint8_t *src, size_t in_len, uint8_t *dst, size_t out_len)
{
        for (int i = 0; i < 8; ++i) {
                ugb_cf::launch_gamma<InT, OutT, SMEM>(lut, src, in_len, dst, out_len, 0);
        }
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        cudaEventRecord(a);
        for (int i = 0; i < 64; ++i) {
                ugb_cf::launch_gamma<InT, OutT, SMEM>(lut, src, in_len, dst, out_len, 0);
        }
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float ms = 0;
        cudaEventElapsedTime(&ms, a, b);
        cudaEventDestroy(a);
        cudaEventDestroy(b);
        return ms * 1e3f / 64;
}

template <typename InT, typename OutT>
static void row(const char *name, const OutT *lut, const uint8_t *src, uint8_t *dst, size_t pixels)
{
        const size_t in_len = pixels * 3 * sizeof(InT), out_len = pixels * 3 * sizeof(OutT);
        const float s = time_us<InT, OutT, true>(lut, src, in_len, dst, out_len);
        const float g = time_us<InT, OutT, false>(lut, src, in_len, dst, out_len);
        printf("%-8s shared %8.1f us (%5.2f TB/s)   global/L1 %8.1f us (%5.2f TB/s)\n", name, s, (in_len + out_len) / (s * 1e-6) / 1e12, g,
               (in_len + out_len) / (g * 1e-6) / 1e12);
}

int main()
{
        const size_t pixels = 7680 * 4320, bytes = pixels * 6;
        uint8_t *host = (uint8_t *) malloc(bytes), *src, *dst;
        srand(1);
        for (size_t i = 0; i < bytes; ++i) {
                host[i] = (uint8_t) rand();
        }
        cudaMalloc(&src, bytes);
        cudaMalloc(&dst, bytes);
        cudaMemcpy(src, host, bytes, cudaMemcpyHostToDevice);
        ugb200_cf_gamma_t g = ugb200_cf_gamma_create(1 / 2.2);
        printf("8K frames of random samples, gamma 1/2.2\n");
        row<uint8_t, uint8_t>("8->8", g->lut8(), src, dst, pixels);
        row<uint8_t, uint16_t>("8->16", g->lut8_16(), src, dst, pixels);
        row<uint16_t, uint8_t>("16->8", g->lut16_8(), src, dst, pixels);
        row<uint16_t, uint16_t>("16->16", g->lut16(), src, dst, pixels);
        printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
        ugb200_cf_gamma_destroy(g);
        cudaFree(src);
        cudaFree(dst);
        free(host);
        return 0;
}
