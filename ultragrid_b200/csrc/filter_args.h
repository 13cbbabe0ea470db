// Argument checks shared by the GPU filters (colour, geometry, interlace, logo, resize).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

// [a, a + na) and [b, b + nb) share a byte; an empty range overlaps nothing
inline bool overlap(const void *a, size_t na, const void *b, size_t nb)
{
        const uintptr_t x = (uintptr_t) a, y = (uintptr_t) b;
        return na && nb && x < y + nb && y < x + na;
}

namespace ugb_il {
// stream-ordered scratch from this library's own pool on the current device (interlace_kernels.cu)
int scratch_alloc(void **p, size_t n, cudaStream_t st);
}
