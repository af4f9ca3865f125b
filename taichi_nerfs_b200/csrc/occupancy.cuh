// occupancy.cuh — the occupancy bitfield's cell addressing (modules/utils.py:60-100), shared by the ray marcher
// (march.cu) and the mesh export's lattice mask (mesh.cu).
#pragma once

#include <stdint.h>

#ifdef __CUDACC__

__device__ __forceinline__ int frexp_bit(float x) {  // utils.py:60-75
    int exponent = 0;
    if (x != 0.0f) {
        uint32_t bits = __float_as_uint(x);
        exponent = (int)((bits & 0x7f800000u) >> 23) - 127;
        bits = (bits & 0x7fffffu) | 0x3f800000u;
        const float frac = __uint_as_float(bits);
        if (frac < 0.5f) exponent -= 1;
        else if (frac > 1.0f) exponent += 1;
    }
    return exponent;
}

__device__ __forceinline__ uint32_t expand_bits(uint32_t v) {  // utils.py:95-100
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
__device__ __forceinline__ uint32_t morton3d(uint32_t x, uint32_t y, uint32_t z) {
    return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2);
}

#endif  // __CUDACC__
