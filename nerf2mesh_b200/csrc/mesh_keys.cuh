// mesh_keys.cuh -- order-preserving float keys shared by the mesh clean-up (meshclean.cu) and the decimation (decimate.cu).
#pragma once

#include <stdint.h>

namespace n2m {

// float -> u32 whose unsigned order is the float order (-0 below +0); fkey_inv inverts it
__device__ __forceinline__ uint32_t fkey(float x) {
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

}  // namespace n2m
