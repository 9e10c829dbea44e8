// n2m_common.cuh -- shared host/device helpers for libn2m_b200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>

#include "../../include/n2m_b200.h"

namespace n2m {

// ---- error plumbing -------------------------------------------------------------------------
extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

inline int fail(const char* what, const char* detail) {
    snprintf(g_err, sizeof(g_err), "n2m_b200: %s: %s", what, detail ? detail : "");
    return 1;
}

inline int check_launch(const char* what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(what, cudaGetErrorString(e));
    return 0;
}

#define N2M_REQUIRE(cond, what, msg) \
    do { if (!(cond)) return ::n2m::fail(what, msg); } while (0)

inline cudaStream_t as_stream(n2m_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename T>
__host__ __device__ inline T div_up(T a, T b) { return (a + b - 1) / b; }

// SM count of the current device, read once per process (grid sizes of the persistent kernels)
inline int num_sms() {
    static int n = 0;
    if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
    return n;
}

// ---- small device helpers ---------------------------------------------------------------------
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(hi, fmaxf(lo, x)); }

// contract() of renderer.py:25-32 (L-inf, in place): where(mag <= 1, x, x * (2 - 1 / mag) / mag), each operation rounded as torch rounds
// it.  The one definition of the stage-1 step (k_s1_points) and the texture bake (k_s1_bake_points).
__device__ __forceinline__ void contract_linf(float p[3]) {
    const float mag = fmaxf(fabsf(p[0]), fmaxf(fabsf(p[1]), fabsf(p[2])));
    if (!(mag <= 1.f)) {
        const float s = __fsub_rn(2.f, __fdiv_rn(1.f, mag));
#pragma unroll
        for (int a = 0; a < 3; ++a) p[a] = __fdiv_rn(__fmul_rn(p[a], s), mag);
    }
}

// Backward of contract_linf at the UNcontracted point x: g <- J(x)^T g.  Outside the unit cube y = x s(m), m = max_k |x_k|,
// s(m) = (2 - 1/m) / m, so J^T g = s g + (g . x) s'(m) dm/dx with s'(m) = 2 (1 - m) / m^3; dm/dx_k = sign(x_k) / t on the t components
// that attain the maximum and 0 elsewhere -- torch's amax backward splits the gradient evenly between ties.
__device__ __forceinline__ void contract_linf_backward(const float x[3], float g[3]) {
    const float ax = fabsf(x[0]), ay = fabsf(x[1]), az = fabsf(x[2]);
    const float m = fmaxf(ax, fmaxf(ay, az));
    if (!(m > 1.f)) return;
    const float r = 1.f / m;
    const float s = (2.f - r) * r;
    const float gx = g[0] * x[0] + g[1] * x[1] + g[2] * x[2];
    const float t = (float)((ax == m) + (ay == m) + (az == m));
    const float c = gx * 2.f * (1.f - m) * r * r * r / t;
    const float a[3] = {ax, ay, az};
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = s * g[k] + (a[k] == m ? (x[k] < 0.f ? -c : c) : 0.f);
}

// 11-bit -> 31-bit spread for 3D Morton codes (bit i of v lands at bit 3i).  Identical to the
// reference's multiply-and-mask form (raymarching.cu:56-63) for every v < 2048 (checked
// exhaustively in tests/test_host_logic.py); the reference documents coords in [0,128).
__host__ __device__ __forceinline__ uint32_t spread3(uint32_t v) {
    v &= 0x7FFu;
    v = (v | (v << 16)) & 0x070000FFu;
    v = (v | (v << 8)) & 0x0700F00Fu;
    v = (v | (v << 4)) & 0x430C30C3u;
    v = (v | (v << 2)) & 0x49249249u;
    return v;
}
__host__ __device__ __forceinline__ uint32_t morton3(uint32_t x, uint32_t y, uint32_t z) {
    return spread3(x) | (spread3(y) << 1) | (spread3(z) << 2);
}
__host__ __device__ __forceinline__ uint32_t compact3(uint32_t x) {
    x &= 0x49249249u;
    x = (x | (x >> 2)) & 0xc30c30c3u;
    x = (x | (x >> 4)) & 0x0f00f00fu;
    x = (x | (x >> 8)) & 0xff0000ffu;
    x = (x | (x >> 16)) & 0x0000ffffu;
    return x;
}


// ---- ray-range parts of a batch (fused stage-0 path) ----------------------------------------------
// The march leaves the sample offsets of rays n*e/8 (e = 0..8) in counters[4..12] (clamped to counters[1]); n is the batch's active
// ray count (counters[16], adaptive ray count) or its N rows.
// Part `part` of `nparts` (1, 2, 4 or 8) covers rays [n*e0/8, n*e1/8) with e0 = part*8/nparts, e1 = (part+1)*8/nparts,
// i.e. the contiguous samples [counters[4+e0], counters[4+e1]).  nparts == 1 reads only counters[1] (callers that
// fill counters by hand, e.g. the explicit-point gather, keep working with a 4-entry array).
constexpr uint32_t kPartSlots = 8;
struct PartRange { uint32_t lo, hi, M; };
__device__ __forceinline__ PartRange part_range(const int32_t* __restrict__ counters, uint32_t part, uint32_t nparts) {
    PartRange r;
    r.M = (uint32_t)counters[1];
    if (nparts <= 1) { r.lo = 0; r.hi = r.M; return r; }
    r.lo = (uint32_t)counters[4 + part * kPartSlots / nparts];
    r.hi = (uint32_t)counters[4 + (part + 1) * kPartSlots / nparts];
    return r;
}
__host__ __device__ __forceinline__ uint32_t part_first_ray(uint32_t N, uint32_t eighth) {
    return (uint32_t)(((unsigned long long)N * eighth) / kPartSlots);
}
__host__ inline bool valid_parts(uint32_t part, uint32_t nparts) {
    return (nparts == 1 || nparts == 2 || nparts == 4 || nparts == 8) && part < nparts;
}

}  // namespace n2m
