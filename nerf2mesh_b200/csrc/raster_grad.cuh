// raster_grad.cuh -- the gradient arithmetic of dr.rasterize and dr.interpolate, written once for the operator kernels of raster.cu
// (n2m_rasterize_backward, n2m_interpolate_backward_rast) and for the colour-field vertex gradient of the stage-1 step (stage1.cu,
// k_s1_offset_grad).
//
// Rasterize (nvdiffrast's gradient): only the (u, v) channels of rast carry one; z/w and the triangle id carry none.  (u, v) are the
// perspective-correct barycentrics of pixel NDC (X, Y) in 2-D homogeneous form: with p'_k = (x_k - X w_k, y_k - Y w_k) and the edge
// functions a_k = p'_{k+1} x p'_{k+2} (indices mod 3), u = a_0 / sum a, v = a_1 / sum a.  The same expression holds for triangles
// that cross the camera plane (k_rast_resolve's homogeneous path solves the same system).  Clip z receives nothing.
#pragma once
#include "n2m_common.cuh"

namespace n2m {
namespace {

// pixel (x, y) of an H x W target -> its NDC centre, the expression of raster.cu's homogeneous path (bary_homog)
__device__ __forceinline__ float2 pixel_ndc(uint32_t x, uint32_t y, uint32_t H, uint32_t W) {
    return make_float2(((float)x + 0.5f) * __fdiv_rn(2.f, (float)W) - 1.f, ((float)y + 0.5f) * __fdiv_rn(2.f, (float)H) - 1.f);
}

// d loss / d (u, v) at pixel NDC (X, Y) of the triangle with clip-space vertices p[0..2] -> d loss / d (x, y, w) of each vertex,
// ACCUMULATED (atomics) into grad_pos [V,4] at rows i[0..2]; the z column is left alone
__device__ __forceinline__ void rasterize_uv_backward(const float4 (&p)[3], const int (&i)[3], float X, float Y, float du, float dv,
                                                      float* __restrict__ grad_pos) {
    float qx[3], qy[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { qx[k] = p[k].x - X * p[k].w; qy[k] = p[k].y - Y * p[k].w; }
    float a[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
        a[k] = qx[k1] * qy[k2] - qy[k1] * qx[k2];
    }
    const float rs = 1.f / (a[0] + a[1] + a[2]);
    const float b0 = a[0] * rs, b1 = a[1] * rs;
    const float G = du * b0 + dv * b1;
    const float ga[3] = {(du - G) * rs, (dv - G) * rs, -G * rs};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
        // a_{k2} = p'_k x p'_{k1} (k first), a_{k1} = p'_{k2} x p'_k (k second)
        const float gx = ga[k2] * qy[k1] - ga[k1] * qy[k2];
        const float gy = ga[k1] * qx[k2] - ga[k2] * qx[k1];
        float* g = grad_pos + 4 * (size_t)i[k];
        atomicAdd(g + 0, gx);
        atomicAdd(g + 1, gy);
        atomicAdd(g + 3, -(X * gx + Y * gy));
    }
}

// dr.interpolate's gradient w.r.t. (u, v) of one pixel: out = u a0 + v a1 + (1 - u - v) a2, so
// du = sum_a g_a (a0 - a2), dv = sum_a g_a (a1 - a2)
template <int A>
__device__ __forceinline__ float2 interpolate_uv_backward(const float (&g)[A], const float (&a0)[A], const float (&a1)[A], const float (&a2)[A]) {
    float du = 0.f, dv = 0.f;
#pragma unroll
    for (int c = 0; c < A; ++c) { du += g[c] * (a0[c] - a2[c]); dv += g[c] * (a1[c] - a2[c]); }
    return make_float2(du, dv);
}

}  // namespace
}  // namespace n2m
