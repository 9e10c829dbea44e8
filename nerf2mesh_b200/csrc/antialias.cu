// antialias.cu -- stage-1 mesh path, third operator: silhouette antialiasing of a rasterised image with gradients to the colours AND
// to the clip-space vertex positions, replacing `dr.antialias` of nvdiffrast as the reference calls it at nerf/renderer.py:886-887
//     alphas = dr.antialias(alphas, rast, vertices_clip, self.triangles, pos_gradient_boost=...)
//     rgbs   = dr.antialias(rgbs,   rast, vertices_clip, self.triangles, pos_gradient_boost=...)
// (the only differentiable path from the image loss to `vertices_offsets` when enable_offset_nerf_grad is off).  Algorithm as
// published (Laine et al. 2020, section 3.4) and restated in oracle/antialias_oracle.py, which is the checker of these kernels:
// per pair of horizontally / vertically adjacent pixels with different triangle ids, the first edge of the FOREGROUND pixel's
// triangle that crosses strictly between the two pixel centres, if it is a silhouette edge, blends the two colours by the position
// of the crossing: alpha = t - 0.5;  out[alpha > 0 ? Q : P] += alpha * (in[P] - in[Q]).
//
// Shape of the work (HBM / L2-atomic bound integer + fp32 work, no tensor cores):
//   k_aa_topology : one thread per triangle inserts its three edges into an open-addressing hash (64-bit key (min, max) vertex,
//                   value = the opposing vertex of up to two triangles) with atomicCAS; built once per mesh (the reference's mesh
//                   only changes at re-meshing), 16 B per slot, load factor <= 0.5
//   k_aa_forward  : one thread per pixel analyses its right and its lower pair INLINE (at F ~ 3e5 triangles on 1600^2 most pairs
//                   have different ids, so a discontinuity work queue would hold nearly every pair); the silhouette test costs one
//                   hash probe and runs only for the one edge that crosses; blends land with red.global.add.f32 on `out`, which the
//                   entry point pre-fills with a device-to-device copy of the input
//   k_aa_backward : the same analysis (recomputed, nothing is stored by the forward pass), colour gradients +-alpha * g, and the
//                   gradient of t through the crossing point to x, y, w of the edge's two vertices
// All geometry is evaluated relative to the foreground pixel's centre, so the fp32 decisions (straddle, 0 < t < 1, fold test) agree
// with the float64 oracle except for crossings within rounding of a pixel centre.
#include "n2m_common.cuh"
#include "topology_hash.cuh"
#include "../../include/n2m_b200_raster.h"

namespace n2m {
namespace {

__global__ void __launch_bounds__(256)
k_aa_topology(const int32_t* __restrict__ tri, uint32_t F, unsigned long long* __restrict__ keys, int32_t* __restrict__ opp, uint32_t mask) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int v[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int a = v[e], b = v[(e + 1) % 3], o = v[(e + 2) % 3];
        if (a == b) continue;
        const unsigned long long key = ((unsigned long long)(uint32_t)min(a, b) << 32) | (unsigned long long)(uint32_t)max(a, b);
        uint32_t h = aa_hash(key) & mask;
        for (uint32_t probe = 0; probe <= mask; ++probe) {
            const unsigned long long prev = atomicCAS(keys + h, kEmptyKey, key);
            if (prev == kEmptyKey || prev == key) {
                if (atomicCAS(opp + 2 * h, -1, o) != -1) atomicCAS(opp + 2 * h + 1, -1, o);       // a third triangle on the edge is dropped
                break;
            }
            h = (h + 1) & mask;
        }
    }
}

// the other triangle's opposing vertex of edge (a, b) seen from the triangle whose opposing vertex is o:  -1 = boundary edge
__device__ __forceinline__ int aa_other_opp(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ opp, uint32_t mask,
                                            int a, int b, int o, bool& found) {
    const unsigned long long key = ((unsigned long long)(uint32_t)min(a, b) << 32) | (unsigned long long)(uint32_t)max(a, b);
    uint32_t h = aa_hash(key) & mask;
    found = false;
    for (uint32_t probe = 0; probe <= mask; ++probe) {
        const unsigned long long k = keys[h];
        if (k == key) {
            found = true;
            const int o0 = opp[2 * h], o1 = opp[2 * h + 1];
            return (o0 == o) ? o1 : o0;
        }
        if (k == kEmptyKey) return -1;
        h = (h + 1) & mask;
    }
    return -1;
}

struct AAHit {
    uint32_t P, Q, dst;          // flat pixel indices
    float alpha;
    int va, vb;                  // the edge's vertices
    float gax, gay, gbx, gby;    // d t / d (screen x, y) of va, vb
};

// analysis of the pair (pixel i, its right (d = 0) or lower (d = 1) neighbour); see oracle/antialias_oracle.py:analyze_pair
__device__ __forceinline__ bool aa_analyze(uint32_t px, uint32_t py, int d, const float4* __restrict__ rast, const float4* __restrict__ pos,
                                           const int32_t* __restrict__ tri, const unsigned long long* __restrict__ keys,
                                           const int32_t* __restrict__ opp, uint32_t mask, uint32_t H, uint32_t W, float4 r0, AAHit& hit) {
    const uint32_t qx = px + (d == 0), qy = py + (d == 1);
    if (qx >= W || qy >= H) return false;
    const float4 r1 = rast[(size_t)qy * W + qx];
    const int id0 = (int)r0.w, id1 = (int)r1.w;
    if (id0 == id1) return false;
    int fg;
    if (id0 == 0) fg = 1;
    else if (id1 == 0) fg = 0;
    else fg = (r0.z < r1.z) ? 0 : 1;
    const uint32_t Px = fg ? qx : px, Py = fg ? qy : py, Qx = fg ? px : qx, Qy = fg ? py : qy;
    const float s = fg ? -1.f : 1.f;                              // Q lies in the positive (fg == 0) or negative direction from P
    const uint32_t f = (uint32_t)(fg ? id1 : id0) - 1u;
    const int v[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
    const float4 p[3] = {__ldg(pos + v[0]), __ldg(pos + v[1]), __ldg(pos + v[2])};
    if (!(p[0].w > 0.f && p[1].w > 0.f && p[2].w > 0.f)) return false;
    const float cx = (float)Px + 0.5f, cy = (float)Py + 0.5f;
    float sx[3], sy[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float rw = __fdiv_rn(1.f, p[k].w);
        sx[k] = (p[k].x * rw * 0.5f + 0.5f) * (float)W - cx;       // relative to P's centre
        sy[k] = (p[k].y * rw * 0.5f + 0.5f) * (float)H - cy;
    }
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int ia = e, ib = (e + 1) % 3, io = (e + 2) % 3;
        const float ax = sx[ia], ay = sy[ia], bx = sx[ib], by = sy[ib];
        float t, gax, gay, gbx, gby;
        if (d == 0) {
            if ((ay < 0.f) == (by < 0.f)) continue;
            const float inv = __fdiv_rn(1.f, by - ay);
            const float u = -ay * inv;
            t = s * (ax + (bx - ax) * u);
            gax = s * (1.f - u); gay = -s * (bx - ax) * (1.f - u) * inv; gbx = s * u; gby = -s * (bx - ax) * u * inv;
        } else {
            if ((ax < 0.f) == (bx < 0.f)) continue;
            const float inv = __fdiv_rn(1.f, bx - ax);
            const float u = -ax * inv;
            t = s * (ay + (by - ay) * u);
            gax = -s * (by - ay) * (1.f - u) * inv; gay = s * (1.f - u); gbx = -s * (by - ay) * u * inv; gby = s * u;
        }
        if (!(t > 0.f && t < 1.f)) continue;
        bool found;
        const int o2 = aa_other_opp(keys, opp, mask, v[ia], v[ib], v[io], found);
        if (!found) return false;                                  // degenerate edge (a == b): not in the table
        if (o2 >= 0) {
            const float4 q = __ldg(pos + o2);
            if (!(q.w > 0.f)) return false;
            const float rw = __fdiv_rn(1.f, q.w);
            const float ox2 = (q.x * rw * 0.5f + 0.5f) * (float)W - cx, oy2 = (q.y * rw * 0.5f + 0.5f) * (float)H - cy;
            const float ex = bx - ax, ey = by - ay;
            const float s1 = ex * (sy[io] - ay) - ey * (sx[io] - ax);
            const float s2 = ex * (oy2 - ay) - ey * (ox2 - ax);
            if (!(s1 * s2 > 0.f)) return false;                    // the neighbour continues on the other side: an interior edge
        }
        hit.alpha = t - 0.5f;
        hit.P = Py * W + Px; hit.Q = Qy * W + Qx;
        hit.dst = hit.alpha > 0.f ? hit.Q : hit.P;
        hit.va = v[ia]; hit.vb = v[ib];
        hit.gax = gax; hit.gay = gay; hit.gbx = gbx; hit.gby = gby;
        return true;
    }
    return false;
}

template <int C>
__global__ void __launch_bounds__(256)
k_aa_forward(const float* __restrict__ color, const float4* __restrict__ rast, const float4* __restrict__ pos, const int32_t* __restrict__ tri,
             const unsigned long long* __restrict__ keys, const int32_t* __restrict__ opp, uint32_t mask, uint32_t H, uint32_t W,
             float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const uint32_t px = i % W, py = i / W;
    const float4 r0 = rast[i];
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        AAHit h;
        if (!aa_analyze(px, py, d, rast, pos, tri, keys, opp, mask, H, W, r0, h)) continue;
#pragma unroll
        for (int c = 0; c < C; ++c)
            atomicAdd(out + (size_t)h.dst * C + c, h.alpha * (color[(size_t)h.P * C + c] - color[(size_t)h.Q * C + c]));
    }
}

template <int C>
__global__ void __launch_bounds__(256)
k_aa_backward(const float* __restrict__ color, const float4* __restrict__ rast, const float4* __restrict__ pos, const int32_t* __restrict__ tri,
              const unsigned long long* __restrict__ keys, const int32_t* __restrict__ opp, uint32_t mask, uint32_t H, uint32_t W,
              const float* __restrict__ grad_out, float boost, float* __restrict__ grad_color, float* __restrict__ grad_pos) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const uint32_t px = i % W, py = i / W;
    const float4 r0 = rast[i];
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        AAHit h;
        if (!aa_analyze(px, py, d, rast, pos, tri, keys, opp, mask, H, W, r0, h)) continue;
        float dt = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const float g = grad_out[(size_t)h.dst * C + c];
            dt += g * (color[(size_t)h.P * C + c] - color[(size_t)h.Q * C + c]);
            if (grad_color) {
                atomicAdd(grad_color + (size_t)h.P * C + c, h.alpha * g);
                atomicAdd(grad_color + (size_t)h.Q * C + c, -h.alpha * g);
            }
        }
        if (!grad_pos || dt == 0.f) continue;
        dt *= boost;
        const int vs[2] = {h.va, h.vb};
        const float gx[2] = {h.gax, h.gbx}, gy[2] = {h.gay, h.gby};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float4 q = __ldg(pos + vs[k]);
            const float rw = __fdiv_rn(1.f, q.w);
            const float dsx = dt * gx[k] * 0.5f * (float)W * rw, dsy = dt * gy[k] * 0.5f * (float)H * rw;      // d / d clip x, y
            atomicAdd(grad_pos + 4 * (size_t)vs[k] + 0, dsx);
            atomicAdd(grad_pos + 4 * (size_t)vs[k] + 1, dsy);
            atomicAdd(grad_pos + 4 * (size_t)vs[k] + 3, -(dsx * q.x + dsy * q.y) * rw);
        }
    }
}

__global__ void __launch_bounds__(256)
k_aa_clear(unsigned long long* __restrict__ keys, int32_t* __restrict__ opp, uint32_t slots) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < slots) { keys[i] = kEmptyKey; opp[2 * i] = -1; opp[2 * i + 1] = -1; }
}

inline bool pow2(uint32_t x) { return x && !(x & (x - 1)); }

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

uint32_t n2m_antialias_topology_slots(uint32_t F) {
    uint32_t s = 16;
    while (s < 3u * F && s < (1u << 31)) s <<= 1;
    return s;
}

int n2m_antialias_topology(const int32_t* tri, uint32_t F, void* keys, int32_t* opp, uint32_t slots, n2m_stream_t stream) {
    N2M_REQUIRE(tri && keys && opp, "antialias_topology", "null pointer");
    N2M_REQUIRE(pow2(slots) && (uint64_t)slots >= 3ull * F, "antialias_topology", "slots must be a power of two >= 3 F (n2m_antialias_topology_slots)");
    cudaStream_t st = as_stream(stream);
    k_aa_clear<<<div_up(slots, 256u), 256, 0, st>>>(static_cast<unsigned long long*>(keys), opp, slots);
    if (int e = check_launch("antialias_topology(clear)")) return e;
    if (F == 0) return 0;
    k_aa_topology<<<div_up(F, 256u), 256, 0, st>>>(tri, F, static_cast<unsigned long long*>(keys), opp, slots - 1);
    return check_launch("antialias_topology");
}

int n2m_antialias_forward(const float* color, const float* rast, const float* pos, const int32_t* tri, const void* keys, const int32_t* opp,
                          uint32_t slots, uint32_t H, uint32_t W, uint32_t C, float* out, n2m_stream_t stream) {
    N2M_REQUIRE(color && rast && pos && tri && keys && opp && out, "antialias_forward", "null pointer");
    N2M_REQUIRE(pow2(slots), "antialias_forward", "slots must be a power of two");
    N2M_REQUIRE(C >= 1 && C <= 4, "antialias_forward", "1..4 channels are supported");
    const uint32_t n = H * W;
    if (n == 0) return 0;
    cudaStream_t st = as_stream(stream);
    if (out != color) {
        cudaError_t e = cudaMemcpyAsync(out, color, (size_t)n * C * sizeof(float), cudaMemcpyDeviceToDevice, st);
        if (e != cudaSuccess) return fail("antialias_forward(copy)", cudaGetErrorString(e));
    } else {
        return fail("antialias_forward", "out must not alias color");
    }
    const float4* r = reinterpret_cast<const float4*>(rast);
    const float4* p = reinterpret_cast<const float4*>(pos);
    const unsigned long long* k = static_cast<const unsigned long long*>(keys);
    const uint32_t g = div_up(n, 256u);
    switch (C) {
        case 1: k_aa_forward<1><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, out); break;
        case 2: k_aa_forward<2><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, out); break;
        case 3: k_aa_forward<3><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, out); break;
        default: k_aa_forward<4><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, out); break;
    }
    return check_launch("antialias_forward");
}

int n2m_antialias_backward(const float* color, const float* rast, const float* pos, const int32_t* tri, const void* keys, const int32_t* opp,
                           uint32_t slots, uint32_t H, uint32_t W, uint32_t C, const float* grad_out, float pos_gradient_boost,
                           float* grad_color, float* grad_pos, n2m_stream_t stream) {
    N2M_REQUIRE(color && rast && pos && tri && keys && opp && grad_out, "antialias_backward", "null pointer");
    N2M_REQUIRE(grad_color || grad_pos, "antialias_backward", "nothing to compute");
    N2M_REQUIRE(pow2(slots), "antialias_backward", "slots must be a power of two");
    N2M_REQUIRE(C >= 1 && C <= 4, "antialias_backward", "1..4 channels are supported");
    N2M_REQUIRE(grad_color != grad_out, "antialias_backward", "grad_color must not alias grad_out");
    const uint32_t n = H * W;
    if (n == 0) return 0;
    cudaStream_t st = as_stream(stream);
    if (grad_color) {
        cudaError_t e = cudaMemcpyAsync(grad_color, grad_out, (size_t)n * C * sizeof(float), cudaMemcpyDeviceToDevice, st);
        if (e != cudaSuccess) return fail("antialias_backward(copy)", cudaGetErrorString(e));
    }
    const float4* r = reinterpret_cast<const float4*>(rast);
    const float4* p = reinterpret_cast<const float4*>(pos);
    const unsigned long long* k = static_cast<const unsigned long long*>(keys);
    const uint32_t g = div_up(n, 256u);
    switch (C) {
        case 1: k_aa_backward<1><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, grad_out, pos_gradient_boost, grad_color, grad_pos); break;
        case 2: k_aa_backward<2><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, grad_out, pos_gradient_boost, grad_color, grad_pos); break;
        case 3: k_aa_backward<3><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, grad_out, pos_gradient_boost, grad_color, grad_pos); break;
        default: k_aa_backward<4><<<g, 256, 0, st>>>(color, r, p, tri, k, opp, slots - 1, H, W, grad_out, pos_gradient_boost, grad_color, grad_pos); break;
    }
    return check_launch("antialias_backward");
}

}  // extern "C"
