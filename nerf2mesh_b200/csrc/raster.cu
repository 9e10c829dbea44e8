// raster.cu -- stage-1 mesh path: triangle rasterization and attribute interpolation as
// sm_90a kernels, replacing the two nvdiffrast operators the reference calls at nerf/renderer.py:860-863 (`dr.rasterize`,
// `dr.interpolate`); output convention (u, v, z/w, triangle_id + 1) as consumed at renderer.py:890,894.
//
// Design (HBM / L2-atomic bound integer work, no tensor cores): a VISIBILITY BUFFER of one 64-bit word per pixel,
//     key = (order-preserving 32-bit image of z/w) << 32 | (triangle_id + 1),
// resolved with atomicMin -- the nearest fragment wins, ties go to the lower triangle id, and the result does not depend on the
// order in which triangles are processed (deterministic, unlike a read-modify-write z-buffer).
//   k_rast_clear     : keys = ~0
//   k_rast_small     : one thread per triangle: clip -> NDC -> pixel coordinates, bounding box; triangles covering <= 64 pixel centres
//                      of bounding box are rasterised inline (the common case at F ~ 3e5 on a 1600^2 target: a few pixels each),
//                      larger ones go to a queue
//   k_rast_large     : one block per queued triangle, threads stride over its bounding box (persistent grid sized by the SM count,
//                      queue length read on the device: no host synchronisation)
//   k_rast_resolve   : one thread per pixel: decode the winner, recompute its screen-space barycentrics with the SAME fp32 expressions,
//                      make them perspective-correct with the clip-space w, write (u, v, z/w, id + 1) as one float4
//   k_interp_fwd/bwd : attr = u a0 + v a1 + (1-u-v) a2 per pixel; backward scatters to the three vertices with red.global.add
//   k_interp_bwd_rast, k_rast_bwd : the gradients of interpolate w.r.t. rast's (u, v) and of rasterize w.r.t. pos through (u, v), as
//                      nvdiffrast defines them (arithmetic in raster_grad.cuh, shared with the stage-1 step's k_s1_offset_grad)
// Near / far clipping: triangles in front of the camera plane (all w > 0) are tested per pixel against -1 <= z/w <= 1.  Triangles that
// CROSS the camera plane (some w <= 0: ground or shell triangles around a camera inside the scene) are rasterised in 2-D homogeneous
// coordinates (Olano & Greer 1997): for pixel NDC (X, Y) the solution of sum_i b'_i (x_i, y_i, w_i) = (X, Y, 1) is non-negative exactly
// on the part of the triangle in front of the camera, z/w = sum_i b'_i z_i gets the same [-1, 1] test, (u, v) = (b'_0, b'_1) / sum b'
// -- the result of clipping against the near plane without building clipped polygons; only the bounding box comes from the clipped
// outline.  Not reproduced (oracle/raster_oracle.py): the exact OpenGL top-left fill rule for pixel centres exactly on an edge.
#include "n2m_common.cuh"
#include "raster_grad.cuh"
#include "../../include/n2m_b200_raster.h"

namespace n2m {
namespace {

constexpr uint32_t kInlinePixels = 64;

struct TriSetup {
    float x0, y0, x1, y1, x2, y2;     // pixel coordinates (pixel centre x + 0.5);  homogeneous path: rows 0 / 1 of adj(M) (A, B) pairs
    float z0, z1, z2;                 // NDC depth;  homogeneous path: clip-space z
    float w0, w1, w2;                 // clip w;  homogeneous path: the constant terms C_k of the three solutions
    float inv_area;                   // homogeneous path: 1 / det(M)
    float a2, b2;                     // homogeneous path: (A_2, B_2)
    int xa, xb, ya, yb;               // inclusive pixel bounding box, clamped to the target
    bool valid;
    bool homog;                       // the triangle crosses the camera plane (one or two vertices at w <= 0)
};

// pixel bounding box of the triangle clipped against the near plane z >= -w (Sutherland-Hodgman, at most four points)
__device__ __forceinline__ bool near_clip_bbox(const float4 p0, const float4 p1, const float4 p2, uint32_t H, uint32_t W, int& xa, int& xb, int& ya, int& yb) {
    const float4 poly[3] = {p0, p1, p2};
    float xmin = 3.4e38f, xmax = -3.4e38f, ymin = 3.4e38f, ymax = -3.4e38f;
    bool any = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 a = poly[k], b = poly[(k + 1) % 3];
        const float da = a.z + a.w, db = b.z + b.w;
        float4 q[2]; int n = 0;
        if (da >= 0.f) q[n++] = a;
        if ((da >= 0.f) != (db >= 0.f)) {
            const float t = __fdiv_rn(da, da - db);
            q[n++] = make_float4(a.x + t * (b.x - a.x), a.y + t * (b.y - a.y), a.z + t * (b.z - a.z), a.w + t * (b.w - a.w));
        }
        for (int j = 0; j < n; ++j) {
            const float rw = __fdiv_rn(1.f, fmaxf(q[j].w, 1e-30f));
            const float sx = (q[j].x * rw * 0.5f + 0.5f) * (float)W, sy = (q[j].y * rw * 0.5f + 0.5f) * (float)H;
            xmin = fminf(xmin, sx); xmax = fmaxf(xmax, sx); ymin = fminf(ymin, sy); ymax = fmaxf(ymax, sy);
            any = true;
        }
    }
    if (!any) return false;
    xa = max((int)floorf(fminf(xmin, (float)W + 1.f) - 0.5f), 0); xb = min((int)ceilf(fmaxf(xmax, -1.f) - 0.5f), (int)W - 1);
    ya = max((int)floorf(fminf(ymin, (float)H + 1.f) - 0.5f), 0); yb = min((int)ceilf(fmaxf(ymax, -1.f) - 0.5f), (int)H - 1);
    return xa <= xb && ya <= yb;
}

__device__ __forceinline__ TriSetup setup_tri(const float4* __restrict__ pos, const int32_t* __restrict__ tri, uint32_t f, uint32_t H, uint32_t W) {
    TriSetup t;
    const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
    const float4 p0 = __ldg(pos + i0), p1 = __ldg(pos + i1), p2 = __ldg(pos + i2);
    t.homog = false;
    t.a2 = t.b2 = 0.f;
    t.valid = p0.w > 0.f && p1.w > 0.f && p2.w > 0.f;
    if (!t.valid && (p0.w > 0.f || p1.w > 0.f || p2.w > 0.f)) {
        // crosses the camera plane: b'_k = (A_k X + B_k Y + C_k) / det, (A_k, B_k, C_k) = row k of adj(M), M = [x; y; w] of the vertices
        t.homog = true;
        t.x0 = p1.y * p2.w - p2.y * p1.w; t.y0 = p2.x * p1.w - p1.x * p2.w; t.w0 = p1.x * p2.y - p2.x * p1.y;
        t.x1 = p2.y * p0.w - p0.y * p2.w; t.y1 = p0.x * p2.w - p2.x * p0.w; t.w1 = p2.x * p0.y - p0.x * p2.y;
        t.a2 = p0.y * p1.w - p1.y * p0.w; t.b2 = p1.x * p0.w - p0.x * p1.w; t.w2 = p0.x * p1.y - p1.x * p0.y;
        t.x2 = t.y2 = 0.f;
        const float det = p0.x * t.x0 + p1.x * t.x1 + p2.x * t.a2;
        t.z0 = p0.z; t.z1 = p1.z; t.z2 = p2.z;
        t.valid = det != 0.f && isfinite(det);
        t.inv_area = t.valid ? __fdiv_rn(1.f, det) : 0.f;
        t.xa = t.ya = 0; t.xb = t.yb = -1;
        if (t.valid) t.valid = near_clip_bbox(p0, p1, p2, H, W, t.xa, t.xb, t.ya, t.yb);
        return t;
    }
    t.w0 = p0.w; t.w1 = p1.w; t.w2 = p2.w;
    const float r0 = __fdiv_rn(1.f, p0.w), r1 = __fdiv_rn(1.f, p1.w), r2 = __fdiv_rn(1.f, p2.w);
    const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;
    t.x0 = (p0.x * r0 * 0.5f + 0.5f) * (float)W; t.y0 = (p0.y * r0 * 0.5f + 0.5f) * (float)H;
    t.x1 = (p1.x * r1 * 0.5f + 0.5f) * (float)W; t.y1 = (p1.y * r1 * 0.5f + 0.5f) * (float)H;
    t.x2 = (p2.x * r2 * 0.5f + 0.5f) * (float)W; t.y2 = (p2.y * r2 * 0.5f + 0.5f) * (float)H;
    (void)hw; (void)hh;
    t.z0 = p0.z * r0; t.z1 = p1.z * r1; t.z2 = p2.z * r2;
    const float area = (t.x1 - t.x0) * (t.y2 - t.y0) - (t.x2 - t.x0) * (t.y1 - t.y0);
    t.valid = t.valid && area != 0.f && isfinite(area);
    t.inv_area = t.valid ? __fdiv_rn(1.f, area) : 0.f;
    const float xmin = fminf(t.x0, fminf(t.x1, t.x2)), xmax = fmaxf(t.x0, fmaxf(t.x1, t.x2));
    const float ymin = fminf(t.y0, fminf(t.y1, t.y2)), ymax = fmaxf(t.y0, fmaxf(t.y1, t.y2));
    // pixel x is a candidate when its centre x + 0.5 lies in [xmin, xmax]
    t.xa = max((int)floorf(xmin - 0.5f), 0); t.xb = min((int)ceilf(xmax - 0.5f), (int)W - 1);
    t.ya = max((int)floorf(ymin - 0.5f), 0); t.yb = min((int)ceilf(ymax - 0.5f), (int)H - 1);
    if (!(xmax >= 0.f && xmin <= (float)W && ymax >= 0.f && ymin <= (float)H)) t.valid = false;      // also rejects NaN
    if (t.xa > t.xb || t.ya > t.yb) t.valid = false;
    return t;
}

// screen-space barycentrics of pixel centre (px, py); returns false when the centre is outside the triangle
__device__ __forceinline__ bool bary(const TriSetup& t, float px, float py, float& b0, float& b1, float& b2) {
    b0 = ((t.x1 - px) * (t.y2 - py) - (t.x2 - px) * (t.y1 - py)) * t.inv_area;
    b1 = ((t.x2 - px) * (t.y0 - py) - (t.x0 - px) * (t.y2 - py)) * t.inv_area;
    b2 = 1.0f - b0 - b1;
    return b0 >= 0.f && b1 >= 0.f && b2 >= 0.f;
}

// homogeneous path: the three solutions b'_k at pixel (x, y); false when the pixel is not covered in front of the camera
__device__ __forceinline__ bool bary_homog(const TriSetup& t, int x, int y, uint32_t H, uint32_t W, float& b0, float& b1, float& b2) {
    const float X = ((float)x + 0.5f) * __fdiv_rn(2.f, (float)W) - 1.f, Y = ((float)y + 0.5f) * __fdiv_rn(2.f, (float)H) - 1.f;
    b0 = (t.x0 * X + t.y0 * Y + t.w0) * t.inv_area;
    b1 = (t.x1 * X + t.y1 * Y + t.w1) * t.inv_area;
    b2 = (t.a2 * X + t.b2 * Y + t.w2) * t.inv_area;
    return b0 >= 0.f && b1 >= 0.f && b2 >= 0.f;
}

__device__ __forceinline__ uint32_t depth_key(float z) {          // order-preserving map float -> uint32
    const uint32_t u = __float_as_uint(z);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ void shade_pixel(const TriSetup& t, uint32_t f, int x, int y, uint32_t H, uint32_t W, unsigned long long* __restrict__ vis) {
    float b0, b1, b2;
    if (t.homog) { if (!bary_homog(t, x, y, H, W, b0, b1, b2)) return; }
    else if (!bary(t, (float)x + 0.5f, (float)y + 0.5f, b0, b1, b2)) return;
    const float z = b0 * t.z0 + b1 * t.z1 + b2 * t.z2;
    if (!(z >= -1.f && z <= 1.f)) return;
    const unsigned long long key = ((unsigned long long)depth_key(z) << 32) | (unsigned long long)(f + 1u);
    atomicMin(vis + (size_t)y * W + x, key);
}

__global__ void __launch_bounds__(256)
k_rast_clear(unsigned long long* __restrict__ vis, uint32_t n, uint32_t* __restrict__ queue) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) vis[i] = ~0ull;
    if (i == 0) queue[0] = 0;
}

__global__ void __launch_bounds__(256)
k_rast_small(const float4* __restrict__ pos, const int32_t* __restrict__ tri, uint32_t F, uint32_t H, uint32_t W,
             unsigned long long* __restrict__ vis, uint32_t* __restrict__ queue) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const TriSetup t = setup_tri(pos, tri, f, H, W);
    if (!t.valid) return;
    const uint32_t bw = (uint32_t)(t.xb - t.xa + 1), bh = (uint32_t)(t.yb - t.ya + 1);
    if (bw * bh > kInlinePixels) { queue[1 + atomicAdd(queue, 1u)] = f; return; }
    for (int y = t.ya; y <= t.yb; ++y)
        for (int x = t.xa; x <= t.xb; ++x) shade_pixel(t, f, x, y, H, W, vis);
}

__global__ void __launch_bounds__(256)
k_rast_large(const float4* __restrict__ pos, const int32_t* __restrict__ tri, uint32_t H, uint32_t W,
             unsigned long long* __restrict__ vis, const uint32_t* __restrict__ queue) {
    const uint32_t count = queue[0];
    for (uint32_t q = blockIdx.x; q < count; q += gridDim.x) {
        const uint32_t f = queue[1 + q];
        const TriSetup t = setup_tri(pos, tri, f, H, W);
        const uint32_t bw = (uint32_t)(t.xb - t.xa + 1), n = bw * (uint32_t)(t.yb - t.ya + 1);
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) shade_pixel(t, f, t.xa + (int)(i % bw), t.ya + (int)(i / bw), H, W, vis);
    }
}

__global__ void __launch_bounds__(256)
k_rast_resolve(const float4* __restrict__ pos, const int32_t* __restrict__ tri, uint32_t H, uint32_t W,
               const unsigned long long* __restrict__ vis, float4* __restrict__ rast) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const unsigned long long key = vis[i];
    if (key == ~0ull) { rast[i] = make_float4(0.f, 0.f, 0.f, 0.f); return; }
    const uint32_t f = (uint32_t)(key & 0xffffffffull) - 1u;
    const TriSetup t = setup_tri(pos, tri, f, H, W);
    float b0, b1, b2;
    if (t.homog) {
        bary_homog(t, (int)(i % W), (int)(i / W), H, W, b0, b1, b2);
        const float zh = b0 * t.z0 + b1 * t.z1 + b2 * t.z2;
        const float invs = __fdiv_rn(1.f, b0 + b1 + b2);
        rast[i] = make_float4(b0 * invs, b1 * invs, zh, (float)(f + 1u));
        return;
    }
    bary(t, (float)(i % W) + 0.5f, (float)(i / W) + 0.5f, b0, b1, b2);
    const float z = b0 * t.z0 + b1 * t.z1 + b2 * t.z2;
    const float p0 = __fdiv_rn(b0, t.w0), p1 = __fdiv_rn(b1, t.w1), p2 = __fdiv_rn(b2, t.w2);
    const float inv = __fdiv_rn(1.f, p0 + p1 + p2);
    rast[i] = make_float4(p0 * inv, p1 * inv, z, (float)(f + 1u));
}

template <int A>
__global__ void __launch_bounds__(256)
k_interp_fwd(const float* __restrict__ attr, const float4* __restrict__ rast, const int32_t* __restrict__ tri, uint32_t n,
             float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 r = rast[i];
    float v[A];
#pragma unroll
    for (int a = 0; a < A; ++a) v[a] = 0.f;
    if (r.w > 0.f) {
        const uint32_t f = (uint32_t)r.w - 1u;
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        const float u = r.x, vv = r.y, w = 1.f - r.x - r.y;
#pragma unroll
        for (int a = 0; a < A; ++a) v[a] = u * __ldg(attr + (size_t)i0 * A + a) + vv * __ldg(attr + (size_t)i1 * A + a) + w * __ldg(attr + (size_t)i2 * A + a);
    }
#pragma unroll
    for (int a = 0; a < A; ++a) out[(size_t)i * A + a] = v[a];
}

template <int A>
__global__ void __launch_bounds__(256)
k_interp_bwd(const float* __restrict__ grad_out, const float4* __restrict__ rast, const int32_t* __restrict__ tri, uint32_t n,
             float* __restrict__ grad_attr) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 r = rast[i];
    if (!(r.w > 0.f)) return;
    const uint32_t f = (uint32_t)r.w - 1u;
    const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
    const float u = r.x, v = r.y, w = 1.f - r.x - r.y;
#pragma unroll
    for (int a = 0; a < A; ++a) {
        const float g = grad_out[(size_t)i * A + a];
        atomicAdd(grad_attr + (size_t)i0 * A + a, u * g);
        atomicAdd(grad_attr + (size_t)i1 * A + a, v * g);
        atomicAdd(grad_attr + (size_t)i2 * A + a, w * g);
    }
}

// dr.rasterize backward: one thread per pixel, d loss / d (u, v) of the covered pixels -> grad_pos [V,4] (raster_grad.cuh)
__global__ void __launch_bounds__(256)
k_rast_bwd(const float4* __restrict__ pos, const int32_t* __restrict__ tri, const float4* __restrict__ rast, const float4* __restrict__ grad_rast,
           uint32_t H, uint32_t W, float* __restrict__ grad_pos) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const float4 r = rast[i];
    if (!(r.w > 0.f)) return;
    const float4 g = grad_rast[i];
    if (g.x == 0.f && g.y == 0.f) return;
    const uint32_t f = (uint32_t)r.w - 1u;
    const int vi[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
    const float4 p[3] = {__ldg(pos + vi[0]), __ldg(pos + vi[1]), __ldg(pos + vi[2])};
    const float2 ndc = pixel_ndc(i % W, i / W, H, W);
    rasterize_uv_backward(p, vi, ndc.x, ndc.y, g.x, g.y, grad_pos);
}

// dr.interpolate backward w.r.t. rast: grad_rast [n,4] = (du, dv, 0, 0) at covered pixels, zeros elsewhere (raster_grad.cuh)
template <int A>
__global__ void __launch_bounds__(256)
k_interp_bwd_rast(const float* __restrict__ grad_out, const float* __restrict__ attr, const float4* __restrict__ rast, const int32_t* __restrict__ tri,
                  uint32_t n, float4* __restrict__ grad_rast) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 r = rast[i];
    float2 d = make_float2(0.f, 0.f);
    if (r.w > 0.f) {
        const uint32_t f = (uint32_t)r.w - 1u;
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        float g[A], a0[A], a1[A], a2[A];
#pragma unroll
        for (int a = 0; a < A; ++a) {
            g[a] = grad_out[(size_t)i * A + a];
            a0[a] = __ldg(attr + (size_t)i0 * A + a); a1[a] = __ldg(attr + (size_t)i1 * A + a); a2[a] = __ldg(attr + (size_t)i2 * A + a);
        }
        d = interpolate_uv_backward<A>(g, a0, a1, a2);
    }
    grad_rast[i] = make_float4(d.x, d.y, 0.f, 0.f);
}

// covered-pixel compaction for the texture-MLP step (renderer.py:865-880: xyzs[mask_flatten], dirs[mask_flatten]): one thread per
// pixel, warp-aggregated atomic counter; writes the pixel index, its interpolated position and its (unnormalised) view direction
__global__ void __launch_bounds__(256)
k_compact_covered(const float4* __restrict__ rast, const float* __restrict__ xyz, const float* __restrict__ dirs, uint32_t n, uint32_t cap,
                  int32_t* __restrict__ counter, int32_t* __restrict__ pix, float* __restrict__ pts, float* __restrict__ pdirs) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool cov = i < n && rast[i].w > 0.f;
    const uint32_t mask = __ballot_sync(0xffffffffu, cov);
    if (mask == 0) return;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t base = 0;
    if (lane == (uint32_t)(__ffs(mask) - 1)) base = (uint32_t)atomicAdd(counter, (int)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, __ffs(mask) - 1);
    if (!cov) return;
    const uint32_t k = base + __popc(mask & ((1u << lane) - 1u));
    if (k >= cap) return;
    pix[k] = (int32_t)i;
#pragma unroll
    for (int a = 0; a < 3; ++a) { pts[3 * k + a] = xyz[3 * (size_t)i + a]; pdirs[3 * k + a] = dirs[3 * (size_t)i + a]; }
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_rasterize(const float* pos, uint32_t V, const int32_t* tri, uint32_t F, uint32_t H, uint32_t W, void* vis, uint32_t* queue,
                  float* rast, n2m_stream_t stream) {
    N2M_REQUIRE(pos && tri && vis && queue && rast, "rasterize", "null pointer");
    N2M_REQUIRE(H > 0 && W > 0 && (uint64_t)H * W < (1ull << 31), "rasterize", "bad resolution");
    (void)V;
    cudaStream_t st = as_stream(stream);
    const uint32_t n = H * W;
    k_rast_clear<<<div_up(n, 256u), 256, 0, st>>>(static_cast<unsigned long long*>(vis), n, queue);
    if (int e = check_launch("rasterize(clear)")) return e;
    if (F > 0) {
        k_rast_small<<<div_up(F, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(pos), tri, F, H, W, static_cast<unsigned long long*>(vis), queue);
        if (int e = check_launch("rasterize(small)")) return e;
        k_rast_large<<<num_sms() * 8, 256, 0, st>>>(reinterpret_cast<const float4*>(pos), tri, H, W, static_cast<unsigned long long*>(vis), queue);
        if (int e = check_launch("rasterize(large)")) return e;
    }
    k_rast_resolve<<<div_up(n, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(pos), tri, H, W, static_cast<const unsigned long long*>(vis),
                                                    reinterpret_cast<float4*>(rast));
    return check_launch("rasterize(resolve)");
}

int n2m_interpolate_forward(const float* attr, uint32_t V, uint32_t A, const float* rast, const int32_t* tri, uint32_t num_pixels,
                            float* out, n2m_stream_t stream) {
    N2M_REQUIRE(attr && rast && tri && out, "interpolate_forward", "null pointer");
    (void)V;
    if (num_pixels == 0) return 0;
    const float4* r = reinterpret_cast<const float4*>(rast);
    cudaStream_t st = as_stream(stream);
    const uint32_t g = div_up(num_pixels, 256u);
    switch (A) {
        case 1: k_interp_fwd<1><<<g, 256, 0, st>>>(attr, r, tri, num_pixels, out); break;
        case 2: k_interp_fwd<2><<<g, 256, 0, st>>>(attr, r, tri, num_pixels, out); break;
        case 3: k_interp_fwd<3><<<g, 256, 0, st>>>(attr, r, tri, num_pixels, out); break;
        case 4: k_interp_fwd<4><<<g, 256, 0, st>>>(attr, r, tri, num_pixels, out); break;
        default: return fail("interpolate_forward", "attribute count must be 1..4");
    }
    return check_launch("interpolate_forward");
}

int n2m_interpolate_backward(const float* grad_out, const float* rast, const int32_t* tri, uint32_t num_pixels, uint32_t V, uint32_t A,
                             float* grad_attr, n2m_stream_t stream) {
    N2M_REQUIRE(grad_out && rast && tri && grad_attr, "interpolate_backward", "null pointer");
    (void)V;
    if (num_pixels == 0) return 0;
    const float4* r = reinterpret_cast<const float4*>(rast);
    cudaStream_t st = as_stream(stream);
    const uint32_t g = div_up(num_pixels, 256u);
    switch (A) {
        case 1: k_interp_bwd<1><<<g, 256, 0, st>>>(grad_out, r, tri, num_pixels, grad_attr); break;
        case 2: k_interp_bwd<2><<<g, 256, 0, st>>>(grad_out, r, tri, num_pixels, grad_attr); break;
        case 3: k_interp_bwd<3><<<g, 256, 0, st>>>(grad_out, r, tri, num_pixels, grad_attr); break;
        case 4: k_interp_bwd<4><<<g, 256, 0, st>>>(grad_out, r, tri, num_pixels, grad_attr); break;
        default: return fail("interpolate_backward", "attribute count must be 1..4");
    }
    return check_launch("interpolate_backward");
}

int n2m_rasterize_backward(const float* pos, uint32_t V, const int32_t* tri, const float* rast, const float* grad_rast, uint32_t H, uint32_t W,
                           float* grad_pos, n2m_stream_t stream) {
    N2M_REQUIRE(pos && tri && rast && grad_rast && grad_pos, "rasterize_backward", "null pointer");
    N2M_REQUIRE((uint64_t)H * W < (1ull << 31), "rasterize_backward", "bad resolution");
    (void)V;
    if (H == 0 || W == 0) return 0;
    k_rast_bwd<<<div_up(H * W, 256u), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(pos), tri, reinterpret_cast<const float4*>(rast),
                                                                   reinterpret_cast<const float4*>(grad_rast), H, W, grad_pos);
    return check_launch("rasterize_backward");
}

int n2m_interpolate_backward_rast(const float* grad_out, const float* attr, const float* rast, const int32_t* tri, uint32_t num_pixels, uint32_t A,
                                  float* grad_rast, n2m_stream_t stream) {
    N2M_REQUIRE(grad_out && attr && rast && tri && grad_rast, "interpolate_backward_rast", "null pointer");
    if (num_pixels == 0) return 0;
    const float4* r = reinterpret_cast<const float4*>(rast);
    float4* gr = reinterpret_cast<float4*>(grad_rast);
    cudaStream_t st = as_stream(stream);
    const uint32_t g = div_up(num_pixels, 256u);
    switch (A) {
        case 1: k_interp_bwd_rast<1><<<g, 256, 0, st>>>(grad_out, attr, r, tri, num_pixels, gr); break;
        case 2: k_interp_bwd_rast<2><<<g, 256, 0, st>>>(grad_out, attr, r, tri, num_pixels, gr); break;
        case 3: k_interp_bwd_rast<3><<<g, 256, 0, st>>>(grad_out, attr, r, tri, num_pixels, gr); break;
        case 4: k_interp_bwd_rast<4><<<g, 256, 0, st>>>(grad_out, attr, r, tri, num_pixels, gr); break;
        default: return fail("interpolate_backward_rast", "attribute count must be 1..4");
    }
    return check_launch("interpolate_backward_rast");
}

int n2m_compact_covered(const float* rast, const float* xyz, const float* dirs, uint32_t num_pixels, uint32_t cap, int32_t* counter,
                        int32_t* pix, float* pts, float* pdirs, n2m_stream_t stream) {
    N2M_REQUIRE(rast && xyz && dirs && counter && pix && pts && pdirs, "compact_covered", "null pointer");
    cudaStream_t st = as_stream(stream);
    cudaMemsetAsync(counter, 0, sizeof(int32_t), st);
    if (num_pixels == 0) return 0;
    k_compact_covered<<<div_up(num_pixels, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(rast), xyz, dirs, num_pixels, cap, counter, pix, pts, pdirs);
    return check_launch("compact_covered");
}

}  // extern "C"
