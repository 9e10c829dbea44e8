// stage1.cu -- the texture-MLP step of the reference's stage 1 (NeRFRenderer.render_stage1, nerf/renderer.py:806-935, and the
// stage-1 branch of Trainer.train_step, nerf/utils.py:703-716) around the rasterizer of raster.cu and the stage-0 kernels:
//
//   n2m_rasterize                     dr.rasterize at the super-sampled resolution (h, w) = ssaa * (h0, w0)        renderer.py:824-860
//   n2m_s1_points                     covered pixels -> surface points: attribute interpolation of the vertex positions (dr.interpolate,
//                                     renderer.py:862), nearest-neighbour up-sampling of the view directions (:828-829), compaction
//                                     (xyzs[mask_flatten], :875-877) -- one kernel, no boolean-mask host sync; writes the march-record
//                                     form (t = 0, origin = point) the stage-0 gather / backward kernels consume;
//                                     n2m_s1_points_contract also applies contract() to the points (unbounded scenes, renderer.py:25-32)
//   n2m_s0_encode_points, n2m_s0_mlp_fwd   self.rgb(x, d) (network.py:170-189) on tensor cores (sigma is computed and ignored)
//   n2m_s1_loss                       alphas * rgbs, ssaa average (scale_img_hwc bilinear at factor 2 == 2x2 mean, :899-901), background
//                                     mix (:907), MSE (+ mask) loss (utils.py:707-712) and its gradient w.r.t. every covered pixel's rgb
//   n2m_s0_mlp_bwd, n2m_s0_encode_bwd, n2m_s0_adam_*   backward of the colour MLPs + colour hash table, optimizer
// With dr.antialias (renderer.py:886-887; csrc/antialias.cu) the middle of the step becomes
//   n2m_s1_rgba                       scatter of the per-point colours into a full-resolution (r, g, b, mask) image (`rgbs[mask_flatten] =
//                                     mask_rgbs`, `alphas = mask`, :881-884) -- ONE 4-channel image, so that one antialias launch serves both
//                                     of the reference's calls (the operator is linear and channel-wise)
//   n2m_antialias_forward             alphas, rgbs = dr.antialias(...)                                                  :886-887
//   n2m_s1_loss_aa                    clamp, alphas * rgbs, ssaa average, background mix, loss; gradient w.r.t. the antialiased image
//   n2m_antialias_backward            -> gradient w.r.t. the (r, g, b, mask) image and w.r.t. the clip-space vertices (vertices_offsets)
//   n2m_s1_dout                       gather of the colour gradient back to the compacted points
// With --enable_offset_nerf_grad (xyzs not detached, renderer.py:877-879) the backward adds
//   n2m_s1_offset_grad                after the MLP backward: every point's colour-net + colour-grid input gradient (through contract()),
//                                     back through dr.interpolate and dr.rasterize's (u, v) to the vertices (grad_vworld, grad_vclip)
// and the vertex step becomes n2m_s1_vert_step_world.
// With mesh refinement on (opt.refine), n2m_s1_loss_err / n2m_s1_loss_aa_err replace the two loss launches: the same kernels, which also
// accumulate each pixel's loss and a hit into the face it sees (update_triangles_errors, renderer.py:893-903,923-943; utils.py:720-721).
// Evaluation (render_stage1 at inference: eval_step / test_step, utils.py:853,882) runs the forward part of the step and then
//   n2m_s1_render_compose             clamp, alphas * rgbs, ssaa average, background mix, weights_sum and depth -- no gt, no loss, no gradient
#include "n2m_common.cuh"
#include "raster_grad.cuh"
#include "s0_geom.cuh"
#include "topology_hash.cuh"
#include "../../include/n2m_b200_raster.h"

namespace n2m {
namespace {

// CONTRACT (Stage0Config.contract): the interpolated point goes through contract() (n2m_common.cuh) before it is stored, as the reference
// contracts xyzs before querying the colour field in an unbounded scene; the view directions are unchanged
template <bool CONTRACT>
__global__ void __launch_bounds__(256)
k_s1_points(const float4* __restrict__ rast, const float* __restrict__ verts, const int32_t* __restrict__ tri,
            const float* __restrict__ rays_d, uint32_t h, uint32_t w, uint32_t ssaa, uint32_t cap, int32_t* __restrict__ counters,
            int32_t* __restrict__ inv, float* __restrict__ pts, float* __restrict__ pdirs, float4* __restrict__ recs) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n = h * w;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < n) r = rast[i];
    const bool cov = i < n && r.w > 0.f;
    const uint32_t mask = __ballot_sync(0xffffffffu, cov);
    const uint32_t lane = threadIdx.x & 31;
    uint32_t base = 0;
    if (mask != 0) {
        const int leader = __ffs(mask) - 1;
        if ((int)lane == leader) base = (uint32_t)atomicAdd(counters + 0, (int)__popc(mask));       // [0]: covered pixels (uncapped)
        base = __shfl_sync(0xffffffffu, base, leader);
    }
    if (i >= n) return;
    int32_t slot = -1;
    if (cov) {
        const uint32_t k = base + __popc(mask & ((1u << lane) - 1u));
        if (k < cap) {
            slot = (int32_t)k;
            const uint32_t f = (uint32_t)r.w - 1u;
            const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
            const float u = r.x, v = r.y, ww = 1.f - r.x - r.y;
            const uint32_t y = i / w, x = i % w;
            const uint32_t q = (y / ssaa) * (w / ssaa) + x / ssaa;            // nearest-neighbour source pixel of the low-res direction
            if constexpr (CONTRACT) {
                float p[3];
#pragma unroll
                for (int a = 0; a < 3; ++a)
                    p[a] = u * __ldg(verts + 3 * (size_t)i0 + a) + v * __ldg(verts + 3 * (size_t)i1 + a) + ww * __ldg(verts + 3 * (size_t)i2 + a);
                contract_linf(p);
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    pts[3 * (size_t)k + a] = p[a];
                    pdirs[3 * (size_t)k + a] = __ldg(rays_d + 3 * (size_t)q + a);
                }
            } else {
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    pts[3 * (size_t)k + a] = u * __ldg(verts + 3 * (size_t)i0 + a) + v * __ldg(verts + 3 * (size_t)i1 + a) + ww * __ldg(verts + 3 * (size_t)i2 + a);
                    pdirs[3 * (size_t)k + a] = __ldg(rays_d + 3 * (size_t)q + a);
                }
            }
            recs[k] = make_float4(0.f, 0.f, 0.f, __int_as_float((int)k));      // t = 0: the "sample" is its origin
        }
    }
    inv[i] = slot;
}

// counters[1] = min(counters[0], cap)  (the sample count the stage-0 kernels read), [2] = overflow flag
__global__ void k_s1_finish_count(int32_t* __restrict__ counters, uint32_t cap) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int32_t c = counters[0];
    counters[1] = c < (int32_t)cap ? c : (int32_t)cap;
    counters[2] = c > (int32_t)cap ? 1 : 0;
    counters[3] = 0;
}

// ERR (refinement on): face_err[f] += the pixel's loss before the 1/Q, face_cnt[f] += 1, for the face f seen at the pixel's top-left
// super-sample (y0 * ssaa, x0 * ssaa) of rast -- update_triangles_errors (renderer.py:893-903,923-943): the nearest-neighbour minification
// of trig_id picks that sample, and a pixel whose sample is background charges nothing.  The face id comes from rast, not from inv, so a
// pixel whose point fell beyond the max_points cap still charges its face.
__device__ __forceinline__ void s1_face_error(const float* __restrict__ rast, uint32_t y0, uint32_t x0, uint32_t w, uint32_t ssaa, float loss_q,
                                              float* __restrict__ face_err, float* __restrict__ face_cnt, uint32_t F) {
    const float id = rast[4 * ((size_t)(y0 * ssaa) * w + x0 * ssaa) + 3];
    if (id > 0.f) {
        const uint32_t f = (uint32_t)id - 1u;
        if (f < F) { atomicAdd(face_err + f, loss_q); atomicAdd(face_cnt + f, 1.f); }
    }
}

// one thread per low-resolution pixel
template <bool ERR>
__global__ void __launch_bounds__(256)
k_s1_loss(const float4* __restrict__ out, const int32_t* __restrict__ inv, const float* __restrict__ gt, uint32_t gt_channels,
          const float* __restrict__ bg, uint32_t h0, uint32_t w0, uint32_t ssaa, float lambda_mask, const float* __restrict__ loss_scale,
          float4* __restrict__ dout, float* __restrict__ image, float* __restrict__ weights_sum, float* __restrict__ loss_out,
          const float* __restrict__ rast, float* __restrict__ face_err, float* __restrict__ face_cnt, uint32_t F) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t Q = h0 * w0;
    float my_loss = 0.f;
    if (q < Q) {
        const uint32_t y0 = q / w0, x0 = q % w0, w = w0 * ssaa;
        const float inv_s2 = 1.0f / (float)(ssaa * ssaa);
        float r = 0.f, g = 0.f, b = 0.f, a = 0.f;
        for (uint32_t dy = 0; dy < ssaa; ++dy)
            for (uint32_t dx = 0; dx < ssaa; ++dx) {
                const int32_t k = inv[(size_t)(y0 * ssaa + dy) * w + x0 * ssaa + dx];
                if (k >= 0) {
                    const float4 o = out[k];
                    // alphas * rgbs with both clamped to [0, 1] (renderer.py:886-889; the colour is already in [0, 1])
                    r += fminf(fmaxf(o.y, 0.f), 1.f); g += fminf(fmaxf(o.z, 0.f), 1.f); b += fminf(fmaxf(o.w, 0.f), 1.f); a += 1.f;
                }
            }
        r *= inv_s2; g *= inv_s2; b *= inv_s2; a *= inv_s2;
        const float T = 1.f - a;
        const float b0 = bg[3 * q], b1 = bg[3 * q + 1], b2 = bg[3 * q + 2];
        const float pr = r + T * b0, pg = g + T * b1, pb = b + T * b2;
        float t0, t1, t2, m = 0.f;
        if (gt_channels == 4) {          // utils.py:662-667
            m = gt[4 * q + 3];
            t0 = gt[4 * q] * m + b0 * (1 - m); t1 = gt[4 * q + 1] * m + b1 * (1 - m); t2 = gt[4 * q + 2] * m + b2 * (1 - m);
        } else {
            t0 = gt[3 * q]; t1 = gt[3 * q + 1]; t2 = gt[3 * q + 2];
        }
        const float e0 = pr - t0, e1 = pg - t1, e2 = pb - t2;
        my_loss = (e0 * e0 + e1 * e1 + e2 * e2) * (1.0f / 3.0f);
        if (gt_channels == 4 && lambda_mask > 0) { const float em = a - m; my_loss += lambda_mask * em * em; }
        image[3 * q] = pr; image[3 * q + 1] = pg; image[3 * q + 2] = pb;
        weights_sum[q] = a;
        const float sc = loss_scale[0] / (float)Q * (2.0f / 3.0f) * inv_s2;
        const float4 d = make_float4(0.f, sc * e0, sc * e1, sc * e2);
        for (uint32_t dy = 0; dy < ssaa; ++dy)
            for (uint32_t dx = 0; dx < ssaa; ++dx) {
                const int32_t k = inv[(size_t)(y0 * ssaa + dy) * w + x0 * ssaa + dx];
                if (k >= 0) dout[k] = d;
            }
        if constexpr (ERR) s1_face_error(rast, y0, x0, w, ssaa, my_loss, face_err, face_cnt, F);
        my_loss /= (float)Q;
    }
    // block reduction -> one atomic per block
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) my_loss += __shfl_xor_sync(0xffffffffu, my_loss, o);
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = my_loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < 8; ++i) s += red[i];
        atomicAdd(loss_out, s);
    }
}

// ---- antialiased variant ----
__global__ void __launch_bounds__(256)
k_s1_rgba(const float4* __restrict__ out, const int32_t* __restrict__ inv, uint32_t n, float4* __restrict__ rgba) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t k = inv[i];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k >= 0) { const float4 o = out[k]; v = make_float4(o.y, o.z, o.w, 1.f); }
    rgba[i] = v;
}

__global__ void __launch_bounds__(256)
k_s1_dout(const float4* __restrict__ grad_rgba, const int32_t* __restrict__ inv, uint32_t n, float4* __restrict__ dout) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t k = inv[i];
    if (k >= 0) { const float4 g = grad_rgba[i]; dout[k] = make_float4(0.f, g.x, g.y, g.z); }
}

// one thread per low-resolution pixel; aa [h*w] float4 = antialiased (r, g, b, alpha); d_aa = d loss / d aa * loss_scale; ERR as in k_s1_loss
template <bool ERR>
__global__ void __launch_bounds__(256)
k_s1_loss_aa(const float4* __restrict__ aa, const float* __restrict__ gt, uint32_t gt_channels, const float* __restrict__ bg, uint32_t h0,
             uint32_t w0, uint32_t ssaa, float lambda_mask, const float* __restrict__ loss_scale, float4* __restrict__ d_aa,
             float* __restrict__ image, float* __restrict__ weights_sum, float* __restrict__ loss_out,
             const float* __restrict__ rast, float* __restrict__ face_err, float* __restrict__ face_cnt, uint32_t F) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t Q = h0 * w0;
    float my_loss = 0.f;
    if (q < Q) {
        const uint32_t y0 = q / w0, x0 = q % w0, w = w0 * ssaa;
        const float inv_s2 = 1.0f / (float)(ssaa * ssaa);
        float r = 0.f, g = 0.f, b = 0.f, a = 0.f;
        for (uint32_t dy = 0; dy < ssaa; ++dy)
            for (uint32_t dx = 0; dx < ssaa; ++dx) {
                const float4 v = aa[(size_t)(y0 * ssaa + dy) * w + x0 * ssaa + dx];
                const float al = clampf(v.w, 0.f, 1.f);                                 // .clamp(0, 1) of both (renderer.py:886-887)
                r += al * clampf(v.x, 0.f, 1.f); g += al * clampf(v.y, 0.f, 1.f); b += al * clampf(v.z, 0.f, 1.f); a += al;
            }
        r *= inv_s2; g *= inv_s2; b *= inv_s2; a *= inv_s2;
        const float T = 1.f - a;
        const float b0 = bg[3 * q], b1 = bg[3 * q + 1], b2 = bg[3 * q + 2];
        const float pr = r + T * b0, pg = g + T * b1, pb = b + T * b2;
        float t0, t1, t2, m = 0.f;
        if (gt_channels == 4) {
            m = gt[4 * q + 3];
            t0 = gt[4 * q] * m + b0 * (1 - m); t1 = gt[4 * q + 1] * m + b1 * (1 - m); t2 = gt[4 * q + 2] * m + b2 * (1 - m);
        } else {
            t0 = gt[3 * q]; t1 = gt[3 * q + 1]; t2 = gt[3 * q + 2];
        }
        const float e0 = pr - t0, e1 = pg - t1, e2 = pb - t2;
        my_loss = (e0 * e0 + e1 * e1 + e2 * e2) * (1.0f / 3.0f);
        float dmask = 0.f;
        if (gt_channels == 4 && lambda_mask > 0) {
            const float em = a - m;
            my_loss += lambda_mask * em * em;
            dmask = loss_scale[0] / (float)Q * 2.0f * lambda_mask * em * inv_s2;
        }
        image[3 * q] = pr; image[3 * q + 1] = pg; image[3 * q + 2] = pb;
        weights_sum[q] = a;
        const float sc = loss_scale[0] / (float)Q * (2.0f / 3.0f) * inv_s2;
        for (uint32_t dy = 0; dy < ssaa; ++dy)
            for (uint32_t dx = 0; dx < ssaa; ++dx) {
                const size_t i = (size_t)(y0 * ssaa + dy) * w + x0 * ssaa + dx;
                const float4 v = aa[i];
                const float al = clampf(v.w, 0.f, 1.f);
                const float cr = clampf(v.x, 0.f, 1.f), cg = clampf(v.y, 0.f, 1.f), cb = clampf(v.z, 0.f, 1.f);
                float4 d;
                // clamp passes the gradient inside [0, 1] (bounds included, as torch.clamp does)
                d.x = (v.x >= 0.f && v.x <= 1.f) ? sc * e0 * al : 0.f;
                d.y = (v.y >= 0.f && v.y <= 1.f) ? sc * e1 * al : 0.f;
                d.z = (v.z >= 0.f && v.z <= 1.f) ? sc * e2 * al : 0.f;
                d.w = (v.w >= 0.f && v.w <= 1.f) ? sc * (e0 * (cr - b0) + e1 * (cg - b1) + e2 * (cb - b2)) + dmask : 0.f;
                d_aa[i] = d;
            }
        if constexpr (ERR) s1_face_error(rast, y0, x0, w, ssaa, my_loss, face_err, face_cnt, F);
        my_loss /= (float)Q;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) my_loss += __shfl_xor_sync(0xffffffffu, my_loss, o);
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = my_loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < 8; ++i) s += red[i];
        atomicAdd(loss_out, s);
    }
}

// ---- evaluation (render_stage1 at inference, renderer.py:886-907): the image part of k_s1_loss_aa, plus depth ----
// One thread per low-resolution pixel over img [h*w] float4 = (r, g, b, alpha), antialiased or the n2m_s1_rgba image (alpha exactly 0 or
// 1).  The float operations are those of k_s1_loss_aa in the same order, so image / weights_sum equal its outputs bit for bit; on the
// n2m_s1_rgba image they also equal k_s1_loss's (al = 1: al * c == c; al = 0 adds +0 to a non-negative sum).  depth = mean over the
// super-samples of alpha * rast.z (z/w; :889,:900).
__global__ void __launch_bounds__(256)
k_s1_render_compose(const float4* __restrict__ img, const float4* __restrict__ rast, const float* __restrict__ bg, uint32_t h0, uint32_t w0,
                    uint32_t ssaa, float* __restrict__ image, float* __restrict__ weights_sum, float* __restrict__ depth) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= h0 * w0) return;
    const uint32_t y0 = q / w0, x0 = q % w0, w = w0 * ssaa;
    const float inv_s2 = 1.0f / (float)(ssaa * ssaa);
    float r = 0.f, g = 0.f, b = 0.f, a = 0.f, d = 0.f;
    for (uint32_t dy = 0; dy < ssaa; ++dy)
        for (uint32_t dx = 0; dx < ssaa; ++dx) {
            const size_t i = (size_t)(y0 * ssaa + dy) * w + x0 * ssaa + dx;
            const float4 v = img[i];
            const float al = clampf(v.w, 0.f, 1.f);
            r += al * clampf(v.x, 0.f, 1.f); g += al * clampf(v.y, 0.f, 1.f); b += al * clampf(v.z, 0.f, 1.f); a += al;
            d += al * rast[i].z;
        }
    r *= inv_s2; g *= inv_s2; b *= inv_s2; a *= inv_s2; d *= inv_s2;
    const float T = 1.f - a;
    const float b0 = bg[3 * q], b1 = bg[3 * q + 1], b2 = bg[3 * q + 2];
    const float pr = r + T * b0, pg = g + T * b1, pb = b + T * b2;
    image[3 * q] = pr; image[3 * q + 1] = pg; image[3 * q + 2] = pb;
    weights_sum[q] = a;
    depth[q] = d;
}

// ---- colour-field path of the vertex gradient (--enable_offset_nerf_grad: renderer.py:877-879 with xyzs[mask_flatten] not detached) ----
// One thread per super-sampled pixel with a point (inv[i] >= 0).  The loss-scaled gradient w.r.t. the point the colour field saw is
//   the direct term: tile columns kColXyz..+2 of its denc row (x is an input of color_net.0; dS1 is zero in stage 1), plus
//   the hash-grid term: per level, d(colour feature)/du of the trilinear interpolation (the reference's dy_dx, gridencoder.cu:198-240:
//   per dimension the weights of the other two dimensions times (right - left corner) times the level scale) dotted with the feature's
//   denc columns, times inv_2gb for u = (x + bound) / (2 bound); zero outside [0,1]^3, where the encoder outputs zeros;
// CONTRACT: then through the Jacobian of contract() at the uncontracted point (recomputed from rast and the vertices as k_s1_points
// does).  The scatter is dr.interpolate's backward: b_k dx into grad_vworld [V,3], and (du, dv) through dr.rasterize's backward into
// grad_vclip [V,4] beside the antialias gradient (raster_grad.cuh).  A non-finite gradient (fp16 overflow of the x columns) sets found_inf
// (st[3]) and is not scattered.
template <bool CONTRACT>
__global__ void __launch_bounds__(256)
k_s1_offset_grad(const n2m_s0_params p, const float4* __restrict__ rast, const float* __restrict__ verts, const float4* __restrict__ vclip,
                 const int32_t* __restrict__ tri, const int32_t* __restrict__ inv, uint32_t h, uint32_t w, const float* __restrict__ pts,
                 const uint8_t* __restrict__ denc_tiles, const TableEntry* __restrict__ table, const int32_t* __restrict__ offsets,
                 float* __restrict__ grad_vclip, float* __restrict__ grad_vworld, float* __restrict__ st) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= h * w) return;
    const int32_t k = inv[i];
    if (k < 0) return;
    const uint8_t* img = denc_tiles + (size_t)(k / kTile) * kTileBytes + (k % kTile) * 16;
    float g[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) g[a] = denc_col(img, kColXyz + a);
    const float x = pts[3 * (size_t)k], y = pts[3 * (size_t)k + 1], z = pts[3 * (size_t)k + 2];
    const float u = __fmul_rn(__fadd_rn(x, p.grid_bound), p.inv_2gb);       // encode_fwd_features (POINTS)
    const float v = __fmul_rn(__fadd_rn(y, p.grid_bound), p.inv_2gb);
    const float ww = __fmul_rn(__fadd_rn(z, p.grid_bound), p.inv_2gb);
    if (!((u < 0 || u > 1) || (v < 0 || v > 1) || (ww < 0 || ww > 1))) {
        float gu[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
        for (uint32_t l = 0; l < kLevels; ++l) {
            const float g0 = denc_col(img, kColColor + 2 * l), g1 = denc_col(img, kColColor + 2 * l + 1);
            const LevelGeom lg = level_geom(offsets, l, p.S, p.base_res);
            Corners c; uint32_t base[3]; bool hashed;
            corners_of(lg, u, v, ww, c, base, hashed, nullptr);
            const float fr[3] = {(u * lg.scale + 0.5f) - (float)base[0], (v * lg.scale + 0.5f) - (float)base[1], (ww * lg.scale + 0.5f) - (float)base[2]};
            const TableEntry* tab = table + lg.row0;
            float f[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const uint2 raw = __ldg(reinterpret_cast<const uint2*>(tab + c.row[q]));
                const float2 cc = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
                f[q] = g0 * cc.x + g1 * cc.y;                  // the feature gradient dotted with the corner's two features
            }
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int d1 = (d + 1) % 3, d2 = (d + 2) % 3;
                float s = 0.f;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float w1 = ((q >> d1) & 1) ? fr[d1] : 1.f - fr[d1], w2 = ((q >> d2) & 1) ? fr[d2] : 1.f - fr[d2];
                    s += ((q >> d) & 1) ? w1 * w2 * f[q] : -(w1 * w2 * f[q]);
                }
                gu[d] += lg.scale * s;
            }
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) g[a] += gu[a] * p.inv_2gb;
    }
    const float4 r = rast[i];
    const uint32_t f = (uint32_t)r.w - 1u;
    const int vi[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
    float vx[3][3];
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int a = 0; a < 3; ++a) vx[q][a] = __ldg(verts + 3 * (size_t)vi[q] + a);
    if constexpr (CONTRACT) {
        float xu[3];
        const float bw = 1.f - r.x - r.y;
#pragma unroll
        for (int a = 0; a < 3; ++a) xu[a] = r.x * vx[0][a] + r.y * vx[1][a] + bw * vx[2][a];
        contract_linf_backward(xu, g);
    }
    if (!(isfinite(g[0]) && isfinite(g[1]) && isfinite(g[2]))) { st[3] = 1.f; return; }
    const float b[3] = {r.x, r.y, 1.f - r.x - r.y};
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int a = 0; a < 3; ++a) atomicAdd(grad_vworld + 3 * (size_t)vi[q] + a, b[q] * g[a]);
    const float2 duv = interpolate_uv_backward<3>(g, vx[0], vx[1], vx[2]);
    const float4 pc[3] = {__ldg(vclip + vi[0]), __ldg(vclip + vi[1]), __ldg(vclip + vi[2])};
    const float2 ndc = pixel_ndc(i % w, i / w, h, w);
    rasterize_uv_backward(pc, vi, ndc.x, ndc.y, duv.x, duv.y, grad_vclip);
}

// ---- vertex-offset optimizer (NeRFRenderer.vertices_offsets: renderer.py:160,180 -- Adam group with lr_vert; regularisers
// utils.py:750-779: lambda_lap * laplacian_smooth_loss (uniform Laplacian, utils.py:176-221) + lambda_offsets * mean(sum(offsets^2))) ----
// y += L x for the uniform Laplacian L = D - A, one thread per slot of the edge hash of csrc/antialias.cu (one slot = one undirected edge)
__global__ void __launch_bounds__(256)
k_s1_laplacian(const unsigned long long* __restrict__ keys, uint32_t slots, const float* __restrict__ x, float* __restrict__ y) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    const unsigned long long k = keys[i];
    if (k == ~0ull) return;
    const uint32_t a = (uint32_t)(k >> 32), b = (uint32_t)(k & 0xffffffffull);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float d = x[3 * (size_t)a + c] - x[3 * (size_t)b + c];
        atomicAdd(y + 3 * (size_t)a + c, d);
        atomicAdd(y + 3 * (size_t)b + c, -d);
    }
}

// u [V,3] = L v  ->  u_i / |u_i| in place (0 where |u_i| = 0: the subgradient torch.norm uses), loss_out[0] += lambda_lap * mean |u_i|
__global__ void __launch_bounds__(256)
k_s1_lap_normalize(float* __restrict__ u, uint32_t V, float lambda_lap, float* __restrict__ loss_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float n = 0.f;
    if (i < V) {
        const float a = u[3 * (size_t)i], b = u[3 * (size_t)i + 1], c = u[3 * (size_t)i + 2];
        n = sqrtf(a * a + b * b + c * c);
        const float r = n > 0.f ? __fdiv_rn(1.f, n) : 0.f;
        u[3 * (size_t)i] = a * r; u[3 * (size_t)i + 1] = b * r; u[3 * (size_t)i + 2] = c * r;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (loss_out && (threadIdx.x & 31) == 0 && n != 0.f) atomicAdd(loss_out, lambda_lap * n / (float)V);
}

// non-finite scan of the loss-scaled clip-space gradient -> found_inf (GradScaler.unscale_ over the vertices_offsets group)
__global__ void __launch_bounds__(256)
k_s1_vert_check(const float* __restrict__ g, uint32_t n, float* __restrict__ st) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool bad = i < n && !isfinite(g[i]);
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) st[3] = 1.f;
}

// grad = (grad_vclip . mvp[:, :3]) / loss_scale + (lambda_lap / V) * (L w) + (2 lambda_offsets / V) * offsets; Adam(eps) on the offsets with
// its own step count vst[0]; vertices = base + offsets.  Skipped as a whole when found_inf is set (st[3]).  WORLD: the image-loss part is
// (grad_vclip . mvp[:, :3] + grad_vworld) / loss_scale (the colour-field path, k_s1_offset_grad); grad_vworld is the last parameter, so
// the WORLD = false instantiation keeps the parameter offsets, and the code, of the kernel without it.  REG (the overload below):
// reg_grad [V,3] (the mesh regularisers' gradient, k_s1_mesh_reg, already weighted) is added to the gradient and grad_vworld is nullable.
template <bool WORLD, bool REG>
__device__ __forceinline__ void vert_adam(const float4* __restrict__ grad_vclip, const float* __restrict__ mvp, const float* __restrict__ lap_grad,
                                          const float* __restrict__ base, float* __restrict__ offsets, float* __restrict__ m, float* __restrict__ v,
                                          float* __restrict__ vertices, float* __restrict__ grad_out, uint32_t V, float lambda_lap,
                                          float lambda_offsets, float lr, float eps, const float* __restrict__ st, const float* __restrict__ vst,
                                          const float* __restrict__ grad_vworld, const float* __restrict__ reg_grad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    if (lr < 0.f) lr = vst[1];                                          // learning rate kept on the device (graph-replayed steps)
    const bool skip = st[3] != 0.f;
    const float inv_scale = st[7];
    const float t = vst[0] + (skip ? 0.f : 1.f);                       // this step's count (k_s1_vert_tick advances it afterwards)
    const float bc1 = 1.f - powf(0.9f, fmaxf(t, 1.f)), bc2s = sqrtf(1.f - powf(0.999f, fmaxf(t, 1.f)));
    const float4 gc = grad_vclip[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const size_t j = 3 * (size_t)i + c;
        float gi;
        if constexpr (WORLD) gi = (gc.x * mvp[c] + gc.y * mvp[4 + c] + gc.z * mvp[8 + c] + gc.w * mvp[12 + c] + grad_vworld[j]) * inv_scale;
        else if constexpr (REG) gi = (gc.x * mvp[c] + gc.y * mvp[4 + c] + gc.z * mvp[8 + c] + gc.w * mvp[12 + c] + (grad_vworld ? grad_vworld[j] : 0.f)) * inv_scale;
        else gi = (gc.x * mvp[c] + gc.y * mvp[4 + c] + gc.z * mvp[8 + c] + gc.w * mvp[12 + c]) * inv_scale;
        const float off = offsets[j];
        float g = gi + (lambda_lap > 0.f ? lambda_lap / (float)V * lap_grad[j] : 0.f) + 2.f * lambda_offsets / (float)V * off;
        if constexpr (REG) g += reg_grad[j];
        if (grad_out) grad_out[j] = g;
        if (skip) continue;
        const float mi = 0.9f * m[j] + 0.1f * g;
        const float vi = 0.999f * v[j] + 0.001f * g * g;
        m[j] = mi; v[j] = vi;
        const float denom = __fdiv_rn(__fsqrt_rn(vi), bc2s) + eps;
        const float o2 = off - __fdiv_rn(lr, bc1) * __fdiv_rn(mi, denom);
        offsets[j] = o2;
        vertices[j] = base[j] + o2;
    }
}

template <bool WORLD>
__global__ void __launch_bounds__(256)
k_s1_vert_adam(const float4* __restrict__ grad_vclip, const float* __restrict__ mvp, const float* __restrict__ lap_grad, const float* __restrict__ base,
               float* __restrict__ offsets, float* __restrict__ m, float* __restrict__ v, float* __restrict__ vertices, float* __restrict__ grad_out,
               uint32_t V, float lambda_lap, float lambda_offsets, float lr, float eps, const float* __restrict__ st, const float* __restrict__ vst,
               const float* __restrict__ grad_vworld) {
    vert_adam<WORLD, false>(grad_vclip, mvp, lap_grad, base, offsets, m, v, vertices, grad_out, V, lambda_lap, lambda_offsets, lr, eps, st, vst,
                            grad_vworld, nullptr);
}

// the mesh-regulariser step: one overload serves it with and without the colour-field path (grad_vworld nullable)
__global__ void __launch_bounds__(256)
k_s1_vert_adam(const float4* __restrict__ grad_vclip, const float* __restrict__ mvp, const float* __restrict__ lap_grad, const float* __restrict__ base,
               float* __restrict__ offsets, float* __restrict__ m, float* __restrict__ v, float* __restrict__ vertices, float* __restrict__ grad_out,
               uint32_t V, float lambda_lap, float lambda_offsets, float lr, float eps, const float* __restrict__ st, const float* __restrict__ vst,
               const float* __restrict__ grad_vworld, const float* __restrict__ reg_grad) {
    vert_adam<false, true>(grad_vclip, mvp, lap_grad, base, offsets, m, v, vertices, grad_out, V, lambda_lap, lambda_offsets, lr, eps, st, vst,
                           grad_vworld, reg_grad);
}

// ---- mesh regularisers of the vertex offsets (utils.py:759-769: lambda_normal * mesh_normal_consistency + lambda_edgelen * mesh_edge_loss of
// pytorch3d, on vertices = base + offsets before the update), over the slots of the edge hash (csrc/topology_hash.cuh) ----
// once per mesh: faces per slot into cnt[slot] (one thread per face, one probe per edge with two distinct ends), and faces with a repeated
// vertex index into res[3]
__global__ void __launch_bounds__(256)
k_s1_mesh_reg_faces(const int32_t* __restrict__ tri, uint32_t F, const unsigned long long* __restrict__ keys, uint32_t mask,
                    uint32_t* __restrict__ cnt, uint32_t* __restrict__ res) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int v[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
    if (v[0] == v[1] || v[1] == v[2] || v[0] == v[2]) atomicAdd(res + 3, 1u);
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int a = v[e], b = v[(e + 1) % 3];
        if (a == b) continue;
        const int64_t s = topo_find(keys, mask, a, b);
        if (s >= 0) atomicAdd(cnt + s, 1u);
    }
}

// res[0] += occupied slots (E, the unique edges), res[1] += slots with exactly two faces (P, the normal pairs), res[2] += slots with more
__global__ void __launch_bounds__(256)
k_s1_mesh_reg_slots(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ cnt, uint32_t slots, uint32_t* __restrict__ res) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool occ = i < slots && keys[i] != kEmptyKey;
    const uint32_t c = occ ? cnt[i] : 0u;
    const uint32_t ne = __popc(__ballot_sync(0xffffffffu, occ)), np = __popc(__ballot_sync(0xffffffffu, c == 2u)),
                   nm = __popc(__ballot_sync(0xffffffffu, c > 2u));
    if ((threadIdx.x & 31) == 0) {
        if (ne) atomicAdd(res, ne);
        if (np) atomicAdd(res + 1, np);
        if (nm) atomicAdd(res + 2, nm);
    }
}

constexpr float kCosEps = 1e-8f;          // torch.cosine_similarity's default eps (mesh_normal_consistency uses the default)

__device__ __forceinline__ void cross3(const float a[3], const float b[3], float r[3]) {
    r[0] = a[1] * b[2] - a[2] * b[1]; r[1] = a[2] * b[0] - a[0] * b[2]; r[2] = a[0] * b[1] - a[1] * b[0];
}

// One thread per slot; the slot holds edge (a, b), a < b, and the opposite vertices c, d of up to two faces.
//   edge:   we * |v_a - v_b|^2,  we = lambda_edgelen / E
//   normal (two faces): wn * (1 - cos(n_c, -n_d)),  wn = lambda_normal / P,  n_c = (v_b - v_a) x (v_c - v_a), n_d likewise; torch's
//           cosine_similarity divides each vector by max(|n|, eps) and differentiates the branch taken, so a zero-area face gives 1 - 0 and
//           the gradient n_other / eps.  With both norms >= eps, 1 - cos = |u + w|^2 / 2 for the unit vectors u = n_c / |n_c|,
//           w = n_d / |n_d|, and d/dn_c = (u + w - loss u) / |n_c|: no cancellation between nearly opposite unit vectors on a smooth mesh.
// The gradient w.r.t. the vertices is ACCUMULATED into grad [V,3] (6 atomics per edge, 12 per edge with a pair); loss_out[0] += the sum.
__global__ void __launch_bounds__(256)
k_s1_mesh_reg(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ opp, uint32_t slots, const float* __restrict__ x,
              float wn, float we, float* __restrict__ grad, float* __restrict__ loss_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float loss = 0.f;
    const unsigned long long k = i < slots ? keys[i] : kEmptyKey;
    if (k != kEmptyKey) {
        const uint32_t a = (uint32_t)(k >> 32), b = (uint32_t)(k & 0xffffffffull);
        float pa[3], e[3], ga[3], gb[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            pa[c] = x[3 * (size_t)a + c];
            e[c] = x[3 * (size_t)b + c] - pa[c];
            ga[c] = 0.f; gb[c] = 0.f;
        }
        if (we > 0.f) {
            loss += we * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
#pragma unroll
            for (int c = 0; c < 3; ++c) { ga[c] = -2.f * we * e[c]; gb[c] = 2.f * we * e[c]; }
        }
        const int oc = opp[2 * (size_t)i], od = opp[2 * (size_t)i + 1];
        if (wn > 0.f && od >= 0) {
            float qc[3], qd[3], nc[3], nd[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) { qc[c] = x[3 * (size_t)oc + c] - pa[c]; qd[c] = x[3 * (size_t)od + c] - pa[c]; }
            cross3(e, qc, nc);
            cross3(e, qd, nd);
            const float lc = __fsqrt_rn(nc[0] * nc[0] + nc[1] * nc[1] + nc[2] * nc[2]);
            const float ld = __fsqrt_rn(nd[0] * nd[0] + nd[1] * nd[1] + nd[2] * nd[2]);
            const float rc = __frcp_rn(fmaxf(lc, kCosEps)), rd = __frcp_rn(fmaxf(ld, kCosEps));
            float u[3], w[3], gc[3], gd[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) { u[c] = nc[c] * rc; w[c] = nd[c] * rd; }
            float L;
            if (lc >= kCosEps && ld >= kCosEps) {
                float s[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) s[c] = u[c] + w[c];
                L = 0.5f * (s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
#pragma unroll
                for (int c = 0; c < 3; ++c) { gc[c] = (s[c] - L * u[c]) * rc; gd[c] = (s[c] - L * w[c]) * rd; }
            } else {
                const float dp = u[0] * w[0] + u[1] * w[1] + u[2] * w[2];
                L = 1.f + dp;
                const float pc = lc >= kCosEps ? dp : 0.f, pd = ld >= kCosEps ? dp : 0.f;        // the clamped branch has no projection
#pragma unroll
                for (int c = 0; c < 3; ++c) { gc[c] = (w[c] - pc * u[c]) * rc; gd[c] = (u[c] - pd * w[c]) * rd; }
            }
            loss += wn * L;
#pragma unroll
            for (int c = 0; c < 3; ++c) { gc[c] *= wn; gd[c] *= wn; }
            // n = e x q: d/de = q x g, d/dq = g x e; e = v_b - v_a, q = v_o - v_a
            float t1[3], t2[3], gqc[3], gqd[3];
            cross3(qc, gc, t1);
            cross3(qd, gd, t2);
            cross3(gc, e, gqc);
            cross3(gd, e, gqd);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float ge = t1[c] + t2[c];
                gb[c] += ge;
                ga[c] -= ge + gqc[c] + gqd[c];
                atomicAdd(grad + 3 * (size_t)oc + c, gqc[c]);
                atomicAdd(grad + 3 * (size_t)od + c, gqd[c]);
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            atomicAdd(grad + 3 * (size_t)a + c, ga[c]);
            atomicAdd(grad + 3 * (size_t)b + c, gb[c]);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (loss_out && (threadIdx.x & 31) == 0 && loss != 0.f) atomicAdd(loss_out, loss);
}

__global__ void k_s1_vert_tick(const float* __restrict__ st, float* __restrict__ vst) {
    if (threadIdx.x == 0 && blockIdx.x == 0 && st[3] == 0.f) vst[0] += 1.f;
}

// the two entry points of each loss kernel: ERR = false (refinement off) and ERR = true (+ the per-face error scatter)
template <bool ERR>
int launch_s1_loss(const void* out, const int32_t* inv, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0,
                   uint32_t ssaa, float lambda_mask, const float* loss_scale, void* dout, float* image, float* weights_sum, float* loss_out,
                   const float* rast, float* face_err, float* face_cnt, uint32_t F, n2m_stream_t stream, const char* what) {
    N2M_REQUIRE(out && inv && gt && bg && loss_scale && dout && image && weights_sum && loss_out, what, "null pointer");
    N2M_REQUIRE(gt_channels == 3 || gt_channels == 4, what, "gt must have 3 or 4 channels");
    N2M_REQUIRE(!ERR || (rast && face_err && face_cnt), what, "null pointer");
    k_s1_loss<ERR><<<div_up(h0 * w0, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(out), inv, gt, gt_channels, bg, h0, w0, ssaa,
                                                                        lambda_mask, loss_scale, static_cast<float4*>(dout), image, weights_sum,
                                                                        loss_out, rast, face_err, face_cnt, F);
    return check_launch(what);
}

template <bool ERR>
int launch_s1_loss_aa(const void* aa, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa,
                      float lambda_mask, const float* loss_scale, void* d_aa, float* image, float* weights_sum, float* loss_out,
                      const float* rast, float* face_err, float* face_cnt, uint32_t F, n2m_stream_t stream, const char* what) {
    N2M_REQUIRE(aa && gt && bg && loss_scale && d_aa && image && weights_sum && loss_out, what, "null pointer");
    N2M_REQUIRE(gt_channels == 3 || gt_channels == 4, what, "gt must have 3 or 4 channels");
    N2M_REQUIRE(ssaa >= 1, what, "ssaa must be >= 1");
    N2M_REQUIRE(!ERR || (rast && face_err && face_cnt), what, "null pointer");
    k_s1_loss_aa<ERR><<<div_up(h0 * w0, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(aa), gt, gt_channels, bg, h0, w0, ssaa,
                                                                           lambda_mask, loss_scale, static_cast<float4*>(d_aa), image,
                                                                           weights_sum, loss_out, rast, face_err, face_cnt, F);
    return check_launch(what);
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_s1_points_contract(const float* rast, const float* verts, const int32_t* tri, const float* rays_d, uint32_t h, uint32_t w,
                           uint32_t ssaa, uint32_t cap, int32_t* counters, int32_t* inv, float* pts, float* pdirs, void* recs,
                           uint32_t contract, n2m_stream_t stream) {
    N2M_REQUIRE(rast && verts && tri && rays_d && counters && inv && pts && pdirs && recs, "s1_points", "null pointer");
    N2M_REQUIRE(ssaa >= 1 && h % ssaa == 0 && w % ssaa == 0 && h > 0 && w > 0, "s1_points", "resolution must be a multiple of ssaa");
    cudaStream_t st = as_stream(stream);
    cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), st);
    auto kernel = contract ? k_s1_points<true> : k_s1_points<false>;
    kernel<<<div_up(h * w, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(rast), verts, tri, rays_d, h, w, ssaa, cap, counters, inv,
                                               pts, pdirs, static_cast<float4*>(recs));
    if (int e = check_launch("s1_points")) return e;
    k_s1_finish_count<<<1, 32, 0, st>>>(counters, cap);
    return check_launch("s1_points(count)");
}

int n2m_s1_points(const float* rast, const float* verts, const int32_t* tri, const float* rays_d, uint32_t h, uint32_t w, uint32_t ssaa,
                  uint32_t cap, int32_t* counters, int32_t* inv, float* pts, float* pdirs, void* recs, n2m_stream_t stream) {
    return n2m_s1_points_contract(rast, verts, tri, rays_d, h, w, ssaa, cap, counters, inv, pts, pdirs, recs, 0, stream);
}

int n2m_s1_loss(const void* out, const int32_t* inv, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0,
                uint32_t ssaa, float lambda_mask, const float* loss_scale, void* dout, float* image, float* weights_sum, float* loss_out,
                n2m_stream_t stream) {
    return launch_s1_loss<false>(out, inv, gt, gt_channels, bg, h0, w0, ssaa, lambda_mask, loss_scale, dout, image, weights_sum, loss_out,
                                 nullptr, nullptr, nullptr, 0, stream, "s1_loss");
}

int n2m_s1_loss_err(const void* out, const int32_t* inv, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0,
                    uint32_t ssaa, float lambda_mask, const float* loss_scale, void* dout, float* image, float* weights_sum, float* loss_out,
                    const float* rast, float* face_err, float* face_cnt, uint32_t F, n2m_stream_t stream) {
    return launch_s1_loss<true>(out, inv, gt, gt_channels, bg, h0, w0, ssaa, lambda_mask, loss_scale, dout, image, weights_sum, loss_out,
                                rast, face_err, face_cnt, F, stream, "s1_loss_err");
}

int n2m_s1_rgba(const void* out, const int32_t* inv, uint32_t num_pixels, void* rgba, n2m_stream_t stream) {
    N2M_REQUIRE(out && inv && rgba, "s1_rgba", "null pointer");
    if (num_pixels == 0) return 0;
    k_s1_rgba<<<div_up(num_pixels, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(out), inv, num_pixels, static_cast<float4*>(rgba));
    return check_launch("s1_rgba");
}

int n2m_s1_dout(const void* grad_rgba, const int32_t* inv, uint32_t num_pixels, void* dout, n2m_stream_t stream) {
    N2M_REQUIRE(grad_rgba && inv && dout, "s1_dout", "null pointer");
    if (num_pixels == 0) return 0;
    k_s1_dout<<<div_up(num_pixels, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(grad_rgba), inv, num_pixels, static_cast<float4*>(dout));
    return check_launch("s1_dout");
}

int n2m_s1_loss_aa(const void* aa, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa,
                   float lambda_mask, const float* loss_scale, void* d_aa, float* image, float* weights_sum, float* loss_out,
                   n2m_stream_t stream) {
    return launch_s1_loss_aa<false>(aa, gt, gt_channels, bg, h0, w0, ssaa, lambda_mask, loss_scale, d_aa, image, weights_sum, loss_out,
                                    nullptr, nullptr, nullptr, 0, stream, "s1_loss_aa");
}

int n2m_s1_loss_aa_err(const void* aa, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa,
                       float lambda_mask, const float* loss_scale, void* d_aa, float* image, float* weights_sum, float* loss_out,
                       const float* rast, float* face_err, float* face_cnt, uint32_t F, n2m_stream_t stream) {
    return launch_s1_loss_aa<true>(aa, gt, gt_channels, bg, h0, w0, ssaa, lambda_mask, loss_scale, d_aa, image, weights_sum, loss_out,
                                   rast, face_err, face_cnt, F, stream, "s1_loss_aa_err");
}

int n2m_s1_render_compose(const void* img, const float* rast, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa, float* image,
                          float* weights_sum, float* depth, n2m_stream_t stream) {
    N2M_REQUIRE(img && rast && bg && image && weights_sum && depth, "s1_render_compose", "null pointer");
    N2M_REQUIRE(ssaa >= 1, "s1_render_compose", "ssaa must be >= 1");
    if (h0 == 0 || w0 == 0) return 0;
    k_s1_render_compose<<<div_up(h0 * w0, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(img), reinterpret_cast<const float4*>(rast),
                                                                             bg, h0, w0, ssaa, image, weights_sum, depth);
    return check_launch("s1_render_compose");
}

int n2m_s1_vert_check(const float* grad_vclip, uint32_t V, float* opt_state, n2m_stream_t stream) {
    N2M_REQUIRE(grad_vclip && opt_state, "s1_vert_check", "null pointer");
    if (V == 0) return 0;
    k_s1_vert_check<<<div_up(4 * V, 256u), 256, 0, as_stream(stream)>>>(grad_vclip, 4 * V, opt_state);
    return check_launch("s1_vert_check");
}

int n2m_s1_offset_grad(const n2m_s0_params* p, const float* rast, const float* verts, const float* vclip, const int32_t* tri, const int32_t* inv,
                       uint32_t h, uint32_t w, const float* pts, const void* denc_tiles, const void* table, const int32_t* offsets,
                       float* grad_vclip, float* grad_vworld, float* opt_state, n2m_stream_t stream) {
    N2M_REQUIRE(p && rast && verts && vclip && tri && inv && pts && denc_tiles && table && offsets && grad_vclip && grad_vworld && opt_state,
                "s1_offset_grad", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s1_offset_grad", "the colour grid must have 16 levels");
    N2M_REQUIRE((uint64_t)h * w < (1ull << 31), "s1_offset_grad", "bad resolution");
    if (h == 0 || w == 0) return 0;
    auto kernel = p->contract ? k_s1_offset_grad<true> : k_s1_offset_grad<false>;
    kernel<<<div_up(h * w, 256u), 256, 0, as_stream(stream)>>>(*p, reinterpret_cast<const float4*>(rast), verts, reinterpret_cast<const float4*>(vclip),
                                                                tri, inv, h, w, pts, static_cast<const uint8_t*>(denc_tiles),
                                                                static_cast<const TableEntry*>(table), offsets, grad_vclip, grad_vworld, opt_state);
    return check_launch("s1_offset_grad");
}

int n2m_s1_mesh_reg_setup(const int32_t* tri, uint32_t F, const void* topo_keys, uint32_t topo_slots, uint32_t* scratch, uint32_t* counts,
                          n2m_stream_t stream) {
    N2M_REQUIRE(tri && topo_keys && scratch && counts, "s1_mesh_reg_setup", "null pointer");
    N2M_REQUIRE(topo_slots && !(topo_slots & (topo_slots - 1)), "s1_mesh_reg_setup", "slots must be a power of two");
    cudaStream_t st = as_stream(stream);
    const unsigned long long* keys = static_cast<const unsigned long long*>(topo_keys);
    uint32_t* res = scratch + topo_slots;
    cudaError_t e = cudaMemsetAsync(scratch, 0, ((size_t)topo_slots + 4) * sizeof(uint32_t), st);
    if (e != cudaSuccess) return fail("s1_mesh_reg_setup(memset)", cudaGetErrorString(e));
    if (F > 0) {
        k_s1_mesh_reg_faces<<<div_up(F, 256u), 256, 0, st>>>(tri, F, keys, topo_slots - 1, scratch, res);
        if (int err = check_launch("s1_mesh_reg_setup(faces)")) return err;
    }
    k_s1_mesh_reg_slots<<<div_up(topo_slots, 256u), 256, 0, st>>>(keys, scratch, topo_slots, res);
    if (int err = check_launch("s1_mesh_reg_setup(slots)")) return err;
    e = cudaMemcpyAsync(counts, res, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail("s1_mesh_reg_setup(read)", cudaGetErrorString(e));
    return 0;
}

int n2m_s1_mesh_reg(const void* topo_keys, const int32_t* topo_opp, uint32_t topo_slots, uint32_t num_edges, uint32_t num_pairs,
                    const float* vertices, float lambda_normal, float lambda_edgelen, float* grad, float* loss_out, n2m_stream_t stream) {
    N2M_REQUIRE(topo_keys && topo_opp && vertices && grad, "s1_mesh_reg", "null pointer");
    N2M_REQUIRE(lambda_normal >= 0.f && lambda_edgelen >= 0.f, "s1_mesh_reg", "the weights must be >= 0");
    const float wn = num_pairs ? lambda_normal / (float)num_pairs : 0.f, we = num_edges ? lambda_edgelen / (float)num_edges : 0.f;
    if (topo_slots == 0 || (wn == 0.f && we == 0.f)) return 0;
    k_s1_mesh_reg<<<div_up(topo_slots, 256u), 256, 0, as_stream(stream)>>>(static_cast<const unsigned long long*>(topo_keys), topo_opp, topo_slots,
                                                                          vertices, wn, we, grad, loss_out);
    return check_launch("s1_mesh_reg");
}

static int s1_vert_step(const float* grad_vclip, const float* grad_vworld, const float* mvp, const void* topo_keys, const int32_t* topo_opp,
                        uint32_t topo_slots, uint32_t num_edges, uint32_t num_pairs, const float* base, float* offsets, float* m, float* v,
                        float* vertices, float* scratch, float* grad_out, uint32_t V, float lambda_lap, float lambda_offsets, float lambda_normal,
                        float lambda_edgelen, float lr_vert, float eps, const float* opt_state, float* vert_state, float* loss_out,
                        n2m_stream_t stream) {
    N2M_REQUIRE(grad_vclip && mvp && base && offsets && m && v && vertices && scratch && opt_state && vert_state, "s1_vert_step", "null pointer");
    N2M_REQUIRE(lambda_lap <= 0.f || (topo_keys && topo_slots > 0), "s1_vert_step", "the Laplacian term needs the mesh's edge hash");
    const bool reg = lambda_normal > 0.f || lambda_edgelen > 0.f;
    N2M_REQUIRE(!reg || (topo_keys && topo_opp && topo_slots > 0), "s1_vert_step", "the mesh regularisers need the mesh's edge hash");
    if (V == 0) return 0;
    cudaStream_t st = as_stream(stream);
    float* u = scratch;                       // [V,3]: L v, then its row-normalised form
    float* lg = scratch + 3 * (size_t)V;      // [V,3]: L (u / |u|)
    float* rg = scratch + 6 * (size_t)V;      // [V,3]: the mesh regularisers' gradient (reg only)
    if (lambda_lap > 0.f) {
        const unsigned long long* keys = static_cast<const unsigned long long*>(topo_keys);
        cudaError_t e = cudaMemsetAsync(scratch, 0, 6 * (size_t)V * sizeof(float), st);
        if (e != cudaSuccess) return fail("s1_vert_step(memset)", cudaGetErrorString(e));
        k_s1_laplacian<<<div_up(topo_slots, 256u), 256, 0, st>>>(keys, topo_slots, vertices, u);
        if (int err = check_launch("s1_vert_step(L v)")) return err;
        k_s1_lap_normalize<<<div_up(V, 256u), 256, 0, st>>>(u, V, lambda_lap, loss_out);
        if (int err = check_launch("s1_vert_step(normalize)")) return err;
        k_s1_laplacian<<<div_up(topo_slots, 256u), 256, 0, st>>>(keys, topo_slots, u, lg);
        if (int err = check_launch("s1_vert_step(L w)")) return err;
    }
    if (reg) {
        cudaError_t e = cudaMemsetAsync(rg, 0, 3 * (size_t)V * sizeof(float), st);
        if (e != cudaSuccess) return fail("s1_vert_step(memset)", cudaGetErrorString(e));
        if (int err = n2m_s1_mesh_reg(topo_keys, topo_opp, topo_slots, num_edges, num_pairs, vertices, lambda_normal, lambda_edgelen, rg, loss_out,
                                      stream))
            return err;
        k_s1_vert_adam<<<div_up(V, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(grad_vclip), mvp, lg, base, offsets, m, v, vertices, grad_out,
                                                        V, lambda_lap, lambda_offsets, lr_vert, eps, opt_state, vert_state, grad_vworld, rg);
    } else {
        auto adam = grad_vworld ? k_s1_vert_adam<true> : k_s1_vert_adam<false>;
        adam<<<div_up(V, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(grad_vclip), mvp, lg, base, offsets, m, v, vertices, grad_out, V,
                                              lambda_lap, lambda_offsets, lr_vert, eps, opt_state, vert_state, grad_vworld);
    }
    if (int err = check_launch("s1_vert_step(adam)")) return err;
    k_s1_vert_tick<<<1, 32, 0, st>>>(opt_state, vert_state);
    return check_launch("s1_vert_step(tick)");
}

int n2m_s1_vert_step(const float* grad_vclip, const float* mvp, const void* topo_keys, uint32_t topo_slots, const float* base, float* offsets,
                     float* m, float* v, float* vertices, float* scratch, float* grad_out, uint32_t V, float lambda_lap, float lambda_offsets,
                     float lr_vert, float eps, const float* opt_state, float* vert_state, float* loss_out, n2m_stream_t stream) {
    return s1_vert_step(grad_vclip, nullptr, mvp, topo_keys, nullptr, topo_slots, 0, 0, base, offsets, m, v, vertices, scratch, grad_out, V,
                        lambda_lap, lambda_offsets, 0.f, 0.f, lr_vert, eps, opt_state, vert_state, loss_out, stream);
}

int n2m_s1_vert_step_reg(const float* grad_vclip, const float* grad_vworld, const float* mvp, const void* topo_keys, const int32_t* topo_opp,
                         uint32_t topo_slots, uint32_t num_edges, uint32_t num_pairs, const float* base, float* offsets, float* m, float* v,
                         float* vertices, float* scratch, float* grad_out, uint32_t V, float lambda_lap, float lambda_offsets, float lambda_normal,
                         float lambda_edgelen, float lr_vert, float eps, const float* opt_state, float* vert_state, float* loss_out,
                         n2m_stream_t stream) {
    N2M_REQUIRE(lambda_normal >= 0.f && lambda_edgelen >= 0.f, "s1_vert_step_reg", "the weights must be >= 0");
    return s1_vert_step(grad_vclip, grad_vworld, mvp, topo_keys, topo_opp, topo_slots, num_edges, num_pairs, base, offsets, m, v, vertices, scratch,
                        grad_out, V, lambda_lap, lambda_offsets, lambda_normal, lambda_edgelen, lr_vert, eps, opt_state, vert_state, loss_out,
                        stream);
}

int n2m_s1_vert_step_world(const float* grad_vclip, const float* grad_vworld, const float* mvp, const void* topo_keys, uint32_t topo_slots,
                           const float* base, float* offsets, float* m, float* v, float* vertices, float* scratch, float* grad_out, uint32_t V,
                           float lambda_lap, float lambda_offsets, float lr_vert, float eps, const float* opt_state, float* vert_state,
                           float* loss_out, n2m_stream_t stream) {
    N2M_REQUIRE(grad_vworld, "s1_vert_step_world", "null pointer");
    return s1_vert_step(grad_vclip, grad_vworld, mvp, topo_keys, nullptr, topo_slots, 0, 0, base, offsets, m, v, vertices, scratch, grad_out, V,
                        lambda_lap, lambda_offsets, 0.f, 0.f, lr_vert, eps, opt_state, vert_state, loss_out, stream);
}

}  // extern "C"
