/* n2m_b200_raster.h -- C ABI of the stage-1 mesh path of libn2m_b200.so.
 *
 * The reference's stage 1 (NeRFRenderer.render_stage1, nerf/renderer.py:806-935) rasterizes the refined mesh with the third-party
 * nvdiffrast library and runs the colour MLPs on the covered pixels.  These entry points replace the two nvdiffrast operators on
 * that path, with nvdiffrast's documented output convention; the reference-side binding is `nerf2mesh_b200.raster`
 * (`rasterize`, `interpolate` with the argument order of `nvdiffrast.torch`), see INTEGRATION.md.
 *
 *   n2m_rasterize             dr.rasterize(glctx, pos, tri, (H, W))   (renderer.py:860; also :338, :968)
 *       pos  [V,4] f32 clip-space vertices, tri [F,3] i32, rast [H,W,4] f32 = (u, v, z/w, triangle_id + 1), zeros where empty;
 *       pixel (x, y) samples NDC ((x+0.5)/W*2-1, (y+0.5)/H*2-1); (u, v) perspective-correct barycentrics of vertices 0 / 1;
 *       vis [H*W] u64 and queue [F+1] u32 are caller-allocated scratch.  Fragments outside -1 <= z/w <= 1 are clipped; triangles that
 *       cross the camera plane (some w <= 0) are rasterised in homogeneous coordinates (the part in front of the near plane).
 *   n2m_interpolate_forward   dr.interpolate(attr, rast, tri)         (renderer.py:862-863): out [H*W,A] = u a0 + v a1 + (1-u-v) a2
 *   n2m_interpolate_backward  its gradient w.r.t. attr [V,A] (accumulated into the caller's zero-initialised buffer)
 *   n2m_interpolate_backward_rast  its gradient w.r.t. rast: grad_rast [H*W,4] = (du, dv, 0, 0) with du = sum_a g_a (a0_a - a2_a),
 *                             dv = sum_a g_a (a1_a - a2_a) at covered pixels, zeros elsewhere (written, not accumulated)
 *   n2m_rasterize_backward    dr.rasterize's gradient w.r.t. pos, as nvdiffrast defines it: only the (u, v) channels of grad_rast [H*W,4]
 *       carry gradient; (u, v) = (a0, a1) / (a0 + a1 + a2) with the edge functions a_k = p'_{k+1} x p'_{k+2} of p'_k = (x_k - X w_k,
 *       y_k - Y w_k) at the pixel's NDC centre (X, Y) -- the same expression for triangles that cross the camera plane.  d/d(x, y, w)
 *       ACCUMULATED into the caller's grad_pos [V,4]; clip z gets nothing.
 *   n2m_compact_covered      xyzs[mask], dirs[mask] of renderer.py:865-880 without the boolean-mask host sync: covered pixel
 *                             indices + their positions / view directions, count in *counter (device)
 *   n2m_antialias_*           dr.antialias(color, rast, pos, tri, pos_gradient_boost=b)   (renderer.py:886-887), csrc/antialias.cu:
 *       topology: edge -> opposing-vertex hash of the mesh (the library's "topology hash"), `keys` [slots] u64 and `opp` [2*slots] i32
 *       caller-allocated, slots = n2m_antialias_topology_slots(F) (a power of two >= 3 F); rebuilt only when `tri` changes;
 *       forward: out [H*W,C] = color + silhouette blends, C = 1..4, out must not alias color;
 *       backward: grad_color [H*W,C] (may be NULL) and grad_pos [V,4] (may be NULL; ACCUMULATED into the caller's zero-initialised
 *       buffer: gradients w.r.t. clip-space x, y, w, multiplied by pos_gradient_boost), from grad_out [H*W,C] and the forward inputs.
 */
#ifndef N2M_B200_RASTER_H
#define N2M_B200_RASTER_H

#include "n2m_b200.h"
#include "n2m_b200_fused.h"   /* n2m_s0_params (n2m_s1_offset_grad) */

#ifdef __cplusplus
extern "C" {
#endif

int n2m_rasterize(const float* pos, uint32_t V, const int32_t* tri, uint32_t F, uint32_t H, uint32_t W, void* vis, uint32_t* queue,
                  float* rast, n2m_stream_t stream);
int n2m_interpolate_forward(const float* attr, uint32_t V, uint32_t A, const float* rast, const int32_t* tri, uint32_t num_pixels,
                            float* out, n2m_stream_t stream);
int n2m_interpolate_backward(const float* grad_out, const float* rast, const int32_t* tri, uint32_t num_pixels, uint32_t V, uint32_t A,
                             float* grad_attr, n2m_stream_t stream);
int n2m_interpolate_backward_rast(const float* grad_out, const float* attr, const float* rast, const int32_t* tri, uint32_t num_pixels, uint32_t A,
                                  float* grad_rast, n2m_stream_t stream);
int n2m_rasterize_backward(const float* pos, uint32_t V, const int32_t* tri, const float* rast, const float* grad_rast, uint32_t H, uint32_t W,
                           float* grad_pos, n2m_stream_t stream);
int n2m_compact_covered(const float* rast, const float* xyz, const float* dirs, uint32_t num_pixels, uint32_t cap, int32_t* counter,
                        int32_t* pix, float* pts, float* pdirs, n2m_stream_t stream);

uint32_t n2m_antialias_topology_slots(uint32_t F);
int n2m_antialias_topology(const int32_t* tri, uint32_t F, void* keys, int32_t* opp, uint32_t slots, n2m_stream_t stream);
int n2m_antialias_forward(const float* color, const float* rast, const float* pos, const int32_t* tri, const void* keys, const int32_t* opp,
                          uint32_t slots, uint32_t H, uint32_t W, uint32_t C, float* out, n2m_stream_t stream);
int n2m_antialias_backward(const float* color, const float* rast, const float* pos, const int32_t* tri, const void* keys, const int32_t* opp,
                           uint32_t slots, uint32_t H, uint32_t W, uint32_t C, const float* grad_out, float pos_gradient_boost,
                           float* grad_color, float* grad_pos, n2m_stream_t stream);

/* ---- stage-1 texture-MLP step (csrc/stage1.cu; host side nerf2mesh_b200/stage1.py) ----
 * n2m_s1_points: covered pixels of `rast` [h,w,4] -> compacted surface points for the stage-0 gather / MLP / backward kernels:
 *   pts [cap,3] = dr.interpolate(vertices, rast, tri) at the covered pixels, pdirs [cap,3] = rays_d [h/ssaa * w/ssaa, 3] up-sampled
 *   nearest-neighbour (renderer.py:828-829), recs [cap] float4 = (0, 0, 0, k) (a march record whose sample is its own origin),
 *   inv [h*w] = slot of each pixel or -1; counters (>= 16 int32): [0] covered pixels, [1] min([0], cap), [2] overflow flag.
 * n2m_s1_loss: per low-res pixel: image = mean(alpha * rgb) + (1 - mean(alpha)) * bg, MSE (+ lambda_mask * mask term for rgba targets)
 *   averaged over the h0*w0 pixels into loss_out[0]; dout [cap] float4 = (0, dL/drgb) * loss_scale for the covered pixels. */
int n2m_s1_points(const float* rast, const float* verts, const int32_t* tri, const float* rays_d, uint32_t h, uint32_t w, uint32_t ssaa,
                  uint32_t cap, int32_t* counters, int32_t* inv, float* pts, float* pdirs, void* recs, n2m_stream_t stream);
/* n2m_s1_points_contract: n2m_s1_points with contract != 0 applying the L-inf contract() of renderer.py:25-32 to each interpolated point
 * before it is stored (unbounded scenes, Stage0Config.contract; the texture bake's n2m_s1_bake_points uses the same expression); pdirs are
 * unchanged.  contract = 0 is n2m_s1_points. */
int n2m_s1_points_contract(const float* rast, const float* verts, const int32_t* tri, const float* rays_d, uint32_t h, uint32_t w,
                           uint32_t ssaa, uint32_t cap, int32_t* counters, int32_t* inv, float* pts, float* pdirs, void* recs,
                           uint32_t contract, n2m_stream_t stream);
int n2m_s1_loss(const void* out, const int32_t* inv, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0,
                uint32_t ssaa, float lambda_mask, const float* loss_scale, void* dout, float* image, float* weights_sum, float* loss_out,
                n2m_stream_t stream);


/* antialiased variant of the step (renderer.py:881-907 with dr.antialias): n2m_s1_rgba scatters the per-point colours `out` [cap] float4
 * (sigma, r, g, b) into rgba [h*w] float4 = (r, g, b, mask) (zero where uncovered); after n2m_antialias_forward (C = 4),
 * n2m_s1_loss_aa evaluates clamp, alphas * rgbs, the ssaa average, the background mix and the loss of n2m_s1_loss on the antialiased
 * image aa [h*w] float4 and writes d_aa = d loss / d aa * loss_scale; after n2m_antialias_backward, n2m_s1_dout gathers the colour
 * part of the image gradient into dout [cap] float4 = (0, dr, dg, db) for the covered pixels. */
int n2m_s1_rgba(const void* out, const int32_t* inv, uint32_t num_pixels, void* rgba, n2m_stream_t stream);
int n2m_s1_loss_aa(const void* aa, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa,
                   float lambda_mask, const float* loss_scale, void* d_aa, float* image, float* weights_sum, float* loss_out,
                   n2m_stream_t stream);
int n2m_s1_dout(const void* grad_rgba, const int32_t* inv, uint32_t num_pixels, void* dout, n2m_stream_t stream);

/* evaluation (render_stage1 at inference, renderer.py:886-907): n2m_s1_render_compose, one thread per low-res pixel of h0 x w0, over
 * img [h*w] float4 = (r, g, b, alpha) at (h, w) = ssaa * (h0, w0) -- the antialiased image, or n2m_s1_rgba's (alpha 0 or 1) --, and
 * rast [h,w,4] of the same view: image [h0*w0,3] = mean(clamp(alpha) * clamp(rgb)) + (1 - mean(clamp(alpha))) * bg [h0*w0,3],
 * weights_sum [h0*w0] = mean(clamp(alpha)), depth [h0*w0] = mean(clamp(alpha) * rast.z).  image and weights_sum are bit-identical to
 * those n2m_s1_loss_aa writes for the same img (and n2m_s1_loss for the n2m_s1_rgba image); nothing else is written. */
int n2m_s1_render_compose(const void* img, const float* rast, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa, float* image,
                          float* weights_sum, float* depth, n2m_stream_t stream);

/* mesh refinement (opt.refine: update_triangles_errors, renderer.py:893-903,923-943; utils.py:720-721): n2m_s1_loss_err and
 * n2m_s1_loss_aa_err are n2m_s1_loss / n2m_s1_loss_aa that also, for every low-res pixel whose top-left super-sample (y0*ssaa, x0*ssaa)
 * of rast [h,w,4] is covered by face f (rast.w = f + 1, f < F), add the pixel's loss (before the 1/(h0*w0) mean and without loss_scale)
 * to face_err[f] and 1 to face_cnt[f].  face_err, face_cnt [F] f32 accumulate across calls (the caller zeroes them); fp32 atomics, so
 * face_err is deterministic up to summation order and face_cnt is exact below 2^24 hits per face. */
int n2m_s1_loss_err(const void* out, const int32_t* inv, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0,
                    uint32_t ssaa, float lambda_mask, const float* loss_scale, void* dout, float* image, float* weights_sum, float* loss_out,
                    const float* rast, float* face_err, float* face_cnt, uint32_t F, n2m_stream_t stream);
int n2m_s1_loss_aa_err(const void* aa, const float* gt, uint32_t gt_channels, const float* bg, uint32_t h0, uint32_t w0, uint32_t ssaa,
                       float lambda_mask, const float* loss_scale, void* d_aa, float* image, float* weights_sum, float* loss_out,
                       const float* rast, float* face_err, float* face_cnt, uint32_t F, n2m_stream_t stream);

/* vertex-offset optimizer of stage 1 (`vertices_offsets`: nn.Parameter at renderer.py:160, Adam group with lr_vert at :180; regularisers
 * utils.py:750-779).  n2m_s1_vert_check: non-finite scan of the loss-scaled clip-space gradient grad_vclip [V,4] into found_inf
 * (opt_state[3]) -- call it BEFORE the optimizer head.  n2m_s1_vert_step (between the optimizer head and its post kernel):
 *   grad = (grad_vclip . mvp[:, :3]) / loss_scale + lambda_lap * d/dv mean_i |(L v)_i| + lambda_offsets * d/doff mean_i sum_c off_ic^2
 * with the uniform Laplacian L = D - A over the unique edges of the mesh (the edge hash of n2m_antialias_topology), Adam(0.9, 0.999, eps)
 * with its own step count vert_state[0] on offsets [V,3], vertices = base + offsets; skipped when found_inf is set.  scratch [6 V] f32;
 * grad_out [V,3] (nullable) receives the total gradient; loss_out (nullable) += lambda_lap * mean |L v| (the offsets term is left to
 * the caller: it needs no kernel).  mvp [4,4] row-major on the device; lr_vert < 0: the learning rate is read from vert_state[1]. */
int n2m_s1_vert_check(const float* grad_vclip, uint32_t V, float* opt_state, n2m_stream_t stream);
int n2m_s1_vert_step(const float* grad_vclip, const float* mvp, const void* topo_keys, uint32_t topo_slots, const float* base, float* offsets,
                     float* m, float* v, float* vertices, float* scratch, float* grad_out, uint32_t V, float lambda_lap, float lambda_offsets,
                     float lr_vert, float eps, const float* opt_state, float* vert_state, float* loss_out, n2m_stream_t stream);

/* colour-field path of the vertex gradient (--enable_offset_nerf_grad: renderer.py:877-879 with xyzs[mask_flatten] not detached).
 * n2m_s1_offset_grad (after n2m_s0_mlp_bwd, before n2m_s1_vert_check): for every super-sampled pixel with a point (inv[i] >= 0), the
 * loss-scaled gradient w.r.t. its surface point = the colour-net input columns kColXyz..+2 of its denc_tiles row + the colour hash grid's
 * input gradient (the reference's dy_dx over the fp16 colour features of `table`, zero outside [0,1]^3), through the Jacobian of
 * contract() when p->contract; then dr.interpolate's backward: b_k dx ACCUMULATED into grad_vworld [V,3] (world space), and (du, dv)
 * through n2m_rasterize_backward's expression ACCUMULATED into grad_vclip [V,4] (clip space, beside n2m_antialias_backward's gradient).
 * rast [h,w,4], verts [V,3], vclip [V,4], tri, inv, pts: those of the step (n2m_rasterize, n2m_s1_points).  A non-finite gradient sets
 * found_inf (opt_state[3]) and is not scattered.  p->num_levels must be 16.
 * n2m_s1_vert_step_world: n2m_s1_vert_step with the image-loss part (grad_vclip . mvp[:, :3] + grad_vworld) / loss_scale. */
int n2m_s1_offset_grad(const n2m_s0_params* p,const float* rast, const float* verts, const float* vclip, const int32_t* tri, const int32_t* inv,
                       uint32_t h, uint32_t w, const float* pts, const void* denc_tiles, const void* table, const int32_t* offsets,
                       float* grad_vclip, float* grad_vworld, float* opt_state, n2m_stream_t stream);
int n2m_s1_vert_step_world(const float* grad_vclip, const float* grad_vworld, const float* mvp, const void* topo_keys, uint32_t topo_slots,
                           const float* base, float* offsets, float* m, float* v, float* vertices, float* scratch, float* grad_out, uint32_t V,
                           float lambda_lap, float lambda_offsets, float lr_vert, float eps, const float* opt_state, float* vert_state,
                           float* loss_out, n2m_stream_t stream);

/* mesh regularisers of the vertex offsets (utils.py:759-769: lambda_normal * pytorch3d mesh_normal_consistency + lambda_edgelen *
 * pytorch3d mesh_edge_loss with target length 0), over the edge hash of n2m_antialias_topology (topo_keys, topo_opp, topo_slots).
 * n2m_s1_mesh_reg_setup (once per mesh; synchronises `stream`): counts[0] = E, the unique edges (occupied slots), counts[1] = P, the
 *   edges with exactly two faces, counts[2] = edges with more than two faces (the hash keeps two of them: the normal term needs a mesh
 *   without), counts[3] = faces with a repeated vertex index; counts is host memory [4], scratch device memory [topo_slots + 4] u32.
 * n2m_s1_mesh_reg: for vertices [V,3], ACCUMULATES into grad [V,3] the gradient of
 *   lambda_edgelen / E * sum_edges |v_a - v_b|^2 + lambda_normal / P * sum_pairs (1 - cos(n_c, -n_d))
 *   with n_c = (v_b - v_a) x (v_c - v_a), n_d likewise, for the edge (a < b) and the opposite vertices c, d of its two faces; cos as
 *   torch.cosine_similarity(eps = 1e-8) computes and differentiates it (each vector divided by max(|n|, eps)); loss_out (nullable) += the
 *   value.  A weight whose count (E or P) is 0 contributes nothing.
 * n2m_s1_vert_step_reg: n2m_s1_vert_step with grad_vworld nullable (non-null: n2m_s1_vert_step_world's image-loss part) and both
 *   regularisers added to the gradient and to loss_out, on vertices before the update; scratch [9 V] f32.  With lambda_normal =
 *   lambda_edgelen = 0 it is n2m_s1_vert_step / n2m_s1_vert_step_world. */
int n2m_s1_mesh_reg_setup(const int32_t* tri, uint32_t F, const void* topo_keys, uint32_t topo_slots, uint32_t* scratch, uint32_t* counts,
                          n2m_stream_t stream);
int n2m_s1_mesh_reg(const void* topo_keys, const int32_t* topo_opp, uint32_t topo_slots, uint32_t num_edges, uint32_t num_pairs,
                    const float* vertices, float lambda_normal, float lambda_edgelen, float* grad, float* loss_out, n2m_stream_t stream);
int n2m_s1_vert_step_reg(const float* grad_vclip, const float* grad_vworld, const float* mvp, const void* topo_keys, const int32_t* topo_opp,
                         uint32_t topo_slots, uint32_t num_edges, uint32_t num_pairs, const float* base, float* offsets, float* m, float* v,
                         float* vertices, float* scratch, float* grad_out, uint32_t V, float lambda_lap, float lambda_offsets, float lambda_normal,
                         float lambda_edgelen, float lr_vert, float eps, const float* opt_state, float* vert_state, float* loss_out,
                         n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_RASTER_H */
