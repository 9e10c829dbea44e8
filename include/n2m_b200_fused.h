/* n2m_b200_fused.h -- C ABI of the FUSED stage-0 train path of libn2m_b200.so.
 *
 * The operator-level entry points in n2m_b200.h are the drop-in replacements for the reference's
 * pybind functions.  The entry points here implement the same arithmetic as ONE pipeline with a
 * GPU-native data layout, no host synchronisation and no per-step allocation, so the whole train
 * step can be captured in a CUDA graph.  What each stage replaces in the reference:
 *
 *   n2m_s0_march          raymarching.near_far_from_aabb + march_rays_train (raymarching.py:19-49,181-245;
 *                          raymarching.cu:92-145,338-475) without the .item() sync (raymarching.py:232)
 *   n2m_s0_encode_fwd     GridEncoder.forward x2 (grid.py:151-168; gridencoder.cu:88-196) + cat + safe_normalize
 *   n2m_s0_tv             grad_total_variation (gridencoder.cu:506-609; utils.py:801-823), its own launch
 *   n2m_s0_mlp_fwd        sigma_net / color_net / specular_net + trunc_exp / sigmoid / clamp
 *                          (nerf/network.py:81-108,159-189) on wgmma tensor cores
 *   n2m_s0_composite_loss composite_rays_train fwd+bwd (raymarching.cu:501-694), background mix
 *                          (renderer.py:804) and the MSE(+mask, +specular) loss (utils.py:660-738)
 *   n2m_s0_mlp_bwd        autograd of the three MLPs (dgrad + wgrad) on wgmma
 *   n2m_s0_encode_bwd     grid_encode backward x2 (gridencoder.cu:248-339)
 *   n2m_s0_adam_*         GradScaler.unscale_/step/update + Adam(eps 1e-15) + the per-step fp32->fp16
 *                          table cast (grid.py:45-46) + zero_grad  (utils.py:549,1163,1176-1177)
 * One function per stage; the five between march and optimizer take a ray-range part (see "Ray-range parts" below).
 *
 * Data layout (all buffers allocated by the caller, see nerf2mesh_b200/stage0.py):
 *   table      [rows]  8-byte entries {float density_feature; half2 colour_features}: the density table
 *              (fp32, C=1) and the fp16 working copy of the colour table (C=2) interleaved so that one
 *              64-bit access serves both encoders.  fp32 colour masters live in `color_master [rows] float2`.
 *   gtable     [rows]  float4 {g_density, g_colour0, g_colour1, 0}, loss-scaled, reduced with one
 *              red.global.add.v4.f32 per lattice corner.
 *   enc_tiles  one 16 KiB image per 128 samples: fp16 [128 x 64] in the no-swizzle core-matrix layout
 *              (chunk-major, wg.cuh): cols 0-2 xyz, 3-18 density features, 19-50 colour features,
 *              51-53 unit view direction, 54..53+ind_dim appearance codes, rest zero (see "Per-image appearance codes").  It is the A operand of every first-layer GEMM and is
 *              staged global->shared with a single bulk async copy.
 *   recs       [Mcap] float4 {t_before, dt, t_after, ray_id (bits)} per sample, ray order.
 *   counters   int32 [17]: [0] M (total samples marched), [1] min(M, Mcap), [2] overflow flag, [3] / [15] samples inside / outside the
 *              unit cube (counted by the TV pass, read by n2m_s0_tv_random),
 *              [4..12] sample offset of the first ray of every eighth of the batch (ray n*e/8, e = 0..8; [4] = 0,
 *              [12] = [1]): the boundaries of the ray-range parts (see "Ray-range parts" below).
 *              [13] += 1 for every march whose M exceeded Mcap, [14] = largest M seen (persistent capacity accounting: the rays
 *              that do not fit -- always the last rays of the batch -- are rendered as background and get no gradient, which
 *              the reference never does (it allocates exactly M, raymarching.py:232-238); hosts must watch [13] and grow Mcap).
 *              [16] n, the active ray count of the batch (adaptive ray count only: written by n2m_s0_march when it is given a
 *              control block; the batch is the first n of the N rows and n = N otherwise).
 *              Entry points without parts (and nparts == 1) read only [1], so hand-filled 4-entry arrays work there.
 *   ray_ctl    int32 [4], persistent, adaptive ray count only (the reference's --adaptive_num_rays, nerf/utils.py:795-797):
 *              [0] ray count n of the next march, in [1, N]; the host sets it to the first step's count.  [1] += 1 for every march
 *              whose requested count exceeded N and was clamped to it; [2] = largest count requested before that clamp (saturated
 *              at INT32_MAX); [3] unused.  The host zeroes [1] / [2] when it reads them.
 *   wpack      packed fp16 MLP weights in tensor-core tile layout (n2m_s0_pack_weights).
 */
#ifndef N2M_B200_FUSED_H
#define N2M_B200_FUSED_H

#include "n2m_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    float bound;            /* marching bound (renderer.real_bound) */
    float grid_bound;       /* bound that normalises positions for the hash grid (renderer.bound) */
    float inv_2gb;          /* float32(1) / float32(2 * grid_bound) -- torch divides by a scalar this way */
    float dt_gamma;
    float min_near;
    float T_thresh;
    float S;                /* log2(per_level_scale) as float32 (grid.py:38) */
    float lambda_mask;
    float lambda_specular;
    float lambda_tv;
    float lambda_entropy;   /* utils.py:728-733: entropy of the per-sample weights and of weights_sum (0 = off) */
    uint32_t contract;
    uint32_t max_steps;
    uint32_t cascades;
    uint32_t grid_size;
    uint32_t num_levels;    /* must be 16 */
    uint32_t base_res;
    uint32_t shading_full;  /* 0 = 'diffuse' (first diffuse_step iterations), 1 = 'full'; 2 = 'specular': n2m_s0_mlp_fwd only (evaluation),
                               which then writes (sigma, specular) -- the training and backward kernels take 0 or 1 */
    uint32_t gt_has_alpha;  /* gt is rgba: blend with bg and add the mask loss (utils.py:662-667,681-683) */
    uint32_t ind_dim;       /* width D of the per-image appearance codes, 0..10 (0 = none).  Read by the *_codes / code entry points; the
                               plain gather entry points write no code columns, and n2m_s0_render_rounds refuses ind_dim > 0 (it has no
                               code row: use n2m_s0_render_rounds_codes) */
} n2m_s0_params;

/* one-time per-process setup (kernel attributes of every stage); call before the first launch / graph capture */
int n2m_s0_init(void);

/* test hook: 1 = sequential one-thread-per-ray marcher, 0 = warp-per-ray marcher (default); same results */
int n2m_s0_set_serial_march(int on);

/* test hook: launch form of the scatter (n2m_s0_encode_bwd).  0 = chosen from the part count (default), 1 = 128-thread CTAs on the
 * resident slots of every SM, 2 = 1024-thread CTAs, one per SM, on 1/nparts of the SMs; same results up to the order of the fp32
 * additions */
int n2m_s0_set_scatter_form(int form);

/* the TV gradient of the step's samples: reads recs/table, adds into gtable, counts counters[3] / [15]; independent of the MLP kernels,
 * so a host may run it on a forked stream beside them */
int n2m_s0_tv(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
              const float* rays_d, const void* table, const int32_t* offsets, void* gtable, const float* loss_scale,
              n2m_stream_t stream);
/* GridEncoder.grad_total_variation's fallback (grid.py:181-183): a TV call of post_train_step (utils.py:815-823) that received no sample
 * position evaluates the TV gradient at `num_points` (reference: 10^6) uniformly random points instead.  The TV pass of the step counts the
 * samples inside / outside the unit cube into counters[3] / counters[15]; this launch (after it, same stream) adds the fallback of every
 * group that stayed empty and exits at once otherwise.  Points: counter-based hash of (optimizer step, index).  `dump` (nullable,
 * [num_points,3]): test hook -- run unconditionally with weight lambda_tv and store the points. */
int n2m_s0_tv_random(const n2m_s0_params* p, const int32_t* counters, const void* table, const int32_t* offsets, void* gtable,
                     const float* loss_scale, uint32_t num_points, float* dump, n2m_stream_t stream);

/* sizes of the packed weight blob (bytes) and of the flat fp32 MLP parameter / gradient vector (floats) */
uint32_t n2m_s0_wpack_bytes(void);
uint32_t n2m_s0_mlp_param_count(void);      /* 7648 = 608+32 + 2240+4096+384 + 192+96 */

/* fp32 masters (reference nn.Linear layouts [out,in], concatenated: sigma0, sigma1, color0, color1, color2,
 * spec0, spec1) -> packed fp16 tiles */
int n2m_s0_pack_weights(const float* mlp_params, void* wpack, n2m_stream_t stream);

/* interleave / de-interleave the hash tables (import / export of reference-format tensors) */
int n2m_s0_pack_tables(const float* emb_density, const float* emb_color, uint32_t rows,
                       void* table, void* color_master, n2m_stream_t stream);
int n2m_s0_unpack_tables(const void* table, const void* color_master, uint32_t rows,
                         float* emb_density, float* emb_color, n2m_stream_t stream);
/* gtable (loss-scaled float4) -> reference-format gradients, divided by *loss_scale */
int n2m_s0_unpack_grads(const void* gtable, uint32_t rows, const float* loss_scale,
                        float* g_density, float* g_color, n2m_stream_t stream);

/* march: near/far + count + scan + sample records.  cam_near_far [N,2] nullable (renderer.py:689-691).
 * ray_ctl (nullable): adaptive ray count.  NULL marches all N rays.  Given a control block the march takes n = min(ray_ctl[0], N), records
 * n in counters[16], marches rays [0, n) only (rays >= n get zero samples and their rows are never read, NaN included), cuts the parts at
 * ray n*e/8, and leaves the next march's count in ray_ctl[0]:  rint(((double)num_points / (double)M) * (double)n), M = counters[0]
 * (never capped by Mcap), clamped to [1, N].  M == 0 keeps n (the reference would divide by zero there). */
int n2m_s0_march(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const float* aabb,
                 const float* cam_near_far, const uint8_t* bitfield, const float* noises, uint32_t N,
                 int32_t* rays, int32_t* counters, float* tbuf, void* recs, uint32_t Mcap,
                 int32_t* ray_ctl, uint32_t num_points, n2m_stream_t stream);

/* the hash-grid gather of the march records into enc_tiles */
int n2m_s0_encode_fwd(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap,
                      const float* rays_o, const float* rays_d, const void* table, const int32_t* offsets,
                      void* enc_tiles, uint32_t part, uint32_t nparts, n2m_stream_t stream);

/* same gather for explicit positions xyz [P,3] in [-bound, bound] (dirs [P,3] nullable); counters[1] = P.  Used by the
 * density-grid update and by tests. */
int n2m_s0_encode_points(const n2m_s0_params* p, const float* xyz, const float* dirs, const int32_t* counters, uint32_t Pcap,
                         const void* table, const int32_t* offsets, void* enc_tiles, n2m_stream_t stream);

/* density-grid update pieces (NeRFRenderer.update_extra_state, renderer.py:1074-1149):
 *   grid_points : jittered centres of cells [first_cell, first_cell+count) of one cascade, Morton order; noise [H^3,3] in [0,1) is the
 *                 cascade's whole draw in the reference's meshgrid order (row x*H*H + y*H + z), i.e. torch.rand_like(cas_xyzs)
 *   grid_update : cells[i] = max(cells[i] * decay, sigma_i) where both >= 0 (sigma_i = out[i].x)
 *   packbits_dev: bit = grid > min(*mean_density, density_thresh), threshold read on the device */
int n2m_s0_grid_points(uint32_t H, uint32_t first_cell, uint32_t count, float cas_bound, const float* noise, float* xyz,
                       n2m_stream_t stream);
int n2m_s0_grid_update(const void* out, uint32_t count, float decay, float* grid_cells, n2m_stream_t stream);
int n2m_s0_packbits_dev(const float* grid, uint32_t nbytes, const float* mean_density, float density_thresh, uint8_t* bitfield,
                        n2m_stream_t stream);

/* NeRFRenderer.mark_untrained_grid (renderer.py:985-1071; called once by Trainer.train, utils.py:925): density_grid [cascades, H^3]
 * cells (Morton order) that no camera sees (camera-space z > near, |x| < cx/fx * z + 2 * half_cell, same for y) or that lie outside
 * aabb (+- half a cell) are set to -1.  poses [num_poses,4,4] camera-to-world; intrinsics [intr_count,4] = (fx, fy, cx, cy) on the
 * DEVICE with intr_count 1 or num_poses; cam_near [num_poses] nullable (else min_near); *count_out (nullable) = marked cells. */
int n2m_mark_untrained_grid(const float* poses, uint32_t num_poses, const float* intrinsics, uint32_t intr_count,
                            const float* cam_near, float min_near, const float* aabb, float bound, uint32_t cascades,
                            uint32_t H, float* density_grid, int32_t* count_out, n2m_stream_t stream);

/* batch sampling on the device = get_rays (nerf/utils.py:236-290) + the stage-0 training collate (nerf/provider.py:300-331)
 * for N random (image, pixel) pairs: poses [num_poses,4,4] (device), intrinsics_host float[4] {fx, fy, cx, cy} (HOST),
 * img_idx / pix_idx int32 [N] (device; pix = j * W + i), images uint8 [num_poses, H, W, C] (device, nullable with gt).
 * Writes rays_o, rays_d [N,3] (unnormalised directions) and gt [N,C] = pixel / 255.  Indices are not range-checked. */
int n2m_s0_gen_rays(const float* poses, uint32_t num_poses, const float* intrinsics_host, uint32_t H, uint32_t W,
                    const int32_t* img_idx, const int32_t* pix_idx, const uint8_t* images, uint32_t C, uint32_t N,
                    float* rays_o, float* rays_d, float* gt, n2m_stream_t stream);

/* out [Mcap] float4 {sigma, r, g, b}; spec_sq_sum: += sum over samples of |specular|^2 (for the loss value) */
int n2m_s0_mlp_fwd(const n2m_s0_params* p, const void* enc_tiles, const int32_t* counters, uint32_t Mcap,
                   const void* wpack, void* out, float* spec_sq_sum, uint32_t part, uint32_t nparts, n2m_stream_t stream);

/* per ray: composite, loss, composite backward.  gt [N,4] (rgba) or [N,3]; bg [N,3].
 * dout [Mcap] float4 {dL/dsigma, dL/dr, dL/dg, dL/db} * loss_scale (zero beyond each ray's break).
 * loss_out float[4]: [0] += sum_rays per-ray loss / n (rgb + mask + ray-level entropy), [1] is the MLP forward's sum |spec|^2,
 * [2] += sum of H(weights_k) over the weights the compositor touched, [3] += their count (lambda_entropy > 0 only);
 * image/ws/depth [N] outputs.  active_rays (nullable, = counters + 16 after a march given a control block): the batch is its first
 * n = *active_rays rays -- the parts, the loss's 1/n and the outputs cover those, rows >= n are neither read nor written; NULL: n = N. */
int n2m_s0_composite_loss(const n2m_s0_params* p, const void* out, const void* recs, const int32_t* rays,
                          const int32_t* counters, uint32_t N, uint32_t Mcap, const float* gt, const float* bg,
                          const float* loss_scale, void* dout, float* image, float* weights_sum, float* depth,
                          float* loss_out, const int32_t* active_rays, uint32_t part, uint32_t nparts, n2m_stream_t stream);

/* MLP backward: denc_tiles (same tile layout as enc_tiles, fp16, loss-scaled), g_mlp flat fp32 [7648] += */
int n2m_s0_mlp_bwd(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters,
                   uint32_t Mcap, const void* wpack, void* denc_tiles, float* g_mlp, const float* loss_scale,
                   uint32_t part, uint32_t nparts, n2m_stream_t stream);

/* scatter denc into gtable */
int n2m_s0_encode_bwd(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap,
                      const float* rays_o, const float* rays_d, const void* denc_tiles, const void* table,
                      const int32_t* offsets, void* gtable, const float* loss_scale, uint32_t part, uint32_t nparts,
                      n2m_stream_t stream);

/* Ray-range parts.  The five stages above between march and optimizer run on part `part` of `nparts` (1, 2, 4 or 8) contiguous
 * ray ranges of the batch -- part k covers rays [n*k/nparts, n*(k+1)/nparts) of its n rays and their (contiguous, ray-ordered) samples -- so that
 * independent chains  gather -> MLP -> composite -> MLP backward -> scatter  of different parts can be in flight on
 * different streams: the latency-bound tensor-core MLP kernels of one part then share the SMs with the memory-bound
 * gather / scatter kernels of another.  A 128-sample tile that straddles a part boundary is computed by both parts,
 * each one reading / writing only its own rows (rows are masked by the [lo, hi) sample range taken from counters[4..12]);
 * losses, weight gradients and table gradients accumulate atomically, so the union of all parts equals the un-split call
 * up to fp32 summation order.  part = 0, nparts = 1 is the whole batch; it reads only counters[1]. */

/* optimizer state block (device, float[8]): [0] loss_scale, [1] growth_tracker, [2] adam step t,
 * [3] found_inf, [4] lr (host-written each step), [5] 1-beta1^t, [6] sqrt(1-beta2^t), [7] 1/loss_scale.
 * Every `loss_scale` pointer argument above is the base of this block: the kernels read [0] and set [3]
 * when they see a non-finite gradient (instead of GradScaler's separate unscale_/inf-check pass). */

/* Adam (betas 0.9/0.999, eps) on tables + MLP as four launches: head (MLP-gradient inf scan + step constants), tables, mlp
 * (+ weight repack), post (GradScaler update).  They unscale by loss_scale, skip everything when found_inf, refresh the fp16 working
 * copies (table, wpack) and zero gtable / g_mlp.  `tables` and `mlp` only read opt_state and touch disjoint buffers: a host may run
 * them on two streams between head and post (nerf2mesh_b200/stage0.py does). */
int n2m_s0_adam_head(const float* g_mlp, float* opt_state, n2m_stream_t stream);
int n2m_s0_adam_tables(void* table, void* color_master, void* gtable, float* m_table, float* v_table, uint32_t rows,
                       const float* opt_state, float eps, n2m_stream_t stream);
/* `tables` without zeroing the gradient rows: the host zeroes that gradient table on a side stream under the next step's forward pass
 * (which accumulates into the other parity table) */
int n2m_s0_adam_tables_keep(void* table, void* color_master, const void* gtable, float* m_table, float* v_table, uint32_t rows,
                            const float* opt_state, float eps, n2m_stream_t stream);
int n2m_s0_adam_mlp(float* mlp_params, float* g_mlp, float* m_mlp, float* v_mlp, void* wpack, const float* opt_state, float eps,
                    n2m_stream_t stream);
int n2m_s0_adam_post(float* opt_state, n2m_stream_t stream);

/* Fused forward (csrc/fused.cu): hash-grid gather + MLP forward of the WHOLE batch (nparts == 1) in one persistent, warp-specialised
 * launch -- two gather groups of four warps fill double-buffered tile images in shared memory, warps 0-3 run the tensor-core MLP rounds on
 * them; a copy of every image is stored to enc_tiles by the TMA unit for the backward pass.  Same arithmetic as n2m_s0_encode_fwd followed
 * by n2m_s0_mlp_fwd (bit-identical enc_tiles / out). */
int n2m_s0_fwd_fused(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                     const float* rays_d, const void* table, const int32_t* offsets, const void* wpack, void* enc_tiles, void* out,
                     float* spec_sq_sum, n2m_stream_t stream);

/* Evaluation renderer with the alive-ray bookkeeping on the device (csrc/render.cu) = NeRFRenderer.render, inference branch
 * (nerf/renderer.py:749-802: per round march_rays -> model -> composite_rays -> mask compaction, one host read-back per round).
 *   render_begin : near / far (+ per-ray camera clamp, nullable), zeroed weights_sum / depth / image [N], rays_t, the first alive list;
 *                  alive [2 N] i32, ctl [16] i32 (control block: [1] sample rows of the round -- the counters the forward kernels read --,
 *                  [8] alive rays, [9] slab width, [10] survivors appended so far, [11] list parity, [12] rounds run, [13] sample rows evaluated)
 *   render_rounds: `num_rounds` rounds of plan -> march (records {t, dt, t + dt, ray} in slab order) -> n2m_s0_encode_fwd -> n2m_s0_mlp_fwd
 *                  -> slab compositor (raymarching.cu:842-924) + survivor compaction, all sizes read on the device; `schedule` (HOST
 *                  array) = slab widths, clipped on the device to Mcap / alive; recs [Mcap] float4, enc_tiles [Mcap*64] half,
 *                  out [Mcap] float4; Mcap a multiple of 128 and >= N.  Afterwards ctl[10] = rays still alive.
 *   render_finish: image += (1 - weights_sum) * bg (renderer.py:804), bg [N,3] or NULL (then bg_scalar). */
int n2m_s0_render_begin(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const float* aabb, const float* cam_near_far,
                        uint32_t N, float* rays_t, float* rays_far, int32_t* alive, int32_t* ctl, float* weights_sum, float* depth,
                        float* image, n2m_stream_t stream);
int n2m_s0_render_rounds(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const uint8_t* bitfield, uint32_t N,
                         const uint32_t* schedule, uint32_t num_rounds, float* rays_t, float* rays_far, int32_t* alive, int32_t* ctl,
                         void* recs, void* enc_tiles, void* out, uint32_t Mcap, const void* table, const int32_t* offsets, const void* wpack,
                         float* weights_sum, float* depth, float* image, n2m_stream_t stream);
int n2m_s0_render_finish(float* image, const float* weights_sum, const float* bg, float bg_scalar, uint32_t N, n2m_stream_t stream);

/* EMA of the parameters = torch_ema.ExponentialMovingAverage as the reference's Trainer holds it (nerf/utils.py:544-545, decay 0.95
 * from main.py:241): `update` once per EPOCH (utils.py:1213-1214), parameters swapped with the shadow for evaluation
 * (utils.py:1250-1252,1340-1341) and for the 'best' checkpoint (utils.py:1389-1401).  shadow_density [rows] f32, shadow_color [rows] float2,
 * shadow_mlp [7648] f32.  ema_update: shadow -= one_minus_decay * (shadow - param).  ema_swap: params <-> shadow in place, fp16 working
 * copies (table colour half2, wpack) refreshed. */
int n2m_s0_ema_update(const void* table, const void* color_master, const float* mlp_params, float* shadow_density, void* shadow_color,
                      float* shadow_mlp, uint32_t rows, float one_minus_decay, n2m_stream_t stream);
int n2m_s0_ema_swap(void* table, void* color_master, float* mlp_params, float* shadow_density, void* shadow_color, float* shadow_mlp,
                    uint32_t rows, void* wpack, n2m_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Per-image appearance codes (the reference's --ind_dim D / --ind_num, renderer.py:97-104, network.py:72,159-166).
 * color_net.0 then reads [xyz | colour features | code of the sample's image]; the code enters the tile image at columns 54..53+D
 * (1 <= D <= 10, p->ind_dim = D), where W_C1 has room, so every GEMM keeps its shape.  The parameters of the feature live outside the
 * flat 7648-float MLP vector, in a second block `ind` [64*D + ind_num*D] fp32:
 *   ind[o*D + j]               = color_net.net.0.weight[o, 35 + j]   (the code columns of the colour net's first layer; lr)
 *   ind[64*D + i*D + j]        = individual_codes[i, j]              (one code per training image; 0.1 * lr)
 * with a gradient block g_ind of the same layout (loss-scaled, like g_mlp).  The *_codes entry points are the ones above plus the
 * code source; with p->ind_dim == 0 they do exactly what the plain ones do.  Code sources:
 *   codes + ray_img : codes = the [ind_num, D] code table, ray_img [N] int32 = image index of every ray (looked up through the ray id
 *                     of the march record; indices are not range-checked, as in n2m_s0_gen_rays);
 *   ray_img == NULL : `codes` points at the ONE code row [D] used for every sample of the launch (evaluation, stage 1).
 * ---------------------------------------------------------------------------------------- */
int n2m_s0_encode_fwd_codes(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                            const float* rays_d, const void* table, const int32_t* offsets, const float* codes, const int32_t* ray_img,
                            void* enc_tiles, uint32_t part, uint32_t nparts, n2m_stream_t stream);
/* n2m_s0_encode_points with one code row `code_row` [D] for every point */
int n2m_s0_encode_points_codes(const n2m_s0_params* p, const float* xyz, const float* dirs, const int32_t* counters, uint32_t Pcap,
                               const void* table, const int32_t* offsets, const float* code_row, void* enc_tiles, n2m_stream_t stream);
int n2m_s0_fwd_fused_codes(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                           const float* rays_d, const void* table, const int32_t* offsets, const float* codes, const int32_t* ray_img,
                           const void* wpack, void* enc_tiles, void* out, float* spec_sq_sum, n2m_stream_t stream);
/* n2m_s0_render_rounds with one code row `code_row` [D] for every sample (the reference evaluates with code 0, renderer.py:702-703) */
int n2m_s0_render_rounds_codes(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const uint8_t* bitfield, uint32_t N,
                               const uint32_t* schedule, uint32_t num_rounds, float* rays_t, float* rays_far, int32_t* alive, int32_t* ctl,
                               void* recs, void* enc_tiles, void* out, uint32_t Mcap, const void* table, const int32_t* offsets,
                               const void* wpack, const float* code_row, float* weights_sum, float* depth, float* image,
                               n2m_stream_t stream);
/* n2m_s0_mlp_bwd that also adds the weight gradient of the code columns to g_ind[0 .. 64*D) (loss-scaled, fp32).  The code columns'
 * input gradient is in denc_tiles columns 54..53+D either way. */
int n2m_s0_mlp_bwd_codes(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters, uint32_t Mcap,
                         const void* wpack, void* denc_tiles, float* g_mlp, float* g_ind, const float* loss_scale, uint32_t part,
                         uint32_t nparts, n2m_stream_t stream);
/* code gradient: g_codes[ray_img[n] * D + j] += sum over the samples of ray n of denc[sample, 54 + j] (fp16 loss-scaled terms summed in
 * fp32; one reduction per ray, one RED per ray and dimension), for the rays of part `part` of `nparts` (rays (offset, count) from the
 * march), samples below counters[1].  g_codes = g_ind + 64*D.  ray_img NULL: every ray adds into the one row at g_codes.  active_rays
 * (nullable, = counters + 16 after an adaptive march): the batch is its first n rays.  A non-finite term sets opt_state[3]. */
int n2m_s0_code_grad(const n2m_s0_params* p, const int32_t* rays, const int32_t* counters, uint32_t N, const void* denc_tiles,
                     const int32_t* ray_img, float* g_codes, float* opt_state, const int32_t* active_rays, uint32_t part, uint32_t nparts,
                     n2m_stream_t stream);
/* the code gradient of a launch with ONE code row (stage 1: the view's image): g_row[j] += sum over the sample rows below counters[1] of
 * denc[row, 54 + j]; Mcap = the capacity of denc_tiles (sizes the grid).  A non-finite term sets opt_state[3]. */
int n2m_s0_code_grad_row(const n2m_s0_params* p, const int32_t* counters, uint32_t Mcap, const void* denc_tiles, float* g_row,
                         float* opt_state, n2m_stream_t stream);
/* the code columns ind[0 .. 64*D) -> W_C1 columns 54..53+D of wpack (after n2m_s0_pack_weights, which zeroes them) */
int n2m_s0_pack_code_weights(const float* ind, uint32_t ind_dim, void* wpack, n2m_stream_t stream);
/* optimizer of the `ind` block (Adam, weight decay 0): `head` ORs a non-finite entry of g_ind[0, n) into found_inf and runs BEFORE
 * n2m_s0_adam_head; `codes` runs between n2m_s0_adam_head and n2m_s0_adam_post, after n2m_s0_adam_mlp on the same stream (whose repack
 * zeroes the code columns): it unscales, skips on found_inf, steps the code columns at lr and the codes at 0.1 * lr (renderer.py:173-174),
 * zeroes g_ind and repacks the code columns into wpack. */
int n2m_s0_adam_codes_head(const float* g_ind, uint32_t n, float* opt_state, n2m_stream_t stream);
int n2m_s0_adam_codes(float* ind, float* g_ind, float* m_ind, float* v_ind, uint32_t ind_dim, uint32_t ind_num, void* wpack,
                      const float* opt_state, float eps, n2m_stream_t stream);
/* EMA of the `ind` block, as n2m_s0_ema_update / n2m_s0_ema_swap (the swap runs after n2m_s0_ema_swap and repacks the code columns) */
int n2m_s0_codes_ema_update(const float* ind, float* shadow_ind, uint32_t n, float one_minus_decay, n2m_stream_t stream);
int n2m_s0_codes_ema_swap(float* ind, float* shadow_ind, uint32_t ind_dim, uint32_t ind_num, void* wpack, n2m_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Data-parallel optimizer fused with its collective over NVLink peer memory (csrc/dp.cu).
 * One process per GPU; buffers of the other ranks are mapped with CUDA IPC.
 * ---------------------------------------------------------------------------------------- */
int n2m_ipc_export(const void* ptr, void* handle_out /* 64 bytes */, uint64_t* offset_out);
int n2m_ipc_open(const void* handle, void** base_out);
int n2m_ipc_close(void* base);
uint32_t n2m_dp_ctx_bytes(void);
/* host image of the device context: per-peer pointers to gradient tables (two parities), working tables, MLP
 * gradient vectors, optimizer state blocks and flag arrays (>= 16 uint32 each, zero-initialised) */
int n2m_dp_ctx_fill(void* host_ctx, uint32_t world, uint32_t rank, uint32_t rows, uint32_t n_mlp,
                    void* const* gtab0, void* const* gtab1, void* const* table, void* const* gmlp0, void* const* gmlp1,
                    void* const* opt, void* const* flags, void* epoch);
int n2m_dp_barrier(const void* ctx, n2m_stream_t stream);
/* barrier -> reduce-scatter + Adam + all-gather on this rank's row slice -> MLP -> zero next-parity grads -> barrier.
 * color_master / m / v are slice-sized: ceil(rows / world) rounded up to a multiple of 4 rows. */
int n2m_dp_adam(const void* ctx, uint32_t parity, uint32_t world, uint32_t rows, uint32_t n_mlp, void* color_master_slice,
                float* m_slice, float* v_slice, float* mlp_params, float* m_mlp, float* v_mlp, void* wpack,
                void* gtab_next, float* gmlp_next, float* opt_state, float eps, n2m_stream_t stream);

/* NVLS variant: the table gradients are reduced INSIDE the NVSwitch (multimem.ld_reduce on a multicast address that maps the gradient
 * table of every rank) and the refreshed 8-byte entries are broadcast with one multimem.st; mc_gtab / mc_table are the multicast addresses
 * (torch.distributed._symmetric_memory) of this parity's gradient table and of the working table.  Per rank and step the links carry 16 B x rows out
 * (the switch pulls every replica of a row once) against 16 B x rows x (W-1)/W each way with P2P loads, and the all-gather 8 B x rows / W
 * out instead of 8 B x rows x (W-1)/W, so it moves fewer bytes than n2m_dp_adam for W > 4.  In both entry points gtab_next / gmlp_next may be NULL: the caller then zeroes the next-parity gradient buffers itself. */
int n2m_dp_adam_nvls(const void* ctx, const void* mc_gtab, void* mc_table, uint32_t parity, uint32_t world, uint32_t rows, uint32_t n_mlp,
                     void* color_master_slice, float* m_slice, float* v_slice, float* mlp_params, float* m_mlp, float* v_mlp, void* wpack,
                     void* gtab_next, float* gmlp_next, float* opt_state, float eps, n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_FUSED_H */
