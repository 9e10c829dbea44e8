/* n2m_b200.h -- C ABI of libn2m_b200.so: the sm_90a (H100) replacement for the
 * native layer of nerf2mesh's stage-0 hot path.
 *
 * Every entry point replaces one function the reference binds through pybind11
 * (reference file:line given per function).  Conventions:
 *   - plain device pointers + explicit sizes, no torch types;
 *   - the CALLER allocates every output (and zero-initialises the ones marked [zero-init]);
 *     the library never allocates, frees or retains device memory and holds no state
 *     between calls except a thread-local error string;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - nullable pointers stand in for the reference's at::optional<Tensor>;
 *   - return 0 on success, non-zero on error; n2m_last_error() returns the message
 *     (the Python layer raises RuntimeError with it, mirroring TORCH_CHECK behaviour
 *     at gridencoder.cu:448-464).  Unlike the reference every launch is followed by
 *     cudaGetLastError().
 */
#ifndef N2M_B200_H
#define N2M_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* n2m_stream_t;

/* library info / errors */
const char* n2m_last_error(void);
int n2m_version(void);
/* number of kernel launches issued by this library in this process since load
 * (bench.py's gpu_launches evidence) */
uint64_t n2m_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * raymarching  (reference: raymarching/src/raymarching.h:7-19, bindings.cpp:5-19)
 * ---------------------------------------------------------------------------------------- */

/* raymarching.cu:148 near_far_from_aabb.  rays_o/d [N,3], aabb [6], nears/fars [N]. */
int n2m_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb,
                           uint32_t N, float min_near, float* nears, float* fars,
                           n2m_stream_t stream);

/* raymarching.cu:201 sph_from_ray.  coords [N,2]. */
int n2m_sph_from_ray(const float* rays_o, const float* rays_d, float radius, uint32_t N,
                     float* coords, n2m_stream_t stream);

/* raymarching.cu:229 morton3D / :257 morton3D_invert.  coords int32 [N,3], indices int32 [N]. */
int n2m_morton3D(const int32_t* coords, uint32_t N, int32_t* indices, n2m_stream_t stream);
int n2m_morton3D_invert(const int32_t* indices, uint32_t N, int32_t* coords, n2m_stream_t stream);

/* raymarching.cu:292 packbits.  grid float [8*N], bitfield u8 [N]; bit i of byte n = grid[8n+i] > thresh. */
int n2m_packbits(const float* grid, uint32_t N, float density_thresh, uint8_t* bitfield,
                 n2m_stream_t stream);

/* raymarching.cu:321 flatten_rays.  rays int32 [N,2] (offset,count) -> res int32 [M] (ray id per sample). */
int n2m_flatten_rays(const int32_t* rays, uint32_t N, uint32_t M, int32_t* res, n2m_stream_t stream);

/* raymarching.cu:477 march_rays_train.  Same two-call protocol as the reference wrapper
 * (raymarching.py:229-241):
 *   call 1: xyzs == NULL  -> counting pass: writes rays[n] = (offset, count) and counter[0] = M.
 *           Unlike the reference (atomicAdd order, raymarching.cu:471) offsets are the exclusive
 *           prefix sum of the counts in ray order, i.e. deterministic.
 *           `tbuf` (float [N * max_steps * 2], caller scratch, may be NULL) receives each ray's
 *           (t_before_step, dt) pairs so that call 2 need not re-march.
 *   call 2: xyzs/dirs/ts != NULL -> writes xyzs [M,3], dirs [M,3], ts [M,2] at rays[n].offset.
 *           With tbuf != NULL samples are regenerated in parallel (one warp per ray); with
 *           tbuf == NULL the ray is re-marched sequentially as in the reference.
 * grid = density bitfield u8 [C*H^3/8]; nears/fars/noises [N]. */
int n2m_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* grid,
                         float bound, int contract, float dt_gamma, uint32_t max_steps,
                         uint32_t N, uint32_t C, uint32_t H,
                         const float* nears, const float* fars,
                         float* xyzs, float* dirs, float* ts,
                         int32_t* rays, int32_t* counter, const float* noises,
                         float* tbuf, n2m_stream_t stream);

/* raymarching.cu:581 composite_rays_train_forward.  weights [M] [zero-init]; weights_sum/depth [N], image [N,3]. */
int n2m_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* ts,
                                     const int32_t* rays, uint32_t M, uint32_t N, float T_thresh,
                                     int alpha_mode, float* weights, float* weights_sum,
                                     float* depth, float* image, n2m_stream_t stream);

/* raymarching.cu:697 composite_rays_train_backward.  grad_sigmas [M], grad_rgbs [M,3] [zero-init]. */
int n2m_composite_rays_train_backward(const float* grad_weights, const float* grad_weights_sum,
                                      const float* grad_depth, const float* grad_image,
                                      const float* sigmas, const float* rgbs, const float* ts,
                                      const int32_t* rays, const float* weights_sum,
                                      const float* depth, const float* image,
                                      uint32_t M, uint32_t N, float T_thresh, int alpha_mode,
                                      float* grad_sigmas, float* grad_rgbs, n2m_stream_t stream);

/* raymarching.cu:831 march_rays (inference).  xyzs/dirs [n_alive*n_step,3], ts [n_alive*n_step,2] [zero-init]. */
int n2m_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t* rays_alive, const float* rays_t,
                   const float* rays_o, const float* rays_d, float bound, int contract,
                   float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H, const uint8_t* grid,
                   const float* nears, const float* fars, float* xyzs, float* dirs, float* ts,
                   const float* noises, n2m_stream_t stream);

/* raymarching.cu:927 composite_rays (inference, in place on weights_sum/depth/image; rays_alive[n] = -1 on termination). */
int n2m_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int alpha_mode,
                       int32_t* rays_alive, float* rays_t, const float* sigmas, const float* rgbs,
                       const float* ts, float* weights_sum, float* depth, float* image,
                       n2m_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * gridencoder  (reference: gridencoder/src/gridencoder.h:12-15, bindings.cpp:5-8)
 * dtype: 0 = float32 table/outputs, 1 = float16 table/outputs (inputs are always float32,
 * gridencoder.cu:468).  gridtype: 0 hash, 1 tiled.  interp: 0 linear, 1 smoothstep.
 * ---------------------------------------------------------------------------------------- */

/* gridencoder.cu:447 grid_encode_forward.  inputs [B,D] in [0,1]; embeddings [rows,C]; offsets int32 [L+1];
 * outputs [L,B,C] (level-major, as the reference kernel writes it); dy_dx [B,L*D*C] or NULL. */
int n2m_grid_encode_forward(const float* inputs, const void* embeddings, const int32_t* offsets,
                            void* outputs, uint32_t B, uint32_t D, uint32_t C, uint32_t L,
                            uint32_t max_level, float S, uint32_t H, void* dy_dx,
                            uint32_t gridtype, int align_corners, uint32_t interp, int dtype,
                            n2m_stream_t stream);

/* gridencoder.cu:472 grid_encode_backward.  grad [L,B,C]; grad_embeddings [rows,C] [zero-init];
 * dy_dx/grad_inputs nullable ([B,L*D*C] / [B,D] in the table dtype). */
int n2m_grid_encode_backward(const void* grad, const float* inputs, const void* embeddings,
                             const int32_t* offsets, void* grad_embeddings, uint32_t B, uint32_t D,
                             uint32_t C, uint32_t L, uint32_t max_level, float S, uint32_t H,
                             const void* dy_dx, void* grad_inputs, uint32_t gridtype,
                             int align_corners, uint32_t interp, int dtype, n2m_stream_t stream);

/* gridencoder.cu:638 grad_total_variation (fp32 only; the reference forces autocast off, grid.py:171).
 * Adds the TV gradient into `grad` [rows,C] in place. */
int n2m_grad_total_variation(const float* inputs, const float* embeddings, float* grad,
                             const int32_t* offsets, float weight, uint32_t B, uint32_t D, uint32_t C,
                             uint32_t L, float S, uint32_t H, uint32_t gridtype, int align_corners,
                             n2m_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * shencoder  (reference: shencoder/src/shencoder.h:9-10, bindings.cpp:5-7)
 * ---------------------------------------------------------------------------------------- */

/* shencoder.cu:400 sh_encode_forward.  inputs [B,3]; outputs [B,degree^2]; dy_dx [B,3*degree^2] or NULL. */
int n2m_sh_encode_forward(const float* inputs, float* outputs, uint32_t B, uint32_t D, uint32_t degree,
                          float* dy_dx, n2m_stream_t stream);

/* shencoder.cu:419 sh_encode_backward.  grad [B,degree^2]; grad_inputs [B,3] (accumulated into, so [zero-init]). */
int n2m_sh_encode_backward(const float* grad, const float* inputs, uint32_t B, uint32_t D, uint32_t degree,
                           const float* dy_dx, float* grad_inputs, n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_H */
