// render.cu -- evaluation renderer of the fused stage-0 path with the alive-ray bookkeeping ON THE DEVICE.
//
// Reference: NeRFRenderer.render, inference branch (nerf/renderer.py:749-802): a Python loop that, per round, reads n_alive back to the
// host, picks n_step = max(min(N // n_alive, 8), 1), calls raymarching.march_rays (raymarching.cu:713-828), the model, and
// raymarching.composite_rays (raymarching.cu:842-924), then compacts `rays_alive` with a boolean mask -- hundreds of launches and one
// host synchronisation per round for a 640 000-ray image.
//
// Here a chunk of rays is rendered by ONE host call that enqueues a fixed schedule of rounds without reading anything back:
//   k_r_begin     : near / far (raymarching.cu:92-145, renderer.py:689-691 clamp), zeroed accumulators, first alive list (rays that hit
//                   the volume), warp-aggregated append
//   k_r_plan      : (one thread) next list's length -> n_alive, n_step = min(schedule[round], capacity / n_alive), rows = n_alive * n_step
//                   into the counters block the stage-0 gather / MLP kernels size themselves by, list parity flipped
//   k_r_march     : one thread per alive ray: up to n_step occupied samples from rays_t with the sequential marcher core
//                   (march_core.cuh; the reference's arithmetic), written as march RECORDS {t, dt, t + dt, ray} in slab order
//                   i * n_step + k, zero records behind a ray that ran out -- the same record form the training path uses, so
//   n2m_s0_encode_fwd + n2m_s0_mlp_fwd : the training forward kernels (hash-grid gather into tensor-core tile images, wgmma MLPs)
//                   evaluate the slab unchanged
//   k_r_composite : one thread per alive ray: the reference's slab compositor (transmittance carried through weights_sum, stop at
//                   T < T_thresh or at the zero tail), ray state in the output arrays, survivors appended to the OTHER alive list
// and k_r_finish mixes the background (renderer.py:804).  Every kernel is launched for the chunk's worst case and reads the round's
// actual sizes from the device, so a round in which nothing is alive costs a few empty launches.  The slab widths double
// (8, 8, 16, 16, 32, 64, ...): early rounds are narrow so that rays stop soon after their first surface, late rounds wide because few
// rays are left; the widths are clipped on the device to what the sample slab holds.  The caller checks the remaining alive count
// once per chunk (one read-back) and runs further rounds in the rare case the clipped schedule did not exhaust the rays.
#include "n2m_common.cuh"
#include "march_core.cuh"
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

using namespace march;

// control block (int32[16]); [0..2] are the counters the stage-0 forward kernels read (whole-batch mode reads [1] only)
enum : int { kRows = 1, kAlive = 8, kStep = 9, kAppend = 10, kParity = 11, kRounds = 12, kRowsTotal = 13 };

__device__ __forceinline__ void append_alive(bool keep, int ray, int32_t* __restrict__ list, int32_t* __restrict__ counter) {
    const uint32_t mask = __ballot_sync(0xffffffffu, keep);
    if (mask == 0) return;
    const uint32_t lane = threadIdx.x & 31;
    const int leader = __ffs(mask) - 1;
    int base = 0;
    if ((int)lane == leader) base = atomicAdd(counter, (int)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (keep) list[base + __popc(mask & ((1u << lane) - 1u))] = ray;
}

__global__ void __launch_bounds__(256)
k_r_begin(n2m_s0_params p, const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ aabb,
          const float* __restrict__ cam_nf, uint32_t N, float* __restrict__ rays_t, float* __restrict__ rays_far,
          int32_t* __restrict__ alive, int32_t* __restrict__ ctl, float* __restrict__ weights_sum, float* __restrict__ depth,
          float* __restrict__ image) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (n < N) {
        float near, far;
        near_far_aabb(rays_o + 3 * n, rays_d + 3 * n, aabb, p.min_near, near, far);
        if (cam_nf) { near = fmaxf(near, cam_nf[2 * n]); far = fminf(far, cam_nf[2 * n + 1]); }
        rays_t[n] = near; rays_far[n] = far;
        weights_sum[n] = 0.f; depth[n] = 0.f;
        image[3 * n] = 0.f; image[3 * n + 1] = 0.f; image[3 * n + 2] = 0.f;
        hit = near < far;
    }
    // the first list goes where the compositor would have left it: the half the first k_r_plan flips TO (parity 0 -> 1)
    append_alive(hit, (int)n, alive + N, ctl + kAppend);
}

__global__ void k_r_plan(int32_t* __restrict__ ctl, uint32_t n_step, uint32_t Mcap) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const uint32_t n_alive = (uint32_t)ctl[kAppend];
    uint32_t step = n_step;
    if (n_alive > 0 && (unsigned long long)n_alive * step > Mcap) step = max(1u, Mcap / n_alive);
    ctl[kAlive] = (int32_t)n_alive;
    ctl[kStep] = (int32_t)step;
    ctl[kAppend] = 0;
    ctl[kParity] ^= 1;
    const unsigned long long rows = (unsigned long long)n_alive * step;
    ctl[0] = (int32_t)min(rows, (unsigned long long)0x7fffffff);
    ctl[kRows] = (int32_t)min(rows, (unsigned long long)Mcap);
    ctl[2] = rows > Mcap ? 1 : 0;                    // only if Mcap < n_alive (the host allocates Mcap >= chunk rays)
    ctl[kRounds] += 1;
    ctl[kRowsTotal] = (int32_t)min((unsigned long long)ctl[kRowsTotal] + min(rows, (unsigned long long)Mcap), (unsigned long long)0x7fffffff);
}

struct RecSink {
    float4* recs; int ray;
    __device__ __forceinline__ void put(uint32_t k, float t_before, float t_after, float dt, const Probe&, float, float, float) const {
        recs[k] = make_float4(t_before, dt, t_after, __int_as_float(ray));
    }
};

__global__ void __launch_bounds__(128)
k_r_march(n2m_s0_params p, const float* __restrict__ rays_o, const float* __restrict__ rays_d, const uint8_t* __restrict__ bits,
          const float* __restrict__ rays_t, const float* __restrict__ rays_far, const int32_t* __restrict__ alive, uint32_t N,
          const int32_t* __restrict__ ctl, float4* __restrict__ recs) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_alive = (uint32_t)ctl[kAlive], n_step = (uint32_t)ctl[kStep];
    if (i >= n_alive || (unsigned long long)(i + 1) * n_step > (unsigned long long)(uint32_t)ctl[kRows]) return;
    const int ray = alive[(size_t)ctl[kParity] * N + i];
    const MarchCfg c = make_cfg(p.bound, p.contract != 0, p.dt_gamma, p.max_steps, p.cascades, p.grid_size, bits);
    const float ox = rays_o[3 * ray], oy = rays_o[3 * ray + 1], oz = rays_o[3 * ray + 2];
    const float dx = rays_d[3 * ray], dy = rays_d[3 * ray + 1], dz = rays_d[3 * ray + 2];
    float4* slab = recs + (size_t)i * n_step;
    // reciprocal directions as the reference's INFERENCE marcher forms them (raymarching.cu:744; its training kernel divides by d itself)
    const uint32_t got = march_one(c, rays_t[ray], rays_far[ray], n_step, ox, oy, oz, dx, dy, dz, 1 / (dx + 1e-10f), 1 / (dy + 1e-10f), 1 / (dz + 1e-10f),
                                   RecSink{slab, ray});
    for (uint32_t k = got; k < n_step; ++k) slab[k] = make_float4(0.f, 0.f, 0.f, __int_as_float(ray));     // the ray ran out: zero tail
}

// raymarching.cu:842-924 on the records / the MLP output rows (sigma, r, g, b) of this round's slab
__global__ void __launch_bounds__(128)
k_r_composite(n2m_s0_params p, const float4* __restrict__ out, const float4* __restrict__ recs, int32_t* __restrict__ ctl,
              int32_t* __restrict__ alive, uint32_t N, float* __restrict__ rays_t, float* __restrict__ weights_sum,
              float* __restrict__ depth, float* __restrict__ image) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_alive = (uint32_t)ctl[kAlive], n_step = (uint32_t)ctl[kStep];
    const uint32_t parity = (uint32_t)ctl[kParity];
    bool keep = false;
    int ray = 0;
    if (i < n_alive && (unsigned long long)(i + 1) * n_step <= (unsigned long long)(uint32_t)ctl[kRows]) {
        ray = alive[(size_t)parity * N + i];
        const size_t base = (size_t)i * n_step;
        float t = 0.f;
        float d = depth[ray], r = image[3 * ray], g = image[3 * ray + 1], b = image[3 * ray + 2], wsum = weights_sum[ray];
        uint32_t k = 0;
        for (; k < n_step; ++k) {
            const float4 rec = recs[base + k];
            if (rec.z == 0.f) break;                      // zero tail: the ray ran out (raymarching.cu:877)
            const float4 o = out[base + k];
            const float alpha = 1.0f - __expf(-o.x * rec.y);
            const float T = 1.f - wsum;
            const float w = alpha * T;
            wsum += w;
            t = rec.z;
            d += w * t;
            r += w * o.y; g += w * o.z; b += w * o.w;
            if (T < p.T_thresh) break;                    // tested after accumulating, as in the reference (:905-906)
        }
        keep = k == n_step;
        if (keep) rays_t[ray] = t;
        weights_sum[ray] = wsum; depth[ray] = d;
        image[3 * ray] = r; image[3 * ray + 1] = g; image[3 * ray + 2] = b;
    }
    append_alive(keep, ray, alive + (size_t)(parity ^ 1u) * N, ctl + kAppend);
}

__global__ void __launch_bounds__(256)
k_r_finish(float* __restrict__ image, const float* __restrict__ weights_sum, const float* __restrict__ bg, float bg_scalar, uint32_t N) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float T = 1.f - weights_sum[n];
#pragma unroll
    for (int c = 0; c < 3; ++c) image[3 * n + c] += T * (bg ? bg[3 * n + c] : bg_scalar);             // renderer.py:804
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_s0_render_rounds(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const uint8_t* bitfield, uint32_t N,
                         const uint32_t* schedule, uint32_t num_rounds, float* rays_t, float* rays_far, int32_t* alive, int32_t* ctl,
                         void* recs, void* enc_tiles, void* out, uint32_t Mcap, const void* table, const int32_t* offsets, const void* wpack,
                         float* weights_sum, float* depth, float* image, n2m_stream_t stream) {
    return n2m_s0_render_rounds_codes(p, rays_o, rays_d, bitfield, N, schedule, num_rounds, rays_t, rays_far, alive, ctl, recs, enc_tiles,
                                      out, Mcap, table, offsets, wpack, nullptr, weights_sum, depth, image, stream);
}

int n2m_s0_render_rounds_codes(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const uint8_t* bitfield, uint32_t N,
                               const uint32_t* schedule, uint32_t num_rounds, float* rays_t, float* rays_far, int32_t* alive, int32_t* ctl,
                               void* recs, void* enc_tiles, void* out, uint32_t Mcap, const void* table, const int32_t* offsets,
                               const void* wpack, const float* code_row, float* weights_sum, float* depth, float* image,
                               n2m_stream_t stream) {
    N2M_REQUIRE(p && (p->ind_dim == 0 || code_row), "s0_render_rounds", "ind_dim > 0 needs a code row");
    N2M_REQUIRE(p && rays_o && rays_d && bitfield && schedule && rays_t && rays_far && alive && ctl && recs && enc_tiles && out && table &&
                offsets && wpack && weights_sum && depth && image, "s0_render_rounds", "null pointer");
    N2M_REQUIRE(Mcap % 128 == 0 && Mcap >= N && N > 0, "s0_render_rounds", "Mcap must be a multiple of 128 and >= the chunk's rays");
    cudaStream_t st = as_stream(stream);
    for (uint32_t r = 0; r < num_rounds; ++r) {
        N2M_REQUIRE(schedule[r] >= 1, "s0_render_rounds", "slab widths must be >= 1");
        k_r_plan<<<1, 32, 0, st>>>(ctl, schedule[r], Mcap);
        if (int e = check_launch("s0_render(plan)")) return e;
        k_r_march<<<div_up(N, 128u), 128, 0, st>>>(*p, rays_o, rays_d, bitfield, rays_t, rays_far, alive, N, ctl, static_cast<float4*>(recs));
        if (int e = check_launch("s0_render(march)")) return e;
        if (int e = code_row ? n2m_s0_encode_fwd_codes(p, recs, ctl, Mcap, rays_o, rays_d, table, offsets, code_row, nullptr, enc_tiles, 0, 1,
                                                       stream)
                             : n2m_s0_encode_fwd(p, recs, ctl, Mcap, rays_o, rays_d, table, offsets, enc_tiles, 0, 1, stream))
            return e;
        if (int e = n2m_s0_mlp_fwd(p, enc_tiles, ctl, Mcap, wpack, out, nullptr, 0, 1, stream)) return e;
        k_r_composite<<<div_up(N, 128u), 128, 0, st>>>(*p, static_cast<const float4*>(out), static_cast<const float4*>(recs), ctl, alive, N,
                                                      rays_t, weights_sum, depth, image);
        if (int e = check_launch("s0_render(composite)")) return e;
    }
    // ctl[10] now holds the number of rays still alive (the caller's one read-back); the lists are ready for further rounds
    return 0;
}

int n2m_s0_render_begin(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const float* aabb, const float* cam_near_far,
                        uint32_t N, float* rays_t, float* rays_far, int32_t* alive, int32_t* ctl, float* weights_sum, float* depth,
                        float* image, n2m_stream_t stream) {
    N2M_REQUIRE(p && rays_o && rays_d && aabb && rays_t && rays_far && alive && ctl && weights_sum && depth && image, "s0_render_begin",
                "null pointer");
    N2M_REQUIRE(N > 0, "s0_render_begin", "no rays");
    cudaStream_t st = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(ctl, 0, 16 * sizeof(int32_t), st);
    if (e != cudaSuccess) return fail("s0_render_begin(memset)", cudaGetErrorString(e));
    k_r_begin<<<div_up(N, 256u), 256, 0, st>>>(*p, rays_o, rays_d, aabb, cam_near_far, N, rays_t, rays_far, alive, ctl, weights_sum, depth, image);
    return check_launch("s0_render_begin");
}

/* image += (1 - weights_sum) * bg (renderer.py:804); bg [N,3] or NULL (then bg_scalar) */
int n2m_s0_render_finish(float* image, const float* weights_sum, const float* bg, float bg_scalar, uint32_t N, n2m_stream_t stream) {
    N2M_REQUIRE(image && weights_sum, "s0_render_finish", "null pointer");
    if (N == 0) return 0;
    k_r_finish<<<div_up(N, 256u), 256, 0, as_stream(stream)>>>(image, weights_sum, bg, bg_scalar, N);
    return check_launch("s0_render_finish");
}

}  // extern "C"
