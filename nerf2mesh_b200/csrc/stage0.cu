// stage0.cu -- fused stage-0 train path, the non-tensor-core stages (see include/n2m_b200_fused.h):
//   march (near/far + count + scan + sample records), hash-grid encode forward into tensor-core
//   tile images, composite + loss + composite-backward per ray, hash-grid scatter (+TV) backward,
//   table (de)interleave helpers.  The MLP stages live in mlp_tc.cu, the optimizer in optim.cu.
//   The scatter and the TV pass walk the hash grid level group by level group rather than sample by sample: their RED target,
//   the 97.6 MB gradient table, is twice the H100's L2, one group's slice of it fits (see "Level-group walk" below).
#include "march_core.cuh"
#include "s0_geom.cuh"
#include <cstdlib>
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

using namespace march;

// ------------------------------------------------------------------------------------------------
// march
// ------------------------------------------------------------------------------------------------
// Adaptive ray count (--adaptive_num_rays): a batch is the first n rays of the N-row buffers.  The march takes n from the control
// block's ray_ctl[0] (left there by the previous march's scan), the composite from counters[16]; rays >= n march no sample and are
// never read.  Without a count n = N.
__device__ __forceinline__ uint32_t ray_count(const int32_t* __restrict__ count, uint32_t N) {
    return count ? min((uint32_t)max(*count, 1), N) : N;
}

template <bool ADAPTIVE>
__global__ void __launch_bounds__(128)
k_s0_count(const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ aabb,
           const float* __restrict__ cam_nf, const uint8_t* __restrict__ bits, const float* __restrict__ noises,
           n2m_s0_params p, uint32_t N, const int32_t* __restrict__ ray_ctl, int32_t* __restrict__ rays, float2* __restrict__ tbuf) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    if (ADAPTIVE && n >= ray_count(ray_ctl, N)) { rays[2 * n + 1] = 0; return; }
    const MarchCfg c = make_cfg(p.bound, p.contract != 0, p.dt_gamma, p.max_steps, p.cascades, p.grid_size, bits);
    float near, far;
    near_far_aabb(rays_o + 3 * n, rays_d + 3 * n, aabb, p.min_near, near, far);
    if (cam_nf) {                      // renderer.py:689-691
        near = fmaxf(near, cam_nf[2 * n]);
        far = fminf(far, cam_nf[2 * n + 1]);
    }
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
    const float rdx = 1 / dx, rdy = 1 / dy, rdz = 1 / dz;
    float t0 = near;
    t0 += clampf(t0 * c.dt_gamma, c.dt_min, c.dt_max) * noises[n];
    CountSink sink{tbuf + (size_t)n * p.max_steps};
    const uint32_t cnt = march_one(c, t0, far, p.max_steps, ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, sink);
    rays[2 * n + 1] = (int32_t)cnt;
}

// Warp-per-ray marcher.  The sequential marcher's t only ever advances by dt(t) = clamp(t * dt_gamma,
// dt_min, dt_max) -- in the "emit" branch and in every hop of the "skip" branch alike -- so every t it visits
// belongs to the one-parameter sequence tau_0 = t0, tau_{j+1} = tau_j + dt(tau_j).  The warp generates 32
// consecutive tau's (serial fp32 adds, identical rounding), probes all 32 positions in parallel (cell,
// cascade, occupancy bit, voxel-exit time: the expensive part), and then replays the sequential control flow
// over the precomputed probes with ballots: runs of occupied samples are consumed in one go, an empty probe
// jumps to the first tau that is not < its exit time.  Same visited set, same (t, dt) per sample, bit for bit.
template <bool ADAPTIVE>
__global__ void __launch_bounds__(128)
k_s0_count_warp(const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ aabb,
                const float* __restrict__ cam_nf, const uint8_t* __restrict__ bits, const float* __restrict__ noises,
                n2m_s0_params p, uint32_t N, const int32_t* __restrict__ ray_ctl, int32_t* __restrict__ rays,
                float2* __restrict__ tbuf) {
    const uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (n >= N) return;
    if (ADAPTIVE && n >= ray_count(ray_ctl, N)) { if (lane == 0) rays[2 * n + 1] = 0; return; }
    const MarchCfg c = make_cfg(p.bound, p.contract != 0, p.dt_gamma, p.max_steps, p.cascades, p.grid_size, bits);
    float near, far;
    near_far_aabb(rays_o + 3 * n, rays_d + 3 * n, aabb, p.min_near, near, far);
    if (cam_nf) {
        near = fmaxf(near, cam_nf[2 * n]);
        far = fminf(far, cam_nf[2 * n + 1]);
    }
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
    const float rdx = 1 / dx, rdy = 1 / dy, rdz = 1 / dz;
    float t_start = near;
    t_start += clampf(t_start * c.dt_gamma, c.dt_min, c.dt_max) * noises[n];
    float2* slab = tbuf + (size_t)n * p.max_steps;

    uint32_t step = 0;
    bool pending = false;          // a hop whose target lies beyond the chunk it started in
    float pending_tt = 0.f;
    bool done = !(t_start < far);
    uint32_t chunks = 0;
    while (!done && ++chunks < (1u << 20)) {       // the cap only guards against a t that cannot advance
        // tau for this lane: `lane` serial steps from the chunk start (all lanes run the loop in lock step)
        float tau = t_start;
        float t_next = t_start;    // value after 32 steps = next chunk start
        if (c.dt_gamma == 0.f) {
            // dt(t) = clamp(t * 0, dt_min, dt_max) is the same constant for every t (also inf/NaN: fmaxf drops
            // the NaN), so the chain is 32 dependent FADDs
            const float dt0 = clampf(0.f, c.dt_min, c.dt_max);
#pragma unroll
            for (uint32_t i = 0; i < 32; ++i) {
                const float adv = t_next + dt0;
                if (i < lane) tau = adv;
                t_next = adv;
            }
        } else {
#pragma unroll 1
            for (uint32_t i = 0; i < 32; ++i) {
                const float adv = t_next + clampf(t_next * c.dt_gamma, c.dt_min, c.dt_max);
                if (i < lane) tau = adv;
                t_next = adv;
            }
        }
        const float dt = clampf(tau * c.dt_gamma, c.dt_min, c.dt_max);
        const bool in_range = tau < far;
        bool emit = false;
        float tt = 0.f;
        if (in_range) {
            const Probe pr = probe_at(c, tau, ox, oy, oz, dx, dy, dz);
            emit = pr.emit;
            if (!emit) tt = exit_time(c, pr, tau, dx, dy, dz, rdx, rdy, rdz);
        }
        const uint32_t range_mask = __ballot_sync(0xffffffffu, in_range);     // a prefix of the warp (tau increases)
        const uint32_t emit_mask = __ballot_sync(0xffffffffu, emit);
        uint32_t cur = 0;
        if (pending) {
            const uint32_t ge = __ballot_sync(0xffffffffu, !(tau < pending_tt));
            if (ge == 0) cur = 32; else { cur = __ffs(ge) - 1; pending = false; }
        }
        while (cur < 32) {
            if (!((range_mask >> cur) & 1u) || step >= p.max_steps) { done = true; break; }
            if ((emit_mask >> cur) & 1u) {
                // run of consecutive occupied probes starting at `cur`
                const uint32_t run_bits = ~(emit_mask >> cur);
                uint32_t run = run_bits ? (uint32_t)(__ffs(run_bits) - 1) : 32u;
                run = min(run, 32u - cur);
                run = min(run, p.max_steps - step);
                if (lane >= cur && lane < cur + run) slab[step + (lane - cur)] = make_float2(tau, dt);
                step += run;
                cur += run;
            } else {
                const float tt_c = __shfl_sync(0xffffffffu, tt, cur);
                uint32_t ge = __ballot_sync(0xffffffffu, !(tau < tt_c));
                ge &= (cur >= 31) ? 0u : (0xffffffffu << (cur + 1));             // at least one dt step is taken
                if (ge == 0) { pending = true; pending_tt = tt_c; cur = 32; }
                else cur = __ffs(ge) - 1;
            }
        }
        t_start = __shfl_sync(0xffffffffu, t_next, 31);
        if (!done && !(t_start < far) ) {
            // the next chunk starts beyond `far`: nothing left to visit (a pending hop lands past far too)
            done = true;
        }
    }
    if (lane == 0) rays[2 * n + 1] = (int32_t)step;
}

// single-block exclusive scan (N is a few thousand rays) -> offsets + counters
// With a control block (adaptive ray count) it also records this batch's n in counters[16] and leaves the next march's count in
// ray_ctl[0]: the reference's rule, utils.py:795-797, num_rays = int(round((num_points / M) * num_rays)), in float64 and in that order
// (rint rounds half to even as round() does), M unclamped by Mcap as the reference never caps it, clamped to [1, N].  Steps clamped at N
// are counted in ray_ctl[1], the largest count asked for before the clamp is kept in ray_ctl[2].  A batch with M == 0 keeps n, where the
// reference would divide by zero.
__global__ void __launch_bounds__(1024)
k_s0_scan(int32_t* __restrict__ rays, uint32_t N, uint32_t Mcap, int32_t* __restrict__ counters, int32_t* __restrict__ ray_ctl,
          uint32_t num_points) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s, n_s;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry_s = 0; n_s = ray_count(ray_ctl, N); }       // read before thread 0 rewrites ray_ctl[0] below
    __syncthreads();
    const uint32_t n_act = n_s;
    for (uint32_t base = 0; base < N; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < N ? (uint32_t)rays[2 * i + 1] : 0u;
        uint32_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += u;
        }
        if (lane == 31) warp_tot[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = warp_tot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += u;
            }
            warp_tot[lane] = w;
        }
        __syncthreads();
        const uint32_t carry = carry_s;
        if (i < N) rays[2 * i] = (int32_t)(carry + (wid ? warp_tot[wid - 1] : 0u) + inc - v);
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    const uint32_t M = carry_s;
    if (threadIdx.x == 0) {
        counters[0] = (int32_t)M;
        counters[1] = (int32_t)min(M, Mcap);
        counters[2] = M > Mcap ? 1 : 0;
        counters[3] = 0;                 // samples inside the unit cube   } counted by this step's n2m_s0_tv (k_s0_encode_bwd<false, true>),
        counters[15] = 0;                // samples outside the unit cube  } read by k_s0_tv_random (grid.py:181-183 fallback)
        // persistent capacity accounting (never reset by the march): steps that overflowed the sample slab, largest M seen
        if (M > Mcap) counters[13] += 1;
        counters[14] = max(counters[14], (int32_t)M);
        if (ray_ctl) {
            counters[16] = (int32_t)n_act;
            uint32_t next = n_act;
            if (M > 0) {
                const double want = rint(__dmul_rn(__ddiv_rn((double)num_points, (double)M), (double)n_act));
                if (want > (double)N) ray_ctl[1] += 1;
                ray_ctl[2] = max(ray_ctl[2], (int32_t)fmin(want, 2147483647.0));
                next = (uint32_t)fmin(fmax(want, 1.0), (double)N);
            }
            ray_ctl[0] = (int32_t)next;
        }
    }
    // part boundaries (n2m_common.cuh part_range): sample offset of the first active ray of every eighth of the batch
    if (threadIdx.x <= kPartSlots) {
        const uint32_t e = threadIdx.x;
        const uint32_t first = part_first_ray(n_act, e);
        const uint32_t off = (e == kPartSlots || first >= n_act) ? M : (uint32_t)rays[2 * first];
        counters[4 + e] = (int32_t)min(min(off, M), Mcap);
    }
}

// one warp per ray: sample records {t_before, dt, t_after, ray}
__global__ void __launch_bounds__(256)
k_s0_records(const int32_t* __restrict__ rays, const float2* __restrict__ tbuf, uint32_t N, uint32_t max_steps,
             uint32_t Mcap, float4* __restrict__ recs) {
    const uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (n >= N) return;
    const uint32_t off = (uint32_t)rays[2 * n], cnt = (uint32_t)rays[2 * n + 1];
    const float2* slab = tbuf + (size_t)n * max_steps;
    for (uint32_t k = lane; k < cnt; k += 32) {
        const uint32_t j = off + k;
        if (j >= Mcap) break;
        const float2 td = slab[k];
        recs[j] = make_float4(td.x, td.y, td.x + td.y, __int_as_float((int)n));
    }
}

// ------------------------------------------------------------------------------------------------
// encode forward: one block = one 128-sample tile image.
// ------------------------------------------------------------------------------------------------
// POINTS = false: samples come from the march records (training / eval rendering);
// POINTS = true : explicit positions xyz [P,3] (rays_o) and optional directions [P,3] (rays_d) -- used for the
//                 density-grid update (renderer.py:1112-1113 evaluates self.density on cell centres), stage 1 and tests.
// (The TV gradient is not evaluated here although 4 of its 7 stencil values are in registers: it slows this kernel by more than a
// separate TV launch costs, and that launch hides under the MLP kernels.)
//
// Where the time goes (profiles/gather_time.py, H100 80GB HBM3 at 700 W, bench.py's batches).  Lego (M = 285,107): the whole
// batch takes 114 us with a warm L2 and 124 us with a cold one, a part 70-72 us warm and 78-84 us cold; garden (M = 823,460):
// 284 / 294 us.  The batch touches 1.19 M sectors (38 MB) of the table, but its warp loads request 17.3 M sectors (554 MB) from L2,
// every corner of a hashed level a sector of its own: 4.9 TB/s at 114 us, more than HBM could deliver.  So the table sectors come
// from L2, and the 10 us between cold and warm is all an L2-resident table could save.  What follows from it, measured the same way:
//  * A level-group walk like the scatter's, writing each level's three fp16 features to per-level planes (1 KiB per tile and level,
//    whole sectors) and then building each tile image from its 16 planes in place, gave bit-identical images but 134 us for the
//    lego batch, 87-103 us per part, a 1.16 ms step timeline instead of 1.03 ms and 7 % fewer samples/s in bench.py.  The walk
//    leaves the sector requests as they were, already served by L2, and adds a re-read of the records per group and the planes.
//  * Issuing the 8 loads of level l + 1 before the sums of level l (two levels in flight): 110 us on lego, 250 us on garden, same
//    bits, but the step is no faster (lego 285.8-286.0 M samples/s against 286.0-288.3, garden 371.2-371.8 against 372.1-373.4).
//    In the step the gathers share the device with TV (half of it) and with each other: part 0's gather ended 44 us earlier, but its
//    k_mlp_fwd started 13 us later, queued behind part 1's gather for SM slots, and TV ended 16 us later.
//  * One 16 B load for the two x-neighbour corners whenever their rows form an aligned pair: 132 us on lego.
template <bool POINTS>
__device__ __forceinline__ void
encode_fwd_tile(const n2m_s0_params& p, const float4* __restrict__ recs,
                const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                const TableEntry* __restrict__ table, const int32_t* __restrict__ offsets,
                uint8_t* __restrict__ enc_tiles, const PartRange pr, uint32_t nparts, uint32_t tile,
                const float* __restrict__ codes, const int32_t* __restrict__ ray_img) {
    float feat[kTileCols];
    const bool own = encode_fwd_features<POINTS>(p, recs, rays_o, rays_d, table, offsets, pr, tile * kTile + threadIdx.x, feat, codes,
                                                 ray_img);
    if (nparts > 1 && !own) return;                  // (whole-batch mode also zero-fills the rows past M of the last tile)
    store_tile_row(enc_tiles + (size_t)tile * kTileBytes, threadIdx.x, feat);
}

// one block per 128-sample tile of the part's range [lo, hi) (grid-stride, so any grid size is correct: the host sizes
// the grid for the expected share of the part and the loop covers an unbalanced one).  CODES = false compiles the code columns out
// (the kernel without appearance codes is the one it was before they existed).
template <bool POINTS, bool CODES>
__global__ void __launch_bounds__(kTile, 6)
k_s0_encode_fwd(n2m_s0_params p, const float4* __restrict__ recs, const int32_t* __restrict__ counters,
                const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                const TableEntry* __restrict__ table, const int32_t* __restrict__ offsets,
                uint8_t* __restrict__ enc_tiles, uint32_t part, uint32_t nparts, const float* __restrict__ codes,
                const int32_t* __restrict__ ray_img) {
    const PartRange pr = part_range(counters, part, nparts);
    if (pr.hi <= pr.lo) return;
    const uint32_t t1 = (pr.hi + kTile - 1) / kTile;
#pragma unroll 1
    for (uint32_t tile = pr.lo / kTile + blockIdx.x; tile < t1; tile += gridDim.x)
        encode_fwd_tile<POINTS>(p, recs, rays_o, rays_d, table, offsets, enc_tiles, pr, nparts, tile, CODES ? codes : nullptr,
                                CODES ? ray_img : nullptr);
}

// ------------------------------------------------------------------------------------------------
// appearance-code gradient (n2m_s0_code_grad): one warp per ray.  The ray's samples are contiguous rows of denc_tiles; every lane sums
// the code columns of every 32nd sample in fp32, the warp reduces, lane j < D issues the ray's one RED for dimension j.  Samples of a
// ray share its image, so the REDs are per ray and not per sample: with random_image_batch 4096 rays fall on ~100 code rows.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_s0_code_grad(uint32_t D, const int32_t* __restrict__ rays, const int32_t* __restrict__ counters, uint32_t N,
               const uint8_t* __restrict__ denc_tiles, const int32_t* __restrict__ ray_img, float* __restrict__ g_codes,
               float* __restrict__ opt_state, const int32_t* __restrict__ active_rays, uint32_t e0, uint32_t e1) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_act = ray_count(active_rays, N);
    const uint32_t ray_lo = part_first_ray(n_act, e0), ray_hi = part_first_ray(n_act, e1);
    const uint32_t M = (uint32_t)counters[1];                 // rows past the sample capacity hold no sample
    bool bad = false;
    for (uint32_t n = ray_lo + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5); n < ray_hi; n += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t off = (uint32_t)rays[2 * n], end = min(off + (uint32_t)rays[2 * n + 1], M);
        float acc[kMaxIndDim];
#pragma unroll
        for (uint32_t k = 0; k < kMaxIndDim; ++k) acc[k] = 0.f;
        for (uint32_t j = off + lane; j < end; j += 32) {
            const uint8_t* row = denc_tiles + (size_t)(j / kTile) * kTileBytes + (j % kTile) * 16;
            // columns 54, 55 are the last word of chunk 6, columns 56..63 all of chunk 7
            const uint32_t w6 = __ldg(reinterpret_cast<const uint32_t*>(row + 6 * kChunkBytes + 12));
            const uint4 w7 = D > 2 ? __ldg(reinterpret_cast<const uint4*>(row + 7 * kChunkBytes)) : make_uint4(0, 0, 0, 0);
            const uint32_t w[5] = {w6, w7.x, w7.y, w7.z, w7.w};
#pragma unroll
            for (uint32_t k = 0; k < kMaxIndDim; ++k) {
                if (k < D) {
                    const __half2 h = *reinterpret_cast<const __half2*>(&w[k / 2]);
                    const float v = (k & 1) ? __high2float(h) : __low2float(h);
                    bad |= !isfinite(v);
                    acc[k] += v;
                }
            }
        }
        float* dst = ray_img ? g_codes + (size_t)ray_img[n] * D : g_codes;
#pragma unroll
        for (uint32_t k = 0; k < kMaxIndDim; ++k) {
            if (k < D) {
                float v = acc[k];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane == k && end > off) atomicAdd(dst + k, v);
            }
        }
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) opt_state[3] = 1.f;
}

// the same sum when ONE code row serves the whole launch (stage 1: one view, one image): every sample row below counters[1] adds into
// g_row; each thread sums a grid-stride share of the rows, the CTA reduces, one RED per CTA and dimension
__global__ void __launch_bounds__(256)
k_s0_code_grad_row(uint32_t D, const int32_t* __restrict__ counters, const uint8_t* __restrict__ denc_tiles, float* __restrict__ g_row,
                   float* __restrict__ opt_state) {
    __shared__ float red[8][kMaxIndDim];
    const uint32_t M = (uint32_t)counters[1];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float acc[kMaxIndDim];
#pragma unroll
    for (uint32_t k = 0; k < kMaxIndDim; ++k) acc[k] = 0.f;
    bool bad = false;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < M; j += gridDim.x * blockDim.x) {
        const uint8_t* row = denc_tiles + (size_t)(j / kTile) * kTileBytes + (j % kTile) * 16;
        const uint32_t w6 = __ldg(reinterpret_cast<const uint32_t*>(row + 6 * kChunkBytes + 12));
        const uint4 w7 = D > 2 ? __ldg(reinterpret_cast<const uint4*>(row + 7 * kChunkBytes)) : make_uint4(0, 0, 0, 0);
        const uint32_t w[5] = {w6, w7.x, w7.y, w7.z, w7.w};
#pragma unroll
        for (uint32_t k = 0; k < kMaxIndDim; ++k) {
            if (k < D) {
                const __half2 h = *reinterpret_cast<const __half2*>(&w[k / 2]);
                const float v = (k & 1) ? __high2float(h) : __low2float(h);
                bad |= !isfinite(v);
                acc[k] += v;
            }
        }
    }
#pragma unroll
    for (uint32_t k = 0; k < kMaxIndDim; ++k) {
        float v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][k] = v;
    }
    bad = __syncthreads_or(bad);
    if (threadIdx.x < D) {
        float v = 0.f;
        for (uint32_t w_ = 0; w_ < blockDim.x / 32; ++w_) v += red[w_][threadIdx.x];
        atomicAdd(g_row + threadIdx.x, v);
    }
    if (threadIdx.x == 0 && bad) opt_state[3] = 1.f;
}

// TV gradient of the density feature at one lattice cell of one level (gridencoder.cu:506-609), times weight w: centre, +1
// neighbours = corners 1, 2, 4, -1 neighbours = left[] (corners_of).  Used by the TV pass of the step's samples and by the
// random-point fallback.
__device__ __forceinline__ float tv_grad(const TableEntry* __restrict__ tab, const Corners& c, const uint32_t base[3],
                                         const uint32_t left[3], uint32_t res, float w) {
    const int right_corner[3] = {1, 2, 4};
    const float centre = __ldg(&tab[c.row[0]].d);
    float rv[3], lv[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {          // all seven loads are independent: issue them back to back
        rv[d] = __ldg(&tab[c.row[right_corner[d]]].d);
        lv[d] = base[d] > 0 ? __ldg(&tab[left[d]].d) : 0.f;
    }
    float sum = 0.f, sq = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        if (base[d] < res) { const float dv = centre - rv[d]; sum += dv; sq += dv * dv; }
        if (base[d] > 0) { const float dv = centre - lv[d]; sum += dv; sq += dv * dv; }
    }
    return w * sum * rsqrtf(sq + 1e-9f);
}

// ------------------------------------------------------------------------------------------------
// encode backward: scatter the (loss-scaled, fp16) feature gradients (template SCATTER = n2m_s0_encode_bwd) or add the TV
// gradient of the density features (template TV = n2m_s0_tv, its own launch that the host overlaps with the MLP kernels).
// L2 atomic throughput bounds this kernel, so at the coarse levels -- where the
// consecutive samples of a ray (= consecutive lanes) sit in the same lattice cell -- the 8 corner
// contributions are first summed across each run of same-cell lanes with a segmented warp scan and only the
// last lane of a run issues the red.global.add.v4.f32.  Fine levels (every lane its own cell) go straight to the atomics.
//
// Duplicate rows of neighbouring cells are not summed first.  Adjacent cells share corners, so on bench's lego batch the run merge
// leaves 69.9 REDs per sample for 48.7 distinct rows per 128-sample tile (per-level counts: profiles/grid_pass_time.py).  But the RED
// count alone does not bound this kernel: it issues those 19.9 M REDs at 56 G/s, where a kernel that only fires random REDs into one
// 8 MiB slice reaches 89 G/s.  Measured on an H100 80GB HBM3 (700 W), the scatter of one lego part takes 195 us with the code
// below.  Summing rows in a 1024-slot open-addressing table in shared memory first -- fp32 CAS loops (there is no shared fp32
// atomic add) or one 128-bit CAS per contribution, per CTA or per warp, at the levels below a cut from 5 to 13 -- took 266-470 us.
// Handing the corners shared with the previous issuing lane's cell over by shuffles took 182 us, but 391 us instead of 357 for the
// whole batch and more on garden (64 registers, 8 CTAs per SM), and left the step's concurrent backward passes no faster.
//
// Level-group walk.  The RED target is the whole gradient table: 6.1 M float4 rows = 97.6 MB at the default config (16 levels,
// 2^19 rows per hashed level), twice the H100's 50 MB L2.  A thread that walks all 16 levels of its sample sends its REDs anywhere
// in those 97.6 MB, so most of them miss L2 and cost a sector fill plus a write-back.  The work items of a launch are therefore
// (level group, tile) pairs, ordered group-major and walked by a grid-stride loop: the CTAs resident at any moment work on
// consecutive items, i.e. inside one or two groups, and the REDs land in one group's slice of the table (the dense levels 0-4
// together, 13 MB; then one hashed level, 8 MiB, at a time).  The price is that every group re-reads the sample's march record
// and the tile-image chunks that hold its own gradient columns -- small, L2-resident streams next to the RED traffic.  No result
// depends on the order in which the items run: every item adds its own contributions and the TV sample counts are taken once,
// by the items of group 0.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kDenseGroupLevels = 5;         // levels 0-4: 13 MB of gradient rows together at the default config
constexpr uint32_t kHashedGroupLevels = 1;        // every later level its own group (two per group: slower step on the H100)
constexpr uint32_t kLevelGroups = 1 + (kLevels - kDenseGroupLevels + kHashedGroupLevels - 1) / kHashedGroupLevels;

__device__ __forceinline__ uint32_t group_first_level(uint32_t grp) {
    return grp == 0 ? 0u : min(kLevels, kDenseGroupLevels + (grp - 1) * kHashedGroupLevels);
}

// The scatter's REDs carry an L2 evict-last hint: the lines of the current group's slice then outlast the streamed reads (march
// records, tile images, the parameter table) between two REDs to the same sector.
__device__ __forceinline__ uint64_t l2_evict_last() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void red_add_v4(float4* dst, float a, float b, float c, uint64_t pol) {
    asm volatile("red.global.add.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 :: "l"(dst), "f"(a), "f"(b), "f"(c), "f"(0.f), "l"(pol) : "memory");
}

template <bool SCATTER, bool TV>
__device__ __forceinline__ void
encode_bwd_visit(const n2m_s0_params& p, const float4* __restrict__ recs,
                 const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                 const uint8_t* __restrict__ denc_tiles, const TableEntry* __restrict__ table,
                 const int32_t* __restrict__ offsets, float4* __restrict__ gtable, float* __restrict__ loss_scale,
                 const PartRange pr, uint32_t tile, uint32_t l0, uint32_t l1, int32_t* tv_counts) {
    static_assert(SCATTER != TV, "a launch either scatters the feature gradients or evaluates TV");
    const uint32_t r = threadIdx.x & (kTile - 1);          // this thread's row of the tile (a CTA may hold several walkers)
    const uint32_t lane = r & 31;
    const uint32_t j = tile * kTile + r;
    Sample s;
    bool active = j >= pr.lo && j < pr.hi;
    if (active) {
        s = sample_of(recs[j], rays_o, rays_d, p);
        active = !((s.u < 0 || s.u > 1) || (s.v < 0 || s.v > 1) || (s.w < 0 || s.w > 1));
    } else {
        s.x = s.y = s.z = s.u = s.v = s.w = 0.5f; s.dx = s.dy = s.dz = 0.f;
    }

    // this row's gradients: cols 3..18 density, 19..50 colour (chunks 0..6); a group reads the columns of its own levels only
    const uint8_t* img = denc_tiles + (size_t)tile * kTileBytes + r * 16;
    bool bad = false;          // fp16 overflow of the loss-scaled gradients => GradScaler semantics: flag, step is skipped
    // TV weight: lambda inside the unit cube, 10 lambda outside when bound > 1 (utils.py:815-821); w = weight / (2 D),
    // kept in the loss-scaled domain
    float tvw_lane = 0.f;
    if (TV) {
        const float mag = fmaxf(fabsf(s.x), fmaxf(fabsf(s.y), fabsf(s.z)));
        const bool outer = p.grid_bound > 1 && mag > 1;
        const float lam = outer ? p.lambda_tv * 10 : p.lambda_tv;
        tvw_lane = active ? lam / 6 * loss_scale[0] : 0.f;
        // how many samples each of the reference's TV calls would receive (utils.py:815-823: xyzs_inner / xyzs_outer, or all of
        // them): counted once per sample, by the visit of the first level group
        const bool mine = j >= pr.lo && j < pr.hi;
        const uint32_t m_out = __ballot_sync(0xffffffffu, mine && outer), m_in = __ballot_sync(0xffffffffu, mine && !outer);
        if (lane == 0 && l0 == 0) {
            if (m_in) atomicAdd(tv_counts + 3, (int)__popc(m_in));
            if (m_out) atomicAdd(tv_counts + 15, (int)__popc(m_out));
        }
    }
#pragma unroll 1
    for (uint32_t l = l0; l < l1; ++l) {
        const LevelGeom lg = level_geom(offsets, l, p.S, p.base_res);
        Corners c; uint32_t base[3]; bool hashed; uint32_t left[3];
        corners_of(lg, s.u, s.v, s.w, c, base, hashed, TV ? left : nullptr);
        float tvw = tvw_lane;
        float4* gt = gtable + lg.row0;
        float gd = 0.f, g0 = 0.f, g1 = 0.f;
        if (SCATTER && active) {
            gd = denc_col(img, kColDens + l);
            g0 = denc_col(img, kColColor + 2 * l); g1 = denc_col(img, kColColor + 2 * l + 1);
            bad |= !isfinite(gd) || !isfinite(g0) || !isfinite(g1);
        }
        float vd[8], v0[8], v1[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { vd[k] = c.w[k] * gd; v0[k] = c.w[k] * g0; v1[k] = c.w[k] * g1; }
        // runs of consecutive lanes in the same cell
        const uint32_t key = active ? (base[0] | (base[1] << 10) | (base[2] << 20)) : 0xffffffffu;
        const uint32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || key != prev);
        const bool merge = lg.res < 1023u && (SCATTER ? __popc(heads) <= 20 : heads != 0xffffffffu);
        bool issue = active;
        if (merge) {
            const uint32_t run_start = 31u - __clz(heads & (0xffffffffu >> (31u - lane)));
            // segmented inclusive scan; only as many doubling rounds as the longest run of this warp needs (the later ones add nothing)
            const uint32_t longest = __reduce_max_sync(0xffffffffu, lane - run_start);
#pragma unroll 1
            for (uint32_t o = 1; o <= longest; o <<= 1) {
                const bool take = lane >= run_start + o;
                if (SCATTER) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float a = __shfl_up_sync(0xffffffffu, vd[k], o), b = __shfl_up_sync(0xffffffffu, v0[k], o),
                                    cc = __shfl_up_sync(0xffffffffu, v1[k], o);
                        if (take) { vd[k] += a; v0[k] += b; v1[k] += cc; }
                    }
                }
                if (TV) {
                    const float t = __shfl_up_sync(0xffffffffu, tvw, o);
                    if (take) tvw += t;
                }
            }
            const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
            issue = active && tail;
        }
        if (issue) {
            if (SCATTER) {
#pragma unroll
                const uint64_t pol = l2_evict_last();
#pragma unroll
                for (int k = 0; k < 8; ++k) red_add_v4(gt + c.row[k], vd[k], v0[k], v1[k], pol);
            }
            if (TV) atomicAdd(&gt[c.row[0]].x, tv_grad(table + lg.row0, c, base, left, lg.res, tvw));
        }
    }
    if (SCATTER && bad) loss_scale[3] = 1.f;
}

// grid-stride over the (level group, tile) items of the part's range [lo, hi), group-major (see "Level-group walk" above); the
// host sizes the grid to no more CTAs than fit on the device at once (encode_bwd_grid)
template <bool SCATTER, bool TV>
__global__ void __launch_bounds__(kTile)
k_s0_encode_bwd(n2m_s0_params p, const float4* __restrict__ recs, const int32_t* __restrict__ counters,
                const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                const uint8_t* __restrict__ denc_tiles, const TableEntry* __restrict__ table,
                const int32_t* __restrict__ offsets, float4* __restrict__ gtable, float* __restrict__ loss_scale,
                uint32_t part, uint32_t nparts) {
    const PartRange pr = part_range(counters, part, nparts);
    if (pr.hi <= pr.lo) return;
    const uint32_t t0 = pr.lo / kTile, nt = (pr.hi + kTile - 1) / kTile - t0;
#pragma unroll 1
    for (uint32_t item = blockIdx.x; item < kLevelGroups * nt; item += gridDim.x) {
        const uint32_t grp = item / nt;
        encode_bwd_visit<SCATTER, TV>(p, recs, rays_o, rays_d, denc_tiles, table, offsets, gtable, loss_scale, pr, t0 + item % nt,
                                      group_first_level(grp), group_first_level(grp + 1), const_cast<int32_t*>(counters));
    }
}

// The whole-SM form of the scatter (see "Launch geometry" below): a CTA of kWholeSmThreads threads is kWholeSmThreads / kTile independent
// 128-thread walkers, each visiting one (level group, tile) item at a time as a k_s0_encode_bwd CTA does; walker w of the grid starts at
// item w and strides by the grid's walker count, so the group-major order is kept.  The walkers share nothing (no CTA barrier).  The
// register cap (the fewest without a spill; the per-item loop of eight walkers needs 8 more than k_s0_encode_bwd) makes a CTA take
// more than half the register file, so the hardware places one per SM.  A kernel of its own, so that the per-slot form keeps its
// 48 registers and 10 CTAs per SM.
constexpr uint32_t kWholeSmThreads = 1024;

__global__ void __maxnreg__(56)
k_s0_scatter_walkers(n2m_s0_params p, const float4* __restrict__ recs, const int32_t* __restrict__ counters,
                     const float* __restrict__ rays_o, const float* __restrict__ rays_d, const uint8_t* __restrict__ denc_tiles,
                     const int32_t* __restrict__ offsets, float4* __restrict__ gtable, float* __restrict__ loss_scale,
                     uint32_t part, uint32_t nparts) {
    const PartRange pr = part_range(counters, part, nparts);
    if (pr.hi <= pr.lo) return;
    const uint32_t t0 = pr.lo / kTile, nt = (pr.hi + kTile - 1) / kTile - t0;
#pragma unroll 1
    for (uint32_t item = blockIdx.x * (kWholeSmThreads / kTile) + threadIdx.x / kTile; item < kLevelGroups * nt;
         item += gridDim.x * (kWholeSmThreads / kTile)) {
        const uint32_t grp = item / nt;
        encode_bwd_visit<true, false>(p, recs, rays_o, rays_d, denc_tiles, nullptr, offsets, gtable, loss_scale, pr, t0 + item % nt,
                                      group_first_level(grp), group_first_level(grp + 1), nullptr);
    }
}

// ------------------------------------------------------------------------------------------------
// TV fallback of GridEncoder.grad_total_variation (grid.py:181-183): a TV call that receives NO sample positions evaluates the TV
// gradient at B = 10^6 uniformly random points of [0,1]^3 instead.  In the reference's post_train_step (utils.py:815-823) that happens
// to the inner call (weight lambda) when no sample lies inside the unit cube, to the outer call (10 lambda) when none lies outside
// (bound > 1), and to the single call of bound <= 1 when the batch marched no sample at all.  The group counts come from the TV pass of
// this step (counters[3], [15]); the points from a counter-based hash of (optimizer step, point index) -- the reference draws
// torch.rand, so the point SETS differ while the estimator is the same (tests feed the same points to the reference kernel).
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t h) {
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}
__host__ __device__ __forceinline__ float tv_random_coord(uint32_t seed, uint32_t idx, uint32_t axis) {
    return (float)(mix32(mix32(idx * 3u + axis) ^ (seed * 0x9e3779b9u)) >> 8) * (1.0f / 16777216.0f);
}

__global__ void __launch_bounds__(128)
k_s0_tv_random(n2m_s0_params p, const int32_t* __restrict__ counters, const TableEntry* __restrict__ table,
               const int32_t* __restrict__ offsets, float4* __restrict__ gtable, const float* __restrict__ loss_scale, uint32_t B,
               float* __restrict__ dump) {
    // which of the reference's TV calls of this step would have been empty
    float lam = 0.f;
    if (p.grid_bound > 1) {
        if (counters[3] == 0) lam += p.lambda_tv;
        if (counters[15] == 0) lam += p.lambda_tv * 10;
    } else if (counters[3] + counters[15] == 0) lam = p.lambda_tv;
    if (dump) lam = p.lambda_tv;                    // test hook: always run, plain weight, record the points
    if (!(lam > 0.f)) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const uint32_t seed = (uint32_t)loss_scale[2];            // optimizer step count (opt_state[2]): a new point set every step
    const float u = tv_random_coord(seed, i, 0), v = tv_random_coord(seed, i, 1), w = tv_random_coord(seed, i, 2);
    if (dump) { dump[3 * i] = u; dump[3 * i + 1] = v; dump[3 * i + 2] = w; }
    const float tvw = lam / 6 * loss_scale[0];
#pragma unroll 1
    for (uint32_t l = 0; l < kLevels; ++l) {
        const LevelGeom lg = level_geom(offsets, l, p.S, p.base_res);
        Corners c; uint32_t base[3]; bool hashed; uint32_t left[3];
        corners_of(lg, u, v, w, c, base, hashed, left);
        atomicAdd(&gtable[lg.row0 + c.row[0]].x, tv_grad(table + lg.row0, c, base, left, lg.res, tvw));
    }
}

// ------------------------------------------------------------------------------------------------
// composite forward + loss + composite backward: one WARP per ray.
// The reference walks each ray sequentially in one thread (raymarching.cu:541-568, 651-693); here the
// transmittance is a warp prefix product, the accumulations are warp scans / reductions and early
// termination is a ballot, so a 70-sample ray costs ~3 chunk iterations instead of 140 dependent steps.
// Same formulas; the summation order differs (1e-6-level), which is why the bit-exact drop-in operator
// (raymarching.cu in this repo) keeps the sequential order and this fused stage is tolerance-checked.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_incl_scan_add(float v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const float u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= (uint32_t)o) v += u; }
    return v;
}
__device__ __forceinline__ float warp_incl_scan_mul(float v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const float u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= (uint32_t)o) v *= u; }
    return v;
}

// binary entropy in bits of w clamped to [1e-5, 1 - 1e-5] and its derivative (zero where the clamp is active), utils.py:729-732
__device__ __forceinline__ float entropy_bits(float w, float& dH) {
    const float wc = fminf(fmaxf(w, 1e-5f), 1.0f - 1e-5f);
    const float l1 = __log2f(wc), l0 = __log2f(1.0f - wc);
    dH = (w > 1e-5f && w < 1.0f - 1e-5f) ? l0 - l1 : 0.f;
    return -wc * l1 - (1.0f - wc) * l0;
}

template <bool ADAPTIVE>
__global__ void __launch_bounds__(128)
k_s0_composite_loss(n2m_s0_params p, const float4* __restrict__ out, const float4* __restrict__ recs,
                    const int32_t* __restrict__ rays, const int32_t* __restrict__ counters, uint32_t N,
                    const float* __restrict__ gt, const float* __restrict__ bg, const float* __restrict__ loss_scale,
                    float4* __restrict__ dout, float* __restrict__ image, float* __restrict__ weights_sum,
                    float* __restrict__ depth, float* __restrict__ loss_out, const int32_t* __restrict__ active, uint32_t lo,
                    uint32_t hi) {
    // rays [lo, hi) of the N-ray batch (a part of the batch, n2m_common.cuh part_range).  ADAPTIVE: the batch is its first n = *active
    // rays (the count the march recorded) and this launch takes rays [n*lo/8, n*hi/8).  All means are over the batch's rays
    uint32_t n_act = N, ray_lo = lo, ray_hi = hi;
    if (ADAPTIVE) {
        n_act = ray_count(active, N);
        ray_lo = part_first_ray(n_act, lo);
        ray_hi = part_first_ray(n_act, hi);
    }
    const uint32_t n = ray_lo + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const uint32_t lane = threadIdx.x & 31;
    if (n >= ray_hi) return;
    const uint32_t M = (uint32_t)counters[1];
    const uint32_t off = rays[2 * n], cnt = rays[2 * n + 1];
    const bool live = cnt != 0 && off + cnt <= M;

    // ---- forward ----
    float T_in = 1.0f, r = 0, g = 0, b = 0, ws = 0, d = 0;
    uint32_t n_used = 0;                 // samples up to and including the one that crossed T_thresh
    const bool ent = p.lambda_entropy > 0.f;
    float ent_sum = 0.f;                 // per lane: entropy of the weights this ray's loop touched
    if (live) {
        for (uint32_t base = 0; base < cnt; base += 32) {
            const uint32_t k = base + lane;
            const bool valid = k < cnt;
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f); float4 rc = o;
            if (valid) { o = out[off + k]; rc = recs[off + k]; }
            const float alpha = valid ? 1.0f - __expf(-o.x * rc.y) : 0.f;
            const float Tpost = T_in * warp_incl_scan_mul(1.0f - alpha, lane);      // transmittance after sample k
            float Tpre = __shfl_up_sync(0xffffffffu, Tpost, 1);
            if (lane == 0) Tpre = T_in;
            const uint32_t stop = __ballot_sync(0xffffffffu, valid && Tpost < p.T_thresh);
            const uint32_t last = stop ? (uint32_t)(__ffs(stop) - 1) : 31u;           // last contributing lane
            const bool use = valid && lane <= last;
            const float w = use ? alpha * Tpre : 0.f;
            r += warp_sum(w * o.y); g += warp_sum(w * o.z); b += warp_sum(w * o.w);
            ws += warp_sum(w); d += warp_sum(w * rc.z);
            if (ent) { float dH; ent_sum += use ? entropy_bits(w, dH) : 0.f; }
            n_used = base + min(last + 1u, cnt - base);
            if (stop) break;
            T_in = __shfl_sync(0xffffffffu, Tpost, 31);
        }
    }
    // ---- background mix (renderer.py:804) and loss (utils.py:660-683): identical on all lanes ----
    const float b0 = bg[3 * n], b1 = bg[3 * n + 1], b2 = bg[3 * n + 2];
    const float om = 1 - ws;
    const float pr = r + om * b0, pg = g + om * b1, pb = b + om * b2;
    float t0, t1, t2, mask = 0.f;
    if (p.gt_has_alpha) {
        mask = gt[4 * n + 3];
        t0 = gt[4 * n] * mask + b0 * (1 - mask);
        t1 = gt[4 * n + 1] * mask + b1 * (1 - mask);
        t2 = gt[4 * n + 2] * mask + b2 * (1 - mask);
    } else {
        t0 = gt[3 * n]; t1 = gt[3 * n + 1]; t2 = gt[3 * n + 2];
    }
    const float e0 = pr - t0, e1 = pg - t1, e2 = pb - t2;
    float my_loss = (e0 * e0 + e1 * e1 + e2 * e2) * (1.0f / 3.0f);
    const float invN = 1.0f / (float)n_act;
    const float sc = loss_scale[0] * invN;
    const float gi0 = sc * (2.0f / 3.0f) * e0, gi1 = sc * (2.0f / 3.0f) * e1, gi2 = sc * (2.0f / 3.0f) * e2;
    float gws = -(gi0 * b0 + gi1 * b1 + gi2 * b2);          // pred = image + (1 - ws) * bg
    if (p.gt_has_alpha && p.lambda_mask > 0) {
        const float em = ws - mask;
        my_loss += p.lambda_mask * em * em;
        gws += sc * p.lambda_mask * 2.0f * em;
    }
    // entropy regulariser (utils.py:728-733): lambda * (mean_k H(weights_k) + mean_n H(weights_sum_n)).  The ray-level term
    // joins this ray's loss; the sample-level sum goes to loss_out[2] (+ the count of touched weights in [3], the untouched
    // entries of `weights` are 0 and contribute the constant H(1e-5)); gw_scale feeds grad_weights below.
    float gw_scale = 0.f;
    if (ent) {
        float dH2;
        my_loss += p.lambda_entropy * entropy_bits(ws, dH2);
        gws += sc * p.lambda_entropy * dH2;
        gw_scale = M > 0 ? loss_scale[0] * p.lambda_entropy / (float)M : 0.f;
        ent_sum = warp_sum(ent_sum);
        if (lane == 0 && live) { atomicAdd(loss_out + 2, ent_sum); atomicAdd(loss_out + 3, (float)n_used); }
    }
    if (lane == 0) {
        image[3 * n] = pr; image[3 * n + 1] = pg; image[3 * n + 2] = pb;
        weights_sum[n] = ws;
        depth[n] = d;
        atomicAdd(loss_out, my_loss * invN);
    }

    // ---- backward (raymarching.cu:605-694 with grad_weights = grad_depth = 0) ----
    if (live) {
        float Tc = 1.0f, cr = 0, cg = 0, cb = 0, cw = 0;     // carries: transmittance and prefix sums
        for (uint32_t base = 0; base < cnt; base += 32) {
            const uint32_t k = base + lane;
            if (base >= n_used) {                            // past the break: zero gradient
                if (k < cnt) dout[off + k] = make_float4(0.f, 0.f, 0.f, 0.f);
                continue;
            }
            const bool use = k < n_used;
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f); float dtk = 0.f;
            if (use) { o = out[off + k]; dtk = recs[off + k].y; }
            const float alpha = use ? 1.0f - __expf(-o.x * dtk) : 0.f;
            const float Tpost = Tc * warp_incl_scan_mul(1.0f - alpha, lane);
            float Tpre = __shfl_up_sync(0xffffffffu, Tpost, 1);
            if (lane == 0) Tpre = Tc;
            const float w = alpha * Tpre;
            const float sr = cr + warp_incl_scan_add(w * o.y, lane), sg = cg + warp_incl_scan_add(w * o.z, lane);
            const float sb = cb + warp_incl_scan_add(w * o.w, lane), sw = cw + warp_incl_scan_add(w, lane);
            if (k < cnt) {
                float4 gq = make_float4(0.f, 0.f, 0.f, 0.f);
                if (use) {
                    // grad_weights_k rides with grad_weights_sum exactly as in raymarching.cu:676
                    float gwk = 0.f;
                    if (ent) { float dH; entropy_bits(w, dH); gwk = gw_scale * dH; }
                    gq.x = dtk * (gi0 * (Tpost * o.y - (r - sr)) + gi1 * (Tpost * o.z - (g - sg)) +
                                  gi2 * (Tpost * o.w - (b - sb)) + (gws + gwk) * (Tpost - (ws - sw)));
                    gq.y = gi0 * w; gq.z = gi1 * w; gq.w = gi2 * w;
                }
                dout[off + k] = gq;
            }
            Tc = __shfl_sync(0xffffffffu, Tpost, 31);
            cr = __shfl_sync(0xffffffffu, sr, 31); cg = __shfl_sync(0xffffffffu, sg, 31);
            cb = __shfl_sync(0xffffffffu, sb, 31); cw = __shfl_sync(0xffffffffu, sw, 31);
        }
    } else if (cnt != 0) {
        for (uint32_t k = lane; k < cnt && off + k < M; k += 32) dout[off + k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// ------------------------------------------------------------------------------------------------
// density-grid update (NeRFRenderer.update_extra_state, renderer.py:1074-1149)
// ------------------------------------------------------------------------------------------------
// jittered cell centres of one cascade, cells enumerated in MORTON order (cell m <-> coords morton3D_invert(m)),
// so sigma lands directly at density_grid[cas, m] (renderer.py:1100-1118).  `noise` is the cascade's whole [H^3, 3] draw in the
// reference's MESHGRID order (row x*H*H + y*H + z, renderer.py:1098-1099,1110: torch.rand_like(cas_xyzs)), so that the same torch
// generator state gives every cell the same jitter as in the reference.
__global__ void __launch_bounds__(256)
k_s0_grid_points(uint32_t H, uint32_t first_cell, uint32_t count, float cas_bound, const float* __restrict__ noise,
                 float* __restrict__ xyz) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t m = first_cell + i;
    const float hgs = cas_bound / (float)H;                  // half_grid_size = bound / grid_size (:1105)
    const float span = cas_bound - hgs;
    const uint32_t c[3] = {compact3(m), compact3(m >> 1), compact3(m >> 2)};
    const uint32_t lin = (c[0] * H + c[1]) * H + c[2];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float base = __fadd_rn(__fdiv_rn(__fmul_rn(2.0f, (float)c[a]), (float)(H - 1)), -1.0f);   // 2*coord/(H-1) - 1
        const float jit = __fmul_rn(__fadd_rn(__fmul_rn(noise[3 * (size_t)lin + a], 2.0f), -1.0f), hgs);   // (rand*2-1)*hgs
        xyz[3 * i + a] = __fadd_rn(__fmul_rn(base, span), jit);
    }
}

// grid = max(grid * decay, sigma) where both are >= 0 (renderer.py:1121-1124); sigma = out[i].x
__global__ void __launch_bounds__(256)
k_s0_grid_update(const float4* __restrict__ out, uint32_t count, float decay, float* __restrict__ cells) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const float g = cells[i], sg = out[i].x;
    if (g >= 0.f && sg >= 0.f) cells[i] = fmaxf(g * decay, sg);
}

// packbits with the threshold min(mean_density, density_thresh) read from device memory (no .item() sync)
__global__ void __launch_bounds__(256)
k_s0_packbits_dev(const float* __restrict__ grid, uint32_t nbytes, const float* __restrict__ mean_density, float density_thresh,
                  uint8_t* __restrict__ bits) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nbytes) return;
    const float thresh = fminf(mean_density[0], density_thresh);
    const float4 a = reinterpret_cast<const float4*>(grid)[2 * n], b = reinterpret_cast<const float4*>(grid)[2 * n + 1];
    uint32_t v = 0;
    v |= (a.x > thresh) << 0; v |= (a.y > thresh) << 1; v |= (a.z > thresh) << 2; v |= (a.w > thresh) << 3;
    v |= (b.x > thresh) << 4; v |= (b.y > thresh) << 5; v |= (b.z > thresh) << 6; v |= (b.w > thresh) << 7;
    bits[n] = (uint8_t)v;
}

// ------------------------------------------------------------------------------------------------
// batch sampling on the device: get_rays (utils.py:236-290) + the training collate of the provider
// (provider.py:300-331) for random (image, pixel) pairs over a device-resident pose / image set.
// One thread per ray: pixel centre (+0.5), camera-space direction ((i-cx)/fx, -(j-cy)/fy, -1), rotated by the
// pose (row-times-R^T == R times column), origin = pose translation, ground truth = images[idx, j, i] / 255.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_s0_gen_rays(const float* __restrict__ poses, float fx, float fy, float cx, float cy, uint32_t W,
              const int32_t* __restrict__ img_idx, const int32_t* __restrict__ pix_idx, const uint8_t* __restrict__ images,
              uint32_t HW, uint32_t C, uint32_t N, float* __restrict__ rays_o, float* __restrict__ rays_d, float* __restrict__ gt) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const uint32_t b = (uint32_t)img_idx[n], pix = (uint32_t)pix_idx[n];
    const float i = __fadd_rn((float)(pix % W), 0.5f), j = __fadd_rn((float)(pix / W), 0.5f);
    const float x = __fdiv_rn(__fsub_rn(i, cx), fx), y = -__fdiv_rn(__fsub_rn(j, cy), fy), z = -1.0f;
    const float* P = poses + (size_t)b * 16;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        // fp32 dot product in index order, no FMA contraction (as a reference matmul of a [1,3] row does on CUDA cores)
        rays_d[3 * n + r] = __fadd_rn(__fadd_rn(__fmul_rn(P[4 * r], x), __fmul_rn(P[4 * r + 1], y)), __fmul_rn(P[4 * r + 2], z));
        rays_o[3 * n + r] = P[4 * r + 3];
    }
    if (gt) {
        const uint8_t* px = images + ((size_t)b * HW + pix) * C;
        for (uint32_t c = 0; c < C; ++c) gt[(size_t)n * C + c] = __fdiv_rn((float)px[c], 255.0f);
    }
}

// ------------------------------------------------------------------------------------------------
// table (de)interleave
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_s0_pack_tables(const float* __restrict__ ed, const float* __restrict__ ec, uint32_t rows,
                 TableEntry* __restrict__ table, float2* __restrict__ cmaster) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const float2 c = make_float2(ec[2 * i], ec[2 * i + 1]);
    TableEntry e; e.d = ed[i]; e.c = __floats2half2_rn(c.x, c.y);
    table[i] = e;
    cmaster[i] = c;
}

__global__ void __launch_bounds__(256)
k_s0_unpack_tables(const TableEntry* __restrict__ table, const float2* __restrict__ cmaster, uint32_t rows,
                   float* __restrict__ ed, float* __restrict__ ec) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    ed[i] = table[i].d;
    ec[2 * i] = cmaster[i].x; ec[2 * i + 1] = cmaster[i].y;
}

__global__ void __launch_bounds__(256)
k_s0_unpack_grads(const float4* __restrict__ gtable, uint32_t rows, const float* __restrict__ loss_scale,
                  float* __restrict__ gd, float* __restrict__ gc) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const float inv = 1.0f / loss_scale[0];
    const float4 g = gtable[i];
    gd[i] = g.x * inv; gc[2 * i] = g.y * inv; gc[2 * i + 1] = g.z * inv;
}

}  // namespace
}  // namespace n2m

using namespace n2m;

static bool g_serial_march = false;

// blocks for one part's gather / scatter launch: the part's expected share of the sample slab plus one boundary tile
// (the kernels are grid-stride over the part's tiles, so an unbalanced part is still covered)
static inline uint32_t part_grid(uint32_t Mcap, uint32_t nparts) {
    return nparts <= 1 ? Mcap / kTile : div_up(Mcap / kTile, nparts) + 1;
}

// Launch geometry of one scatter / TV launch.  Every walk is persistent: its CTAs keep their SM resources until the last item, and
// the launch takes 1/(nparts * share) of the device, so that the walks the step runs side by side (the parts' scatters, TV) each get
// their own share and walk the level groups at the same time.
//  * A scatter with nparts > 1 runs beside the other parts' chains, whose k_mlp_bwd (384 threads x 160 registers, 217 KB of shared
//    memory) only starts on an SM with no other CTA on it.  It takes the whole-SM form (k_s0_scatter_walkers): one CTA per SM on
//    S / nparts of the S SMs, so the other SMs are free of it as soon as one part's k_mlp_bwd leaves them.  In the per-slot form the
//    part-0 scatter's CTAs queued behind part 1's k_mlp_bwd on every SM (33 us on lego, 87 us on garden).  On an H100 80GB HBM3
//    (700 W) this took the lego step from 1.070-1.077 to 1.034-1.036 ms and the garden step from 2.321-2.332 to 2.199-2.207 ms.  A
//    whole-SM grid of S CTAs per part measured 1.091-1.093 / 2.271-2.283 ms.
//  * Every other launch (TV; the scatter with nparts == 1: stage 1, the fused forward, single-part stage 0) takes the per-slot form
//    (k_s0_encode_bwd) on its share of every SM's resident slots: TV runs underneath the forward chains, whose CTAs are small, and a
//    lone scatter has nothing beside it.  TV in the whole-SM form on half of the SMs measured 1.026-1.030 / 2.259 ms, on a third
//    1.032-1.034 / 2.220 ms, against 1.032-1.033 / 2.201-2.202 ms for the per-slot TV (scatters whole-SM in all three).
// Never more CTAs than the launch has items.
static int g_scatter_form = 0;        // test hook n2m_s0_set_scatter_form: 0 = by part count, 1 = per-slot, 2 = whole-SM

template <bool SCATTER, bool TV>
static uint32_t encode_bwd_grid(uint32_t Mcap, uint32_t nparts, uint32_t share = 1) {
    static int per_sm = 0;
    if (!per_sm) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_s0_encode_bwd<SCATTER, TV>, kTile, 0);
        if (per_sm <= 0) per_sm = 1;
    }
    return min(max(1u, (uint32_t)(per_sm * num_sms()) / (nparts * share)), kLevelGroups * part_grid(Mcap, nparts));
}

static uint32_t scatter_walkers_grid(uint32_t Mcap, uint32_t nparts) {
    return min(max(1u, (uint32_t)num_sms() / nparts), div_up(kLevelGroups * part_grid(Mcap, nparts), kWholeSmThreads / kTile));
}

// The TV launch gets half of the device.  The step forks it at its start, beside the parts' gather -> MLP -> composite chains.  A
// grid of every CTA the device holds at once is a persistent grid-stride walk that keeps its slots until the last item, so the
// kernels of those chains find no room on the SMs beside it; with half the slots TV runs underneath them.  On an H100 80GB HBM3
// (700 W) this took the lego step from 1.139-1.142 to 1.076 ms and the garden step from 2.463-2.472 to 2.328-2.331 ms.  A third
// of the device measured 1.083 / 2.327 ms, a quarter 1.081 / 2.363 ms, a sixth 1.121 ms on lego.
constexpr uint32_t kTvDeviceShare = 2;

extern "C" {

/* test hook: 1 = one-thread-per-ray sequential marcher (the reference's structure), 0 = warp-per-ray (default) */
int n2m_s0_set_serial_march(int on) { g_serial_march = on != 0; return 0; }
/* test hook: launch form of the scatter, 0 = chosen from its part count (default), 1 = per-slot, 2 = whole-SM */
int n2m_s0_set_scatter_form(int form) {
    N2M_REQUIRE(form >= 0 && form <= 2, "s0_set_scatter_form", "form must be 0, 1 or 2");
    g_scatter_form = form;
    return 0;
}
int n2m_s0_pack_tables(const float* emb_density, const float* emb_color, uint32_t rows, void* table, void* color_master,
                       n2m_stream_t stream) {
    N2M_REQUIRE(emb_density && emb_color && table && color_master, "s0_pack_tables", "null pointer");
    k_s0_pack_tables<<<div_up(rows, 256u), 256, 0, as_stream(stream)>>>(emb_density, emb_color, rows,
                                                                         static_cast<TableEntry*>(table), static_cast<float2*>(color_master));
    return check_launch("s0_pack_tables");
}

int n2m_s0_unpack_tables(const void* table, const void* color_master, uint32_t rows, float* emb_density, float* emb_color,
                         n2m_stream_t stream) {
    N2M_REQUIRE(emb_density && emb_color && table && color_master, "s0_unpack_tables", "null pointer");
    k_s0_unpack_tables<<<div_up(rows, 256u), 256, 0, as_stream(stream)>>>(static_cast<const TableEntry*>(table),
                                                                           static_cast<const float2*>(color_master), rows, emb_density, emb_color);
    return check_launch("s0_unpack_tables");
}

int n2m_s0_unpack_grads(const void* gtable, uint32_t rows, const float* loss_scale, float* g_density, float* g_color,
                        n2m_stream_t stream) {
    N2M_REQUIRE(gtable && loss_scale && g_density && g_color, "s0_unpack_grads", "null pointer");
    k_s0_unpack_grads<<<div_up(rows, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(gtable), rows, loss_scale, g_density, g_color);
    return check_launch("s0_unpack_grads");
}

int n2m_s0_march(const n2m_s0_params* p, const float* rays_o, const float* rays_d, const float* aabb,
                 const float* cam_near_far, const uint8_t* bitfield, const float* noises, uint32_t N, int32_t* rays,
                 int32_t* counters, float* tbuf, void* recs, uint32_t Mcap, int32_t* ray_ctl, uint32_t num_points,
                 n2m_stream_t stream) {
    N2M_REQUIRE(p && rays && counters, "s0_march", "null pointer");
    cudaStream_t st = as_stream(stream);
    if (N == 0) { cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), st); return 0; }
    N2M_REQUIRE(rays_o && rays_d && aabb && bitfield && noises && tbuf && recs, "s0_march", "null pointer");
    N2M_REQUIRE(p->max_steps > 0 && p->grid_size > 0 && p->cascades > 0, "s0_march", "bad params");
    N2M_REQUIRE(!ray_ctl || num_points > 0, "s0_march", "adaptive ray count needs num_points > 0");
    auto count = g_serial_march ? (ray_ctl ? k_s0_count<true> : k_s0_count<false>)
                                : (ray_ctl ? k_s0_count_warp<true> : k_s0_count_warp<false>);
    count<<<g_serial_march ? div_up(N, 128u) : div_up(N * 32u, 128u), 128, 0, st>>>(rays_o, rays_d, aabb, cam_near_far, bitfield, noises,
                                                                                   *p, N, ray_ctl, rays, reinterpret_cast<float2*>(tbuf));
    if (int e = check_launch("s0_march(count)")) return e;
    k_s0_scan<<<1, 1024, 0, st>>>(rays, N, Mcap, counters, ray_ctl, num_points);
    if (int e = check_launch("s0_march(scan)")) return e;
    k_s0_records<<<div_up(N * 32u, 256u), 256, 0, st>>>(rays, reinterpret_cast<const float2*>(tbuf), N, p->max_steps, Mcap,
                                                        static_cast<float4*>(recs));
    return check_launch("s0_march(records)");
}

int n2m_s0_encode_fwd(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap,
                      const float* rays_o, const float* rays_d, const void* table, const int32_t* offsets, void* enc_tiles,
                      uint32_t part, uint32_t nparts, n2m_stream_t stream) {
    N2M_REQUIRE(p && recs && counters && rays_o && rays_d && table && offsets && enc_tiles, "s0_encode_fwd", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_encode_fwd", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_encode_fwd", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_encode_fwd", "nparts must be 1, 2, 4 or 8 and part < nparts");
    k_s0_encode_fwd<false, false><<<part_grid(Mcap, nparts), kTile, 0, as_stream(stream)>>>(
        *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const TableEntry*>(table), offsets,
        static_cast<uint8_t*>(enc_tiles), part, nparts, nullptr, nullptr);
    return check_launch("s0_encode_fwd");
}

int n2m_s0_encode_fwd_codes(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                            const float* rays_d, const void* table, const int32_t* offsets, const float* codes, const int32_t* ray_img,
                            void* enc_tiles, uint32_t part, uint32_t nparts, n2m_stream_t stream) {
    N2M_REQUIRE(p && p->ind_dim <= kMaxIndDim, "s0_encode_fwd_codes", "ind_dim must be at most 10");
    if (p->ind_dim == 0) return n2m_s0_encode_fwd(p, recs, counters, Mcap, rays_o, rays_d, table, offsets, enc_tiles, part, nparts, stream);
    N2M_REQUIRE(recs && counters && rays_o && rays_d && table && offsets && enc_tiles && codes, "s0_encode_fwd_codes", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_encode_fwd_codes", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_encode_fwd_codes", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_encode_fwd_codes", "nparts must be 1, 2, 4 or 8 and part < nparts");
    k_s0_encode_fwd<false, true><<<part_grid(Mcap, nparts), kTile, 0, as_stream(stream)>>>(
        *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const TableEntry*>(table), offsets,
        static_cast<uint8_t*>(enc_tiles), part, nparts, codes, ray_img);
    return check_launch("s0_encode_fwd_codes");
}

int n2m_s0_code_grad_row(const n2m_s0_params* p, const int32_t* counters, uint32_t Mcap, const void* denc_tiles, float* g_row,
                         float* opt_state, n2m_stream_t stream) {
    N2M_REQUIRE(p && p->ind_dim <= kMaxIndDim, "s0_code_grad_row", "ind_dim must be at most 10");
    if (p->ind_dim == 0 || Mcap == 0) return 0;
    N2M_REQUIRE(counters && denc_tiles && g_row && opt_state, "s0_code_grad_row", "null pointer");
    const uint32_t grid = min(div_up(Mcap, 256u * 8u), (uint32_t)(4 * num_sms()));
    k_s0_code_grad_row<<<grid, 256, 0, as_stream(stream)>>>(p->ind_dim, counters, static_cast<const uint8_t*>(denc_tiles), g_row, opt_state);
    return check_launch("s0_code_grad_row");
}

int n2m_s0_code_grad(const n2m_s0_params* p, const int32_t* rays, const int32_t* counters, uint32_t N, const void* denc_tiles,
                     const int32_t* ray_img, float* g_codes, float* opt_state, const int32_t* active_rays, uint32_t part, uint32_t nparts,
                     n2m_stream_t stream) {
    N2M_REQUIRE(p && p->ind_dim <= kMaxIndDim, "s0_code_grad", "ind_dim must be at most 10");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_code_grad", "nparts must be 1, 2, 4 or 8 and part < nparts");
    if (p->ind_dim == 0 || N == 0) return 0;
    N2M_REQUIRE(rays && counters && denc_tiles && g_codes && opt_state, "s0_code_grad", "null pointer");
    const uint32_t e0 = part * kPartSlots / nparts, e1 = (part + 1) * kPartSlots / nparts;
    // the part's rays may be known on the device only (adaptive count): cover the largest part any n <= N gives
    const uint32_t most = active_rays ? div_up(N, nparts) + 1 : part_first_ray(N, e1) - part_first_ray(N, e0);
    if (most == 0) return 0;
    k_s0_code_grad<<<div_up(most * 32u, 128u), 128, 0, as_stream(stream)>>>(p->ind_dim, rays, counters, N,
                                                                          static_cast<const uint8_t*>(denc_tiles), ray_img, g_codes,
                                                                          opt_state, active_rays, e0, e1);
    return check_launch("s0_code_grad");
}

int n2m_s0_encode_points(const n2m_s0_params* p, const float* xyz, const float* dirs, const int32_t* counters, uint32_t Pcap,
                         const void* table, const int32_t* offsets, void* enc_tiles, n2m_stream_t stream) {
    N2M_REQUIRE(p && xyz && counters && table && offsets && enc_tiles, "s0_encode_points", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_encode_points", "fused path supports num_levels == 16");
    N2M_REQUIRE(Pcap % kTile == 0 && Pcap > 0, "s0_encode_points", "Pcap must be a positive multiple of 128");
    k_s0_encode_fwd<true, false><<<Pcap / kTile, kTile, 0, as_stream(stream)>>>(*p, nullptr, counters, xyz, dirs,
                                                                                static_cast<const TableEntry*>(table), offsets,
                                                                                static_cast<uint8_t*>(enc_tiles), 0, 1, nullptr, nullptr);
    return check_launch("s0_encode_points");
}

int n2m_s0_encode_points_codes(const n2m_s0_params* p, const float* xyz, const float* dirs, const int32_t* counters, uint32_t Pcap,
                               const void* table, const int32_t* offsets, const float* code_row, void* enc_tiles, n2m_stream_t stream) {
    N2M_REQUIRE(p && p->ind_dim <= kMaxIndDim, "s0_encode_points_codes", "ind_dim must be at most 10");
    if (p->ind_dim == 0) return n2m_s0_encode_points(p, xyz, dirs, counters, Pcap, table, offsets, enc_tiles, stream);
    N2M_REQUIRE(xyz && counters && table && offsets && enc_tiles && code_row, "s0_encode_points_codes", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_encode_points_codes", "fused path supports num_levels == 16");
    N2M_REQUIRE(Pcap % kTile == 0 && Pcap > 0, "s0_encode_points_codes", "Pcap must be a positive multiple of 128");
    k_s0_encode_fwd<true, true><<<Pcap / kTile, kTile, 0, as_stream(stream)>>>(*p, nullptr, counters, xyz, dirs,
                                                                               static_cast<const TableEntry*>(table), offsets,
                                                                               static_cast<uint8_t*>(enc_tiles), 0, 1, code_row, nullptr);
    return check_launch("s0_encode_points_codes");
}

int n2m_s0_grid_points(uint32_t H, uint32_t first_cell, uint32_t count, float cas_bound, const float* noise, float* xyz,
                       n2m_stream_t stream) {
    N2M_REQUIRE(noise && xyz && H > 1, "s0_grid_points", "bad arguments");
    if (count == 0) return 0;
    k_s0_grid_points<<<div_up(count, 256u), 256, 0, as_stream(stream)>>>(H, first_cell, count, cas_bound, noise, xyz);
    return check_launch("s0_grid_points");
}

int n2m_s0_grid_update(const void* out, uint32_t count, float decay, float* grid_cells, n2m_stream_t stream) {
    N2M_REQUIRE(out && grid_cells, "s0_grid_update", "null pointer");
    if (count == 0) return 0;
    k_s0_grid_update<<<div_up(count, 256u), 256, 0, as_stream(stream)>>>(static_cast<const float4*>(out), count, decay, grid_cells);
    return check_launch("s0_grid_update");
}

int n2m_s0_packbits_dev(const float* grid, uint32_t nbytes, const float* mean_density, float density_thresh, uint8_t* bitfield,
                        n2m_stream_t stream) {
    N2M_REQUIRE(grid && mean_density && bitfield, "s0_packbits_dev", "null pointer");
    if (nbytes == 0) return 0;
    k_s0_packbits_dev<<<div_up(nbytes, 256u), 256, 0, as_stream(stream)>>>(grid, nbytes, mean_density, density_thresh, bitfield);
    return check_launch("s0_packbits_dev");
}

int n2m_s0_gen_rays(const float* poses, uint32_t num_poses, const float* intrinsics_host, uint32_t H, uint32_t W,
                    const int32_t* img_idx, const int32_t* pix_idx, const uint8_t* images, uint32_t C, uint32_t N,
                    float* rays_o, float* rays_d, float* gt, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(poses && intrinsics_host && img_idx && pix_idx && rays_o && rays_d, "s0_gen_rays", "null pointer");
    N2M_REQUIRE(num_poses > 0 && H > 0 && W > 0, "s0_gen_rays", "empty pose set or image");
    N2M_REQUIRE(!gt || (images && (C == 3 || C == 4)), "s0_gen_rays", "gt requested without images, or channels not 3 / 4");
    k_s0_gen_rays<<<div_up(N, 256u), 256, 0, as_stream(stream)>>>(poses, intrinsics_host[0], intrinsics_host[1], intrinsics_host[2],
                                                                 intrinsics_host[3], W, img_idx, pix_idx, images, H * W, C, N,
                                                                 rays_o, rays_d, gt);
    return check_launch("s0_gen_rays");
}

int n2m_s0_encode_bwd(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap,
                      const float* rays_o, const float* rays_d, const void* denc_tiles, const void* table,
                      const int32_t* offsets, void* gtable, const float* loss_scale, uint32_t part, uint32_t nparts,
                      n2m_stream_t stream) {
    N2M_REQUIRE(p && recs && counters && rays_o && rays_d && denc_tiles && table && offsets && gtable && loss_scale,
                "s0_encode_bwd", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_encode_bwd", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_encode_bwd", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_encode_bwd", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const bool whole_sm = g_scatter_form ? g_scatter_form == 2 : nparts > 1;
    if (whole_sm)
        k_s0_scatter_walkers<<<scatter_walkers_grid(Mcap, nparts), kWholeSmThreads, 0, as_stream(stream)>>>(
            *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const uint8_t*>(denc_tiles), offsets,
            static_cast<float4*>(gtable), const_cast<float*>(loss_scale), part, nparts);
    else
        k_s0_encode_bwd<true, false><<<encode_bwd_grid<true, false>(Mcap, nparts), kTile, 0, as_stream(stream)>>>(
            *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const uint8_t*>(denc_tiles),
            static_cast<const TableEntry*>(table), offsets, static_cast<float4*>(gtable), const_cast<float*>(loss_scale), part, nparts);
    return check_launch("s0_encode_bwd");
}

/* TV-gradient launch: the same per-sample walk as the scatter, adding the TV gradient instead of the feature gradients */
int n2m_s0_tv(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
              const float* rays_d, const void* table, const int32_t* offsets, void* gtable, const float* loss_scale,
              n2m_stream_t stream) {
    N2M_REQUIRE(p && recs && counters && rays_o && rays_d && table && offsets && gtable && loss_scale, "s0_tv", "null pointer");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_tv", "Mcap must be a positive multiple of 128");
    if (!(p->lambda_tv > 0)) return 0;
    k_s0_encode_bwd<false, true><<<encode_bwd_grid<false, true>(Mcap, 1, kTvDeviceShare), kTile, 0, as_stream(stream)>>>(
        *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, nullptr, static_cast<const TableEntry*>(table), offsets,
        static_cast<float4*>(gtable), const_cast<float*>(loss_scale), 0, 1);
    return check_launch("s0_tv");
}

/* the random-point fallback of the TV calls that received no sample this step (see k_s0_tv_random); launch after n2m_s0_tv on the
 * same stream.  `dump` (nullable, [num_points,3]) is a test hook: run unconditionally with weight
 * lambda_tv and store the points. */
int n2m_s0_tv_random(const n2m_s0_params* p, const int32_t* counters, const void* table, const int32_t* offsets, void* gtable,
                     const float* loss_scale, uint32_t num_points, float* dump, n2m_stream_t stream) {
    N2M_REQUIRE(p && counters && table && offsets && gtable && loss_scale, "s0_tv_random", "null pointer");
    if (!(p->lambda_tv > 0) || num_points == 0) return 0;
    k_s0_tv_random<<<div_up(num_points, 128u), 128, 0, as_stream(stream)>>>(*p, counters, static_cast<const TableEntry*>(table), offsets,
                                                                            static_cast<float4*>(gtable), loss_scale, num_points, dump);
    return check_launch("s0_tv_random");
}

int n2m_s0_composite_loss(const n2m_s0_params* p, const void* out, const void* recs, const int32_t* rays,
                          const int32_t* counters, uint32_t N, uint32_t Mcap, const float* gt, const float* bg,
                          const float* loss_scale, void* dout, float* image, float* weights_sum, float* depth,
                          float* loss_out, const int32_t* active_rays, uint32_t part, uint32_t nparts, n2m_stream_t stream) {
    (void)Mcap;
    if (N == 0) return 0;
    N2M_REQUIRE(p && out && recs && rays && counters && gt && bg && loss_scale && dout && image && weights_sum && depth && loss_out,
                "s0_composite_loss", "null pointer");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_composite_loss", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const uint32_t e0 = part * kPartSlots / nparts, e1 = (part + 1) * kPartSlots / nparts;
    if (active_rays) {
        // the part's rays are known on the device only: the grid covers the largest part any n <= N can give, ceil(N / nparts)
        k_s0_composite_loss<true><<<div_up(div_up(N, nparts) * 32u, 128u), 128, 0, as_stream(stream)>>>(
            *p, static_cast<const float4*>(out), static_cast<const float4*>(recs), rays, counters, N, gt, bg, loss_scale,
            static_cast<float4*>(dout), image, weights_sum, depth, loss_out, active_rays, e0, e1);
        return check_launch("s0_composite_loss");
    }
    const uint32_t ray_lo = part_first_ray(N, e0), ray_hi = part_first_ray(N, e1);
    if (ray_hi == ray_lo) return 0;
    k_s0_composite_loss<false><<<div_up((ray_hi - ray_lo) * 32u, 128u), 128, 0, as_stream(stream)>>>(
        *p, static_cast<const float4*>(out), static_cast<const float4*>(recs), rays, counters, N, gt, bg, loss_scale,
        static_cast<float4*>(dout), image, weights_sum, depth, loss_out, nullptr, ray_lo, ray_hi);
    return check_launch("s0_composite_loss");
}

}  // extern "C"
