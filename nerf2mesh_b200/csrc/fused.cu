// fused.cu -- warp-specialised fused kernels of the stage-0 train path.
//
// k_s0_bwd_fused: the whole per-sample backward (autograd of the three MLPs on wgmma + the hash-grid scatter of
// gridencoder.cu:248-339) in ONE persistent kernel.  The stand-alone kernels (k_mlp_bwd: a latency-bound chain of ten dependent
// tensor-core rounds per tile, low occupancy; k_s0_encode_bwd: bound by the rate of spread red.global.add.v4.f32, no tensor or
// shared-memory use) leave each other's resources idle and run back to back.  Here one CTA per SM holds
//     warps 0-3  : the MLP backward, one 128-sample tile at a time: one warpgroup runs the chain of k_mlp_bwd and issues each
//                  weight-gradient step itself as soon as the chain has published its tiles (mlp_common.cuh, InlineWgrad);
//                  the feature gradients of a finished tile go to a double-buffered shared-memory image instead of HBM,
//     warps 4-19 : the scatter of the previous tile: warp = (32-sample group, level l mod 4), lane = sample, so consecutive lanes
//                  are consecutive samples of a ray and runs of same-cell lanes are merged before the RED as before (the scatter is
//                  instruction-bound at low warp counts -- see n2m_s0_set_fused_debug to time each role alone --
//                  hence sixteen warps, register budgets by setmaxnreg, lattice constants in smem),
// handing tiles over through two mbarrier pairs (full / empty).  The tensor chain of tile k+1 runs under the REDs of tile k, the
// `denc_tiles` round trip through HBM (2 x 128 B per sample) disappears, and the step loses one launch per part.
#include "n2m_common.cuh"
#include "s0_geom.cuh"
#include "mlp_common.cuh"
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

constexpr uint32_t kMlpThreads = 128, kScatWarps = 16, kFusedThreads = kMlpThreads + 32 * kScatWarps;     // 640
// register budget (setmaxnreg, multiples of 8).  The kernel starts with 96 registers per thread; setmaxnreg.inc can only take what
// setmaxnreg.dec of the other warps returned to the CTA pool: 512 x (96 - 72) = 12 288 >= 128 x (184 - 96) = 11 264.
// ptxas (CUDA 12.9, sm_90a) compiles this 640-thread kernel at 96 registers per thread whatever these budgets say, and the MLP
// warps' wgmma accumulators (120 weight-gradient registers beside a layer's 64) spill: 656 B of stack, 1,168 B of spill stores
// and 1,124 B of spill loads per thread, and one C7512 advisory (wgmma serialised for lack of registers; -Xptxas -v).  On an
// H100 80GB HBM3 at 700 W it takes 0.67 ms of a 1.33 ms lego step, where the two-launch backward (k_mlp_bwd + k_s0_encode_bwd)
// gives a 1.27 ms step; the two launches are therefore the default (stage0.py).
constexpr uint32_t kMlpRegs = 184, kScatRegs = 72;
static_assert(kScatWarps * 32 * (96 - kScatRegs) >= kMlpThreads * (kMlpRegs - 96), "setmaxnreg.inc must fit in what setmaxnreg.dec releases");
constexpr uint32_t D_CHUNKS = 7;                          // gradient columns 0..55 (cols 3..50 are used)
constexpr uint32_t D_BYTES = D_CHUNKS * kChunk;           // 14336
constexpr uint32_t FB_DENC = B_SET + T_BYTES;             // weights + one tile set
constexpr uint32_t FB_BYTES = FB_DENC + 2 * D_BYTES;      // 152576

__device__ __forceinline__ void bar_mlp() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// MLP warps only: make generic smem writes visible to the tensor core, meet at named barrier 1
__device__ __forceinline__ void sync_mlp() {
    wg::fence_async_smem();
    bar_mlp();
}
__device__ __forceinline__ void mbar_arrive1(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(wg::smem_u32(bar)) : "memory");
}

// per-level lattice constants, computed once per CTA into shared memory (level_geom + the dense / hashed index decision of
// corners_of): the scatter warps are instruction-bound, not RED-bound, at the warp counts a fused CTA can afford
struct LevelConst { float scale; uint32_t res, rows, row0, mx, my, mz, flags; };      // flags: bit 0 hashed, bit 1 rows is a power of two

__device__ __forceinline__ LevelConst make_level_const(const int32_t* __restrict__ offsets, uint32_t l, float S, uint32_t H) {
    const LevelGeom g = level_geom(offsets, l, S, H);
    LevelConst c;
    c.scale = g.scale; c.res = g.res; c.rows = g.rows; c.row0 = g.row0;
    const uint32_t s1 = g.res + 1;
    uint32_t stride = 1;
    c.mx = c.my = c.mz = 0;
    if (stride <= g.rows) { c.mx = stride; stride *= s1; }
    if (stride <= g.rows) { c.my = stride; stride *= s1; }
    if (stride <= g.rows) { c.mz = stride; stride *= s1; }
    c.flags = (stride > g.rows ? 1u : 0u) | (((g.rows & (g.rows - 1)) == 0) ? 2u : 0u);
    return c;
}

// ---- scatter of one tile by one warp: rows [32 * sg, 32 * sg + 32) of the tile, levels lq, lq + 4, lq + 8, lq + 12 ----
__device__ __forceinline__ void scatter_levels(const LevelConst* __restrict__ lc, uint32_t lq, const Sample& s, bool active,
                                               const uint8_t* __restrict__ row, float4* __restrict__ gtable, uint32_t lane, bool no_red) {
#pragma unroll 1
    for (uint32_t i = 0; i < 4; ++i) {
        const uint32_t l = lq + 4 * i;
        // this level's gradients from the shared-memory image: column kColDens + l, columns kColColor + 2l, + 2l + 1
        const uint32_t cd = kColDens + l, cc = kColColor + 2 * l;
        const float gd = active ? __half2float(*reinterpret_cast<const __half*>(row + (cd >> 3) * kChunk + (cd & 7) * 2)) : 0.f;
        const float g0 = active ? __half2float(*reinterpret_cast<const __half*>(row + (cc >> 3) * kChunk + (cc & 7) * 2)) : 0.f;
        const float g1 = active ? __half2float(*reinterpret_cast<const __half*>(row + ((cc + 1) >> 3) * kChunk + ((cc + 1) & 7) * 2)) : 0.f;
        const LevelConst L = lc[l];
        // corners (same expressions as corners_of in s0_geom.cuh)
        const float pu = s.u * L.scale + 0.5f, pv = s.v * L.scale + 0.5f, pw = s.w * L.scale + 0.5f;
        const float fu0 = floorf(pu), fv0 = floorf(pv), fw0 = floorf(pw);
        const uint32_t x0 = fu0, y0 = fv0, z0 = fw0;
        const float fx = pu - (float)x0, fy = pv - (float)y0, fz = pw - (float)z0;
        const bool hashed = (L.flags & 1u) != 0, pow2 = (L.flags & 2u) != 0;
        uint32_t xs[2], ys[2], zs[2];
        if (hashed) {
            xs[0] = x0;                 xs[1] = x0 + 1u;
            ys[0] = y0 * 2654435761u;   ys[1] = ys[0] + 2654435761u;
            zs[0] = z0 * 805459861u;    zs[1] = zs[0] + 805459861u;
        } else {
            xs[0] = x0 * L.mx;          xs[1] = xs[0] + L.mx;
            ys[0] = y0 * L.my;          ys[1] = ys[0] + L.my;
            zs[0] = z0 * L.mz;          zs[1] = zs[0] + L.mz;
        }
        const float wx[2] = {1 - fx, fx}, wy[2] = {1 - fy, fy}, wz[2] = {1 - fz, fz};
        uint32_t rowi[8];
        float vd[8], v0[8], v1[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ix = k & 1, iy = (k >> 1) & 1, iz = (k >> 2) & 1;
            const uint32_t raw = hashed ? (xs[ix] ^ ys[iy] ^ zs[iz]) : (xs[ix] + ys[iy] + zs[iz]);
            rowi[k] = wrap_row(raw, L.rows, pow2);
            const float w = wx[ix] * wy[iy] * wz[iz];
            vd[k] = w * gd; v0[k] = w * g0; v1[k] = w * g1;
        }
        float4* gt = gtable + L.row0;
        // runs of consecutive lanes in the same cell: sum them first, the last lane of a run issues the REDs
        const uint32_t key = active ? (x0 | (y0 << 10) | (z0 << 20)) : 0xffffffffu;
        const uint32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || key != prev);
        const bool merge = L.res < 1023u && __popc(heads) <= 20;
        bool issue = active;
        if (merge) {
            const uint32_t run_start = 31u - __clz(heads & (0xffffffffu >> (31u - lane)));
            // segmented inclusive scan; only as many doubling rounds as the longest run of this warp needs (the later ones add nothing)
            const uint32_t longest = __reduce_max_sync(0xffffffffu, lane - run_start);
#pragma unroll 1
            for (uint32_t o = 1; o <= longest; o <<= 1) {
                const bool take = lane >= run_start + o;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float a = __shfl_up_sync(0xffffffffu, vd[k], o), b = __shfl_up_sync(0xffffffffu, v0[k], o),
                                cq = __shfl_up_sync(0xffffffffu, v1[k], o);
                    if (take) { vd[k] += a; v0[k] += b; v1[k] += cq; }
                }
            }
            issue = active && (lane == 31 || ((heads >> (lane + 1)) & 1u));
        }
        if (issue && !no_red) {
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(gt + rowi[k], make_float4(vd[k], v0[k], v1[k], 0.f));
        }
        if (no_red && issue && vd[0] == 12345.678f) gt[rowi[0]].w = v0[3] + v1[5];       // keeps the arithmetic alive in the probe mode
    }
}

__global__ void __launch_bounds__(kFusedThreads, 1)
k_s0_bwd_fused(n2m_s0_params p, const uint8_t* __restrict__ enc_tiles, const float4* __restrict__ dout,
               const float4* __restrict__ recs, const int32_t* __restrict__ counters, const float* __restrict__ rays_o,
               const float* __restrict__ rays_d, const uint8_t* __restrict__ wpack, const int32_t* __restrict__ offsets,
               float4* __restrict__ gtable, float* __restrict__ g_mlp, float* __restrict__ loss_scale, uint32_t part, uint32_t nparts,
               uint32_t dbg) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bar_tma, bar_full[2], bar_empty[2];
    __shared__ LevelConst s_lc[kLevels];
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const PartRange pr = part_range(counters, part, nparts);
    const uint32_t M = pr.M;
    const uint32_t t0 = pr.lo / kTile, t1 = (pr.hi + kTile - 1) / kTile;
    if (pr.hi <= pr.lo || t0 + blockIdx.x >= t1) return;

    if (tid == 0) {
        wg::mbar_init(&bar_tma, 1);
        wg::mbar_init(&bar_full[0], 1); wg::mbar_init(&bar_full[1], 1);
        wg::mbar_init(&bar_empty[0], kScatWarps); wg::mbar_init(&bar_empty[1], kScatWarps);
        wg::mbar_init_fence();
    }
    if (tid >= kMlpThreads && tid < kMlpThreads + kLevels) s_lc[tid - kMlpThreads] = make_level_const(offsets, tid - kMlpThreads, p.S, p.base_res);
    for (uint32_t i = tid; i < W_BYTES / 16; i += kFusedThreads)
        reinterpret_cast<uint4*>(smem + B_W)[i] = __ldg(reinterpret_cast<const uint4*>(wpack) + i);
    uint8_t* set = smem + B_SET;
    uint8_t* sA = set + T_A;
    uint8_t* sD = smem + FB_DENC;
    if (tid < kMlpThreads) zero_narrow_tiles(set, tid);
    wg::fence_async_smem();
    __syncthreads();

    if (warp >= 4) {
        // =========================================== scatter warps ===========================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kScatRegs));
        const uint32_t sw = warp - 4, sg = sw & 3, lq = sw >> 2;
        uint32_t it = 0;
        for (uint32_t tile = t0 + blockIdx.x; tile < t1; tile += gridDim.x, ++it) {
            const uint32_t buf = it & 1, use = it >> 1;
            const uint32_t r = sg * 32 + lane;
            const uint32_t j = tile * kTile + r;
            Sample s;
            bool active = j >= pr.lo && j < pr.hi;
            if (active) {
                s = sample_of(recs[j], rays_o, rays_d, p);
                active = !((s.u < 0 || s.u > 1) || (s.v < 0 || s.v > 1) || (s.w < 0 || s.w > 1));
            } else {
                s.x = s.y = s.z = s.u = s.v = s.w = 0.5f; s.dx = s.dy = s.dz = 0.f;
            }
            wg::mbar_wait(&bar_full[buf], use & 1);
            const uint8_t* row = sD + buf * D_BYTES + r * 16;
            if (lq == 0 && active) {   // fp16 overflow of the loss-scaled gradients => GradScaler semantics: flag, the step is skipped
                bool bad = false;
#pragma unroll
                for (uint32_t ch = 0; ch < D_CHUNKS; ++ch) {
                    const uint4 q = *reinterpret_cast<const uint4*>(row + ch * kChunk);
                    const uint32_t ww[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&ww[i]));
                        const uint32_t col = 8 * ch + 2 * i;
                        if (col >= kColDens && col < kColDir) bad |= !isfinite(f.x);
                        if (col + 1 >= kColDens && col + 1 < kColDir) bad |= !isfinite(f.y);
                    }
                }
                if (bad) loss_scale[3] = 1.f;
            }
            scatter_levels(s_lc, lq, s, active, row, gtable, lane, (dbg & 1u) != 0);
            __syncwarp();
            if (lane == 0) mbar_arrive1(&bar_empty[buf]);          // the image of this tile is no longer needed by this warp
        }
    } else {
        // =========================================== MLP warps (k_mlp_bwd) ===========================================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kMlpRegs));
        uint32_t ph_tma = 0;
        const bool full = p.shading_full != 0;
        const float ls = loss_scale[0];
        const float spec_reg = (M > 0) ? 2.0f * p.lambda_specular / (float)M * ls : 0.f;
        const uint32_t r = sample_row(tid);
        WgradAcc wa;
        wa.zero();
        uint32_t it = 0;
        for (uint32_t tile = t0 + blockIdx.x; tile < t1; tile += gridDim.x, ++it) {
            const uint32_t buf = it & 1, use = it >> 1;
            if (dbg & 2u) {          // probe mode: no tensor-core work, hand a zero image over at once (measures the scatter warps alone)
                wg::mbar_wait(&bar_empty[buf], (use & 1) ^ 1);
#pragma unroll
                for (uint32_t ch = 0; ch < D_CHUNKS; ++ch) *reinterpret_cast<uint4*>(sD + buf * D_BYTES + ch * kChunk + tid * 16) = make_uint4(0x3c003c00u, 0x3c003c00u, 0x3c003c00u, 0x3c003c00u);
                bar_mlp();
                if (tid == 0) mbar_arrive1(&bar_full[buf]);
                continue;
            }
            if (tid == 0) bulk_g2s(sA, enc_tiles + (size_t)tile * kTileBytes, kTileBytes, &bar_tma);
            const uint32_t j = tile * kTile + r;
            float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
            const bool own = j >= pr.lo && j < pr.hi;
            if (own) dv = dout[j];
            wg::mbar_wait(&bar_tma, ph_tma); ph_tma ^= 1;
            InlineWgrad<void (*)()> wgrad{set, wa, sync_mlp};     // the chain and the weight-gradient steps on this one warpgroup
            mlp_bwd_chain(smem + B_W, set, dv, own, full, spec_reg, tid, sync_mlp, wgrad, [&](const float (&d)[2][32]) {
                // the scatter warps must have taken the buffer's previous contents (two tiles ago) before it is overwritten
                wg::mbar_wait(&bar_empty[buf], (use & 1) ^ 1);
                // the feature gradients -> the shared-memory gradient image (zeros for rows of other parts)
                uint8_t* dst = sD + buf * D_BYTES;
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                    for (int i = 0; i < 4 * (int)D_CHUNKS; i += 2) {
                        const uint32_t row = frag_row(hh, i, tid), jr = tile * kTile + row;
                        const bool mine = jr >= pr.lo && jr < pr.hi;
                        *reinterpret_cast<uint32_t*>(dst + wg::tile_off(row, frag_col(i, tid), kTile)) = mine ? pack2(d[hh][i], d[hh][i + 1]) : 0u;
                    }
            });
            sync_mlp();          // every row of the image is written, all reads of this tile's smem are done
            if (tid == 0) mbar_arrive1(&bar_full[buf]);
        }
        flush_wgrad(wa, g_mlp, full, tid);
    }
}


// ================================================================================================================================
// k_s0_fwd_fused: hash-grid gather + the three MLPs' forward in ONE persistent kernel (north_star's "fused march+encode+MLP"; the march
// itself stays a separate, prefetched launch: it does not depend on the parameters and runs under the previous step).
//   warps 0-3   : the MLP forward of k_mlp_fwd on the tile image in shared memory (one warpgroup issuing the wgmma rounds),
//   warps 4-7   : gather group 0, warps 8-11: gather group 1.  A group gathers one 128-sample tile (thread = sample, all 16 levels: the
//                 code of the stand-alone gather), writes the core-matrix-layout rows straight into ITS shared-memory buffer -- the image never
//                 makes the HBM round trip -- and has the TMA unit store a copy to `enc_tiles` for the backward pass (cp.async.bulk
//                 shared -> global, 16 KiB per instruction).
// Two CTAs per SM (86 KB of shared memory, 80 registers per thread each): 16 gather warps per SM keep the L1 / L2 gather pipe
// busy while two tensor-core chains run underneath.  Whole-batch only (nparts == 1): the bulk store writes complete tiles.
// ================================================================================================================================
constexpr uint32_t kFwdThreads = 384;
constexpr uint32_t FF_W = 0, FF_A0 = FF_W + W_BYTES, FF_A1 = FF_A0 + kTileBytes, FF_H = FF_A1 + kTileBytes, FF_S1 = FF_H + kTileBytes,
                   FF_AS2 = FF_S1 + 8192, FF_BYTES = FF_AS2 + 4096;          // 86,528 B

__device__ __forceinline__ void bar_group(uint32_t g) {          // named barriers 2 / 3 (immediate ids: a register id makes ptxas reserve all 16)
    if (g == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
    else asm volatile("bar.sync 3, 128;" ::: "memory");
}

__global__ void __launch_bounds__(kFwdThreads, 2)
k_s0_fwd_fused(n2m_s0_params p, const float4* __restrict__ recs, const int32_t* __restrict__ counters, const float* __restrict__ rays_o,
               const float* __restrict__ rays_d, const TableEntry* __restrict__ table, const int32_t* __restrict__ offsets,
               const uint8_t* __restrict__ wpack, uint8_t* __restrict__ enc_tiles, float4* __restrict__ out, float* __restrict__ spec_sq_sum) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bar_full[2], bar_empty[2];
    __shared__ float red[4];
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    const PartRange pr = part_range(counters, 0, 1);
    const uint32_t t1 = (pr.hi + kTile - 1) / kTile;
    if (pr.hi == 0 || blockIdx.x >= t1) return;
    const uint32_t my_tiles = (t1 - blockIdx.x + gridDim.x - 1) / gridDim.x;        // tiles blockIdx.x, + gridDim.x, ...

    if (tid == 0) {
        wg::mbar_init(&bar_full[0], 1); wg::mbar_init(&bar_full[1], 1);
        wg::mbar_init(&bar_empty[0], 1); wg::mbar_init(&bar_empty[1], 1);
        wg::mbar_init_fence();
    }
    for (uint32_t i = tid; i < W_BYTES / 16; i += kFwdThreads)
        reinterpret_cast<uint4*>(smem + FF_W)[i] = __ldg(reinterpret_cast<const uint4*>(wpack) + i);
    if (tid < 128) *reinterpret_cast<uint4*>(smem + FF_AS2 + kChunk + tid * 16) = make_uint4(0, 0, 0, 0);     // second K chunk of the specular input: zero
    wg::fence_async_smem();
    __syncthreads();

    if (warp >= 4) {
        // =========================================== gather groups ===========================================
        const uint32_t g = (warp - 4) >> 2, r = tid - 128 - g * 128;
        uint8_t* buf = smem + (g ? FF_A1 : FF_A0);
        uint32_t k = 0;
        for (uint32_t it = g; it < my_tiles; it += 2, ++k) {
            const uint32_t tile = blockIdx.x + it * gridDim.x;
            float feat[kTileCols];
            encode_fwd_features<false>(p, recs, rays_o, rays_d, table, offsets, pr, tile * kTile + r, feat);
            // the buffer is free once the TMA store of its previous image has read it and the MLP warps are done with that tile
            if (r == 0) {
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                wg::mbar_wait(&bar_empty[g], (k & 1) ^ 1);
            }
            bar_group(g);
            store_tile_row(buf, r, feat);
            wg::fence_async_smem();                  // generic-proxy writes -> visible to the tensor core and to the bulk copy engine
            bar_group(g);
            if (r == 0) {
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                             :: "l"(enc_tiles + (size_t)tile * kTileBytes), "r"(wg::smem_u32(buf)), "r"(kTileBytes) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                mbar_arrive1(&bar_full[g]);
            }
        }
        if (r == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");        // the last stores complete before the CTA exits
    } else {
        // =========================================== MLP warps (k_mlp_fwd) ===========================================
        float spec_sq = 0.f;
        const uint32_t r = sample_row(tid);
        for (uint32_t it = 0; it < my_tiles; ++it) {
            const uint32_t tile = blockIdx.x + it * gridDim.x, g = it & 1;
            const uint8_t* sA = smem + (g ? FF_A1 : FF_A0);
            wg::mbar_wait(&bar_full[g], (it >> 1) & 1);
            float sp[3];
            const float4 o = mlp_fwd_tile(sA, smem + FF_W, smem + FF_H, smem + FF_S1, smem + FF_S1, smem + FF_AS2, p.shading_full != 0,
                                          tid, sp, sync_mlp);
            const uint32_t j = tile * kTile + r;
            if (j < pr.hi) {
                out[j] = o;
                spec_sq += sp[0] * sp[0] + sp[1] * sp[1] + sp[2] * sp[2];
            }
            sync_mlp();                                   // every read of this tile's image is done
            if (tid == 0) mbar_arrive1(&bar_empty[g]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) spec_sq += __shfl_xor_sync(0xffffffffu, spec_sq, o);
        if ((tid & 31) == 0) red[warp] = spec_sq;
        bar_mlp();
        if (tid == 0 && spec_sq_sum) atomicAdd(spec_sq_sum, red[0] + red[1] + red[2] + red[3]);
    }
}

}  // namespace
}  // namespace n2m

using namespace n2m;

static uint32_t g_fused_dbg = 0;

static int fused_num_sms() {
    static int n = 0;
    if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
    return n;
}

extern "C" {

/* profiling hook: bit 0 = the scatter warps skip their REDs, bit 1 = the MLP warps skip the tensor-core rounds (results are then
 * meaningless; used to time each role of the fused backward alone) */
int n2m_s0_set_fused_debug(int mode) { g_fused_dbg = (uint32_t)mode; return 0; }

int n2m_s0_fused_init(void) {
    cudaError_t e = cudaFuncSetAttribute(k_s0_bwd_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FB_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_s0_fwd_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FF_BYTES);
    if (e != cudaSuccess) return fail("s0_fused_init", cudaGetErrorString(e));
    fused_num_sms();
    return 0;
}

/* MLP backward + hash-grid scatter of one part of the batch in one persistent launch (replaces n2m_s0_mlp_bwd_part followed by
 * n2m_s0_encode_bwd_part; the TV gradient stays with n2m_s0_tv) */
int n2m_s0_bwd_fused_part(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const void* recs, const int32_t* counters,
                          uint32_t Mcap, const float* rays_o, const float* rays_d, const void* wpack, const int32_t* offsets,
                          void* gtable, float* g_mlp, float* loss_scale, uint32_t part, uint32_t nparts, n2m_stream_t stream) {
    N2M_REQUIRE(p && enc_tiles && dout && recs && counters && rays_o && rays_d && wpack && offsets && gtable && g_mlp && loss_scale,
                "s0_bwd_fused", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_bwd_fused", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_bwd_fused", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_bwd_fused", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)fused_num_sms());
    k_s0_bwd_fused<<<grid, kFusedThreads, FB_BYTES, as_stream(stream)>>>(
        *p, static_cast<const uint8_t*>(enc_tiles), static_cast<const float4*>(dout), static_cast<const float4*>(recs), counters,
        rays_o, rays_d, static_cast<const uint8_t*>(wpack), offsets, static_cast<float4*>(gtable), g_mlp, loss_scale, part, nparts, g_fused_dbg);
    return check_launch("s0_bwd_fused");
}

/* hash-grid gather + MLP forward of the WHOLE batch in one persistent launch (replaces n2m_s0_encode_fwd followed by n2m_s0_mlp_fwd):
 * the tile images go from the gather warps to the tensor core through shared memory; a copy is stored to enc_tiles (TMA bulk store) for
 * the backward pass */
int n2m_s0_fwd_fused(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                     const float* rays_d, const void* table, const int32_t* offsets, const void* wpack, void* enc_tiles, void* out,
                     float* spec_sq_sum, n2m_stream_t stream) {
    N2M_REQUIRE(p && recs && counters && rays_o && rays_d && table && offsets && wpack && enc_tiles && out, "s0_fwd_fused", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_fwd_fused", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_fwd_fused", "Mcap must be a positive multiple of 128");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)(2 * fused_num_sms()));
    k_s0_fwd_fused<<<grid, kFwdThreads, FF_BYTES, as_stream(stream)>>>(
        *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const TableEntry*>(table), offsets,
        static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(enc_tiles), static_cast<float4*>(out), spec_sq_sum);
    return check_launch("s0_fwd_fused");
}

}  // extern "C"
