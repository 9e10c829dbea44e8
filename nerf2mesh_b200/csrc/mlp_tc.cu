// mlp_tc.cu -- the three tiny MLPs of NeRFNetwork (nerf/network.py:66-189) forward and backward on
// Hopper tensor cores: hand-written wgmma (m64nNk16, fp16 operands from shared memory, fp32 accumulation
// in registers), operands staged in shared memory as core-matrix tiles, first-layer activations brought
// in with one bulk async copy (TMA unit, cp.async.bulk) per 128-sample tile.
//
// Mapping: one warpgroup of 128 threads works on one 128-sample tile = the M dimension of every
// forward / dgrad GEMM (two m64 halves).  Layer epilogues (ReLU, masks) work on the accumulator
// fragments directly; the per-sample chain (sigmoid, exp, clamp, loss-side chain rule) runs one
// sample per thread, its few columns gathered from the fragments by warp shuffles (mlp_common.cuh).
// Weight gradients are GEMMs whose reduction dimension is the SAMPLE index; the same shared-memory
// activation / gradient tiles are re-read MN-major for them (wg.cuh).  In the backward kernel a
// warpgroup of its own issues them, and its accumulators stay resident in registers across all
// tiles a persistent CTA processes, then are flushed once with atomics.  Numerics follow torch.autocast(fp16): operands and layer outputs rounded to
// fp16, fp32 accumulation; gradients are carried loss-scaled in fp16 like GradScaler does.
#include "n2m_common.cuh"
#include "mlp_common.cuh"
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

__global__ void __launch_bounds__(256)
k_pack_weights(const float* __restrict__ P, uint8_t* __restrict__ wpack) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;      // one fp16 element
    if (i >= W_BYTES / 2) return;
    const uint32_t byte = i * 2;
    uint32_t base, rows; int which;
    if (byte < W_C2) { base = W_C1; rows = 64; which = 0; }
    else if (byte < W_C3) { base = W_C2; rows = 64; which = 1; }
    else if (byte < W_S1) { base = W_C3; rows = 16; which = 2; }
    else if (byte < W_S2) { base = W_S1; rows = 32; which = 3; }
    else if (byte < W_P1) { base = W_S2; rows = 16; which = 4; }
    else if (byte < W_P2) { base = W_P1; rows = 32; which = 5; }
    else { base = W_P2; rows = 16; which = 6; }
    // invert tile_off: byte offset -> (r, c)
    const uint32_t off = byte - base;
    const uint32_t chunk_bytes = rows * 16;
    const uint32_t ch = off / chunk_bytes, rem = off % chunk_bytes;
    const uint32_t r = rem / 16, c = ch * 8 + (rem % 16) / 2;
    float v = 0.f;
    switch (which) {
        case 0: { const int k = map_c1(c); if (k >= 0) v = P[P_C0 + r * 35 + k]; break; }
        case 1: v = P[P_C1 + r * 64 + c]; break;
        case 2: if (r < 6) v = P[P_C2 + r * 64 + c]; break;
        case 3: { const int k = map_s1(c); if (k >= 0) v = P[P_S0 + r * 19 + k]; break; }
        case 4: if (r < 1) v = P[P_S1 + c]; break;
        case 5: if (c < 6) v = P[P_P0 + r * 6 + c]; break;
        case 6: if (r < 3) v = P[P_P1 + r * 32 + c]; break;
    }
    *reinterpret_cast<__half*>(wpack + byte) = __float2half_rn(v);
}

// ================================================================================================
// forward
// ================================================================================================
// The specular hidden tile P1 aliases the sigma hidden tile S1, which is dead once sigma_net.1 has completed in round 2 (P1 is written in
// round 4, S1 again in round 1 of the next tile): 71 KB of shared memory per CTA, i.e. three CTAs per SM.
constexpr uint32_t F_W = 0, F_A = F_W + W_BYTES, F_H = F_A + kTileBytes, F_S1 = F_H + kTileBytes, F_AS2 = F_S1 + 8192, F_BYTES = F_AS2 + 4096;

__global__ void __launch_bounds__(128)
k_mlp_fwd(n2m_s0_params p, const uint8_t* __restrict__ enc_tiles, const int32_t* __restrict__ counters,
          const uint8_t* __restrict__ wpack, float4* __restrict__ out, float* __restrict__ spec_sq_sum,
          uint32_t part, uint32_t nparts) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bar_tma;
    __shared__ float red[4];
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    // samples [lo, hi) of this part: tiles [t0, t1); the boundary tiles are also computed by the neighbouring parts,
    // every part writes only its own rows
    const PartRange pr = part_range(counters, part, nparts);
    const uint32_t t0 = pr.lo / kTile, t1 = (pr.hi + kTile - 1) / kTile;
    if (pr.hi <= pr.lo || t0 + blockIdx.x >= t1) return;

    if (tid == 0) { wg::mbar_init(&bar_tma, 1); wg::mbar_init_fence(); }
    for (uint32_t i = tid; i < W_BYTES / 16; i += 128)
        reinterpret_cast<uint4*>(smem + F_W)[i] = __ldg(reinterpret_cast<const uint4*>(wpack) + i);
    {   // second K chunk of the specular input tile is always zero
        *reinterpret_cast<uint4*>(smem + F_AS2 + kChunk + tid * 16) = make_uint4(0, 0, 0, 0);
    }
    sync_before_mma();
    uint32_t ph_tma = 0;
    float spec_sq = 0.f;
    const uint32_t r = sample_row(tid);

    for (uint32_t tile = t0 + blockIdx.x; tile < t1; tile += gridDim.x) {
        if (tid == 0) bulk_g2s(smem + F_A, enc_tiles + (size_t)tile * kTileBytes, kTileBytes, &bar_tma);
        wg::mbar_wait(&bar_tma, ph_tma); ph_tma ^= 1;
        float sp[3];
        const float4 o = mlp_fwd_tile(smem + F_A, smem + F_W, smem + F_H, smem + F_S1, smem + F_S1, smem + F_AS2, p.shading_full != 0,
                                      tid, sp, sync_before_mma);
        const uint32_t j = tile * kTile + r;
        if (j >= pr.lo && j < pr.hi) {
            out[j] = o;
            spec_sq += sp[0] * sp[0] + sp[1] * sp[1] + sp[2] * sp[2];
        }
        sync_before_mma();          // all reads of this tile's smem are done before the next bulk copy
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) spec_sq += __shfl_xor_sync(0xffffffffu, spec_sq, o);
    if ((tid & 31) == 0) red[warp] = spec_sq;
    __syncthreads();
    if (tid == 0 && spec_sq_sum) atomicAdd(spec_sq_sum, red[0] + red[1] + red[2] + red[3]);
}

// ================================================================================================
// backward (forward recompute + dgrad + wgrad)
// ================================================================================================
// One CTA per SM of three warpgroups: two chain warpgroups (mlp_bwd_chain) work on alternating tiles of the CTA, each in its own
// tile set, and one weight-gradient warpgroup runs the wgrad steps (mlp_wgrad_step) of both, tile after tile in the CTA's order,
// holding the weight-gradient accumulators (WgradAcc, 120 fp32 registers per thread) across all of them.  While one chain waits on
// a round's MMAs, a TMA load or a barrier, the other chain and the wgrad GEMMs use the tensor core.
// Shared memory: 25,600 B of weights + 2 x 98,304 B tile sets = 222,208 B (+ 144 B of mbarriers).  Registers: 384 threads at
// __launch_bounds__(384, 1), at most 168 per thread.
// Hand-over per tile set (mbarriers, one phase per tile of the set; mbar_wait traps instead of hanging):
//   ready[s][k]  chain -> wgrad, 1 arrival (chain thread 0, after the barrier that publishes step k's tiles);
//                the wgrad warpgroup waits for phase `it` of its it-th tile of the set
//   rel[s][0]    wgrad -> chain, 128 arrivals, after step 0 (S1, P1 free): the chain waits for phase `it` of its own tile
//   rel[s][1]    wgrad -> chain, 128 arrivals, after step 3 (dH2 free): as rel[s][0]
//   rel[s][2]    wgrad -> chain, 128 arrivals, after step 4 (the tile set free): the chain waits for phase it - 1 before it
//                loads its next tile (parity (it & 1) ^ 1, which a fresh barrier passes at it = 0)
// A barrier never runs more than one phase ahead of its waiter: the chain's arrivals of tile it + 1 of a set follow its wait on
// rel[s][2] of tile it, which follows the wgrad warpgroup's last wait on that set's ready barriers of tile it.
// -Xptxas -v (CUDA 12.9, sm_90a): 159 registers, no stack frame, no spills, no wgmma serialisation advisories
// (tests/test_mlp_bwd_compile.py keeps it so).  On an H100 80GB HBM3 at 700 W, on bench.py's lego batch (2.85e5 samples):
// 80 us per launch against 180 us for the single-warpgroup kernel it replaces (profiles/mlp_bwd_time.py), 0.086 against
// 0.193 ms as bench.py's cold-L2 stage time, and the lego step 1.272 against 1.334 ms.
constexpr uint32_t kBwdChains = 2, kBwdThreads = 128 * (kBwdChains + 1);
constexpr uint32_t B_BYTES = B_SET + kBwdChains * T_BYTES;            // 222,208

// chain warpgroup c: make generic smem writes visible to the tensor core, meet the warpgroup's 128 threads at named barrier 1 + c.
// One code path serves both chains (two inlined copies would let the compiler hoist their common descriptor arithmetic above the
// role branch and hold it in registers through both); the register barrier id makes ptxas reserve all 16 named barriers.
struct SyncChain {
    uint32_t id;
    __device__ __forceinline__ void operator()() const {
        wg::fence_async_smem();
        asm volatile("bar.sync %0, 128;" :: "r"(id) : "memory");
    }
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(wg::smem_u32(bar)) : "memory");
}

struct BwdBars {
    uint64_t tma[kBwdChains], ready[kBwdChains][kWgradSteps], rel[kBwdChains][REL_SET + 1];
};

// chain side of the hand-over for the it-th tile of tile set s
struct ChainHandover {
    BwdBars* b; uint32_t s, it, tid;
    __device__ __forceinline__ void ready(int step) { if (tid == 0) mbar_arrive(&b->ready[s][step]); }
    __device__ __forceinline__ void released(int what) { wg::mbar_wait(&b->rel[s][what], it & 1); }
};

__device__ __forceinline__ void mlp_bwd_chain_role(uint32_t c, const n2m_s0_params& p, const uint8_t* __restrict__ enc_tiles,
                                                   const float4* __restrict__ dout, uint8_t* __restrict__ denc_tiles, const PartRange& pr,
                                                   uint32_t t0, uint32_t t1, uint32_t nparts, float spec_reg, uint8_t* smem, BwdBars* bars) {
    const uint32_t tid = threadIdx.x & 127u;
    const bool full = p.shading_full != 0;
    const uint32_t r = sample_row(tid);
    uint8_t* set = smem + B_SET + c * T_BYTES;
    const SyncChain sync{1 + c};
    uint32_t it = 0;
    for (uint32_t tile = t0 + blockIdx.x + c * gridDim.x; tile < t1; tile += kBwdChains * gridDim.x, ++it) {
        wg::mbar_wait(&bars->rel[c][REL_SET], (it & 1) ^ 1);        // the wgrad steps of this set's previous tile are complete
        if (tid == 0) bulk_g2s(set + T_A, enc_tiles + (size_t)tile * kTileBytes, kTileBytes, &bars->tma[c]);
        const uint32_t j = tile * kTile + r;
        float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool own = j >= pr.lo && j < pr.hi;
        if (own) dv = dout[j];
        wg::mbar_wait(&bars->tma[c], it & 1);
        ChainHandover h{bars, c, it, tid};
        mlp_bwd_chain(smem + B_W, set, dv, own, full, spec_reg, tid, sync, h, [&](const float (&d)[2][32]) {
            // the feature gradients -> the tile's rows of the denc tile image (global)
            uint8_t* img = denc_tiles + (size_t)tile * kTileBytes;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                    const uint32_t row = frag_row(hh, i, tid), jr = tile * kTile + row;
                    if (nparts == 1 || (jr >= pr.lo && jr < pr.hi))
                        *reinterpret_cast<uint32_t*>(img + wg::tile_off(row, frag_col(i, tid), kTile)) = pack2(d[hh][i], d[hh][i + 1]);
                }
        });
        // every chain warp's B5 MMAs have read dS1 (in S1) and dH1 before the next tile's recompute writes S1 and H1 and its
        // epilogues write dH
        sync();
    }
}

__global__ void __launch_bounds__(kBwdThreads, 1)
k_mlp_bwd(n2m_s0_params p, const uint8_t* __restrict__ enc_tiles, const float4* __restrict__ dout,
          const int32_t* __restrict__ counters, const uint8_t* __restrict__ wpack, uint8_t* __restrict__ denc_tiles,
          float* __restrict__ g_mlp, const float* __restrict__ loss_scale, uint32_t part, uint32_t nparts) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ BwdBars bars;
    const uint32_t tid = threadIdx.x, wgi = tid >> 7;
    // rows outside [lo, hi) of a boundary tile belong to a neighbouring part: zero upstream gradient (so they add
    // nothing to the weight gradients; their activations are whatever finite values the tile holds) and no store
    const PartRange pr = part_range(counters, part, nparts);
    const uint32_t M = pr.M;
    const uint32_t t0 = pr.lo / kTile, t1 = (pr.hi + kTile - 1) / kTile;
    if (pr.hi <= pr.lo || t0 + blockIdx.x >= t1) return;

    if (tid == 0) {
        for (uint32_t c = 0; c < kBwdChains; ++c) {
            wg::mbar_init(&bars.tma[c], 1);
            for (int k = 0; k < kWgradSteps; ++k) wg::mbar_init(&bars.ready[c][k], 1);
            for (int k = 0; k <= REL_SET; ++k) wg::mbar_init(&bars.rel[c][k], 128);
        }
        wg::mbar_init_fence();
    }
    for (uint32_t i = tid; i < W_BYTES / 16; i += kBwdThreads)
        reinterpret_cast<uint4*>(smem + B_W)[i] = __ldg(reinterpret_cast<const uint4*>(wpack) + i);
    if (wgi < kBwdChains) zero_narrow_tiles(smem + B_SET + wgi * T_BYTES, tid & 127u);
    sync_before_mma();
    const bool full = p.shading_full != 0;
    const float ls = loss_scale[0];
    const float spec_reg = (M > 0) ? 2.0f * p.lambda_specular / (float)M * ls : 0.f;   // d/dspec of lambda * mean_j sum_c spec^2

    if (wgi < kBwdChains) {
        mlp_bwd_chain_role(wgi, p, enc_tiles, dout, denc_tiles, pr, t0, t1, nparts, spec_reg, smem, &bars);
    } else {
        // weight-gradient warpgroup (the last one): the CTA's tiles in order, tile k in set k % kBwdChains
        WgradAcc wa;
        wa.zero();
        uint32_t k = 0;
        for (uint32_t tile = t0 + blockIdx.x; tile < t1; tile += gridDim.x, ++k) {
            const uint32_t s = k % kBwdChains, par = (k / kBwdChains) & 1;
            const uint8_t* set = smem + B_SET + s * T_BYTES;
#pragma unroll
            for (int step = 0; step < kWgradSteps; ++step) {
                wg::mbar_wait(&bars.ready[s][step], par);
                mlp_wgrad_step(step, set, wa);
                if (step == 0) mbar_arrive(&bars.rel[s][REL_S1P1]);
                if (step == 3) mbar_arrive(&bars.rel[s][REL_DH]);
                if (step == 4) mbar_arrive(&bars.rel[s][REL_SET]);
            }
        }
        flush_wgrad(wa, g_mlp, full, tid & 127u);
    }
}


}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

uint32_t n2m_s0_wpack_bytes(void) { return W_BYTES; }
uint32_t n2m_s0_mlp_param_count(void) { return P_COUNT; }

int n2m_s0_pack_weights(const float* mlp_params, void* wpack, n2m_stream_t stream) {
    N2M_REQUIRE(mlp_params && wpack, "s0_pack_weights", "null pointer");
    k_pack_weights<<<div_up(W_BYTES / 2, 256u), 256, 0, as_stream(stream)>>>(mlp_params, static_cast<uint8_t*>(wpack));
    return check_launch("s0_pack_weights");
}

static int num_sms() {
    static int n = 0;
    if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
    return n;
}


/* one-time function attributes (dynamic shared memory opt-in); safe to call repeatedly */
int n2m_s0_init(void) {
    cudaError_t e = cudaFuncSetAttribute(k_mlp_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)B_BYTES);
    if (e != cudaSuccess) return fail("s0_init", cudaGetErrorString(e));
    num_sms();
    return 0;
}

int n2m_s0_mlp_fwd_part(const n2m_s0_params* p, const void* enc_tiles, const int32_t* counters, uint32_t Mcap, const void* wpack,
                        void* out, float* spec_sq_sum, uint32_t part, uint32_t nparts, n2m_stream_t stream) {
    N2M_REQUIRE(p && enc_tiles && counters && wpack && out, "s0_mlp_fwd", "null pointer");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_mlp_fwd", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_mlp_fwd", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)(3 * num_sms()));          // 71 KB of shared memory: 3 CTAs per SM
    k_mlp_fwd<<<grid, 128, F_BYTES, as_stream(stream)>>>(*p, static_cast<const uint8_t*>(enc_tiles), counters,
                                                                static_cast<const uint8_t*>(wpack), static_cast<float4*>(out), spec_sq_sum,
                                                                part, nparts);
    return check_launch("s0_mlp_fwd");
}

int n2m_s0_mlp_fwd(const n2m_s0_params* p, const void* enc_tiles, const int32_t* counters, uint32_t Mcap, const void* wpack,
                   void* out, float* spec_sq_sum, n2m_stream_t stream) {
    return n2m_s0_mlp_fwd_part(p, enc_tiles, counters, Mcap, wpack, out, spec_sq_sum, 0, 1, stream);
}

int n2m_s0_mlp_bwd_part(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters, uint32_t Mcap,
                        const void* wpack, void* denc_tiles, float* g_mlp, const float* loss_scale, uint32_t part, uint32_t nparts,
                        n2m_stream_t stream) {
    N2M_REQUIRE(p && enc_tiles && dout && counters && wpack && denc_tiles && g_mlp && loss_scale, "s0_mlp_bwd", "null pointer");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_mlp_bwd", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_mlp_bwd", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)num_sms());
    k_mlp_bwd<<<grid, kBwdThreads, B_BYTES, as_stream(stream)>>>(*p, static_cast<const uint8_t*>(enc_tiles), static_cast<const float4*>(dout),
                                                         counters, static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(denc_tiles),
                                                         g_mlp, loss_scale, part, nparts);
    return check_launch("s0_mlp_bwd");
}

int n2m_s0_mlp_bwd(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters, uint32_t Mcap,
                   const void* wpack, void* denc_tiles, float* g_mlp, const float* loss_scale, n2m_stream_t stream) {
    return n2m_s0_mlp_bwd_part(p, enc_tiles, dout, counters, Mcap, wpack, denc_tiles, g_mlp, loss_scale, 0, 1, stream);
}

}  // extern "C"
