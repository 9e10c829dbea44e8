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

// appearance-code columns of color_net.0: ind[o * D + j] -> W_C1 (o, 54 + j)
__global__ void __launch_bounds__(256)
k_pack_code_weights(const float* __restrict__ ind, uint32_t D, uint8_t* __restrict__ wpack) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 64 * D) return;
    const uint32_t o = i / D, j = i % D;
    *reinterpret_cast<__half*>(wpack + W_C1 + wg::tile_off(o, kColCode + j, 64)) = __float2half_rn(ind[i]);
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
            // shading 'specular' (network.py:183-184, evaluation only): the colour is the specular term alone
            out[j] = p.shading_full == 2 ? make_float4(o.x, sp[0], sp[1], sp[2]) : o;
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

// ---- shared memory: the packed weights, then one tile set per chain warpgroup -------------------------------------------------
// A tile set, 48 chunks: A | H2 | H1 | S1 | P1 | As2 | dH | dO | dOs | dO2.  dS1 and dP1 are written in place over S1 and P1 (the
// B1 epilogue reads each mask element and writes the gradient element of the same thread and offset), once the weight-gradient
// GEMMs that read S1 and P1 are complete.  dH holds dH2, then dH1.  The wgrad GEMMs' 64-column MN-major reads of the narrower
// tiles S1, P1 and As2 run on into the next tiles of the set; the rows they produce there are never used.
constexpr uint32_t B_W = 0;
constexpr uint32_t T_A = 0, T_H2 = 16384, T_H1 = 32768, T_S1 = 49152, T_P1 = 57344, T_AS2 = 65536, T_DH = 69632, T_DO = 86016,
                   T_DOS = 90112, T_DO2 = 94208, T_BYTES = 98304;
constexpr uint32_t B_SET = B_W + W_BYTES;            // first tile set
constexpr uint32_t kBwdChains = 2, kBwdThreads = 128 * (kBwdChains + 1);
constexpr uint32_t B_BYTES = B_SET + kBwdChains * T_BYTES;            // 222,208

// constant-zero parts of the narrow backward tiles (their second K chunk, and unused columns of the first), and the specular
// tiles As2, P1 / dP1 and dO2, which only full shading writes
__device__ __forceinline__ void zero_narrow_tiles(uint8_t* set, uint32_t tid) {
    const uint4 z = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(set + T_AS2 + kChunk + tid * 16) = z;
    *reinterpret_cast<uint4*>(set + T_DO + kChunk + tid * 16) = z;
    *reinterpret_cast<uint4*>(set + T_DOS + kChunk + tid * 16) = z;
    *reinterpret_cast<uint4*>(set + T_DO2 + kChunk + tid * 16) = z;
    *reinterpret_cast<uint4*>(set + T_DO2 + tid * 16) = z;
    *reinterpret_cast<uint4*>(set + T_AS2 + tid * 16) = z;
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) *reinterpret_cast<uint4*>(set + T_P1 + ch * kChunk + tid * 16) = z;
}

// weight-gradient accumulators of one CTA, summed over all its tiles (rows = input feature of the layer, m64 fragments)
struct WgradAcc {
    float c1[32], c2[32], c3[8], s1[16], s2[8], p2[8], p1[16];
    __device__ __forceinline__ void zero() {
#pragma unroll
        for (int i = 0; i < 32; ++i) { c1[i] = 0.f; c2[i] = 0.f; }
#pragma unroll
        for (int i = 0; i < 16; ++i) { s1[i] = 0.f; p1[i] = 0.f; }
#pragma unroll
        for (int i = 0; i < 8; ++i) { c3[i] = 0.f; s2[i] = 0.f; p2[i] = 0.f; }
    }
};

// ---- the backward of one tile in two roles ---------------------------------------------------------------------------------
// The chain (mlp_bwd_chain) runs the forward recompute, the per-sample chain rule and the dgrad GEMMs down to the encoding
// gradient; it holds one round's accumulators at a time.  The weight gradients (mlp_wgrad_step) are GEMMs over the tile's
// activation and gradient tiles, in five steps, each issued once the chain has written the tiles it reads:
//     step 0 (after the chain rule): S1^T dOs, P1^T dO2                -> then S1 / P1 may be overwritten (dS1 / dP1 in place)
//     step 1 (after B1): A^T dS1, As2^T dP1
//     step 2 (after B2): H2^T dO
//     step 3 (after B3): H1^T dH2                                       -> then dH may be overwritten (dH1)
//     step 4 (after B4): A^T dH1                                        -> then the whole tile set is free
// The chain calls hooks.ready(step) after the barrier that publishes a step's tiles, and hooks.released(what) before it overwrites
// a tile that step 0 / step 3 read; released() returns once the weight-gradient MMAs of every warp that read the tile are
// complete.  Both are mbarrier arrivals / waits between the chain and the weight-gradient warpgroup (ChainHandover below).
constexpr int kWgradSteps = 5;
enum { REL_S1P1 = 0, REL_DH = 1, REL_SET = 2 };

// weight-gradient step `step` of the tile in tile set `set`, issued and completed by the calling warpgroup
// The specular GEMMs are issued in both shading modes (a wgmma under a branch makes ptxas fence the accumulator registers of the
// whole group); without full shading their operand tiles stay zero, and nothing reads what they accumulate.
__device__ __forceinline__ void mlp_wgrad_step(int step, const uint8_t* set, WgradAcc& wa) {
    const uint8_t* sA = set + T_A; const uint8_t* sH2 = set + T_H2; const uint8_t* sH1 = set + T_H1;
    const uint8_t* sS1 = set + T_S1; const uint8_t* sP1 = set + T_P1; const uint8_t* sAs2 = set + T_AS2;
    const uint8_t* sdS1 = set + T_S1; const uint8_t* sdP1 = set + T_P1; const uint8_t* sdH = set + T_DH;
    const uint8_t* sdO = set + T_DO; const uint8_t* sdOs = set + T_DOS; const uint8_t* sdO2 = set + T_DO2;
    wg::wgmma_fence();
    switch (step) {
        case 0:
            wg::gemm64<16, 8, true, true>(wa.s2, opMN(sS1, 128), opMN(sdOs, 128), true);             // rows 0..31: S1^T dOs
            wg::gemm64<16, 8, true, true>(wa.p2, opMN(sP1, 128), opMN(sdO2, 128), true);             // rows 0..31: P1^T dO2
            wg::commit(); wg::wait(wa.s2, wa.p2);
            break;
        case 1:
            wg::gemm64<32, 8, true, true>(wa.s1, opMN(sA, 128), opMN(sdS1, 128), true);              // rows 0..63: A^T dS1
            wg::gemm64<32, 8, true, true>(wa.p1, opMN(sAs2, 128), opMN(sdP1, 128), true);            // rows 0..5: As2^T dP1
            wg::commit(); wg::wait(wa.s1, wa.p1);
            break;
        case 2:
            wg::gemm64<16, 8, true, true>(wa.c3, opMN(sH2, 128), opMN(sdO, 128), true);              // rows 0..63: H2^T dO
            wg::commit(); wg::wait(wa.c3);
            break;
        case 3:
            wg::gemm64<64, 8, true, true>(wa.c2, opMN(sH1, 128), opMN(sdH, 128), true);              // rows 0..63: H1^T dH2
            wg::commit(); wg::wait(wa.c2);
            break;
        default:
            wg::gemm64<64, 8, true, true>(wa.c1, opMN(sA, 128), opMN(sdH, 128), true);               // rows 0..63: A^T dH1
            wg::commit(); wg::wait(wa.c1);
            break;
    }
}

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

// chain role of the backward of one tile in tile set `set` (forward recompute, dgrad).  dv: upstream gradient of this thread's
// sample (zero if not owned); emit(d_enc) receives the 128 x 64 accumulator of the encoding gradient.  `tid`: 0..127 in the
// chain's warpgroup; `sync()` makes generic smem writes visible to the tensor core and meets the warpgroup's 128 threads.
template <class Emit>
__device__ __forceinline__ void mlp_bwd_chain(const uint8_t* sW, uint8_t* set, float4 dv, bool own, bool full, float spec_reg,
                                              uint32_t tid, SyncChain sync, ChainHandover& hooks, Emit emit) {
    uint8_t* sA = set + T_A; uint8_t* sH2 = set + T_H2; uint8_t* sH1 = set + T_H1; uint8_t* sS1 = set + T_S1;
    uint8_t* sP1 = set + T_P1; uint8_t* sAs2 = set + T_AS2;
    uint8_t* sdH = set + T_DH; uint8_t* sdS1 = set + T_S1; uint8_t* sdP1 = set + T_P1; uint8_t* sdO = set + T_DO;
    uint8_t* sdOs = set + T_DOS; uint8_t* sdO2 = set + T_DO2;
    const uint32_t r = sample_row(tid);

    // ---------------- forward recompute (one layer per round, the rounds of the reference numerics) ----------------
    {
        float c[2][32];
        wg::wgmma_fence();
        wg::gemm128<64, 4, false, false>(c, opK(sA, 128), opK(sW + W_C1, 64), false);
        wg::commit(); wg::wait(c);
        epi_store<64, true>(c, sH1, tid, nullptr);
    }
    {
        float s[2][16];
        wg::wgmma_fence();
        wg::gemm128<32, 4, false, false>(s, opK(sA, 128), opK(sW + W_S1, 32), false);
        wg::commit(); wg::wait(s);
        epi_store<32, true>(s, sS1, tid, nullptr);
    }
    sync();
    float h_sig;
    {
        float s[2][8], v[8];
        wg::wgmma_fence();
        wg::gemm128<16, 2, false, false>(s, opK(sS1, 128), opK(sW + W_S2, 16), false);
        wg::commit(); wg::wait(s);
        row_cols<16, 1>(s, v, tid);
        h_sig = round_h(v[0]);
    }
    {
        float c[2][32];
        wg::wgmma_fence();
        wg::gemm128<64, 4, false, false>(c, opK(sH1, 128), opK(sW + W_C2, 64), false);
        wg::commit(); wg::wait(c);
        epi_store<64, true>(c, sH2, tid, nullptr);
    }
    sync();
    float feat[6];
    {
        float c[2][8], v[8];
        wg::wgmma_fence();
        wg::gemm128<16, 4, false, false>(c, opK(sH2, 128), opK(sW + W_C3, 16), false);
        wg::commit(); wg::wait(c);
        row_cols<16, 6>(c, v, tid);
#pragma unroll
        for (int i = 0; i < 6; ++i) feat[i] = sigmoid_h(v[i]);
    }
    float sp[3] = {0.f, 0.f, 0.f};
    if (full) {
        const uint4 dq = *reinterpret_cast<const uint4*>(sA + 6 * kChunk + r * 16);
        const __half2 d01 = *reinterpret_cast<const __half2*>(&dq.y);
        const __half2 d23 = *reinterpret_cast<const __half2*>(&dq.z);
        const float in[8] = {__high2float(d01), __low2float(d23), __high2float(d23), feat[3], feat[4], feat[5], 0.f, 0.f};
        store_chunk(sAs2, 0, r, in);
        sync();
        {
            float c[2][16];
            wg::wgmma_fence();
            wg::gemm128<32, 1, false, false>(c, opK(sAs2, 128), opK(sW + W_P1, 32), false);
            wg::commit(); wg::wait(c);
            epi_store<32, true>(c, sP1, tid, nullptr);
        }
        sync();
        float c[2][8], v[8];
        wg::wgmma_fence();
        wg::gemm128<16, 2, false, false>(c, opK(sP1, 128), opK(sW + W_P2, 16), false);
        wg::commit(); wg::wait(c);
        row_cols<16, 3>(c, v, tid);
#pragma unroll
        for (int i = 0; i < 3; ++i) sp[i] = sigmoid_h(v[i]);
    }

    // ---------------- output-side chain rule (thread-per-sample) ----------------
    float dfeat[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    {
        const float dcol[3] = {dv.y, dv.z, dv.w};
        float dO2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float g = dcol[c];
            if (full) {
                const float cs = round_h(sp[c] + feat[c]);
                if (!(cs >= 0.f && cs <= 1.f)) g = 0.f;            // clamp(0,1) backward
                const float dsp = own ? g + spec_reg * sp[c] : 0.f;
                dO2[c] = dsp * sp[c] * (1.0f - sp[c]);            // sigmoid backward
            }
            dfeat[c] = g;
        }
        float dOs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        dOs[0] = dv.x * __expf(fminf(fmaxf(h_sig, -15.f), 15.f));   // trunc_exp backward (activation.py:13-17)
        store_chunk(sdOs, 0, r, dOs);
        if (full) store_chunk(sdO2, 0, r, dO2);
    }
    sync();
    hooks.ready(0);

    // ---------------- B1: specular_net.1 / sigma_net.1 dgrad ----------------
    {
        float d[2][16], e[2][16];
        wg::wgmma_fence();
        wg::gemm128<32, 1, false, true>(d, opK(sdOs, 128), opMN(sW + W_S2, 16), false);           // dS1 (pre-mask)
        wg::gemm128<32, 1, false, true>(e, opK(sdO2, 128), opMN(sW + W_P2, 16), false);           // dP1 (pre-mask)
        wg::commit(); wg::wait(d, e);
        hooks.released(REL_S1P1);                        // dS1 / dP1 overwrite S1 / P1
        epi_store<32, false>(d, sdS1, tid, sS1);
        if (full) epi_store<32, false>(e, sdP1, tid, sP1);
    }
    sync();
    hooks.ready(1);

    // ---------------- B2: specular_net.0 dgrad ----------------
    {
        float e[2][8], v[8];
        if (full) {
            wg::wgmma_fence();
            wg::gemm128<16, 2, false, true>(e, opK(sdP1, 128), opMN(sW + W_P1, 32), false);       // d As2
            wg::commit(); wg::wait(e);
            row_cols<16, 6>(e, v, tid);
            dfeat[3] = v[3]; dfeat[4] = v[4]; dfeat[5] = v[5];
        }
        float dO[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 6; ++i) dO[i] = dfeat[i] * feat[i] * (1.0f - feat[i]);
        store_chunk(sdO, 0, r, dO);
    }
    sync();
    hooks.ready(2);

    // ---------------- B3: color_net.2 dgrad ----------------
    {
        float d[2][32];
        wg::wgmma_fence();
        wg::gemm128<64, 1, false, true>(d, opK(sdO, 128), opMN(sW + W_C3, 16), false);            // dH2 (pre-mask)
        wg::commit(); wg::wait(d);
        epi_store<64, false>(d, sdH, tid, sH2);
    }
    sync();
    hooks.ready(3);

    // ---------------- B4: color_net.1 dgrad ----------------
    {
        float d[2][32];
        wg::wgmma_fence();
        wg::gemm128<64, 4, false, true>(d, opK(sdH, 128), opMN(sW + W_C2, 64), false);            // dH1 (pre-mask)
        wg::commit(); wg::wait(d);
        sync();                                          // dH1 overwrites dH2: every warp's MMAs have read it
        hooks.released(REL_DH);
        epi_store<64, false>(d, sdH, tid, sH1);
    }
    sync();
    hooks.ready(4);

    // ---------------- B5: encoding dgrad (sigma_net.0 + color_net.0) ----------------
    {
        float d[2][32];
        wg::wgmma_fence();
        wg::gemm128<64, 2, false, true>(d, opK(sdS1, 128), opMN(sW + W_S1, 32), false);           // d enc  = dS1 W_s1
        wg::gemm128<64, 4, false, true>(d, opK(sdH, 128), opMN(sW + W_C1, 64), true);             // d enc += dH1 W_c1
        wg::commit(); wg::wait(d);
        emit(d);
    }
}

// apply f(row, col, value) to every element of an m64 accumulator fragment
template <int N, class F>
__device__ __forceinline__ void for_frag64(const float (&d)[N / 2], uint32_t tid, F f) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) f(frag_row(0, i, tid), frag_col(i, tid), d[i]);
}

// the weight-gradient accumulators of a CTA -> g_mlp (flat reference layout), atomically; with g_ind the appearance-code columns
// 54..53+D of W_C1 -> g_ind[o * D + (f - 54)] (include/n2m_b200_fused.h "Per-image appearance codes")
__device__ __forceinline__ void flush_wgrad(const WgradAcc& wa, float* g_mlp, float* g_ind, uint32_t D, bool full, uint32_t tid) {
    for_frag64<64>(wa.c1, tid, [&](uint32_t f, uint32_t o, float v) {
        const int k = map_c1(f);
        if (k >= 0) atomicAdd(g_mlp + P_C0 + o * 35 + k, v);
        else if (g_ind && f >= kColCode && f < kColCode + D) atomicAdd(g_ind + o * D + (f - kColCode), v);
    });
    for_frag64<64>(wa.c2, tid, [&](uint32_t f, uint32_t o, float v) { atomicAdd(g_mlp + P_C1 + o * 64 + f, v); });
    for_frag64<16>(wa.c3, tid, [&](uint32_t f, uint32_t o, float v) { if (o < 6) atomicAdd(g_mlp + P_C2 + o * 64 + f, v); });
    for_frag64<32>(wa.s1, tid, [&](uint32_t f, uint32_t o, float v) { const int k = map_s1(f); if (k >= 0) atomicAdd(g_mlp + P_S0 + o * 19 + k, v); });
    for_frag64<16>(wa.s2, tid, [&](uint32_t f, uint32_t o, float v) { if (f < 32 && o == 0) atomicAdd(g_mlp + P_S1 + f, v); });
    if (full) {
        for_frag64<16>(wa.p2, tid, [&](uint32_t f, uint32_t o, float v) { if (f < 32 && o < 3) atomicAdd(g_mlp + P_P1 + o * 32 + f, v); });
        for_frag64<32>(wa.p1, tid, [&](uint32_t f, uint32_t o, float v) { if (f < 6) atomicAdd(g_mlp + P_P0 + o * 6 + f, v); });
    }
}

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
          float* __restrict__ g_mlp, const float* __restrict__ loss_scale, uint32_t part, uint32_t nparts, float* __restrict__ g_ind) {
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
        flush_wgrad(wa, g_mlp, g_ind, p.ind_dim, full, tid & 127u);
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

/* one-time function attributes (dynamic shared memory opt-in) of every stage-0 kernel; safe to call repeatedly */
int n2m_s0_init(void) {
    cudaError_t e = cudaFuncSetAttribute(k_mlp_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_mlp_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)B_BYTES);
    if (e == cudaSuccess) e = fwd_fused_set_attributes();
    if (e != cudaSuccess) return fail("s0_init", cudaGetErrorString(e));
    num_sms();
    return 0;
}

int n2m_s0_mlp_fwd(const n2m_s0_params* p, const void* enc_tiles, const int32_t* counters, uint32_t Mcap, const void* wpack,
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

int n2m_s0_mlp_bwd(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters, uint32_t Mcap,
                   const void* wpack, void* denc_tiles, float* g_mlp, const float* loss_scale, uint32_t part, uint32_t nparts,
                   n2m_stream_t stream) {
    N2M_REQUIRE(p && enc_tiles && dout && counters && wpack && denc_tiles && g_mlp && loss_scale, "s0_mlp_bwd", "null pointer");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_mlp_bwd", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_mlp_bwd", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)num_sms());
    k_mlp_bwd<<<grid, kBwdThreads, B_BYTES, as_stream(stream)>>>(*p, static_cast<const uint8_t*>(enc_tiles), static_cast<const float4*>(dout),
                                                         counters, static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(denc_tiles),
                                                         g_mlp, loss_scale, part, nparts, nullptr);
    return check_launch("s0_mlp_bwd");
}

int n2m_s0_mlp_bwd_codes(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters, uint32_t Mcap,
                         const void* wpack, void* denc_tiles, float* g_mlp, float* g_ind, const float* loss_scale, uint32_t part,
                         uint32_t nparts, n2m_stream_t stream) {
    N2M_REQUIRE(p && p->ind_dim <= kMaxIndDim, "s0_mlp_bwd_codes", "ind_dim must be at most 10");
    N2M_REQUIRE(p->ind_dim == 0 || g_ind, "s0_mlp_bwd_codes", "null pointer");
    N2M_REQUIRE(enc_tiles && dout && counters && wpack && denc_tiles && g_mlp && loss_scale, "s0_mlp_bwd_codes", "null pointer");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_mlp_bwd_codes", "Mcap must be a positive multiple of 128");
    N2M_REQUIRE(valid_parts(part, nparts), "s0_mlp_bwd_codes", "nparts must be 1, 2, 4 or 8 and part < nparts");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)num_sms());
    k_mlp_bwd<<<grid, kBwdThreads, B_BYTES, as_stream(stream)>>>(*p, static_cast<const uint8_t*>(enc_tiles), static_cast<const float4*>(dout),
                                                         counters, static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(denc_tiles),
                                                         g_mlp, loss_scale, part, nparts, p->ind_dim ? g_ind : nullptr);
    return check_launch("s0_mlp_bwd_codes");
}

int n2m_s0_pack_code_weights(const float* ind, uint32_t ind_dim, void* wpack, n2m_stream_t stream) {
    N2M_REQUIRE(ind_dim <= kMaxIndDim, "s0_pack_code_weights", "ind_dim must be at most 10");
    if (ind_dim == 0) return 0;
    N2M_REQUIRE(ind && wpack, "s0_pack_code_weights", "null pointer");
    k_pack_code_weights<<<div_up(64u * ind_dim, 256u), 256, 0, as_stream(stream)>>>(ind, ind_dim, static_cast<uint8_t*>(wpack));
    return check_launch("s0_pack_code_weights");
}

}  // extern "C"
