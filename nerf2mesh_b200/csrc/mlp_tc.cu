// mlp_tc.cu -- the three tiny MLPs of NeRFNetwork (nerf/network.py:66-189) forward and backward on
// Hopper tensor cores: hand-written wgmma (m64nNk16, fp16 operands from shared memory, fp32 accumulation
// in registers), operands staged in shared memory as core-matrix tiles, first-layer activations brought
// in with one bulk async copy (TMA unit, cp.async.bulk) per 128-sample tile.
//
// Mapping: one CTA = one warpgroup of 128 threads = one 128-sample tile = the M dimension of every
// forward / dgrad GEMM (two m64 halves).  Layer epilogues (ReLU, masks) work on the accumulator
// fragments directly; the per-sample chain (sigmoid, exp, clamp, loss-side chain rule) runs one
// sample per thread, its few columns gathered from the fragments by warp shuffles (mlp_common.cuh).
// Weight gradients are GEMMs whose reduction dimension is the SAMPLE index; the same shared-memory
// activation / gradient tiles are re-read MN-major for them (wg.cuh) and the accumulators stay
// resident in registers across all tiles a persistent CTA processes, then are flushed once with
// atomics.  Numerics follow torch.autocast(fp16): operands and layer outputs rounded to
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
// One CTA per SM: 255 registers per thread (-Xptxas -v, CUDA 12.9: 84 B of spills, and ptxas serialises some wgmma issues around
// register use, C7519).  On an H100 SXM 80 GB at 700 W the kernel takes 0.19 ms of the 1.33 ms lego step (bench.py, stage times).
__global__ void __launch_bounds__(128, 1)
k_mlp_bwd(n2m_s0_params p, const uint8_t* __restrict__ enc_tiles, const float4* __restrict__ dout,
          const int32_t* __restrict__ counters, const uint8_t* __restrict__ wpack, uint8_t* __restrict__ denc_tiles,
          float* __restrict__ g_mlp, const float* __restrict__ loss_scale, uint32_t part, uint32_t nparts) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bar_tma;
    const uint32_t tid = threadIdx.x;
    // rows outside [lo, hi) of a boundary tile belong to a neighbouring part: zero upstream gradient (so they add
    // nothing to the weight gradients; their activations are whatever finite values the tile holds) and no store
    const PartRange pr = part_range(counters, part, nparts);
    const uint32_t M = pr.M;
    const uint32_t t0 = pr.lo / kTile, t1 = (pr.hi + kTile - 1) / kTile;
    if (pr.hi <= pr.lo || t0 + blockIdx.x >= t1) return;

    if (tid == 0) { wg::mbar_init(&bar_tma, 1); wg::mbar_init_fence(); }
    for (uint32_t i = tid; i < W_BYTES / 16; i += 128)
        reinterpret_cast<uint4*>(smem + B_W)[i] = __ldg(reinterpret_cast<const uint4*>(wpack) + i);
    zero_narrow_tiles(smem, tid);
    sync_before_mma();
    uint32_t ph_tma = 0;
    const bool full = p.shading_full != 0;
    const float ls = loss_scale[0];
    const float spec_reg = (M > 0) ? 2.0f * p.lambda_specular / (float)M * ls : 0.f;   // d/dspec of lambda * mean_j sum_c spec^2
    const uint32_t r = sample_row(tid);
    WgradAcc wa;
    wa.zero();

    for (uint32_t tile = t0 + blockIdx.x; tile < t1; tile += gridDim.x) {
        if (tid == 0) bulk_g2s(smem + B_ACT + A_A, enc_tiles + (size_t)tile * kTileBytes, kTileBytes, &bar_tma);
        const uint32_t j = tile * kTile + r;
        float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool own = j >= pr.lo && j < pr.hi;
        if (own) dv = dout[j];
        wg::mbar_wait(&bar_tma, ph_tma); ph_tma ^= 1;
        mlp_bwd_tile(smem, dv, own, full, spec_reg, tid, wa, sync_before_mma, [&](const float (&d)[2][32]) {
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
        sync_before_mma();
    }
    flush_wgrad(wa, g_mlp, full, tid);
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
    k_mlp_bwd<<<grid, 128, B_BYTES, as_stream(stream)>>>(*p, static_cast<const uint8_t*>(enc_tiles), static_cast<const float4*>(dout),
                                                         counters, static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(denc_tiles),
                                                         g_mlp, loss_scale, part, nparts);
    return check_launch("s0_mlp_bwd");
}

int n2m_s0_mlp_bwd(const n2m_s0_params* p, const void* enc_tiles, const void* dout, const int32_t* counters, uint32_t Mcap,
                   const void* wpack, void* denc_tiles, float* g_mlp, const float* loss_scale, n2m_stream_t stream) {
    return n2m_s0_mlp_bwd_part(p, enc_tiles, dout, counters, Mcap, wpack, denc_tiles, g_mlp, loss_scale, 0, 1, stream);
}

}  // extern "C"
