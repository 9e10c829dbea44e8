// fused.cu -- k_s0_fwd_fused: hash-grid gather + the three MLPs' forward of the stage-0 train path in ONE persistent,
// warp-specialised kernel (the march stays a separate, prefetched launch: it does not depend on the parameters and runs under the
// previous step).
//   warps 0-3   : the MLP forward of k_mlp_fwd on the tile image in shared memory (one warpgroup issuing the wgmma rounds),
//   warps 4-7   : gather group 0, warps 8-11: gather group 1.  A group gathers one 128-sample tile (thread = sample, all 16 levels: the
//                 code of the stand-alone gather), writes the core-matrix-layout rows straight into ITS shared-memory buffer -- the image never
//                 makes the HBM round trip -- and has the TMA unit store a copy to `enc_tiles` for the backward pass (cp.async.bulk
//                 shared -> global, 16 KiB per instruction).
// Two CTAs per SM (86 KB of shared memory, 80 registers per thread each): 16 gather warps per SM keep the L1 / L2 gather pipe
// busy while two tensor-core chains run underneath.  Whole-batch only (nparts == 1): the bulk store writes complete tiles.
#include "n2m_common.cuh"
#include "s0_geom.cuh"
#include "mlp_common.cuh"
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

__device__ __forceinline__ void bar_mlp() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// MLP warps only: make generic smem writes visible to the tensor core, meet at named barrier 1
__device__ __forceinline__ void sync_mlp() {
    wg::fence_async_smem();
    bar_mlp();
}
__device__ __forceinline__ void mbar_arrive1(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(wg::smem_u32(bar)) : "memory");
}

constexpr uint32_t kFwdThreads = 384;
constexpr uint32_t FF_W = 0, FF_A0 = FF_W + W_BYTES, FF_A1 = FF_A0 + kTileBytes, FF_H = FF_A1 + kTileBytes, FF_S1 = FF_H + kTileBytes,
                   FF_AS2 = FF_S1 + 8192, FF_BYTES = FF_AS2 + 4096;          // 86,528 B

__device__ __forceinline__ void bar_group(uint32_t g) {          // named barriers 2 / 3 (immediate ids: a register id makes ptxas reserve all 16)
    if (g == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
    else asm volatile("bar.sync 3, 128;" ::: "memory");
}

// CODES = false compiles the appearance-code columns out of the gather (include/n2m_b200_fused.h "Per-image appearance codes")
template <bool CODES>
__global__ void __launch_bounds__(kFwdThreads, 2)
k_s0_fwd_fused(n2m_s0_params p, const float4* __restrict__ recs, const int32_t* __restrict__ counters, const float* __restrict__ rays_o,
               const float* __restrict__ rays_d, const TableEntry* __restrict__ table, const int32_t* __restrict__ offsets,
               const uint8_t* __restrict__ wpack, uint8_t* __restrict__ enc_tiles, float4* __restrict__ out, float* __restrict__ spec_sq_sum,
               const float* __restrict__ codes, const int32_t* __restrict__ ray_img) {
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
            encode_fwd_features<false>(p, recs, rays_o, rays_d, table, offsets, pr, tile * kTile + r, feat, CODES ? codes : nullptr,
                                       CODES ? ray_img : nullptr);
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

cudaError_t fwd_fused_set_attributes() {
    const cudaError_t e = cudaFuncSetAttribute(k_s0_fwd_fused<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FF_BYTES);
    return e != cudaSuccess ? e : cudaFuncSetAttribute(k_s0_fwd_fused<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FF_BYTES);
}
}  // namespace n2m

using namespace n2m;

extern "C" {

/* hash-grid gather + MLP forward of the WHOLE batch in one persistent launch (replaces n2m_s0_encode_fwd followed by n2m_s0_mlp_fwd):
 * the tile images go from the gather warps to the tensor core through shared memory; a copy is stored to enc_tiles (TMA bulk store) for
 * the backward pass */
int n2m_s0_fwd_fused(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                     const float* rays_d, const void* table, const int32_t* offsets, const void* wpack, void* enc_tiles, void* out,
                     float* spec_sq_sum, n2m_stream_t stream) {
    N2M_REQUIRE(p && recs && counters && rays_o && rays_d && table && offsets && wpack && enc_tiles && out, "s0_fwd_fused", "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_fwd_fused", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_fwd_fused", "Mcap must be a positive multiple of 128");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)(2 * num_sms()));
    k_s0_fwd_fused<false><<<grid, kFwdThreads, FF_BYTES, as_stream(stream)>>>(
        *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const TableEntry*>(table), offsets,
        static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(enc_tiles), static_cast<float4*>(out), spec_sq_sum, nullptr, nullptr);
    return check_launch("s0_fwd_fused");
}

int n2m_s0_fwd_fused_codes(const n2m_s0_params* p, const void* recs, const int32_t* counters, uint32_t Mcap, const float* rays_o,
                           const float* rays_d, const void* table, const int32_t* offsets, const float* codes, const int32_t* ray_img,
                           const void* wpack, void* enc_tiles, void* out, float* spec_sq_sum, n2m_stream_t stream) {
    N2M_REQUIRE(p && p->ind_dim <= kMaxIndDim, "s0_fwd_fused_codes", "ind_dim must be at most 10");
    if (p->ind_dim == 0)
        return n2m_s0_fwd_fused(p, recs, counters, Mcap, rays_o, rays_d, table, offsets, wpack, enc_tiles, out, spec_sq_sum, stream);
    N2M_REQUIRE(recs && counters && rays_o && rays_d && table && offsets && wpack && enc_tiles && out && codes, "s0_fwd_fused_codes",
                "null pointer");
    N2M_REQUIRE(p->num_levels == kLevels, "s0_fwd_fused_codes", "fused path supports num_levels == 16");
    N2M_REQUIRE(Mcap % kTile == 0 && Mcap > 0, "s0_fwd_fused_codes", "Mcap must be a positive multiple of 128");
    const uint32_t grid = min(Mcap / kTile, (uint32_t)(2 * num_sms()));
    k_s0_fwd_fused<true><<<grid, kFwdThreads, FF_BYTES, as_stream(stream)>>>(
        *p, static_cast<const float4*>(recs), counters, rays_o, rays_d, static_cast<const TableEntry*>(table), offsets,
        static_cast<const uint8_t*>(wpack), static_cast<uint8_t*>(enc_tiles), static_cast<float4*>(out), spec_sq_sum, codes, ray_img);
    return check_launch("s0_fwd_fused_codes");
}

}  // extern "C"
