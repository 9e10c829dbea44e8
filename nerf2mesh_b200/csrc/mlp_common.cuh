// mlp_common.cuh -- what the tensor-core MLP forward kernels share (k_mlp_fwd in mlp_tc.cu, k_s0_fwd_fused in fused.cu,
// k_s1_geo_feat in texture.cu): packed-weight layout, flat parameter layout, epilogue helpers (wgmma register accumulators ->
// fp16 chunk-major smem tile, -> the per-sample values of the thread that owns the sample), and the forward of one tile
// (mlp_fwd_tile).  The backward's tile-set layout and routines live beside their one kernel, k_mlp_bwd (mlp_tc.cu).
#pragma once
#include "n2m_common.cuh"
#include "wg.cuh"
#include "s0_geom.cuh"

namespace n2m {
namespace {

constexpr uint32_t kChunk = kChunkBytes;     // 2048: one 8-column chunk of a 128-row tile (kTile / kTileBytes: s0_geom.cuh)

// ---- packed weights: fp16 chunk-major tiles [rows = out (padded), cols = in (padded)] --------------
constexpr uint32_t W_C1 = 0;                        // color_net.0   64 x 64  (in: enc tile cols)
constexpr uint32_t W_C2 = W_C1 + 64 * 64 * 2;       // color_net.1   64 x 64
constexpr uint32_t W_C3 = W_C2 + 64 * 64 * 2;       // color_net.2   16 x 64  (6 real outputs)
constexpr uint32_t W_S1 = W_C3 + 16 * 64 * 2;       // sigma_net.0   32 x 64
constexpr uint32_t W_S2 = W_S1 + 32 * 64 * 2;       // sigma_net.1   16 x 32  (1 real output)
constexpr uint32_t W_P1 = W_S2 + 16 * 32 * 2;       // specular_net.0 32 x 16 (6 real inputs)
constexpr uint32_t W_P2 = W_P1 + 32 * 16 * 2;       // specular_net.1 16 x 32 (3 real outputs)
constexpr uint32_t W_BYTES = W_P2 + 16 * 32 * 2;    // 25600

// flat fp32 parameter vector (reference nn.Linear layouts [out, in])
constexpr uint32_t P_S0 = 0, P_S1 = 608, P_C0 = 640, P_C1 = 2880, P_C2 = 6976, P_P0 = 7360, P_P1 = 7552, P_COUNT = 7648;

// enc tile column -> input index of the first-layer weights (-1: not an input of that net; the appearance-code columns
// kColCode.. of color_net.0 live outside the flat vector, see k_pack_code_weights)
__host__ __device__ __forceinline__ int map_c1(uint32_t k) { return k < 3 ? (int)k : (k >= 19 && k < 51) ? (int)(k - 16) : -1; }
__host__ __device__ __forceinline__ int map_s1(uint32_t k) { return k < 19 ? (int)k : -1; }

// ---- small device helpers ---------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(wg::smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(wg::smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(wg::smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float round_h(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float sigmoid_h(float pre_acc) {          // torch.sigmoid on an fp16 tensor
    const float x = round_h(pre_acc);
    return round_h(1.0f / (1.0f + __expf(-x)));
}

// everyone: make generic smem writes visible to the tensor core, then barrier
__device__ __forceinline__ void sync_before_mma() {
    wg::fence_async_smem();
    __syncthreads();
}

// Sample row of a 128-row tile owned by thread `tid` of the MLP warpgroup for the thread-per-sample parts (input gradients,
// sigmoid / exp epilogues, outputs): warp w, lane l -> 64 (l / 16) + 16 w + l % 16, i.e. the 32 rows whose accumulator
// fragments the warp holds, so that a sample's values move between lanes of one warp by shuffles.
__device__ __forceinline__ uint32_t sample_row(uint32_t tid) {
    const uint32_t w = tid >> 5, l = tid & 31;
    return 64u * (l >> 4) + 16u * w + (l & 15u);
}
// accumulator fragment (half h, register i) of lane l of warp w -> tile row / column (wg.cuh)
__device__ __forceinline__ uint32_t frag_row(uint32_t h, uint32_t i, uint32_t tid) {
    return 64u * h + 16u * (tid >> 5) + ((tid & 31u) >> 2) + 8u * ((i >> 1) & 1u);
}
__device__ __forceinline__ uint32_t frag_col(uint32_t i, uint32_t tid) { return 8u * (i >> 2) + 2u * (tid & 3u) + (i & 1u); }

// columns 0 .. NC-1 of this thread's sample row (sample_row) of a 128-row accumulator, gathered from the lanes holding them
template <int N, int NC>
__device__ __forceinline__ void row_cols(const float (&acc)[2][N / 2], float (&v)[8], uint32_t tid) {
    const uint32_t l = tid & 31u, h = l >> 4, r = l & 15u;
#pragma unroll
    for (int q = 0; q < (NC + 1) / 2; ++q) {
        const int src = 4 * (r & 7u) + q;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float x = __shfl_sync(0xffffffffu, acc[hh][2 * rr + e], src);
                    if (hh == (int)h && rr == (int)(r >> 3)) v[2 * q + e] = x;
                }
    }
}

// 128 x NCOL accumulator -> optional ReLU / mask -> fp16 128-row chunk-major tile.  mask_tile != nullptr: +0 where the fp16
// activation stored there is <= 0.  ReLU and the mask are applied on packed half2 values, bit-identical to the fp32 formulation
// (rounding to fp16 commutes with max(., 0) and with zeroing).  The mask is a select (bitwise AND with __hgt2_mask), as the
// backward of torch's relu (threshold_backward) is: a multiply by 0 would turn a masked gradient that overflowed fp16 into NaN.
// Shared-memory accesses by 32-bit shared-window address: one base register per tile and immediate offsets, where generic
// pointers would take a 64-bit address register pair per access of an unrolled epilogue.
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ __half2 bits_h2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }

template <int NCOL, bool RELU>
__device__ __forceinline__ void epi_store(const float (&acc)[2][NCOL / 2], uint8_t* tile, uint32_t tid, const uint8_t* mask_tile) {
    const __half2 zero2 = __float2half2_rn(0.f);
    const uint32_t t = wg::smem_u32(tile) + wg::tile_off(frag_row(0, 0, tid), frag_col(0, tid), kTile);
    const uint32_t m = mask_tile ? wg::smem_u32(mask_tile) + wg::tile_off(frag_row(0, 0, tid), frag_col(0, tid), kTile) : 0u;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int i = 0; i < NCOL / 2; i += 2) {
            // offset of this fragment pair from the thread's first one: a compile-time constant
            const uint32_t off = wg::tile_off(64u * hh + 8u * ((i >> 1) & 1), 8u * (i >> 2), kTile);
            __half2 h = __floats2half2_rn(acc[hh][i], acc[hh][i + 1]);
            if (RELU) h = __hmax2(h, zero2);
            uint32_t hb = h2_bits(h);
            if (mask_tile) hb &= __hgt2_mask(bits_h2(lds32(m + off)), zero2);
            sts32(t + off, hb);
        }
}

__device__ __forceinline__ void store_chunk(uint8_t* tile, uint32_t chunk, uint32_t r, const float (&v)[8]) {
    const uint32_t a = wg::smem_u32(tile) + chunk * kChunk + r * 16;
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                 :: "r"(a), "r"(pack2(v[0], v[1])), "r"(pack2(v[2], v[3])), "r"(pack2(v[4], v[5])), "r"(pack2(v[6], v[7])) : "memory");
}

__device__ __forceinline__ wg::Operand opK(const uint8_t* tile, uint32_t rows) { return wg::Operand{wg::smem_u32(tile), rows, false}; }
__device__ __forceinline__ wg::Operand opMN(const uint8_t* tile, uint32_t rows) { return wg::Operand{wg::smem_u32(tile), rows, true}; }

// ================================================================================================
// forward of one 128-sample tile of the MLPs on one warpgroup (wgmma, accumulators in registers)
// ================================================================================================
// The caller's `sync()` makes generic smem writes visible to the tensor core and meets all 128 threads at a barrier.
// Every round waits for its MMAs; a barrier follows the wait where the epilogue overwrites a tile other warps' MMAs read.

// returns (sigma, color); `sp` = specular colour (zero unless full shading)
template <class Sync>
__device__ __forceinline__ float4 mlp_fwd_tile(const uint8_t* sA, const uint8_t* sW, uint8_t* sH, uint8_t* sS1, uint8_t* sP1, uint8_t* sAs2,
                                               bool full, uint32_t tid, float (&sp)[3], Sync sync) {
    const uint32_t r = sample_row(tid);
    {   // round 1: first layers of color_net and sigma_net
        float c[2][32], s[2][16];
        wg::wgmma_fence();
        wg::gemm128<64, 4, false, false>(c, opK(sA, 128), opK(sW + W_C1, 64), false);
        wg::gemm128<32, 4, false, false>(s, opK(sA, 128), opK(sW + W_S1, 32), false);
        wg::commit(); wg::wait(c, s);
        epi_store<64, true>(c, sH, tid, nullptr);
        epi_store<32, true>(s, sS1, tid, nullptr);
    }
    sync();
    float sigma;
    {   // round 2: color_net.1, sigma_net.1
        float c[2][32], s[2][8], v[8];
        wg::wgmma_fence();
        wg::gemm128<64, 4, false, false>(c, opK(sH, 128), opK(sW + W_C2, 64), false);
        wg::gemm128<16, 2, false, false>(s, opK(sS1, 128), opK(sW + W_S2, 16), false);
        wg::commit(); wg::wait(c, s);
        row_cols<16, 1>(s, v, tid);
        sigma = __expf(round_h(v[0]));                   // trunc_exp forward (activation.py:5-11)
        sync();                                          // H2 overwrites H1: every warp's MMAs have read it
        epi_store<64, true>(c, sH, tid, nullptr);
    }
    sync();
    float feat[6];
    {   // round 3: color_net.2
        float c[2][8], v[8];
        wg::wgmma_fence();
        wg::gemm128<16, 4, false, false>(c, opK(sH, 128), opK(sW + W_C3, 16), false);
        wg::commit(); wg::wait(c);
        row_cols<16, 6>(c, v, tid);
#pragma unroll
        for (int i = 0; i < 6; ++i) feat[i] = sigmoid_h(v[i]);
    }
    float cr = feat[0], cg = feat[1], cb = feat[2];
    sp[0] = sp[1] = sp[2] = 0.f;
    if (full) {
        // specular input [dir(3), feat[3:6]]; dir sits in enc cols 51..53 = chunk 6, elements 3..5
        const uint4 dq = *reinterpret_cast<const uint4*>(sA + 6 * kChunk + r * 16);
        const __half2 d01 = *reinterpret_cast<const __half2*>(&dq.y);     // elements 2,3
        const __half2 d23 = *reinterpret_cast<const __half2*>(&dq.z);     // elements 4,5
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
        // color = (specular + diffuse).clamp(0, 1) on fp16 tensors (network.py:187)
        cr = fminf(fmaxf(round_h(sp[0] + cr), 0.f), 1.f);
        cg = fminf(fmaxf(round_h(sp[1] + cg), 0.f), 1.f);
        cb = fminf(fmaxf(round_h(sp[2] + cb), 0.f), 1.f);
    }
    return make_float4(sigma, cr, cg, cb);
}

}  // namespace

// dynamic shared memory opt-in of k_s0_fwd_fused (fused.cu); n2m_s0_init calls it with the attributes of the MLP kernels
cudaError_t fwd_fused_set_attributes();
}  // namespace n2m
