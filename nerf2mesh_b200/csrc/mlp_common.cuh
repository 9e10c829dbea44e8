// mlp_common.cuh -- constants and device helpers shared by the tensor-core MLP kernels (mlp_tc.cu) and the fused kernels (fused.cu):
// packed-weight layout, flat parameter layout, epilogue helpers (wgmma register accumulators -> fp16 chunk-major smem tile,
// -> the per-sample values of the thread that owns the sample).
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

// enc tile column -> input index of the first-layer weights (-1: not an input of that net)
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

// 128 x NCOL accumulator -> optional ReLU / mask -> fp16 128-row chunk-major tile.  mask_tile != nullptr: zero where the fp16
// activation stored there is <= 0.  ReLU and the mask are applied on packed half2 values, bit-identical to the fp32 formulation
// (rounding to fp16 commutes with max(., 0) and with zeroing).
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
            if (mask_tile) h = __hmul2(h, __hgt2(bits_h2(lds32(m + off)), zero2));
            sts32(t + off, h2_bits(h));
        }
}

__device__ __forceinline__ void store_chunk(uint8_t* tile, uint32_t chunk, uint32_t r, const float (&v)[8]) {
    const uint32_t a = wg::smem_u32(tile) + chunk * kChunk + r * 16;
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                 :: "r"(a), "r"(pack2(v[0], v[1])), "r"(pack2(v[2], v[3])), "r"(pack2(v[4], v[5])), "r"(pack2(v[6], v[7])) : "memory");
}

__device__ __forceinline__ wg::Operand opK(const uint8_t* tile, uint32_t rows) { return wg::Operand{wg::smem_u32(tile), rows, false}; }
__device__ __forceinline__ wg::Operand opMN(const uint8_t* tile, uint32_t rows) { return wg::Operand{wg::smem_u32(tile), rows, true}; }

// ---- backward shared memory: the packed weights, then one or more tile sets (one per 128-sample tile in flight) --------------
// A tile set, 48 chunks: A | H2 | H1 | S1 | P1 | As2 | dH | dO | dOs | dO2.  dS1 and dP1 are written in place over S1 and P1 (the
// B1 epilogue reads each mask element and writes the gradient element of the same thread and offset), once the weight-gradient
// GEMMs that read S1 and P1 are complete.  dH holds dH2, then dH1.  The wgrad GEMMs' 64-column MN-major reads of the narrower
// tiles S1, P1 and As2 run on into the next tiles of the set; the rows they produce there are never used.
constexpr uint32_t B_W = 0;
constexpr uint32_t T_A = 0, T_H2 = 16384, T_H1 = 32768, T_S1 = 49152, T_P1 = 57344, T_AS2 = 65536, T_DH = 69632, T_DO = 86016,
                   T_DOS = 90112, T_DO2 = 94208, T_BYTES = 98304;
constexpr uint32_t B_SET = B_W + W_BYTES;            // first tile set

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

// ================================================================================================
// one 128-sample tile of the MLPs on one warpgroup (wgmma, accumulators in registers)
// ================================================================================================
// The caller's `sync()` makes generic smem writes visible to the tensor core and meets all 128 threads at a barrier.
// Every round waits for its MMAs; a barrier follows the wait where the epilogue overwrites a tile other warps' MMAs read.

// forward: returns (sigma, color); `sp` = specular colour (zero unless full shading)
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
// complete.  In the warp-specialised kernel ready() / released() are mbarrier arrivals / waits between the chain and a
// weight-gradient warpgroup; a warpgroup that runs both roles issues the step from ready() and meets at its barrier in released().
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

// both roles on one warpgroup: each weight-gradient step runs as soon as its tiles are published.  wgmma.wait_group waits for the
// calling warp's share of the MMAs only, so before the chain overwrites a tile a step read (the B1 epilogue writes dS1 / dP1 over
// S1 / P1 in every column of its warp's rows), the warpgroup meets at its barrier: every warp has then waited for its step MMAs.
template <class Sync>
struct InlineWgrad {
    const uint8_t* set; WgradAcc& wa; Sync sync;
    __device__ __forceinline__ void ready(int step) { mlp_wgrad_step(step, set, wa); }
    __device__ __forceinline__ void released(int) { sync(); }
};

// chain role of the backward of one tile in tile set `set` (forward recompute, dgrad).  dv: upstream gradient of this thread's
// sample (zero if not owned); emit(d_enc) receives the 128 x 64 accumulator of the encoding gradient.  `tid`: 0..127 in the
// chain's warpgroup; `sync()` makes generic smem writes visible to the tensor core and meets the warpgroup's 128 threads.
template <class Sync, class Hooks, class Emit>
__device__ __forceinline__ void mlp_bwd_chain(const uint8_t* sW, uint8_t* set, float4 dv, bool own, bool full, float spec_reg,
                                              uint32_t tid, Sync sync, Hooks& hooks, Emit emit) {
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

// the weight-gradient accumulators of a CTA -> g_mlp (flat reference layout), atomically
__device__ __forceinline__ void flush_wgrad(const WgradAcc& wa, float* g_mlp, bool full, uint32_t tid) {
    for_frag64<64>(wa.c1, tid, [&](uint32_t f, uint32_t o, float v) { const int k = map_c1(f); if (k >= 0) atomicAdd(g_mlp + P_C0 + o * 35 + k, v); });
    for_frag64<64>(wa.c2, tid, [&](uint32_t f, uint32_t o, float v) { atomicAdd(g_mlp + P_C1 + o * 64 + f, v); });
    for_frag64<16>(wa.c3, tid, [&](uint32_t f, uint32_t o, float v) { if (o < 6) atomicAdd(g_mlp + P_C2 + o * 64 + f, v); });
    for_frag64<32>(wa.s1, tid, [&](uint32_t f, uint32_t o, float v) { const int k = map_s1(f); if (k >= 0) atomicAdd(g_mlp + P_S0 + o * 19 + k, v); });
    for_frag64<16>(wa.s2, tid, [&](uint32_t f, uint32_t o, float v) { if (f < 32 && o == 0) atomicAdd(g_mlp + P_S1 + f, v); });
    if (full) {
        for_frag64<16>(wa.p2, tid, [&](uint32_t f, uint32_t o, float v) { if (f < 32 && o < 3) atomicAdd(g_mlp + P_P1 + o * 32 + f, v); });
        for_frag64<32>(wa.p1, tid, [&](uint32_t f, uint32_t o, float v) { if (f < 6) atomicAdd(g_mlp + P_P0 + o * 6 + f, v); });
    }
}

}  // namespace
}  // namespace n2m
