// dp.cu -- data-parallel optimizer step fused with its collective, over NVLink peer memory.
//
// With rays sharded across W GPUs every rank ends its backward pass with a full-size gradient table
// (98 MB).  The library baseline (NCCL all-reduce of 98 MB, then a full Adam on every rank) moves the whole table over
// NVLink and streams it through HBM on every rank.  This file does it as ONE pass:
//
//   reduce-scatter : rank r reads rows [r R/W, (r+1) R/W) of every peer's gradient table straight from the
//                    peers' HBM (P2P loads over NVLink / NVSwitch) and sums them,
//   optimizer      : applies GradScaler-unscale + Adam to that 1/W slice only (moments and fp32 colour
//                    masters exist only for the slice it owns: the Adam stream shrinks W-fold),
//   all-gather     : writes the updated 8-byte table entries into every peer's table (P2P stores),
//
// so the NVLink payload per rank is (W-1)/W * (16 + 8) bytes per row instead of 2 * (W-1)/W * 16 for the
// ring all-reduce, and it overlaps with the arithmetic row by row.  Two system-scope flag barriers
// (k_dp_barrier) order it against the backward pass before and the forward pass after; gradient tables
// are double-buffered per step parity so the table being reduced by peers is never the one being zeroed.
#include "n2m_common.cuh"
#include "../../include/n2m_b200_fused.h"
#include <cuda.h>
#include <cstdlib>

namespace n2m {
namespace {

constexpr int kMaxWorld = 8;
constexpr float kBeta1 = 0.9f, kBeta2 = 0.999f;

struct __align__(8) TableEntry { float d; __half2 c; };

struct DpCtx {
    uint32_t world, rank;
    uint32_t rows, n_mlp;
    float4* gtab[kMaxWorld][2];        // [peer][parity] gradient tables (peer pointers mapped through CUDA IPC)
    TableEntry* table[kMaxWorld];      // [peer] working tables
    float* gmlp[kMaxWorld][2];         // [peer][parity] MLP gradient vectors
    float* opt[kMaxWorld];             // [peer] optimizer state blocks (found_inf at [3])
    uint32_t* flags[kMaxWorld];        // [peer] flag arrays: slots 0..7 barrier epochs, slots 8+parity "this rank saw inf"
    uint32_t* epoch;                   // local barrier epoch counter (device)
};

// system-scope flag barrier: every rank bumps its slot in every peer's flag array, then waits until all
// slots of its own array have reached the new epoch.
__global__ void k_dp_barrier(const DpCtx* __restrict__ ctx) {
    const uint32_t p = threadIdx.x;
    const uint32_t W = ctx->world, r = ctx->rank;
    const uint32_t e = *ctx->epoch + 1;
    if (p < W) {
        __threadfence_system();
        volatile uint32_t* remote = ctx->flags[p] + r;
        *remote = e;
        __threadfence_system();
        volatile uint32_t* mine = ctx->flags[r] + p;
        uint64_t spins = 0;
        while ((int32_t)(*mine - e) < 0) {
            if (++spins > (1ull << 31)) __trap();          // a missing peer traps instead of hanging forever
        }
    }
    __syncthreads();
    if (p == 0) *ctx->epoch = e;
}

__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, float lr_over_bc1, float bc2s, float eps) {
    m = kBeta1 * m + (1.f - kBeta1) * g;
    v = kBeta2 * v + (1.f - kBeta2) * g * g;
    const float denom = __fdiv_rn(__fsqrt_rn(v), bc2s) + eps;
    return p - lr_over_bc1 * __fdiv_rn(m, denom);
}

// publish this rank's found_inf for the step (parity-indexed slot: rewritten only two steps later, so a slow peer
// can still read it after this rank has moved on)
__global__ void k_dp_publish_inf(const DpCtx* __restrict__ ctx, uint32_t parity, const float* __restrict__ st) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    ctx->flags[ctx->rank][kMaxWorld + parity] = st[3] != 0.f ? 1u : 0u;
    __threadfence_system();
}

// found_inf = OR over ranks (every rank computes the same value), then the usual per-step constants
__global__ void k_dp_prep(const DpCtx* __restrict__ ctx, uint32_t parity, float* __restrict__ st) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float inf = 0.f;
    for (uint32_t p = 0; p < ctx->world; ++p)
        if (*reinterpret_cast<volatile uint32_t*>(ctx->flags[p] + kMaxWorld + parity) != 0u) inf = 1.f;
    st[3] = inf;
    if (inf == 0.f) st[2] += 1.f;
    const float t = fmaxf(st[2], 1.f);
    st[5] = 1.f - powf(kBeta1, t);
    st[6] = sqrtf(1.f - powf(kBeta2, t));
    st[7] = 1.f / (st[0] * (float)ctx->world);          // unscale and average over ranks in one factor
}

constexpr int kRowsPerThread = 2;

// rows owned by one rank: ceil(rows / world) rounded up to a multiple of 4, so that the float2 colour moments that
// follow the `per` density moments in the slice-sized m / v arrays stay 8-byte aligned (764983 rows at world 8 is odd)
__host__ __device__ __forceinline__ uint32_t slice_rows(uint32_t rows, uint32_t world) {
    return ((rows + world - 1) / world + 3u) & ~3u;
}

__device__ __forceinline__ void mc_st_entry(TableEntry* mc, TableEntry e) {
    const float lo = e.d, hi = __uint_as_float(*reinterpret_cast<const uint32_t*>(&e.c));
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" :: "l"(mc), "f"(lo), "f"(hi) : "memory");
}


// reduce-scatter + Adam + all-gather on this rank's row slice.  All 2 x W peer loads of a thread are issued before the first use (a
// 128-bit load over NVLink has microseconds of latency; the slice is streamed with 16 of them in flight per thread).
__global__ void __launch_bounds__(256)
k_dp_adam_tables(const DpCtx* __restrict__ ctx, uint32_t parity, float2* __restrict__ cmaster,
                 float* __restrict__ m, float* __restrict__ v, const float* __restrict__ st, float eps) {
    const uint32_t W = ctx->world, r = ctx->rank, rows = ctx->rows;
    const uint32_t per = slice_rows(rows, W);
    const uint32_t lo = min(rows, r * per), hi = min(rows, lo + per);
    const bool skip = st[3] != 0.f;
    const float inv = st[7];
    const float lr1 = __fdiv_rn(st[4], st[5]), bc2s = st[6];
    // slice-local optimizer state: index i - lo
    float2* mc_p = reinterpret_cast<float2*>(m + per);
    float2* vc_p = reinterpret_cast<float2*>(v + per);
    const uint32_t i0 = lo + blockIdx.x * (256 * kRowsPerThread) + threadIdx.x;

    float4 q[kRowsPerThread][kMaxWorld];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
        const uint32_t i = i0 + j * 256;
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
            if (p < (int)W && i < hi) q[j][p] = __ldcv(ctx->gtab[p][parity] + i);       // peer HBM over NVLink (L2-bypassing on the reader)
    }
    if (skip) return;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
        const uint32_t i = i0 + j * 256;
        if (i >= hi) continue;
        float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
            if (p < (int)W) { gx += q[j][p].x; gy += q[j][p].y; gz += q[j][p].z; }
        gx *= inv; gy *= inv; gz *= inv;
        const uint32_t k = i - lo;
        float md = m[k], vd = v[k];
        float2 mc = mc_p[k], vc = vc_p[k];
        if (gx == 0.f && gy == 0.f && gz == 0.f && md == 0.f && vd == 0.f && mc.x == 0.f && mc.y == 0.f && vc.x == 0.f && vc.y == 0.f)
            continue;
        TableEntry e = ctx->table[r][i];
        float2 pc = cmaster[k];
        e.d = adam_update(e.d, gx, md, vd, lr1, bc2s, eps);
        pc.x = adam_update(pc.x, gy, mc.x, vc.x, lr1, bc2s, eps);
        pc.y = adam_update(pc.y, gz, mc.y, vc.y, lr1, bc2s, eps);
        e.c = __floats2half2_rn(pc.x, pc.y);
        cmaster[k] = pc;
        m[k] = md; v[k] = vd; mc_p[k] = mc; vc_p[k] = vc;
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
            if (p < (int)W) ctx->table[p][i] = e;                                       // all-gather: P2P stores
    }
}

// ---- NVLS variant: the same reduce-scatter + Adam + all-gather with the reduction done INSIDE the NVSwitch -----------------------
// `mc_gtab` / `mc_table` are multicast addresses (one virtual address mapped onto the same buffer of every rank, created by
// torch.distributed._symmetric_memory): multimem.ld_reduce returns the sum of the W ranks' copies of a 16-byte row in one load -- the
// switch adds them, each GPU's link carries 1/W of the traffic of the peer-load version -- and multimem.st stores the refreshed 8-byte
// table entry into all W tables with one store.  NVLink bytes per rank per step: 16 B x rows / W in, 8 B x rows / W out, instead of
// (W-1)/W x 16 B x rows in and (W-1)/W x 8 B x rows out.
__device__ __forceinline__ float4 mc_ld_reduce_add(const float4* mc) {
    float4 r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
    return r;
}
constexpr int kMcRowsPerThread = 4;

__global__ void __launch_bounds__(256)
k_dp_adam_tables_mc(const DpCtx* __restrict__ ctx, const float4* __restrict__ mc_gtab, TableEntry* __restrict__ mc_table,
                    float2* __restrict__ cmaster, float* __restrict__ m, float* __restrict__ v, const float* __restrict__ st, float eps) {
    const uint32_t W = ctx->world, r = ctx->rank, rows = ctx->rows;
    const uint32_t per = slice_rows(rows, W);
    const uint32_t lo = min(rows, r * per), hi = min(rows, lo + per);
    const bool skip = st[3] != 0.f;
    const float inv = st[7];
    const float lr1 = __fdiv_rn(st[4], st[5]), bc2s = st[6];
    float2* mc_p = reinterpret_cast<float2*>(m + per);
    float2* vc_p = reinterpret_cast<float2*>(v + per);
    const uint32_t i0 = lo + blockIdx.x * (256 * kMcRowsPerThread) + threadIdx.x;
    float4 g[kMcRowsPerThread]; float md[kMcRowsPerThread], vd[kMcRowsPerThread];
    float2 mcv[kMcRowsPerThread], vcv[kMcRowsPerThread], pc[kMcRowsPerThread];
    TableEntry e[kMcRowsPerThread];
#pragma unroll
    for (int j = 0; j < kMcRowsPerThread; ++j) {          // all loads first: the in-switch reductions and the local state stream together
        const uint32_t i = i0 + j * 256;
        if (i < hi) {
            g[j] = mc_ld_reduce_add(mc_gtab + i);
            if (!skip) {
                const uint32_t k = i - lo;
                md[j] = m[k]; vd[j] = v[k]; mcv[j] = mc_p[k]; vcv[j] = vc_p[k]; e[j] = ctx->table[r][i]; pc[j] = cmaster[k];
            }
        }
    }
    if (skip) return;
#pragma unroll
    for (int j = 0; j < kMcRowsPerThread; ++j) {
        const uint32_t i = i0 + j * 256;
        if (i >= hi) continue;
        const uint32_t k = i - lo;
        const float gx = g[j].x * inv, gy = g[j].y * inv, gz = g[j].z * inv;
        if (gx == 0.f && gy == 0.f && gz == 0.f && md[j] == 0.f && vd[j] == 0.f && mcv[j].x == 0.f && mcv[j].y == 0.f && vcv[j].x == 0.f &&
            vcv[j].y == 0.f)
            continue;
        e[j].d = adam_update(e[j].d, gx, md[j], vd[j], lr1, bc2s, eps);
        pc[j].x = adam_update(pc[j].x, gy, mcv[j].x, vcv[j].x, lr1, bc2s, eps);
        pc[j].y = adam_update(pc[j].y, gz, mcv[j].y, vcv[j].y, lr1, bc2s, eps);
        e[j].c = __floats2half2_rn(pc[j].x, pc[j].y);
        cmaster[k] = pc[j];
        m[k] = md[j]; v[k] = vd[j]; mc_p[k] = mcv[j]; vc_p[k] = vcv[j];
        mc_st_entry(mc_table + i, e[j]);                                            // all-gather: one multicast store
    }
}

// zero the local gradient buffers of the next parity (full size, local HBM only)
__global__ void __launch_bounds__(256)
k_dp_zero(float4* __restrict__ gtab, uint32_t rows, float* __restrict__ gmlp, uint32_t n_mlp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows) gtab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < n_mlp) gmlp[i] = 0.f;
}

// MLP parameters: every rank reduces all peers' (tiny) gradient vectors and applies the same update
__global__ void __launch_bounds__(256)
k_dp_adam_mlp(const DpCtx* __restrict__ ctx, uint32_t parity, float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
              const float* __restrict__ st, float eps) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ctx->n_mlp) return;
    float g = 0.f;
    for (uint32_t q = 0; q < ctx->world; ++q) g += __ldcv(ctx->gmlp[q][parity] + i);
    if (st[3] != 0.f) return;
    g *= st[7];
    float mi = m[i], vi = v[i];
    p[i] = adam_update(p[i], g, mi, vi, __fdiv_rn(st[4], st[5]), st[6], eps);
    m[i] = mi; v[i] = vi;
}

__global__ void k_dp_post(float* __restrict__ st) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (st[3] != 0.f) { st[0] *= 0.5f; st[1] = 0.f; }
    else {
        st[1] += 1.f;
        if (st[1] >= 2000.f) { st[0] *= 2.0f; st[1] = 0.f; }
    }
    st[3] = 0.f;
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_s0_pack_weights(const float* mlp_params, void* wpack, n2m_stream_t stream);

/* ---- CUDA IPC helpers (one process per GPU): export the allocation that contains `ptr` ---- */
int n2m_ipc_export(const void* ptr, void* handle_out, uint64_t* offset_out) {
    N2M_REQUIRE(ptr && handle_out && offset_out, "ipc_export", "null pointer");
    CUdeviceptr base = 0; size_t size = 0;
    // driver entry point resolved at run time: the library must stay loadable on hosts without libcuda.so
    typedef CUresult (*range_fn)(CUdeviceptr*, size_t*, CUdeviceptr);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn)
        return fail("ipc_export", "cuMemGetAddressRange entry point not available");
    if (reinterpret_cast<range_fn>(fn)(&base, &size, (CUdeviceptr)ptr) != CUDA_SUCCESS) return fail("ipc_export", "cuMemGetAddressRange failed");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, (void*)base);
    if (e != cudaSuccess) return fail("ipc_export", cudaGetErrorString(e));
    memcpy(handle_out, &h, sizeof(h));
    *offset_out = (uint64_t)((CUdeviceptr)ptr - base);
    return 0;
}

int n2m_ipc_open(const void* handle, void** base_out) {
    N2M_REQUIRE(handle && base_out, "ipc_open", "null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    cudaError_t e = cudaIpcOpenMemHandle(base_out, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail("ipc_open", cudaGetErrorString(e));
    return 0;
}

int n2m_ipc_close(void* base) {
    cudaError_t e = cudaIpcCloseMemHandle(base);
    if (e != cudaSuccess) return fail("ipc_close", cudaGetErrorString(e));
    return 0;
}

uint32_t n2m_dp_ctx_bytes(void) { return (uint32_t)sizeof(DpCtx); }

/* host-side fill of a DpCtx image (then cudaMemcpy'd to the device by the caller) */
int n2m_dp_ctx_fill(void* host_ctx, uint32_t world, uint32_t rank, uint32_t rows, uint32_t n_mlp,
                    void* const* gtab0, void* const* gtab1, void* const* table, void* const* gmlp0, void* const* gmlp1,
                    void* const* opt, void* const* flags, void* epoch) {
    N2M_REQUIRE(host_ctx && world >= 1 && world <= (uint32_t)kMaxWorld && rank < world, "dp_ctx_fill", "bad arguments");
    DpCtx c;
    memset(&c, 0, sizeof(c));
    c.world = world; c.rank = rank; c.rows = rows; c.n_mlp = n_mlp;
    for (uint32_t p = 0; p < world; ++p) {
        c.gtab[p][0] = (float4*)gtab0[p]; c.gtab[p][1] = (float4*)gtab1[p];
        c.table[p] = (TableEntry*)table[p];
        c.gmlp[p][0] = (float*)gmlp0[p]; c.gmlp[p][1] = (float*)gmlp1[p];
        c.opt[p] = (float*)opt[p]; c.flags[p] = (uint32_t*)flags[p];
    }
    c.epoch = (uint32_t*)epoch;
    memcpy(host_ctx, &c, sizeof(c));
    return 0;
}

int n2m_dp_barrier(const void* ctx, n2m_stream_t stream) {
    N2M_REQUIRE(ctx, "dp_barrier", "null pointer");
    k_dp_barrier<<<1, 32, 0, as_stream(stream)>>>(static_cast<const DpCtx*>(ctx));
    return check_launch("dp_barrier");
}

static int dp_adam_impl(const void* ctx, const void* mc_gtab, void* mc_table, uint32_t parity, uint32_t world, uint32_t rows, uint32_t n_mlp,
                        void* color_master_slice, float* m_slice, float* v_slice, float* mlp_params, float* m_mlp, float* v_mlp, void* wpack,
                        void* gtab_next, float* gmlp_next, float* opt_state, float eps, n2m_stream_t stream);

/* barrier -> [found_inf OR, step constants] -> reduce-scatter + Adam + all-gather (tables) -> MLP -> repack ->
 * zero next-parity gradients -> scaler update -> barrier.   m/v/color_master are SLICE-sized (ceil(rows/world) rows). */
int n2m_dp_adam(const void* ctx, uint32_t parity, uint32_t world, uint32_t rows, uint32_t n_mlp, void* color_master_slice,
                float* m_slice, float* v_slice, float* mlp_params, float* m_mlp, float* v_mlp, void* wpack,
                void* gtab_next, float* gmlp_next, float* opt_state, float eps, n2m_stream_t stream) {
    return dp_adam_impl(ctx, nullptr, nullptr, parity, world, rows, n_mlp, color_master_slice, m_slice, v_slice, mlp_params, m_mlp, v_mlp, wpack,
                        gtab_next, gmlp_next, opt_state, eps, stream);
}

/* the same with the table reduce / broadcast through NVSwitch multicast (NVLS): mc_gtab = multicast address of THIS parity's gradient
 * table, mc_table = multicast address of the working table (both mapped on every rank's buffer) */
int n2m_dp_adam_nvls(const void* ctx, const void* mc_gtab, void* mc_table, uint32_t parity, uint32_t world, uint32_t rows, uint32_t n_mlp,
                     void* color_master_slice, float* m_slice, float* v_slice, float* mlp_params, float* m_mlp, float* v_mlp, void* wpack,
                     void* gtab_next, float* gmlp_next, float* opt_state, float eps, n2m_stream_t stream) {
    N2M_REQUIRE(mc_gtab && mc_table, "dp_adam_nvls", "null multicast pointer");
    return dp_adam_impl(ctx, mc_gtab, mc_table, parity, world, rows, n_mlp, color_master_slice, m_slice, v_slice, mlp_params, m_mlp, v_mlp, wpack,
                        gtab_next, gmlp_next, opt_state, eps, stream);
}

static int dp_adam_impl(const void* ctx, const void* mc_gtab, void* mc_table, uint32_t parity, uint32_t world, uint32_t rows, uint32_t n_mlp,
                        void* color_master_slice, float* m_slice, float* v_slice, float* mlp_params, float* m_mlp, float* v_mlp, void* wpack,
                        void* gtab_next, float* gmlp_next, float* opt_state, float eps, n2m_stream_t stream) {
    N2M_REQUIRE(ctx && color_master_slice && m_slice && v_slice && mlp_params && m_mlp && v_mlp && wpack && opt_state, "dp_adam", "null pointer");
    N2M_REQUIRE((gtab_next == nullptr) == (gmlp_next == nullptr), "dp_adam", "gtab_next and gmlp_next must both be given or both be NULL");
    cudaStream_t st = as_stream(stream);
    const DpCtx* c = static_cast<const DpCtx*>(ctx);
    // N2M_DP_TRACE=1 (eager launches only, never under graph capture): CUDA events between the sub-launches, printed per call
    static const bool trace = getenv("N2M_DP_TRACE") != nullptr;
    cudaEvent_t ev[8];
    int nev = 0;
    auto mark = [&]() { if (trace && nev < 8) { cudaEventCreate(&ev[nev]); cudaEventRecord(ev[nev], st); ++nev; } };
    mark();
    k_dp_publish_inf<<<1, 32, 0, st>>>(c, parity, opt_state);
    if (int e = check_launch("dp_adam(publish)")) return e;
    k_dp_barrier<<<1, 32, 0, st>>>(c);
    if (int e = check_launch("dp_adam(barrier A)")) return e;
    k_dp_prep<<<1, 32, 0, st>>>(c, parity, opt_state);
    if (int e = check_launch("dp_adam(prep)")) return e;
    mark();
    const uint32_t per = slice_rows(rows, world);
    if (mc_gtab)
        k_dp_adam_tables_mc<<<div_up(per, 256u * kMcRowsPerThread), 256, 0, st>>>(c, static_cast<const float4*>(mc_gtab), static_cast<TableEntry*>(mc_table),
                                                                                  static_cast<float2*>(color_master_slice), m_slice, v_slice, opt_state, eps);
    else
        k_dp_adam_tables<<<div_up(per, 256u * kRowsPerThread), 256, 0, st>>>(c, parity, static_cast<float2*>(color_master_slice), m_slice, v_slice,
                                                                           opt_state, eps);
    if (int e = check_launch("dp_adam(tables)")) return e;
    mark();
    k_dp_adam_mlp<<<div_up(n_mlp, 256u), 256, 0, st>>>(c, parity, mlp_params, m_mlp, v_mlp, opt_state, eps);
    if (int e = check_launch("dp_adam(mlp)")) return e;
    if (int e = n2m_s0_pack_weights(mlp_params, wpack, stream)) return e;
    if (gtab_next) {          // NULL: the caller zeroes the next-parity gradient buffers off the critical path
        k_dp_zero<<<div_up(rows, 256u), 256, 0, st>>>(static_cast<float4*>(gtab_next), rows, gmlp_next, n_mlp);
        if (int e = check_launch("dp_adam(zero)")) return e;
    }
    k_dp_post<<<1, 32, 0, st>>>(opt_state);
    if (int e = check_launch("dp_adam(post)")) return e;
    mark();
    k_dp_barrier<<<1, 32, 0, st>>>(c);
    if (int e = check_launch("dp_adam(barrier B)")) return e;
    mark();
    if (trace && nev == 5) {
        cudaEventSynchronize(ev[4]);
        float a = 0, b = 0, cc = 0, d = 0;
        cudaEventElapsedTime(&a, ev[0], ev[1]); cudaEventElapsedTime(&b, ev[1], ev[2]); cudaEventElapsedTime(&cc, ev[2], ev[3]);
        cudaEventElapsedTime(&d, ev[3], ev[4]);
        fprintf(stderr, "[n2m dp trace] publish+barrierA+prep %.1f us | tables %.1f us | mlp+pack(+zero)+post %.1f us | barrierB %.1f us\n",
                a * 1e3f, b * 1e3f, cc * 1e3f, d * 1e3f);
        for (int i = 0; i < nev; ++i) cudaEventDestroy(ev[i]);
    }
    return 0;
}

}  // extern "C"
