// optim.cu -- optimizer stage of the fused train path: GradScaler bookkeeping + Adam (torch
// semantics: betas (0.9, 0.999), eps 1e-15 as main.py:221, no weight decay) over the interleaved hash
// tables and the MLP parameters, fused with the passes the reference runs separately every step:
// unscale_ (utils.py:812), the fp32 -> fp16 colour-table cast (grid.py:45-46), zero_grad
// (utils.py:1163) and GradScaler.step/update (utils.py:1176-1177).
//
// opt_state (device float[8]): [0] loss_scale  [1] growth_tracker  [2] adam step t  [3] found_inf
//                              [4] lr (host-written)  [5] 1 - beta1^t  [6] sqrt(1 - beta2^t)  [7] 1 / loss_scale
#include "n2m_common.cuh"
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

constexpr float kBeta1 = 0.9f, kBeta2 = 0.999f;
constexpr float kGrowth = 2.0f, kBackoff = 0.5f;
constexpr float kGrowthInterval = 2000.f;

struct __align__(8) TableEntry { float d; __half2 c; };

__global__ void k_adam_post(float* __restrict__ st) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    // torch.amp.GradScaler.update: back off on inf, otherwise grow every growth_interval clean steps
    if (st[3] != 0.f) { st[0] *= kBackoff; st[1] = 0.f; }
    else {
        st[1] += 1.f;
        if (st[1] >= kGrowthInterval) { st[0] *= kGrowth; st[1] = 0.f; }
    }
    st[3] = 0.f;
}

__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, float lr_over_bc1, float bc2s, float eps) {
    m = kBeta1 * m + (1.f - kBeta1) * g;
    v = kBeta2 * v + (1.f - kBeta2) * g * g;
    const float denom = __fdiv_rn(__fsqrt_rn(v), bc2s) + eps;
    return p - lr_over_bc1 * __fdiv_rn(m, denom);
}

// Table rows: {density feature fp32 (master lives in the table), 2 colour features (fp32 masters in cmaster,
// fp16 copy in the table)}.  m/v: [rows] density then [rows][2] colour.  Pure streaming (112 B/row, ~0.7 GB per
// step): each thread handles kRowsPerThread rows, block-strided so every access stays coalesced, and issues ALL
// of its loads before the first dependent instruction -- with one row per thread the kernel is latency bound.
constexpr int kRowsPerThread = 4;

// ZERO = false: the gradient rows are left as they are; the host zeroes that table on a side stream while the NEXT step (which
// accumulates into the other gradient-table parity) runs its forward pass -- 16 of the 112 bytes per row leave the critical path.
template <bool ZERO>
__global__ void __launch_bounds__(256)
k_adam_tables(TableEntry* __restrict__ table, float2* __restrict__ cmaster, float4* __restrict__ gtable,
              float* __restrict__ m, float* __restrict__ v, uint32_t rows, const float* __restrict__ st, float eps) {
    const uint32_t i0 = blockIdx.x * (256 * kRowsPerThread) + threadIdx.x;
    const bool skip = st[3] != 0.f;
    const float inv = st[7];
    const float lr1 = __fdiv_rn(st[4], st[5]), bc2s = st[6];
    float2* mc_p = reinterpret_cast<float2*>(m + rows);
    float2* vc_p = reinterpret_cast<float2*>(v + rows);
    float4 g[kRowsPerThread]; float md[kRowsPerThread], vd[kRowsPerThread];
    float2 mc[kRowsPerThread], vc[kRowsPerThread], pc[kRowsPerThread];
    TableEntry e[kRowsPerThread];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
        const uint32_t i = i0 + j * 256;
        if (i < rows) {
            g[j] = gtable[i];
            if (!skip) { md[j] = m[i]; vd[j] = v[i]; mc[j] = mc_p[i]; vc[j] = vc_p[i]; e[j] = table[i]; pc[j] = cmaster[i]; }
        }
    }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
        const uint32_t i = i0 + j * 256;
        if (i >= rows) continue;
        if (ZERO) gtable[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (skip) continue;
        const float gx = g[j].x * inv, gy = g[j].y * inv, gz = g[j].z * inv;
        // untouched row with empty moments: the update is exactly zero -- skip the writes
        if (gx == 0.f && gy == 0.f && gz == 0.f && md[j] == 0.f && vd[j] == 0.f && mc[j].x == 0.f && mc[j].y == 0.f &&
            vc[j].x == 0.f && vc[j].y == 0.f)
            continue;
        e[j].d = adam_update(e[j].d, gx, md[j], vd[j], lr1, bc2s, eps);
        pc[j].x = adam_update(pc[j].x, gy, mc[j].x, vc[j].x, lr1, bc2s, eps);
        pc[j].y = adam_update(pc[j].y, gz, mc[j].y, vc[j].y, lr1, bc2s, eps);
        e[j].c = __floats2half2_rn(pc[j].x, pc[j].y);
        table[i] = e[j];
        cmaster[i] = pc[j];
        m[i] = md[j]; v[i] = vd[j];
        mc_p[i] = mc[j]; vc_p[i] = vc[j];
    }
}

__global__ void __launch_bounds__(256)
k_adam_mlp(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, uint32_t n,
           const float* __restrict__ st, float eps) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool skip = st[3] != 0.f;
    const float gi = g[i] * st[7];
    g[i] = 0.f;
    if (skip) return;
    float mi = m[i], vi = v[i];
    p[i] = adam_update(p[i], gi, mi, vi, __fdiv_rn(st[4], st[5]), st[6], eps);
    m[i] = mi; v[i] = vi;
}

// head of the optimizer stage, one block: non-finite scan of the MLP gradient vector (the table gradients are checked
// where they are produced) OR-ed into found_inf, then the per-step constants (bias corrections, 1 / loss_scale)
__global__ void __launch_bounds__(1024)
k_adam_head(const float* __restrict__ g, uint32_t n, float* __restrict__ st) {
    int bad = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) bad |= !isfinite(g[i]);
    bad = __syncthreads_or(bad);
    if (threadIdx.x != 0) return;
    if (bad) st[3] = 1.f;
    const bool skip = st[3] != 0.f;
    if (!skip) st[2] += 1.f;
    const float t = fmaxf(st[2], 1.f);
    st[5] = 1.f - powf(kBeta1, t);
    st[6] = sqrtf(1.f - powf(kBeta2, t));
    st[7] = 1.f / st[0];
}

// ---- EMA of the parameters (torch_ema.ExponentialMovingAverage as the reference's Trainer uses it: created at
// nerf/utils.py:544-545 with decay 0.95, `update()` ONCE PER EPOCH at utils.py:1213-1214, swapped in for evaluation at
// utils.py:1250-1252 / 1340-1341 and for the 'best' checkpoint at :1389-1401).  shadow -= (1 - decay) * (shadow - param), in the
// library's operation order (tmp = shadow - param; tmp *= one_minus_decay; shadow -= tmp).
__global__ void __launch_bounds__(256)
k_ema_update(const TableEntry* __restrict__ table, const float2* __restrict__ cmaster, const float* __restrict__ mlp,
             float* __restrict__ sh_d, float2* __restrict__ sh_c, float* __restrict__ sh_mlp, uint32_t rows, uint32_t n_mlp,
             float one_minus_decay) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows) {
        const float pd = table[i].d; const float2 pc = cmaster[i];
        float sd = sh_d[i]; float2 sc = sh_c[i];
        sd = __fsub_rn(sd, __fmul_rn(__fsub_rn(sd, pd), one_minus_decay));
        sc.x = __fsub_rn(sc.x, __fmul_rn(__fsub_rn(sc.x, pc.x), one_minus_decay));
        sc.y = __fsub_rn(sc.y, __fmul_rn(__fsub_rn(sc.y, pc.y), one_minus_decay));
        sh_d[i] = sd; sh_c[i] = sc;
    }
    if (i < n_mlp) {
        const float s = sh_mlp[i];
        sh_mlp[i] = __fsub_rn(s, __fmul_rn(__fsub_rn(s, mlp[i]), one_minus_decay));
    }
}

// parameters <-> shadow, in place (ema.store(); ema.copy_to()  ==  swap;   ema.restore()  ==  swap back); the fp16 working copy of
// the colour features is refreshed from the swapped-in fp32 values
__global__ void __launch_bounds__(256)
k_ema_swap(TableEntry* __restrict__ table, float2* __restrict__ cmaster, float* __restrict__ mlp,
           float* __restrict__ sh_d, float2* __restrict__ sh_c, float* __restrict__ sh_mlp, uint32_t rows, uint32_t n_mlp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows) {
        TableEntry e = table[i]; const float2 pc = cmaster[i];
        const float sd = sh_d[i]; const float2 sc = sh_c[i];
        sh_d[i] = e.d; sh_c[i] = pc;
        e.d = sd; e.c = __floats2half2_rn(sc.x, sc.y);
        table[i] = e; cmaster[i] = sc;
    }
    if (i < n_mlp) { const float s = sh_mlp[i]; sh_mlp[i] = mlp[i]; mlp[i] = s; }
}

// ---- the appearance-code block `ind` [64 D code columns of color_net.0 | ind_num * D codes] (include/n2m_b200_fused.h): two Adam groups,
// lr and 0.1 lr (renderer.py:173-174), weight decay 0 for both
__global__ void __launch_bounds__(256)
k_adam_codes(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, uint32_t n_cols, uint32_t n,
             const float* __restrict__ st, float eps) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool skip = st[3] != 0.f;
    const float gi = g[i] * st[7];
    g[i] = 0.f;
    if (skip) return;
    const float lr = i < n_cols ? st[4] : __fmul_rn(st[4], 0.1f);
    float mi = m[i], vi = v[i];
    p[i] = adam_update(p[i], gi, mi, vi, __fdiv_rn(lr, st[5]), st[6], eps);
    m[i] = mi; v[i] = vi;
}

__global__ void __launch_bounds__(1024)
k_adam_codes_head(const float* __restrict__ g, uint32_t n, float* __restrict__ st) {
    int bad = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) bad |= !isfinite(g[i]);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0 && bad) st[3] = 1.f;
}

__global__ void __launch_bounds__(256)
k_codes_ema(float* __restrict__ p, float* __restrict__ sh, uint32_t n, float one_minus_decay, bool swap) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float s = sh[i];
    if (swap) { sh[i] = p[i]; p[i] = s; }
    else sh[i] = __fsub_rn(s, __fmul_rn(__fsub_rn(s, p[i]), one_minus_decay));
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" int n2m_s0_pack_code_weights(const float* ind, uint32_t ind_dim, void* wpack, n2m_stream_t stream);

extern "C" int n2m_s0_adam_codes_head(const float* g_ind, uint32_t n, float* opt_state, n2m_stream_t stream) {
    N2M_REQUIRE(g_ind && opt_state, "s0_adam_codes_head", "null pointer");
    if (n == 0) return 0;
    k_adam_codes_head<<<1, 1024, 0, as_stream(stream)>>>(g_ind, n, opt_state);
    return check_launch("s0_adam_codes_head");
}

extern "C" int n2m_s0_adam_codes(float* ind, float* g_ind, float* m_ind, float* v_ind, uint32_t ind_dim, uint32_t ind_num, void* wpack,
                                 const float* opt_state, float eps, n2m_stream_t stream) {
    N2M_REQUIRE(ind_dim <= 10, "s0_adam_codes", "ind_dim must be at most 10");
    if (ind_dim == 0) return 0;
    N2M_REQUIRE(ind && g_ind && m_ind && v_ind && wpack && opt_state, "s0_adam_codes", "null pointer");
    const uint32_t n = (64 + ind_num) * ind_dim;
    k_adam_codes<<<div_up(n, 256u), 256, 0, as_stream(stream)>>>(ind, g_ind, m_ind, v_ind, 64 * ind_dim, n, opt_state, eps);
    if (int e = check_launch("s0_adam_codes")) return e;
    return n2m_s0_pack_code_weights(ind, ind_dim, wpack, stream);
}

extern "C" int n2m_s0_codes_ema_update(const float* ind, float* shadow_ind, uint32_t n, float one_minus_decay, n2m_stream_t stream) {
    N2M_REQUIRE(ind && shadow_ind, "s0_codes_ema_update", "null pointer");
    if (n == 0) return 0;
    k_codes_ema<<<div_up(n, 256u), 256, 0, as_stream(stream)>>>(const_cast<float*>(ind), shadow_ind, n, one_minus_decay, false);
    return check_launch("s0_codes_ema_update");
}

extern "C" int n2m_s0_codes_ema_swap(float* ind, float* shadow_ind, uint32_t ind_dim, uint32_t ind_num, void* wpack, n2m_stream_t stream) {
    N2M_REQUIRE(ind_dim <= 10, "s0_codes_ema_swap", "ind_dim must be at most 10");
    if (ind_dim == 0) return 0;
    N2M_REQUIRE(ind && shadow_ind && wpack, "s0_codes_ema_swap", "null pointer");
    const uint32_t n = (64 + ind_num) * ind_dim;
    k_codes_ema<<<div_up(n, 256u), 256, 0, as_stream(stream)>>>(ind, shadow_ind, n, 0.f, true);
    if (int e = check_launch("s0_codes_ema_swap")) return e;
    return n2m_s0_pack_code_weights(ind, ind_dim, wpack, stream);
}

extern "C" int n2m_s0_pack_weights(const float* mlp_params, void* wpack, n2m_stream_t stream);
extern "C" uint32_t n2m_s0_mlp_param_count(void);

/* The optimizer stage in four launches.  adam_mlp (+ weight repack) and adam_tables are independent of each other (both only
 * READ opt_state), so a host may run them on two streams between head and post. */
extern "C" int n2m_s0_adam_head(const float* g_mlp, float* opt_state, n2m_stream_t stream) {
    N2M_REQUIRE(g_mlp && opt_state, "s0_adam_head", "null pointer");
    k_adam_head<<<1, 1024, 0, as_stream(stream)>>>(g_mlp, n2m_s0_mlp_param_count(), opt_state);
    return check_launch("s0_adam(head)");
}

extern "C" int n2m_s0_adam_tables(void* table, void* color_master, void* gtable, float* m_table, float* v_table, uint32_t rows,
                                  const float* opt_state, float eps, n2m_stream_t stream) {
    N2M_REQUIRE(table && color_master && gtable && m_table && v_table && opt_state, "s0_adam_tables", "null pointer");
    if (rows == 0) return 0;
    k_adam_tables<true><<<div_up(rows, 256u * kRowsPerThread), 256, 0, as_stream(stream)>>>(
        static_cast<TableEntry*>(table), static_cast<float2*>(color_master), static_cast<float4*>(gtable), m_table, v_table, rows,
        opt_state, eps);
    return check_launch("s0_adam(tables)");
}

/* the same without zeroing the gradient rows (the caller zeroes that table off the critical path, see k_adam_tables) */
extern "C" int n2m_s0_adam_tables_keep(void* table, void* color_master, const void* gtable, float* m_table, float* v_table, uint32_t rows,
                                       const float* opt_state, float eps, n2m_stream_t stream) {
    N2M_REQUIRE(table && color_master && gtable && m_table && v_table && opt_state, "s0_adam_tables_keep", "null pointer");
    if (rows == 0) return 0;
    k_adam_tables<false><<<div_up(rows, 256u * kRowsPerThread), 256, 0, as_stream(stream)>>>(
        static_cast<TableEntry*>(table), static_cast<float2*>(color_master), static_cast<float4*>(const_cast<void*>(gtable)), m_table, v_table,
        rows, opt_state, eps);
    return check_launch("s0_adam(tables, keep)");
}

extern "C" int n2m_s0_adam_mlp(float* mlp_params, float* g_mlp, float* m_mlp, float* v_mlp, void* wpack, const float* opt_state,
                               float eps, n2m_stream_t stream) {
    N2M_REQUIRE(mlp_params && g_mlp && m_mlp && v_mlp && wpack && opt_state, "s0_adam_mlp", "null pointer");
    const uint32_t n = n2m_s0_mlp_param_count();
    k_adam_mlp<<<div_up(n, 256u), 256, 0, as_stream(stream)>>>(mlp_params, g_mlp, m_mlp, v_mlp, n, opt_state, eps);
    if (int e = check_launch("s0_adam(mlp)")) return e;
    return n2m_s0_pack_weights(mlp_params, wpack, stream);
}

extern "C" int n2m_s0_adam_post(float* opt_state, n2m_stream_t stream) {
    N2M_REQUIRE(opt_state, "s0_adam_post", "null pointer");
    k_adam_post<<<1, 32, 0, as_stream(stream)>>>(opt_state);
    return check_launch("s0_adam(post)");
}


/* EMA shadow update over the hash tables (fp32 density feature in the table, fp32 colour masters) and the MLP parameters */
extern "C" int n2m_s0_ema_update(const void* table, const void* color_master, const float* mlp_params, float* shadow_density,
                                 void* shadow_color, float* shadow_mlp, uint32_t rows, float one_minus_decay, n2m_stream_t stream) {
    N2M_REQUIRE(table && color_master && mlp_params && shadow_density && shadow_color && shadow_mlp, "s0_ema_update", "null pointer");
    const uint32_t n = n2m_s0_mlp_param_count();
    const uint32_t work = rows > n ? rows : n;
    if (work == 0) return 0;
    k_ema_update<<<div_up(work, 256u), 256, 0, as_stream(stream)>>>(static_cast<const TableEntry*>(table), static_cast<const float2*>(color_master),
                                                                     mlp_params, shadow_density, static_cast<float2*>(shadow_color), shadow_mlp,
                                                                     rows, n, one_minus_decay);
    return check_launch("s0_ema_update");
}

/* swap parameters and EMA shadow in place (+ weight repack) */
extern "C" int n2m_s0_ema_swap(void* table, void* color_master, float* mlp_params, float* shadow_density, void* shadow_color,
                               float* shadow_mlp, uint32_t rows, void* wpack, n2m_stream_t stream) {
    N2M_REQUIRE(table && color_master && mlp_params && shadow_density && shadow_color && shadow_mlp && wpack, "s0_ema_swap", "null pointer");
    const uint32_t n = n2m_s0_mlp_param_count();
    const uint32_t work = rows > n ? rows : n;
    if (work == 0) return 0;
    k_ema_swap<<<div_up(work, 256u), 256, 0, as_stream(stream)>>>(static_cast<TableEntry*>(table), static_cast<float2*>(color_master), mlp_params,
                                                                   shadow_density, static_cast<float2*>(shadow_color), shadow_mlp, rows, n);
    if (int e = check_launch("s0_ema_swap")) return e;
    return n2m_s0_pack_weights(mlp_params, wpack, stream);
}
