// raymarching.cu -- occupancy-grid ray marching + volume compositing for sm_90a.
//
// Replaces the native layer behind the reference's `raymarching.*` operators
// (reference: raymarching/src/raymarching.cu).  Arithmetic contract: every value that decides
// a sample (t sequence, cascade level, cell index, occupancy bit, voxel-exit distance) is
// evaluated with the same operation order, literal types and -use_fast_math semantics as the
// reference so that per-ray sample COUNTS and positions are bit-identical; the structure around
// it is different:
//   * one sequential march per ray instead of two: the counting pass records (t, dt) of every
//     emitted sample in a scratch slab, a block scan produces DETERMINISTIC ray-order offsets
//     (the reference's atomicAdd order is not, raymarching.cu:471), and the output pass
//     regenerates xyz/dir/ts for all samples in parallel, one warp per ray, coalesced;
//   * the cell test uses only fp32/integer instructions (the reference's double sub-expressions
//     `0.5 * (..) * H` and `dt * H * 0.5` are exact products of <= 48 significant bits, so a
//     single fp32 multiply rounds identically);
//   * every launch goes to the caller's stream and is checked.
#include "march_core.cuh"

namespace n2m {

thread_local char g_err[512] = {0};
std::atomic<uint64_t> g_launches{0};

namespace {

constexpr float kInvPi = 0.3183098861837907f;
constexpr int kRayBlock = 128;
using namespace march;

// ---- training: counting pass ------------------------------------------------------------------
__global__ void __launch_bounds__(kRayBlock)
k_march_train_count(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                    const uint8_t* __restrict__ bits, float bound, bool contract, float dt_gamma,
                    uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H,
                    const float* __restrict__ nears, const float* __restrict__ fars,
                    const float* __restrict__ noises, int32_t* __restrict__ rays,
                    float2* __restrict__ tbuf) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const MarchCfg c = make_cfg(bound, contract, dt_gamma, max_steps, C, H, bits);
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
    const float rdx = 1 / dx, rdy = 1 / dy, rdz = 1 / dz;
    const float near = nears[n], far = fars[n], noise = noises[n];
    float t0 = near;
    t0 += clampf(t0 * c.dt_gamma, c.dt_min, c.dt_max) * noise;     // raymarching.cu:389-390
    CountSink sink{tbuf ? tbuf + (size_t)n * max_steps : nullptr};
    const uint32_t cnt = march_one(c, t0, far, max_steps, ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, sink);
    rays[2 * n + 1] = (int32_t)cnt;
}

// ---- training: exclusive scan of counts -> offsets (single block; N is a few thousand rays) -----
__global__ void __launch_bounds__(1024)
k_scan_counts(int32_t* __restrict__ rays, uint32_t N, int32_t* __restrict__ counter) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
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
            warp_tot[lane] = w;     // inclusive over warps
        }
        __syncthreads();
        const uint32_t carry = carry_s;
        const uint32_t excl = carry + (wid ? warp_tot[wid - 1] : 0u) + inc - v;
        if (i < N) rays[2 * i] = (int32_t)excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) counter[0] = (int32_t)carry_s;
}

// ---- training: parallel output pass from the (t, dt) slab: one warp per ray ---------------------
__global__ void __launch_bounds__(256)
k_march_train_emit(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                   float bound, bool contract, uint32_t max_steps, uint32_t N,
                   const int32_t* __restrict__ rays, const float2* __restrict__ tbuf,
                   float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ ts) {
    const uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (n >= N) return;
    const uint32_t off = (uint32_t)rays[2 * n], cnt = (uint32_t)rays[2 * n + 1];
    if (cnt == 0) return;
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
    const float2* slab = tbuf + (size_t)n * max_steps;
    for (uint32_t k = lane; k < cnt; k += 32) {
        const float2 td = slab[k];
        const float t = td.x;
        float cx = clampf(ox + t * dx, -bound, bound);
        float cy = clampf(oy + t * dy, -bound, bound);
        float cz = clampf(oz + t * dz, -bound, bound);
        const float mag = fmaxf(fabsf(cx), fmaxf(fabsf(cy), fabsf(cz)));
        if (contract && mag > 1) {
            const float s = (2 - 1 / mag) / mag;
            cx *= s; cy *= s; cz *= s;
        }
        const size_t j = (size_t)off + k;
        xyzs[3 * j + 0] = cx; xyzs[3 * j + 1] = cy; xyzs[3 * j + 2] = cz;
        dirs[3 * j + 0] = dx; dirs[3 * j + 1] = dy; dirs[3 * j + 2] = dz;
        ts[2 * j + 0] = t + td.y;
        ts[2 * j + 1] = td.y;
    }
}

// ---- training: sequential output pass (no slab) --------------------------------------------------
__global__ void __launch_bounds__(kRayBlock)
k_march_train_rewalk(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                     const uint8_t* __restrict__ bits, float bound, bool contract, float dt_gamma,
                     uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H,
                     const float* __restrict__ nears, const float* __restrict__ fars,
                     const float* __restrict__ noises, const int32_t* __restrict__ rays,
                     float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ ts) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const MarchCfg c = make_cfg(bound, contract, dt_gamma, max_steps, C, H, bits);
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
    const float rdx = 1 / dx, rdy = 1 / dy, rdz = 1 / dz;
    const float near = nears[n], far = fars[n], noise = noises[n];
    float t0 = near;
    t0 += clampf(t0 * c.dt_gamma, c.dt_min, c.dt_max) * noise;
    const size_t off = (size_t)(uint32_t)rays[2 * n];
    WriteSink sink{xyzs + 3 * off, dirs + 3 * off, ts + 2 * off};
    march_one(c, t0, far, (uint32_t)rays[2 * n + 1], ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, sink);
}

// ---- inference marcher (raymarching.cu:713-828) -------------------------------------------------
__global__ void __launch_bounds__(kRayBlock)
k_march_infer(uint32_t n_alive, uint32_t n_step, const int32_t* __restrict__ rays_alive,
              const float* __restrict__ rays_t, const float* __restrict__ rays_o,
              const float* __restrict__ rays_d, float bound, bool contract, float dt_gamma,
              uint32_t max_steps, uint32_t C, uint32_t H, const uint8_t* __restrict__ bits,
              const float* __restrict__ nears, const float* __restrict__ fars,
              float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ ts,
              const float* __restrict__ noises) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int r = rays_alive[n];
    const float noise = noises[n];
    const MarchCfg c = make_cfg(bound, contract, dt_gamma, max_steps, C, H, bits);
    const float ox = rays_o[3 * r], oy = rays_o[3 * r + 1], oz = rays_o[3 * r + 2];
    const float dx = rays_d[3 * r], dy = rays_d[3 * r + 1], dz = rays_d[3 * r + 2];
    // the inference kernel regularises the reciprocal, the training kernel does not (:744 vs :377)
    const float rdx = 1 / (dx + 1e-10f), rdy = 1 / (dy + 1e-10f), rdz = 1 / (dz + 1e-10f);
    const float far = fars[r];
    (void)nears;
    float t = rays_t[r];
    t += clampf(t * c.dt_gamma, c.dt_min, c.dt_max) * noise;
    const size_t base = (size_t)n * n_step;
    WriteSink sink{xyzs + 3 * base, dirs + 3 * base, ts + 2 * base};
    march_one(c, t, far, n_step, ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, sink);
}

// ---------------------------------------------------------------------------------------------
// compositing
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float alpha_of(float sigma, float dt, bool alpha_mode) {
    return alpha_mode ? sigma : (1.0f - __expf(-sigma * dt));
}

// raymarching.cu:501-578
__global__ void __launch_bounds__(kRayBlock)
k_composite_train_fwd(const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                      const float* __restrict__ ts, const int32_t* __restrict__ rays,
                      uint32_t M, uint32_t N, float T_thresh, bool alpha_mode,
                      float* __restrict__ weights, float* __restrict__ weights_sum,
                      float* __restrict__ depth, float* __restrict__ image) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const uint32_t off = rays[2 * n], cnt = rays[2 * n + 1];
    float T = 1.0f, r = 0, g = 0, b = 0, ws = 0, d = 0;
    if (cnt != 0 && off + cnt <= M) {
        for (uint32_t k = 0; k < cnt; ++k) {
            const size_t j = (size_t)off + k;
            const float tj = ts[2 * j], dtj = ts[2 * j + 1];
            const float alpha = alpha_of(sigmas[j], dtj, alpha_mode);
            const float w = alpha * T;
            weights[j] = w;
            r += w * rgbs[3 * j];
            g += w * rgbs[3 * j + 1];
            b += w * rgbs[3 * j + 2];
            ws += w;
            d += w * tj;
            T *= 1.0f - alpha;
            if (T < T_thresh) break;    // tested after accumulating, as in the reference (:554-557)
        }
    }
    weights_sum[n] = ws;
    depth[n] = d;
    image[3 * n] = r; image[3 * n + 1] = g; image[3 * n + 2] = b;
}

// raymarching.cu:605-694
__global__ void __launch_bounds__(kRayBlock)
k_composite_train_bwd(const float* __restrict__ g_weights, const float* __restrict__ g_wsum,
                      const float* __restrict__ g_depth, const float* __restrict__ g_image,
                      const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                      const float* __restrict__ ts, const int32_t* __restrict__ rays,
                      const float* __restrict__ weights_sum, const float* __restrict__ depth,
                      const float* __restrict__ image, uint32_t M, uint32_t N, float T_thresh,
                      bool alpha_mode, float* __restrict__ g_sigmas, float* __restrict__ g_rgbs) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const uint32_t off = rays[2 * n], cnt = rays[2 * n + 1];
    if (cnt == 0 || off + cnt > M) return;
    const float gi0 = g_image[3 * n], gi1 = g_image[3 * n + 1], gi2 = g_image[3 * n + 2];
    const float gws = g_wsum[n], gd = g_depth[n];
    const float r_fin = image[3 * n], g_fin = image[3 * n + 1], b_fin = image[3 * n + 2];
    const float ws_fin = weights_sum[n], d_fin = depth[n];
    float T = 1.0f, r = 0, g = 0, b = 0, ws = 0, d = 0;
    for (uint32_t k = 0; k < cnt; ++k) {
        const size_t j = (size_t)off + k;
        const float tj = ts[2 * j], dtj = ts[2 * j + 1];
        const float c0 = rgbs[3 * j], c1 = rgbs[3 * j + 1], c2 = rgbs[3 * j + 2];
        const float alpha = alpha_of(sigmas[j], dtj, alpha_mode);
        const float w = alpha * T;
        r += w * c0; g += w * c1; b += w * c2;
        ws += w;
        d += w * tj;
        T *= 1.0f - alpha;          // post-update transmittance enters the formula (:662 before :672)
        g_rgbs[3 * j] = gi0 * w;
        g_rgbs[3 * j + 1] = gi1 * w;
        g_rgbs[3 * j + 2] = gi2 * w;
        const float scale = alpha_mode ? (1.0f / (1.0f - alpha)) : dtj;
        g_sigmas[j] = scale * (
            gi0 * (T * c0 - (r_fin - r)) +
            gi1 * (T * c1 - (g_fin - g)) +
            gi2 * (T * c2 - (b_fin - b)) +
            (gws + g_weights[j]) * (T - (ws_fin - ws)) +
            gd * (T * tj - (d_fin - d)));
        if (T < T_thresh) break;
    }
}

// raymarching.cu:842-924
__global__ void __launch_bounds__(kRayBlock)
k_composite_infer(uint32_t n_alive, uint32_t n_step, float T_thresh, bool alpha_mode,
                  int32_t* __restrict__ rays_alive, float* __restrict__ rays_t,
                  const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                  const float* __restrict__ ts, float* __restrict__ weights_sum,
                  float* __restrict__ depth, float* __restrict__ image) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int idx = rays_alive[n];
    const size_t base = (size_t)n * n_step;
    float t = 0;
    float d = depth[idx], r = image[3 * idx], g = image[3 * idx + 1], b = image[3 * idx + 2];
    float wsum = weights_sum[idx];
    uint32_t k = 0;
    for (; k < n_step; ++k) {
        const size_t j = base + k;
        const float tj = ts[2 * j];
        if (tj == 0) break;                 // zero-initialised tail = the ray ran out (:877)
        const float alpha = alpha_of(sigmas[j], ts[2 * j + 1], alpha_mode);
        const float T = 1 - wsum;           // transmittance carried across slabs through weights_sum
        const float w = alpha * T;
        wsum += w;
        t = tj;
        d += w * t;
        r += w * rgbs[3 * j];
        g += w * rgbs[3 * j + 1];
        b += w * rgbs[3 * j + 2];
        if (T < T_thresh) break;
    }
    if (k < n_step) rays_alive[n] = -1;
    else rays_t[idx] = t;
    weights_sum[idx] = wsum;
    depth[idx] = d;
    image[3 * idx] = r; image[3 * idx + 1] = g; image[3 * idx + 2] = b;
}

// ---------------------------------------------------------------------------------------------
// utilities
// ---------------------------------------------------------------------------------------------
// Slab test against the AABB (raymarching.cu:92-145).
__global__ void __launch_bounds__(kRayBlock)
k_near_far(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
           const float* __restrict__ aabb, uint32_t N, float min_near,
           float* __restrict__ nears, float* __restrict__ fars) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float near, far;
    near_far_aabb(rays_o + 3 * n, rays_d + 3 * n, aabb, min_near, near, far);
    nears[n] = near;
    fars[n] = far;
}

// raymarching.cu:163-198
__global__ void __launch_bounds__(kRayBlock)
k_sph_from_ray(const float* __restrict__ rays_o, const float* __restrict__ rays_d, float radius,
               uint32_t N, float* __restrict__ coords) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
    const float A = dx * dx + dy * dy + dz * dz;
    const float B = ox * dx + oy * dy + oz * dz;
    const float Cq = ox * ox + oy * oy + oz * oz - radius * radius;
    const float t = (-B + sqrtf(B * B - A * Cq)) / A;
    const float x = ox + t * dx, y = oy + t * dy, z = oz + t * dz;
    const float theta = atan2(sqrtf(x * x + z * z), y);
    const float phi = atan2(z, x);
    coords[2 * n] = 2 * theta * kInvPi - 1;
    coords[2 * n + 1] = phi * kInvPi;
}

__global__ void __launch_bounds__(256)
k_morton(const int32_t* __restrict__ coords, uint32_t N, int32_t* __restrict__ out) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    out[n] = (int32_t)morton3(coords[3 * n], coords[3 * n + 1], coords[3 * n + 2]);
}

__global__ void __launch_bounds__(256)
k_morton_inv(const int32_t* __restrict__ idx, uint32_t N, int32_t* __restrict__ coords) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int32_t v = idx[n];
    coords[3 * n] = (int32_t)compact3(v >> 0);
    coords[3 * n + 1] = (int32_t)compact3(v >> 1);
    coords[3 * n + 2] = (int32_t)compact3(v >> 2);
}

// One thread packs 32 cells -> 4 bytes: two float4 x4 loads, one 32-bit store (HBM-bound byte
// work: coalesced 128 B per thread in, 4 B out).  Tail bytes handled scalar.
__global__ void __launch_bounds__(256)
k_packbits(const float* __restrict__ grid, uint32_t nbytes, float thresh, uint8_t* __restrict__ bits) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;     // 4-byte word index
    const uint32_t nwords = nbytes / 4;
    if (w < nwords) {
        const float4* g4 = reinterpret_cast<const float4*>(grid) + (size_t)w * 8;
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 v = __ldg(g4 + q);
            word |= (v.x > thresh ? 1u : 0u) << (4 * q + 0);
            word |= (v.y > thresh ? 1u : 0u) << (4 * q + 1);
            word |= (v.z > thresh ? 1u : 0u) << (4 * q + 2);
            word |= (v.w > thresh ? 1u : 0u) << (4 * q + 3);
        }
        reinterpret_cast<uint32_t*>(bits)[w] = word;
    } else if (w == nwords) {
        for (uint32_t n = nwords * 4; n < nbytes; ++n) {
            uint8_t b = 0;
            for (int i = 0; i < 8; ++i) b |= (grid[(size_t)n * 8 + i] > thresh) ? (uint8_t)(1u << i) : 0;
            bits[n] = b;
        }
    }
}

// generic (unaligned pointers) fallback: one thread per byte
__global__ void __launch_bounds__(256)
k_packbits_bytes(const float* __restrict__ grid, uint32_t nbytes, float thresh, uint8_t* __restrict__ bits) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nbytes) return;
    uint8_t b = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) b |= (grid[(size_t)n * 8 + i] > thresh) ? (uint8_t)(1u << i) : 0;
    bits[n] = b;
}

// one warp per ray, coalesced
__global__ void __launch_bounds__(256)
k_flatten_rays(const int32_t* __restrict__ rays, uint32_t N, uint32_t M, int32_t* __restrict__ res) {
    const uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (n >= N) return;
    const uint32_t off = rays[2 * n], cnt = rays[2 * n + 1];
    for (uint32_t k = lane; k < cnt; k += 32)
        if (off + k < M) res[off + k] = (int32_t)n;
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

const char* n2m_last_error(void) { return g_err; }
int n2m_version(void) { return 100; }
uint64_t n2m_launch_count(void) { return g_launches.load(); }

int n2m_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb, uint32_t N,
                           float min_near, float* nears, float* fars, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(rays_o && rays_d && aabb && nears && fars, "near_far_from_aabb", "null pointer");
    k_near_far<<<div_up(N, (uint32_t)kRayBlock), kRayBlock, 0, as_stream(stream)>>>(rays_o, rays_d, aabb, N, min_near, nears, fars);
    return check_launch("near_far_from_aabb");
}

int n2m_sph_from_ray(const float* rays_o, const float* rays_d, float radius, uint32_t N, float* coords,
                     n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(rays_o && rays_d && coords, "sph_from_ray", "null pointer");
    k_sph_from_ray<<<div_up(N, (uint32_t)kRayBlock), kRayBlock, 0, as_stream(stream)>>>(rays_o, rays_d, radius, N, coords);
    return check_launch("sph_from_ray");
}

int n2m_morton3D(const int32_t* coords, uint32_t N, int32_t* indices, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(coords && indices, "morton3D", "null pointer");
    k_morton<<<div_up(N, 256u), 256, 0, as_stream(stream)>>>(coords, N, indices);
    return check_launch("morton3D");
}

int n2m_morton3D_invert(const int32_t* indices, uint32_t N, int32_t* coords, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(coords && indices, "morton3D_invert", "null pointer");
    k_morton_inv<<<div_up(N, 256u), 256, 0, as_stream(stream)>>>(indices, N, coords);
    return check_launch("morton3D_invert");
}

int n2m_packbits(const float* grid, uint32_t N, float density_thresh, uint8_t* bitfield, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(grid && bitfield, "packbits", "null pointer");
    const bool aligned = (reinterpret_cast<uintptr_t>(grid) % 16 == 0) && (reinterpret_cast<uintptr_t>(bitfield) % 4 == 0);
    if (aligned) {
        const uint32_t nthreads = N / 4 + 1;
        k_packbits<<<div_up(nthreads, 256u), 256, 0, as_stream(stream)>>>(grid, N, density_thresh, bitfield);
    } else {
        k_packbits_bytes<<<div_up(N, 256u), 256, 0, as_stream(stream)>>>(grid, N, density_thresh, bitfield);
    }
    return check_launch("packbits");
}

int n2m_flatten_rays(const int32_t* rays, uint32_t N, uint32_t M, int32_t* res, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(rays && res, "flatten_rays", "null pointer");
    k_flatten_rays<<<div_up(N * 32u, 256u), 256, 0, as_stream(stream)>>>(rays, N, M, res);
    return check_launch("flatten_rays");
}

int n2m_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* grid, float bound,
                         int contract, float dt_gamma, uint32_t max_steps, uint32_t N, uint32_t C,
                         uint32_t H, const float* nears, const float* fars, float* xyzs, float* dirs,
                         float* ts, int32_t* rays, int32_t* counter, const float* noises, float* tbuf,
                         n2m_stream_t stream) {
    cudaStream_t st = as_stream(stream);
    if (N == 0) {          // empty batch: M = 0 (rays is a zero-size tensor, possibly NULL)
        if (!xyzs && counter) { cudaMemsetAsync(counter, 0, sizeof(int32_t), st); }
        return 0;
    }
    N2M_REQUIRE(rays && counter, "march_rays_train", "rays/counter must not be null");
    N2M_REQUIRE(rays_o && rays_d && grid && nears && fars && noises, "march_rays_train", "null pointer");
    N2M_REQUIRE(max_steps > 0 && H > 0 && C > 0, "march_rays_train", "max_steps, H, C must be positive");
    if (!xyzs) {
        k_march_train_count<<<div_up(N, (uint32_t)kRayBlock), kRayBlock, 0, st>>>(
            rays_o, rays_d, grid, bound, contract != 0, dt_gamma, max_steps, N, C, H, nears, fars, noises,
            rays, reinterpret_cast<float2*>(tbuf));
        if (int e = check_launch("march_rays_train(count)")) return e;
        k_scan_counts<<<1, 1024, 0, st>>>(rays, N, counter);
        return check_launch("march_rays_train(scan)");
    }
    N2M_REQUIRE(dirs && ts, "march_rays_train", "xyzs given but dirs/ts null");
    if (tbuf) {
        k_march_train_emit<<<div_up(N * 32u, 256u), 256, 0, st>>>(
            rays_o, rays_d, bound, contract != 0, max_steps, N, rays, reinterpret_cast<const float2*>(tbuf),
            xyzs, dirs, ts);
        return check_launch("march_rays_train(emit)");
    }
    k_march_train_rewalk<<<div_up(N, (uint32_t)kRayBlock), kRayBlock, 0, st>>>(
        rays_o, rays_d, grid, bound, contract != 0, dt_gamma, max_steps, N, C, H, nears, fars, noises, rays,
        xyzs, dirs, ts);
    return check_launch("march_rays_train(rewalk)");
}

int n2m_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* ts,
                                     const int32_t* rays, uint32_t M, uint32_t N, float T_thresh,
                                     int alpha_mode, float* weights, float* weights_sum, float* depth,
                                     float* image, n2m_stream_t stream) {
    if (N == 0) return 0;
    N2M_REQUIRE(rays && weights_sum && depth && image, "composite_rays_train_forward", "null pointer");
    N2M_REQUIRE(M == 0 || (sigmas && rgbs && ts && weights), "composite_rays_train_forward", "null sample pointer");
    k_composite_train_fwd<<<div_up(N, (uint32_t)kRayBlock), kRayBlock, 0, as_stream(stream)>>>(
        sigmas, rgbs, ts, rays, M, N, T_thresh, alpha_mode != 0, weights, weights_sum, depth, image);
    return check_launch("composite_rays_train_forward");
}

int n2m_composite_rays_train_backward(const float* grad_weights, const float* grad_weights_sum,
                                      const float* grad_depth, const float* grad_image,
                                      const float* sigmas, const float* rgbs, const float* ts,
                                      const int32_t* rays, const float* weights_sum, const float* depth,
                                      const float* image, uint32_t M, uint32_t N, float T_thresh,
                                      int alpha_mode, float* grad_sigmas, float* grad_rgbs,
                                      n2m_stream_t stream) {
    if (N == 0 || M == 0) return 0;
    N2M_REQUIRE(grad_weights && grad_weights_sum && grad_depth && grad_image && sigmas && rgbs && ts &&
                rays && weights_sum && depth && image && grad_sigmas && grad_rgbs,
                "composite_rays_train_backward", "null pointer");
    k_composite_train_bwd<<<div_up(N, (uint32_t)kRayBlock), kRayBlock, 0, as_stream(stream)>>>(
        grad_weights, grad_weights_sum, grad_depth, grad_image, sigmas, rgbs, ts, rays, weights_sum, depth,
        image, M, N, T_thresh, alpha_mode != 0, grad_sigmas, grad_rgbs);
    return check_launch("composite_rays_train_backward");
}

int n2m_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t* rays_alive, const float* rays_t,
                   const float* rays_o, const float* rays_d, float bound, int contract, float dt_gamma,
                   uint32_t max_steps, uint32_t C, uint32_t H, const uint8_t* grid, const float* nears,
                   const float* fars, float* xyzs, float* dirs, float* ts, const float* noises,
                   n2m_stream_t stream) {
    if (n_alive == 0 || n_step == 0) return 0;
    N2M_REQUIRE(rays_alive && rays_t && rays_o && rays_d && grid && fars && xyzs && dirs && ts && noises,
                "march_rays", "null pointer");
    k_march_infer<<<div_up(n_alive, (uint32_t)kRayBlock), kRayBlock, 0, as_stream(stream)>>>(
        n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, contract != 0, dt_gamma, max_steps, C, H,
        grid, nears, fars, xyzs, dirs, ts, noises);
    return check_launch("march_rays");
}

int n2m_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int alpha_mode,
                       int32_t* rays_alive, float* rays_t, const float* sigmas, const float* rgbs,
                       const float* ts, float* weights_sum, float* depth, float* image,
                       n2m_stream_t stream) {
    if (n_alive == 0) return 0;
    N2M_REQUIRE(rays_alive && rays_t && weights_sum && depth && image, "composite_rays", "null pointer");
    N2M_REQUIRE(n_step == 0 || (sigmas && rgbs && ts), "composite_rays", "null sample pointer");
    k_composite_infer<<<div_up(n_alive, (uint32_t)kRayBlock), kRayBlock, 0, as_stream(stream)>>>(
        n_alive, n_step, T_thresh, alpha_mode != 0, rays_alive, rays_t, sigmas, rgbs, ts, weights_sum, depth, image);
    return check_launch("composite_rays");
}

}  // extern "C"
