// texture.cu -- the stage-1 texture export of the reference (NeRFRenderer.export_stage1 / _export_obj, nerf/renderer.py:298-439) after the
// UV raster (n2m_rasterize of (vt * 2 - 1, 0, 1) / ft, renderer.py:329-338), C ABI include/n2m_b200_texture.h:
//
//   n2m_s1_bake_points     covered texels of a band of rows -> texel index + interpolated position (renderer.py:339-352), compacted
//   n2m_s0_encode_points   the hash-grid gather of stage 0 (encoder_color(x) and x into the 64-column tile image)
//   n2m_s1_geo_feat        geo_feat = sigmoid(color_net([x, encoder_color(x)])) (network.py:159-168) on tensor cores, quantised to uint8
//                          and scattered into the full-resolution feature image (renderer.py:349-376)
//   n2m_s1_inpaint         gutter inpaint (renderer.py:378-394): morphological classification + exact windowed nearest-neighbour search
//   n2m_s1_ssaa_down2      the 2x down-sample (cv2.resize INTER_LINEAR at half size, renderer.py:400-402) and the channel split
// and the viewer's side of the export (renderer.html:54-160):
//   n2m_s1_asset_shade     the fragment shader on the rasterized asset: nearest texel of feat0 / feat1, specular_net in fp32, modes
#include "n2m_common.cuh"
#include "mlp_common.cuh"
#include "../../include/n2m_b200_texture.h"

namespace n2m {
namespace {

// ================================================================================================
// points of one band of rows
// ================================================================================================
__global__ void __launch_bounds__(256)
k_s1_bake_points(const float4* __restrict__ rast, const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t first,
                 uint32_t n, uint32_t cap, uint32_t contract, int32_t* __restrict__ counters, int32_t* __restrict__ pix,
                 float* __restrict__ pts) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t i = first + t;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < n) r = rast[i];
    const bool cov = t < n && r.w > 0.f;
    const uint32_t mask = __ballot_sync(0xffffffffu, cov);
    if (mask == 0) return;
    const uint32_t lane = threadIdx.x & 31;
    const int leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if ((int)lane == leader) base = (uint32_t)atomicAdd(counters + 0, (int)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (!cov) return;
    const uint32_t k = base + __popc(mask & ((1u << lane) - 1u));
    if (k >= cap) return;
    // dr.interpolate(v, rast, f): the expression of k_interp_fwd (raster.cu) and k_s1_points (stage1.cu)
    const uint32_t f = (uint32_t)r.w - 1u;
    const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
    const float u = r.x, vv = r.y, w = 1.f - r.x - r.y;
    float p[3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
        p[a] = u * __ldg(verts + (size_t)i0 * 3 + a) + vv * __ldg(verts + (size_t)i1 * 3 + a) + w * __ldg(verts + (size_t)i2 * 3 + a);
    if (contract) contract_linf(p);         // contract() of renderer.py:25-32 (n2m_common.cuh)
    pix[k] = (int32_t)i;
#pragma unroll
    for (int a = 0; a < 3; ++a) pts[3 * (size_t)k + a] = p[a];
}

// counters[1] = min(counters[0], cap) (the point count the gather and geo_feat read), [2] = overflow flag
__global__ void k_s1_bake_count(int32_t* __restrict__ counters, uint32_t cap) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int32_t c = counters[0];
    counters[1] = c < (int32_t)cap ? c : (int32_t)cap;
    counters[2] = c > (int32_t)cap ? 1 : 0;
}

// ================================================================================================
// geo_feat: color_net on one warpgroup per CTA (wgmma, accumulators in registers)
// ================================================================================================
// The colour rounds of mlp_fwd_tile (mlp_common.cuh) with the same GEMM shapes, K order and fp16 rounding points, so the features equal
// the forward kernel's bit for bit; the sigma and specular nets are not evaluated.  Shared memory: the packed colour weights C1..C3
// (the first 18,432 B of wpack), two A tiles (the TMA load of the CTA's next tile runs underneath the current one) and the hidden tile:
// 67,584 B, three CTAs per SM.
constexpr uint32_t G_W = 0, G_A0 = G_W + W_S1, G_A1 = G_A0 + kTileBytes, G_H = G_A1 + kTileBytes, G_BYTES = G_H + kTileBytes;

__global__ void __launch_bounds__(128)
k_s1_geo_feat(const uint8_t* __restrict__ enc_tiles, const int32_t* __restrict__ counters, const uint8_t* __restrict__ wpack,
              const int32_t* __restrict__ pix, uint8_t* __restrict__ feats, float* __restrict__ feats_f32) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bar[2];
    const uint32_t tid = threadIdx.x;
    const uint32_t M = (uint32_t)counters[1];
    const uint32_t nt = (M + kTile - 1) / kTile;
    if (blockIdx.x >= nt) return;

    if (tid == 0) { wg::mbar_init(&bar[0], 1); wg::mbar_init(&bar[1], 1); wg::mbar_init_fence(); }
    for (uint32_t i = tid; i < W_S1 / 16; i += 128)
        reinterpret_cast<uint4*>(smem + G_W)[i] = __ldg(reinterpret_cast<const uint4*>(wpack) + i);
    sync_before_mma();
    if (tid == 0) bulk_g2s(smem + G_A0, enc_tiles + (size_t)blockIdx.x * kTileBytes, kTileBytes, &bar[0]);
    const uint8_t* sW = smem + G_W;
    uint8_t* sH = smem + G_H;
    const uint32_t r = sample_row(tid);

    uint32_t k = 0;
    for (uint32_t tile = blockIdx.x; tile < nt; tile += gridDim.x, ++k) {
        const uint32_t buf = k & 1u, next = tile + gridDim.x;
        // the other A buffer was last read by the previous tile's round 1, which every warp completed before the barrier ending it
        if (tid == 0 && next < nt) bulk_g2s(smem + (buf ? G_A0 : G_A1), enc_tiles + (size_t)next * kTileBytes, kTileBytes, &bar[buf ^ 1u]);
        wg::mbar_wait(&bar[buf], (k >> 1) & 1u);
        const uint8_t* sA = smem + (buf ? G_A1 : G_A0);
        {   // round 1: color_net.0
            float c[2][32];
            wg::wgmma_fence();
            wg::gemm128<64, 4, false, false>(c, opK(sA, 128), opK(sW + W_C1, 64), false);
            wg::commit(); wg::wait(c);
            epi_store<64, true>(c, sH, tid, nullptr);
        }
        sync_before_mma();
        {   // round 2: color_net.1
            float c[2][32];
            wg::wgmma_fence();
            wg::gemm128<64, 4, false, false>(c, opK(sH, 128), opK(sW + W_C2, 64), false);
            wg::commit(); wg::wait(c);
            sync_before_mma();                           // H2 overwrites H1: every warp's MMAs have read it
            epi_store<64, true>(c, sH, tid, nullptr);
        }
        sync_before_mma();
        {   // round 3: color_net.2, sigmoid, quantisation
            float c[2][8], v[8];
            wg::wgmma_fence();
            wg::gemm128<16, 4, false, false>(c, opK(sH, 128), opK(sW + W_C3, 16), false);
            wg::commit(); wg::wait(c);
            row_cols<16, 6>(c, v, tid);
            const uint32_t j = tile * kTile + r;
            if (j < M) {
                float f[6];
#pragma unroll
                for (int i = 0; i < 6; ++i) f[i] = sigmoid_h(v[i]);
                // (feats * 255).astype(np.uint8) on float32: one rounded product, truncated
                uint32_t q[6];
#pragma unroll
                for (int i = 0; i < 6; ++i) q[i] = (uint32_t)__fmul_rn(f[i], 255.f);
                uint16_t* dst = reinterpret_cast<uint16_t*>(feats + (size_t)pix[j] * 6);
                dst[0] = (uint16_t)(q[0] | (q[1] << 8)); dst[1] = (uint16_t)(q[2] | (q[3] << 8)); dst[2] = (uint16_t)(q[4] | (q[5] << 8));
                if (feats_f32) {
#pragma unroll
                    for (int i = 0; i < 6; ++i) feats_f32[(size_t)j * 6 + i] = f[i];
                }
            }
        }
        sync_before_mma();          // every warp's round-3 MMAs have read H, round 1 has read this A buffer
    }
}

// ================================================================================================
// inpaint
// ================================================================================================
// L1 balls: binary_dilation(mask, iterations=32) is "L1 distance to the mask <= 32", binary_erosion(mask, iterations=3) (border value 0)
// is "every texel within L1 distance 3 lies in the image and in the mask".  An inpaint texel's Euclidean-nearest search texel is as far
// as its nearest mask texel (the nearest mask texel has a non-mask 4-neighbour), at most 32 away, so a separable search over a +-32
// window is exact: a column pass g(x, y) = the smallest dy^2 to a search texel of column x, then a row pass min_dx dx^2 + g(x + dx, y).
constexpr int kDilate = 32, kErode = 3;
constexpr uint8_t C_NONE = 0, C_INTERIOR = 1, C_SEARCH = 2;
constexpr int8_t kNoSource = 127;

// cls: 0 non-mask, 1 mask interior, 2 search
__global__ void __launch_bounds__(256)
k_inpaint_classify(const uint8_t* __restrict__ mask, uint32_t H, uint32_t W, uint8_t* __restrict__ cls) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    uint8_t c = C_NONE;
    if (mask[i]) {
        const int x = (int)(i % W), y = (int)(i / W);
        bool interior = true;
        for (int dy = -kErode; dy <= kErode && interior; ++dy) {
            const int rx = kErode - abs(dy), yy = y + dy;
            for (int dx = -rx; dx <= rx; ++dx) {
                const int xx = x + dx;
                if (yy < 0 || yy >= (int)H || xx < 0 || xx >= (int)W || !mask[(size_t)yy * W + xx]) { interior = false; break; }
            }
        }
        c = interior ? C_INTERIOR : C_SEARCH;
    }
    cls[i] = c;
}

// column pass: hm = smallest |dy| to a mask texel of the column (255: none within 32); gd = the dy of the nearest search texel of the
// column (kNoSource: none within 32), the upper one of two at equal distance
__global__ void __launch_bounds__(256)
k_inpaint_columns(const uint8_t* __restrict__ cls, uint32_t H, uint32_t W, uint8_t* __restrict__ hm, int8_t* __restrict__ gd) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const int x = (int)(i % W), y = (int)(i / W);
    int best_m = 255, best_s = kNoSource, best_s2 = 1 << 30;
    const int lo = max(-kDilate, -y), hi = min(kDilate, (int)H - 1 - y);
    for (int dy = lo; dy <= hi; ++dy) {
        const uint8_t c = cls[(size_t)(y + dy) * W + x];
        if (c != C_NONE) best_m = min(best_m, abs(dy));
        if (c == C_SEARCH && dy * dy < best_s2) { best_s2 = dy * dy; best_s = dy; }
    }
    hm[i] = (uint8_t)best_m;
    gd[i] = (int8_t)best_s;
}

// row pass: classify the non-mask texels (inpaint: L1 distance to the mask <= 32) and copy the nearest search texel's features;
// ties: smallest distance^2, then smallest source row, then smallest source column
__global__ void __launch_bounds__(256)
k_inpaint_rows(uint8_t* __restrict__ feats, const uint8_t* __restrict__ cls, const uint8_t* __restrict__ hm, const int8_t* __restrict__ gd,
               uint32_t H, uint32_t W, int32_t* __restrict__ source) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    if (cls[i] != C_NONE) {
        if (source) source[i] = -1;
        return;
    }
    const int x = (int)(i % W), y = (int)(i / W);
    const size_t row = (size_t)y * W;
    int best_l1 = 1 << 30, best_d2 = 1 << 30, best_y = 0, best_x = -1;
    const int lo = max(-kDilate, -x), hi = min(kDilate, (int)W - 1 - x);
    for (int dx = lo; dx <= hi; ++dx) {
        const uint8_t m = hm[row + x + dx];
        if (m != 255) best_l1 = min(best_l1, abs(dx) + (int)m);
        const int g = gd[row + x + dx];
        if (g != kNoSource) {
            const int d2 = dx * dx + g * g, sy = y + g;
            if (d2 < best_d2 || (d2 == best_d2 && sy < best_y)) { best_d2 = d2; best_y = sy; best_x = x + dx; }
        }
    }
    uint16_t* dst = reinterpret_cast<uint16_t*>(feats + (size_t)i * 6);
    if (best_l1 <= kDilate && best_x >= 0) {
        const size_t s = (size_t)best_y * W + best_x;
        const uint16_t* src = reinterpret_cast<const uint16_t*>(feats + s * 6);
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
        if (source) source[i] = (int32_t)s;
    } else {
        dst[0] = 0; dst[1] = 0; dst[2] = 0;
        if (source) source[i] = -1;
    }
}

// ================================================================================================
// down-sample + channel split
// ================================================================================================
__global__ void __launch_bounds__(256)
k_ssaa_down2(const uint8_t* __restrict__ feats, uint32_t h0, uint32_t w0, uint32_t ssaa, uint8_t* __restrict__ feat0,
             uint8_t* __restrict__ feat1) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= h0 * w0) return;
    const uint32_t y = q / w0, x = q % w0;
    uint8_t out[6];
    if (ssaa == 1) {
#pragma unroll
        for (int c = 0; c < 6; ++c) out[c] = feats[(size_t)q * 6 + c];
    } else {
        const size_t w = (size_t)w0 * 2;
        const uint8_t* a = feats + ((size_t)(2 * y) * w + 2 * x) * 6;
        const uint8_t* b = a + w * 6;
#pragma unroll
        for (int c = 0; c < 6; ++c) out[c] = (uint8_t)(((uint32_t)a[c] + a[6 + c] + b[c] + b[6 + c] + 2u) >> 2);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { feat0[(size_t)q * 3 + c] = out[c]; feat1[(size_t)q * 3 + c] = out[3 + c]; }
}

// ================================================================================================
// the exported asset as the viewer draws it (renderer.html:54-160, textures :441-450)
// ================================================================================================
constexpr int kSpecIn = 6, kSpecHidden = 32, kSpecOut = 3, kSpecWeights = kSpecHidden * kSpecIn + kSpecOut * kSpecHidden;

// u * a0 + v * a1 + (1 - u - v) * a2 with every product and sum rounded on its own (no contraction), so a float32 restatement of the
// expression gives the same bits and the same nearest texel
__device__ __forceinline__ float bary_rn(float u, float v, float ww, float a0, float a1, float a2) {
    return __fadd_rn(__fadd_rn(__fmul_rn(u, a0), __fmul_rn(v, a1)), __fmul_rn(ww, a2));
}

// nearest texel of an RGB uint8 texture [H,W,3] at (s, t), three.js NearestFilter + flipY + clamp-to-edge
__device__ __forceinline__ const uint8_t* nearest_texel(const uint8_t* tex, int H, int W, float s, float t) {
    const int x = min(max((int)floorf(__fmul_rn(s, (float)W)), 0), W - 1);
    const int y = min(max(H - 1 - (int)floorf(__fmul_rn(t, (float)H)), 0), H - 1);
    return tex + ((size_t)y * W + x) * 3;
}

// one thread per super-sample: covered ones -> (r, g, b, 1), the others -> 0
__global__ void __launch_bounds__(256)
k_s1_asset_shade(const float4* __restrict__ rast, uint32_t n, const float* __restrict__ verts, const int32_t* __restrict__ tri,
                 const float* __restrict__ st, const int32_t* __restrict__ ft, const int32_t* __restrict__ face_offsets, uint32_t cascades,
                 const uint8_t* const* __restrict__ feat0, const uint8_t* const* __restrict__ feat1, const int32_t* __restrict__ tex_size,
                 const float* __restrict__ mlp, float cx, float cy, float cz, uint32_t mode, float4* __restrict__ img) {
    __shared__ float sw[kSpecWeights];
    for (int k = threadIdx.x; k < kSpecWeights; k += blockDim.x) sw[k] = mlp[k];
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 r = rast[i];
    if (!(r.w > 0.f)) { img[i] = make_float4(0.f, 0.f, 0.f, 0.f); return; }
    const int32_t f = (int32_t)r.w - 1;
    uint32_t c = 0;
    while (c + 1 < cascades && f >= face_offsets[c + 1]) ++c;
    const float u = r.x, v = r.y, ww = __fsub_rn(__fsub_rn(1.f, r.x), r.y);
    const int t0 = ft[3 * f], t1 = ft[3 * f + 1], t2 = ft[3 * f + 2];
    const float s = bary_rn(u, v, ww, st[2 * t0], st[2 * t1], st[2 * t2]);
    const float t = bary_rn(u, v, ww, st[2 * t0 + 1], st[2 * t1 + 1], st[2 * t2 + 1]);
    const int H = tex_size[2 * c], W = tex_size[2 * c + 1];
    const uint8_t* d = nearest_texel(feat0[c], H, W, s, t);
    float rgb[3] = {d[0] / 255.f, d[1] / 255.f, d[2] / 255.f};
    if (mode != 1) {
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        const float cam[3] = {cx, cy, cz};
        float x[kSpecIn];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            x[a] = bary_rn(u, v, ww, verts[3 * (size_t)i0 + a], verts[3 * (size_t)i1 + a], verts[3 * (size_t)i2 + a]) - cam[a];
        const float inv_len = 1.f / sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);        // normalize(rayDirection)
#pragma unroll
        for (int a = 0; a < 3; ++a) x[a] *= inv_len;
        const uint8_t* p = nearest_texel(feat1[c], H, W, s, t);
#pragma unroll
        for (int a = 0; a < 3; ++a) x[3 + a] = p[a] / 255.f;
        float o[kSpecOut] = {0.f, 0.f, 0.f};
#pragma unroll 4
        for (int j = 0; j < kSpecHidden; ++j) {
            float hj = 0.f;
#pragma unroll
            for (int k = 0; k < kSpecIn; ++k) hj += sw[j * kSpecIn + k] * x[k];
            hj = fmaxf(hj, 0.f);
#pragma unroll
            for (int q = 0; q < kSpecOut; ++q) o[q] += sw[kSpecHidden * kSpecIn + q * kSpecHidden + j] * hj;
        }
#pragma unroll
        for (int q = 0; q < kSpecOut; ++q) {
            const float spec = 1.f / (1.f + expf(-o[q]));
            rgb[q] = mode == 2 ? spec : fminf(fmaxf(rgb[q] + spec, 0.f), 1.f);
        }
    }
    img[i] = make_float4(rgb[0], rgb[1], rgb[2], 1.f);
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_s1_bake_points(const float* rast, const float* verts, const int32_t* tri, uint32_t W, uint32_t y0, uint32_t y1, uint32_t cap,
                       uint32_t contract, int32_t* counters, int32_t* pix, float* pts, n2m_stream_t stream) {
    N2M_REQUIRE(rast && verts && tri && counters && pix && pts, "s1_bake_points", "null pointer");
    N2M_REQUIRE(W > 0 && y1 >= y0 && (uint64_t)y1 * W < (1ull << 31), "s1_bake_points", "bad band");
    cudaStream_t st = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), st);
    if (e != cudaSuccess) return fail("s1_bake_points(memset)", cudaGetErrorString(e));
    const uint32_t n = (y1 - y0) * W;
    if (n > 0) {
        k_s1_bake_points<<<div_up(n, 256u), 256, 0, st>>>(reinterpret_cast<const float4*>(rast), verts, tri, y0 * W, n, cap, contract, counters,
                                                         pix, pts);
        if (int err = check_launch("s1_bake_points")) return err;
    }
    k_s1_bake_count<<<1, 32, 0, st>>>(counters, cap);
    return check_launch("s1_bake_points(count)");
}

int n2m_s1_geo_feat(const void* enc_tiles, const int32_t* counters, uint32_t Pcap, const void* wpack, const int32_t* pix, uint8_t* feats,
                    float* feats_f32, n2m_stream_t stream) {
    N2M_REQUIRE(enc_tiles && counters && wpack && pix && feats, "s1_geo_feat", "null pointer");
    N2M_REQUIRE(Pcap % kTile == 0 && Pcap > 0, "s1_geo_feat", "Pcap must be a positive multiple of 128");
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(k_s1_geo_feat, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_BYTES);
        if (e != cudaSuccess) return fail("s1_geo_feat(attribute)", cudaGetErrorString(e));
        attr = true;
    }
    const uint32_t grid = min(Pcap / kTile, (uint32_t)(3 * num_sms()));          // 67.6 KB of shared memory: 3 CTAs per SM
    k_s1_geo_feat<<<grid, 128, G_BYTES, as_stream(stream)>>>(static_cast<const uint8_t*>(enc_tiles), counters, static_cast<const uint8_t*>(wpack),
                                                             pix, feats, feats_f32);
    return check_launch("s1_geo_feat");
}

int n2m_s1_inpaint(uint8_t* feats, const uint8_t* mask, uint32_t H, uint32_t W, uint8_t* scratch, int32_t* source, n2m_stream_t stream) {
    N2M_REQUIRE(feats && mask && scratch, "s1_inpaint", "null pointer");
    N2M_REQUIRE(H > 0 && W > 0 && (uint64_t)H * W < (1ull << 31), "s1_inpaint", "bad resolution");
    cudaStream_t st = as_stream(stream);
    const uint32_t n = H * W, g = div_up(n, 256u);
    uint8_t* cls = scratch;
    uint8_t* hm = scratch + n;
    int8_t* gd = reinterpret_cast<int8_t*>(scratch + 2 * (size_t)n);
    k_inpaint_classify<<<g, 256, 0, st>>>(mask, H, W, cls);
    if (int e = check_launch("s1_inpaint(classify)")) return e;
    k_inpaint_columns<<<g, 256, 0, st>>>(cls, H, W, hm, gd);
    if (int e = check_launch("s1_inpaint(columns)")) return e;
    k_inpaint_rows<<<g, 256, 0, st>>>(feats, cls, hm, gd, H, W, source);
    return check_launch("s1_inpaint(rows)");
}

int n2m_s1_ssaa_down2(const uint8_t* feats, uint32_t h0, uint32_t w0, uint32_t ssaa, uint8_t* feat0, uint8_t* feat1, n2m_stream_t stream) {
    N2M_REQUIRE(feats && feat0 && feat1, "s1_ssaa_down2", "null pointer");
    N2M_REQUIRE(ssaa == 1 || ssaa == 2, "s1_ssaa_down2", "ssaa must be 1 or 2");
    N2M_REQUIRE((uint64_t)h0 * ssaa * w0 * ssaa < (1ull << 31), "s1_ssaa_down2", "bad resolution");
    if (h0 == 0 || w0 == 0) return 0;
    k_ssaa_down2<<<div_up(h0 * w0, 256u), 256, 0, as_stream(stream)>>>(feats, h0, w0, ssaa, feat0, feat1);
    return check_launch("s1_ssaa_down2");
}

int n2m_s1_asset_shade(const float* rast, uint32_t num_pixels, const float* verts, const int32_t* tri, const float* st, const int32_t* ft,
                       const int32_t* face_offsets, uint32_t cascades, const void* const* feat0, const void* const* feat1, const int32_t* tex_size,
                       const float* mlp, float cam_x, float cam_y, float cam_z, uint32_t mode, float* img, n2m_stream_t stream) {
    N2M_REQUIRE(rast && verts && tri && st && ft && face_offsets && feat0 && feat1 && tex_size && mlp && img, "s1_asset_shade", "null pointer");
    N2M_REQUIRE(cascades >= 1, "s1_asset_shade", "at least one cascade");
    N2M_REQUIRE(mode >= 1 && mode <= 3, "s1_asset_shade", "mode must be 1 (diffuse), 2 (specular) or 3 (full)");
    if (num_pixels == 0) return 0;
    k_s1_asset_shade<<<div_up(num_pixels, 256u), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(rast), num_pixels, verts, tri, st, ft, face_offsets, cascades,
        reinterpret_cast<const uint8_t* const*>(feat0), reinterpret_cast<const uint8_t* const*>(feat1), tex_size, mlp, cam_x, cam_y, cam_z, mode,
        reinterpret_cast<float4*>(img));
    return check_launch("s1_asset_shade");
}

}  // extern "C"
