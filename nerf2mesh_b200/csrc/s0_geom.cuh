// s0_geom.cuh -- sample / lattice geometry shared by the gather, scatter and fused kernels of the stage-0 train path
// (stage0.cu, fused.cu): tile-image constants, the interleaved table entry, sample reconstruction from a march record, hash /
// dense corner indices and trilinear weights of one level (gridencoder.cu:50-84,88-196 of the reference, same expressions).
// Everything here is per level, so a kernel may visit the levels of a sample in any order or split them over launches / work items:
// the scatter and TV passes of stage0.cu visit one level group of a tile at a time, so that the REDs of the CTAs running together
// stay inside one group's slice of the gradient table (8 MiB per hashed level) instead of the whole 97.6 MB, twice the H100's L2.
#pragma once
#include "n2m_common.cuh"
#include "../../include/n2m_b200_fused.h"

namespace n2m {
namespace {

constexpr uint32_t kTile = 128;            // samples per tile image
constexpr uint32_t kTileCols = 64;         // fp16 features per sample
constexpr uint32_t kTileBytes = kTile * kTileCols * 2;
constexpr uint32_t kChunkBytes = kTile * 16;   // one 8-column chunk of a 128-row tile
constexpr uint32_t kColXyz = 0, kColDens = 3, kColColor = 19, kColDir = 51, kColCode = 54;
constexpr uint32_t kMaxIndDim = kTileCols - kColCode;      // appearance-code columns the tile image has room for
constexpr uint32_t kLevels = 16;

struct __align__(8) TableEntry { float d; __half2 c; };

// ------------------------------------------------------------------------------------------------
// shared sample geometry
// ------------------------------------------------------------------------------------------------
struct Sample {
    float x, y, z;        // (contracted) position handed to the network
    float u, v, w;        // position mapped to [0,1]^3 for the grid
    float dx, dy, dz;     // raw ray direction
};

__device__ __forceinline__ Sample sample_of(const float4 rec, const float* __restrict__ rays_o,
                                            const float* __restrict__ rays_d, const n2m_s0_params& p) {
    Sample s;
    const int n = __float_as_int(rec.w);
    const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
    s.dx = rays_d[3 * n]; s.dy = rays_d[3 * n + 1]; s.dz = rays_d[3 * n + 2];
    const float t = rec.x;
    s.x = clampf(ox + t * s.dx, -p.bound, p.bound);
    s.y = clampf(oy + t * s.dy, -p.bound, p.bound);
    s.z = clampf(oz + t * s.dz, -p.bound, p.bound);
    const float mag = fmaxf(fabsf(s.x), fmaxf(fabsf(s.y), fabsf(s.z)));
    if (p.contract && mag > 1) {
        const float k = (2 - 1 / mag) / mag;
        s.x *= k; s.y *= k; s.z *= k;
    }
    // GridEncoder.forward: (x + bound) / (2 * bound); torch divides by a python scalar as a
    // multiplication with float32(1)/float32(2*bound)
    s.u = __fmul_rn(__fadd_rn(s.x, p.grid_bound), p.inv_2gb);
    s.v = __fmul_rn(__fadd_rn(s.y, p.grid_bound), p.inv_2gb);
    s.w = __fmul_rn(__fadd_rn(s.z, p.grid_bound), p.inv_2gb);
    return s;
}

// lattice geometry of one level for one sample: the 8 corner rows and trilinear weights
struct Corners {
    uint32_t row[8];
    float w[8];
};

struct LevelGeom {
    float scale;
    uint32_t res, rows, row0;
};

__device__ __forceinline__ LevelGeom level_geom(const int32_t* __restrict__ offsets, uint32_t level, float S, uint32_t H) {
    LevelGeom g;
    g.row0 = (uint32_t)offsets[level];
    g.rows = (uint32_t)offsets[level + 1] - g.row0;
    g.scale = exp2f(level * S) * H - 1.0f;          // gridencoder.cu:138 (same expression, same flags)
    g.res = (uint32_t)ceil(g.scale) + 1;
    return g;
}

// index % rows of gridencoder.cu:84.  A dense level's index is already below its row count ((res + 1)^3 <= rows and every
// coordinate <= res), a hashed level has 2^k rows: the integer division (~20 instructions per corner) is kept only as the guard
__device__ __forceinline__ uint32_t wrap_row(uint32_t raw, uint32_t rows, bool pow2) {
    if (pow2) return raw & (rows - 1);
    if (raw >= rows) raw %= rows;
    return raw;
}

// returns false when the sample is outside [0,1]^3 (the encoders output zeros there)
__device__ __forceinline__ void corners_of(const LevelGeom& g, float u, float v, float w, Corners& c,
                                           uint32_t (&base)[3], bool& hashed, uint32_t* left = nullptr) {
    const float pu = u * g.scale + 0.5f, pv = v * g.scale + 0.5f, pw = w * g.scale + 0.5f;
    const float fu0 = floorf(pu), fv0 = floorf(pv), fw0 = floorf(pw);
    const uint32_t x0 = fu0, y0 = fv0, z0 = fw0;
    base[0] = x0; base[1] = y0; base[2] = z0;
    const float fx = pu - (float)x0, fy = pv - (float)y0, fz = pw - (float)z0;
    // index: dense while the running stride fits the level's rows, else hashed (gridencoder.cu:66-84)
    const uint32_t s1 = g.res + 1;
    uint32_t stride = 1;
    uint32_t mx = 0, my = 0, mz = 0;          // dense multipliers (0 = dimension not accumulated)
    if (stride <= g.rows) { mx = stride; stride *= s1; }
    if (stride <= g.rows) { my = stride; stride *= s1; }
    if (stride <= g.rows) { mz = stride; stride *= s1; }
    hashed = stride > g.rows;
    uint32_t xs[2], ys[2], zs[2];
    if (hashed) {
        xs[0] = x0;                 xs[1] = x0 + 1u;
        ys[0] = y0 * 2654435761u;   ys[1] = ys[0] + 2654435761u;
        zs[0] = z0 * 805459861u;    zs[1] = zs[0] + 805459861u;
    } else {
        xs[0] = x0 * mx;            xs[1] = xs[0] + mx;
        ys[0] = y0 * my;            ys[1] = ys[0] + my;
        zs[0] = z0 * mz;            zs[1] = zs[0] + mz;
    }
    const float wx[2] = {1 - fx, fx}, wy[2] = {1 - fy, fy}, wz[2] = {1 - fz, fz};
    const bool pow2 = (g.rows & (g.rows - 1)) == 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int ix = k & 1, iy = (k >> 1) & 1, iz = (k >> 2) & 1;
        const uint32_t raw = hashed ? (xs[ix] ^ ys[iy] ^ zs[iz]) : (xs[ix] + ys[iy] + zs[iz]);
        c.row[k] = wrap_row(raw, g.rows, pow2);
        c.w[k] = wx[ix] * wy[iy] * wz[iz];
    }
    if (left) {     // rows of the cells at base - 1 along each axis (TV neighbours); callers check base[d] > 0
        uint32_t lx, ly, lz;
        if (hashed) {
            lx = (x0 - 1u) ^ ys[0] ^ zs[0];
            ly = xs[0] ^ (ys[0] - 2654435761u) ^ zs[0];
            lz = xs[0] ^ ys[0] ^ (zs[0] - 805459861u);
        } else {
            lx = xs[0] - mx + ys[0] + zs[0];
            ly = xs[0] + ys[0] - my + zs[0];
            lz = xs[0] + ys[0] + zs[0] - mz;
        }
        left[0] = wrap_row(lx, g.rows, pow2);
        left[1] = wrap_row(ly, g.rows, pow2);
        left[2] = wrap_row(lz, g.rows, pow2);
    }
}

__device__ __forceinline__ uint32_t pack2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// ---- gather of one sample: the 64 fp16 columns of its tile-image row (xyz | 16 density features | 32 colour features | unit direction
// | p.ind_dim appearance-code columns | zeros), shared by the stand-alone gather kernel (stage0.cu) and the fused forward kernel (fused.cu).
// POINTS = false: the sample comes from march record j; POINTS = true: explicit position rays_o[j] / direction rays_d[j] (density-grid
// update, stage 1, tests).  Codes (include/n2m_b200_fused.h "Per-image appearance codes"): none when `codes` is null, else row
// ray_img[ray of record j] of the code table `codes`, or the one row at `codes` when ray_img is null; rounded to fp16 by the tile store
// as autocast rounds the concatenated input of color_net.0.
// Returns false when row j is outside [pr.lo, pr.hi) (a row of another part, or past the last sample: all zeros). ----
template <bool POINTS>
__device__ __forceinline__ bool
encode_fwd_features(const n2m_s0_params& p, const float4* __restrict__ recs, const float* __restrict__ rays_o,
                    const float* __restrict__ rays_d, const TableEntry* __restrict__ table, const int32_t* __restrict__ offsets,
                    const PartRange pr, uint32_t j, float (&feat)[kTileCols], const float* __restrict__ codes = nullptr,
                    const int32_t* __restrict__ ray_img = nullptr) {
#pragma unroll
    for (uint32_t i = 0; i < kTileCols; ++i) feat[i] = 0.f;
    Sample s;
    const bool own = j >= pr.lo && j < pr.hi;        // rows of a boundary tile outside [lo, hi) belong to another part
    bool active = own;
    if (own) {
        if (POINTS) {
            s.x = rays_o[3 * j]; s.y = rays_o[3 * j + 1]; s.z = rays_o[3 * j + 2];
            s.u = __fmul_rn(__fadd_rn(s.x, p.grid_bound), p.inv_2gb);
            s.v = __fmul_rn(__fadd_rn(s.y, p.grid_bound), p.inv_2gb);
            s.w = __fmul_rn(__fadd_rn(s.z, p.grid_bound), p.inv_2gb);
            s.dx = rays_d ? rays_d[3 * j] : 0.f; s.dy = rays_d ? rays_d[3 * j + 1] : 0.f; s.dz = rays_d ? rays_d[3 * j + 2] : 1.f;
        } else
        s = sample_of(recs[j], rays_o, rays_d, p);
        feat[kColXyz] = s.x; feat[kColXyz + 1] = s.y; feat[kColXyz + 2] = s.z;
        // safe_normalize (utils.py:41-42): d / sqrt(clamp(sum d^2, 1e-20))
        const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(s.dx, s.dx), __fmul_rn(s.dy, s.dy)), __fmul_rn(s.dz, s.dz));
        const float nrm = __fsqrt_rn(fmaxf(n2, 1e-20f));
        feat[kColDir] = __fdiv_rn(s.dx, nrm); feat[kColDir + 1] = __fdiv_rn(s.dy, nrm); feat[kColDir + 2] = __fdiv_rn(s.dz, nrm);
        active = !((s.u < 0 || s.u > 1) || (s.v < 0 || s.v > 1) || (s.w < 0 || s.w > 1));
    } else {
        s.x = s.y = s.z = s.u = s.v = s.w = 0.5f; s.dx = s.dy = s.dz = 0.f;
    }
#pragma unroll
    for (uint32_t l = 0; l < kLevels; ++l) {
        const LevelGeom g = level_geom(offsets, l, p.S, p.base_res);
        Corners c; uint32_t base[3]; bool hashed;
        corners_of(g, s.u, s.v, s.w, c, base, hashed, nullptr);
        const TableEntry* tab = table + g.row0;
        if (active) {
            uint2 raw[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) raw[k] = __ldg(reinterpret_cast<const uint2*>(tab + c.row[k]));
            float d = 0.f, c0 = 0.f, c1 = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float2 cc = __half22float2(*reinterpret_cast<const __half2*>(&raw[k].y));
                d += c.w[k] * __uint_as_float(raw[k].x);
                c0 += c.w[k] * cc.x;
                c1 += c.w[k] * cc.y;
            }
            feat[kColDens + l] = d;
            feat[kColColor + 2 * l] = c0;
            feat[kColColor + 2 * l + 1] = c1;
        }
    }
    // after the level walk, so that the code columns hold no register across it
    if (codes && own) {
        const uint32_t D = p.ind_dim;
        const float* row = codes;
        if (!POINTS && ray_img) row += (size_t)ray_img[__float_as_int(recs[j].w)] * D;
#pragma unroll
        for (uint32_t k = 0; k < kMaxIndDim; ++k)
            if (k < D) feat[kColCode + k] = __ldg(row + k);
    }
    return own;
}

// one fp16 gradient column of a tile-image row (`row` = the row's first byte in chunk 0)
__device__ __forceinline__ float denc_col(const uint8_t* row, uint32_t col) {
    return __half2float(__ldg(reinterpret_cast<const __half*>(row + (col >> 3) * kChunkBytes + (col & 7) * 2)));
}

// row r of a tile image at `img` (global or shared): 8 chunks of 16 bytes, each chunk 2 KiB apart
__device__ __forceinline__ void store_tile_row(uint8_t* img, uint32_t r, const float (&feat)[kTileCols]) {
    uint8_t* dst = img + r * 16;
#pragma unroll
    for (uint32_t ch = 0; ch < 8; ++ch) {
        uint4 q;
        q.x = pack2(feat[8 * ch + 0], feat[8 * ch + 1]);
        q.y = pack2(feat[8 * ch + 2], feat[8 * ch + 3]);
        q.z = pack2(feat[8 * ch + 4], feat[8 * ch + 5]);
        q.w = pack2(feat[8 * ch + 6], feat[8 * ch + 7]);
        *reinterpret_cast<uint4*>(dst + ch * kChunkBytes) = q;
    }
}

}  // namespace
}  // namespace n2m
