// gridencoder.cu -- multiresolution hash / tiled grid encoding for sm_90a (unfused operator form).
//
// Replaces the native layer behind the reference's `grid_encode` / `GridEncoder`
// (reference: gridencoder/src/gridencoder.cu).  Level geometry, corner order, hashing and the
// rounding behaviour of the fp16 path follow the reference so that forward outputs are
// bit-identical on identical inputs; loads are vectorised per corner (one 4/8/16-byte access
// covers all C features), the scatter uses vector reductions (red.global.add.v2.f32 /
// .noftz.f16x2), and every launch goes to the caller's stream.
#include "n2m_common.cuh"
#include <type_traits>

namespace n2m {
namespace {

// ---- scalar semantics of the two table dtypes ---------------------------------------------------
// fp32: plain float arithmetic (the compiler contracts a += w * g into one FFMA, as it does for
// the reference).  fp16: the reference accumulates in at::Half, whose operators round the product
// to half and then round the sum to half again (torch/headeronly/util/Half.h:501-531); reproduce
// exactly that double rounding.
template <typename T> struct Acc;
template <> struct Acc<float> {
    using type = float;
    static __device__ __forceinline__ float zero() { return 0.f; }
    static __device__ __forceinline__ float to_f(float v) { return v; }
    static __device__ __forceinline__ float from_f(float v) { return v; }
    static __device__ __forceinline__ void fma_w(float& acc, float w, float g) { acc += w * g; }
    static __device__ __forceinline__ float sub(float a, float b) { return a - b; }
};
template <> struct Acc<__half> {
    using type = __half;
    static __device__ __forceinline__ __half zero() { return __float2half_rn(0.f); }
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
    static __device__ __forceinline__ void fma_w(__half& acc, float w, __half g) {
        const __half p = __float2half_rn(w * __half2float(g));
        acc = __float2half_rn(__half2float(acc) + __half2float(p));
    }
    static __device__ __forceinline__ __half sub(__half a, __half b) {
        return __float2half_rn(__half2float(a) - __half2float(b));
    }
};

// vector type that moves all C features of one table row in a single access
template <typename T, uint32_t C> struct RowVec { using type = void; };
template <> struct RowVec<float, 1> { using type = float; };
template <> struct RowVec<float, 2> { using type = float2; };
template <> struct RowVec<float, 4> { using type = float4; };
template <> struct RowVec<float, 8> { using type = float4; };      // two accesses
template <> struct RowVec<__half, 1> { using type = __half; };
template <> struct RowVec<__half, 2> { using type = __half2; };
template <> struct RowVec<__half, 4> { using type = uint2; };
template <> struct RowVec<__half, 8> { using type = uint4; };

template <typename T, uint32_t C>
__device__ __forceinline__ void load_row(const T* __restrict__ row, T (&out)[C]) {
    using V = typename RowVec<T, C>::type;
    constexpr uint32_t NV = (sizeof(T) * C) / sizeof(V);
    V tmp[NV];
#pragma unroll
    for (uint32_t i = 0; i < NV; ++i) tmp[i] = __ldg(reinterpret_cast<const V*>(row) + i);
    const T* p = reinterpret_cast<const T*>(tmp);
#pragma unroll
    for (uint32_t c = 0; c < C; ++c) out[c] = p[c];
}

// ---- level geometry -------------------------------------------------------------------------
struct Level {
    float scale;
    uint32_t res;        // resolution (cells per axis + 1 when !align_corners is added at use)
    uint32_t rows;       // padded row count of this level = "hashmap_size"
    uint32_t row0;       // first row of the level
};

__device__ __forceinline__ Level level_geom(const int32_t* __restrict__ offsets, uint32_t level, float S, uint32_t H) {
    Level g;
    g.row0 = (uint32_t)offsets[level];
    g.rows = (uint32_t)offsets[level + 1] - g.row0;
    g.scale = exp2f(level * S) * H - 1.0f;              // gridencoder.cu:138
    g.res = (uint32_t)ceil(g.scale) + 1;                // gridencoder.cu:139
    return g;
}

// per-axis multipliers of the spatial hash (instant-ngp's "coherent" primes, gridencoder.cu:54)
template <uint32_t AXIS> __device__ __forceinline__ constexpr uint32_t hash_prime() {
    return AXIS == 0 ? 1u : AXIS == 1 ? 2654435761u : AXIS == 2 ? 805459861u : AXIS == 3 ? 3674653429u
         : AXIS == 4 ? 2097192037u : AXIS == 5 ? 1434869437u : 2165219737u;
}
template <uint32_t D, uint32_t AXIS = 0>
__device__ __forceinline__ uint32_t hash_xor(const uint32_t (&p)[D]) {
    if constexpr (AXIS >= D) return 0u;
    else return (p[AXIS] * hash_prime<AXIS>()) ^ hash_xor<D, AXIS + 1>(p);
}

// row index of a lattice point (gridencoder.cu:66-84): dense while the running stride still fits
// the level's rows, else the XOR-of-primes hash (hash gridtype only); always wrapped by `rows`.
template <uint32_t D>
__device__ __forceinline__ uint32_t lattice_row(const uint32_t (&p)[D], const Level& g, uint32_t gridtype, bool align_corners) {
    uint32_t stride = 1, idx = 0;
    const uint32_t step = align_corners ? g.res : (g.res + 1);
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) {
        if (stride <= g.rows) {
            idx += p[d] * stride;
            stride *= step;
        }
    }
    if (gridtype == 0 && stride > g.rows) {
        idx = hash_xor<D>(p);
    }
    // idx % rows without the integer division where it is an identity or a mask (dense levels, 2^k-row hashed levels)
    if ((g.rows & (g.rows - 1)) == 0) return idx & (g.rows - 1);
    return idx < g.rows ? idx : idx % g.rows;
}

__device__ __forceinline__ float smooth(float v) { return v * v * (3.0f - 2.0f * v); }
__device__ __forceinline__ float smooth_d(float v) { return 6 * v * (1.0f - v); }

template <uint32_t D>
__device__ __forceinline__ bool outside_unit(const float* __restrict__ x) {
    bool oob = false;
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) oob |= (x[d] < 0 || x[d] > 1);
    return oob;
}

// fractional position + base lattice point of a sample at one level (gridencoder.cu:146-158)
template <uint32_t D>
__device__ __forceinline__ void locate(const float* __restrict__ x, const Level& g, bool align_corners, uint32_t interp,
                                       float (&frac)[D], float (&dfrac)[D], uint32_t (&base)[D]) {
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) {
        float p = x[d] * g.scale + (align_corners ? 0.0f : 0.5f);
        base[d] = floorf(p);
        p -= (float)base[d];
        if (interp == 1) { dfrac[d] = smooth_d(p); p = smooth(p); }
        else dfrac[d] = 1.0f;
        frac[d] = p;
    }
}

// ---- forward --------------------------------------------------------------------------------
template <typename T, uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256)
k_grid_fwd(const float* __restrict__ inputs, const T* __restrict__ table, const int32_t* __restrict__ offsets,
           T* __restrict__ outputs, uint32_t B, uint32_t L, float S, uint32_t H, T* __restrict__ dy_dx,
           uint32_t gridtype, bool align_corners, uint32_t interp) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    const float* x = inputs + (size_t)b * D;
    T* out = outputs + ((size_t)level * B + b) * C;
    T* dout = dy_dx ? dy_dx + ((size_t)b * L + level) * D * C : nullptr;     // [B, L, D, C]

    if (outside_unit<D>(x)) {          // out-of-range sample: zeros (gridencoder.cu:110-135)
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) out[c] = Acc<T>::zero();
        if (dout) {
#pragma unroll
            for (uint32_t i = 0; i < D * C; ++i) dout[i] = Acc<T>::zero();
        }
        return;
    }

    const Level g = level_geom(offsets, level, S, H);
    const T* tab = table + (size_t)g.row0 * C;
    float frac[D], dfrac[D];
    uint32_t base[D];
    locate<D>(x, g, align_corners, interp, frac, dfrac, base);

    T acc[C];
#pragma unroll
    for (uint32_t c = 0; c < C; ++c) acc[c] = Acc<T>::zero();

#pragma unroll
    for (uint32_t corner = 0; corner < (1u << D); ++corner) {
        float w = 1;
        uint32_t p[D];
#pragma unroll
        for (uint32_t d = 0; d < D; ++d) {
            if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; p[d] = base[d]; }
            else { w *= frac[d]; p[d] = base[d] + 1; }
        }
        const uint32_t row = lattice_row<D>(p, g, gridtype, align_corners);
        T v[C];
        load_row<T, C>(tab + (size_t)row * C, v);
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) Acc<T>::fma_w(acc[c], w, v[c]);
    }
#pragma unroll
    for (uint32_t c = 0; c < C; ++c) out[c] = acc[c];

    if (dout) {                       // d(out)/d(x) per axis (gridencoder.cu:200-243)
#pragma unroll
        for (uint32_t gd = 0; gd < D; ++gd) {
            T gacc[C];
#pragma unroll
            for (uint32_t c = 0; c < C; ++c) gacc[c] = Acc<T>::zero();
#pragma unroll
            for (uint32_t corner = 0; corner < (1u << (D - 1)); ++corner) {
                float w = g.scale;
                uint32_t p[D];
#pragma unroll
                for (uint32_t nd = 0; nd < D - 1; ++nd) {
                    const uint32_t d = (nd >= gd) ? (nd + 1) : nd;
                    if ((corner & (1u << nd)) == 0) { w *= 1 - frac[d]; p[d] = base[d]; }
                    else { w *= frac[d]; p[d] = base[d] + 1; }
                }
                p[gd] = base[gd];
                const uint32_t r_lo = lattice_row<D>(p, g, gridtype, align_corners);
                p[gd] = base[gd] + 1;
                const uint32_t r_hi = lattice_row<D>(p, g, gridtype, align_corners);
                T lo[C], hi[C];
                load_row<T, C>(tab + (size_t)r_lo * C, lo);
                load_row<T, C>(tab + (size_t)r_hi * C, hi);
#pragma unroll
                for (uint32_t c = 0; c < C; ++c) {
                    if constexpr (std::is_same<T, float>::value) {
                        gacc[c] += w * (hi[c] - lo[c]) * dfrac[gd];
                    } else {
                        // Half - Half rounds to half; (w * diff) * dfrac is float; += rounds twice
                        const __half diff = Acc<T>::sub(hi[c], lo[c]);
                        const float term = w * __half2float(diff) * dfrac[gd];
                        const __half th = __float2half_rn(term);
                        gacc[c] = __float2half_rn(__half2float(gacc[c]) + __half2float(th));
                    }
                }
            }
#pragma unroll
            for (uint32_t c = 0; c < C; ++c) dout[gd * C + c] = gacc[c];
        }
    }
}

// ---- backward: scatter to the table gradient ---------------------------------------------------
__device__ __forceinline__ void red_add(float* addr, const float (&v)[1]) { atomicAdd(addr, v[0]); }
__device__ __forceinline__ void red_add(float* addr, const float (&v)[2]) {
    atomicAdd(reinterpret_cast<float2*>(addr), make_float2(v[0], v[1]));
}
__device__ __forceinline__ void red_add(__half* addr, const __half (&v)[2]) {
    atomicAdd(reinterpret_cast<__half2*>(addr), __halves2half2(v[0], v[1]));
}

// thread <-> (sample, group of G channels); G = min(2, C) as in the reference (gridencoder.cu:404)
template <typename T, uint32_t D, uint32_t C, uint32_t G>
__global__ void __launch_bounds__(256)
k_grid_bwd(const T* __restrict__ grad, const float* __restrict__ inputs, const int32_t* __restrict__ offsets,
           T* __restrict__ grad_table, uint32_t B, uint32_t L, float S, uint32_t H, uint32_t gridtype,
           bool align_corners, uint32_t interp) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t b = tid * G / C;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    const uint32_t ch = tid * G - b * C;
    const float* x = inputs + (size_t)b * D;
    if (outside_unit<D>(x)) return;

    const Level g = level_geom(offsets, level, S, H);
    T* gt = grad_table + (size_t)g.row0 * C;
    float frac[D], dfrac[D];
    uint32_t base[D];
    locate<D>(x, g, align_corners, interp, frac, dfrac, base);

    T gin[G];
#pragma unroll
    for (uint32_t c = 0; c < G; ++c) gin[c] = grad[((size_t)level * B + b) * C + ch + c];

#pragma unroll
    for (uint32_t corner = 0; corner < (1u << D); ++corner) {
        float w = 1;
        uint32_t p[D];
#pragma unroll
        for (uint32_t d = 0; d < D; ++d) {
            if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; p[d] = base[d]; }
            else { w *= frac[d]; p[d] = base[d] + 1; }
        }
        const uint32_t row = lattice_row<D>(p, g, gridtype, align_corners);
        T v[G];
#pragma unroll
        for (uint32_t c = 0; c < G; ++c) v[c] = Acc<T>::from_f(w * Acc<T>::to_f(gin[c]));
        if constexpr (std::is_same<T, __half>::value && G == 1) {
            // fp16 table with a single channel: the reference never reaches this (grid.py:45);
            // use the native half atomic so the entry point is still well defined.
            atomicAdd(gt + (size_t)row * C + ch, v[0]);
        } else {
            red_add(gt + (size_t)row * C + ch, v);
        }
    }
}

// grad_inputs[b, d] = sum_{l, c} grad[l, b, c] * dy_dx[b, l, d, c]   (gridencoder.cu:343-368)
template <typename T, uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256)
k_grid_input_bwd(const T* __restrict__ grad, const T* __restrict__ dy_dx, T* __restrict__ grad_inputs, uint32_t B, uint32_t L) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * D) return;
    const uint32_t b = t / D, d = t - b * D;
    const T* dd = dy_dx + (size_t)b * L * D * C;
    T acc = Acc<T>::zero();
    for (uint32_t l = 0; l < L; ++l) {
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) {
            const T gv = grad[((size_t)l * B + b) * C + c];
            const T dv = dd[(l * D + d) * C + c];
            if constexpr (std::is_same<T, float>::value) acc += gv * dv;
            else {
                const __half p = __float2half_rn(__half2float(gv) * __half2float(dv));
                acc = __float2half_rn(__half2float(acc) + __half2float(p));
            }
        }
    }
    grad_inputs[t] = acc;
}

// ---- total-variation gradient, fp32, added in place into `grad` (gridencoder.cu:506-609) --------
template <uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256)
k_grid_tv(const float* __restrict__ inputs, const float* __restrict__ table, float* __restrict__ grad,
          const int32_t* __restrict__ offsets, float weight, uint32_t B, uint32_t L, float S, uint32_t H,
          uint32_t gridtype, bool align_corners) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    const float* x = inputs + (size_t)b * D;
    if (outside_unit<D>(x)) return;

    const Level g = level_geom(offsets, level, S, H);
    const float* tab = table + (size_t)g.row0 * C;
    float* gt = grad + (size_t)g.row0 * C;

    uint32_t p[D];
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) {
        const float pos = x[d] * g.scale + (align_corners ? 0.0f : 0.5f);
        p[d] = floorf(pos);
    }
    const uint32_t row = lattice_row<D>(p, g, gridtype, align_corners);
    float centre[C];
    load_row<float, C>(tab + (size_t)row * C, centre);

    float sum[C], sq[C];
#pragma unroll
    for (uint32_t c = 0; c < C; ++c) { sum[c] = 0; sq[c] = 0; }
    const float w = weight / (2 * D);

#pragma unroll
    for (uint32_t d = 0; d < D; ++d) {
        const uint32_t cur = p[d];
        if (cur < g.res) {                                  // right neighbour
            p[d] = cur + 1;
            float nb[C];
            load_row<float, C>(tab + (size_t)lattice_row<D>(p, g, gridtype, align_corners) * C, nb);
#pragma unroll
            for (uint32_t c = 0; c < C; ++c) { const float dv = centre[c] - nb[c]; sum[c] += dv; sq[c] += dv * dv; }
        }
        if (cur > 0) {                                      // left neighbour
            p[d] = cur - 1;
            float nb[C];
            load_row<float, C>(tab + (size_t)lattice_row<D>(p, g, gridtype, align_corners) * C, nb);
#pragma unroll
            for (uint32_t c = 0; c < C; ++c) { const float dv = centre[c] - nb[c]; sum[c] += dv; sq[c] += dv * dv; }
        }
        p[d] = cur;
    }
#pragma unroll
    for (uint32_t c = 0; c < C; ++c)
        atomicAdd(gt + (size_t)row * C + c, w * sum[c] * rsqrtf(sq[c] + 1e-9f));
}

// ---- dispatch -------------------------------------------------------------------------------
template <typename T, uint32_t D, uint32_t C>
int launch_fwd(const float* inputs, const void* emb, const int32_t* offsets, void* out, uint32_t B, uint32_t L,
               uint32_t max_level, float S, uint32_t H, void* dy_dx, uint32_t gridtype, bool ac, uint32_t interp,
               cudaStream_t st) {
    const dim3 grid(div_up(B, 256u), max_level, 1);
    k_grid_fwd<T, D, C><<<grid, 256, 0, st>>>(inputs, static_cast<const T*>(emb), offsets, static_cast<T*>(out), B, L, S, H,
                                              static_cast<T*>(dy_dx), gridtype, ac, interp);
    return check_launch("grid_encode_forward");
}

template <typename T, uint32_t D, uint32_t C>
int launch_bwd(const void* grad, const float* inputs, const int32_t* offsets, void* gemb, uint32_t B, uint32_t L,
               uint32_t max_level, float S, uint32_t H, const void* dy_dx, void* ginputs, uint32_t gridtype, bool ac,
               uint32_t interp, cudaStream_t st) {
    constexpr uint32_t G = C < 2 ? C : 2;
    const dim3 grid(div_up(B * C / G, 256u), max_level, 1);
    k_grid_bwd<T, D, C, G><<<grid, 256, 0, st>>>(static_cast<const T*>(grad), inputs, offsets, static_cast<T*>(gemb), B, L, S, H,
                                                  gridtype, ac, interp);
    if (int e = check_launch("grid_encode_backward")) return e;
    if (dy_dx) {
        k_grid_input_bwd<T, D, C><<<div_up(B * D, 256u), 256, 0, st>>>(static_cast<const T*>(grad), static_cast<const T*>(dy_dx),
                                                                        static_cast<T*>(ginputs), B, L);
        return check_launch("grid_encode_backward(inputs)");
    }
    return 0;
}

template <uint32_t D, uint32_t C>
int launch_tv(const float* inputs, const float* emb, float* grad, const int32_t* offsets, float weight, uint32_t B, uint32_t L,
              float S, uint32_t H, uint32_t gridtype, bool ac, cudaStream_t st) {
    const dim3 grid(div_up(B, 256u), L, 1);
    k_grid_tv<D, C><<<grid, 256, 0, st>>>(inputs, emb, grad, offsets, weight, B, L, S, H, gridtype, ac);
    return check_launch("grad_total_variation");
}

#define N2M_DISPATCH_DC(D, C, CALL)                                                        \
    switch (D) {                                                                           \
        case 2: switch (C) { case 1: return CALL(2, 1); case 2: return CALL(2, 2);         \
                             case 4: return CALL(2, 4); case 8: return CALL(2, 8); } break; \
        case 3: switch (C) { case 1: return CALL(3, 1); case 2: return CALL(3, 2);         \
                             case 4: return CALL(3, 4); case 8: return CALL(3, 8); } break; \
        case 4: switch (C) { case 1: return CALL(4, 1); case 2: return CALL(4, 2);         \
                             case 4: return CALL(4, 4); case 8: return CALL(4, 8); } break; \
        case 5: switch (C) { case 1: return CALL(5, 1); case 2: return CALL(5, 2);         \
                             case 4: return CALL(5, 4); case 8: return CALL(5, 8); } break; \
    }

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_grid_encode_forward(const float* inputs, const void* embeddings, const int32_t* offsets, void* outputs,
                            uint32_t B, uint32_t D, uint32_t C, uint32_t L, uint32_t max_level, float S, uint32_t H,
                            void* dy_dx, uint32_t gridtype, int align_corners, uint32_t interp, int dtype,
                            n2m_stream_t stream) {
    if (B == 0 || max_level == 0) return 0;
    N2M_REQUIRE(inputs && embeddings && offsets && outputs, "grid_encode_forward", "null pointer");
    N2M_REQUIRE(max_level <= L, "grid_encode_forward", "max_level > L");
    N2M_REQUIRE(dtype == 0 || dtype == 1, "grid_encode_forward", "dtype must be 0 (float32) or 1 (float16)");
    cudaStream_t st = as_stream(stream);
    const bool ac = align_corners != 0;
    if (dtype == 0) {
#define CALL(DD, CC) launch_fwd<float, DD, CC>(inputs, embeddings, offsets, outputs, B, L, max_level, S, H, dy_dx, gridtype, ac, interp, st)
        N2M_DISPATCH_DC(D, C, CALL)
#undef CALL
    } else {
#define CALL(DD, CC) launch_fwd<__half, DD, CC>(inputs, embeddings, offsets, outputs, B, L, max_level, S, H, dy_dx, gridtype, ac, interp, st)
        N2M_DISPATCH_DC(D, C, CALL)
#undef CALL
    }
    return fail("grid_encode_forward", "GridEncoding: D must be 2..5 and C must be 1, 2, 4, or 8.");
}

int n2m_grid_encode_backward(const void* grad, const float* inputs, const void* embeddings, const int32_t* offsets,
                             void* grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, uint32_t max_level,
                             float S, uint32_t H, const void* dy_dx, void* grad_inputs, uint32_t gridtype,
                             int align_corners, uint32_t interp, int dtype, n2m_stream_t stream) {
    (void)embeddings;
    if (B == 0 || max_level == 0) return 0;
    N2M_REQUIRE(grad && inputs && offsets && grad_embeddings, "grid_encode_backward", "null pointer");
    N2M_REQUIRE(max_level <= L, "grid_encode_backward", "max_level > L");
    N2M_REQUIRE(!dy_dx || grad_inputs, "grid_encode_backward", "dy_dx given but grad_inputs null");
    N2M_REQUIRE(dtype == 0 || dtype == 1, "grid_encode_backward", "dtype must be 0 (float32) or 1 (float16)");
    cudaStream_t st = as_stream(stream);
    const bool ac = align_corners != 0;
    if (dtype == 0) {
#define CALL(DD, CC) launch_bwd<float, DD, CC>(grad, inputs, offsets, grad_embeddings, B, L, max_level, S, H, dy_dx, grad_inputs, gridtype, ac, interp, st)
        N2M_DISPATCH_DC(D, C, CALL)
#undef CALL
    } else {
#define CALL(DD, CC) launch_bwd<__half, DD, CC>(grad, inputs, offsets, grad_embeddings, B, L, max_level, S, H, dy_dx, grad_inputs, gridtype, ac, interp, st)
        N2M_DISPATCH_DC(D, C, CALL)
#undef CALL
    }
    return fail("grid_encode_backward", "GridEncoding: D must be 2..5 and C must be 1, 2, 4, or 8.");
}

int n2m_grad_total_variation(const float* inputs, const float* embeddings, float* grad, const int32_t* offsets,
                             float weight, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
                             uint32_t gridtype, int align_corners, n2m_stream_t stream) {
    if (B == 0 || L == 0) return 0;
    N2M_REQUIRE(inputs && embeddings && grad && offsets, "grad_total_variation", "null pointer");
    cudaStream_t st = as_stream(stream);
    const bool ac = align_corners != 0;
#define CALL(DD, CC) launch_tv<DD, CC>(inputs, embeddings, grad, offsets, weight, B, L, S, H, gridtype, ac, st)
    N2M_DISPATCH_DC(D, C, CALL)
#undef CALL
    return fail("grad_total_variation", "GridEncoding: D must be 2..5 and C must be 1, 2, 4, or 8.");
}

}  // extern "C"
