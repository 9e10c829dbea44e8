// meshclean.cu -- the stage-0 mesh clean-up on the device: remove_masked_trigs and clean_mesh(..., remesh=False) of meshutils.py:63-93,
// 146-188 (pymeshlab in the reference) restated as exact combinatorics.  C ABI include/n2m_b200_mesh.h, host side nerf2mesh_b200/mesh.py
// (remove_masked_faces, clean_mesh), CPU restatement tests/meshclean_oracle.py.
//
// The kernels never move the mesh: faces are dropped through a keep flag, merged / split vertices are re-indexed in place in the face
// array, and the caller compacts once at the end with k_rsv_emit (cascade.cu).  Every decision is a function of sets (minimum index,
// count), so the atomics' order does not reach the output.
//
//   k_mark_verts / k_dilate_faces   selection dilation: select the vertices of kept faces, keep every face with a selected vertex
//   k_bbox                          bounding box of the flagged vertices as order-preserving u32 keys (atomicMin / atomicMax)
//   k_merge_bin / k_merge_fill      spatial hash of the referenced vertices: cells of size r, buckets of a power-of-two table (a bucket
//                                   shared by several cells only adds candidates, every candidate is tested exactly)
//   k_merge_round                   one decision round of the greedy merge (lexicographically-first maximal independent set of the
//                                   r-disk graph): i decides once every undecided lower neighbour is above its lowest leader neighbour
//   k_merge_apply                   faces take their vertices' leaders; faces that repeat an index go
//   k_table_insert<EDGE>            open-addressing table of unordered vertex triples (faces) or pairs (face edges), slot value = the
//                                   lowest element with that key
//   k_dup_null                      duplicate faces (not the lowest of their triple) and float64 null faces go
//   k_union_faces / k_comp_*        edge-connected components (lock-free union-find, root = lowest face) and their size / bbox filter
//   k_nme_*                         non-manifold edges: the faces on an edge of > 2 live faces, visited by (float64 area, index) in one CTA
//   k_fan_*                         non-manifold vertices: union-find over face corners joined through an edge at their vertex
#include "n2m_common.cuh"
#include "mesh_keys.cuh"
#include "union_find.cuh"
#include "../../include/n2m_b200_mesh.h"

#include <limits.h>

namespace n2m {
namespace {

constexpr int kSortThreads = 1024;

// ---- the two percentage readings --------------------------------------------------------------------------------------------------

// sqrt((dx*dx + dy*dy) + dz*dz) of a key box, each operation rounded on its own; an empty box (min > max) has diagonal 0
__device__ double box_diag(const uint32_t* lo, const uint32_t* hi) {
    if (lo[0] > hi[0]) return 0.0;
    double s = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double d = __dsub_rn((double)fkey_inv(hi[a]), (double)fkey_inv(lo[a]));
        s = a == 0 ? __dmul_rn(d, d) : __dadd_rn(s, __dmul_rn(d, d));
    }
    return __dsqrt_rn(s);
}
// PercentageValue(v_pct) of meshing_merge_close_vertices read against its parameter range [0, diag / 10]
__device__ __forceinline__ double merge_radius(double diag, double v_pct) { return __ddiv_rn(__dmul_rn(__ddiv_rn(v_pct, 100.0), diag), 10.0); }
// PercentageValue(min_d) of meshing_remove_connected_component_by_diameter read against the whole diagonal
__device__ __forceinline__ double min_component_diag(double diag, double min_d) { return __dmul_rn(__ddiv_rn(min_d, 100.0), diag); }

__device__ __forceinline__ bool live(const uint8_t* fkeep, uint32_t f) { return fkeep == nullptr || fkeep[f] != 0; }

// ---- selection, dilation, bounding box ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_mark_verts(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, uint8_t* __restrict__ vflag) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !live(fkeep, f)) return;
#pragma unroll
    for (int a = 0; a < 3; ++a) vflag[tri[3 * (size_t)f + a]] = 1;
}

__global__ void __launch_bounds__(256)
k_dilate_faces(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ vsel, uint8_t* __restrict__ fkeep) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || fkeep[f]) return;
    if (vsel[tri[3 * (size_t)f]] | vsel[tri[3 * (size_t)f + 1]] | vsel[tri[3 * (size_t)f + 2]]) fkeep[f] = 1;
}

__global__ void __launch_bounds__(256)
k_bbox(const float* __restrict__ verts, uint32_t V, const uint8_t* __restrict__ vflag, uint32_t* __restrict__ bbox) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V || !vflag[i]) return;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const uint32_t k = fkey(verts[3 * (size_t)i + a]);
        atomicMin(bbox + a, k);
        atomicMax(bbox + 3 + a, k);
    }
}

// ---- close-vertex merge ------------------------------------------------------------------------------------------------------------
struct MergeGrid {
    double lo[3], cell, r2;
};
// cells are a hair larger than r, so two points within r always lie in the same or adjacent cells whatever the quotient's rounding;
// cell coordinates are clamped (a clamped pair within r still lands in adjacent cells)
__device__ MergeGrid merge_grid(const uint32_t* bbox, double v_pct) {
    MergeGrid g;
    const double r = merge_radius(box_diag(bbox, bbox + 3), v_pct);
    g.r2 = __dmul_rn(r, r);
    g.cell = r * 1.000001;
#pragma unroll
    for (int a = 0; a < 3; ++a) g.lo[a] = (double)fkey_inv(bbox[a]);
    return g;
}
__device__ __forceinline__ void cell_of(const MergeGrid& g, const float* p, long long c[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double q = g.cell > 0.0 ? floor(((double)p[a] - g.lo[a]) / g.cell) : 0.0;
        c[a] = (long long)fmin(fmax(q, 0.0), 1099511627776.0);
    }
}
__device__ __forceinline__ uint32_t cell_bucket(long long x, long long y, long long z, uint32_t nb) {
    uint64_t h = (uint64_t)x * 0x9E3779B97F4A7C15ull ^ (uint64_t)y * 0xC2B2AE3D27D4EB4Full ^ (uint64_t)z * 0x165667B19E3779F9ull;
    h ^= h >> 31; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 29;
    return (uint32_t)h & (nb - 1);
}
__device__ __forceinline__ double dist2(const float* p, const float* q) {
    const double dx = __dsub_rn((double)p[0], (double)q[0]), dy = __dsub_rn((double)p[1], (double)q[1]), dz = __dsub_rn((double)p[2], (double)q[2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__global__ void __launch_bounds__(256)
k_merge_bin(const float* __restrict__ verts, uint32_t V, const uint8_t* __restrict__ vflag, const uint32_t* __restrict__ bbox, double v_pct,
            uint32_t nb, int32_t* __restrict__ bucket_count, int32_t* __restrict__ vbucket) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V || !vflag[i]) return;
    const MergeGrid g = merge_grid(bbox, v_pct);
    long long c[3];
    cell_of(g, verts + 3 * (size_t)i, c);
    const uint32_t b = cell_bucket(c[0], c[1], c[2], nb);
    vbucket[i] = (int32_t)b;
    atomicAdd(bucket_count + b, 1);
}

__global__ void __launch_bounds__(256)
k_merge_fill(uint32_t V, const uint8_t* __restrict__ vflag, const int32_t* __restrict__ vbucket, int32_t* __restrict__ cursor,
             int32_t* __restrict__ items) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V || !vflag[i]) return;
    items[atomicAdd(cursor + vbucket[i], 1)] = (int32_t)i;
}

// decided[j] = the round j was decided in (0: not yet); a neighbour decided in this very round counts as undecided, so the round count
// and every decision are deterministic.  target[j] is read only for neighbours decided in an earlier round (an earlier launch).
__global__ void __launch_bounds__(256)
k_merge_round(const float* __restrict__ verts, uint32_t V, const uint8_t* __restrict__ vflag, const uint32_t* __restrict__ bbox, double v_pct,
              uint32_t nb, const int32_t* __restrict__ start, const int32_t* __restrict__ items, int32_t round, int32_t* decided,
              int32_t* target, int32_t* __restrict__ pending) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V || !vflag[i] || decided[i] != 0) return;
    const MergeGrid g = merge_grid(bbox, v_pct);
    const float* p = verts + 3 * (size_t)i;
    long long c[3];
    cell_of(g, p, c);
    int32_t lead = INT_MAX, pend = INT_MAX;
#pragma unroll 1
    for (int n = 0; n < 27; ++n) {
        const uint32_t b = cell_bucket(c[0] + n / 9 - 1, c[1] + (n / 3) % 3 - 1, c[2] + n % 3 - 1, nb);
        const int32_t t1 = start[b + 1];
        for (int32_t t = start[b]; t < t1; ++t) {
            const int32_t j = items[t];
            if ((uint32_t)j >= i || j >= lead || j >= pend) continue;
            if (dist2(p, verts + 3 * (size_t)j) > g.r2) continue;
            const int32_t d = ((volatile int32_t*)decided)[j];
            if (d == 0 || d >= round) pend = j;
            else if (target[j] == j) lead = j;
        }
    }
    if (lead < pend) { target[i] = lead; decided[i] = round; }
    else if (pend == INT_MAX) { target[i] = (int32_t)i; decided[i] = round; }
    else *pending = 1;
}

__global__ void __launch_bounds__(256)
k_merge_apply(int32_t* __restrict__ tri, uint32_t F, const int32_t* __restrict__ target, uint8_t* __restrict__ fkeep) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !fkeep[f]) return;
    int32_t v[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) { v[a] = target[tri[3 * (size_t)f + a]]; tri[3 * (size_t)f + a] = v[a]; }
    if (v[0] == v[1] || v[1] == v[2] || v[0] == v[2]) fkeep[f] = 0;
}

// ---- hash table of unordered vertex tuples ----------------------------------------------------------------------------------------
// element e: face e (EDGE = false, key = its sorted triple) or edge e % 3 of face e / 3 (EDGE = true, key = (lo, hi) of corners k, k+1)
struct Key { int32_t a, b, c; };
template <bool EDGE>
__device__ __forceinline__ Key key_of(const int32_t* tri, int32_t e) {
    if (EDGE) {
        const int32_t f = e / 3, k = e % 3;
        const int32_t x = tri[3 * (size_t)f + k], y = tri[3 * (size_t)f + (k + 1) % 3];
        return Key{min(x, y), max(x, y), -1};
    }
    int32_t x = tri[3 * (size_t)e], y = tri[3 * (size_t)e + 1], z = tri[3 * (size_t)e + 2], t;
    if (x > y) { t = x; x = y; y = t; }
    if (y > z) { t = y; y = z; z = t; }
    if (x > y) { t = x; x = y; y = t; }
    return Key{x, y, z};
}
__device__ __forceinline__ uint32_t key_hash(Key k, uint32_t mask) {
    uint64_t h = (uint64_t)(uint32_t)k.a * 0x9E3779B97F4A7C15ull ^ (uint64_t)(uint32_t)k.b * 0xC2B2AE3D27D4EB4Full ^
                 (uint64_t)(uint32_t)k.c * 0x165667B19E3779F9ull;
    h ^= h >> 31; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 29;
    return (uint32_t)h & mask;
}

template <bool EDGE>
__global__ void __launch_bounds__(256)
k_table_insert(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, uint32_t nslots, int32_t* table,
               int32_t* __restrict__ slot_of) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (EDGE ? 3 * F : F) || !fkeep[EDGE ? e / 3 : e]) return;
    const Key k = key_of<EDGE>(tri, (int32_t)e);
    uint32_t s = key_hash(k, nslots - 1);
    for (uint32_t probe = 0; probe < nslots; ++probe, s = (s + 1) & (nslots - 1)) {
        int32_t cur = ((volatile int32_t*)table)[s];
        if (cur == -1) {
            cur = atomicCAS(table + s, -1, (int32_t)e);
            if (cur == -1) { slot_of[e] = (int32_t)s; return; }
        }
        const Key o = key_of<EDGE>(tri, cur);
        if (o.a == k.a && o.b == k.b && o.c == k.c) {
            atomicMin(table + s, (int32_t)e);
            slot_of[e] = (int32_t)s;
            return;
        }
    }
}

__device__ __forceinline__ void face_cross(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t f, double n[3]) {
    double p[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int a = 0; a < 3; ++a) p[c][a] = (double)verts[3 * (size_t)tri[3 * (size_t)f + c] + a];
    double e1[3], e2[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) { e1[a] = __dsub_rn(p[1][a], p[0][a]); e2[a] = __dsub_rn(p[2][a], p[0][a]); }
    n[0] = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
    n[1] = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
    n[2] = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
}

__global__ void __launch_bounds__(256)
k_dup_null(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t F, const int32_t* __restrict__ table,
           const int32_t* __restrict__ slot_of, uint8_t* __restrict__ fkeep) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !fkeep[f]) return;
    double n[3];
    face_cross(verts, tri, f, n);
    if (table[slot_of[f]] != (int32_t)f || (n[0] == 0.0 && n[1] == 0.0 && n[2] == 0.0)) fkeep[f] = 0;
}

// ---- connected components -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_iota(int32_t* __restrict__ x, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = (int32_t)i;
}

__global__ void __launch_bounds__(256)
k_union_faces(uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ table, const int32_t* __restrict__ slot_of,
              int32_t* parent) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F || !fkeep[e / 3]) return;
    const int32_t g = table[slot_of[e]] / 3;
    if (g != (int32_t)(e / 3)) uf_union(parent, (int32_t)(e / 3), g);
}

__global__ void __launch_bounds__(256)
k_comp_stats(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep,
             const int32_t* __restrict__ parent, int32_t* __restrict__ label, int32_t* __restrict__ count, uint32_t* __restrict__ cmin,
             uint32_t* __restrict__ cmax) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !fkeep[f]) return;
    const int32_t r = uf_root(parent, (int32_t)f);
    label[f] = r;
    atomicAdd(count + r, 1);
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const uint32_t k = fkey(verts[3 * (size_t)tri[3 * (size_t)f + c] + a]);
            atomicMin(cmin + 3 * (size_t)r + a, k);
            atomicMax(cmax + 3 * (size_t)r + a, k);
        }
}

__global__ void __launch_bounds__(256)
k_comp_filter(uint32_t F, const int32_t* __restrict__ label, const int32_t* __restrict__ count, const uint32_t* __restrict__ cmin,
              const uint32_t* __restrict__ cmax, const uint32_t* __restrict__ bbox, double min_d, uint32_t min_f, uint8_t* __restrict__ fkeep) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !fkeep[f]) return;
    const int32_t r = label[f];
    bool drop = min_f > 0 && (uint32_t)count[r] < min_f;
    if (min_d > 0.0) drop = drop || box_diag(cmin + 3 * (size_t)r, cmax + 3 * (size_t)r) < min_component_diag(box_diag(bbox, bbox + 3), min_d);
    if (drop) fkeep[f] = 0;
}

// ---- one-CTA sort of (key, value) pairs, lexicographic; n read on the device, buffers hold the next power of two ------------------
__device__ void block_sort(uint64_t* keys, int32_t* vals, uint32_t n) {
    uint32_t p = 1;
    while (p < n) p <<= 1;
    for (uint32_t i = n + threadIdx.x; i < p; i += blockDim.x) { keys[i] = ~0ull; vals[i] = INT_MAX; }
    __syncthreads();
    for (uint32_t k = 2; k <= p; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < p; i += blockDim.x) {
                const uint32_t l = i ^ j;
                if (l <= i) continue;
                const uint64_t ki = keys[i], kl = keys[l];
                const int32_t vi = vals[i], vl = vals[l];
                const bool greater = ki > kl || (ki == kl && vi > vl);
                if (((i & k) == 0) == greater) { keys[i] = kl; keys[l] = ki; vals[i] = vl; vals[l] = vi; }
            }
            __syncthreads();
        }
}

// ---- non-manifold edges -------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_edge_count(uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ slot_of, int32_t* __restrict__ ecount) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < 3 * F && fkeep[e / 3]) atomicAdd(ecount + slot_of[e], 1);
}

__global__ void __launch_bounds__(256)
k_nme_collect(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep,
              const int32_t* __restrict__ slot_of, const int32_t* __restrict__ ecount, int32_t* __restrict__ ncand, uint64_t* __restrict__ keys,
              int32_t* __restrict__ vals) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F || !fkeep[f]) return;
    if (ecount[slot_of[3 * f]] <= 2 && ecount[slot_of[3 * f + 1]] <= 2 && ecount[slot_of[3 * f + 2]] <= 2) return;
    double n[3];
    face_cross(verts, tri, f, n);
    const double area = __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(n[0], n[0]), __dmul_rn(n[1], n[1])), __dmul_rn(n[2], n[2]))));
    const int32_t t = atomicAdd(ncand, 1);
    keys[t] = (uint64_t)__double_as_longlong(area);             // area >= +0: the bit pattern orders as the value
    vals[t] = (int32_t)f;
}

// the visit is sequential by definition (each deletion changes the counts the next face sees): one thread, after the CTA's sort
__global__ void __launch_bounds__(kSortThreads)
k_nme_repair(const int32_t* __restrict__ ncand, uint64_t* keys, int32_t* vals, const int32_t* __restrict__ slot_of, int32_t* ecount,
             uint8_t* fkeep) {
    const uint32_t n = (uint32_t)*ncand;
    block_sort(keys, vals, n);
    if (threadIdx.x != 0) return;
    for (uint32_t t = 0; t < n; ++t) {
        const int32_t f = vals[t];
        const int32_t s0 = slot_of[3 * f], s1 = slot_of[3 * f + 1], s2 = slot_of[3 * f + 2];
        if (ecount[s0] > 2 || ecount[s1] > 2 || ecount[s2] > 2) {
            fkeep[f] = 0;
            --ecount[s0]; --ecount[s1]; --ecount[s2];
        }
    }
}

// ---- non-manifold vertices ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_edge_min(uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ slot_of, int32_t* __restrict__ emin) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < 3 * F && fkeep[e / 3]) atomicMin(emin + slot_of[e], (int32_t)e);
}

__device__ __forceinline__ int32_t corner_at(const int32_t* __restrict__ tri, int32_t g, int32_t v) {
    return 3 * g + (tri[3 * (size_t)g] == v ? 0 : tri[3 * (size_t)g + 1] == v ? 1 : 2);
}

// corner c = 3 f + k stands for face f at vertex tri[c]; the two faces on an edge join their corners at each end of it
__global__ void __launch_bounds__(256)
k_fan_union(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ slot_of,
            const int32_t* __restrict__ emin, int32_t* cparent) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F || !fkeep[e / 3]) return;
    const int32_t f = (int32_t)(e / 3), k = (int32_t)(e % 3);
    const int32_t g = emin[slot_of[e]] / 3;
    if (g == f) return;
    const int32_t a = tri[3 * (size_t)f + k], kb = (k + 1) % 3, b = tri[3 * (size_t)f + kb];
    uf_union(cparent, 3 * f + k, corner_at(tri, g, a));
    uf_union(cparent, 3 * f + kb, corner_at(tri, g, b));
}

__global__ void __launch_bounds__(256)
k_fan_roots(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ cparent,
            int32_t* __restrict__ clabel, int32_t* __restrict__ vmin) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= 3 * F || !fkeep[c / 3]) return;
    const int32_t r = uf_root(cparent, (int32_t)c);
    clabel[c] = r;
    atomicMin(vmin + tri[c], r);
}

// the roots of the fans that do not hold their vertex's lowest face, keyed (vertex, root corner): the root is the fan's lowest corner,
// so its order within a vertex is the order of the fans' lowest faces
__global__ void __launch_bounds__(256)
k_fan_collect(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ clabel,
              const int32_t* __restrict__ vmin, int32_t* __restrict__ nextra, uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= 3 * F || !fkeep[c / 3] || clabel[c] != (int32_t)c || vmin[tri[c]] == (int32_t)c) return;
    const int32_t t = atomicAdd(nextra, 1);
    keys[t] = ((uint64_t)(uint32_t)tri[c] << 32) | c;
    vals[t] = (int32_t)c;
}

__global__ void __launch_bounds__(kSortThreads)
k_fan_number(const int32_t* __restrict__ nextra, uint64_t* keys, int32_t* vals, int32_t* __restrict__ cnew) {
    const uint32_t n = (uint32_t)*nextra;
    block_sort(keys, vals, n);
    for (uint32_t t = threadIdx.x; t < n; t += blockDim.x) cnew[vals[t]] = (int32_t)t;
}

__global__ void __launch_bounds__(256)
k_fan_apply(const float* __restrict__ verts, uint32_t V, int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep,
            const int32_t* __restrict__ clabel, const int32_t* __restrict__ vmin, const int32_t* __restrict__ cnew, float* __restrict__ ext) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= 3 * F || !fkeep[c / 3]) return;
    const int32_t v = tri[c], r = clabel[c];
    if (r == vmin[v]) return;
    const size_t nv = (size_t)V + (size_t)cnew[r];
    tri[c] = (int32_t)nv;
    if (r == (int32_t)c)
#pragma unroll
        for (int a = 0; a < 3; ++a) ext[3 * nv + a] = verts[3 * (size_t)v + a];
}

inline uint32_t grid_of(size_t n) { return (uint32_t)div_up(n, (size_t)256); }
inline bool pow2(uint32_t n) { return n && !(n & (n - 1)); }

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_clean_mark_verts(const int32_t* tri, uint32_t F, const uint8_t* fkeep, uint8_t* vflag, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && vflag, "clean_mark_verts", "null pointer");
    k_mark_verts<<<grid_of(F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, vflag);
    return check_launch("clean_mark_verts");
}

int n2m_clean_dilate(const int32_t* tri, uint32_t F, uint8_t* fkeep, uint8_t* vsel, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && fkeep && vsel, "clean_dilate", "null pointer");
    k_mark_verts<<<grid_of(F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, vsel);
    k_dilate_faces<<<grid_of(F), 256, 0, as_stream(stream)>>>(tri, F, vsel, fkeep);
    return check_launch("clean_dilate");
}

int n2m_clean_bbox(const float* vertices, uint32_t V, const uint8_t* vflag, uint32_t* bbox, n2m_stream_t stream) {
    N2M_REQUIRE(bbox, "clean_bbox", "null pointer");
    cudaMemsetAsync(bbox, 0xFF, 3 * sizeof(uint32_t), as_stream(stream));
    cudaMemsetAsync(bbox + 3, 0, 3 * sizeof(uint32_t), as_stream(stream));
    if (V == 0) return check_launch("clean_bbox");
    N2M_REQUIRE(vertices && vflag, "clean_bbox", "null pointer");
    k_bbox<<<grid_of(V), 256, 0, as_stream(stream)>>>(vertices, V, vflag, bbox);
    return check_launch("clean_bbox");
}

int n2m_clean_merge_bin(const float* vertices, uint32_t V, const uint8_t* vflag, const uint32_t* bbox, double v_pct, uint32_t nbuckets,
                        int32_t* bucket_count, int32_t* vbucket, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(nbuckets) && v_pct > 0.0, "clean_merge_bin", "power-of-two bucket count, v_pct > 0");
    if (V == 0) return 0;
    N2M_REQUIRE(vertices && vflag && bbox && bucket_count && vbucket, "clean_merge_bin", "null pointer");
    k_merge_bin<<<grid_of(V), 256, 0, as_stream(stream)>>>(vertices, V, vflag, bbox, v_pct, nbuckets, bucket_count, vbucket);
    return check_launch("clean_merge_bin");
}

int n2m_clean_merge_fill(uint32_t V, const uint8_t* vflag, const int32_t* vbucket, int32_t* cursor, int32_t* items, n2m_stream_t stream) {
    if (V == 0) return 0;
    N2M_REQUIRE(vflag && vbucket && cursor && items, "clean_merge_fill", "null pointer");
    k_merge_fill<<<grid_of(V), 256, 0, as_stream(stream)>>>(V, vflag, vbucket, cursor, items);
    return check_launch("clean_merge_fill");
}

int n2m_clean_merge_round(const float* vertices, uint32_t V, const uint8_t* vflag, const uint32_t* bbox, double v_pct, uint32_t nbuckets,
                          const int32_t* bucket_start, const int32_t* items, int32_t round, int32_t* decided, int32_t* target,
                          int32_t* pending, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(nbuckets) && v_pct > 0.0 && round >= 1, "clean_merge_round", "power-of-two bucket count, v_pct > 0, round >= 1");
    if (V == 0) return 0;
    N2M_REQUIRE(vertices && vflag && bbox && bucket_start && items && decided && target && pending, "clean_merge_round", "null pointer");
    k_merge_round<<<grid_of(V), 256, 0, as_stream(stream)>>>(vertices, V, vflag, bbox, v_pct, nbuckets, bucket_start, items, round, decided,
                                                             target, pending);
    return check_launch("clean_merge_round");
}

int n2m_clean_merge_apply(int32_t* tri, uint32_t F, const int32_t* target, uint8_t* fkeep, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && target && fkeep, "clean_merge_apply", "null pointer");
    k_merge_apply<<<grid_of(F), 256, 0, as_stream(stream)>>>(tri, F, target, fkeep);
    return check_launch("clean_merge_apply");
}

int n2m_clean_dup_null(const float* vertices, const int32_t* tri, uint32_t F, uint8_t* fkeep, uint32_t nslots, int32_t* table,
                       int32_t* slot_of, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(nslots) && nslots >= 2 * (uint64_t)F, "clean_dup_null", "power-of-two table of at least 2 F slots");
    if (F == 0) return 0;
    N2M_REQUIRE(vertices && tri && fkeep && table && slot_of, "clean_dup_null", "null pointer");
    cudaMemsetAsync(table, 0xFF, nslots * sizeof(int32_t), as_stream(stream));
    k_table_insert<false><<<grid_of(F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, nslots, table, slot_of);
    k_dup_null<<<grid_of(F), 256, 0, as_stream(stream)>>>(vertices, tri, F, table, slot_of, fkeep);
    return check_launch("clean_dup_null");
}

int n2m_clean_edge_table(const int32_t* tri, uint32_t F, const uint8_t* fkeep, uint32_t nslots, int32_t* table, int32_t* slot_of,
                         n2m_stream_t stream) {
    N2M_REQUIRE(pow2(nslots) && nslots >= 6 * (uint64_t)F, "clean_edge_table", "power-of-two table of at least 6 F slots");
    if (F == 0) return 0;
    N2M_REQUIRE(tri && fkeep && table && slot_of, "clean_edge_table", "null pointer");
    cudaMemsetAsync(table, 0xFF, nslots * sizeof(int32_t), as_stream(stream));
    k_table_insert<true><<<grid_of(3 * (size_t)F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, nslots, table, slot_of);
    return check_launch("clean_edge_table");
}

int n2m_clean_components(const float* vertices, const int32_t* tri, uint32_t F, uint8_t* fkeep, const int32_t* table, const int32_t* slot_of,
                         const uint32_t* bbox, double min_d, uint32_t min_f, int32_t* parent, int32_t* label, int32_t* count, uint32_t* cmin,
                         uint32_t* cmax, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(vertices && tri && fkeep && table && slot_of && bbox && parent && label && count && cmin && cmax, "clean_components",
                "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(count, 0, F * sizeof(int32_t), s);
    cudaMemsetAsync(cmin, 0xFF, 3 * (size_t)F * sizeof(uint32_t), s);
    cudaMemsetAsync(cmax, 0, 3 * (size_t)F * sizeof(uint32_t), s);
    k_iota<<<grid_of(F), 256, 0, s>>>(parent, F);
    k_union_faces<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, fkeep, table, slot_of, parent);
    k_comp_stats<<<grid_of(F), 256, 0, s>>>(vertices, tri, F, fkeep, parent, label, count, cmin, cmax);
    k_comp_filter<<<grid_of(F), 256, 0, s>>>(F, label, count, cmin, cmax, bbox, min_d, min_f, fkeep);
    return check_launch("clean_components");
}

int n2m_clean_nm_edges(const float* vertices, const int32_t* tri, uint32_t F, uint8_t* fkeep, const int32_t* slot_of, uint32_t nslots,
                       int32_t* ecount, int32_t* ncand, uint64_t* keys, int32_t* vals, uint32_t capacity, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(capacity) && capacity >= F, "clean_nm_edges", "power-of-two sort buffers of at least F entries");
    if (F == 0) return 0;
    N2M_REQUIRE(vertices && tri && fkeep && slot_of && ecount && ncand && keys && vals, "clean_nm_edges", "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(ecount, 0, nslots * sizeof(int32_t), s);
    cudaMemsetAsync(ncand, 0, sizeof(int32_t), s);
    k_edge_count<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, fkeep, slot_of, ecount);
    k_nme_collect<<<grid_of(F), 256, 0, s>>>(vertices, tri, F, fkeep, slot_of, ecount, ncand, keys, vals);
    k_nme_repair<<<1, kSortThreads, 0, s>>>(ncand, keys, vals, slot_of, ecount, fkeep);
    return check_launch("clean_nm_edges");
}

int n2m_clean_nm_verts_find(const int32_t* tri, uint32_t V, uint32_t F, const uint8_t* fkeep, const int32_t* slot_of, uint32_t nslots,
                            int32_t* emin, int32_t* cparent, int32_t* clabel, int32_t* vmin, int32_t* nextra, uint64_t* keys, int32_t* vals,
                            int32_t* cnew, uint32_t capacity, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(capacity) && capacity >= 3 * (uint64_t)F, "clean_nm_verts_find", "power-of-two sort buffers of at least 3 F entries");
    if (F == 0) return 0;
    N2M_REQUIRE(tri && fkeep && slot_of && emin && cparent && clabel && vmin && nextra && keys && vals && cnew, "clean_nm_verts_find",
                "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(emin, 0x7F, nslots * sizeof(int32_t), s);
    cudaMemsetAsync(vmin, 0x7F, V * sizeof(int32_t), s);
    cudaMemsetAsync(nextra, 0, sizeof(int32_t), s);
    k_edge_min<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, fkeep, slot_of, emin);
    k_iota<<<grid_of(3 * (size_t)F), 256, 0, s>>>(cparent, 3 * F);
    k_fan_union<<<grid_of(3 * (size_t)F), 256, 0, s>>>(tri, F, fkeep, slot_of, emin, cparent);
    k_fan_roots<<<grid_of(3 * (size_t)F), 256, 0, s>>>(tri, F, fkeep, cparent, clabel, vmin);
    k_fan_collect<<<grid_of(3 * (size_t)F), 256, 0, s>>>(tri, F, fkeep, clabel, vmin, nextra, keys, vals);
    k_fan_number<<<1, kSortThreads, 0, s>>>(nextra, keys, vals, cnew);
    return check_launch("clean_nm_verts_find");
}

int n2m_clean_nm_verts_apply(const float* vertices, uint32_t V, int32_t* tri, uint32_t F, const uint8_t* fkeep, const int32_t* clabel,
                             const int32_t* vmin, const int32_t* cnew, float* ext_vertices, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(vertices && tri && fkeep && clabel && vmin && cnew && ext_vertices, "clean_nm_verts_apply", "null pointer");
    k_fan_apply<<<grid_of(3 * (size_t)F), 256, 0, as_stream(stream)>>>(vertices, V, tri, F, fkeep, clabel, vmin, cnew, ext_vertices);
    return check_launch("clean_nm_verts_apply");
}

}  // extern "C"
