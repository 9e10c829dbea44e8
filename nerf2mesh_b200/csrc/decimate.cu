// decimate.cu -- quadric edge-collapse decimation of the stage-0 meshes on the device: the library's parallel reading of
// meshing_decimation_quadric_edge_collapse (pymeshlab / VCG, meshutils.py decimate_mesh) with its defaults.  C ABI
// include/n2m_b200_mesh.h, host side nerf2mesh_b200/mesh.py (decimate_mesh), CPU restatement tests/decimate_oracle.py.
//
// VCG collapses one edge at a time from a heap.  Here a round collapses a set of edges that share no vertex and no adjacency, so the
// collapses are independent and their order does not matter; the face array is re-indexed in place (n2m_clean_merge_apply) and
// compacted once at the end (n2m_rsv_emit).  Every float64 operation is an explicit __d*_rn intrinsic, so no FMA contraction separates
// the kernels from the numpy restatement, and no sum depends on the order of atomics: the atomics only count, fill order-free lists,
// and take minima.
//
//   k_dc_init                 faces that repeat an index go; flive = the live faces (warp-aggregated count)
//   k_dc_vcount / k_dc_vfill  vertex -> live face lists (count, caller's exclusive scan, fill in any order)
//   k_dc_quadrics             Q_v = sum of the faces' plane quadrics, the vertex's list sorted by face index first
//   k_dc_ecount / k_dc_bnd    live faces per edge-table slot; vertices on an edge of one face are boundary vertices
//   k_dc_eval                 per edge (its lowest live face-edge 3f+k): validity, placement, key = fkey(float(cost)) << 32 | 3f+k
//   k_dc_need / k_dc_hist / k_dc_digit   K* by an 8-bit radix select over the keys, each weighted by its edge's face count
//   k_dc_vmin / k_dc_r1 / k_dc_select    the least key at each vertex, over its closed neighbourhood, and the edges equal to both ends'
#include "n2m_common.cuh"
#include "mesh_keys.cuh"
#include "../../include/n2m_b200_mesh.h"

#include <algorithm>

namespace n2m {
namespace {

constexpr uint64_t kNone = ~0ull;            // the key of an edge that may not collapse (a valid key's high word is at most fkey(NaN))
constexpr double kDetRel = 1e-6;             // optimal placement solves A p = -b when det(A) > kDetRel * trace(A)^3

__device__ __forceinline__ bool live(const uint8_t* fkeep, uint32_t f) { return fkeep[f] != 0; }

__device__ __forceinline__ void load_p(const float* __restrict__ verts, int32_t v, double p[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = (double)verts[3 * (size_t)v + a];
}

// float64 cross(b - a, c - a), one rounding per operation (meshclean.cu's face_cross on points)
__device__ __forceinline__ void cross3(const double* a, const double* b, const double* c, double n[3]) {
    double e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { e1[k] = __dsub_rn(b[k], a[k]); e2[k] = __dsub_rn(c[k], a[k]); }
    n[0] = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
    n[1] = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
    n[2] = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
}
__device__ __forceinline__ double dot3(const double* x, const double* y) {
    return __dadd_rn(__dadd_rn(__dmul_rn(x[0], y[0]), __dmul_rn(x[1], y[1])), __dmul_rn(x[2], y[2]));
}

// the plane quadric (a00 a01 a02 a11 a12 a22 b0 b1 b2 c) of face f: unit normal u = cross / |cross|, d = -u.a; zero when |cross| = 0
__device__ void face_quadric(const float* __restrict__ verts, const int32_t* __restrict__ tri, int32_t f, double K[10]) {
    double p[3][3], n[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) load_p(verts, tri[3 * (size_t)f + c], p[c]);
    cross3(p[0], p[1], p[2], n);
    const double ln = __dsqrt_rn(dot3(n, n));
    if (!(ln > 0.0)) {
#pragma unroll
        for (int i = 0; i < 10; ++i) K[i] = 0.0;
        return;
    }
    const double u[3] = {__ddiv_rn(n[0], ln), __ddiv_rn(n[1], ln), __ddiv_rn(n[2], ln)};
    const double d = -dot3(u, p[0]);
    K[0] = __dmul_rn(u[0], u[0]); K[1] = __dmul_rn(u[0], u[1]); K[2] = __dmul_rn(u[0], u[2]);
    K[3] = __dmul_rn(u[1], u[1]); K[4] = __dmul_rn(u[1], u[2]); K[5] = __dmul_rn(u[2], u[2]);
    K[6] = __dmul_rn(d, u[0]); K[7] = __dmul_rn(d, u[1]); K[8] = __dmul_rn(d, u[2]); K[9] = __dmul_rn(d, d);
}

// x^T A x + 2 b.x + c evaluated as ((((x Ax + y Ay) + z Az) + 2 bx) + c), Ax = (a00 x + a01 y) + a02 z, ...
__device__ double quadric_cost(const double* Q, const float* p32) {
    const double x = (double)p32[0], y = (double)p32[1], z = (double)p32[2];
    const double Ax = __dadd_rn(__dadd_rn(__dmul_rn(Q[0], x), __dmul_rn(Q[1], y)), __dmul_rn(Q[2], z));
    const double Ay = __dadd_rn(__dadd_rn(__dmul_rn(Q[1], x), __dmul_rn(Q[3], y)), __dmul_rn(Q[4], z));
    const double Az = __dadd_rn(__dadd_rn(__dmul_rn(Q[2], x), __dmul_rn(Q[4], y)), __dmul_rn(Q[5], z));
    const double bx = __dadd_rn(__dadd_rn(__dmul_rn(Q[6], x), __dmul_rn(Q[7], y)), __dmul_rn(Q[8], z));
    const double q = __dadd_rn(__dadd_rn(__dmul_rn(x, Ax), __dmul_rn(y, Ay)), __dmul_rn(z, Az));
    return __dadd_rn(__dadd_rn(q, __dmul_rn(2.0, bx)), Q[9]);
}

// the merged vertex's float32 position and the float64 cost there; pa is the lower-index endpoint
__device__ double place(const double* Q, const float* pa, const float* pb, bool optimal, float out[3]) {
    float mid[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) mid[a] = __double2float_rn(__dmul_rn(__dadd_rn((double)pa[a], (double)pb[a]), 0.5));
    const double cm = quadric_cost(Q, mid);
    if (optimal) {
        const double C00 = __dsub_rn(__dmul_rn(Q[3], Q[5]), __dmul_rn(Q[4], Q[4]));
        const double C01 = __dsub_rn(__dmul_rn(Q[2], Q[4]), __dmul_rn(Q[1], Q[5]));
        const double C02 = __dsub_rn(__dmul_rn(Q[1], Q[4]), __dmul_rn(Q[3], Q[2]));
        const double det = __dadd_rn(__dadd_rn(__dmul_rn(Q[0], C00), __dmul_rn(Q[1], C01)), __dmul_rn(Q[2], C02));
        const double tr = __dadd_rn(__dadd_rn(Q[0], Q[3]), Q[5]);
        if (det > __dmul_rn(kDetRel, __dmul_rn(__dmul_rn(tr, tr), tr))) {
            const double C11 = __dsub_rn(__dmul_rn(Q[0], Q[5]), __dmul_rn(Q[2], Q[2]));
            const double C12 = __dsub_rn(__dmul_rn(Q[1], Q[2]), __dmul_rn(Q[0], Q[4]));
            const double C22 = __dsub_rn(__dmul_rn(Q[0], Q[3]), __dmul_rn(Q[1], Q[1]));
            out[0] = __double2float_rn(-__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(C00, Q[6]), __dmul_rn(C01, Q[7])), __dmul_rn(C02, Q[8])), det));
            out[1] = __double2float_rn(-__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(C01, Q[6]), __dmul_rn(C11, Q[7])), __dmul_rn(C12, Q[8])), det));
            out[2] = __double2float_rn(-__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(C02, Q[6]), __dmul_rn(C12, Q[7])), __dmul_rn(C22, Q[8])), det));
            return quadric_cost(Q, out);
        }
        double best = quadric_cost(Q, pa);
        int which = 0;
        const double cb = quadric_cost(Q, pb);
        if (cb < best) { best = cb; which = 1; }
        if (cm < best) { best = cm; which = 2; }
#pragma unroll
        for (int a = 0; a < 3; ++a) out[a] = which == 0 ? pa[a] : which == 1 ? pb[a] : mid[a];
        return best;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) out[a] = mid[a];
    return cm;
}

__device__ __forceinline__ bool has_vertex(const int32_t* __restrict__ tri, int32_t g, int32_t v) {
    return tri[3 * (size_t)g] == v || tri[3 * (size_t)g + 1] == v || tri[3 * (size_t)g + 2] == v;
}
__device__ __forceinline__ bool adjacent(const int32_t* __restrict__ tri, const int32_t* __restrict__ vstart, const int32_t* __restrict__ vfaces,
                                         int32_t x, int32_t w) {
    for (int32_t t = vstart[x]; t < vstart[x + 1]; ++t)
        if (has_vertex(tri, vfaces[t], w)) return true;
    return false;
}
// a live face around x whose vertices are {x, c, d}
__device__ __forceinline__ bool has_face(const int32_t* __restrict__ tri, const int32_t* __restrict__ vstart, const int32_t* __restrict__ vfaces,
                                         int32_t x, int32_t c, int32_t d) {
    for (int32_t t = vstart[x]; t < vstart[x + 1]; ++t) {
        const int32_t g = vfaces[t];
        if (has_vertex(tri, g, c) && has_vertex(tri, g, d)) return true;
    }
    return false;
}

// ---- set-up ---------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_dc_init(const int32_t* __restrict__ tri, uint32_t F, uint8_t* __restrict__ fkeep, int32_t* __restrict__ flive) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    bool ok = false;
    if (f < F) {
        const int32_t a = tri[3 * (size_t)f], b = tri[3 * (size_t)f + 1], c = tri[3 * (size_t)f + 2];
        ok = a != b && b != c && a != c;
        fkeep[f] = ok ? 1 : 0;
    }
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(flive, __popc(m));
}

__global__ void __launch_bounds__(256)
k_dc_vcount(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, int32_t* __restrict__ vcount) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < 3 * F && live(fkeep, c / 3)) atomicAdd(vcount + tri[c], 1);
}

__global__ void __launch_bounds__(256)
k_dc_vfill(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, int32_t* __restrict__ cursor, int32_t* __restrict__ vfaces) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < 3 * F && live(fkeep, c / 3)) vfaces[atomicAdd(cursor + tri[c], 1)] = (int32_t)(c / 3);
}

// the vertex's face list is sorted in place (insertion sort: the lists are the vertex valences), then summed in that order from +0
__global__ void __launch_bounds__(256)
k_dc_quadrics(const float* __restrict__ verts, uint32_t V, const int32_t* __restrict__ tri, const int32_t* __restrict__ vstart,
              int32_t* __restrict__ vfaces, double* __restrict__ Q) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const int32_t s = vstart[v], t1 = vstart[v + 1];
    for (int32_t i = s + 1; i < t1; ++i) {
        const int32_t x = vfaces[i];
        int32_t j = i - 1;
        while (j >= s && vfaces[j] > x) { vfaces[j + 1] = vfaces[j]; --j; }
        vfaces[j + 1] = x;
    }
    double q[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) q[i] = 0.0;
    for (int32_t t = s; t < t1; ++t) {
        double K[10];
        face_quadric(verts, tri, vfaces[t], K);
#pragma unroll
        for (int i = 0; i < 10; ++i) q[i] = __dadd_rn(q[i], K[i]);
    }
#pragma unroll
    for (int i = 0; i < 10; ++i) Q[10 * (size_t)v + i] = q[i];
}

// ---- per round: edges ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_dc_ecount(uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ slot_of, int32_t* __restrict__ ecount) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < 3 * F && live(fkeep, e / 3)) atomicAdd(ecount + slot_of[e], 1);
}

__global__ void __launch_bounds__(256)
k_dc_bnd(const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ slot_of,
         const int32_t* __restrict__ ecount, uint8_t* __restrict__ vbnd) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F || !live(fkeep, e / 3) || ecount[slot_of[e]] != 1) return;
    vbnd[tri[e]] = 1;
    vbnd[tri[3 * (e / 3) + (e % 3 + 1) % 3]] = 1;
}

// keys[e] for every face-edge e: the collapse key where e is its edge's lowest live face-edge and the collapse is valid, else kNone;
// pos[e] the merged position
__global__ void __launch_bounds__(256)
k_dc_eval(const float* __restrict__ verts, const double* __restrict__ Qv, const int32_t* __restrict__ tri, uint32_t F,
          const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ table, const int32_t* __restrict__ slot_of,
          const int32_t* __restrict__ ecount, const uint8_t* __restrict__ vbnd, const int32_t* __restrict__ vstart,
          const int32_t* __restrict__ vfaces, int optimal, uint64_t* __restrict__ keys, float* __restrict__ pos) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F) return;
    keys[e] = kNone;
    const uint32_t f = e / 3, k = e % 3;
    if (!live(fkeep, f) || table[slot_of[e]] != (int32_t)e) return;
    const int32_t cnt = ecount[slot_of[e]];
    if (cnt < 1 || cnt > 2) return;
    const int32_t x = tri[3 * (size_t)f + k], y = tri[3 * (size_t)f + (k + 1) % 3];
    const int32_t a = min(x, y), b = max(x, y), c = tri[3 * (size_t)f + (k + 2) % 3];
    int32_t d = -1;
    if (cnt == 2)
        for (int32_t t = vstart[a]; t < vstart[a + 1]; ++t) {
            const int32_t g = vfaces[t];
            if (g != (int32_t)f && has_vertex(tri, g, b)) {
                const int32_t* G = tri + 3 * (size_t)g;
                d = G[0] != a && G[0] != b ? G[0] : G[1] != a && G[1] != b ? G[1] : G[2];
            }
        }
    // boundary: an interior edge between two boundary vertices would pinch the mesh, and a boundary edge whose face has its other two
    // edges on the boundary as well would delete a lone triangle
    if (cnt == 2 && vbnd[a] && vbnd[b]) return;
    if (cnt == 1 && ecount[slot_of[3 * f + (k + 1) % 3]] == 1 && ecount[slot_of[3 * f + (k + 2) % 3]] == 1) return;
    // link condition: every common neighbour of a and b is an opposite vertex
    for (int32_t t = vstart[a]; t < vstart[a + 1]; ++t) {
        const int32_t* G = tri + 3 * (size_t)vfaces[t];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int32_t w = G[j];
            if (w == a || w == b || w == c || w == d) continue;
            if (adjacent(tri, vstart, vfaces, b, w)) return;
        }
    }
    // tetrahedron: (a, c, d) and (b, c, d) both live
    if (cnt == 2 && c != d && has_face(tri, vstart, vfaces, a, c, d) && has_face(tri, vstart, vfaces, b, c, d)) return;
    double Q[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) Q[i] = __dadd_rn(Qv[10 * (size_t)a + i], Qv[10 * (size_t)b + i]);
    float pa[3], pb[3], p[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { pa[i] = verts[3 * (size_t)a + i]; pb[i] = verts[3 * (size_t)b + i]; }
    const double cost = place(Q, pa, pb, optimal != 0, p);
    // no surviving face around a or b may flip or degenerate: dot(n_old, n_new) > 0
    const double pd[3] = {(double)p[0], (double)p[1], (double)p[2]};
#pragma unroll 1
    for (int end = 0; end < 2; ++end) {
        const int32_t m = end ? b : a;
        for (int32_t t = vstart[m]; t < vstart[m + 1]; ++t) {
            const int32_t g = vfaces[t];
            if (has_vertex(tri, g, end ? a : b)) continue;
            double q[3][3], n0[3], n1[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) load_p(verts, tri[3 * (size_t)g + j], q[j]);
            cross3(q[0], q[1], q[2], n0);
#pragma unroll
            for (int j = 0; j < 3; ++j)
                if (tri[3 * (size_t)g + j] == m) { q[j][0] = pd[0]; q[j][1] = pd[1]; q[j][2] = pd[2]; }
            cross3(q[0], q[1], q[2], n1);
            if (!(dot3(n0, n1) > 0.0)) return;
        }
    }
    keys[e] = ((uint64_t)fkey(__double2float_rn(cost)) << 32) | e;
#pragma unroll
    for (int i = 0; i < 3; ++i) pos[3 * (size_t)e + i] = p[i];
}

// ---- per round: K* -----------------------------------------------------------------------------------------------------------------
// state [4] u64: prefix, the faces still needed below it, "every valid edge" flag, K*
__global__ void k_dc_need(const int32_t* __restrict__ flive, uint32_t target, uint64_t* __restrict__ state, unsigned long long* __restrict__ hist) {
    if (threadIdx.x == 0) { state[0] = 0; state[1] = (uint64_t)(*flive - (int64_t)target); state[2] = 0; state[3] = 0; }
    hist[threadIdx.x] = 0;
}

__global__ void __launch_bounds__(256)
k_dc_hist(const uint64_t* __restrict__ keys, uint32_t n, const int32_t* __restrict__ slot_of, const int32_t* __restrict__ ecount,
          const uint64_t* __restrict__ state, int shift, unsigned long long* __restrict__ hist) {
    __shared__ unsigned int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const bool all = state[2] != 0;
    const uint64_t prefix = state[0], mask = shift >= 56 ? 0ull : (~0ull << (shift + 8));
    if (!all)
        for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
            const uint64_t key = keys[e];
            if (key == kNone || ((key ^ prefix) & mask) != 0) continue;
            atomicAdd(h + ((key >> shift) & 0xFF), (unsigned int)ecount[slot_of[e]]);
        }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(hist + threadIdx.x, (unsigned long long)h[threadIdx.x]);
}

// one thread walks the 256 digit weights; the others clear them for the next pass
__global__ void k_dc_digit(uint64_t* __restrict__ state, unsigned long long* __restrict__ hist, int shift) {
    __shared__ unsigned long long h[256];
    h[threadIdx.x] = hist[threadIdx.x];
    hist[threadIdx.x] = 0;
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (shift == 56) {
        unsigned long long total = 0;
        for (int d = 0; d < 256; ++d) total += h[d];
        if (total < state[1]) state[2] = 1;
    }
    if (!state[2]) {
        unsigned long long cum = 0;
        for (int d = 0; d < 256; ++d) {
            if (cum + h[d] >= state[1]) { state[0] |= (uint64_t)d << shift; state[1] -= cum; break; }
            cum += h[d];
        }
    }
    if (shift == 0) state[3] = state[2] ? kNone - 1 : state[0];
}

// ---- per round: selection and apply --------------------------------------------------------------------------------------------------
__device__ __forceinline__ void edge_ends(const int32_t* __restrict__ tri, uint32_t e, int32_t& a, int32_t& b) {
    const int32_t x = tri[e], y = tri[3 * (e / 3) + (e % 3 + 1) % 3];
    a = min(x, y); b = max(x, y);
}

__global__ void __launch_bounds__(256)
k_dc_vmin(const uint64_t* __restrict__ keys, uint32_t n, const int32_t* __restrict__ tri, const uint64_t* __restrict__ state,
          unsigned long long* __restrict__ vmin) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const uint64_t key = keys[e];
    if (key == kNone || key > state[3]) return;
    int32_t a, b;
    edge_ends(tri, e, a, b);
    atomicMin(vmin + a, (unsigned long long)key);
    atomicMin(vmin + b, (unsigned long long)key);
}

// r1[v] = min of vmin over v and its neighbours; target reset to the identity for the selection
__global__ void __launch_bounds__(256)
k_dc_r1(uint32_t V, const int32_t* __restrict__ tri, const int32_t* __restrict__ vstart, const int32_t* __restrict__ vfaces,
        const unsigned long long* __restrict__ vmin, unsigned long long* __restrict__ r1, int32_t* __restrict__ target) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    unsigned long long r = vmin[v];
    for (int32_t t = vstart[v]; t < vstart[v + 1]; ++t) {
        const int32_t* G = tri + 3 * (size_t)vfaces[t];
        r = min(r, min(vmin[G[0]], min(vmin[G[1]], vmin[G[2]])));
    }
    r1[v] = r;
    target[v] = (int32_t)v;
}

// Independence: let (a, b) and (c, d) be selected with keys k1 < k2.  r1[c] = k2 is the least vmin over c and its neighbours, and vmin[a],
// vmin[b] <= k1 < k2, so neither a nor b is c or a neighbour of c; the same holds for d.  The endpoints of two selected edges are thus
// distinct and pairwise non-adjacent: no face holds endpoints of both, so the two collapses change disjoint face sets, neither moves a
// vertex the other's validity test read, and each removes exactly its edge's faces.
__global__ void __launch_bounds__(256)
k_dc_select(const uint64_t* __restrict__ keys, uint32_t n, const int32_t* __restrict__ tri, const int32_t* __restrict__ slot_of,
            const int32_t* __restrict__ ecount, const uint64_t* __restrict__ state, const unsigned long long* __restrict__ r1,
            const float* __restrict__ pos, float* __restrict__ verts, double* __restrict__ Q, int32_t* __restrict__ target,
            int32_t* __restrict__ flive) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const uint64_t key = keys[e];
    if (key == kNone || key > state[3]) return;
    int32_t a, b;
    edge_ends(tri, e, a, b);
    if (r1[a] != key || r1[b] != key) return;
    target[b] = a;
#pragma unroll
    for (int i = 0; i < 3; ++i) verts[3 * (size_t)a + i] = pos[3 * (size_t)e + i];
#pragma unroll
    for (int i = 0; i < 10; ++i) Q[10 * (size_t)a + i] = __dadd_rn(Q[10 * (size_t)a + i], Q[10 * (size_t)b + i]);
    atomicSub(flive, ecount[slot_of[e]]);
}

inline uint32_t grid_of(size_t n) { return (uint32_t)div_up(n, (size_t)256); }

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_decim_init(const int32_t* tri, uint32_t F, uint8_t* fkeep, int32_t* flive, n2m_stream_t stream) {
    N2M_REQUIRE(flive, "decim_init", "null pointer");
    cudaMemsetAsync(flive, 0, sizeof(int32_t), as_stream(stream));
    if (F == 0) return check_launch("decim_init");
    N2M_REQUIRE(tri && fkeep, "decim_init", "null pointer");
    k_dc_init<<<grid_of(F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, flive);
    return check_launch("decim_init");
}

int n2m_decim_vcount(const int32_t* tri, uint32_t F, const uint8_t* fkeep, int32_t* vcount, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && fkeep && vcount, "decim_vcount", "null pointer");
    k_dc_vcount<<<grid_of(3 * (size_t)F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, vcount);
    return check_launch("decim_vcount");
}

int n2m_decim_vfill(const int32_t* tri, uint32_t F, const uint8_t* fkeep, int32_t* cursor, int32_t* vfaces, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && fkeep && cursor && vfaces, "decim_vfill", "null pointer");
    k_dc_vfill<<<grid_of(3 * (size_t)F), 256, 0, as_stream(stream)>>>(tri, F, fkeep, cursor, vfaces);
    return check_launch("decim_vfill");
}

int n2m_decim_quadrics(const float* vertices, uint32_t V, const int32_t* tri, const int32_t* vstart, int32_t* vfaces, double* Q,
                       n2m_stream_t stream) {
    if (V == 0) return 0;
    N2M_REQUIRE(vertices && tri && vstart && vfaces && Q, "decim_quadrics", "null pointer");
    k_dc_quadrics<<<grid_of(V), 256, 0, as_stream(stream)>>>(vertices, V, tri, vstart, vfaces, Q);
    return check_launch("decim_quadrics");
}

int n2m_decim_edges(const int32_t* tri, uint32_t V, uint32_t F, const uint8_t* fkeep, const int32_t* slot_of, uint32_t nslots, int32_t* ecount,
                    uint8_t* vbnd, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && fkeep && slot_of && ecount && vbnd, "decim_edges", "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(ecount, 0, nslots * sizeof(int32_t), s);
    cudaMemsetAsync(vbnd, 0, V, s);
    k_dc_ecount<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, fkeep, slot_of, ecount);
    k_dc_bnd<<<grid_of(3 * (size_t)F), 256, 0, s>>>(tri, F, fkeep, slot_of, ecount, vbnd);
    return check_launch("decim_edges");
}

int n2m_decim_eval(const float* vertices, const double* Q, const int32_t* tri, uint32_t F, const uint8_t* fkeep, const int32_t* table,
                   const int32_t* slot_of, const int32_t* ecount, const uint8_t* vbnd, const int32_t* vstart, const int32_t* vfaces, int optimal,
                   uint64_t* keys, float* pos, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(vertices && Q && tri && fkeep && table && slot_of && ecount && vbnd && vstart && vfaces && keys && pos, "decim_eval",
                "null pointer");
    k_dc_eval<<<grid_of(3 * (size_t)F), 256, 0, as_stream(stream)>>>(vertices, Q, tri, F, fkeep, table, slot_of, ecount, vbnd, vstart, vfaces,
                                                                    optimal, keys, pos);
    return check_launch("decim_eval");
}

int n2m_decim_threshold(const uint64_t* keys, uint32_t F, const int32_t* slot_of, const int32_t* ecount, const int32_t* flive, uint32_t target,
                        uint64_t* hist, uint64_t* state, n2m_stream_t stream) {
    N2M_REQUIRE(keys && slot_of && ecount && flive && hist && state, "decim_threshold", "null pointer");
    cudaStream_t s = as_stream(stream);
    unsigned long long* h = reinterpret_cast<unsigned long long*>(hist);
    const uint32_t n = 3 * F, blocks = n ? (uint32_t)std::min<size_t>(grid_of(n), 8 * (size_t)num_sms()) : 1;
    k_dc_need<<<1, 256, 0, s>>>(flive, target, state, h);
    for (int shift = 56; shift >= 0; shift -= 8) {
        k_dc_hist<<<blocks, 256, 0, s>>>(keys, n, slot_of, ecount, state, shift, h);
        k_dc_digit<<<1, 256, 0, s>>>(state, h, shift);
    }
    return check_launch("decim_threshold");
}

int n2m_decim_select(const uint64_t* keys, uint32_t V, uint32_t F, const int32_t* tri, const int32_t* slot_of, const int32_t* ecount,
                     const int32_t* vstart, const int32_t* vfaces, const uint64_t* state, const float* pos, uint64_t* vmin, uint64_t* r1,
                     float* vertices, double* Q, int32_t* target, int32_t* flive, n2m_stream_t stream) {
    if (F == 0 || V == 0) return 0;
    N2M_REQUIRE(keys && tri && slot_of && ecount && vstart && vfaces && state && pos && vmin && r1 && vertices && Q && target && flive,
                "decim_select", "null pointer");
    cudaStream_t s = as_stream(stream);
    unsigned long long* vm = reinterpret_cast<unsigned long long*>(vmin);
    unsigned long long* r = reinterpret_cast<unsigned long long*>(r1);
    cudaMemsetAsync(vmin, 0xFF, V * sizeof(uint64_t), s);
    k_dc_vmin<<<grid_of(3 * (size_t)F), 256, 0, s>>>(keys, 3 * F, tri, state, vm);
    k_dc_r1<<<grid_of(V), 256, 0, s>>>(V, tri, vstart, vfaces, vm, r, target);
    k_dc_select<<<grid_of(3 * (size_t)F), 256, 0, s>>>(keys, 3 * F, tri, slot_of, ecount, state, r, pos, vertices, Q, target, flive);
    return check_launch("decim_select");
}

}  // extern "C"
