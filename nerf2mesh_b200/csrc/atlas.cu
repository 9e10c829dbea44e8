// atlas.cu -- the UV atlas of a stage-1 mesh on the device: the library's own deterministic unwrap (normal-cone charts, one shared texel
// scale, shelf packing on the final-texel grid, a texel-conflict check at the bake raster).  C ABI include/n2m_b200_atlas.h, host side
// nerf2mesh_b200/texture.py (uv_unwrap), CPU restatement tests/atlas_oracle.py.
//
// The rule, step by step (the host drives the rounds; every float64 operation is an explicit __d*_rn intrinsic, so no FMA contraction
// separates the kernels from the numpy restatement, and the atomics only count, fill order-free lists and take minima / maxima):
//   1. k_at_faces     float64 unit normal n = cross(b - a, c - a) / |.|; bucket = the argmax of dot(n, axis_i) over the 26 axes
//                     normalize(i, j, k), (i, j, k) in {-1, 0, 1}^3 \ 0, the lowest index on a tie.  A face that repeats an index or whose
//                     cross product is zero is degenerate: bucket -1, a chart of its own, projected along axis 0.
//   2. k_at_ecount / k_at_mates / k_at_union / k_at_labels   base charts: faces across a 2-manifold edge of the non-degenerate faces'
//                     edge table (n2m_clean_edge_table) with the same bucket share a chart (union-find, root = the lowest face).
//   3. k_at_count / k_at_fill / k_at_propose / k_at_accept   one merge round: a chart of fewer than `small` faces proposes to the
//                     neighbouring chart it shares the most manifold edges with (ties: the lowest chart id) when every one of its faces has
//                     dot(n, axis of that chart) >= 0.5; the proposal is accepted unless the target proposes too.  The merged chart keeps
//                     the target's id and axis.
//   4. k_at_boxes / k_at_orient   per chart and angle k of the host's table: the bounding box of (cos u - sin v, sin u + cos v), (u, v) =
//                     (p.e1, p.e2) in the axis's basis; the least area wins (ties: the lowest k), then a box taller than wide turns by
//                     +90 degrees ((x, y) -> (-y, x)).
//   5. k_at_bitonic / k_at_pack   charts sorted by (box height desc, chart index); one CTA bisects the largest common scale s (final
//                     texels per unit length) at which next-fit-decreasing-height shelves of ceil(s W) x ceil(s H) rectangles, PAD texels
//                     apart and from the border, fit the texture.
//   6. k_at_texels<0, 1> / k_at_merged / k_at_split        the bake-raster texel centres strictly inside two faces (float64 edge
//                     functions of the float32 vt); a chart holding one re-splits into its base charts when it is a merged chart, else
//                     into single faces.
//   7. k_at_corner_keys / k_at_bitonic / k_at_row_flags / k_at_emit   one vt row per distinct (chart, vertex), in key order.
#include "n2m_common.cuh"
#include "union_find.cuh"
#include "../../include/n2m_b200_atlas.h"

#include <limits.h>

namespace n2m {
namespace {

constexpr int kAxes = 26;
constexpr int kMaxSmall = 32;              // the merge's small-chart bound is below this (local candidate list of 3 (small - 1) charts)
constexpr int kMaxAngles = 64;
constexpr int kPackThreads = 1024;

__device__ __forceinline__ double dot3(const double* x, const double* y) {
    return __dadd_rn(__dadd_rn(__dmul_rn(x[0], y[0]), __dmul_rn(x[1], y[1])), __dmul_rn(x[2], y[2]));
}
__device__ __forceinline__ void load_p(const float* __restrict__ verts, int32_t v, double p[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = (double)verts[3 * (size_t)v + a];
}
// double -> u64 whose unsigned order is the value order
__device__ __forceinline__ uint64_t dkey(double x) {
    const uint64_t u = (uint64_t)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double dkey_inv(uint64_t k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
}
__device__ __forceinline__ int32_t chart_index(const int32_t* __restrict__ incl, const int32_t* __restrict__ label, int32_t f) {
    return incl[label[f]] - 1;
}

// (x, y) of point p in chart coordinates before the turn: (u, v) = (p.e1, p.e2) of the axis's basis, rotated by the angle (c, s)
__device__ __forceinline__ void rotated(const double* p, const double* basis, double c, double s, double& x, double& y) {
    const double u = dot3(p, basis), v = dot3(p, basis + 3);
    x = __dsub_rn(__dmul_rn(c, u), __dmul_rn(s, v));
    y = __dadd_rn(__dmul_rn(s, u), __dmul_rn(c, v));
}

struct Chart {
    const double* basis;
    double c, s, ox, oy;
    int turn;
    int32_t tx, ty;
};
__device__ __forceinline__ Chart chart_of(int32_t ci, int32_t axis, const double* __restrict__ basis, const double* __restrict__ rot,
                                          const int32_t* __restrict__ orient, const double* __restrict__ org, const int32_t* __restrict__ off) {
    Chart ch;
    const int32_t o = orient[ci];
    ch.basis = basis + 6 * axis;
    ch.c = rot[2 * (o & 0xFFFF)]; ch.s = rot[2 * (o & 0xFFFF) + 1];
    ch.turn = o >> 16;
    ch.ox = org[2 * (size_t)ci]; ch.oy = org[2 * (size_t)ci + 1];
    ch.tx = off[2 * (size_t)ci]; ch.ty = off[2 * (size_t)ci + 1];
    return ch;
}
// vt of point p in chart ch: (offset + s (xy - origin)) / resolution, rounded once to float32
__device__ __forceinline__ float2 chart_vt(const Chart& ch, const double* p, double scale, double res) {
    double x, y;
    rotated(p, ch.basis, ch.c, ch.s, x, y);
    if (ch.turn) { const double t = x; x = -y; y = t; }
    const double u = __ddiv_rn(__dadd_rn((double)ch.tx, __dmul_rn(scale, __dsub_rn(x, ch.ox))), res);
    const double v = __ddiv_rn(__dadd_rn((double)ch.ty, __dmul_rn(scale, __dsub_rn(y, ch.oy))), res);
    return make_float2(__double2float_rn(u), __double2float_rn(v));
}

// ---- 1. faces ------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_at_faces(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t F, const double* __restrict__ axes, double* __restrict__ nrm,
           int32_t* __restrict__ bucket, uint8_t* __restrict__ fkeep) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int32_t a = tri[3 * (size_t)f], b = tri[3 * (size_t)f + 1], c = tri[3 * (size_t)f + 2];
    double p[3][3], e1[3], e2[3], n[3];
    load_p(verts, a, p[0]); load_p(verts, b, p[1]); load_p(verts, c, p[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) { e1[k] = __dsub_rn(p[1][k], p[0][k]); e2[k] = __dsub_rn(p[2][k], p[0][k]); }
    n[0] = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
    n[1] = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
    n[2] = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
    const double ln = __dsqrt_rn(dot3(n, n));
    if (a == b || b == c || a == c || !(ln > 0.0)) {
        bucket[f] = -1; fkeep[f] = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) nrm[3 * (size_t)f + k] = 0.0;
        return;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { n[k] = __ddiv_rn(n[k], ln); nrm[3 * (size_t)f + k] = n[k]; }
    int32_t best = 0;
    double bd = dot3(n, axes);
    for (int i = 1; i < kAxes; ++i) {
        const double d = dot3(n, axes + 3 * i);
        if (d > bd) { bd = d; best = i; }
    }
    bucket[f] = best; fkeep[f] = 1;
}

// ---- 2. base charts ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_at_ecount(uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ slot_of, int32_t* __restrict__ ecount) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < 3 * F && fkeep[e / 3]) atomicAdd(ecount + slot_of[e], 1);
}

// mate[e] = the other face-edge of a 2-manifold edge (-1 elsewhere, caller-initialised): the higher of the two writes both
__global__ void __launch_bounds__(256)
k_at_mates(uint32_t F, const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ table, const int32_t* __restrict__ slot_of,
           const int32_t* __restrict__ ecount, int32_t* __restrict__ mate) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F || !fkeep[e / 3]) return;
    const int32_t s = slot_of[e], lo = table[s];
    if (ecount[s] != 2 || lo == (int32_t)e) return;
    mate[e] = lo;
    mate[lo] = (int32_t)e;
}

__global__ void __launch_bounds__(256) k_at_iota(int32_t* __restrict__ x, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = (int32_t)i;
}

__global__ void __launch_bounds__(256)
k_at_union(uint32_t F, const int32_t* __restrict__ mate, const int32_t* __restrict__ bucket, int32_t* parent) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F || mate[e] < 0) return;
    const int32_t f = (int32_t)(e / 3), g = mate[e] / 3;
    if (f < g && bucket[f] == bucket[g]) uf_union(parent, f, g);
}

__global__ void __launch_bounds__(256)
k_at_labels(uint32_t F, const int32_t* __restrict__ parent, const int32_t* __restrict__ bucket, int32_t* __restrict__ base,
            int32_t* __restrict__ label, int32_t* __restrict__ fax) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int32_t r = uf_root(parent, (int32_t)f);
    base[f] = r; label[f] = r;
    fax[f] = max(bucket[f], 0);
}

// ---- 3. merging small charts ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_at_count(uint32_t F, const int32_t* __restrict__ label, int32_t* __restrict__ count) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F) atomicAdd(count + label[f], 1);
}

__global__ void __launch_bounds__(256)
k_at_fill(uint32_t F, const int32_t* __restrict__ label, int32_t* __restrict__ cursor, int32_t* __restrict__ items) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F) items[atomicAdd(cursor + label[f], 1)] = (int32_t)f;
}

// one thread per chart id c (a face with label[c] == c); every decision is a function of sets, so the fill order does not matter
__global__ void __launch_bounds__(128)
k_at_propose(uint32_t F, uint32_t small, const double* __restrict__ nrm, const double* __restrict__ axes, const int32_t* __restrict__ bucket,
             const int32_t* __restrict__ label, const int32_t* __restrict__ fax, const int32_t* __restrict__ mate, const int32_t* __restrict__ count,
             const int32_t* __restrict__ start, const int32_t* __restrict__ items, int32_t* __restrict__ propose) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= F || label[c] != (int32_t)c || bucket[c] < 0) return;
    const int32_t n = count[c];
    if ((uint32_t)n >= small) return;
    int32_t cand[3 * (kMaxSmall - 1)];
    int nc = 0;
    for (int32_t t = 0; t < n; ++t) {
        const int32_t f = items[start[c] + t];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int32_t m = mate[3 * (size_t)f + k];
            if (m < 0) continue;
            const int32_t g = label[m / 3];
            if (g != (int32_t)c) cand[nc++] = g;
        }
    }
    int32_t best = -1, bc = 0;
    for (int i = 0; i < nc; ++i) {
        int cnt = 0;
        for (int j = 0; j < nc; ++j) cnt += cand[j] == cand[i];
        if (cnt > bc || (cnt == bc && cand[i] < best)) { bc = cnt; best = cand[i]; }
    }
    if (best < 0) return;
    const double* ax = axes + 3 * fax[best];
    for (int32_t t = 0; t < n; ++t)
        if (!(dot3(nrm + 3 * (size_t)items[start[c] + t], ax) >= 0.5)) return;
    propose[c] = best;
}

__global__ void __launch_bounds__(256)
k_at_accept(uint32_t F, const int32_t* __restrict__ propose, int32_t* __restrict__ label, int32_t* __restrict__ fax) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int32_t b = propose[label[f]];
    if (b >= 0 && propose[b] < 0) { label[f] = b; fax[f] = fax[b]; }      // b's chart does not move this round
}

__global__ void __launch_bounds__(256) k_at_roots(uint32_t F, const int32_t* __restrict__ label, int32_t* __restrict__ flag) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F) flag[f] = label[f] == (int32_t)f;
}

// ---- 4. projection and rotation ------------------------------------------------------------------------------------------------------
// bmin / bmax [C, K, 2] u64 (dkey of x, y); one thread per face, its three corners reduced before the atomics
__global__ void __launch_bounds__(256)
k_at_boxes(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t F, const int32_t* __restrict__ label,
           const int32_t* __restrict__ incl, const int32_t* __restrict__ fax, const double* __restrict__ basis, const double* __restrict__ rot,
           uint32_t K, unsigned long long* __restrict__ bmin, unsigned long long* __restrict__ bmax) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const size_t ci = (size_t)chart_index(incl, label, (int32_t)f);
    double p[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) load_p(verts, tri[3 * (size_t)f + c], p[c]);
    const double* B = basis + 6 * fax[f];
    for (uint32_t k = 0; k < K; ++k) {
        uint64_t x0 = ~0ull, y0 = ~0ull, x1 = 0, y1 = 0;             // in key order, so -0 stays below +0 as in the atomics
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double x, y;
            rotated(p[c], B, rot[2 * k], rot[2 * k + 1], x, y);
            const uint64_t kx = dkey(x), ky = dkey(y);
            x0 = min(x0, kx); x1 = max(x1, kx); y0 = min(y0, ky); y1 = max(y1, ky);
        }
        const size_t o = 2 * (ci * K + k);
        atomicMin(bmin + o, x0); atomicMin(bmin + o + 1, y0);
        atomicMax(bmax + o, x1); atomicMax(bmax + o + 1, y1);
    }
}

__global__ void __launch_bounds__(256)
k_at_orient(uint32_t C, uint32_t K, const unsigned long long* __restrict__ bmin, const unsigned long long* __restrict__ bmax,
            int32_t* __restrict__ orient, double* __restrict__ org, double* __restrict__ ext, uint64_t* __restrict__ skey,
            int32_t* __restrict__ sval) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    uint32_t bk = 0;
    double x0 = 0, y0 = 0, x1 = 0, y1 = 0, ba = 0;
    for (uint32_t k = 0; k < K; ++k) {
        const size_t o = 2 * ((size_t)c * K + k);
        const double a0 = dkey_inv(bmin[o]), b0 = dkey_inv(bmin[o + 1]), a1 = dkey_inv(bmax[o]), b1 = dkey_inv(bmax[o + 1]);
        const double area = __dmul_rn(__dsub_rn(a1, a0), __dsub_rn(b1, b0));
        if (k == 0 || area < ba) { bk = k; ba = area; x0 = a0; y0 = b0; x1 = a1; y1 = b1; }
    }
    double w = __dsub_rn(x1, x0), h = __dsub_rn(y1, y0);
    int turn = 0;
    if (h > w) {                            // (x, y) -> (-y, x): the new x runs over [-y1, -y0], the new y over [x0, x1]
        turn = 1;
        const double t = w; w = h; h = t;
        const double nx0 = -y1;
        y0 = x0; x0 = nx0;
    }
    orient[c] = (int32_t)(bk | (turn << 16));
    org[2 * (size_t)c] = x0; org[2 * (size_t)c + 1] = y0;
    ext[2 * (size_t)c] = w; ext[2 * (size_t)c + 1] = h;
    const double bh = h;
    skey[c] = ~(uint64_t)__double_as_longlong(bh);          // bh >= +0: the bit pattern orders as the value; ~ sorts descending
    sval[c] = (int32_t)c;
}

// ---- sort of (key, value) pairs, lexicographic: bitonic, one launch per merge step ----------------------------------------------------
__global__ void __launch_bounds__(256) k_at_pad(uint64_t* __restrict__ keys, int32_t* __restrict__ vals, uint32_t n, uint32_t cap) {
    const uint32_t i = n + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cap) { keys[i] = ~0ull; vals[i] = INT_MAX; }
}
__global__ void __launch_bounds__(256) k_at_bitonic(uint64_t* keys, int32_t* vals, uint32_t cap, uint32_t k, uint32_t j) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    const uint32_t l = i ^ j;
    if (l <= i) return;
    const uint64_t ki = keys[i], kl = keys[l];
    const int32_t vi = vals[i], vl = vals[l];
    const bool greater = ki > kl || (ki == kl && vi > vl);
    if (((i & k) == 0) == greater) { keys[i] = kl; keys[l] = ki; vals[i] = vl; vals[l] = vi; }
}

// ---- 5. packing: one CTA -------------------------------------------------------------------------------------------------------------
struct PackBuf {
    int32_t *wid, *hgt, *nxt, *shelf_a, *shelf_y;
    long long* P;
};

// Next-fit decreasing height at scale s over the charts in `order`: chart i of the order is ceil(s W) x ceil(s H) final texels (at
// least 1), x_0 = pad, x_{i+1} = x_i + w_i + pad within a shelf, a shelf is as tall as its first chart and the next starts pad texels
// above it.  Returns whether it fits in res x res with pad texels to the border; `write` also stores the offsets.
__device__ bool layout(const double* __restrict__ ext, const int32_t* __restrict__ order, uint32_t C, double s, int res, int pad,
                       const PackBuf& b, bool write, int32_t* __restrict__ off) {
    __shared__ long long part[kPackThreads];
    __shared__ int ok_sh, nshelf_sh;
    const uint32_t t = threadIdx.x, chunk = (C + kPackThreads - 1) / kPackThreads;
    const uint32_t i0 = min(C, t * chunk), i1 = min(C, i0 + chunk);
    long long sum = 0;
    for (uint32_t i = i0; i < i1; ++i) {
        const int32_t c = order[i];
        const int32_t w = max(1, (int32_t)ceil(__dmul_rn(s, ext[2 * (size_t)c])));
        const int32_t h = max(1, (int32_t)ceil(__dmul_rn(s, ext[2 * (size_t)c + 1])));
        b.wid[i] = w; b.hgt[i] = h;
        sum += w + pad;
    }
    part[t] = sum;
    __syncthreads();
    for (uint32_t d = 1; d < kPackThreads; d <<= 1) {           // inclusive scan of the chunk sums
        const long long v = t >= d ? part[t - d] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    long long run = part[t] - sum;
    for (uint32_t i = i0; i < i1; ++i) { b.P[i] = run; run += b.wid[i] + pad; }
    if (t == kPackThreads - 1) b.P[C] = part[t];
    __syncthreads();
    const long long room = res - pad;
    for (uint32_t i = t; i < C; i += kPackThreads) {             // nxt[i] = the largest e with P[e] - P[i] <= room
        uint32_t lo = i, hi = C;
        const long long lim = b.P[i] + room;
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if (b.P[mid] <= lim) lo = mid; else hi = mid - 1;
        }
        b.nxt[i] = (int32_t)lo;
    }
    __syncthreads();
    if (t == 0) {
        int ok = 1, ns = 0;
        long long y = pad;
        for (uint32_t a = 0; a < C;) {
            const uint32_t e = (uint32_t)b.nxt[a];
            if (e == a || y + b.hgt[a] + pad > res) { ok = 0; break; }
            if (write) { b.shelf_a[ns] = (int32_t)a; b.shelf_y[ns] = (int32_t)y; }
            ++ns;
            y += b.hgt[a] + pad;
            a = e;
        }
        ok_sh = ok; nshelf_sh = ns;
    }
    __syncthreads();
    const bool ok = ok_sh != 0;
    if (write && ok) {
        const int ns = nshelf_sh;
        for (uint32_t i = t; i < C; i += kPackThreads) {
            int lo = 0, hi = ns - 1;                             // the last shelf start <= i
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if ((uint32_t)b.shelf_a[mid] <= i) lo = mid; else hi = mid - 1;
            }
            const int32_t c = order[i];
            off[2 * (size_t)c] = (int32_t)(pad + b.P[i] - b.P[b.shelf_a[lo]]);
            off[2 * (size_t)c + 1] = b.shelf_y[lo];
        }
    }
    __syncthreads();
    return ok;
}

// state[0] = s, state[1] = 1 when the charts fit at the smallest scale (else 0 and no offsets)
__global__ void __launch_bounds__(kPackThreads)
k_at_pack(const double* __restrict__ ext, const int32_t* __restrict__ order, uint32_t C, int res, int pad, int steps, PackBuf b,
          int32_t* __restrict__ off, double* __restrict__ state) {
    __shared__ double wmax[kPackThreads];
    double m = 0.0;
    for (uint32_t i = threadIdx.x; i < C; i += kPackThreads) m = fmax(m, ext[2 * (size_t)i]);
    wmax[threadIdx.x] = m;
    __syncthreads();
    for (uint32_t d = kPackThreads / 2; d > 0; d >>= 1) {
        if (threadIdx.x < d) wmax[threadIdx.x] = fmax(wmax[threadIdx.x], wmax[threadIdx.x + d]);
        __syncthreads();
    }
    const double W = wmax[0];
    double hi = W > 0.0 ? __ddiv_rn((double)(res - 2 * pad), W) : (double)res;
    double lo = __dmul_rn(hi, 0x1p-20);
    if (!layout(ext, order, C, lo, res, pad, b, false, off)) {
        if (threadIdx.x == 0) { state[0] = lo; state[1] = 0.0; }
        return;
    }
    if (layout(ext, order, C, hi, res, pad, b, false, off)) {
        lo = hi;
    } else {
        for (int it = 0; it < steps; ++it) {
            const double mid = __dsqrt_rn(__dmul_rn(lo, hi));
            if (layout(ext, order, C, mid, res, pad, b, false, off)) lo = mid; else hi = mid;
        }
    }
    layout(ext, order, C, lo, res, pad, b, true, off);
    if (threadIdx.x == 0) { state[0] = lo; state[1] = 1.0; }
}

// ---- 6. texel conflicts --------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double edge_fn(double ax, double ay, double bx, double by, double px, double py) {
    return __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(py, ay)), __dmul_rn(__dsub_rn(by, ay), __dsub_rn(px, ax)));
}

struct FaceUV { double x[3], y[3]; int32_t i0, i1, j0, j1; };
__device__ __forceinline__ FaceUV face_uv(const float* __restrict__ verts, const int32_t* __restrict__ tri, int32_t f, const Chart& ch,
                                          double scale, double res, uint32_t R) {
    FaceUV u;
    double p[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        load_p(verts, tri[3 * (size_t)f + k], p);
        const float2 t = chart_vt(ch, p, scale, res);
        u.x[k] = __dmul_rn((double)t.x, (double)R); u.y[k] = __dmul_rn((double)t.y, (double)R);     // exact: 24 x 32 bits
    }
    // texel (i, j) has its centre at (i + 0.5, j + 0.5): the candidates of the face's bounding box, clamped to the raster
    const double x0 = fmin(u.x[0], fmin(u.x[1], u.x[2])), x1 = fmax(u.x[0], fmax(u.x[1], u.x[2]));
    const double y0 = fmin(u.y[0], fmin(u.y[1], u.y[2])), y1 = fmax(u.y[0], fmax(u.y[1], u.y[2]));
    u.i0 = max(0, (int32_t)ceil(x0 - 0.5)); u.i1 = min((int32_t)R - 1, (int32_t)floor(x1 - 0.5));
    u.j0 = max(0, (int32_t)ceil(y0 - 0.5)); u.j1 = min((int32_t)R - 1, (int32_t)floor(y1 - 0.5));
    return u;
}
__device__ __forceinline__ bool strictly_inside(const FaceUV& u, double px, double py) {
    return edge_fn(u.x[0], u.y[0], u.x[1], u.y[1], px, py) > 0.0 && edge_fn(u.x[1], u.y[1], u.x[2], u.y[2], px, py) > 0.0 &&
           edge_fn(u.x[2], u.y[2], u.x[0], u.y[0], px, py) > 0.0;
}

struct ChartArgs {
    const int32_t *label, *incl, *fax, *orient, *off;
    const double *basis, *rot, *org, *state;
};

// one warp per face; PASS 0: owner[texel] = the lowest face strictly over it; PASS 1: a face over a texel another face owns marks its chart
template <int PASS>
__global__ void __launch_bounds__(256)
k_at_texels(const float* __restrict__ verts, const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ fkeep, ChartArgs a,
            int res, uint32_t R, int32_t* __restrict__ owner, uint8_t* __restrict__ conf, int32_t* __restrict__ nconf) {
    const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (f >= F || !fkeep[f]) return;
    const int32_t ci = chart_index(a.incl, a.label, (int32_t)f);
    const Chart ch = chart_of(ci, a.fax[f], a.basis, a.rot, a.orient, a.org, a.off);
    const FaceUV u = face_uv(verts, tri, (int32_t)f, ch, a.state[0], (double)res, R);
    if (u.i1 < u.i0 || u.j1 < u.j0) return;
    const uint32_t nw = (uint32_t)(u.i1 - u.i0 + 1), n = nw * (uint32_t)(u.j1 - u.j0 + 1);
    int hits = 0;
    for (uint32_t q = lane; q < n; q += 32) {
        const int32_t i = u.i0 + (int32_t)(q % nw), j = u.j0 + (int32_t)(q / nw);
        if (!strictly_inside(u, i + 0.5, j + 0.5)) continue;
        const size_t t = (size_t)j * R + i;
        if (PASS == 0) atomicMin(owner + t, (int32_t)f);
        else hits += owner[t] != (int32_t)f;
    }
    if (PASS == 1) {
        hits = __reduce_add_sync(0xFFFFFFFFu, hits);
        if (lane == 0 && hits) { conf[ci] = 1; atomicAdd(nconf, hits); }
    }
}

__global__ void __launch_bounds__(256)
k_at_merged(uint32_t F, const int32_t* __restrict__ label, const int32_t* __restrict__ incl, const int32_t* __restrict__ base,
            uint8_t* __restrict__ merged) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < F && base[f] != label[f]) merged[chart_index(incl, label, (int32_t)f)] = 1;
}

__global__ void __launch_bounds__(256)
k_at_split(uint32_t F, const int32_t* __restrict__ incl, const int32_t* __restrict__ base, const int32_t* __restrict__ bucket,
           const uint8_t* __restrict__ conf, const uint8_t* __restrict__ merged, int32_t* __restrict__ label, int32_t* __restrict__ fax) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int32_t ci = incl[label[f]] - 1;
    if (!conf[ci]) return;
    label[f] = merged[ci] ? base[f] : (int32_t)f;
    fax[f] = max(bucket[f], 0);
}

// ---- 7. emit -------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_at_corner_keys(const int32_t* __restrict__ tri, uint32_t F, const int32_t* __restrict__ label, const int32_t* __restrict__ incl,
                 uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * F) return;
    keys[e] = ((uint64_t)(uint32_t)chart_index(incl, label, (int32_t)(e / 3)) << 32) | (uint32_t)tri[e];
    vals[e] = (int32_t)e;
}

__global__ void __launch_bounds__(256) k_at_row_flags(const uint64_t* __restrict__ keys, uint32_t n, int32_t* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = i == 0 || keys[i] != keys[i - 1];
}

__global__ void __launch_bounds__(256)
k_at_emit(const float* __restrict__ verts, const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint32_t n,
          const int32_t* __restrict__ rows, ChartArgs a, int res, float* __restrict__ vt, int32_t* __restrict__ ft, int32_t* __restrict__ vmap) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t row = rows[i] - 1, e = vals[i];
    ft[e] = row;
    if (i > 0 && keys[i] == keys[i - 1]) return;
    const int32_t v = (int32_t)(uint32_t)keys[i], ci = (int32_t)(keys[i] >> 32);
    const Chart ch = chart_of(ci, a.fax[e / 3], a.basis, a.rot, a.orient, a.org, a.off);
    double p[3];
    load_p(verts, v, p);
    const float2 t = chart_vt(ch, p, a.state[0], (double)res);
    vt[2 * (size_t)row] = t.x; vt[2 * (size_t)row + 1] = t.y;
    vmap[row] = v;
}

// contract() of the unwrap's positions: the one definition of the step and the bake (n2m_common.cuh)
__global__ void __launch_bounds__(256) k_at_contract(const float* __restrict__ verts, uint32_t V, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    float p[3] = {verts[3 * (size_t)i], verts[3 * (size_t)i + 1], verts[3 * (size_t)i + 2]};
    contract_linf(p);
#pragma unroll
    for (int a = 0; a < 3; ++a) out[3 * (size_t)i + a] = p[a];
}

inline uint32_t grid_of(size_t n) { return (uint32_t)div_up(n, (size_t)256); }
inline bool pow2(uint32_t n) { return n && !(n & (n - 1)); }

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_atlas_contract(const float* vertices, uint32_t V, float* out, n2m_stream_t stream) {
    if (V == 0) return 0;
    N2M_REQUIRE(vertices && out, "atlas_contract", "null pointer");
    k_at_contract<<<grid_of(V), 256, 0, as_stream(stream)>>>(vertices, V, out);
    return check_launch("atlas_contract");
}

int n2m_atlas_faces(const float* vertices, const int32_t* tri, uint32_t F, const double* axes, double* nrm, int32_t* bucket, uint8_t* fkeep,
                    n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(vertices && tri && axes && nrm && bucket && fkeep, "atlas_faces", "null pointer");
    k_at_faces<<<grid_of(F), 256, 0, as_stream(stream)>>>(vertices, tri, F, axes, nrm, bucket, fkeep);
    return check_launch("atlas_faces");
}

int n2m_atlas_base(uint32_t F, const uint8_t* fkeep, const int32_t* bucket, const int32_t* table, const int32_t* slot_of, uint32_t nslots,
                   int32_t* ecount, int32_t* mate, int32_t* parent, int32_t* base, int32_t* label, int32_t* fax, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(nslots) && nslots >= 6 * (uint64_t)F, "atlas_base", "power-of-two table of at least 6 F slots");
    if (F == 0) return 0;
    N2M_REQUIRE(fkeep && bucket && table && slot_of && ecount && mate && parent && base && label && fax, "atlas_base", "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(ecount, 0, nslots * sizeof(int32_t), s);
    cudaMemsetAsync(mate, 0xFF, 3 * (size_t)F * sizeof(int32_t), s);
    k_at_ecount<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, fkeep, slot_of, ecount);
    k_at_mates<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, fkeep, table, slot_of, ecount, mate);
    k_at_iota<<<grid_of(F), 256, 0, s>>>(parent, F);
    k_at_union<<<grid_of(3 * (size_t)F), 256, 0, s>>>(F, mate, bucket, parent);
    k_at_labels<<<grid_of(F), 256, 0, s>>>(F, parent, bucket, base, label, fax);
    return check_launch("atlas_base");
}

int n2m_atlas_chart_count(uint32_t F, const int32_t* label, int32_t* count, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(label && count, "atlas_chart_count", "null pointer");
    cudaMemsetAsync(count, 0, F * sizeof(int32_t), as_stream(stream));
    k_at_count<<<grid_of(F), 256, 0, as_stream(stream)>>>(F, label, count);
    return check_launch("atlas_chart_count");
}

int n2m_atlas_merge_round(uint32_t F, uint32_t small, const double* nrm, const double* axes, const int32_t* bucket, const int32_t* mate,
                          const int32_t* count, const int32_t* start, int32_t* cursor, int32_t* items, int32_t* propose, int32_t* label,
                          int32_t* fax, n2m_stream_t stream) {
    N2M_REQUIRE(small <= kMaxSmall, "atlas_merge_round", "small-chart bound above 32 faces");
    if (F == 0) return 0;
    N2M_REQUIRE(nrm && axes && bucket && mate && count && start && cursor && items && propose && label && fax, "atlas_merge_round",
                "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemcpyAsync(cursor, start, F * sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
    cudaMemsetAsync(propose, 0xFF, F * sizeof(int32_t), s);
    k_at_fill<<<grid_of(F), 256, 0, s>>>(F, label, cursor, items);
    k_at_propose<<<(uint32_t)div_up(F, 128u), 128, 0, s>>>(F, small, nrm, axes, bucket, label, fax, mate, count, start, items, propose);
    k_at_accept<<<grid_of(F), 256, 0, s>>>(F, propose, label, fax);
    return check_launch("atlas_merge_round");
}

int n2m_atlas_roots(uint32_t F, const int32_t* label, int32_t* flag, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(label && flag, "atlas_roots", "null pointer");
    k_at_roots<<<grid_of(F), 256, 0, as_stream(stream)>>>(F, label, flag);
    return check_launch("atlas_roots");
}

int n2m_atlas_orient(const float* vertices, const int32_t* tri, uint32_t F, const int32_t* label, const int32_t* incl, const int32_t* fax,
                     const double* basis, const double* rot, uint32_t K, uint32_t C, uint64_t* bmin, uint64_t* bmax, int32_t* orient,
                     double* org, double* ext, uint64_t* skey, int32_t* sval, n2m_stream_t stream) {
    N2M_REQUIRE(K >= 1 && K <= kMaxAngles, "atlas_orient", "1 to 64 angles");
    if (F == 0 || C == 0) return 0;
    N2M_REQUIRE(vertices && tri && label && incl && fax && basis && rot && bmin && bmax && orient && org && ext && skey && sval, "atlas_orient",
                "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(bmin, 0xFF, 2 * (size_t)C * K * sizeof(uint64_t), s);
    cudaMemsetAsync(bmax, 0, 2 * (size_t)C * K * sizeof(uint64_t), s);
    k_at_boxes<<<grid_of(F), 256, 0, s>>>(vertices, tri, F, label, incl, fax, basis, rot, K, (unsigned long long*)bmin,
                                                     (unsigned long long*)bmax);
    k_at_orient<<<grid_of(C), 256, 0, s>>>(C, K, (const unsigned long long*)bmin, (const unsigned long long*)bmax, orient, org, ext, skey, sval);
    return check_launch("atlas_orient");
}

int n2m_atlas_sort(uint64_t* keys, int32_t* vals, uint32_t n, uint32_t cap, n2m_stream_t stream) {
    N2M_REQUIRE(pow2(cap) && cap >= n, "atlas_sort", "power-of-two buffers of at least n entries");
    if (n <= 1) return 0;
    N2M_REQUIRE(keys && vals, "atlas_sort", "null pointer");
    cudaStream_t s = as_stream(stream);
    uint32_t p = 1;
    while (p < n) p <<= 1;
    k_at_pad<<<grid_of(p - n + 1), 256, 0, s>>>(keys, vals, n, p);
    for (uint32_t k = 2; k <= p; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) k_at_bitonic<<<grid_of(p), 256, 0, s>>>(keys, vals, p, k, j);
    return check_launch("atlas_sort");
}

int n2m_atlas_pack(const double* ext, const int32_t* order, uint32_t C, int32_t res, int32_t pad, int32_t steps, int32_t* wid, int32_t* hgt,
                   int32_t* nxt, int32_t* shelf_a, int32_t* shelf_y, long long* prefix, int32_t* off, double* state, n2m_stream_t stream) {
    N2M_REQUIRE(C >= 1 && res > 2 * pad && pad >= 0 && steps >= 0, "atlas_pack", "C >= 1, res > 2 pad, pad >= 0, steps >= 0");
    N2M_REQUIRE(ext && order && wid && hgt && nxt && shelf_a && shelf_y && prefix && off && state, "atlas_pack", "null pointer");
    PackBuf b{wid, hgt, nxt, shelf_a, shelf_y, prefix};
    k_at_pack<<<1, kPackThreads, 0, as_stream(stream)>>>(ext, order, C, res, pad, steps, b, off, state);
    return check_launch("atlas_pack");
}

int n2m_atlas_conflicts(const float* vertices, const int32_t* tri, uint32_t F, const uint8_t* fkeep, const int32_t* label, const int32_t* incl,
                        const int32_t* fax, const double* basis, const double* rot, const int32_t* orient, const double* org, const int32_t* off,
                        const double* state, uint32_t C, int32_t res, uint32_t R, int32_t* owner, uint8_t* conf, int32_t* nconf,
                        n2m_stream_t stream) {
    N2M_REQUIRE((uint64_t)R * R < (1ull << 31) && R >= 1 && res >= 1, "atlas_conflicts", "raster of fewer than 2^31 texels");
    N2M_REQUIRE(nconf, "atlas_conflicts", "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(nconf, 0, sizeof(int32_t), s);
    if (F == 0 || C == 0) return check_launch("atlas_conflicts");
    N2M_REQUIRE(vertices && tri && fkeep && label && incl && fax && basis && rot && orient && org && off && state && owner && conf,
                "atlas_conflicts", "null pointer");
    cudaMemsetAsync(owner, 0x7F, (size_t)R * R * sizeof(int32_t), s);
    cudaMemsetAsync(conf, 0, C, s);
    const ChartArgs a{label, incl, fax, orient, off, basis, rot, org, state};
    const uint32_t blocks = (uint32_t)div_up((size_t)F * 32, (size_t)256);
    k_at_texels<0><<<blocks, 256, 0, s>>>(vertices, tri, F, fkeep, a, res, R, owner, conf, nconf);
    k_at_texels<1><<<blocks, 256, 0, s>>>(vertices, tri, F, fkeep, a, res, R, owner, conf, nconf);
    return check_launch("atlas_conflicts");
}

int n2m_atlas_split(uint32_t F, uint32_t C, const int32_t* incl, const int32_t* base, const int32_t* bucket, const uint8_t* conf,
                    uint8_t* merged, int32_t* label, int32_t* fax, n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(incl && base && bucket && conf && merged && label && fax, "atlas_split", "null pointer");
    cudaStream_t s = as_stream(stream);
    cudaMemsetAsync(merged, 0, C, s);
    k_at_merged<<<grid_of(F), 256, 0, s>>>(F, label, incl, base, merged);
    k_at_split<<<grid_of(F), 256, 0, s>>>(F, incl, base, bucket, conf, merged, label, fax);
    return check_launch("atlas_split");
}

int n2m_atlas_corner_keys(const int32_t* tri, uint32_t F, const int32_t* label, const int32_t* incl, uint64_t* keys, int32_t* vals,
                          n2m_stream_t stream) {
    if (F == 0) return 0;
    N2M_REQUIRE(tri && label && incl && keys && vals, "atlas_corner_keys", "null pointer");
    k_at_corner_keys<<<grid_of(3 * (size_t)F), 256, 0, as_stream(stream)>>>(tri, F, label, incl, keys, vals);
    return check_launch("atlas_corner_keys");
}

int n2m_atlas_row_flags(const uint64_t* keys, uint32_t n, int32_t* flag, n2m_stream_t stream) {
    if (n == 0) return 0;
    N2M_REQUIRE(keys && flag, "atlas_row_flags", "null pointer");
    k_at_row_flags<<<grid_of(n), 256, 0, as_stream(stream)>>>(keys, n, flag);
    return check_launch("atlas_row_flags");
}

int n2m_atlas_emit(const float* vertices, const uint64_t* keys, const int32_t* vals, uint32_t n, const int32_t* rows, const int32_t* fax,
                   const double* basis, const double* rot, const int32_t* orient, const double* org, const int32_t* off, const double* state,
                   int32_t res, float* vt, int32_t* ft, int32_t* vmapping, n2m_stream_t stream) {
    if (n == 0) return 0;
    N2M_REQUIRE(vertices && keys && vals && rows && fax && basis && rot && orient && org && off && state && vt && ft && vmapping, "atlas_emit",
                "null pointer");
    const ChartArgs a{nullptr, nullptr, fax, orient, off, basis, rot, org, state};
    k_at_emit<<<grid_of(n), 256, 0, as_stream(stream)>>>(vertices, keys, vals, n, rows, a, res, vt, ft, vmapping);
    return check_launch("atlas_emit");
}

}  // extern "C"
