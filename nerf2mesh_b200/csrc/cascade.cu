// cascade.cu -- the outer-cascade meshes of an unbounded scene (NeRFRenderer.export_stage0, non-SDF branch for cas = 1 .. C-1,
// nerf/renderer.py:606-672) on the device, up to the reference's CPU clean-up / decimation, and the visibility test that follows them
// (mark_unseen_triangles, renderer.py:947-981).  C ABI include/n2m_b200_mesh.h, host side nerf2mesh_b200/mesh.py:
//
//   k_outer_occupancy   density_grid[cas] (Morton order, straight from the trainer) -> trilinear up-sampling to [R,R,R] with torch's
//                       upsample_trilinear3d arithmetic (align_corners=False) -> nan_to_num(., 0) > thresh as a float 0/1 volume
//   (marching cubes at iso 0.5: mcubes.cu, unchanged)
//   k_outer_select      index coordinates -> p = idx / (R - 1) * 2 - 1 -> p * (bound - half), in float64 (PyMCubes returns float64 and the
//                       reference's numpy chain stays float64) rounded once to float32; flags the centre-box and out-of-AABB vertices of
//                       both remove_selected_verts calls in one pass
//   k_rsv_count / k_rsv_emit   remove_selected_verts (meshutils.py:122-144, pymeshlab): flagged vertices and every face touching one go,
//                       unflagged vertices stay even when unreferenced, survivors keep their order, faces are re-indexed -- two kernels
//                       around the exclusive prefix sums of the keep flags, as n2m_mc_count / n2m_mc_emit
//   k_mark_seen_faces   the faces a rasterised view covers (the `mask[trig_id] += 1` of renderer.py:970-973 as a 0/1 flag)
// HBM-bound streaming work; no tensor cores.
#include "n2m_common.cuh"
#include "../../include/n2m_b200_mesh.h"

namespace n2m {
namespace {

// one thread per output cell (x, y, z), x-major, z fastest; the input cell (i, j, k) is grid[morton3(i, j, k)].
// The source index, weights and the nested sum are those of torch's CUDA upsample_trilinear3d (accscalar_t = float): a NaN tap makes the
// sum NaN even where its weight is 0, and nan_to_num then gives 0.  With R == H torch copies the input (its "just copy" special case), so
// only the cell itself is read.
__global__ void __launch_bounds__(256)
k_outer_occupancy(const float* __restrict__ grid, uint32_t H, uint32_t R, float thresh, float* __restrict__ out) {
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n = (size_t)R * R * R;
    if (p >= n) return;
    const uint32_t z = (uint32_t)(p % R), y = (uint32_t)((p / R) % R), x = (uint32_t)(p / ((size_t)R * R));
    float v;
    if (R == H) {
        v = __ldg(grid + morton3(x, y, z));
    } else {
        const float scale = (float)H / (float)R;
        const uint32_t dst[3] = {x, y, z};
        uint32_t i0[3], i1[3];
        float l0[3], l1[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float src = fmaxf(scale * ((float)dst[a] + 0.5f) - 0.5f, 0.f);
            i0[a] = (uint32_t)src;
            i1[a] = i0[a] + (i0[a] < H - 1 ? 1u : 0u);
            l1[a] = src - (float)i0[a];
            l0[a] = 1.f - l1[a];
        }
        const float v000 = __ldg(grid + morton3(i0[0], i0[1], i0[2])), v001 = __ldg(grid + morton3(i0[0], i0[1], i1[2]));
        const float v010 = __ldg(grid + morton3(i0[0], i1[1], i0[2])), v011 = __ldg(grid + morton3(i0[0], i1[1], i1[2]));
        const float v100 = __ldg(grid + morton3(i1[0], i0[1], i0[2])), v101 = __ldg(grid + morton3(i1[0], i0[1], i1[2]));
        const float v110 = __ldg(grid + morton3(i1[0], i1[1], i0[2])), v111 = __ldg(grid + morton3(i1[0], i1[1], i1[2]));
        v = l0[0] * (l0[1] * (l0[2] * v000 + l1[2] * v001) + l1[1] * (l0[2] * v010 + l1[2] * v011)) +
            l1[0] * (l0[1] * (l0[2] * v100 + l1[2] * v101) + l1[1] * (l0[2] * v110 + l1[2] * v111));
    }
    if (isnan(v)) v = 0.f;                                            // torch.nan_to_num(occ, 0)
    out[p] = v > thresh ? 1.f : 0.f;
}

// float64 throughout with explicit rounding (no contraction into FMAs): numpy evaluates each operation on its own
__global__ void __launch_bounds__(256)
k_outer_select(const float* __restrict__ idx, uint32_t V, uint32_t R, double scale, double xmn, double ymn, double zmn, double xmx,
               double ymx, double zmx, float* __restrict__ out, uint8_t* __restrict__ removed) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    const double rm1 = (double)R - 1.0;
    double p[3], s[3];
    bool centre = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        p[a] = __dadd_rn(__dmul_rn(__ddiv_rn((double)idx[3 * (size_t)i + a], rm1), 2.0), -1.0);       // renderer.py:631
        centre = centre && p[a] <= 0.45 && p[a] >= -0.45;                                             // :634-635
        s[a] = __dmul_rn(p[a], scale);                                                                // :638
        out[3 * (size_t)i + a] = (float)s[a];
    }
    const bool outside = s[0] <= xmn || s[0] >= xmx || s[1] <= ymn || s[1] >= ymx || s[2] <= zmn || s[2] >= zmx;     // :641-649
    removed[i] = (centre || outside) ? 1 : 0;
}

// one thread per vertex AND per face (max(V, F) threads): vkeep = !removed, fkeep = no corner removed
__global__ void __launch_bounds__(256)
k_rsv_count(const uint8_t* __restrict__ removed, uint32_t V, const int32_t* __restrict__ tri, uint32_t F, uint8_t* __restrict__ vkeep,
            uint8_t* __restrict__ fkeep) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < V) vkeep[i] = removed[i] ? 0 : 1;
    if (i < F) fkeep[i] = (removed[tri[3 * (size_t)i]] | removed[tri[3 * (size_t)i + 1]] | removed[tri[3 * (size_t)i + 2]]) ? 0 : 1;
}

// voff / foff: EXCLUSIVE prefix sums of vkeep / fkeep; a kept vertex i lands at voff[i], so a kept face's corners re-index through voff
__global__ void __launch_bounds__(256)
k_rsv_emit(const float* __restrict__ verts, uint32_t V, const int32_t* __restrict__ tri, uint32_t F, const uint8_t* __restrict__ vkeep,
           const uint8_t* __restrict__ fkeep, const int32_t* __restrict__ voff, const int32_t* __restrict__ foff, float* __restrict__ out_v,
           int32_t* __restrict__ out_f) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < V && vkeep[i]) {
        const size_t k = (size_t)voff[i];
#pragma unroll
        for (int a = 0; a < 3; ++a) out_v[3 * k + a] = verts[3 * (size_t)i + a];
    }
    if (i < F && fkeep[i]) {
        const size_t k = (size_t)foff[i];
#pragma unroll
        for (int a = 0; a < 3; ++a) out_f[3 * k + a] = voff[tri[3 * (size_t)i + a]];
    }
}

// trig_id = (long)rast.w - 1 indexes the face mask: an uncovered pixel (rast.w = 0) gives -1, which python indexing wraps to the LAST face
__global__ void __launch_bounds__(256)
k_mark_seen_faces(const float4* __restrict__ rast, uint32_t num_pixels, uint32_t F, uint8_t* __restrict__ seen) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_pixels) return;
    const int64_t id = (int64_t)__ldg(&rast[i].w) - 1;
    const int64_t f = id < 0 ? id + (int64_t)F : id;
    if (f >= 0 && f < (int64_t)F) seen[f] = 1;
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" {

int n2m_outer_occupancy(const float* density_grid, uint32_t H, uint32_t R, float thresh, float* volume, n2m_stream_t stream) {
    N2M_REQUIRE(density_grid && volume, "outer_occupancy", "null pointer");
    N2M_REQUIRE(H >= 1 && H <= 2048 && R >= 2 && R <= 1024, "outer_occupancy", "grid size 1..2048, volume resolution 2..1024");
    const size_t n = (size_t)R * R * R;
    k_outer_occupancy<<<(uint32_t)div_up(n, (size_t)256), 256, 0, as_stream(stream)>>>(density_grid, H, R, thresh, volume);
    return check_launch("outer_occupancy");
}

int n2m_outer_select(const float* vertices, uint32_t V, uint32_t R, double scale, double xmn, double ymn, double zmn, double xmx,
                     double ymx, double zmx, float* out, uint8_t* removed, n2m_stream_t stream) {
    N2M_REQUIRE(R >= 2, "outer_select", "volume resolution >= 2");
    if (V == 0) return 0;
    N2M_REQUIRE(vertices && out && removed, "outer_select", "null pointer");
    k_outer_select<<<div_up(V, 256u), 256, 0, as_stream(stream)>>>(vertices, V, R, scale, xmn, ymn, zmn, xmx, ymx, zmx, out, removed);
    return check_launch("outer_select");
}

int n2m_rsv_count(const uint8_t* removed, uint32_t V, const int32_t* tri, uint32_t F, uint8_t* vkeep, uint8_t* fkeep, n2m_stream_t stream) {
    const uint32_t n = V > F ? V : F;
    if (n == 0) return 0;
    N2M_REQUIRE(removed && vkeep && (F == 0 || (tri && fkeep)), "rsv_count", "null pointer");
    k_rsv_count<<<div_up(n, 256u), 256, 0, as_stream(stream)>>>(removed, V, tri, F, vkeep, fkeep);
    return check_launch("rsv_count");
}

int n2m_rsv_emit(const float* vertices, uint32_t V, const int32_t* tri, uint32_t F, const uint8_t* vkeep, const uint8_t* fkeep,
                 const int32_t* voff, const int32_t* foff, float* out_v, int32_t* out_f, n2m_stream_t stream) {
    const uint32_t n = V > F ? V : F;
    if (n == 0) return 0;
    N2M_REQUIRE(vertices && vkeep && voff && (F == 0 || (tri && fkeep && foff)), "rsv_emit", "null pointer");
    k_rsv_emit<<<div_up(n, 256u), 256, 0, as_stream(stream)>>>(vertices, V, tri, F, vkeep, fkeep, voff, foff, out_v, out_f);
    return check_launch("rsv_emit");
}

int n2m_mark_seen_faces(const float* rast, uint32_t num_pixels, uint32_t F, uint8_t* seen, n2m_stream_t stream) {
    N2M_REQUIRE(rast && seen, "mark_seen_faces", "null pointer");
    if (num_pixels == 0 || F == 0) return 0;
    k_mark_seen_faces<<<div_up(num_pixels, 256u), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(rast), num_pixels, F, seen);
    return check_launch("mark_seen_faces");
}

}  // extern "C"
