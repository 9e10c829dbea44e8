/* n2m_b200_mesh.h -- C ABI of the stage-0 -> stage-1 mesh hand-off of libn2m_b200.so.
 *
 * NeRFRenderer.export_stage0 (nerf/renderer.py:471-545) evaluates the density on a regular grid, copies it to the host and calls the
 * third-party PyMCubes `mcubes.marching_cubes(sigmas, density_thresh)` (:526-529; not vendored, version unpinned) before cleaning /
 * decimating the mesh with CPU mesh libraries.  These entry points replace the marching-cubes call on the device; the volume comes from
 * Stage0Trainer.density_volume (the reference's own arithmetic up to that call, tests/test_gpu_reference_parity.py), the cleaning /
 * decimation stays the reference's CPU code.  Python binding: nerf2mesh_b200/mesh.py (`marching_cubes(volume, isovalue)` returns
 * vertices in index coordinates and int32 triangles like PyMCubes).
 *
 *   n2m_mc_count : volume [X,Y,Z] f32 (z fastest), per grid point: vcount = iso-crossings on its +x / +y / +z edges, tcount = triangles
 *                  of the cell it is the minimum corner of; num_tris [256] i32 (device) from nerf2mesh_b200/mc_table.py
 *   n2m_mc_emit  : with voff / toff = EXCLUSIVE prefix sums of vcount / tcount (i32): vertices [V,3] f32 (index coordinates, linear
 *                  interpolation), triangles [F,3] i32; tri_table [256,16] i8 (device).  "inside" = value > iso; triangle normals
 *                  point from inside to outside; shared vertices, deterministic order.
 *
 * Outer-cascade meshes of an unbounded scene (export_stage0's non-SDF branch for cas = 1 .. C-1, renderer.py:606-672; csrc/cascade.cu;
 * Python: mesh.export_outer_meshes):
 *   n2m_outer_occupancy : density_grid [H^3] f32 of one cascade in Morton order -> volume [R,R,R] f32 (x-major, z fastest) =
 *                         nan_to_num(F.interpolate(occ, [R]*3, mode='trilinear'), 0) > thresh as 0/1, with torch's CUDA upsample_trilinear3d
 *                         arithmetic (align_corners=False; a NaN tap gives NaN, hence 0, whatever its weight; R == H copies)
 *   n2m_outer_select    : vertices [V,3] f32 in index coordinates (marching cubes of that volume at 0.5) -> out [V,3] f32 =
 *                         (idx / (R-1) * 2 - 1) * scale computed in float64 and rounded once; removed [V] u8 = 1 where every normalised
 *                         |p| <= 0.45 (the centre box) or where the scaled point is outside the open box (xmn, xmx) x (ymn, ymx) x (zmn, zmx)
 *   n2m_rsv_count       : remove_selected_verts (meshutils.py:122-144): vkeep [V] u8 = !removed, fkeep [F] u8 = no corner removed
 *   n2m_rsv_emit        : with voff / foff = EXCLUSIVE prefix sums of vkeep / fkeep (i32): the kept vertices in order -> out_v, the kept
 *                         faces re-indexed -> out_f.  Unreferenced kept vertices stay.
 *   n2m_mark_seen_faces : rast [num_pixels,4] f32 of one view -> seen[(long)rast.w - 1] = 1 (caller zeroes seen [F] u8).  The index of an
 *                         uncovered pixel is -1, which the reference's torch indexing wraps to the last face: face F-1 counts as seen
 *                         whenever the view has an empty pixel (mark_unseen_triangles, renderer.py:947-981, kept as is).
 */
#ifndef N2M_B200_MESH_H
#define N2M_B200_MESH_H

#include "n2m_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int n2m_mc_count(const float* volume, uint32_t X, uint32_t Y, uint32_t Z, float iso, const int32_t* num_tris, uint8_t* vcount,
                 uint8_t* tcount, n2m_stream_t stream);
int n2m_mc_emit(const float* volume, uint32_t X, uint32_t Y, uint32_t Z, float iso, const int8_t* tri_table, const uint8_t* tcount,
                const int32_t* voff, const int32_t* toff, float* vertices, int32_t* triangles, n2m_stream_t stream);

int n2m_outer_occupancy(const float* density_grid, uint32_t H, uint32_t R, float thresh, float* volume, n2m_stream_t stream);
int n2m_outer_select(const float* vertices, uint32_t V, uint32_t R, double scale, double xmn, double ymn, double zmn, double xmx,
                     double ymx, double zmx, float* out, uint8_t* removed, n2m_stream_t stream);
int n2m_rsv_count(const uint8_t* removed, uint32_t V, const int32_t* tri, uint32_t F, uint8_t* vkeep, uint8_t* fkeep, n2m_stream_t stream);
int n2m_rsv_emit(const float* vertices, uint32_t V, const int32_t* tri, uint32_t F, const uint8_t* vkeep, const uint8_t* fkeep,
                 const int32_t* voff, const int32_t* foff, float* out_v, int32_t* out_f, n2m_stream_t stream);
int n2m_mark_seen_faces(const float* rast, uint32_t num_pixels, uint32_t F, uint8_t* seen, n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_MESH_H */
