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

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_MESH_H */
