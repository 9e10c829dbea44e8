/* n2m_b200_mesh.h -- C ABI of the stage-0 -> stage-1 mesh hand-off of libn2m_b200.so.
 *
 * NeRFRenderer.export_stage0 (nerf/renderer.py:471-545) evaluates the density on a regular grid, copies it to the host and calls the
 * third-party PyMCubes `mcubes.marching_cubes(sigmas, density_thresh)` (:526-529; not vendored, version unpinned) before cleaning /
 * decimating the mesh with CPU mesh libraries.  These entry points replace the marching-cubes call on the device; the volume comes from
 * Stage0Trainer.density_volume (the reference's own arithmetic up to that call, tests/test_gpu_reference_parity.py); the cleaning and
 * the decimation that follow run on the device too (below).  Python binding: nerf2mesh_b200/mesh.py (`marching_cubes(volume, isovalue)` returns
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
 *
 * Mesh clean-up (remove_masked_trigs and clean_mesh(..., remesh=False) of meshutils.py:63-93,146-188, pymeshlab in the reference;
 * csrc/meshclean.cu; Python: mesh.remove_masked_faces, mesh.clean_mesh).  The steps never move the mesh: faces are dropped through
 * fkeep [F] u8, merged and split vertices are re-indexed in place in tri [F,3] i32, and the caller compacts once with n2m_rsv_emit.  Power-
 * of-two tables and sort buffers are the caller's; each entry initialises what it documents.
 *   n2m_clean_mark_verts    : vflag[v] = 1 for every corner of a face with fkeep set (fkeep NULL: every face); caller zeroes vflag [V] u8
 *   n2m_clean_dilate        : one selection dilation: vsel [V] u8 |= the corners of kept faces, then fkeep[f] = 1 where a corner is selected
 *   n2m_clean_bbox          : bbox [6] u32 = order-preserving keys of the min / max xyz over the vertices with vflag set (initialised here)
 *   n2m_clean_merge_bin     : close-vertex merge, radius r = v_pct / 100 * diag / 10 (float64, diag of bbox): vbucket [V] i32 = the
 *                             bucket of the vertex's cell of size r in a table of nbuckets, bucket_count [nbuckets] i32 += 1 (caller zeroes)
 *   n2m_clean_merge_fill    : cursor = EXCLUSIVE prefix sum of bucket_count (advanced here) -> items [V] i32 grouped by bucket
 *   n2m_clean_merge_round   : one decision round (round = 1, 2, ...) over the flagged, undecided vertices; decided [V] i32 zeroed by the
 *                             caller before round 1, target [V] i32 = the vertex's leader once decided; pending [1] i32 = 1 (caller
 *                             zeroes) while a vertex is still undecided.  bucket_start [nbuckets+1] i32: inclusive prefix after a 0.
 *                             Leader rule: i leads unless a leader j < i lies within r, dx*dx + dy*dy + dz*dz <= r*r in float64
 *   n2m_clean_merge_apply   : tri <- target[tri] for kept faces; a face repeating an index is dropped
 *   n2m_clean_dup_null      : drop the kept faces whose unordered vertex triple a lower kept face has, and those whose float64
 *                             cross(b - a, c - a) is the zero vector; table [nslots >= 2F] i32 and slot_of [F] i32 are scratch
 *   n2m_clean_edge_table    : table [nslots >= 6F] i32 of the kept faces' unordered edges (slot value = lowest face-edge 3f+k with the
 *                             edge), slot_of [3F] i32 = the slot of face-edge 3f+k (edge from corner k to corner k+1)
 *   n2m_clean_components    : edge-connected components of the kept faces over that table; drop a component whose bbox diagonal is
 *                             < min_d / 100 * diag (diag of bbox; min_d > 0) or whose face count is < min_f (min_f > 0).  parent,
 *                             label, count [F] i32, cmin, cmax [3F] u32 are scratch
 *   n2m_clean_nm_edges      : the kept faces with an edge of > 2 kept faces, visited by (float64 area, face index); a face goes when one
 *                             of its edges still has > 2 kept faces.  ecount [nslots] i32, ncand [1] i32, keys [capacity] u64,
 *                             vals [capacity] i32 are scratch (capacity a power of two >= F)
 *   n2m_clean_nm_verts_find : fans of every vertex (kept faces joined through an edge at the vertex); nextra [1] i32 = the number of fans
 *                             that do not hold the vertex's lowest face, cnew [3F] i32 numbers them in (vertex, lowest face) order.
 *                             emin [nslots], cparent, clabel [3F], vmin [V] i32, keys / vals [capacity >= 3F] are scratch; clabel (each
 *                             corner's fan root) and vmin feed n2m_clean_nm_verts_apply
 *   n2m_clean_nm_verts_apply: the corners of those fans take vertex V + cnew, ext_vertices [V + nextra, 3] f32 rows V.. get the copies'
 *                             positions (the caller copies rows 0..V-1)
 *
 * Decimation (meshing_decimation_quadric_edge_collapse of meshutils.py decimate_mesh, pymeshlab in the reference; csrc/decimate.cu;
 * Python: mesh.decimate_mesh).  Rounds of independent edge collapses over fkeep / tri as above: each round rebuilds the edge table
 * (n2m_clean_edge_table) and the vertex -> live face lists, keys every valid collapse, selects, moves the survivors and re-indexes the
 * faces with n2m_clean_merge_apply; the caller reads flive once per round and compacts once with n2m_rsv_emit.  The lower vertex of a
 * collapsed edge survives.  Q [V,10] f64 holds a00 a01 a02 a11 a12 a22 b0 b1 b2 c of each vertex quadric.
 *   n2m_decim_init      : fkeep [F] u8 = the face repeats no index; flive [1] i32 = the number of such faces (initialised here)
 *   n2m_decim_vcount    : vcount [V] i32 += the live faces at each vertex (caller zeroes)
 *   n2m_decim_vfill     : cursor = EXCLUSIVE prefix sum of vcount (advanced here) -> vfaces [3 * live] i32, each vertex's live faces in
 *                         any order
 *   n2m_decim_quadrics  : Q [V,10] = the sum over the vertex's live faces, in ascending face index from +0, of the plane quadric of the
 *                         float64 unit normal u = cross(b - a, c - a) / |.| and d = -u.a (zero for |cross| = 0); sorts each list of vfaces
 *   n2m_decim_edges     : ecount [nslots] i32 = live face-edges per slot of n2m_clean_edge_table's slot_of; vbnd [V] u8 = the vertex is
 *                         on an edge of one live face (both initialised here)
 *   n2m_decim_eval      : keys [3F] u64, pos [3F,3] f32: for the lowest live face-edge e of an edge (a < b) whose collapse is valid,
 *                         pos[e] = the merged position and keys[e] = fkey(float(cost)) << 32 | e, else keys[e] = ~0.  Valid: 1 or 2
 *                         faces; every common neighbour of a and b is an opposite vertex; a boundary edge or not both ends boundary; a
 *                         boundary edge's face has not both other edges on the boundary; not (a,c,d) and (b,c,d) both live; no other
 *                         face at a or b gets float64 dot(n_old, n_new) <= 0.  Position (optimal
 *                         != 0): A p = -b of Q_a + Q_b by cofactors when det > 1e-6 trace^3, else the cheapest of a, b, the midpoint
 *                         (ties in that order); optimal == 0: the float64 midpoint; rounded once to f32, cost = the quadric there
 *   n2m_decim_threshold : state [4] u64, state[3] = K*: the least key at which the valid keys in order, weighted by their edge's face
 *                         count, reach flive - target (every valid key when they do not); hist [256] u64 and state[0..2] are scratch
 *   n2m_decim_select    : the valid edges with key <= K* equal to the least such key over the closed neighbourhoods of both ends:
 *                         target [V] i32 = b -> a (identity elsewhere), vertices[a] = pos, Q[a] += Q[b], flive -= the edge's faces;
 *                         vmin, r1 [V] u64 are scratch.  The caller then runs n2m_clean_merge_apply with target
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

int n2m_clean_mark_verts(const int32_t* tri, uint32_t F, const uint8_t* fkeep, uint8_t* vflag, n2m_stream_t stream);
int n2m_clean_dilate(const int32_t* tri, uint32_t F, uint8_t* fkeep, uint8_t* vsel, n2m_stream_t stream);
int n2m_clean_bbox(const float* vertices, uint32_t V, const uint8_t* vflag, uint32_t* bbox, n2m_stream_t stream);
int n2m_clean_merge_bin(const float* vertices, uint32_t V, const uint8_t* vflag, const uint32_t* bbox, double v_pct, uint32_t nbuckets,
                        int32_t* bucket_count, int32_t* vbucket, n2m_stream_t stream);
int n2m_clean_merge_fill(uint32_t V, const uint8_t* vflag, const int32_t* vbucket, int32_t* cursor, int32_t* items, n2m_stream_t stream);
int n2m_clean_merge_round(const float* vertices, uint32_t V, const uint8_t* vflag, const uint32_t* bbox, double v_pct, uint32_t nbuckets,
                          const int32_t* bucket_start, const int32_t* items, int32_t round, int32_t* decided, int32_t* target,
                          int32_t* pending, n2m_stream_t stream);
int n2m_clean_merge_apply(int32_t* tri, uint32_t F, const int32_t* target, uint8_t* fkeep, n2m_stream_t stream);
int n2m_clean_dup_null(const float* vertices, const int32_t* tri, uint32_t F, uint8_t* fkeep, uint32_t nslots, int32_t* table,
                       int32_t* slot_of, n2m_stream_t stream);
int n2m_clean_edge_table(const int32_t* tri, uint32_t F, const uint8_t* fkeep, uint32_t nslots, int32_t* table, int32_t* slot_of,
                         n2m_stream_t stream);
int n2m_clean_components(const float* vertices, const int32_t* tri, uint32_t F, uint8_t* fkeep, const int32_t* table, const int32_t* slot_of,
                         const uint32_t* bbox, double min_d, uint32_t min_f, int32_t* parent, int32_t* label, int32_t* count, uint32_t* cmin,
                         uint32_t* cmax, n2m_stream_t stream);
int n2m_clean_nm_edges(const float* vertices, const int32_t* tri, uint32_t F, uint8_t* fkeep, const int32_t* slot_of, uint32_t nslots,
                       int32_t* ecount, int32_t* ncand, uint64_t* keys, int32_t* vals, uint32_t capacity, n2m_stream_t stream);
int n2m_clean_nm_verts_find(const int32_t* tri, uint32_t V, uint32_t F, const uint8_t* fkeep, const int32_t* slot_of, uint32_t nslots,
                            int32_t* emin, int32_t* cparent, int32_t* clabel, int32_t* vmin, int32_t* nextra, uint64_t* keys, int32_t* vals,
                            int32_t* cnew, uint32_t capacity, n2m_stream_t stream);
int n2m_clean_nm_verts_apply(const float* vertices, uint32_t V, int32_t* tri, uint32_t F, const uint8_t* fkeep, const int32_t* clabel,
                             const int32_t* vmin, const int32_t* cnew, float* ext_vertices, n2m_stream_t stream);

int n2m_decim_init(const int32_t* tri, uint32_t F, uint8_t* fkeep, int32_t* flive, n2m_stream_t stream);
int n2m_decim_vcount(const int32_t* tri, uint32_t F, const uint8_t* fkeep, int32_t* vcount, n2m_stream_t stream);
int n2m_decim_vfill(const int32_t* tri, uint32_t F, const uint8_t* fkeep, int32_t* cursor, int32_t* vfaces, n2m_stream_t stream);
int n2m_decim_quadrics(const float* vertices, uint32_t V, const int32_t* tri, const int32_t* vstart, int32_t* vfaces, double* Q,
                       n2m_stream_t stream);
int n2m_decim_edges(const int32_t* tri, uint32_t V, uint32_t F, const uint8_t* fkeep, const int32_t* slot_of, uint32_t nslots, int32_t* ecount,
                    uint8_t* vbnd, n2m_stream_t stream);
int n2m_decim_eval(const float* vertices, const double* Q, const int32_t* tri, uint32_t F, const uint8_t* fkeep, const int32_t* table,
                   const int32_t* slot_of, const int32_t* ecount, const uint8_t* vbnd, const int32_t* vstart, const int32_t* vfaces, int optimal,
                   uint64_t* keys, float* pos, n2m_stream_t stream);
int n2m_decim_threshold(const uint64_t* keys, uint32_t F, const int32_t* slot_of, const int32_t* ecount, const int32_t* flive, uint32_t target,
                        uint64_t* hist, uint64_t* state, n2m_stream_t stream);
int n2m_decim_select(const uint64_t* keys, uint32_t V, uint32_t F, const int32_t* tri, const int32_t* slot_of, const int32_t* ecount,
                     const int32_t* vstart, const int32_t* vfaces, const uint64_t* state, const float* pos, uint64_t* vmin, uint64_t* r1,
                     float* vertices, double* Q, int32_t* target, int32_t* flive, n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_MESH_H */
