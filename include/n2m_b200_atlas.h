/* n2m_b200_atlas.h -- C ABI of the stage-1 UV atlas of libn2m_b200.so (csrc/atlas.cu; Python: texture.uv_unwrap).
 *
 * The reference unwraps the stage-1 mesh with xatlas on the CPU (renderer.py:313-321).  These entry points build the library's own atlas
 * on the device instead: normal-cone charts, one texel scale shared by every chart, next-fit-decreasing-height shelves on the final
 * texture's texel grid, and a texel-conflict check at the bake raster.  The rule is deterministic and its float64 steps are single
 * rounded operations, so tests/atlas_oracle.py restates it bit for bit.  The host drives the rounds and reads back the chart count, the
 * scale and fit flag, the conflict count and the row count only.
 *
 * Faces f (F of them), face-edges e = 3f + k (corner k to corner k+1), chart ids = the id face of the chart (label[f] == f), chart
 * indices 0 .. C-1 = the chart ids in ascending order (incl = the INCLUSIVE prefix sum of n2m_atlas_roots' flags, index = incl[id] - 1).
 * axes [26,3] f64: normalize(i, j, k) over {-1, 0, 1}^3 \ 0 in lexicographic order; basis [26,6] f64: per axis a right-handed (e1, e2)
 * with e1 x e2 = axis; rot [K,2] f64: (cos, sin) of the K angles.
 *
 *   n2m_atlas_contract    : out [V,3] f32 = contract(vertices) of renderer.py:25-32, the arithmetic of the stage-1 step and the bake (the
 *                           positions an unbounded scene's cascades are unwrapped at)
 *   n2m_atlas_faces       : nrm [F,3] f64 = the unit normal cross(b - a, c - a) / |.| (each operation rounded once), bucket [F] i32 = the
 *                           argmax of dot(nrm, axes[i]) (lowest i on a tie), fkeep [F] u8 = 1; a face that repeats an index or whose cross
 *                           product is zero gets bucket -1, fkeep 0, nrm 0
 *   n2m_atlas_base        : over n2m_clean_edge_table(tri, F, fkeep, ...)'s table / slot_of: ecount [nslots] = face-edges per slot, mate [3F]
 *                           = the other face-edge of a slot with exactly two (-1 elsewhere), parent [F] scratch; faces across a mate with the
 *                           same bucket join; base [F] = label [F] = the lowest face of the chart, fax [F] = max(bucket, 0)
 *   n2m_atlas_chart_count : count [F] i32 = the faces of each chart id (initialised here)
 *   n2m_atlas_merge_round : start = EXCLUSIVE prefix sum of count; cursor, items [F] i32 and propose [F] i32 are scratch.  A chart of fewer
 *                           than `small` (<= 32) non-degenerate faces proposes the chart id it shares the most mates with (ties: the lowest
 *                           id) when dot(nrm, axes[fax of that chart]) >= 0.5 for each of its faces; a proposal whose target does not
 *                           propose is accepted: label and fax of the small chart's faces take the target's
 *   n2m_atlas_roots       : flag [F] i32 = (label[f] == f)
 *   n2m_atlas_orient      : bmin / bmax [C,K,2] u64 (scratch): per chart and angle the box of (c u - s v, s u + c v), (u, v) = (p.e1, p.e2)
 *                           of the chart's axis; orient [C] i32 = k | turn << 16 with k the least-area angle (lowest k on a tie) and turn = 1
 *                           when that box is taller than wide ((x, y) -> (-y, x)); org [C,2] f64 = the turned box's minimum, ext [C,2] f64 =
 *                           its (width, height); skey [C] u64 / sval [C] i32 = sort pairs ordering by height desc, then chart index
 *   n2m_atlas_sort        : sorts (keys, vals) pairs lexicographically in place; buffers of cap (a power of two >= n) entries
 *   n2m_atlas_pack        : order [C] = the chart indices sorted as above.  Chart i of the order is w_i = max(1, ceil(s W)) x h_i =
 *                           max(1, ceil(s H)) final texels; shelves fill left to right from x = pad with pad texels between rectangles, a shelf
 *                           is as tall as its first chart and the next starts pad above it, everything pad texels inside res x res.  s is
 *                           the largest scale found by `steps` geometric bisection steps on [hi 2^-20, hi], hi = (res - 2 pad) / max W
 *                           (res when every W is 0).  state [2] f64 = (s, 1) and off [C,2] i32 = the rectangles' corners, or (.., 0) when
 *                           even hi 2^-20 does not fit.  wid, hgt, nxt, shelf_a, shelf_y [C] i32 and prefix [C+1] i64 are scratch
 *   n2m_atlas_conflicts   : at the bake raster R x R (texel (i, j) centred at (i + 0.5, j + 0.5) in units of vt * R): conf [C] u8 = 1 for the
 *                           charts with a non-degenerate face strictly inside which (float64 edge functions > 0) a texel centre lies that a
 *                           lower face also covers strictly; nconf [1] i32 = the number of such (face, texel) pairs.  owner [R*R] i32 scratch
 *   n2m_atlas_split       : the faces of a chart with conf set take base[f] when the chart is a merged one (a face with base != label),
 *                           else become charts of their own; fax = max(bucket, 0).  merged [C] u8 scratch
 *   n2m_atlas_corner_keys : keys [3F] u64 = chart index << 32 | vertex of each corner, vals [3F] = the corner
 *   n2m_atlas_row_flags   : flag [n] i32 = 1 where a sorted key differs from the one before
 *   n2m_atlas_emit        : rows = INCLUSIVE prefix sum of those flags: ft[corner] = row, and per distinct key vmapping[row] = vertex, vt[row]
 *                           = ((off + s (xy - org)) / res) rounded once to f32, xy the vertex's turned chart coordinates
 */
#ifndef N2M_B200_ATLAS_H
#define N2M_B200_ATLAS_H

#include "n2m_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int n2m_atlas_contract(const float* vertices, uint32_t V, float* out, n2m_stream_t stream);
int n2m_atlas_faces(const float* vertices, const int32_t* tri, uint32_t F, const double* axes, double* nrm, int32_t* bucket, uint8_t* fkeep,
                    n2m_stream_t stream);
int n2m_atlas_base(uint32_t F, const uint8_t* fkeep, const int32_t* bucket, const int32_t* table, const int32_t* slot_of, uint32_t nslots,
                   int32_t* ecount, int32_t* mate, int32_t* parent, int32_t* base, int32_t* label, int32_t* fax, n2m_stream_t stream);
int n2m_atlas_chart_count(uint32_t F, const int32_t* label, int32_t* count, n2m_stream_t stream);
int n2m_atlas_merge_round(uint32_t F, uint32_t small, const double* nrm, const double* axes, const int32_t* bucket, const int32_t* mate,
                          const int32_t* count, const int32_t* start, int32_t* cursor, int32_t* items, int32_t* propose, int32_t* label,
                          int32_t* fax, n2m_stream_t stream);
int n2m_atlas_roots(uint32_t F, const int32_t* label, int32_t* flag, n2m_stream_t stream);
int n2m_atlas_orient(const float* vertices, const int32_t* tri, uint32_t F, const int32_t* label, const int32_t* incl, const int32_t* fax,
                     const double* basis, const double* rot, uint32_t K, uint32_t C, uint64_t* bmin, uint64_t* bmax, int32_t* orient,
                     double* org, double* ext, uint64_t* skey, int32_t* sval, n2m_stream_t stream);
int n2m_atlas_sort(uint64_t* keys, int32_t* vals, uint32_t n, uint32_t cap, n2m_stream_t stream);
int n2m_atlas_pack(const double* ext, const int32_t* order, uint32_t C, int32_t res, int32_t pad, int32_t steps, int32_t* wid, int32_t* hgt,
                   int32_t* nxt, int32_t* shelf_a, int32_t* shelf_y, long long* prefix, int32_t* off, double* state, n2m_stream_t stream);
int n2m_atlas_conflicts(const float* vertices, const int32_t* tri, uint32_t F, const uint8_t* fkeep, const int32_t* label, const int32_t* incl,
                        const int32_t* fax, const double* basis, const double* rot, const int32_t* orient, const double* org, const int32_t* off,
                        const double* state, uint32_t C, int32_t res, uint32_t R, int32_t* owner, uint8_t* conf, int32_t* nconf,
                        n2m_stream_t stream);
int n2m_atlas_split(uint32_t F, uint32_t C, const int32_t* incl, const int32_t* base, const int32_t* bucket, const uint8_t* conf,
                    uint8_t* merged, int32_t* label, int32_t* fax, n2m_stream_t stream);
int n2m_atlas_corner_keys(const int32_t* tri, uint32_t F, const int32_t* label, const int32_t* incl, uint64_t* keys, int32_t* vals,
                          n2m_stream_t stream);
int n2m_atlas_row_flags(const uint64_t* keys, uint32_t n, int32_t* flag, n2m_stream_t stream);
int n2m_atlas_emit(const float* vertices, const uint64_t* keys, const int32_t* vals, uint32_t n, const int32_t* rows, const int32_t* fax,
                   const double* basis, const double* rot, const int32_t* orient, const double* org, const int32_t* off, const double* state,
                   int32_t res, float* vt, int32_t* ft, int32_t* vmapping, n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_ATLAS_H */
