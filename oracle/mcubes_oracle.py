"""oracle/mcubes_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT.  PARITY UNPINNED (see below).

CPU (numpy, float64, plain loops over the active cells) marching cubes with the conventions of csrc/mcubes.cu, the checker of those
kernels.  The reference calls the third-party PyMCubes (`mcubes.marching_cubes`, nerf/renderer.py:526-529), which is neither vendored
in the reference tree nor installed here, and pins no version: its output cannot be produced, and the classic 256-case table it ships
is not transcribed here -- the case table is GENERATED (nerf2mesh_b200/mc_table.py: crossing points traced around the cube's faces,
inside corners cut off separately on ambiguous faces).  What is shared with the library by construction: vertices lie on the grid edges
at the linear-interpolation crossing, in index coordinates, shared between cells.  What may differ: the triangulation inside a cell, the
resolution of ambiguous faces, the output order.  PARITY UNPINNED; tests/test_mcubes_oracle.py checks the properties any correct
marching cubes has (closed 2-manifold, Euler characteristic, outward orientation, area / volume of analytic shapes).
"""
import numpy as np

from nerf2mesh_b200 import mc_table as T


def marching_cubes(volume, iso):
    """volume [X,Y,Z], iso -> (vertices [V,3] float64 in index coordinates, triangles [F,3] int64); output order as csrc/mcubes.cu:
    vertices by (x-major point index, axis), triangles by (x-major cell index, table order)"""
    vol = np.asarray(volume, np.float64)
    X, Y, Z = vol.shape
    inside = vol > iso
    # crossings owned by each grid point
    cross = np.zeros((X, Y, Z, 3), bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    vid = np.full((X, Y, Z, 3), -1, np.int64)
    flat = cross.reshape(-1)
    vid.reshape(-1)[flat] = np.arange(flat.sum())
    pts = np.argwhere(cross)                                        # sorted by (x, y, z, axis): the kernel's order
    verts = pts[:, :3].astype(np.float64)
    for k, (x, y, z, a) in enumerate(pts):
        q = [x, y, z]; q[a] += 1
        f0, f1 = vol[x, y, z], vol[tuple(q)]
        verts[k, a] += (iso - f0) / (f1 - f0)
    case = np.zeros((X - 1, Y - 1, Z - 1), np.int64)
    for c in range(8):
        ox, oy, oz = T.corner_offset(c)
        case |= inside[ox:X - 1 + ox, oy:Y - 1 + oy, oz:Z - 1 + oz].astype(np.int64) << c
    tris = []
    for x, y, z in np.argwhere((case != 0) & (case != 255)):
        row = T.TRI_TABLE[case[x, y, z]]
        for t in range(T.NUM_TRIS[case[x, y, z]]):
            tri = []
            for e in row[3 * t:3 * t + 3]:
                axis, b1, b2 = int(e) >> 2, int(e) & 1, (int(e) >> 1) & 1
                o = [x, y, z]
                others = [a for a in range(3) if a != axis]
                o[others[0]] += b1; o[others[1]] += b2
                tri.append(vid[o[0], o[1], o[2], axis])
            tris.append(tri)
    return verts, np.array(tris, np.int64).reshape(-1, 3)


def mesh_properties(verts, tris):
    """edge-manifoldness, Euler characteristic, area, signed volume (positive when normals point outward)"""
    e = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    und = np.sort(e, axis=1)
    uniq, counts = np.unique(und, axis=0, return_counts=True)
    # orientation consistency: every directed edge appears once in each direction
    d = {}
    for a, b in e:
        d[(int(a), int(b))] = d.get((int(a), int(b)), 0) + 1
    consistent = all(v == 1 and d.get((b, a), 0) == 1 for (a, b), v in d.items())
    p0, p1, p2 = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    cr = np.cross(p1 - p0, p2 - p0)
    return dict(closed=bool((counts == 2).all()), consistent=bool(consistent),
                euler=int(len(np.unique(tris)) - len(uniq) + len(tris)),
                area=float(0.5 * np.linalg.norm(cr, axis=1).sum()), volume=float((p0 * cr).sum() / 6.0),
                degenerate=int((np.linalg.norm(cr, axis=1) == 0).sum()))
