"""CPU: the decimation rule (nerf2mesh_b200/mesh.py decimate_mesh) through its numpy restatement (tests/decimate_oracle.py) on hand-built
meshes with their results written out and on analytic marching-cubes meshes, against the sequential greedy yardstick -- and the C ABI of
csrc/decimate.cu: every n2m_decim_* entry is exported, bound and documented, and no kernel spills."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import decimate_oracle as D
from nerf2mesh_b200 import build as B
from oracle import mcubes_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "n2m_b200_mesh.h")


def grid(n):
    """(n+1)^2 vertices on z = 0, row-major; quad (x, y) splits into (p, p+1, p+n+2) and (p, p+n+2, p+n+1), p = y (n+1) + x"""
    v = np.array([(x, y, 0) for y in range(n + 1) for x in range(n + 1)], np.float32)
    f = []
    for y in range(n):
        for x in range(n):
            p = y * (n + 1) + x
            f += [(p, p + 1, p + n + 2), (p, p + n + 2, p + n + 1)]
    return v, np.array(f)


def tetrahedron():
    return np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32), np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])


def octahedron():
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    return v, np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])


def strip(n):
    """n quads along x: a_k = (k, 0) (index k), b_k = (k, 1) (index n + 1 + k); faces (a_k, a_k+1, b_k+1), (a_k, b_k+1, b_k)"""
    v = np.array([(k, 0, 0) for k in range(n + 1)] + [(k, 1, 0) for k in range(n + 1)], np.float32)
    return v, np.array([t for k in range(n) for t in ((k, k + 1, n + 2 + k), (k, n + 2 + k, n + 1 + k))])


def three_on_edge():
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 2, 0], [0.5, 0, 0.5], [0.5, -1, 0]], np.float32)
    return v, np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]])


def fold(x):
    """edge (0, 1) with faces (0, 1, 2) and (0, 3, 1) and a third face (1, 2, 3) folded over them; 2 = (x, 1), 3 = (x, -1)"""
    v = np.array([[0, 0, 0], [1, 0, 0], [x, 1, 0], [x, -1, 0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 3, 1], [1, 2, 3]])


def two_triangles():
    return np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 0, 0], [6, 0, 0], [5, 1, 0]], np.float32), np.array([[0, 1, 2], [3, 4, 5]])


HAND = {"two_triangles": two_triangles(), "grid": grid(3), "tetrahedron": tetrahedron(), "octahedron": octahedron(), "strip": strip(10), "three_on_edge": three_on_edge(),
        "fold": fold(0.7), "fold_open": fold(-0.2)}


def _round1(v, f, target, optimal=True):
    trace, info = [], {}
    out = D.decimate(v, f, target, optimal, info, trace)
    return trace[0], info, out


def _valid_edges(t):
    m = t["key"] != D.NONE
    o = np.argsort(t["key"][m])
    return [(int(a), int(b)) for a, b in zip(t["lo"][m][o], t["hi"][m][o])], t["key"][m][o]


# ---- hand-built meshes ----------------------------------------------------------------------------------------------------------------
def test_flat_grid_keys_follow_edge_ids_and_round_one_takes_the_least():
    v, f = grid(3)                                    # 18 faces; every quadric is the plane z = 0, so every cost is exactly 0
    t, info, (vo, fo) = _round1(v, f, 10)
    edges, keys = _valid_edges(t)
    assert set((keys >> np.uint64(32)).tolist()) == {0x80000000}          # fkey(+0.0)
    assert (keys & np.uint64(0xFFFFFFFF)).tolist() == [0, 1, 2, 4, 5, 6, 7, 8, 10, 12, 13, 16, 19, 20, 22, 23, 25, 26, 28, 31, 32, 34, 37,
                                                        40, 41, 43, 44, 46, 49, 50, 52]
    # interior edges between two boundary vertices are not valid: (1, 4), (2, 5), ... are missing
    assert edges[:6] == [(0, 1), (1, 5), (0, 5), (4, 5), (0, 4), (1, 2)]
    # need = 8: weights 1, 2, 2, 2, 1 reach it at edge id 5; every eligible edge touches (0, 1)'s neighbourhood, so only edge 0 is selected
    assert int(t["K"]) == (0x80000000 << 32) | 5 and t["selected"].tolist() == [0]
    assert info == {"rounds": 6, "stalled": False, "faces": [17, 15, 14, 13, 11, 10]}
    assert len(fo) == 10 and np.all(vo[:, 2] == 0)


def test_tetrahedron_stalls():
    v, f = tetrahedron()
    info = {}
    vo, fo = D.decimate(v, f, 2, True, info)
    assert info == {"rounds": 0, "stalled": True, "faces": []}
    assert np.array_equal(vo, v) and np.array_equal(fo, f)


def test_lone_triangles_stay():
    # each edge is a boundary edge whose face has its other two edges on the boundary: collapsing it would delete a component
    v, f = two_triangles()
    info = {}
    vo, fo = D.decimate(v, f, 1, True, info)
    assert info == {"rounds": 0, "stalled": True, "faces": []}
    assert np.array_equal(vo, v) and np.array_equal(fo, f)


@pytest.mark.parametrize("optimal", [True, False])
def test_octahedron_stops_at_the_tetrahedron(optimal):
    v, f = octahedron()
    info = {}
    vo, fo = D.decimate(v, f, 1, optimal, info)
    assert info == {"rounds": 2, "stalled": True, "faces": [6, 4]}
    assert np.array_equal(fo, [[2, 0, 1], [1, 0, 3], [2, 1, 3], [0, 2, 3]])
    assert np.array_equal(np.abs(vo), [[0.5, 0.5, 0], [0.5, 0, 0.5], [0, 1, 0], [0, 0, 1]])
    # a target of 4 stops there without stalling
    info = {}
    D.decimate(v, f, 4, optimal, info)
    assert info == {"rounds": 2, "stalled": False, "faces": [6, 4]}


def test_open_strip_collapses_boundary_edges_only():
    v, f = strip(10)                                   # every vertex is a boundary vertex: the rungs and diagonals inside may not collapse
    t, info, (vo, fo) = _round1(v, f, 12)
    edges, _ = _valid_edges(t)
    rails = {(k, k + 1) for k in range(10)} | {(11 + k, 12 + k) for k in range(10)}
    assert set(edges) == rails | {(0, 11), (10, 21)}   # the two rails and the two end rungs: the boundary edges
    # zero costs: keys in edge-id order, need = 8 reaches K* at the 8th; every other eligible edge is within one ring of (0, 1)'s ends
    assert t["selected"].tolist() == [0]
    assert info == {"rounds": 8, "stalled": False, "faces": [19, 18, 17, 16, 15, 14, 13, 12]} and len(fo) == 12


def test_edge_of_three_faces_is_left_alone():
    v, f = three_on_edge()
    t, info, (vo, fo) = _round1(v, f, 2)
    edges, _ = _valid_edges(t)
    assert (0, 1) not in edges and len(edges) == 6
    assert len(fo) == 2 and not info["stalled"]
    e = np.sort(np.stack([fo, np.roll(fo, -1, 1)], 2).reshape(-1, 2), 1)
    assert (e == [0, 1]).all(1).sum() == 2             # the crowded edge is still there, with the two faces left


@pytest.mark.parametrize("optimal", [True, False])
def test_fold_is_rejected_by_the_flip_test(optimal):
    # (0, 1) has two faces, its link is {2, 3}, 1 is interior, no (0, 2, 3) face: only the flip test can refuse it.  Every quadric is
    # the plane z = 0, so both placements put 1 at 0 (the cheapest, on a tie the lower end) or at the midpoint (0.5, 0): with 2, 3 at
    # x = 0.7 the face (1, 2, 3) turns over, with them at x = -0.2 it does not
    t, _, _ = _round1(*fold(0.7), 2, optimal)
    assert _valid_edges(t)[0] == [(1, 2), (1, 3)]
    t, _, _ = _round1(*fold(-0.2), 2, optimal)
    assert _valid_edges(t)[0] == [(0, 1), (1, 2), (1, 3)]


def test_target_below_one_and_small_inputs():
    v, f = grid(2)
    with pytest.raises(ValueError):
        D.decimate(v, f, 0)
    v2 = np.concatenate([v, [[9, 9, 9]]]).astype(np.float32)
    info = {}
    vo, fo = D.decimate(v2, f, 8, True, info)           # F <= target: only the unreferenced vertex goes
    assert np.array_equal(vo, v) and np.array_equal(fo, f) and info["rounds"] == 0


# ---- analytic marching-cubes meshes ---------------------------------------------------------------------------------------------------
def sphere_volume(N, r=0.7):
    ax = np.linspace(-1, 1, N)
    x, y, z = np.meshgrid(ax, ax, ax, indexing="ij")
    return r - np.sqrt(x * x + y * y + z * z), lambda p: np.abs(np.linalg.norm(p, axis=1) - r)


def torus_volume(N, R=0.6, r=0.25):
    ax = np.linspace(-1, 1, N)
    x, y, z = np.meshgrid(ax, ax, ax, indexing="ij")
    d = lambda x, y, z: r - np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z)
    return d(x, y, z), lambda p: np.abs(d(p[:, 0], p[:, 1], p[:, 2]))


def mc(vol):
    N = vol.shape[0]
    v, f = MO.marching_cubes(vol, 0.0)
    return (v / (N - 1) * 2 - 1).astype(np.float32), f


def check_mesh(v, f, euler):
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all()
    assert len(np.unique(np.sort(f, 1), axis=0)) == len(f)
    e = np.sort(np.stack([f, np.roll(f, -1, 1)], 2).reshape(-1, 2), 1)
    ue, cnt = np.unique(e, axis=0, return_counts=True)
    assert cnt.max() <= 2
    assert np.array_equal(np.unique(f), np.arange(len(v)))
    assert len(v) - len(ue) + len(f) == euler


def surface_error(v, f, dist):
    """mean distance to the analytic surface over the vertices and the face centroids"""
    p = v.astype(np.float64)
    return float(np.concatenate([dist(p), dist(p[f].mean(1))]).mean())


# the parallel rule's surface error over the greedy yardstick's on these meshes (64^3, 10%), as measured: sphere 0.948 with optimal
# placement and 0.997 with the midpoint, torus 0.985 and 0.998.  The bound is that with a small margin.
ERROR_FACTOR = 1.02


def _decimated(shape, optimal):
    vol, dist = sphere_volume(64) if shape == "sphere" else torus_volume(64)
    v, f = mc(vol)
    target = len(f) // 10
    info = {}
    return v, f, target, dist, info, D.decimate(v, f, target, optimal, info)


@pytest.mark.parametrize("shape,euler", [("sphere", 2), ("torus", 0)])
@pytest.mark.parametrize("optimal", [True, False])
def test_marching_cubes_meshes_keep_their_topology(shape, euler, optimal):
    v, f, target, _, info, (vo, fo) = _decimated(shape, optimal)
    assert 15000 < len(f) < 30000
    check_mesh(v, f, euler)
    assert len(fo) in (target, target - 1) and not info["stalled"] and info["faces"][-1] == len(fo)
    check_mesh(vo, fo, euler)
    if shape == "sphere":
        p = vo.astype(np.float64)
        n = np.cross(p[fo[:, 1]] - p[fo[:, 0]], p[fo[:, 2]] - p[fo[:, 0]])
        assert (np.einsum("ij,ij->i", n, p[fo].mean(1)) > 0).all()


@pytest.mark.parametrize("shape,optimal,euler", [("sphere", True, 2), ("torus", False, 0)])
def test_marching_cubes_surface_error_is_the_greedy_ones(shape, optimal, euler):
    v, f, target, dist, _, (vo, fo) = _decimated(shape, optimal)
    vg, fg = D.decimate_greedy(v, f, target, optimal)
    assert len(fg) in (target, target - 1)
    check_mesh(vg, fg, euler)
    assert surface_error(vo, fo, dist) <= ERROR_FACTOR * surface_error(vg, fg, dist)


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
def test_decim_entries_are_exported_bound_and_documented():
    from nerf2mesh_b200 import _lib, mesh  # noqa: F401  (registers the mesh signatures)
    code = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(n2m_decim_[a-z0-9_]+)\s*\(", code)))
    assert len(syms) == 8, syms
    header = open(HEADER).read()
    for s in syms:
        assert hasattr(_lib.lib, s), f"libn2m_b200.so does not export {s}"
        assert s in _lib.SIGNATURES, f"{s} is not bound in mesh.py"
        assert f"*   {s} " in header or f"*   {s}:" in header, f"{s} has no comment entry in the header"


def test_decimate_mesh_needs_cuda_tensors():
    from nerf2mesh_b200 import mesh as M
    v, f = grid(2)
    with pytest.raises(RuntimeError, match="CUDA"):
        M.decimate_mesh(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), 4)


def test_decimate_kernels_have_no_spills(tmp_path):
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "decimate.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    found = []
    for i, l in enumerate(lines):
        if "Function properties for" in l and "decimate" in l:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            assert m and (int(m.group(2)), int(m.group(3))) == (0, 0), l + "\n" + lines[i + 1]
            found.append(l)
    assert len(found) == 13, found
