"""CPU: the mesh clean-up's specification on hand-built meshes, each with its expected result written out, through the numpy oracle
(tests/meshclean_oracle.py) -- and the C ABI of csrc/meshclean.cu: the header compiles as C99, every entry is exported and bound, no kernel
spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import meshclean_oracle as O
from nerf2mesh_b200 import build as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "n2m_b200_mesh.h")
NO_CLEAN = dict(v_pct=0, min_f=0, min_d=0)


def strip(x0, y0, dx, dy, n, base=0):
    """n quads along x: a_k = (x0 + k dx, y0), b_k = (x0 + k dx, y0 + dy) (indices base + k, base + n + 1 + k), faces 2k = (a_k, a_k+1,
    b_k+1), 2k + 1 = (a_k, b_k+1, b_k)"""
    v = np.array([(x0 + k * dx, y0, 0) for k in range(n + 1)] + [(x0 + k * dx, y0 + dy, 0) for k in range(n + 1)], np.float32)
    a, b = (lambda k: base + k), (lambda k: base + n + 1 + k)
    f = [t for k in range(n) for t in ((a(k), a(k + 1), b(k + 1)), (a(k), b(k + 1), b(k)))]
    return v, np.array(f, np.int64)


def join(*meshes):
    vs, fs, base = [], [], 0
    for v, f in meshes:
        vs.append(v); fs.append(f + base); base += len(v)
    return np.concatenate(vs), np.concatenate(fs)


def bowtie():
    """two fans of two faces on vertex 0, sharing nothing else"""
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [-1, 0, 0.5], [-1, -1, 0.5], [0, -1, 0.5]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3], [0, 4, 5], [0, 5, 6]])


# ---- the oracle on hand-built meshes ------------------------------------------------------------------------------------------------
def test_bowtie_vertex_is_split():
    v, f = bowtie()
    stats = {}
    v2, f2 = O.clean_mesh(v, f, **NO_CLEAN, repair=True, stats=stats)
    assert np.array_equal(v2, np.concatenate([v, v[:1]]))                     # the copy of vertex 0 goes after every vertex
    assert np.array_equal(f2, [[0, 1, 2], [0, 2, 3], [7, 4, 5], [7, 5, 6]])  # the fan holding face 0 keeps vertex 0
    assert stats["split_copies"] == 1
    v3, f3 = O.clean_mesh(v, f, **NO_CLEAN, repair=False)
    assert np.array_equal(v3, v) and np.array_equal(f3, f)


def bowtie3():
    """a bow-tie with a third fan on vertex 0 (faces 4, 5), then a second bow-tie on vertex 10 (faces 6-9)"""
    v, f = bowtie()
    v = np.concatenate([v, np.array([[0, 0.2, -1], [0.3, 1, -1], [0.5, -0.5, -1]], np.float32)])
    f = np.concatenate([f, [[0, 7, 8], [0, 8, 9]]])
    w, g = bowtie()
    return np.concatenate([v, w + np.float32(5)]), np.concatenate([f, g + 10])


def test_two_bowties_number_copies_by_vertex_then_fan():
    # vertex 0 with three fans, vertex 10 with two; the copies come as (0, fan of face 2), (0, fan of face 4), (10, fan of face 8)
    v, f = bowtie3()
    v2, f2 = O.clean_mesh(v, f, **NO_CLEAN, repair=True)
    assert len(v2) == 20 and np.array_equal(v2[17:], v[[0, 0, 10]])
    assert np.array_equal(f2, [[0, 1, 2], [0, 2, 3], [17, 4, 5], [17, 5, 6], [18, 7, 8], [18, 8, 9],
                               [10, 11, 12], [10, 12, 13], [19, 14, 15], [19, 15, 16]])


def test_three_faces_on_one_edge_lose_the_smallest():
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 2, 0], [0.5, 0, 0.5], [0.5, -1, 0]], np.float32)
    f = np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]])                          # areas 1, 0.25, 0.5 on the edge (0, 1)
    stats = {}
    v2, f2 = O.clean_mesh(v, f, **NO_CLEAN, repair=True, stats=stats)
    assert np.array_equal(v2, v[[0, 1, 2, 4]])                               # vertex 3 went with face 1
    assert np.array_equal(f2, [[0, 1, 2], [0, 1, 3]])
    assert stats["nm_edge_faces"] == 1


def test_equal_areas_on_a_crowded_edge_go_by_index():
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0], [0.5, 0, 1], [0.5, 0, -1]], np.float32)
    f = np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [1, 0, 5]])                  # four faces of area 0.5 on one edge: 0 and 1 go
    v2, f2 = O.clean_mesh(v, f, **NO_CLEAN, repair=True)
    assert np.array_equal(v2, v[[0, 1, 4, 5]]) and np.array_equal(f2, [[0, 1, 2], [1, 0, 3]])


def test_duplicates_with_either_winding_keep_the_lowest():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], np.float32)
    f = np.array([[1, 3, 2], [2, 1, 0], [0, 1, 2], [1, 2, 0], [3, 1, 2]])
    stats = {}
    v2, f2 = O.clean_mesh(v, f, **NO_CLEAN, repair=True, stats=stats)
    assert np.array_equal(v2, v) and np.array_equal(f2, [[1, 3, 2], [2, 1, 0]])
    assert stats["duplicates"] == 3


def test_zero_area_face_goes():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.5, 0, 0], [2, 0, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 3, 1], [1, 4, 3]])                          # 0, 3, 1 and 1, 4, 3 lie on the x axis
    stats = {}
    v2, f2 = O.clean_mesh(v, f, **NO_CLEAN, repair=True, stats=stats)
    assert np.array_equal(v2, v[:3]) and np.array_equal(f2, [[0, 1, 2]])
    assert stats["null"] == 2


def test_row_at_nine_tenths_of_r_alternates_leaders():
    # top row t_0..t_5 at (3k, 5, 0) fixes the box: 15 x 5, diag sqrt(250); v_pct = 100 -> r = 0.1 diag = 1.58
    diag = np.sqrt(250.0)
    r = O.merge_radius(diag, 100)
    p = np.array([[0.9 * r * k, 0, 0] for k in range(5)], np.float32)
    t = np.array([[3 * k, 5, 0] for k in range(6)], np.float32)
    v = np.concatenate([p, t])
    f = np.array([[k, 5 + k, 6 + k] for k in range(5)])
    assert O.bbox_diag(v) == diag
    stats = {}
    v2, f2 = O.clean_mesh(v, f, v_pct=100, min_f=0, min_d=0, repair=False, stats=stats)
    # p1 -> p0, p2 leads (p0 is 1.8 r away and p1 is no leader), p3 -> p2, p4 leads: not transitive
    assert np.array_equal(v2, v[[0, 2, 4, 5, 6, 7, 8, 9, 10]])
    assert np.array_equal(f2, [[0, 3, 4], [0, 4, 5], [1, 5, 6], [1, 6, 7], [2, 7, 8]])
    assert stats["merged"] == 2


def test_merge_distance_is_inclusive():
    diag = np.sqrt(250.0)
    r = O.merge_radius(diag, 100)
    t = np.array([[3 * k, 5, 0] for k in range(6)], np.float32)
    for x, merged in ((np.float32(r), None), (np.nextafter(np.float32(r), np.float32(0)), True), (np.nextafter(np.float32(r), np.float32(9)), False)):
        v = np.concatenate([np.array([[0, 0, 0], [x, 0, 0]], np.float32), t])
        f = np.array([[0, 2, 3], [1, 4, 5], [0, 6, 7]])
        stats = {}
        O.clean_mesh(v, f, v_pct=100, min_f=0, min_d=0, repair=False, stats=stats)
        d = float(x)
        assert stats["merged"] == int(d * d <= r * r) and (merged is None or bool(stats["merged"]) == merged)


@pytest.mark.parametrize("dilation,kept", [(0, [10]), (1, [8, 10, 11, 12, 13]), (2, [6, 8, 9, 10, 11, 12, 13, 14, 15])])
def test_dilation_rings_on_a_strip(dilation, kept):
    v, f = strip(0, 0, 1, 1, 10)
    mask = np.ones(20, np.int64); mask[10] = 0
    v2, f2 = O.remove_masked_faces(v, f, mask, dilation)
    used = np.unique(f[kept])
    assert np.array_equal(v2, v[used])
    assert np.array_equal(f2, np.searchsorted(used, f[kept]))


def test_masked_faces_everything_or_nothing():
    v, f = strip(0, 0, 1, 1, 3)
    v2, f2 = O.remove_masked_faces(v, f, np.ones(6), 5)
    assert v2.shape == (0, 3) and f2.shape == (0, 3)
    v2, f2 = O.remove_masked_faces(np.concatenate([v, [[9, 9, 9]]]).astype(np.float32), f, np.zeros(6), 0)
    assert np.array_equal(v2, v) and np.array_equal(f2, f)                   # the unreferenced vertex goes


def test_component_diameter_threshold_is_strict():
    big = strip(0, 0, 6, 80, 10)                          # 60 x 80: diag 100, threshold 5 / 100 * 100 = 5
    at = strip(10, 10, 1.5, 4, 2)                         # 3 x 4: diag 5, kept
    below = strip(20, 0, 1.5, np.nextafter(np.float32(4), np.float32(0)), 2)
    v, f = join(big, at, below)
    assert O.bbox_diag(v) == 100.0 and O.min_component_diag(100.0, 5) == 5.0
    v2, f2 = O.clean_mesh(v, f, v_pct=0, min_f=0, min_d=5, repair=True)
    assert np.array_equal(v2, v[:28]) and np.array_equal(f2, f[:24])


def test_component_face_count_threshold_is_strict():
    big = strip(0, 0, 1, 1, 10)
    four = strip(20, 0, 1, 1, 2)
    three = strip(30, 0, 1, 1, 2)
    three = (three[0], three[1][:3])
    v, f = join(big, four, three)
    v2, f2 = O.clean_mesh(v, f, v_pct=0, min_f=4, min_d=0, repair=True)
    assert np.array_equal(v2, v[:28]) and np.array_equal(f2, f[:24])


def test_components_are_edge_connected():
    v, f = bowtie()                                      # 4 faces on one vertex, two edge-connected pairs
    v2, f2 = O.clean_mesh(v, f, v_pct=0, min_f=3, min_d=0, repair=False)
    assert v2.shape == (0, 3) and f2.shape == (0, 3)
    v2, f2 = O.clean_mesh(v, f, v_pct=0, min_f=2, min_d=0, repair=False)
    assert np.array_equal(v2, v) and np.array_equal(f2, f)


def test_empty_mesh():
    v2, f2 = O.clean_mesh(np.zeros((4, 3), np.float32), np.zeros((0, 3), np.int64))
    assert v2.shape == (0, 3) and f2.shape == (0, 3) and v2.dtype == np.float32 and f2.dtype == np.int32


# ---- the C ABI ----------------------------------------------------------------------------------------------------------------------
def _clean_symbols():
    code = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(n2m_clean_[a-z0-9_]+)\s*\(", code)))


def test_mesh_header_compiles_as_c99():
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", HEADER], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:500]


def test_clean_entries_are_exported_and_bound():
    from nerf2mesh_b200 import _lib, mesh  # noqa: F401  (registers the mesh signatures)
    syms = _clean_symbols()
    assert len(syms) == 13, syms
    header = open(HEADER).read()
    for s in syms:
        assert hasattr(_lib.lib, s), f"libn2m_b200.so does not export {s}"
        assert s in _lib.SIGNATURES, f"{s} is not bound in mesh.py"
        assert f"*   {s} " in header or f"*   {s}:" in header, f"{s} has no comment entry in the header"


def test_clean_functions_need_cuda_tensors():
    from nerf2mesh_b200 import mesh as M
    v, f = bowtie()
    with pytest.raises(RuntimeError, match="CUDA"):
        M.clean_mesh(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)))
    with pytest.raises(RuntimeError, match="CUDA"):
        M.remove_masked_faces(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), torch.zeros(4), 1)


def test_clean_kernels_have_no_spills(tmp_path):
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "meshclean.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    found = []
    for i, l in enumerate(lines):
        if "Function properties for" in l and "meshclean" in l:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            assert m and (int(m.group(2)), int(m.group(3))) == (0, 0), l + "\n" + lines[i + 1]
            found.append(l)
    assert len(found) >= 22, found
