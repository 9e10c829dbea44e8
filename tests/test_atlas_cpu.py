"""CPU: the UV atlas rule (nerf2mesh_b200/texture.py uv_unwrap) through its numpy restatement (tests/atlas_oracle.py) on hand-built meshes
with their results written out, and the atlas's properties on icospheres, marching-cubes spheres and tori and a decimated noisy mesh --
and the C ABI of csrc/atlas.cu: every n2m_atlas_* entry is exported, bound and documented, and no kernel spills."""
import os
import re
import subprocess

import numpy as np
import pytest

import atlas_oracle as A
import test_decimate_cpu as D
from nerf2mesh_b200 import build as B
from nerf2mesh_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "n2m_b200_atlas.h")
RES, SSAA = 512, 2


# ---- meshes ----------------------------------------------------------------------------------------------------------------------------
def cube():
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7],
                  [1, 7, 3]])
    return v, f


def three_on_edge():
    """edge (0, 1) with three faces, all facing +z: none of them may join another"""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0], [0.5, 2, 0.3]], np.float32)
    return v, np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]])


def with_degenerate():
    """grid(2) plus a face repeating an index and a zero-area face along the grid's first row"""
    v, f = D.grid(2)
    return v, np.concatenate([f, [[0, 0, 4], [0, 1, 2]]])


def spiral(turns=2.5, steps=60):
    """an annulus strip winding 2.5 times around z and rising slowly: every face faces +z, so it is one base chart, and its projection
    overlaps itself after one turn"""
    n = int(turns * steps)
    t = np.arange(n + 1) * (2 * np.pi / steps)
    rings = [np.stack([r * np.cos(t), r * np.sin(t), 0.01 * t], 1) for r in (1.0, 1.5)]
    v = np.concatenate(rings).astype(np.float32)
    f = [tri for k in range(n) for tri in ((k, n + 2 + k, k + 1), (k, n + 1 + k, n + 2 + k))]
    return v, np.array(f)


def noisy_decimated(N=64, seed=0):
    """a sphere with floater blobs and surface noise (seeded), marching cubes, decimated to 10 % by the decimation rule"""
    rng = np.random.default_rng(seed)
    ax = np.linspace(-1, 1, N)
    x, y, z = np.meshgrid(ax, ax, ax, indexing="ij")
    d = 0.6 - np.sqrt(x * x + y * y + z * z)
    for c, r in zip(rng.uniform(-0.9, 0.9, (8, 3)), rng.uniform(1, 3, 8) * 2 / N):
        d = np.maximum(d, r - np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2))
    h = 2.0 / (N - 1)
    d = np.where(np.abs(d) < 2 * h, d + rng.standard_normal(d.shape) * 0.5 * h, d)
    v, f = D.mc(d)
    return D.D.decimate(v, f, len(f) // 10)


HAND = {"cube": cube(), "grid": D.grid(6), "tetrahedron": D.tetrahedron(), "three_on_edge": three_on_edge(),
        "degenerate": with_degenerate(), "spiral": spiral()}


def property_meshes():
    return {"icosphere4": S.icosphere(4), "mc_sphere64": D.mc(D.sphere_volume(64)[0]), "mc_torus64": D.mc(D.torus_volume(64)[0]),
            "noisy_decimated": noisy_decimated()}


# ---- hand-built meshes ----------------------------------------------------------------------------------------------------------------
def _unwrap(name, res=RES):
    v, f = HAND[name]
    info = {}
    vt, ft, vm = A.unwrap(v, f, res, SSAA, info)
    assert np.array_equal(vm[ft], f)
    return v, f, vt, ft, vm, info


def test_cube_gives_six_charts_of_two_faces():
    v, f, vt, ft, vm, info = _unwrap("cube")
    assert info["charts"] == 6 and info["split_rounds"] == 0 and len(vt) == 24
    # the two faces of a side share their diagonal's two rows, and the sides share none
    for k in range(0, 12, 2):
        assert len(set(ft[k]) | set(ft[k + 1])) == 4
    assert sorted(np.unique(ft).tolist()) == list(range(24))


def test_flat_grid_is_one_chart():
    v, f, vt, ft, vm, info = _unwrap("grid")
    assert info["charts"] == 1 and len(vt) == len(v) and np.array_equal(np.sort(vm), np.arange(len(v)))
    # one uniform scale, no stretch: the chart is the grid, scaled
    assert abs(A.uv_area(vt, ft) * RES * RES / info["texels_per_unit"] ** 2 - 36) < 1e-3


def test_tetrahedron_gives_a_chart_per_face():
    v, f, vt, ft, vm, info = _unwrap("tetrahedron")
    assert info["charts"] == 4 and len(vt) == 12 and np.array_equal(np.sort(ft, 1).reshape(-1), np.arange(12))


def test_faces_do_not_join_across_a_non_manifold_edge():
    v, f, vt, ft, vm, info = _unwrap("three_on_edge")
    _, bucket = A.faces(v, f, A.tables()[0])
    assert (bucket == bucket[0]).all()                  # one axis, yet three charts: the edge has three faces
    assert info["charts"] == 3 and len(vt) == 9


def test_degenerate_faces_are_charts_of_their_own():
    v, f, vt, ft, vm, info = _unwrap("degenerate")
    assert info["charts"] == 3 and len(vt) == 9 + 2 + 3            # (0, 0, 4) has two distinct vertices
    assert ft[8, 0] == ft[8, 1] and len(set(ft[8]) | set(ft[9])) == 5 and not set(ft[8]) & set(ft[:8].reshape(-1))
    assert len(A.inside_pairs(vt[ft[8:10]], np.arange(2), RES * SSAA)[0]) == 0                  # no texel


def test_empty_mesh():
    info = {}
    vt, ft, vm = A.unwrap(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), RES, SSAA, info)
    assert vt.shape == (0, 2) and ft.shape == (0, 3) and vm.shape == (0,) and info["charts"] == 0


def test_self_overlapping_spiral_splits():
    trace = []
    v, f = spiral()
    info = {}
    vt, ft, vm = A.unwrap(v, f, RES, SSAA, info, trace)
    assert trace[0] == 1 and info["split_rounds"] >= 1 and info["charts"] == len(f)   # one base chart, not merged: into single faces
    check_properties(v, f, vt, ft, vm, info)


# ---- properties -----------------------------------------------------------------------------------------------------------------------
def _charts_of(ft, nt):
    """faces joined through shared vt rows: the atlas's charts as the output shows them"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    F = len(ft)
    g = coo_matrix((np.ones(3 * F), (np.repeat(np.arange(F), 3), F + ft.reshape(-1))), shape=(F + nt, F + nt))
    return connected_components(g, directed=False)[1][:F]


def check_properties(v, f, vt, ft, vm, info, res=RES, ssaa=SSAA):
    s = info["texels_per_unit"]
    assert np.isfinite(vt).all() and vt.min() >= 0 and vt.max() <= 1
    assert np.array_equal(vm[ft], f)
    axes = A.tables()[0]
    nrm, bucket = A.faces(v, f, axes)
    keep = bucket >= 0
    assert (A.dot3(nrm[keep], axes[bucket[keep]]) >= 0.886).all()
    # faces across a 2-manifold edge in one chart share that edge's two rows
    mate = A.mates(f, keep)
    e = np.nonzero(mate >= 0)[0]
    m = mate[e]
    rows = lambda x: np.sort(np.stack([ft.reshape(-1)[x], ft.reshape(-1)[3 * (x // 3) + (x % 3 + 1) % 3]], 1), 1)
    same = (rows(e) == rows(m)).all(1)
    chart = _charts_of(ft, len(vt))
    assert np.array_equal(same, chart[e // 3] == chart[m // 3])
    # positive signed UV area, and the stretch of the one projection
    t = vt.astype(np.float64)[ft]
    uv = 0.5 * ((t[:, 1, 0] - t[:, 0, 0]) * (t[:, 2, 1] - t[:, 0, 1]) - (t[:, 1, 1] - t[:, 0, 1]) * (t[:, 2, 0] - t[:, 0, 0]))
    assert (uv[keep] > 0).all()
    p = v.astype(np.float64)[f]
    a3 = 0.5 * np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1)
    big = keep & (uv * res * res >= 1.0)
    ratio = uv[big] * res * res / (s * s * a3[big])
    assert ratio.max() <= 1 + 1e-3 and ratio.min() >= 0.5 - 1e-3
    first_bucket = np.full(chart.max() + 1, -2)          # charts whose faces all have one bucket: no merge, the 27.6 deg cone
    first_bucket[chart[keep][::-1]] = bucket[keep][::-1]
    mixed = np.zeros(chart.max() + 1, bool)
    np.logical_or.at(mixed, chart[keep], bucket[keep] != first_bucket[chart[keep]])
    pure = big & ~mixed[chart]
    assert (uv[pure] * res * res / (s * s * a3[pure]) >= 0.886 - 1e-3).all()
    # no bake-raster texel centre strictly inside two faces
    fs, ts = A.inside_pairs(vt[ft[keep]], np.nonzero(keep)[0], res * ssaa)
    assert len(np.unique(ts)) == len(ts)
    # PAD final texels between the charts' texels
    lo = np.full((chart.max() + 1, 2), np.inf); hi = np.full_like(lo, -np.inf)
    np.minimum.at(lo, np.repeat(chart, 3), t.reshape(-1, 2) * res); np.maximum.at(hi, np.repeat(chart, 3), t.reshape(-1, 2) * res)
    lo, hi = np.floor(lo + 1e-3), np.ceil(hi - 1e-3)                   # the texels each chart touches: [lo, hi)
    gap = np.maximum(lo[None, :, :] - hi[:, None, :], lo[:, None, :] - hi[None, :, :]).max(-1)
    np.fill_diagonal(gap, np.inf)
    assert gap.min() >= A.PAD and lo.min() >= A.PAD and hi.max() <= res - A.PAD


# utilization of the unit square as measured on each mesh (resolution 512, ssaa 2), and the chart counts the constants give
MEASURED = {"icosphere4": (0.562, 26), "mc_sphere64": (0.654, 26), "mc_torus64": (0.456, 50), "noisy_decimated": (0.381, 897)}


@pytest.fixture(scope="module")
def meshes():
    return property_meshes()


@pytest.mark.parametrize("name", list(MEASURED))
def test_atlas_properties(meshes, name):
    v, f = meshes[name]
    info = {}
    vt, ft, vm = A.unwrap(v, f, RES, SSAA, info)
    print(name, len(f), info)
    check_properties(v, f, vt, ft, vm, info)
    util, charts = MEASURED[name]
    assert info["utilization"] >= util and info["charts"] == charts


# ---- the host tables and the C ABI -----------------------------------------------------------------------------------------------------
def test_tables_and_constants_are_the_libraries():
    from nerf2mesh_b200 import texture as X
    for a, b in zip(A.tables(), X.atlas_tables()):
        assert np.array_equal(a, b)
    axes, basis, _ = A.tables()
    assert np.allclose(np.cross(basis[:, :3], basis[:, 3:]), axes) and np.allclose(A.dot3(basis[:, :3], basis[:, 3:]), 0)
    assert (A.SMALL_CHART, A.MERGE_ROUNDS, A.ANGLES, A.PAD, A.BISECT_STEPS, A.MERGE_COS) == \
        (X.SMALL_CHART, X.MERGE_ROUNDS, X.ANGLES, X.PAD, X.BISECT_STEPS, X.MERGE_COS)
    # a unit vector lies within about 27.6 deg of its bucket's axis: sampled
    u = np.random.default_rng(0).standard_normal((200000, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    assert A.dot3(u[:, None, :], axes[None]).max(1).min() >= 0.886


def test_atlas_entries_are_exported_bound_and_documented():
    from nerf2mesh_b200 import _lib, texture  # noqa: F401  (registers the atlas signatures)
    code = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(n2m_atlas_[a-z0-9_]+)\s*\(", code)))
    assert len(syms) == 14, syms
    header = open(HEADER).read()
    for s in syms:
        assert hasattr(_lib.lib, s), f"libn2m_b200.so does not export {s}"
        assert s in _lib.SIGNATURES, f"{s} is not bound in texture.py"
        assert f"*   {s} " in header or f"*   {s}:" in header, f"{s} has no comment entry in the header"


def test_uv_unwrap_input_checks():
    import torch
    from nerf2mesh_b200 import texture as X
    v, f = cube()
    with pytest.raises(ValueError):
        X.uv_unwrap(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), 64)          # not on a CUDA device


def test_export_stage1_needs_both_vt_and_ft():
    from nerf2mesh_b200 import texture as X
    with pytest.raises(ValueError, match="both"):
        X.export_stage1(type("S1", (), {"t0": None, "cascades": 1})(), "/nonexistent", vt=np.zeros((3, 2), np.float32))


def test_atlas_kernels_have_no_spills(tmp_path):
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "atlas.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    found = []
    for i, l in enumerate(lines):
        if "Function properties for" in l and "atlas" in l:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            assert m and (int(m.group(2)), int(m.group(3))) == (0, 0), l + "\n" + lines[i + 1]
            found.append(l)
    assert len(found) >= 20, found
