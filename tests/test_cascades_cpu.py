"""CPU: the host logic of unbounded scenes through stage 1 with the CUDA layer mocked -- the cascade bookkeeping of Stage1Trainer (v_cumsum /
f_cumsum, cascade_mesh, refine_mask over cascade 0, replace_mesh rebasing the outer cascades), the per-cascade export's files and texture
sizes, load_stage0_meshes -- the numpy float64 oracle of the outer-mesh chain (tests/cascade_oracle.py) on hand-built meshes, and the
compile-time budget of the new kernels."""
import json
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import cascade_oracle as CO
import nerf2mesh_b200.mesh as M
import nerf2mesh_b200.stage1 as S1
import nerf2mesh_b200.texture as X
from nerf2mesh_b200 import build as B
from test_refine_cpu import FWD, _numpy_refine_mask, _step_names, mocked  # noqa: F401  (the mocked CUDA layer fixture)


def _meshes():
    g = torch.Generator().manual_seed(3)
    vs = [torch.rand(5, 3, generator=g), torch.rand(4, 3, generator=g), torch.rand(3, 3, generator=g)]
    fs = [torch.tensor([[0, 1, 2], [2, 3, 4]]), torch.tensor([[0, 1, 2], [1, 2, 3], [0, 2, 3]]), torch.tensor([[0, 1, 2]])]
    return vs, fs


def _make(m, vs, fs, **kw):
    return S1.Stage1Trainer(m.t0, vs, fs, 4, 4, ssaa=2, **kw)


def test_cascaded_trainer_concatenates_with_offsets(mocked):
    vs, fs = _meshes()
    s1 = _make(mocked, vs, fs)
    assert s1.v_cumsum == [0, 5, 9, 12] and s1.f_cumsum == [0, 2, 5, 6] and s1.cascades == 3
    assert all(type(x) is int for x in s1.v_cumsum + s1.f_cumsum)
    assert torch.equal(s1.vertices, torch.cat(vs)) and s1.triangles.dtype == torch.int32
    assert torch.equal(s1.triangles, torch.cat([fs[0], fs[1] + 5, fs[2] + 9]).int())
    for cas in range(3):
        v, f = s1.cascade_mesh(cas)
        assert torch.equal(v, vs[cas]) and torch.equal(f, fs[cas].int())
    # the step over the concatenated mesh launches what a one-mesh step launches, with the total face count
    one = _make(mocked, torch.cat(vs), torch.cat([fs[0], fs[1] + 5, fs[2] + 9]), refine=True)
    many = _make(mocked, vs, fs, refine=True)
    assert _step_names(mocked, many) == _step_names(mocked, one)
    args = next(a for n, a in mocked.calls if n == "n2m_s1_loss_err")
    assert args[-2] == 6


@pytest.mark.parametrize("as_list", [False, True])
def test_single_mesh_is_one_cascade(mocked, as_list):
    v, f = torch.rand(5, 3), torch.tensor([[0, 1, 2], [2, 3, 4]])
    s1 = _make(mocked, [v] if as_list else v, [f] if as_list else f)
    assert s1.v_cumsum == [0, 5] and s1.f_cumsum == [0, 2] and s1.cascades == 1
    assert torch.equal(s1.vertices, v) and torch.equal(s1.triangles, f.int())
    assert _step_names(mocked, s1)[:len(FWD)] == FWD


@pytest.mark.parametrize("vs,fs", [([torch.rand(3, 3)], []), ([], []), ([torch.rand(3, 3)] * 2, [torch.tensor([[0, 1, 2]])])])
def test_cascade_lists_must_pair_up(mocked, vs, fs):
    with pytest.raises(ValueError):
        _make(mocked, vs, fs)


def test_contract_selects_the_contracting_points_entry(mocked):
    vs, fs = _meshes()
    mocked.t0.cfg = types.SimpleNamespace(eps=1e-15, contract=True)
    names = _step_names(mocked, _make(mocked, vs, fs))
    assert names[:len(FWD)] == ["n2m_rasterize", "n2m_s1_points_contract"] + FWD[2:]
    args = next(a for n, a in mocked.calls if n == "n2m_s1_points_contract")
    assert args[-2:] == (1, 0)                                                  # contract flag, stream
    mocked.t0.cfg = types.SimpleNamespace(eps=1e-15, contract=False)
    assert _step_names(mocked, _make(mocked, vs, fs))[:len(FWD)] == FWD


def test_refine_mask_covers_cascade_0_only():
    rng = np.random.default_rng(11)
    f_cumsum = [0, 400, 700, 1000]
    cnt = rng.integers(0, 4, 1000).astype(np.float32)
    errors = (rng.random(1000) * cnt).astype(np.float32)
    errors[400:] *= 100                                                          # outer faces: much larger errors, must not count
    s1 = object.__new__(S1.Stage1Trainer)
    s1.refine, s1.f_cumsum = True, f_cumsum
    s1.face_errors, s1.face_counts = torch.from_numpy(errors.copy()), torch.from_numpy(cnt.copy())
    mask, (t_ref, t_dec) = s1.refine_mask()
    ref_mask, ref_t_ref, ref_t_dec = _numpy_refine_mask(errors[:400], cnt[:400])
    assert mask.shape == (400,) and np.array_equal(mask.numpy(), ref_mask)
    assert t_ref == float(ref_t_ref) and t_dec == float(ref_t_dec)
    cnt[:400] = 0                                                                # only outer faces seen: nothing to threshold
    s1.face_counts = torch.from_numpy(cnt)
    with pytest.raises(ValueError):
        s1.refine_mask()


def test_replace_mesh_rebases_the_outer_cascades(mocked):
    vs, fs = _meshes()
    s1 = _make(mocked, vs, fs, antialias=True, lr_vert=1e-4, refine=True)
    s1.offsets.copy_(torch.rand(12, 3) * 0.01)
    s1.vertices.copy_(s1.base_vertices + s1.offsets)                             # what the vertex step leaves: base + offsets
    for b in (s1.m_vert, s1.v_vert, s1.face_errors, s1.face_counts):
        b.fill_(3.0)
    moved = s1.vertices.clone()
    v0 = torch.rand(7, 3, dtype=torch.float64)
    f0 = torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [0, 3, 6]])
    s1.replace_mesh(v0, f0)
    assert s1.v_cumsum == [0, 7, 11, 14] and s1.f_cumsum == [0, 4, 7, 8]
    assert torch.equal(s1.vertices[:7], v0.float())
    assert torch.equal(s1.vertices[7:], moved[5:]) and torch.equal(s1.base_vertices, s1.vertices)
    assert torch.equal(s1.triangles, torch.cat([f0, fs[1] + 7, fs[2] + 11]).int())
    for name in ("offsets", "m_vert", "v_vert", "face_errors", "face_counts"):
        b = getattr(s1, name)
        assert b.shape[0] == (14 if name in ("offsets", "m_vert", "v_vert") else 8) and not b.any(), name
    assert s1.topology.tri is s1.triangles and s1._graphs == {}


def test_texture_sizes_halve_above_2048():
    assert X.texture_sizes(4096, 5) == [4096, 2048, 2048, 2048, 2048]
    assert X.texture_sizes(8192, 4) == [8192, 4096, 2048, 2048]
    assert X.texture_sizes(2048, 3) == [2048, 2048, 2048]
    assert X.texture_sizes(1024, 1) == [1024]


def test_cascaded_export_writes_one_set_of_files_per_cascade(mocked, monkeypatch, tmp_path):
    vs, fs = _meshes()
    s1 = _make(mocked, vs, fs)
    mocked.t0.cfg = types.SimpleNamespace(eps=1e-15, bound=4.0)
    baked = []

    def fake_bake(t0, v, f, vt, ft, h0, w0, ssaa=2, band_rows=None):
        baked.append((v.shape[0], f.shape[0], h0, w0, ssaa))
        return torch.zeros(h0, w0, 3, dtype=torch.uint8), torch.zeros(h0, w0, 3, dtype=torch.uint8)
    monkeypatch.setattr(X, "bake_features", fake_bake)
    monkeypatch.setattr(X, "specular_weights", lambda t0: {"net.0.weight": np.zeros((32, 6)), "net.1.weight": np.zeros((3, 32))})
    vts = [torch.rand(3 * f.shape[0], 2) for f in fs]
    fts = [torch.arange(3 * f.shape[0], dtype=torch.int32).view(-1, 3) for f in fs]
    out = X.export_stage1(s1, str(tmp_path), vts, fts, resolution=4096)
    assert len(out) == 3
    assert baked == [(5, 2, 4096, 4096, 2), (4, 3, 2048, 2048, 2), (3, 1, 2048, 2048, 2)]
    names = sorted(os.listdir(tmp_path))
    assert names == sorted(["mlp.json"] + [f"{k}_{c}.{e}" for c in range(3) for k, e in
                                           (("mesh", "obj"), ("mesh", "mtl"), ("feat0", "jpg"), ("feat1", "jpg"))])
    for c in range(3):
        obj = open(tmp_path / f"mesh_{c}.obj").read().splitlines()
        assert obj[0].strip() == f"mtllib mesh_{c}.mtl"
        assert sum(l.startswith("v ") for l in obj) == vs[c].shape[0] and sum(l.startswith("f ") for l in obj) == fs[c].shape[0]
        assert f"map_Kd feat0_{c}.jpg" in open(tmp_path / f"mesh_{c}.mtl").read()
    assert json.load(open(tmp_path / "mlp.json"))["cascade"] == 3
    with pytest.raises(ValueError):                                   # a cascaded trainer needs one unwrap per cascade
        X.export_stage1(s1, str(tmp_path), vts[0], fts[0])


def test_load_stage0_meshes_prefers_updated(tmp_path):
    vs, fs = _meshes()
    for c in range(3):
        M.write_ply(tmp_path / f"mesh_{c}.ply", vs[c], fs[c])
    M.write_ply(tmp_path / "mesh_1_updated.ply", vs[2], fs[2])
    v, f = M.load_stage0_meshes(str(tmp_path), 3)
    assert [x.shape[0] for x in v] == [5, 3, 3] and torch.equal(v[1], vs[2]) and torch.equal(f[1], fs[2].int())
    assert v[0].dtype == torch.float32 and f[0].dtype == torch.int32
    os.remove(tmp_path / "mesh_2.ply")
    with pytest.raises(FileNotFoundError, match="mesh_2.ply"):
        M.load_stage0_meshes(str(tmp_path), 3)


# ---- the numpy oracle of the outer-mesh chain on hand-built meshes ------------------------------------------------------------------
def test_oracle_remove_selected_verts_keeps_unreferenced_survivors():
    v = np.arange(18, dtype=np.float64).reshape(6, 3)
    f = np.array([[0, 1, 2], [2, 3, 4], [3, 4, 5], [0, 4, 5]])
    v2, f2 = CO.remove_selected_verts(v, f, np.array([0, 0, 0, 1, 0, 0], bool))
    assert np.array_equal(v2, v[[0, 1, 2, 4, 5]])
    assert np.array_equal(f2, [[0, 1, 2], [0, 3, 4]])                   # vertex 3 gone with faces 1 and 2; 4 -> 3, 5 -> 4
    v3, f3 = CO.remove_selected_verts(v, f, np.array([0, 0, 1, 0, 0, 0], bool))
    assert np.array_equal(v3, v[[0, 1, 3, 4, 5]]) and np.array_equal(f3, [[2, 3, 4], [0, 3, 4]])
    v4, f4 = CO.remove_selected_verts(v, f[:1], np.array([0, 1, 0, 0, 0, 0], bool))
    assert v4.shape == (5, 3) and f4.shape == (0, 3)                     # 3, 4, 5 unreferenced, kept


def test_oracle_outer_chain_on_a_hand_built_mesh():
    R, bound = 9, 4.0
    half = bound / R
    # index coordinates -> p = idx / 8 * 2 - 1 in {-1, -0.75, ..., 1}; 0.45 lies between 0.25 and 0.5
    vidx = np.array([[4, 4, 4],        # p = 0: centre box
                     [5, 4, 3],        # p = (0.25, 0, -0.25): centre box
                     [6, 4, 4],        # p = (0.5, 0, 0): outside the box (0.5 > 0.45), inside the AABB
                     [0, 4, 4],        # p = (-1, 0, 0): x = -(bound - half) <= xmn + half with the AABB at -bound
                     [2, 7, 4],        # p = (-0.5, 0.75, 0): kept
                     [4, 4, 8],        # p = (0, 0, 1): z >= zmx - half
                     [2.5, 2, 6]],     # p = (-0.375, -0.5, 0.5): kept (a marching-cubes midpoint)
                    np.float64)
    f = np.array([[0, 2, 4], [2, 4, 6], [3, 4, 6], [2, 5, 6], [1, 2, 6]])
    aabb = (-bound, -bound, -bound, bound, bound, bound)
    v, tri = CO.outer_chain(vidx, f, R, bound, aabb)
    p = vidx[[2, 4, 6]] / (R - 1.0) * 2 - 1
    assert v.dtype == np.float32 and np.array_equal(v, (p * (bound - half)).astype(np.float32))
    assert tri.dtype == np.int32 and np.array_equal(tri, [[0, 1, 2]])
    # a tighter AABB also removes the vertex at y = 0.75 * (bound - half) = 2.666...
    v, tri = CO.outer_chain(vidx, f, R, bound, (-bound, -bound, -bound, bound, 2.5 + half, bound))
    assert v.shape == (2, 3) and tri.shape == (0, 3)
    # everything in the centre: nothing left
    v, tri = CO.outer_chain(np.array([[4, 4, 4], [4.5, 4, 4], [4, 3.5, 4]]), np.array([[0, 1, 2]]), R, bound, aabb)
    assert v.shape == (0, 3) and tri.shape == (0, 3)


def test_new_kernels_have_no_spills(tmp_path):
    found = []
    for src, pat in (("cascade.cu", r"k_outer_occupancy|k_outer_select|k_rsv_count|k_rsv_emit|k_mark_seen_faces"),
                     ("stage1.cu", r"k_s1_pointsILb1E")):
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, src), "-o", str(tmp_path / "k.o")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        lines = (r.stdout + r.stderr).splitlines()
        for i, l in enumerate(lines):
            if "Function properties for" in l and re.search(pat, l):
                m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
                assert m and (int(m.group(2)), int(m.group(3))) == (0, 0), l + "\n" + lines[i + 1]
                found.append(l)
    assert len(found) == 6, found
