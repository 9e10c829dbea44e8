"""CPU: the stage-1 mesh regularisers of the vertex offsets (Stage1Trainer(lambda_normal=..., lambda_edgelen=...), the reference's
pytorch3d mesh_normal_consistency and mesh_edge_loss terms) -- the float64 oracle (tests/mesh_reg_oracle.py) against closed forms, the
kernel's hand-derived gradient against autograd, the step's launch sequence with the CUDA layer mocked, and the compile-time budget of
the new kernels."""
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import nerf2mesh_b200.stage1 as S1
from nerf2mesh_b200 import build as B

import mesh_reg_oracle as O
from test_offset_grad_cpu import AA, ADAM, BWD, FWD, _step, mocked  # noqa: F401  (the mocked CUDA layer fixture)


def _losses(v, f):
    n, e = O.regularisers(torch.from_numpy(np.asarray(v, np.float64)), f)
    return float(n), float(e)


def test_flat_grid_has_zero_normal_loss():
    v, f = O.grid(4)
    n, e = _losses(v, f)
    assert n == 0.0
    # 40 unique edges: 2 * 4 * 5 axis edges of length 1 and 16 diagonals of length^2 2
    assert abs(e - (40 * 1 + 16 * 2) / 56) < 1e-12


def test_cube_normal_loss():
    """12 cube edges at 90 degrees (1 - cos = 1) and 6 face diagonals at 0 degrees (0): 12 / 18"""
    v, f = O.cube()
    assert len(O.edge_faces(f)) == 18 and O.pairs(f).shape == (18, 4)
    n, e = _losses(v, f)
    assert abs(n - 12 / 18) < 1e-12
    assert abs(e - (12 * 1 + 6 * 2) / 18) < 1e-12


@pytest.mark.parametrize("phi", [0.0, 0.3, np.pi / 2, 2.0, 3.0])
def test_hinge_normal_loss(phi):
    v, f = O.hinge(phi)
    n, _ = _losses(v, f)
    assert abs(n - (1 - np.cos(phi))) < 1e-12


def test_right_triangle_edge_loss():
    v = np.array([[0, 0, 0], [3, 0, 0], [0, 4, 0]], np.float64)
    f = np.array([[0, 1, 2]])
    n, e = _losses(v, f)
    assert n == 0.0 and abs(e - (9 + 16 + 25) / 3) < 1e-12
    _, g = O.loss_and_grad(v, f, 0.0, 1.0)
    # d/dv_i = sum over its two edges of 2 (v_i - v_j), over the mean's 3 edges
    want = np.array([[-6, -8, 0], [12, -8, 0], [-6, 16, 0]], np.float64) / 3
    assert np.allclose(g.numpy(), want, atol=1e-12)


def _meshes():
    rng = np.random.default_rng(0)
    out = {}
    v, f = O.grid(5, z=rng.normal(scale=0.3, size=36))
    out["bumpy_grid"] = (v, f)
    v, f = O.cube()
    out["perturbed_cube"] = (v + rng.normal(scale=0.05, size=v.shape), f)
    for phi in (0.0, 1e-3, 2.5):
        out[f"hinge_{phi}"] = O.hinge(phi)
    # a collinear (zero-area) face on exact coordinates: n = 0 exactly, torch's clamped branch
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0.5, 1, 0.3]], np.float64)
    out["zero_area"] = (v, np.array([[0, 1, 2], [1, 0, 3]], np.int64))
    # two faces on the same three vertices (opposite orientation): each edge pairs the face with its twin
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float64)
    out["twin"] = (v, np.array([[0, 1, 2], [0, 2, 1]], np.int64))
    return out


@pytest.mark.parametrize("name", sorted(_meshes()))
def test_kernel_closed_form_matches_autograd(name):
    """the expressions k_s1_mesh_reg evaluates (|u + w|^2 / 2, the clamped branch below eps) and its hand-derived gradient through
    the cross products == torch autograd of the definition"""
    v, f = _meshes()[name]
    lam_n, lam_e = 0.7, 0.2
    loss_ref, g_ref = O.loss_and_grad(v, f, lam_n, lam_e)
    loss, g = O.closed_form(v, f, lam_n, lam_e)
    assert abs(loss - loss_ref) <= 1e-12 * max(1.0, abs(loss_ref))
    g_ref = g_ref.numpy()
    assert np.abs(g - g_ref).max() <= 1e-9 * max(1.0, np.abs(g_ref).max()), (g, g_ref)
    if name == "zero_area":
        # pair loss 1 - 0; the zero face's normal gets n_other / eps, ~1e8
        _, g_n = O.loss_and_grad(v, f, 1.0, 0.0)
        assert abs(O.regularisers(torch.from_numpy(v), f)[0].item() - 1.0) < 1e-12
        assert np.abs(g_n.numpy()).max() > 1e7


# ---- the host side, with the CUDA layer mocked ----
def _names(m):
    return [n for n, _ in m.calls]


def test_both_lambdas_zero_keep_the_parent_sequence(mocked):
    for kw in ({}, {"offset_nerf_grad": True}):
        s1 = mocked.make(antialias=True, lr_vert=1e-4, lambda_normal=0.0, lambda_edgelen=0.0, **kw)
        assert "n2m_s1_mesh_reg_setup" not in _names(mocked)
        seq = _step(mocked, s1)
        step = "n2m_s1_vert_step_world" if kw else "n2m_s1_vert_step"
        grad = ["n2m_s1_offset_grad"] if kw else []
        assert seq == FWD + AA + BWD + grad + ["n2m_s1_vert_check"] + ADAM[:3] + [step, ADAM[3]]
        assert s1.vert_scratch.shape == (6 * 5,)
        args = dict(mocked.calls)[step]
        assert len(args) == (21 if kw else 20) and args[-8:-5] == (s1.lambda_lap, s1.lambda_offsets, -1.0)


@pytest.mark.parametrize("world", [False, True])
@pytest.mark.parametrize("lams", [(1e-3, 0.0), (0.0, 0.5), (1e-2, 0.5)])
def test_regularised_sequence(mocked, world, lams):
    ln, le = lams
    mocked.calls.clear()
    s1 = mocked.make(antialias=True, lr_vert=1e-4, offset_nerf_grad=world, lambda_normal=ln, lambda_edgelen=le)
    assert _names(mocked).count("n2m_s1_mesh_reg_setup") == 1                      # once at construction
    setup = dict(mocked.calls)["n2m_s1_mesh_reg_setup"]
    th = s1.topology
    assert setup[:4] == (th.tri.data_ptr(), 2, th.keys.data_ptr(), th.slots) and len(setup) == 7
    seq = _step(mocked, s1)
    grad = ["n2m_s1_offset_grad"] if world else []
    assert seq == FWD + AA + BWD + grad + ["n2m_s1_vert_check"] + ADAM[:3] + ["n2m_s1_vert_step_reg", ADAM[3]]
    a = dict(mocked.calls)["n2m_s1_vert_step_reg"]
    assert len(a) == 26
    assert a[:2] == (s1.grad_vclip.data_ptr(), s1.grad_vworld.data_ptr() if world else None)
    assert a[3:8] == (th.keys.data_ptr(), th.opp.data_ptr(), th.slots, s1.mesh_edges, s1.mesh_pairs)
    assert a[13:16] == (s1.vert_scratch.data_ptr(), s1.grad_offsets.data_ptr(), 5)
    assert a[16:22] == (s1.lambda_lap, s1.lambda_offsets, ln, le, -1.0, mocked.t0.cfg.eps)
    assert a[-2] == s1.loss_acc.data_ptr() and s1.vert_scratch.shape == (9 * 5,)
    # replace_mesh: the new mesh is checked before anything changes, then the concatenated mesh's counts are read again
    mocked.calls.clear()
    s1.replace_mesh(torch.rand(9, 3), torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 7, 8]]))
    assert _names(mocked).count("n2m_s1_mesh_reg_setup") == 2
    assert s1.vert_scratch.shape == (9 * 9,)
    assert _step(mocked, s1)[-2] == "n2m_s1_vert_step_reg"


@pytest.fixture
def counts(mocked, monkeypatch):
    """the setup entry reports `counts.value` = (E, P, non-manifold edges, repeated-index faces) into its host array"""
    box = types.SimpleNamespace(value=(3, 1, 0, 0))

    def fake_call(name, *a):
        mocked.calls.append((name, a))
        if name == "n2m_s1_mesh_reg_setup":
            for k, c in enumerate(box.value):
                a[-2][k] = c
    monkeypatch.setattr(S1, "call", fake_call)
    return box


def test_counts_become_launch_constants(mocked, counts):
    counts.value = (7, 5, 0, 0)
    s1 = mocked.make(antialias=True, lr_vert=1e-4, lambda_normal=1e-3)
    assert (s1.mesh_edges, s1.mesh_pairs) == (7, 5)
    _step(mocked, s1)
    assert dict(mocked.calls)["n2m_s1_vert_step_reg"][6:8] == (7, 5)


def test_non_manifold_and_repeated_index_meshes_are_rejected(mocked, counts):
    counts.value = (10, 6, 2, 0)
    with pytest.raises(ValueError, match="2 non-manifold edges"):
        mocked.make(antialias=True, lr_vert=1e-4, lambda_normal=1e-3)
    s1 = mocked.make(antialias=True, lr_vert=1e-4, lambda_edgelen=0.5)            # the edge loss does not care
    assert (s1.mesh_edges, s1.mesh_pairs) == (10, 6)
    counts.value = (10, 6, 0, 3)
    for kw in ({"lambda_normal": 1e-3}, {"lambda_edgelen": 0.5}):
        with pytest.raises(ValueError, match="3 faces with a repeated vertex index"):
            mocked.make(antialias=True, lr_vert=1e-4, **kw)
    # replace_mesh rejects before anything changes: the trainer keeps its mesh and its buffers
    counts.value = (3, 1, 0, 0)
    s1 = mocked.make(antialias=True, lr_vert=1e-4, lambda_normal=1e-3)
    tri, scratch = s1.triangles, s1.vert_scratch
    counts.value = (12, 7, 1, 0)
    with pytest.raises(ValueError, match="replace_mesh: 1 non-manifold edges"):
        s1.replace_mesh(torch.rand(9, 3), torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 7, 8]]))
    assert s1.triangles is tri and s1.vert_scratch is scratch


@pytest.mark.parametrize("kw", [{"lambda_normal": 1e-3}, {"lambda_edgelen": 1.0}, {"lambda_normal": 1e-3, "antialias": True},
                                {"lambda_normal": -1e-3, "antialias": True, "lr_vert": 1e-4},
                                {"lambda_edgelen": -1.0, "antialias": True, "lr_vert": 1e-4}])
def test_regularisers_need_the_vertex_optimizer(mocked, kw):
    with pytest.raises(ValueError):
        mocked.make(**kw)


def test_new_kernels_have_no_spills_and_no_stack(tmp_path):
    """the per-step slot walk (k_s1_mesh_reg), the two setup kernels and the Adam overload that reads the regularisers' gradient"""
    pats = [r"k_s1_mesh_regEP", r"k_s1_mesh_reg_faces", r"k_s1_mesh_reg_slots", r"14k_s1_vert_adamEPK"]
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, "stage1.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    for pat in pats:
        props = [i for i, l in enumerate(lines) if "Function properties for" in l and re.search(pat, l)]
        assert len(props) == 1, (pat, "\n".join(lines))
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[props[0] + 1])
        assert m and (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (0, 0, 0), lines[props[0]] + "\n" + lines[props[0] + 1]
