"""CPU: the colour-field path of the stage-1 vertex gradient (Stage1Trainer(offset_nerf_grad=True), the reference's
--enable_offset_nerf_grad) -- the float64 restatement of the dr.rasterize / dr.interpolate gradients and of contract()'s backward
(tests/raster_grad_oracle.py) against central finite differences and torch autograd, the step's launch sequence with the CUDA layer
mocked, and the compile-time budget of the new kernels."""
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import nerf2mesh_b200.raster as RA
import nerf2mesh_b200.stage0 as S0
import nerf2mesh_b200.stage1 as S1
from nerf2mesh_b200 import build as B

import raster_grad_oracle as O

FWD = ["n2m_rasterize", "n2m_s1_points", "n2m_s0_encode_points", "n2m_s0_mlp_fwd"]
BWD = ["n2m_s0_mlp_bwd", "n2m_s0_encode_bwd"]
ADAM = ["n2m_s0_adam_head", "n2m_s0_adam_mlp", "n2m_s0_adam_tables", "n2m_s0_adam_post"]
AA = ["n2m_s1_rgba", "n2m_antialias_forward", "n2m_s1_loss_aa", "n2m_antialias_backward", "n2m_s1_dout"]


def _triangles(kind, n, rng):
    """random clip-space triangles with a pixel NDC (X, Y) inside the part in front of the camera"""
    out = []
    while len(out) < n:
        P = np.zeros((3, 4))
        P[:, :2] = rng.uniform(-1.5, 1.5, (3, 2))
        P[:, 2] = rng.uniform(-0.5, 0.5, 3)
        P[:, 3] = rng.uniform(0.5, 3.0, 3)
        if kind == "crossing":
            k = rng.integers(0, 3)
            P[k, 3] = -rng.uniform(0.1, 2.0)
        b = rng.dirichlet(np.ones(3) * 2)          # a point of the triangle in front of the camera: sum b'_k p_k with w > 0
        h = b @ P
        if h[3] <= 0.2:
            continue
        X, Y = h[0] / h[3], h[1] / h[3]
        if kind == "crossing":
            assert (P[:, 3] <= 0).any() and (P[:, 3] > 0).any()
        out.append((P, X, Y))
    return out


@pytest.mark.parametrize("kind", ["front", "crossing"])
def test_rasterize_backward_matches_finite_differences(kind):
    rng = np.random.default_rng(11 if kind == "front" else 12)
    for P, X, Y in _triangles(kind, 40, rng):
        u, v = O.uv(P, X, Y)
        assert u >= -1e-9 and v >= -1e-9 and 1 - u - v >= -1e-9          # the pixel is covered
        du, dv = rng.normal(size=2)
        g = O.rasterize_backward(P, X, Y, du, dv)
        fd = np.zeros((3, 4))
        eps = 1e-6
        for k in range(3):
            for c in range(4):
                Pp, Pm = P.copy(), P.copy()
                Pp[k, c] += eps; Pm[k, c] -= eps
                up, vp = O.uv(Pp, X, Y); um, vm = O.uv(Pm, X, Y)
                fd[k, c] = (du * (up - um) + dv * (vp - vm)) / (2 * eps)
        assert np.all(g[:, 2] == 0) and np.allclose(fd[:, 2], 0, atol=1e-9)        # clip z carries nothing
        assert np.allclose(g, fd, rtol=1e-6, atol=1e-7 * max(1.0, np.abs(fd).max())), (g, fd)


def test_closed_form_is_the_perspective_correct_barycentric():
    """in front of the camera, (u, v) of the closed form == screen-space barycentrics made perspective-correct (k_rast_resolve)"""
    rng = np.random.default_rng(3)
    for P, X, Y in _triangles("front", 30, rng):
        s = P[:, :2] / P[:, 3:4]
        area = lambda a, b, c: (b[0] - a[0]) * (c[1] - a[1]) - (c[0] - a[0]) * (b[1] - a[1])
        pnt = np.array([X, Y])
        A = area(s[0], s[1], s[2])
        b = np.array([area(pnt, s[1], s[2]), area(s[0], pnt, s[2]), area(s[0], s[1], pnt)]) / A
        pc = b / P[:, 3]
        pc /= pc.sum()
        u, v = O.uv(P, X, Y)
        assert abs(u - pc[0]) < 1e-10 and abs(v - pc[1]) < 1e-10


def test_interpolate_backward_rast_matches_finite_differences():
    rng = np.random.default_rng(5)
    for A in (1, 2, 3, 4):
        a0, a1, a2, g = (rng.normal(size=A) for _ in range(4))
        u, v = rng.uniform(0, 0.5, 2)
        out = lambda u, v: u * a0 + v * a1 + (1 - u - v) * a2
        du, dv = O.interpolate_backward_rast(g, a0, a1, a2)
        eps = 1e-6
        assert abs(du - g @ (out(u + eps, v) - out(u - eps, v)) / (2 * eps)) < 1e-8
        assert abs(dv - g @ (out(u, v + eps) - out(u, v - eps)) / (2 * eps)) < 1e-8
    # the mask of the reference: interpolate(ones) has an exactly zero (u, v) gradient
    assert O.interpolate_backward_rast([0.37], [1.0], [1.0], [1.0]) == (0.0, 0.0)


@pytest.mark.parametrize("x", [[0.3, -0.5, 0.9], [1.7, 0.2, -0.4], [-0.3, -2.5, 1.1], [1.5, -1.5, 0.2], [1.3, 1.3, -1.3], [3.0, 2.0, 1.0]])
def test_contract_backward_matches_torch_autograd(x):
    """contract() of renderer.py:25-32 by torch autograd (float64), including ties of |x_k| (torch's amax backward splits evenly)"""
    xt = torch.tensor([x], dtype=torch.float64, requires_grad=True)
    mag = torch.amax(torch.abs(xt), dim=1, keepdim=True)
    y = torch.where(mag <= 1, xt, xt * (2 - 1 / mag) / mag)
    g = torch.tensor([[0.7, -1.1, 0.4]], dtype=torch.float64)
    y.backward(g)
    assert np.allclose(O.contract_backward(x, g[0].numpy()), xt.grad[0].numpy(), rtol=1e-12, atol=1e-14)


@pytest.fixture
def mocked(monkeypatch):
    """a CPU Stage0Trainer shell and a Stage1Trainer factory over a recording `call`"""
    calls = []
    for mod in (S0, S1, RA):
        monkeypatch.setattr(mod, "call", lambda name, *a: calls.append((name, a)))
        monkeypatch.setattr(mod, "stream", lambda: 0)

    def fake_rasterize(glctx, pos, tri, resolution, **kw):
        calls.append(("n2m_rasterize", ()))
        return torch.zeros(1, resolution[0], resolution[1], 4), None
    monkeypatch.setattr(RA, "rasterize", fake_rasterize)
    monkeypatch.setattr(RA, "TopologyHash", lambda tri: types.SimpleNamespace(keys=torch.zeros(4, dtype=torch.int64),
                                                                             opp=torch.zeros(4, 2, dtype=torch.int32), slots=4, tri=tri))

    class FakeStream:
        def wait_stream(self, o): pass

    class Ctx:
        def __init__(self, s): pass
        def __enter__(self): return self
        def __exit__(self, *a): return False
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: Ctx(s))

    t0 = object.__new__(S0.Stage0Trainer)
    t0.device = "cpu"
    t0.cfg = types.SimpleNamespace(eps=1e-15)
    for k in ("table", "offsets", "wpack", "color_master", "m_table", "v_table", "mlp", "m_mlp", "v_mlp"):
        setattr(t0, k, torch.zeros(8))
    t0.opt_state = torch.zeros(8)
    t0.gtables, t0.g_mlps, t0.parity, t0.rows, t0._adam_stream, t0.global_step = [torch.zeros(8)] * 2, [torch.zeros(8)], 0, 8, None, 0
    t0.params = S0.S0Params()

    def make(vertices=None, triangles=None, **kw):
        v = torch.rand(5, 3) if vertices is None else vertices
        f = torch.tensor([[0, 1, 2], [2, 3, 4]]) if triangles is None else triangles
        return S1.Stage1Trainer(t0, v, f, 4, 4, ssaa=2, **kw)
    return types.SimpleNamespace(calls=calls, t0=t0, make=make)


def _step(m, s1):
    m.calls.clear()
    s1.step(torch.eye(4), torch.rand(16, 3), torch.rand(16, 4), torch.rand(16, 3))
    return [n for n, _ in m.calls]


def test_offset_grad_launch_sequence(mocked):
    off = _step(mocked, mocked.make(antialias=True, lr_vert=1e-4))
    assert off == FWD + AA + BWD + ["n2m_s1_vert_check"] + ADAM[:3] + ["n2m_s1_vert_step", ADAM[3]]
    s1 = mocked.make(antialias=True, lr_vert=1e-4, offset_nerf_grad=True)
    on = _step(mocked, s1)
    # the colour-field gradient comes after the MLP backward (it reads denc_tiles) and before the overflow scan of the vertex group
    assert on == FWD + AA + BWD + ["n2m_s1_offset_grad", "n2m_s1_vert_check"] + ADAM[:3] + ["n2m_s1_vert_step_world", ADAM[3]]
    assert on.index("n2m_s1_offset_grad") > on.index("n2m_s0_mlp_bwd")
    args = dict(mocked.calls)
    g = args["n2m_s1_offset_grad"]
    assert g[1:6] == (s1.rast.data_ptr(), s1.vertices.data_ptr(), s1.vclip.data_ptr(), s1.triangles.data_ptr(), s1.inv.data_ptr())
    assert g[6:8] == (8, 8) and g[-4:] == (s1.grad_vclip.data_ptr(), s1.grad_vworld.data_ptr(), mocked.t0.opt_state.data_ptr(), 0)
    w = args["n2m_s1_vert_step_world"]
    assert w[:2] == (s1.grad_vclip.data_ptr(), s1.grad_vworld.data_ptr())
    assert len(w) == 21 and s1.grad_vworld.shape == (5, 3) and s1.grad_vworld.dtype == torch.float32


def test_offset_grad_buffers_follow_the_mesh(mocked):
    s1 = mocked.make(antialias=True, lr_vert=1e-4, offset_nerf_grad=True)
    s1.grad_vworld.fill_(3.0)
    s1.replace_mesh(torch.rand(9, 3), torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 7, 8]]))
    assert s1.grad_vworld.shape == (9, 3) and not s1.grad_vworld.any()
    # cascades: one buffer over the concatenated mesh
    s2 = mocked.make([torch.rand(5, 3), torch.rand(4, 3)], [torch.tensor([[0, 1, 2], [2, 3, 4]]), torch.tensor([[0, 1, 2], [1, 2, 3]])],
                     antialias=True, lr_vert=1e-4, offset_nerf_grad=True)
    assert s2.grad_vworld.shape == (9, 3)
    assert not hasattr(mocked.make(antialias=True, lr_vert=1e-4), "grad_vworld")


@pytest.mark.parametrize("kw", [{"offset_nerf_grad": True}, {"offset_nerf_grad": True, "antialias": True},
                                {"offset_nerf_grad": True, "lr_vert": 1e-4}])
def test_offset_grad_needs_the_vertex_optimizer(mocked, kw):
    with pytest.raises(ValueError):
        mocked.make(**kw)


def test_new_kernels_have_no_spills_and_no_stack(tmp_path):
    """one pass over the covered super-samples with a 16-level colour-grid walk (k_s1_offset_grad) and the two operator kernels: a
    spill or a stack frame would add local-memory traffic beside their gathers and atomics"""
    want = {"stage1.cu": [r"k_s1_offset_gradILb0E", r"k_s1_offset_gradILb1E", r"k_s1_vert_adamILb1E"],
            "raster.cu": [r"k_rast_bwd"] + [rf"k_interp_bwd_rastILi{a}E" for a in (1, 2, 3, 4)]}
    for src, pats in want.items():
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, src), "-o", str(tmp_path / "k.o")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        lines = (r.stdout + r.stderr).splitlines()
        for pat in pats:
            props = [i for i, l in enumerate(lines) if "Function properties for" in l and re.search(pat, l)]
            assert len(props) == 1, (pat, "\n".join(lines))
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[props[0] + 1])
            assert m and (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (0, 0, 0), lines[props[0]] + "\n" + lines[props[0] + 1]
