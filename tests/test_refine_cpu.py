"""CPU: stage-1 mesh refinement host logic (nerf2mesh_b200/stage1.py: Stage1Trainer(refine=True), refine_mask, replace_mesh) with the CUDA
layer mocked, and the compile-time budget of the error-scattering loss kernels (csrc/stage1.cu)."""
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

FWD = ["n2m_rasterize", "n2m_s1_points", "n2m_s0_encode_points", "n2m_s0_mlp_fwd"]
BWD = ["n2m_s0_mlp_bwd", "n2m_s0_encode_bwd"]
ADAM = ["n2m_s0_adam_head", "n2m_s0_adam_mlp", "n2m_s0_adam_tables", "n2m_s0_adam_post"]
AA_F = ["n2m_s1_rgba", "n2m_antialias_forward"]


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

    def make(**kw):
        return S1.Stage1Trainer(t0, torch.rand(5, 3), torch.tensor([[0, 1, 2], [2, 3, 4]]), 4, 4, ssaa=2, **kw)
    return types.SimpleNamespace(calls=calls, t0=t0, make=make)


def _step_names(m, s1):
    m.calls.clear()
    s1.step(torch.eye(4), torch.rand(16, 3), torch.rand(16, 4), torch.rand(16, 3))
    return [n for n, _ in m.calls]


@pytest.mark.parametrize("kw,loss", [({}, "n2m_s1_loss"), ({"antialias": True}, "n2m_s1_loss_aa"),
                                     ({"antialias": True, "lr_vert": 1e-4}, "n2m_s1_loss_aa")])
def test_refine_swaps_only_the_loss_launch(mocked, kw, loss):
    off = _step_names(mocked, mocked.make(**kw))
    assert loss in off and not hasattr(mocked.make(**kw), "face_errors")
    s1 = mocked.make(refine=True, **kw)
    on = _step_names(mocked, s1)
    assert on == [loss + "_err" if n == loss else n for n in off]
    assert off[:len(FWD)] == FWD and off[-1] == ADAM[-1]
    # the error variant gets the existing arguments, then rast, face_errors, face_counts, F, then the stream
    args = next(a for n, a in mocked.calls if n == loss + "_err")
    assert args[-5:] == (s1.rast.data_ptr(), s1.face_errors.data_ptr(), s1.face_counts.data_ptr(), 2, 0)
    assert s1.face_errors.shape == (2,) and s1.face_counts.shape == (2,) and s1.face_errors.dtype == torch.float32
    assert not s1.face_errors.any() and not s1.face_counts.any()


def _numpy_refine_mask(errors, cnt):
    """renderer.py:217-240 (non-SDF, one mesh)"""
    errors, cnt = errors.copy(), cnt.copy()
    cnt_mask = cnt > 0
    errors[cnt_mask] = errors[cnt_mask] / cnt[cnt_mask]
    thresh_refine = np.percentile(errors[cnt_mask], 90)
    thresh_decimate = np.percentile(errors[cnt_mask], 50)
    mask = np.zeros_like(errors)
    mask[(errors > thresh_refine) & cnt_mask] = 2
    mask[(errors < thresh_decimate) & cnt_mask] = 1
    return mask, thresh_refine, thresh_decimate


def _trainer_with_errors(errors, cnt):
    s1 = object.__new__(S1.Stage1Trainer)
    s1.refine = True
    s1.face_errors, s1.face_counts = torch.from_numpy(errors.copy()), torch.from_numpy(cnt.copy())
    return s1


def _cases():
    rng = np.random.default_rng(7)
    out = []
    for n in (1, 2, 3, 10, 11, 1000, 4097):                 # random errors, with faces never seen
        cnt = rng.integers(0, 5, n).astype(np.float32)
        cnt[rng.integers(0, n)] = 3.0
        errors = (rng.random(n) * cnt * rng.choice([1e-3, 1.0, 50.0])).astype(np.float32)
        out.append((f"random{n}", errors, cnt))
    cnt = rng.integers(1, 9, 500).astype(np.float32)
    out.append(("all_equal", cnt * np.float32(0.25), cnt))                 # every mean error == 0.25
    cnt = np.zeros(64, np.float32); cnt[17] = 4.0
    errors = np.zeros(64, np.float32); errors[17] = 1.3
    out.append(("single_seen", errors, cnt))
    cnt = rng.integers(0, 3, 300001).astype(np.float32)                    # a refine-sized mesh: float32 virtual index
    out.append(("large", (rng.random(300001) * cnt).astype(np.float32), cnt))
    errors = np.repeat(np.float32([0.1, 0.2, 0.3]), [5, 90, 5]); cnt = np.ones(100, np.float32)  # ties at both thresholds
    out.append(("ties", errors, cnt))
    return out


@pytest.mark.parametrize("name,errors,cnt", _cases(), ids=[c[0] for c in _cases()])
def test_refine_mask_equals_numpy_restatement(name, errors, cnt):
    mask, (t_ref, t_dec) = _trainer_with_errors(errors, cnt).refine_mask()
    ref_mask, ref_t_ref, ref_t_dec = _numpy_refine_mask(errors, cnt)
    assert ref_t_ref.dtype == np.float32 and ref_t_dec.dtype == np.float32
    assert t_ref == float(ref_t_ref) and t_dec == float(ref_t_dec), (t_ref, ref_t_ref, t_dec, ref_t_dec)
    assert mask.dtype == torch.float32 and mask.shape == (errors.shape[0],)
    assert np.array_equal(mask.numpy(), ref_mask)
    if name == "all_equal":
        assert not mask.any()
    if name == "single_seen":
        assert not mask.any() and t_ref == t_dec == pytest.approx(1.3 / 4, rel=1e-7)


def test_refine_mask_without_seen_faces_raises():
    with pytest.raises(ValueError):
        _trainer_with_errors(np.zeros(6, np.float32), np.zeros(6, np.float32)).refine_mask()
    s1 = object.__new__(S1.Stage1Trainer)
    s1.refine = False
    with pytest.raises(RuntimeError):
        s1.refine_mask()


def test_replace_mesh_resizes_and_resets(mocked):
    t0 = mocked.t0
    s1 = mocked.make(antialias=True, lr_vert=1e-4, refine=True)
    s1.step(torch.eye(4), torch.rand(16, 3), torch.rand(16, 4), torch.rand(16, 3))
    for b in (s1.offsets, s1.m_vert, s1.v_vert, s1.vert_state[:1], s1.face_errors, s1.face_counts, s1.grad_vclip):
        b.fill_(3.0)
    s1._graphs[("k",)] = object()
    for k in ("m_table", "v_table", "m_mlp", "v_mlp"):
        getattr(t0, k).fill_(2.0)
    t0.opt_state.copy_(torch.arange(1.0, 9.0))
    v2 = torch.rand(9, 3, dtype=torch.float64)
    f2 = torch.tensor([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 7, 8]], dtype=torch.int64)
    mocked.calls.clear()
    s1.replace_mesh(v2, f2)
    assert s1._graphs == {} and s1._warm is False
    assert s1.vertices.dtype == torch.float32 and torch.equal(s1.vertices, v2.float()) and torch.equal(s1.base_vertices, s1.vertices)
    assert s1.triangles.dtype == torch.int32 and torch.equal(s1.triangles, f2.int())
    for name, shape in (("offsets", (9, 3)), ("m_vert", (9, 3)), ("v_vert", (9, 3)), ("grad_offsets", (9, 3)), ("grad_vclip", (9, 4)),
                        ("vert_scratch", (54,)), ("face_errors", (4,)), ("face_counts", (4,))):
        b = getattr(s1, name)
        assert tuple(b.shape) == shape, name
        assert not b.any(), name
    assert s1.vert_state[0].item() == 0
    assert s1.topology.tri is s1.triangles                                     # edge hash rebuilt on the new triangles
    for k in ("m_table", "v_table", "m_mlp", "v_mlp"):
        assert not getattr(t0, k).any(), k
    assert t0.opt_state.tolist() == [1.0, 2.0, 0.0, 4.0, 5.0, 6.0, 7.0, 8.0]  # step count zeroed, GradScaler state kept
    # the next step runs on the new mesh, eagerly (no graph is warm)
    names = _step_names(mocked, s1)
    assert names == FWD + AA_F + ["n2m_s1_loss_aa_err", "n2m_antialias_backward", "n2m_s1_dout"] + BWD + ["n2m_s1_vert_check"] \
        + ADAM[:3] + ["n2m_s1_vert_step", ADAM[3]]
    args = next(a for n, a in mocked.calls if n == "n2m_s1_loss_aa_err")
    assert args[-2] == 4


def test_replace_mesh_keeps_optimizer_when_asked(mocked):
    t0 = mocked.t0
    s1 = mocked.make(refine=True)
    for k in ("m_table", "v_table", "m_mlp", "v_mlp"):
        getattr(t0, k).fill_(2.0)
    t0.opt_state.fill_(5.0)
    s1.replace_mesh(torch.rand(4, 3), torch.tensor([[0, 1, 2], [1, 2, 3], [0, 2, 3]], dtype=torch.int32), reset_optimizer=False)
    assert all(bool((getattr(t0, k) == 2.0).all()) for k in ("m_table", "v_table", "m_mlp", "v_mlp"))
    assert bool((t0.opt_state == 5.0).all())
    assert s1.face_counts.shape == (3,) and not hasattr(s1, "offsets")


@pytest.mark.parametrize("v,f", [
    (torch.rand(4, 2), torch.tensor([[0, 1, 2]])),                            # vertices not [V,3]
    (torch.rand(4, 3).int(), torch.tensor([[0, 1, 2]])),                      # integer vertices
    (torch.rand(4, 3), torch.tensor([[0.0, 1.0, 2.0]])),                      # float triangles
    (torch.rand(4, 3), torch.tensor([[True, False, True]])),                  # bool triangles
    (torch.rand(4, 3), torch.tensor([0, 1, 2])),                              # triangles not [F,3]
    (torch.rand(4, 3), torch.zeros(0, 3, dtype=torch.int64)),                 # F = 0
    (torch.rand(4, 3), torch.tensor([[0, 1, 4]])),                            # index past V
    (torch.rand(4, 3), torch.tensor([[0, -1, 2]])),                           # negative index
    (torch.tensor([[0.0, 0.0, float("nan")]] * 3), torch.tensor([[0, 1, 2]])),  # non-finite vertex
    (np.zeros((3, 3), np.float32), torch.tensor([[0, 1, 2]])),                # not a tensor
])
def test_replace_mesh_rejects_bad_input(mocked, v, f):
    s1 = mocked.make(antialias=True, lr_vert=1e-4, refine=True)
    before = (s1.vertices, s1.triangles, s1.face_errors)
    with pytest.raises(ValueError):
        s1.replace_mesh(v, f)
    assert (s1.vertices, s1.triangles, s1.face_errors) == before              # nothing was touched


def test_error_scatter_kernels_have_no_spills(tmp_path):
    src = os.path.join(B.CSRC, "stage1.cu")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "stage1.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    props = [i for i, l in enumerate(lines) if "Function properties for" in l and re.search(r"k_s1_loss(_aa)?ILb1E", l)]
    assert len(props) == 2, "\n".join(lines)
    for i in props:
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
        assert m and (int(m.group(2)), int(m.group(3))) == (0, 0), lines[i] + "\n" + lines[i + 1]
