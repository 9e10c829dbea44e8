"""CPU: per-image appearance codes (Stage0Config.ind_dim / ind_num) -- the float64 restatement on hand-built cases with written-out
answers, the host logic of Stage0Trainer with the CUDA layer mocked, and the compile budget of the new kernels."""
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import ind_codes_oracle as O
from nerf2mesh_b200 import build as B
from nerf2mesh_b200 import stage0 as S0
from nerf2mesh_b200.stage0 import Stage0Config


# ------------------------------------------------------------------------------------------------
# restatement, hand-built cases
# ------------------------------------------------------------------------------------------------
def test_gathered_code_columns_follow_the_record_ray():
    codes = np.array([[0.1, -2.0], [1.0 / 3.0, 65504.0 * 2]], np.float32)      # fp16: 0.0999755859375, -2, 0.333251953125, inf
    ray_img = np.array([1, 0, 1])
    rec_ray = np.array([0, 0, 1, 2, 2])
    with np.errstate(over="ignore"):
        got = O.gather_code_cols(codes, ray_img, rec_ray, 5, 2)
    c1 = [0.333251953125, np.inf]
    c0 = [0.0999755859375, -2.0]
    assert np.array_equal(got, np.array([c1, c1, c0, c1, c1]))
    assert np.array_equal(O.gather_code_cols(None, None, None, 2, 1, code_row=[0.1, 5.0]), [[0.0999755859375]] * 2)


def test_code_grad_one_ray():
    denc = np.array([[1.0, 2.0], [0.5, -1.0], [0.25, 0.0]])
    g = O.code_grad(denc, [[0, 3]], [2], ind_num=3, D=2, M=3)
    assert np.array_equal(g, [[0, 0], [0, 0], [1.75, 1.0]])
    # samples past the capacity M are not summed
    assert np.array_equal(O.code_grad(denc, [[0, 3]], [2], 3, 2, M=2)[2], [1.5, 1.0])


def test_code_grad_image_split_across_parts_and_empty_rays():
    # 8 rays, all of image 0 except ray 5 (image 1); rays 2 and 6 have no samples; one sample per ray elsewhere, denc = ray id
    rays = np.array([[0, 1], [1, 1], [2, 0], [2, 1], [3, 1], [4, 1], [5, 0], [5, 1]])
    denc = np.array([[0.0], [1.0], [3.0], [4.0], [5.0], [7.0]])
    img = np.array([0, 0, 0, 0, 0, 1, 0, 0])
    whole = O.code_grad(denc, rays, img, 2, 1, M=6)
    assert np.array_equal(whole, [[0 + 1 + 3 + 4 + 7], [5]])
    # two parts: rays 0-3 | 4-7 -- image 0 is split across the boundary, the parts add up to the whole
    p0 = O.code_grad(denc, rays, img, 2, 1, M=6, part=0, nparts=2)
    p1 = O.code_grad(denc, rays, img, 2, 1, M=6, part=1, nparts=2)
    assert np.array_equal(p0, [[0 + 1 + 3], [0]]) and np.array_equal(p1, [[4 + 7], [5]])
    assert np.array_equal(p0 + p1, whole)
    # eight parts: one ray each
    assert sum(O.code_grad(denc, rays, img, 2, 1, M=6, part=k, nparts=8) for k in range(8)).tolist() == whole.tolist()


def test_code_grad_ignores_rays_past_the_adaptive_count():
    rays = np.array([[0, 2], [2, 1], [3, 4]])
    denc = np.arange(7, dtype=np.float64)[:, None]
    img = [1, 1, 0]
    assert np.array_equal(O.code_grad(denc, rays, img, 2, 1, M=7, n_active=2), [[0], [0 + 1 + 2]])
    assert np.array_equal(O.code_grad(denc, rays, img, 2, 1, M=7), [[3 + 4 + 5 + 6], [3]])
    # parts of an adaptive batch cut its n rays, not the N rows: n = 2, two parts of one ray each
    assert np.array_equal(O.code_grad(denc, rays, img, 2, 1, M=7, n_active=2, part=1, nparts=2), [[0], [2]])


def test_two_group_adam_step():
    D = 1
    ind = np.zeros(64 + 2)
    g = np.zeros(66); g[0] = 2.0; g[64] = 2.0; g[65] = -4.0          # loss scale 2: unscaled 1, 1, -2
    new, m, v = O.adam_two_groups(ind, g, np.zeros(66), np.zeros(66), D, step=1, lr=1e-2, loss_scale=2.0, found_inf=False)
    # the first Adam step moves every parameter with a gradient by -lr * sign(g) (m / sqrt(v) = sign after bias correction)
    assert np.allclose(new[0], -1e-2) and np.allclose(new[64], -1e-3) and np.allclose(new[65], 1e-3)
    assert np.all(new[1:64] == 0)
    assert np.allclose(m[[0, 64, 65]], [0.1, 0.1, -0.2]) and np.allclose(v[[0, 64, 65]], [1e-3, 1e-3, 4e-3])
    skipped = O.adam_two_groups(ind, g, np.zeros(66), np.zeros(66), D, 1, 1e-2, 2.0, found_inf=True)
    assert all(np.all(a == 0) for a in skipped)


# ------------------------------------------------------------------------------------------------
# configuration
# ------------------------------------------------------------------------------------------------
def test_config_validates_code_width_and_count():
    assert Stage0Config().ind_dim == 0 and Stage0Config().ind_num == 500
    assert Stage0Config(ind_dim=10, ind_num=1).ind_dim == 10
    for bad in (dict(ind_dim=11), dict(ind_dim=-1), dict(ind_dim=4, ind_num=0), dict(ind_num=0)):
        with pytest.raises(ValueError):
            Stage0Config(**bad)


def test_data_parallel_paths_reject_codes():
    from nerf2mesh_b200 import parallel
    t = types.SimpleNamespace(ind_dim=4)
    for cls in (parallel.GradSync, parallel.PeerAdam, parallel.NvlsAdam):
        with pytest.raises(ValueError):
            cls(t)


# ------------------------------------------------------------------------------------------------
# Stage0Trainer host logic, CUDA layer mocked
# ------------------------------------------------------------------------------------------------
class _T:
    def zero_(self): return self
    def __getitem__(self, k): return self
    def data_ptr(self): return 0


class _Slot:
    def __init__(self):
        for k in ("rays_o", "rays_d", "gt", "bg", "noises", "rays", "counters", "tbuf", "recs", "cam_nf", "ray_img"):
            setattr(self, k, _T())
        self.has_alpha, self.loaded, self.index = True, 0, None

    def load(self, *a):
        self.loaded += 1

    def load_index(self, index):
        self.index = index


def _mock_trainer(monkeypatch, ind_dim, N=4, ind_num=8):
    calls = []
    monkeypatch.setattr(S0, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(S0, "ptr", lambda t: 0)
    monkeypatch.setattr(S0, "stream", lambda: 0)

    class FakeStream:
        def wait_stream(self, o): pass
        def wait_event(self, e): pass
        def synchronize(self): pass

    class FakeEvent:
        def record(self, s=None): pass

    class Ctx:
        def __init__(self, s): pass
        def __enter__(self): return self
        def __exit__(self, *a): return False

    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: FakeEvent())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: Ctx(s))
    tr = object.__new__(S0.Stage0Trainer)
    tr.cfg = types.SimpleNamespace(lambda_tv=0.0, eps=1e-15, num_levels=16)
    tr.slots, tr.cur = [_Slot(), _Slot()], 0
    for k in ("table", "offsets", "enc_tiles", "opt_state", "wpack", "out", "dout", "image", "weights_sum", "depth", "denc_tiles",
              "color_master", "m_table", "v_table", "mlp", "m_mlp", "v_mlp", "loss_acc", "m_ind", "v_ind", "aabb", "density_bitfield"):
        setattr(tr, k, _T())
    tr.ind = torch.zeros((64 + ind_num) * max(ind_dim, 1))
    tr.g_ind = torch.zeros_like(tr.ind)
    tr.ind_dim, tr.ind_num = ind_dim, ind_num
    tr.gtables, tr.g_mlps, tr.defer_zero, tr._zero_stream = [_T(), _T()], [_T()], False, None
    tr.params = S0.S0Params(); tr.params.shading_full = 1; tr.params.gt_has_alpha = 1; tr.params.ind_dim = ind_dim
    tr.Mcap, tr.N, tr.rows, tr.parity, tr.device = 128, N, 160, 0, "cpu"
    tr._tv_stream, tr._part_streams, tr._adam_stream = None, [], None
    tr.fused_fwd, tr.tv_fallback_points, tr._graphs, tr.nparts = False, 1000, {}, 1
    tr._prefetched, tr._side, tr._ev_march, tr._ev_done = None, None, [None, None], [None, None]
    tr.prefetch_at, tr.global_step, tr.use_cam_near_far = "optimizer", 0, False
    return tr, calls


def _batch(N=4):
    return (torch.zeros(N, 3), torch.ones(N, 3), torch.zeros(N, 4), torch.zeros(N, 3))


def test_index_required_with_codes_and_rejected_without(monkeypatch):
    tr, _ = _mock_trainer(monkeypatch, ind_dim=0)
    with pytest.raises(ValueError):
        tr.step(*_batch(), index=0, use_graph=False)
    tr.step(*_batch(), use_graph=False)
    tr, _ = _mock_trainer(monkeypatch, ind_dim=4)
    with pytest.raises(ValueError):
        tr.step(*_batch(), use_graph=False)
    with pytest.raises(ValueError):
        tr.step(*_batch(), index=3, next_batch=_batch(), use_graph=False)                 # next_batch without next_index
    with pytest.raises(ValueError):
        tr.step(*_batch(), index=3, grad_sync=lambda: None, use_graph=False)             # data parallel
    for bad in (8, -1, torch.tensor([0, 1, 8, 2], dtype=torch.int32), torch.tensor([0, 1, 2], dtype=torch.int32),
                torch.tensor([0, 1, 2, 3]), 1.0, True):
        with pytest.raises(ValueError):
            tr.step(*_batch(), index=bad, use_graph=False)
    tr.step(*_batch(), index=7, use_graph=False)
    assert tr.slots[0].index == 7


def test_index_travels_with_the_prefetched_batch(monkeypatch):
    tr, calls = _mock_trainer(monkeypatch, ind_dim=4)
    idx0 = torch.tensor([0, 1, 2, 3], dtype=torch.int32)
    idx1 = torch.tensor([4, 5, 6, 7], dtype=torch.int32)
    tr.step(*_batch(), index=idx0, next_batch=_batch(), next_index=idx1, use_graph=False)
    assert tr.slots[0].index is idx0 and tr.slots[1].index is idx1 and tr._prefetched == 1
    # the following step runs the prefetched slot: its index was staged with it, the call's own is not loaded again
    tr.step(*_batch(), index=idx1, use_graph=False)
    assert tr.cur == 1 and tr.slots[1].index is idx1 and tr.slots[1].loaded == 1
    names = calls
    assert names.count("n2m_s0_encode_fwd_codes") == 2 and "n2m_s0_encode_fwd" not in names
    assert names.count("n2m_s0_mlp_bwd_codes") == 2 and names.count("n2m_s0_code_grad") == 2
    # optimizer: the code block's inf scan before the head, its Adam after the MLP's (whose repack zeroes the code columns)
    assert names.index("n2m_s0_adam_codes_head") < names.index("n2m_s0_adam_head")
    assert names.index("n2m_s0_adam_mlp") < names.index("n2m_s0_adam_codes") < names.index("n2m_s0_adam_post")


def test_graph_replay_reads_the_staged_index(monkeypatch):
    """with use_graph the index is staged into the slot's persistent buffer before the replay, every step"""
    tr, calls = _mock_trainer(monkeypatch, ind_dim=2)
    replays = []

    class G:
        def replay(self): replays.append(tr.slots[tr.cur].index)

    monkeypatch.setattr(S0.Stage0Trainer, "_graph", lambda self, name, fn: G())
    for k in range(3):
        idx = torch.full((4,), k, dtype=torch.int32)
        tr.step(*_batch(), index=idx, use_graph=True)
        assert replays[-1] is idx and tr.slots[tr.cur].index is idx


def test_without_codes_the_call_sequence_is_unchanged(monkeypatch):
    tr, calls = _mock_trainer(monkeypatch, ind_dim=0)
    tr.step(*_batch(), use_graph=False)
    assert not [n for n in calls if n.endswith("_codes") or "code_grad" in n or "codes_" in n]
    assert calls == ["n2m_s0_march", "n2m_s0_encode_fwd", "n2m_s0_mlp_fwd", "n2m_s0_composite_loss", "n2m_s0_mlp_bwd",
                     "n2m_s0_encode_bwd", "n2m_s0_adam_head", "n2m_s0_adam_mlp", "n2m_s0_adam_tables", "n2m_s0_adam_post"]


def test_state_dict_layout_of_the_code_block():
    tr = object.__new__(S0.Stage0Trainer)
    D, K = 3, 5
    tr.ind_dim, tr.ind_num = D, K
    ind = torch.arange((64 + K) * D, dtype=torch.float32)
    out = tr._with_codes({"color_net.net.0.weight": torch.zeros(64, 35)}, ind)
    assert out["color_net.net.0.weight"].shape == (64, 35 + D) and out["individual_codes"].shape == (K, D)
    assert out["color_net.net.0.weight"][2, 35 + 1] == 2 * D + 1
    assert out["individual_codes"][1, 2] == 64 * D + 1 * D + 2


def test_params_struct_carries_ind_dim():
    assert S0.S0Params._fields_[-1][0] == "ind_dim"


# ------------------------------------------------------------------------------------------------
# compile budget
# ------------------------------------------------------------------------------------------------
def _ptxas(tmp_path, name):
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.CSRC, name), "-o", str(tmp_path / (name + ".o"))],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return (r.stdout + r.stderr).splitlines()


def _spills(lines, kernel):
    props = [i for i, l in enumerate(lines) if "Function properties for" in l and kernel in l]
    assert len(props) == 1, (kernel, "\n".join(lines[-40:]))
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", lines[props[0] + 1])
    assert m, lines[props[0] + 1]
    return int(m.group(1)), int(m.group(2))


@pytest.mark.parametrize("src,kernels", [
    ("stage0.cu", ["k_s0_code_gradEj", "k_s0_code_grad_row", "k_s0_encode_fwdILb0ELb1E", "k_s0_encode_fwdILb1ELb1E"]),
    ("mlp_tc.cu", ["k_pack_code_weights", "k_mlp_bwd"]),
    ("optim.cu", ["k_adam_codesEPfS1", "k_adam_codes_head", "k_codes_ema"]),
])
def test_code_kernels_compile_without_spills(tmp_path, src, kernels):
    lines = _ptxas(tmp_path, src)
    for k in kernels:
        assert _spills(lines, k) == (0, 0), k


def test_fused_forward_with_codes_spills_no_more_than_without(tmp_path):
    """k_s0_fwd_fused runs at 80 registers per thread and spills a little without codes already; the code columns, written after the
    level walk, must not add to it"""
    lines = _ptxas(tmp_path, "fused.cu")
    with_codes, without = _spills(lines, "k_s0_fwd_fusedILb1E"), _spills(lines, "k_s0_fwd_fusedILb0E")
    assert with_codes[0] <= without[0] and with_codes[1] <= without[1], (with_codes, without)
