"""GPU: stage-1 mesh refinement (Stage1Trainer(refine=True), csrc/stage1.cu's error-scattering loss kernels, refine_mask, replace_mesh).

The per-face accumulators are checked against a torch restatement of the reference's update_triangles_errors (nerf/renderer.py:893-903,
923-943): trig_id = rast[0, ::ssaa, ::ssaa, 3] - 1 (the nearest-neighbour minification of the triangle ids), the per-pixel loss rebuilt from
the step's image / weights_sum / gt / bg (utils.py:713-718), scatter-add of the loss and of ones over the covered pixels."""
import numpy as np
import pytest
import torch

from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200.stage1 import Stage1Trainer
from nerf2mesh_b200.train_synthetic import full_image_rays
from oracle import raster_oracle as R
from test_gpu_stage1 import _setup

pytestmark = pytest.mark.gpu

T0_STATE = ["table", "color_master", "mlp", "m_table", "v_table", "m_mlp", "v_mlp", "wpack", "opt_state", "g_mlp"]


def _views(h0, w0, gt_channels, seed=1):
    """three device-resident views of the sphere (the camera of test_gpu_stage1._setup and two more around it)"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for cam in (np.array([1.5, 1.1, 0.9]) * 1.6, np.array([-1.2, 1.4, 1.0]) * 1.6, np.array([0.4, -1.6, 1.2]) * 1.6):
        pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
        intr = S.lego_intrinsics(h0, w0)
        _, rays_d = full_image_rays(pose, intr, h0, w0)
        mvp = R.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0)
        mvp[1] *= -1
        gt = torch.rand(h0 * w0, 4, generator=g); gt[:, 3] = (gt[:, 3] > 0.5).float()
        bg = torch.rand(h0 * w0, 3, generator=g)
        out.append((torch.from_numpy(mvp).cuda(), rays_d.cuda().contiguous(), gt[:, :gt_channels].contiguous().cuda(), bg.cuda()))
    return out


def _restated_update(s1, gt, bg, errors, counts):
    """update_triangles_errors of the step just taken, accumulated into float64 errors / counts"""
    trig_id = (s1.rast[0, ::s1.ssaa, ::s1.ssaa, 3] - 1).reshape(-1).long()
    image, ws = s1.image.double(), s1.weights_sum.double()
    gt, bg = gt.double(), bg.double()
    if gt.shape[-1] == 4:
        m = gt[:, 3]
        gt_rgb = gt[:, :3] * m[:, None] + bg * (1 - m[:, None])
        loss = ((image - gt_rgb) ** 2).mean(-1) + s1.lambda_mask * (ws - m) ** 2
    else:
        loss = ((image - gt) ** 2).mean(-1)
    keep = trig_id >= 0
    errors.index_add_(0, trig_id[keep], loss[keep])
    counts.index_add_(0, trig_id[keep], torch.ones_like(loss[keep]))


def _snapshot(t0):
    snap = {n: getattr(t0, n).clone() for n in T0_STATE}
    snap_g = [g.clone() for g in t0.gtables]

    def restore():
        for n in T0_STATE:
            getattr(t0, n).copy_(snap[n])
        for g, s in zip(t0.gtables, snap_g):
            g.copy_(s)
    return restore


ORDER = [0, 1, 2, 0, 1, 2]


@pytest.mark.parametrize("gt_channels", [3, 4])
@pytest.mark.parametrize("ssaa,antialias", [(1, False), (2, False), (1, True), (2, True)])
def test_face_errors_match_update_triangles_errors(ssaa, antialias, gt_channels):
    t0, s1, *_ = _setup(ssaa=ssaa, antialias=antialias, subdiv=3, steps=8, refine=True)
    views = _views(s1.h0, s1.w0, gt_channels)
    Fn = s1.triangles.shape[0]
    restore = _snapshot(t0)
    errors = torch.zeros(Fn, dtype=torch.float64, device="cuda"); counts = torch.zeros_like(errors)
    for k in ORDER:                                                      # eager steps, restatement read after each
        s1.step(*views[k])
        _restated_update(s1, views[k][2], views[k][3], errors, counts)
    torch.cuda.synchronize()
    assert counts.sum().item() > 0.1 * s1.h0 * s1.w0 * len(ORDER) and (counts > 0).sum().item() > 0.2 * Fn
    assert torch.equal(s1.face_counts.double(), counts)
    assert torch.allclose(s1.face_errors.double(), errors, rtol=1e-5, atol=1e-6), (s1.face_errors.double() - errors).abs().max().item()
    assert s1.refine_mask()[0].eq(2).any()
    eager_err, eager_cnt = s1.face_errors.clone(), s1.face_counts.clone()
    # the same steps replayed as per-view CUDA graphs (first step eager, then captures, then pure replays)
    restore()
    s1.face_errors.zero_(); s1.face_counts.zero_()
    for k in ORDER:
        s1.step(*views[k], use_graph=True)
    torch.cuda.synchronize()
    assert len(s1._graphs) == 3
    assert torch.equal(s1.face_counts, eager_cnt)
    assert torch.allclose(s1.face_errors, eager_err, rtol=1e-4, atol=1e-6), (s1.face_errors - eager_err).abs().max().item()


@pytest.mark.parametrize("antialias", [False, True])
def test_refine_off_step_unchanged_by_refine_on(antialias):
    """the error scatter leaves the step itself alone: image, weights_sum and the loss equal the refine-off step's (up to the order of
    the fp32 atomics of antialias and of the loss sum)"""
    t0, s1, *_ = _setup(ssaa=2, antialias=antialias, subdiv=3, steps=8, refine=True)
    off = Stage1Trainer(t0, s1.vertices, s1.triangles, s1.h0, s1.w0, ssaa=2, antialias=antialias)
    mvp, rays_d, gt, bg = _views(s1.h0, s1.w0, 4)[0]
    for tr in (s1, off):
        tr.forward(mvp, rays_d); tr.loss_backward(gt, bg)
    torch.cuda.synchronize()
    assert (s1.image - off.image).abs().max().item() <= 1e-6 and (s1.weights_sum - off.weights_sum).abs().max().item() <= 1e-6
    assert abs(s1.read_loss() - off.read_loss()) <= 1e-6 * abs(off.read_loss())
    assert s1.face_counts.sum().item() > 0


def _split_refined(v, f, mask):
    """1 -> 3 centroid split of the mask-2 faces: face (a, b, c) keeps its slot as (a, b, m); (b, c, m) and (c, a, m) are appended"""
    sel = np.nonzero(mask == 2)[0]
    m = v.shape[0] + np.arange(len(sel))
    v2 = np.concatenate([v, v[f[sel]].mean(1)]).astype(np.float32)
    f2 = f.copy()
    a, b, c = f[sel, 0], f[sel, 1], f[sel, 2]
    f2[sel] = np.stack([a, b, m], 1)
    f2 = np.concatenate([f2, np.stack([b, c, m], 1), np.stack([c, a, m], 1)]).astype(np.int32)
    return v2, f2


@pytest.mark.parametrize("lr_vert", [0.0, 1e-4])
def test_replace_mesh_then_graph_steps_render_the_new_mesh(lr_vert):
    kw = dict(ssaa=2, antialias=True, lr_vert=lr_vert, refine=True)
    t0, s1, *_ = _setup(subdiv=3, steps=8, **kw)
    views = _views(s1.h0, s1.w0, 4)
    for k in ORDER:
        s1.step(*views[k], use_graph=True)
    assert len(s1._graphs) == 3
    old_F = s1.triangles.shape[0]
    mask, (t_ref, t_dec) = s1.refine_mask()
    assert t_ref >= t_dec and mask.eq(2).sum().item() > 0 and mask.eq(1).sum().item() > 0
    v2, f2 = _split_refined(s1.vertices.cpu().numpy(), s1.triangles.cpu().numpy(), mask.cpu().numpy())
    s1.replace_mesh(torch.from_numpy(v2), torch.from_numpy(f2))
    new_F = f2.shape[0]
    assert new_F > old_F and s1.face_counts.shape == (new_F,) and s1._graphs == {}
    assert t0.opt_state[2].item() == 0 and t0.m_mlp.abs().max().item() == 0
    restore = _snapshot(t0)                                              # the state a fresh trainer starts from
    seq = [0, 1, 0, 1, 0]                                                # eager, capture 1, capture 0, replay 1, replay 0
    for k in seq:
        s1.step(*views[k], use_graph=True)
    torch.cuda.synchronize()
    ids = s1.rast[0, ..., 3]
    assert (ids > old_F).any() and ids.max().item() <= new_F                 # face ids >= old F: the new mesh was rendered
    assert s1.face_counts.shape == (new_F,) and s1.face_counts[old_F:].sum().item() > 0
    if lr_vert > 0:
        # the vertex group restarted on the new vertices: its step count follows the restarted shared one; no exact comparison below,
        # because Adam's first steps turn the summation-order noise of near-zero gradient components into +-lr_vert moves
        assert s1.offsets.shape == (v2.shape[0], 3) and s1.offsets.abs().max().item() > 0 and torch.isfinite(s1.vertices).all()
        assert s1.vert_state[0].item() == t0.opt_state[2].item() > 0
        assert torch.equal(s1.vertices, s1.base_vertices + s1.offsets) and torch.equal(s1.base_vertices.cpu(), torch.from_numpy(v2))
        return
    loss, image, counts = s1.read_loss(), s1.image.clone(), s1.face_counts.clone()
    # a trainer built fresh on the new mesh from the same model state (zeroed moments)
    restore()
    fresh = Stage1Trainer(t0, torch.from_numpy(v2), torch.from_numpy(f2), s1.h0, s1.w0, **kw)
    for k in seq:
        fresh.step(*views[k], use_graph=True)
    torch.cuda.synchronize()
    assert torch.equal(fresh.face_counts, counts)
    assert (fresh.image - image).abs().max().item() <= 2e-3
    assert abs(fresh.read_loss() - loss) <= 1e-3 * abs(loss)
