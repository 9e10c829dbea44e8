"""GPU: stage-1 evaluation -- Stage1Trainer.render (render_stage1 at inference, nerf/renderer.py:816-921) against the training step's
own image, the reference model and the numpy compose oracle; texture.render_exported (the viewer's fragment shader, renderer.html:54-160)
against the numpy shading oracle; the export -> load round trip; and the distance between the two renderers."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import stage1_render_oracle as O
import texture_oracle as TO
from nerf2mesh_b200 import raster as dr
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200 import texture as X
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage1 import Stage1Trainer
from nerf2mesh_b200.train_synthetic import full_image_rays
from oracle import raster_oracle as R
from test_gpu_stage1 import _setup

pytestmark = pytest.mark.gpu

CAM = np.array([1.5, 1.1, 0.9]) * 1.6            # the camera of test_gpu_stage1._setup


def _view(h0, w0, cam=CAM):
    pose = torch.from_numpy(S.look_at_pose(cam).astype(np.float32))
    intr = S.lego_intrinsics(h0, w0)
    _, rays_d = full_image_rays(pose, intr, h0, w0)
    mvp = R.perspective_mvp(cam, fovy=2 * np.arctan(0.5 * h0 / intr[1]), aspect=w0 / h0)
    mvp[1] *= -1
    return torch.from_numpy(np.ascontiguousarray(mvp, np.float32)).cuda(), rays_d.cuda().contiguous()


def _oracle_depth(s1, alpha, bg):
    img = torch.zeros(s1.h * s1.w, 4, device="cuda")
    img[:, 3] = alpha
    return O.compose(img.cpu().numpy(), s1.rast[0, ..., 2].reshape(-1).cpu().numpy(), bg.cpu().numpy(), s1.h0, s1.w0, s1.ssaa)[2]


@pytest.mark.parametrize("ssaa,antialias", [(1, False), (2, False), (1, True), (2, True)])
def test_render_is_the_step_image(ssaa, antialias):
    """render(bg) gives the image and weights_sum the step's loss kernel writes for the same view, depth = the compose oracle on the
    step's rast and alpha"""
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=ssaa, antialias=antialias, subdiv=2 if antialias else 4, steps=8)
    mvp = mvp.cuda()
    s1.forward(mvp, rays_d)
    s1.loss_backward(gt, bg)
    image, ws, depth = s1.render(mvp, rays_d, bg_color=bg, antialias=antialias)
    torch.cuda.synchronize()
    assert image.shape == (s1.h0 * s1.w0, 3) and ws.shape == depth.shape == (s1.h0 * s1.w0,)
    assert (ws > 0).float().mean().item() > 0.1
    if antialias:
        # the compose kernel on the step's antialiased image: the loss kernel's bits
        img2 = torch.empty_like(image); ws2 = torch.empty_like(ws); d2 = torch.empty_like(depth)
        call("n2m_s1_render_compose", ptr(s1.aa), ptr(s1.rast), ptr(bg), s1.h0, s1.w0, ssaa, ptr(img2), ptr(ws2), ptr(d2), stream())
        torch.cuda.synchronize()
        assert torch.equal(img2, s1.image) and torch.equal(ws2, s1.weights_sum) and torch.equal(d2, depth)
        # end to end, the antialias forward adds the silhouette blends with fp32 atomics: a pixel that receives two of them may differ in
        # the last bit between two launches
        assert (image - s1.image).abs().max().item() <= 1e-6 and (ws - s1.weights_sum).abs().max().item() <= 1e-6
        alpha = s1.aa[:, 3]
    else:
        assert torch.equal(image, s1.image) and torch.equal(ws, s1.weights_sum)
        alpha = (s1.inv >= 0).float()
    assert np.abs(depth.cpu().numpy() - _oracle_depth(s1, alpha, bg)).max() <= 1e-6


def _reference_render(ns, ref_stage, t0, s1, mvp, rays_d, bg, shading):
    """render_stage1 in eval (renderer.py:816-921) with the unmodified reference model; this repo's rasterize / interpolate / antialias
    stand in for nvdiffrast as in test_gpu_stage1"""
    opt = ref_stage.default_opt(bound=1.0, dt_gamma=0.0, adaptive_num_rays=False)
    model = ns.make_model(opt)
    model.load_state_dict(t0.export_reference_state(), strict=True)
    model.cuda().eval()
    h0, w0, ssaa = s1.h0, s1.w0, s1.ssaa
    h, w = h0 * ssaa, w0 * ssaa
    dirs = rays_d.view(h0, w0, 3)
    dirs = F.interpolate(dirs.permute(2, 0, 1)[None], (h, w), mode="nearest")[0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    dirs = dirs / torch.sqrt(torch.clamp((dirs * dirs).sum(-1, keepdim=True), min=1e-20))
    vertices = s1.vertices
    vclip = torch.matmul(F.pad(vertices, pad=(0, 1), mode="constant", value=1.0), torch.transpose(mvp, 0, 1)).float().unsqueeze(0)
    rast, _ = dr.rasterize(dr.RasterizeCudaContext(), vclip, s1.triangles, (h, w))
    xyzs, _ = dr.interpolate(vertices.unsqueeze(0), rast, s1.triangles)
    mask, _ = dr.interpolate(torch.ones_like(vertices[:, :1]).unsqueeze(0), rast, s1.triangles)
    mask_flatten = (mask > 0).view(-1)
    xyzs = xyzs.view(-1, 3)
    rgbs = torch.zeros(h * w, 3, device="cuda", dtype=torch.float32)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        mask_rgbs, _ = model.rgb(xyzs[mask_flatten], dirs[mask_flatten], None, shading)
    rgbs[mask_flatten] = mask_rgbs.float()
    rgbs = rgbs.view(1, h, w, 3)
    alphas = dr.antialias(mask.float(), rast, vclip, s1.triangles).squeeze(0).clamp(0, 1)
    rgbs = dr.antialias(rgbs, rast, vclip, s1.triangles).squeeze(0).clamp(0, 1)
    image = alphas * rgbs
    depth = alphas * rast[0, :, :, [2]]
    T = 1 - alphas

    def down(x):
        return F.interpolate(x.permute(2, 0, 1)[None], (h0, w0), mode="bilinear")[0].permute(1, 2, 0).contiguous()

    if ssaa > 1:
        image, depth, T = down(image), down(depth), down(T)
    image = image + T * bg.view(h0, w0, 3)
    return image.view(-1, 3), (1 - T).view(-1), depth.view(-1)


@pytest.mark.parametrize("shading", ["diffuse", "specular", "full"])
def test_render_matches_reference_render_stage1(shading):
    from oracle import ref_stage
    if not ref_stage.staged():
        pytest.skip("reference Python files not staged")
    ns = ref_stage.load("ref")
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, antialias=False)          # render builds its own edge hash
    mvp = mvp.cuda()
    ri, rw, rd = _reference_render(ns, ref_stage, t0, s1, mvp, rays_d, bg, shading)
    image, ws, depth = s1.render(mvp, rays_d, bg_color=bg, shading=shading)
    torch.cuda.synchronize()
    assert (ws > 0).float().mean().item() > 0.1
    assert (image - ri).abs().max().item() <= 2e-3, (image - ri).abs().max().item()
    assert (ws - rw).abs().max().item() <= 1e-5 and (depth - rd).abs().max().item() <= 1e-5


def _state(t0):
    names = ["table", "color_master", "mlp", "m_table", "v_table", "m_mlp", "v_mlp", "wpack", "opt_state", "g_mlp"]
    return {n: getattr(t0, n).clone() for n in names}, [g.clone() for g in t0.gtables]


def _restore(t0, snap):
    for n, v in snap[0].items():
        getattr(t0, n).copy_(v)
    for g, s in zip(t0.gtables, snap[1]):
        g.copy_(s)


def test_render_leaves_training_untouched():
    """render at the training and at another resolution between steps: the step's buffers, the optimizer state and the captured graphs
    are untouched, and the next step (eager or graph-replayed) computes what it computes without the render"""
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, steps=8)
    mvp = mvp.cuda()
    mvp2, rays_d2 = _view(72, 120)
    s1.step(mvp, rays_d, gt, bg)                        # warm-up
    torch.cuda.synchronize()
    bufs = ["out", "inv", "rast", "image", "weights_sum", "loss_acc", "dout", "counters", "pts", "enc_tiles"]
    before = {n: getattr(s1, n).clone() for n in bufs}
    st = _state(t0)
    s1.render(mvp, rays_d, bg_color=bg)
    img2, ws2, _ = s1.render(mvp2, rays_d2, h0=72, w0=120, shading="specular")
    torch.cuda.synchronize()
    assert img2.shape == (72 * 120, 3) and (ws2 > 0).any()
    for n in bufs:
        assert torch.equal(getattr(s1, n), before[n]), n
    after = _state(t0)
    assert all(torch.equal(a, b) for a, b in zip(after[0].values(), st[0].values())) and all(torch.equal(a, b) for a, b in zip(after[1], st[1]))
    # the next step, eager: without and with a render before it
    out = {}
    for with_render in (False, True):
        _restore(t0, st)
        if with_render:
            s1.render(mvp2, rays_d2, h0=72, w0=120)
        s1.step(mvp, rays_d, gt, bg)
        torch.cuda.synchronize()
        out[with_render] = (s1.image.clone(), s1.weights_sum.clone(), t0.mlp.clone(), t0.opt_state.clone())
    assert torch.equal(out[False][0], out[True][0]) and torch.equal(out[False][1], out[True][1])
    for a, b in zip(out[False][2:], out[True][2:]):          # the scatter's fp32 atomics: parameters up to their order
        assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())
    # graph-replayed: capture, then a render at another resolution, then the same graph again
    _restore(t0, st)
    s1.step(mvp, rays_d, gt, bg, use_graph=True)
    torch.cuda.synchronize()
    g_img = s1.image.clone()
    _restore(t0, st)
    s1.render(*_view(144, 240), h0=144, w0=240)
    s1.step(mvp, rays_d, gt, bg, use_graph=True)
    torch.cuda.synchronize()
    assert len(s1._graphs) == 1 and torch.equal(s1.image, g_img) and torch.equal(g_img, out[False][0])


def test_render_cascades_with_contract():
    from test_gpu_cascades import _bound4_trainer, _cascade_meshes, _views
    t0 = _bound4_trainer(contract=True)
    vs, fs = _cascade_meshes()
    s1 = Stage1Trainer(t0, vs, fs, 48, 48, ssaa=2)
    mvp, rays_d, gt, bg = _views(48, 48)[0]
    s1.forward(mvp, rays_d)
    s1.loss_backward(gt, bg)
    image, ws, depth = s1.render(mvp, rays_d, bg_color=bg, antialias=False)
    torch.cuda.synchronize()
    ids = s1.rast[0, ..., 3]
    assert all(((ids > s1.f_cumsum[c]) & (ids <= s1.f_cumsum[c + 1])).any() for c in range(3))
    assert torch.equal(image, s1.image) and torch.equal(ws, s1.weights_sum)
    image_aa, ws_aa, _ = s1.render(mvp, rays_d, bg_color=bg)
    assert torch.isfinite(image_aa).all() and (image_aa - image).abs().max().item() > 0      # the cascades' silhouettes blend


def _two_cascade_asset(seed=0):
    """two spheres side by side, grid atlases, random textures of different sizes, random specular weights"""
    rng = np.random.default_rng(seed)
    meshes = [S.icosphere(2, 0.6), S.icosphere(1, 0.5)]
    vs, fs, sts, fts = [], [], [], []
    for (v, f), dx in zip(meshes, (-0.7, 0.7)):
        vs.append(np.asarray(v, np.float32) + np.float32([dx, 0, 0])); fs.append(np.asarray(f, np.int32))
        vt, ft = TO.grid_atlas(f.shape[0])
        sts.append(np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], 1).astype(np.float32)); fts.append(ft)
    f0 = [rng.integers(0, 256, (64, 64, 3), dtype=np.uint8), rng.integers(0, 256, (32, 48, 3), dtype=np.uint8)]
    f1 = [rng.integers(0, 256, (64, 64, 3), dtype=np.uint8), rng.integers(0, 256, (32, 48, 3), dtype=np.uint8)]
    w = {"net.0.weight": (rng.standard_normal((32, 6)) * 0.5).astype(np.float32), "net.1.weight": (rng.standard_normal((3, 32)) * 0.5).astype(np.float32)}
    return X.ExportedMesh(vs, fs, sts, fts, f0, f1, w)


@pytest.mark.parametrize("ssaa", [1, 2])
@pytest.mark.parametrize("shading", ["diffuse", "specular", "full"])
def test_asset_shade_matches_the_numpy_oracle(ssaa, shading):
    asset = _two_cascade_asset()
    cam = np.array([0.2, 0.5, 2.6])
    h0 = w0 = 48
    mvp, _ = _view(h0, w0, cam)
    bg = torch.rand(h0 * w0, 3, generator=torch.Generator().manual_seed(1)).cuda()
    image, ws, depth = X.render_exported(asset, mvp, cam, h0, w0, ssaa=ssaa, bg_color=bg, shading=shading)
    vclip = (F.pad(asset.vertices, (0, 1), value=1.0) @ mvp.T).contiguous()
    rast, _ = dr.rasterize(dr.RasterizeCudaContext(), vclip[None], asset.triangles, (h0 * ssaa, w0 * ssaa))
    torch.cuda.synchronize()
    rast = rast.reshape(-1, 4).cpu().numpy()
    ids = rast[:, 3]
    assert ((ids > 0) & (ids <= asset.face_offsets[1])).sum() > 50 and (ids > asset.face_offsets[1]).sum() > 50     # both cascades seen
    img = O.asset_shade(rast, asset.vertices.cpu().numpy(), asset.triangles.cpu().numpy(), asset.st.cpu().numpy(), asset.ft.cpu().numpy(),
                        asset.face_offsets, [t.cpu().numpy() for t in asset.feat0], [t.cpu().numpy() for t in asset.feat1],
                        asset.weights["net.0.weight"], asset.weights["net.1.weight"], cam, X.SHADE_MODES[shading])
    ri, rw, rd = O.compose(img, rast[:, 2], bg.cpu().numpy(), h0, w0, ssaa)
    assert np.abs(image.cpu().numpy() - ri).max() <= 1e-5
    assert np.abs(ws.cpu().numpy() - rw).max() <= 1e-6 and np.abs(depth.cpu().numpy() - rd).max() <= 1e-6
    # antialiased: the same samples, blended at the silhouettes
    image_aa, ws_aa, _ = X.render_exported(asset, mvp, cam, h0, w0, ssaa=ssaa, bg_color=bg, shading=shading, antialias=True)
    assert torch.isfinite(image_aa).all() and (ws_aa - ws).abs().max().item() > 0


def test_export_then_load_gives_the_in_memory_asset(tmp_path):
    import cv2
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2, subdiv=2, steps=8)
    v, f = s1.cascade_mesh(0)
    vt, ft = TO.grid_atlas(f.shape[0])
    vt, ft = torch.from_numpy(vt).cuda(), torch.from_numpy(ft).cuda()
    feats = X.export_stage1(s1, str(tmp_path), vt, ft, resolution=128)
    a = X.load_exported(str(tmp_path))
    b = X.ExportedMesh.from_export(s1, vt, ft, feats)
    for n in ("vertices", "triangles", "st", "ft"):
        assert torch.equal(getattr(a, n), getattr(b, n)), n
    assert a.face_offsets == b.face_offsets == [0, f.shape[0]] and a.bound == b.bound
    for k in b.weights:
        assert np.array_equal(a.weights[k], b.weights[k])
    for name, tex, mem in (("feat0_0.jpg", a.feat0[0], feats[0]), ("feat1_0.jpg", a.feat1[0], feats[1])):
        assert np.array_equal(tex.cpu().numpy(), cv2.imread(os.path.join(tmp_path, name))[..., ::-1])
        assert np.abs(tex.cpu().numpy().astype(np.int32) - mem.cpu().numpy().astype(np.int32)).mean() < 8      # JPEG is lossy
    ia, wa, _ = X.render_exported(a, mvp.cuda(), CAM, s1.h0, s1.w0)
    ib, wb, _ = X.render_exported(b, mvp.cuda(), CAM, s1.h0, s1.w0)
    torch.cuda.synchronize()
    assert torch.equal(wa, wb) and (wa > 0).any() and (ia - ib).abs().mean().item() < 8 / 255


def test_baked_asset_is_close_to_the_neural_render():
    """A 2048^2 bake of the _setup sphere rendered as the viewer does, against render_stage1 ('diffuse', ssaa 2, antialiased), over the
    pixels both cover fully: the mean |difference| is bounded by the bake's losses -- the 1/255 truncation of the features, the 2x
    down-sample and the nearest texel on a smooth field: 4/255 (a reasoned bound).  Measured on an H100 80GB HBM3 (700 W power limit):
    0.217/255 over 1844 pixels."""
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2)
    mvp = mvp.cuda()
    v, f = s1.cascade_mesh(0)
    vt, ft = TO.grid_atlas(f.shape[0])
    vt, ft = torch.from_numpy(vt).cuda(), torch.from_numpy(ft).cuda()
    feats = X.bake_features(t0, v, f, vt, ft, 2048, 2048, ssaa=2)
    asset = X.ExportedMesh.from_export(s1, vt, ft, feats)
    ia, wa, _ = X.render_exported(asset, mvp, CAM, s1.h0, s1.w0, ssaa=2, shading="diffuse", antialias=True)
    ineu, wn, _ = s1.render(mvp, rays_d, shading="diffuse")
    torch.cuda.synchronize()
    both = (wa == 1) & (wn == 1)
    assert both.float().mean().item() > 0.1
    err = (ia[both] - ineu[both]).abs().mean().item()
    print(f"mean |asset - neural| over {int(both.sum())} pixels: {err * 255:.3f}/255")
    assert err <= 4 / 255, err * 255
