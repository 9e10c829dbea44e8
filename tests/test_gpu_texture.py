"""GPU: the stage-1 texture export (nerf2mesh_b200/texture.py over csrc/texture.cu) -- geo_feat bit-identical to the forward MLP kernel
and within the stage-1 bound of the UNMODIFIED reference model's `geo_feat` under fp16 autocast, the UV raster / positions / band split,
the inpaint against the reference's scipy + KD-tree post-processing (tests/texture_oracle.py), the down-sample, the files of
export_stage1, and a 4096-texel, ssaa-2 bake of a 327,680-face mesh."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import texture_oracle as O
from nerf2mesh_b200 import raster as dr
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200 import texture as X
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer

pytestmark = pytest.mark.gpu


def _trained(steps=20):
    N = 1024
    t0 = Stage0Trainer(Stage0Config(bound=1.0, num_rays=N, max_samples=N * 256), seed=5)
    grid, bits, bricks = S.occupancy_regime("converged")
    t0.set_occupancy(bits, grid)
    g = torch.Generator().manual_seed(0)
    poses = S.orbit_cameras(100, seed=0)
    for _ in range(steps):       # non-trivial colour parameters
        ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, N, g)
        t0.step(ro, rd, S.render_bricks(ro, rd, bricks), torch.rand(N, 3, generator=g), torch.rand(N, generator=g), use_graph=False)
    torch.cuda.synchronize()
    return t0


@pytest.fixture(scope="module")
def t0():
    return _trained()


def _mesh(subdiv):
    v, f = S.icosphere(subdiv)
    vt, ft = O.grid_atlas(f.shape[0])
    return (torch.from_numpy(np.asarray(v, np.float32)).cuda(), torch.from_numpy(np.asarray(f, np.int32)).cuda(),
            torch.from_numpy(vt).cuda(), torch.from_numpy(ft).cuda())


def _bake_one_band(t0, v, f, vt, ft, h, w):
    rast = X.uv_raster(vt, ft, h, w)
    baker = X.Baker(t0, h * w)
    feats = torch.zeros(h, w, 6, dtype=torch.uint8, device="cuda")
    f32 = torch.zeros(baker.cap, 6, device="cuda")
    baker.band(rast, v, f, w, 0, h, feats, feats_f32=f32)
    torch.cuda.synchronize()
    M = int(baker.counters[1].item())
    return rast, baker, feats, f32, M


def test_geo_feat_is_bit_identical_to_the_forward_kernel(t0):
    P = 1000                                  # not a multiple of 128
    g = torch.Generator(device="cuda").manual_seed(1)
    pts = torch.rand(P, 3, device="cuda", generator=g) * 1.8 - 0.9
    baker = X.Baker(t0, P)
    baker.pts[:P] = pts
    baker.pix[:P] = torch.arange(P, dtype=torch.int32, device="cuda")
    baker.counters.zero_(); baker.counters[1] = P
    params = t0.params_with(shading_full=0)
    call("n2m_s0_encode_points", ctypes.byref(params), ptr(baker.pts), None, ptr(baker.counters), baker.cap, ptr(t0.table), ptr(t0.offsets),
         ptr(baker.enc_tiles), stream())
    feats = torch.zeros(P, 6, dtype=torch.uint8, device="cuda")
    f32 = torch.full((baker.cap, 6), -1.0, device="cuda")
    call("n2m_s1_geo_feat", ptr(baker.enc_tiles), ptr(baker.counters), baker.cap, ptr(t0.wpack), ptr(baker.pix), ptr(feats), ptr(f32), stream())
    out = torch.zeros(baker.cap, 4, device="cuda")
    call("n2m_s0_mlp_fwd", ctypes.byref(params), ptr(baker.enc_tiles), ptr(baker.counters), baker.cap, ptr(t0.wpack), ptr(out), None, 0, 1,
         stream())
    torch.cuda.synchronize()
    assert torch.equal(f32[:P, :3], out[:P, 1:4])
    assert (f32[P:] == -1.0).all()                                     # rows past the count are not written
    quantised = (f32[:P].cpu().numpy() * np.float32(255)).astype(np.uint8)             # (feats * 255).astype(np.uint8)
    assert np.array_equal(feats.cpu().numpy(), quantised)
    assert f32[:P, 3:].std().item() > 1e-3                            # the specular features vary


def test_geo_feat_matches_reference_model(t0):
    from oracle import ref_stage
    if not ref_stage.staged():
        pytest.skip("reference Python files not staged")
    ns = ref_stage.load("ref")
    model = ns.make_model(ref_stage.default_opt(bound=1.0, dt_gamma=0.0, adaptive_num_rays=False))
    model.load_state_dict(t0.export_reference_state(), strict=True)
    model.cuda().eval()
    v, f, vt, ft = _mesh(3)
    rast, baker, feats, f32, M = _bake_one_band(t0, v, f, vt, ft, 256, 256)
    assert M > 10000
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        ref = model.geo_feat(baker.pts[:M].clone()).float()
    assert (ref - f32[:M]).abs().max().item() <= 2e-3
    q_ref = (ref.cpu().numpy() * np.float32(255)).astype(np.uint8).astype(np.int32)
    ours = feats.view(-1, 6)[baker.pix[:M].long()].cpu().numpy().astype(np.int32)
    assert np.abs(q_ref - ours).max() <= 1


def test_uv_raster_positions_and_bands(t0):
    v, f, vt, ft = _mesh(3)
    h, w = 200, 232
    rast, baker, feats, f32, M = _bake_one_band(t0, v, f, vt, ft, h, w)
    clip = torch.cat([vt * 2 - 1, torch.zeros_like(vt[:, :1]), torch.ones_like(vt[:, :1])], 1).contiguous()
    ref_rast, _ = dr.rasterize(dr.RasterizeCudaContext(), clip, ft, (h, w))
    assert torch.equal(rast, ref_rast)
    covered = rast[0, ..., 3] > 0
    assert M == int(covered.sum()) and int(baker.counters[2]) == 0 and M > 0.2 * h * w
    xyz = torch.empty(h * w, 3, device="cuda")
    call("n2m_interpolate_forward", ptr(v), v.shape[0], 3, ptr(rast), ptr(f), h * w, ptr(xyz), stream())
    torch.cuda.synchronize()
    pix = baker.pix[:M].long()
    assert torch.equal(baker.pts[:M], xyz[pix])
    assert torch.equal(torch.sort(pix).values, torch.nonzero(covered.view(-1))[:, 0])
    one, mask = X.uv_features(t0, v, f, vt, ft, h, w)
    assert torch.equal(mask, covered) and torch.equal(one, feats)
    banded, _ = X.uv_features(t0, v, f, vt, ft, h, w, band_rows=37)
    assert torch.equal(banded, one)
    assert (one.view(-1, 6)[~covered.view(-1)] == 0).all()


def _check_inpaint(before, m, after, src):
    """the device inpaint (after, src) of (before, m) against renderer.py:378-394 restated with scipy and the KD-tree"""
    _, inpaint, search, d2 = O.reference_inpaint(before, m)
    w = m.shape[1]
    assert np.array_equal(src >= 0, inpaint)
    ys, xs = np.nonzero(inpaint)
    s = src[ys, xs].astype(np.int64)
    sy, sx = s // w, s % w
    assert search[sy, sx].all()
    assert np.array_equal((sy - ys) ** 2 + (sx - xs) ** 2, d2)
    assert np.array_equal(after[ys, xs], before[sy, sx])
    assert np.array_equal(after[m], before[m])
    assert (after[~m & ~inpaint] == 0).all()
    return inpaint


def test_inpaint_against_reference_post_processing(t0):
    v, f, vt, ft = _mesh(2)
    h, w = 320, 288
    feats, mask = X.uv_features(t0, v, f, vt, ft, h, w)
    before = feats.cpu().numpy(); m = mask.cpu().numpy()
    _, src = X.inpaint(feats, mask, return_source=True)
    inpaint = _check_inpaint(before, m, feats.cpu().numpy(), src.cpu().numpy())
    assert inpaint.sum() > 1000


@pytest.mark.parametrize("name,mask", O.sample_masks(), ids=[n for n, _ in O.sample_masks()])
def test_inpaint_on_oracle_masks(name, mask):
    """masks that touch the image border (the erosion's border rule) and leave texels beyond the L1 radius 32 (the dilation's cut-off)"""
    rng = np.random.default_rng(1)
    h, w = mask.shape
    before = rng.integers(0, 256, (h, w, 6)).astype(np.uint8)           # garbage outside the mask: the kernel must overwrite it
    feats = torch.from_numpy(before).cuda()
    _, src = X.inpaint(feats, torch.from_numpy(mask).cuda(), return_source=True)
    inpaint = _check_inpaint(before, mask, feats.cpu().numpy(), src.cpu().numpy())
    if name in ("blobs", "sparse_blobs", "single_texel", "single_corner_texel"):
        ys, xs = np.nonzero(~mask & ~inpaint)
        assert len(ys) > 0                                                 # texels beyond the cut-off exist and stay 0
    if name == "single_texel":                                             # the diamond |dx| + |dy| <= 32 around (40, 31)
        yy, xx = np.mgrid[0:h, 0:w]
        assert np.array_equal(inpaint, (np.abs(yy - 40) + np.abs(xx - 31) <= 32) & ~mask)


def test_inpaint_beyond_4_gib_of_features():
    """an image whose feature buffer exceeds 2^32 bytes (26,800^2 texels, 4.3 GB): the texel byte offsets must not wrap.  The mask sits in
    the bottom-right corner, where texel * 6 >= 2^32; a 300 x 700 crop around it is an exact sub-problem for the oracle."""
    H = W = 26800
    assert 6 * H * W >= 1 << 32 and H * W < 1 << 31
    ch, cw = 300, 700
    cm = np.zeros((ch, cw), dtype=bool)
    cm[40:, 40:] = O.blob_mask(ch - 40, cw - 40, 8, seed=5, rmax=30)       # touches the image's bottom and right borders
    rng = np.random.default_rng(2)
    crop_before = rng.integers(0, 256, (ch, cw, 6)).astype(np.uint8)
    feats = torch.zeros(H, W, 6, dtype=torch.uint8, device="cuda")
    mask = torch.zeros(H, W, dtype=torch.uint8, device="cuda")
    feats[H - ch:, W - cw:] = torch.from_numpy(crop_before).cuda()
    mask[H - ch:, W - cw:] = torch.from_numpy(cm.astype(np.uint8)).cuda()
    _, src = X.inpaint(feats, mask, return_source=True)
    torch.cuda.synchronize()
    crop_after = feats[H - ch:, W - cw:].cpu().numpy()
    g = src[H - ch:, W - cw:].cpu().numpy().astype(np.int64)
    local = np.where(g >= 0, (g // W - (H - ch)) * cw + (g % W - (W - cw)), -1)
    inpaint = _check_inpaint(crop_before, cm, crop_after, local)
    # inpaint and mask texels in the last 90 rows, whose byte offsets are past 2^32
    assert (H - 90) * W * 6 >= 1 << 32 and inpaint[-90:].sum() > 1000 and cm[-90:].sum() > 1000
    assert torch.count_nonzero(feats[: H - ch]).item() == 0 and torch.count_nonzero(feats[H - ch:, : W - cw]).item() == 0
    assert int((src[: H - ch] >= 0).sum()) == 0


def test_downscale_is_the_rounded_block_mean(t0):
    g = torch.Generator(device="cuda").manual_seed(2)
    feats = torch.randint(0, 256, (130, 198, 6), dtype=torch.uint8, device="cuda", generator=g)
    f0, f1 = X.downscale(feats, 2)
    ref = O.down2(feats.cpu().numpy())
    assert np.array_equal(f0.cpu().numpy(), ref[..., :3]) and np.array_equal(f1.cpu().numpy(), ref[..., 3:])
    g0, g1 = X.downscale(feats, 1)
    assert torch.equal(g0, feats[..., :3]) and torch.equal(g1, feats[..., 3:])


def test_empty_coverage_gives_zero_textures(t0):
    v, f, _, _ = _mesh(1)
    vt = torch.full((3 * f.shape[0], 2), 0.5, device="cuda")          # degenerate UV triangles: nothing is covered
    ft = torch.arange(3 * f.shape[0], dtype=torch.int32, device="cuda").view(-1, 3)
    f0, f1 = X.bake_features(t0, v, f, vt, ft, 64, 64, ssaa=2)
    assert f0.shape == (64, 64, 3) and int(f0.sum()) == 0 and int(f1.sum()) == 0


def test_export_stage1_writes_the_reference_files(t0, tmp_path):
    import cv2
    from nerf2mesh_b200.stage1 import Stage1Trainer
    v, f, vt, ft = _mesh(2)
    s1 = Stage1Trainer(t0, v, f, 16, 16, ssaa=2)
    f0, f1 = X.export_stage1(s1, str(tmp_path), vt, ft, resolution=128)
    names = sorted(os.listdir(tmp_path))
    assert names == ["feat0_0.jpg", "feat1_0.jpg", "mesh_0.mtl", "mesh_0.obj", "mlp.json"]
    img = cv2.imread(str(tmp_path / "feat0_0.jpg"))
    assert img.shape == (128, 128, 3)
    # JPEG is lossy: the decoded BGR image is close to the RGB texture reversed
    assert np.abs(img.astype(np.int32) - f0.cpu().numpy()[..., ::-1].astype(np.int32)).mean() < 8
    d = json.load(open(tmp_path / "mlp.json"))
    st = t0.export_reference_state()
    for k in ("net.0.weight", "net.1.weight"):
        assert np.array_equal(np.array(d[k], dtype=np.float32), st["specular_net." + k].cpu().numpy().T)
    assert d["bound"] == 1.0 and d["cascade"] == 1
    lines = open(tmp_path / "mesh_0.obj").read().splitlines()
    assert sum(l.startswith("v ") for l in lines) == v.shape[0] and sum(l.startswith("vt ") for l in lines) == vt.shape[0]
    assert sum(l.startswith("f ") for l in lines) == f.shape[0]


def test_full_size_bake_is_deterministic(t0):
    v, f, vt, ft = _mesh(7)
    assert f.shape[0] >= 100000
    torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
    a0, a1 = X.bake_features(t0, v, f, vt, ft, 4096, 4096, ssaa=2)        # raises on a point overflow
    b0, b1 = X.bake_features(t0, v, f, vt, ft, 4096, 4096, ssaa=2)
    torch.cuda.synchronize()
    assert a0.shape == (4096, 4096, 3)
    assert torch.equal(a0, b0) and torch.equal(a1, b1)
    assert (a0.view(-1, 3) != 0).any(dim=1).float().mean().item() > 0.3
