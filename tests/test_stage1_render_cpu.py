"""CPU: the numpy oracles of the stage-1 evaluation (stage1_render_oracle.py) against independent restatements, and the OBJ /
mlp.json loaders of the exported asset against their writers."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import stage1_render_oracle as O


def _torch_render_stage1_tail(img, z, bg, h0, w0, ssaa):
    """renderer.py:886-907 restated in torch: clamp, alphas * rgbs, alphas * z, scale_img_hwc (bilinear) minification, background"""
    h, w = h0 * ssaa, w0 * ssaa
    img = torch.from_numpy(img).double().view(h, w, 4)
    alphas = img[..., 3:].clamp(0, 1)
    rgbs = img[..., :3].clamp(0, 1)
    image = alphas * rgbs
    depth = alphas * torch.from_numpy(z).double().view(h, w, 1)
    T = 1 - alphas

    def down(x):
        return F.interpolate(x.permute(2, 0, 1)[None], (h0, w0), mode="bilinear")[0].permute(1, 2, 0)

    if ssaa > 1:
        image, depth, T = down(image), down(depth), down(T)
    image = image + T * torch.from_numpy(bg).double().view(h0, w0, 3)
    return image.reshape(-1, 3).numpy(), (1 - T).reshape(-1).numpy(), depth.reshape(-1).numpy()


@pytest.mark.parametrize("ssaa", [1, 2])
def test_compose_oracle_is_render_stage1(ssaa):
    rng = np.random.default_rng(ssaa)
    h0, w0 = 13, 17
    n = h0 * w0 * ssaa * ssaa
    img = rng.uniform(-0.3, 1.3, (n, 4))                       # outside [0, 1] too: both clamps matter
    img[rng.random(n) < 0.3, 3] = 0.0
    z = rng.uniform(-1, 1, n)
    bg = rng.random((h0 * w0, 3))
    got = O.compose(img, z, bg, h0, w0, ssaa)
    ref = _torch_render_stage1_tail(img, z, bg, h0, w0, ssaa)
    for a, b in zip(got, ref):
        assert np.abs(a - b).max() <= 1e-12


def test_nearest_texel_is_three_js_nearest_flipy_clamp():
    H, W = 4, 8
    tex = np.arange(H * W * 3, dtype=np.uint8).reshape(H, W, 3)
    # (s, t) -> (image row, column): t = 0 is the bottom image row (flipY), exact texel edges go to the texel above them, outside clamps
    cases = [((0.0, 0.0), (3, 0)), ((0.999, 0.999), (0, 7)), ((0.125, 0.25), (2, 1)), ((0.1249, 0.2499), (3, 0)),
             ((-0.5, 1.5), (0, 0)), ((1.0, 1.0), (0, 7)), ((1.5, -0.2), (3, 7))]
    for (s, t), (y, x) in cases:
        assert np.array_equal(O.nearest_texel(tex, np.float32([s]), np.float32([t]))[0], tex[y, x]), (s, t)


def test_specular_oracle_is_the_reference_net():
    rng = np.random.default_rng(3)
    w0 = rng.standard_normal((32, 6)).astype(np.float32); w1 = rng.standard_normal((3, 32)).astype(np.float32)
    x = rng.standard_normal((50, 6))
    net = torch.nn.Sequential(torch.nn.Linear(6, 32, bias=False), torch.nn.ReLU(), torch.nn.Linear(32, 3, bias=False)).double()
    with torch.no_grad():
        net[0].weight.copy_(torch.from_numpy(w0)); net[2].weight.copy_(torch.from_numpy(w1))
        ref = torch.sigmoid(net(torch.from_numpy(x))).numpy()
    assert np.abs(O.specular(w0, w1, x) - ref).max() <= 1e-12


def test_asset_shade_oracle_modes_and_cascades():
    """two cascades with different texture sizes, a face of each: the colour comes from the face's own cascade, the modes compose as the
    viewer's shader does (renderer.html:148-158)"""
    rng = np.random.default_rng(5)
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 2], [1, 0, 2], [0, 1, 2]], np.float32)
    tri = np.array([[0, 1, 2], [3, 4, 5]], np.int64)
    st = np.array([[0.1, 0.1], [0.9, 0.1], [0.1, 0.9], [0.6, 0.6], [0.7, 0.6], [0.6, 0.7]], np.float32)
    ft = np.array([[0, 1, 2], [3, 4, 5]], np.int64)
    feat0 = [rng.integers(0, 256, (8, 8, 3), dtype=np.uint8), rng.integers(0, 256, (4, 16, 3), dtype=np.uint8)]
    feat1 = [rng.integers(0, 256, (8, 8, 3), dtype=np.uint8), rng.integers(0, 256, (4, 16, 3), dtype=np.uint8)]
    w0 = rng.standard_normal((32, 6)).astype(np.float32); w1 = rng.standard_normal((3, 32)).astype(np.float32)
    cam = np.array([0.3, 0.2, 5.0])
    rast = np.array([[0.2, 0.35, 0.1, 1], [0.45, 0.3, 0.4, 2], [0, 0, 0, 0]], np.float32)
    out = {m: O.asset_shade(rast, verts, tri, st, ft, [0, 1, 2], feat0, feat1, w0, w1, cam, m) for m in (1, 2, 3)}
    assert np.array_equal(out[1][2], np.zeros(4)) and np.all(out[1][:2, 3] == 1)
    for k, (c, face) in enumerate([(0, 0), (1, 1)]):
        u, v = rast[k, 0], rast[k, 1]
        b = np.array([u, v, 1 - u - v], np.float64)
        s, t = b @ st[ft[face], 0], b @ st[ft[face], 1]
        H, W = feat0[c].shape[:2]
        y, x = H - 1 - int(np.floor(t * H)), int(np.floor(s * W))
        assert np.array_equal(out[1][k, :3], feat0[c][y, x] / 255.0)
        p = b @ verts[tri[face]]
        d = (p - cam) / np.linalg.norm(p - cam)
        sp = O.specular(w0, w1, np.concatenate([d, feat1[c][y, x] / 255.0])[None])[0]
        assert np.abs(out[2][k, :3] - sp).max() <= 1e-6
        assert np.abs(out[3][k, :3] - np.clip(feat0[c][y, x] / 255.0 + sp, 0, 1)).max() <= 1e-6


def test_obj_and_mlp_json_round_trip(tmp_path):
    from nerf2mesh_b200 import texture as X
    rng = np.random.default_rng(11)
    v = (rng.standard_normal((57, 3)) * np.array([1e-7, 3.0, 1234.5])).astype(np.float32)
    f = rng.integers(0, 57, (40, 3)).astype(np.int32)
    vt = rng.random((71, 2)).astype(np.float32); vt[0] = [0.0, 1.0]; vt[1] = [1.0, 1e-8]
    ft = rng.integers(0, 71, (40, 3)).astype(np.int32)
    X.write_obj(tmp_path / "mesh_0.obj", v, f, vt, ft)
    rv, rst, rf, rft = X.read_obj(tmp_path / "mesh_0.obj")
    assert rv.tobytes() == v.tobytes()
    assert rst.tobytes() == np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], 1).astype(np.float32).tobytes()
    assert np.array_equal(rf, f) and np.array_equal(rft, ft)
    w0 = rng.standard_normal((32, 6)).astype(np.float32); w1 = rng.standard_normal((3, 32)).astype(np.float32)
    X.write_mlp_json(tmp_path / "mlp.json", {"net.0.weight": w0, "net.1.weight": w1}, bound=1.0, cascade=1)
    cv2 = pytest.importorskip("cv2")
    tex = rng.integers(0, 256, (16, 8, 3), dtype=np.uint8)
    X.write_textures(str(tmp_path), tex, tex[::-1].copy(), 0)
    asset = X.load_exported(str(tmp_path), device="cpu")
    assert asset.vertices.numpy().tobytes() == v.tobytes() and np.array_equal(asset.triangles.numpy(), f)
    assert asset.st.numpy().tobytes() == rst.tobytes() and np.array_equal(asset.ft.numpy(), ft)
    assert np.array_equal(asset.weights["net.0.weight"], w0) and np.array_equal(asset.weights["net.1.weight"], w1)
    assert asset.bound == 1.0 and asset.face_offsets == [0, 40] and asset.cascades == 1
    assert np.array_equal(asset.feat0[0].numpy(), cv2.imread(str(tmp_path / "feat0_0.jpg"))[..., ::-1])
    assert json.load(open(tmp_path / "mlp.json"))["cascade"] == 1
