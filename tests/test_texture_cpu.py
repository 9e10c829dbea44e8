"""CPU: the stage-1 texture export without a GPU -- the closed forms the inpaint and down-sample kernels implement (csrc/texture.cu) against
the reference's own post-processing (tests/texture_oracle.py: scipy dilation / erosion, sklearn KD-tree, cv2.resize), the compile-time
budget of the geo_feat kernel, the OBJ / MTL / mlp.json writers and the input validation of nerf2mesh_b200.texture."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import texture_oracle as O
from nerf2mesh_b200 import build as B


@pytest.mark.parametrize("name,mask", O.sample_masks(), ids=[n for n, _ in O.sample_masks()])
def test_windowed_search_equals_kd_tree(name, mask):
    rng = np.random.default_rng(0)
    feats = np.where(mask[..., None], rng.integers(0, 256, mask.shape + (6,)), 0).astype(np.uint8)
    _, inpaint, search, d2 = O.reference_inpaint(feats, mask)
    ci, cs = O.closed_form_regions(mask)
    assert np.array_equal(ci, inpaint) and np.array_equal(cs, search), name
    if inpaint.any():
        ours = O.windowed_min_d2(search)[inpaint]                   # np.nonzero order, as the oracle's
        assert np.array_equal(ours, d2), name
        assert d2.max() <= 32 * 32
    if name == "blobs":
        assert inpaint.sum() > 10000


@pytest.mark.parametrize("h0,w0", [(64, 48), (101, 37), (256, 256)])
def test_rounded_block_mean_equals_cv2_resize(h0, w0):
    img = np.random.default_rng(h0 * w0).integers(0, 256, (2 * h0, 2 * w0, 3)).astype(np.uint8)
    assert np.array_equal(O.down2(img), O.reference_resize(img, w0, h0))


def test_geo_feat_kernel_has_no_spills_and_no_wgmma_advisories(tmp_path):
    src = os.path.join(B.CSRC, "texture.cu")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "texture.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    props = [i for i, l in enumerate(lines) if "Function properties for" in l and "k_s1_geo_feat" in l]
    assert len(props) == 1, "\n".join(lines)
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[props[0] + 1])
    assert m and (int(m.group(2)), int(m.group(3))) == (0, 0), lines[props[0] + 1]
    assert not [l for l in lines if re.search(r"\(C751\d\)", l) and "k_s1_geo_feat" in l]


def _read_obj(path):
    v, vt, f = [], [], []
    with open(path) as fp:
        lines = fp.read().splitlines()
    for line in lines:
        p = line.split()
        if not p:
            continue
        if p[0] == "v":
            v.append([np.float32(x) for x in p[1:]])
        elif p[0] == "vt":
            vt.append([np.float32(x) for x in p[1:]])
        elif p[0] == "f":
            f.append([[int(i) for i in c.split("/")] for c in p[1:]])
    return lines, np.array(v, dtype=np.float32), np.array(vt, dtype=np.float32), np.array(f, dtype=np.int64)


def test_obj_mtl_and_mlp_json_writers(tmp_path):
    from nerf2mesh_b200 import texture as X
    rng = np.random.default_rng(7)
    v = (rng.standard_normal((57, 3)) * np.array([1e-7, 3.0, 1234.5])).astype(np.float32)
    v[0] = [0.1, -0.0, 1.0 / 3.0]
    f = rng.integers(0, 57, (40, 3)).astype(np.int32)
    vt = rng.random((71, 2)).astype(np.float32); vt[0] = [0.0, 1.0]; vt[1] = [1.0, 1e-8]
    ft = rng.integers(0, 71, (40, 3)).astype(np.int32)
    X.write_obj(tmp_path / "mesh_0.obj", torch.from_numpy(v), torch.from_numpy(f), vt, ft)
    lines, rv, rvt, rf = _read_obj(tmp_path / "mesh_0.obj")
    assert lines[0].split() == ["mtllib", "mesh_0.mtl"] and "usemtl defaultMat" in [l.strip() for l in lines]
    assert rv.tobytes() == v.tobytes()
    assert rvt.tobytes() == np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], 1).astype(np.float32).tobytes()
    assert np.array_equal(rf[..., 0], f + 1) and np.array_equal(rf[..., 1], ft + 1)
    X.write_mtl(tmp_path / "mesh_0.mtl")
    mtl = [l.split() for l in open(tmp_path / "mesh_0.mtl").read().splitlines()]
    assert ["newmtl", "defaultMat"] in mtl and ["map_Kd", "feat0_0.jpg"] in mtl
    w0 = rng.standard_normal((32, 6)).astype(np.float32); w1 = rng.standard_normal((3, 32)).astype(np.float32)
    X.write_mlp_json(tmp_path / "mlp.json", {"net.0.weight": w0, "net.1.weight": w1}, bound=1.0, cascade=1)
    d = json.load(open(tmp_path / "mlp.json"))
    assert set(d) == {"net.0.weight", "net.1.weight", "bound", "cascade"} and d["bound"] == 1.0 and d["cascade"] == 1
    assert np.array_equal(np.array(d["net.0.weight"], dtype=np.float32), w0.T)
    assert np.array_equal(np.array(d["net.1.weight"], dtype=np.float32), w1.T)


def test_mesh_validation():
    from nerf2mesh_b200.texture import validate_mesh
    v = torch.zeros(4, 3); f = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    vt = torch.tensor([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]]); ft = f.clone()
    validate_mesh(v, f, vt, ft, 64, 64)
    with pytest.raises(ValueError):
        validate_mesh(v, f, vt, ft[:1], 64, 64)                          # row counts differ
    with pytest.raises(ValueError):
        validate_mesh(v, f, vt, torch.tensor([[0, 1, 2], [0, 2, 4]], dtype=torch.int32), 64, 64)     # ft index out of range
    with pytest.raises(ValueError):
        validate_mesh(v, f, vt * 1.5, ft, 64, 64)                        # vt outside [0, 1]
    with pytest.raises(ValueError):
        validate_mesh(v, f, vt - 0.25, ft, 64, 64)
    with pytest.raises(ValueError):
        validate_mesh(v, f, vt, ft, 65536, 32768)                        # 2^31 texels: more than n2m_rasterize accepts
