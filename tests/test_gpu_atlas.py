"""GPU: the device UV atlas (texture.uv_unwrap, csrc/atlas.cu) is bit for bit its numpy restatement (tests/atlas_oracle.py) on the hand-built
and property meshes of tests/test_atlas_cpu.py and on a 300k-face decimated marching-cubes mesh, and deterministic; export_stage1 without
a caller's unwrap writes the usual files for a cascaded, contracted scene; and a bake on the device atlas renders as close to the neural
render as a bake on the per-face grid atlas."""
import os

import numpy as np
import pytest
import torch

import atlas_oracle as A
import test_atlas_cpu as C
import texture_oracle as TO
from nerf2mesh_b200 import mesh as M
from nerf2mesh_b200 import texture as X
from nerf2mesh_b200.stage1 import Stage1Trainer

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _dev(v, f):
    return torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda(), torch.from_numpy(np.ascontiguousarray(f, np.int32)).cuda()


def _same_as_oracle(v, f, res=C.RES, ssaa=C.SSAA):
    vd, fd = _dev(v, f)
    info = {}
    vt, ft, vm = X.uv_unwrap(vd, fd, res, ssaa=ssaa, info=info)
    again = X.uv_unwrap(vd, fd, res, ssaa=ssaa)
    torch.cuda.synchronize()
    assert vt.dtype == torch.float32 and ft.dtype == torch.int32 and vm.dtype == torch.int32
    assert all(torch.equal(a, b) for a, b in zip((vt, ft, vm), again))                 # deterministic
    ref_info = {}
    rvt, rft, rvm = A.unwrap(v, f, res, ssaa, ref_info)
    vt, ft, vm = vt.cpu().numpy(), ft.cpu().numpy(), vm.cpu().numpy()
    assert vt.shape == rvt.shape and np.array_equal(vt.view(np.uint32), rvt.view(np.uint32))
    assert np.array_equal(ft, rft) and np.array_equal(vm, rvm)
    for k in ("charts", "split_rounds", "texels_per_unit"):
        assert info[k] == ref_info[k], (k, info[k], ref_info[k])
    assert abs(info["utilization"] - ref_info["utilization"]) <= 1e-9
    return vt, ft, vm, info


@pytest.mark.parametrize("name", list(C.HAND))
def test_hand_built_meshes_equal_the_oracle(name):
    v, f = C.HAND[name]
    _same_as_oracle(v, f)


@pytest.mark.parametrize("name", list(C.MEASURED))
def test_property_meshes_equal_the_oracle(name):
    v, f = C.property_meshes()[name]
    vt, ft, vm, info = _same_as_oracle(v, f)
    C.check_properties(v, f, vt, ft, vm, info)


def test_empty_and_invalid_inputs():
    v, f = _dev(*C.cube())
    vt, ft, vm = X.uv_unwrap(v[:0], f[:0], 64)
    assert vt.shape == (0, 2) and ft.shape == (0, 3) and vm.shape == (0,)
    for bad in (dict(triangles=f[:, :2]), dict(triangles=f.float()), dict(vertices=v.double()), dict(triangles=f + 8),
                dict(triangles=f - 1), dict(resolution=1 << 15), dict(resolution=4)):
        args = dict(vertices=v, triangles=f, resolution=64)
        args.update(bad)
        with pytest.raises(ValueError):
            X.uv_unwrap(**args)
    with pytest.raises(ValueError, match="fit"):                     # 12 single-face charts cannot fit 8 x 8 texels with a gap of 2
        X.uv_unwrap(*_dev(*C.spiral()), 8, ssaa=1)


def test_300k_face_mesh_equals_the_oracle():
    from test_gpu_meshclean import mc_mesh
    v, f = mc_mesh(512)
    v, f = M.decimate_mesh(*M.clean_mesh(v, f), 300000)
    assert f.shape[0] in (300000, 299999)
    vn, fn = v.cpu().numpy(), f.cpu().numpy().astype(np.int64)
    del v, f
    vt, ft, vm, info = _same_as_oracle(vn, fn, res=2048, ssaa=2)
    print(f"300k: {info}")


def test_export_stage1_unwraps_every_cascade(tmp_path):
    from test_gpu_cascades import _bound4_trainer, _cascade_meshes
    t0 = _bound4_trainer(contract=True)
    vs, fs = _cascade_meshes()
    s1 = Stage1Trainer(t0, vs, fs, 48, 48, ssaa=2)
    feats = X.export_stage1(s1, str(tmp_path), resolution=512)
    assert len(feats) == 3
    names = sorted(os.listdir(tmp_path))
    assert names == sorted([f"{p}_{c}.{e}" for c in range(3) for p, e in (("feat0", "jpg"), ("feat1", "jpg"), ("mesh", "obj"), ("mesh", "mtl"))]
                           + ["mlp.json"])
    a = X.load_exported(str(tmp_path))
    assert a.cascades == 3 and a.face_offsets == [0] + np.cumsum([x.shape[0] for x in fs]).tolist()
    # the files hold unwrap_stage1's atlas: the contracted positions unwrapped at each cascade's texture size
    vts, fts = X.unwrap_stage1(s1, 512)
    st = torch.cat([torch.stack([x[:, 0], 1 - x[:, 1]], 1) for x in vts]).cpu()
    assert torch.equal(a.st.cpu(), st)
    for cas, size in enumerate(X.texture_sizes(512, 3)):
        v, f = s1.cascade_mesh(cas)
        vc = v.clone()
        mag = vc.abs().amax(1, keepdim=True)
        vc = torch.where(mag <= 1, vc, (2 - 1 / mag) * vc / mag)                       # contract(), renderer.py:25-32
        vt, ft, _ = X.uv_unwrap(vc.contiguous(), f, size, ssaa=2)
        assert torch.equal(vt, vts[cas]) and torch.equal(ft, fts[cas])
    with pytest.raises(ValueError):
        X.export_stage1(s1, str(tmp_path), vt=vts)


def test_device_atlas_bake_is_close_to_the_neural_render():
    """test_gpu_stage1_render.test_baked_asset_is_close_to_the_neural_render at resolution 512, with the device atlas and with the
    per-face grid atlas: the device atlas's mean error is within the same 4/255 bound and no larger than the grid atlas's"""
    from test_gpu_stage1 import _setup
    from test_gpu_stage1_render import CAM
    t0, s1, mvp, rays_d, gt, bg = _setup(ssaa=2)
    mvp = mvp.cuda()
    v, f = s1.cascade_mesh(0)
    vts, fts = X.unwrap_stage1(s1, 512)
    gvt, gft = TO.grid_atlas(f.shape[0])
    errs = {}
    ineu, wn, _ = s1.render(mvp, rays_d, shading="diffuse")
    for name, vt, ft in (("device", vts[0], fts[0]), ("grid", torch.from_numpy(gvt).cuda(), torch.from_numpy(gft).cuda())):
        feats = X.bake_features(t0, v, f, vt, ft, 512, 512, ssaa=2)
        asset = X.ExportedMesh.from_export(s1, vt, ft, feats)
        ia, wa, _ = X.render_exported(asset, mvp, CAM, s1.h0, s1.w0, ssaa=2, shading="diffuse", antialias=True)
        torch.cuda.synchronize()
        both = (wa == 1) & (wn == 1)
        assert both.float().mean().item() > 0.1
        errs[name] = (ia[both] - ineu[both]).abs().mean().item()
        print(f"mean |asset - neural| with the {name} atlas over {int(both.sum())} pixels: {errs[name] * 255:.3f}/255")
    assert errs["device"] <= 4 / 255 and errs["device"] <= errs["grid"], errs
