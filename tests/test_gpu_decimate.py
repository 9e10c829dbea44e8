"""GPU: the decimation of csrc/decimate.cu against the CPU oracle (tests/decimate_oracle.py) -- bit-equal vertices, equal faces -- on the
hand-built meshes of test_decimate_cpu.py and on the seeded noisy marching-cubes meshes of test_gpu_meshclean.py, raw and cleaned;
properties at 512^3; empty, small, invalid and stalling inputs; the exports' `decimate_target=` against the oracle chain; a stage-1
trainer on the decimated meshes."""
import numpy as np
import pytest
import torch

import decimate_oracle as D
import meshclean_oracle as O
import test_decimate_cpu as C
from nerf2mesh_b200 import mesh as M
from nerf2mesh_b200.stage1 import Stage1Trainer
from test_gpu_cascades import _bound4_trainer, _cascade_meshes, _garden_trainer, _views
from test_gpu_meshclean import _dev, _np, _same, _train, mc_mesh
from nerf2mesh_b200 import synthetic as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _check(v, f, target, optimal):
    ref_info, info = {}, {}
    ref = D.decimate(v, f, target, optimal, ref_info)
    _same(M.decimate_mesh(*_dev(v, f), target, optimal_placement=optimal, info=info), ref)
    assert info == ref_info, (info, ref_info)
    return info


@pytest.mark.parametrize("optimal", [True, False])
@pytest.mark.parametrize("name", sorted(C.HAND))
def test_hand_built_cases_equal_the_oracle(name, optimal):
    v, f = C.HAND[name]
    for target in sorted({1, 2, len(f) // 2, len(f) - 1, len(f)} - {0}):
        _check(v, f, target, optimal)


@pytest.mark.parametrize("optimal", [True, False])
def test_analytic_meshes_equal_the_oracle(optimal):
    for vol in (C.sphere_volume(40)[0], C.torus_volume(40)[0]):
        v, f = C.mc(vol)
        for target in (len(f) // 2, len(f) // 10, 7):
            _check(v, f, target, optimal)


@pytest.mark.parametrize("optimal", [True, False])
def test_noisy_marching_cubes_meshes_equal_the_oracle(optimal):
    v, f = mc_mesh(128)
    raw = _np(v, f)
    info = _check(*raw, len(raw[1]) // 10, optimal)
    assert info["rounds"] >= 2 and not info["stalled"]
    vc, fc = M.clean_mesh(v, f)
    cleaned = _np(vc, fc)
    _check(*cleaned, len(cleaned[1]) // 3, optimal)
    _check(*cleaned, len(cleaned[1]) // 20, optimal)


def _edges(f):
    return np.sort(np.stack([f, np.roll(f, -1, 1)], 2).reshape(-1, 2), 1)


def test_512_properties():
    v, f = M.clean_mesh(*mc_mesh(512, seed=3))
    vi, fi = _np(v, f)
    ei = np.unique(_edges(fi), axis=0)
    euler = len(vi) - len(ei) + len(fi)
    target = len(fi) // 5
    info = {}
    vo, fo = M.decimate_mesh(v, f, target, info=info)
    torch.cuda.synchronize()
    vo, fo = _np(vo, fo)
    assert len(fo) in (target, target - 1) and not info["stalled"]
    assert info["rounds"] == len(info["faces"]) >= 2 and info["faces"][-1] == len(fo)
    assert all(a > b for a, b in zip(info["faces"], info["faces"][1:]))
    assert ((fo[:, 0] != fo[:, 1]) & (fo[:, 1] != fo[:, 2]) & (fo[:, 0] != fo[:, 2])).all()
    assert len(np.unique(np.sort(fo, 1), axis=0)) == len(fo)
    eo, cnt = np.unique(_edges(fo), axis=0, return_counts=True)
    assert cnt.max() <= 2
    assert np.array_equal(np.unique(fo), np.arange(len(vo)))
    assert len(vo) - len(eo) + len(fo) == euler
    assert np.isfinite(vo).all()


def test_empty_small_invalid_and_stalling_inputs():
    v, f = C.grid(2)
    vd, fd = _dev(v, f)
    empty_f = torch.empty(0, 3, dtype=torch.int32, device="cuda")
    for out in (M.decimate_mesh(vd, empty_f, 5), M.decimate_mesh(vd[:0], empty_f, 5)):
        torch.cuda.synchronize()
        assert out[0].shape == (0, 3) and out[1].shape == (0, 3) and out[0].dtype == torch.float32 and out[1].dtype == torch.int32
    with pytest.raises(ValueError):
        M.decimate_mesh(vd, fd, 0)
    # F <= target: only the unreferenced vertex goes
    v2 = np.concatenate([v, [[9, 9, 9]]]).astype(np.float32)
    info = {}
    _same(M.decimate_mesh(*_dev(v2, f), len(f), info=info), (v, f.astype(np.int32)))
    assert info == {"rounds": 0, "stalled": False, "faces": []}
    # the tetrahedron stalls at once; faces that repeat an index go before the first round
    info = _check(*C.tetrahedron(), 2, True)
    assert info == {"rounds": 0, "stalled": True, "faces": []}
    tv, tf = C.tetrahedron()
    _check(tv, np.concatenate([tf, [[0, 0, 1], [2, 3, 3]]]), 5, True)


# ---- the exports' decimation ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["bound4", "garden16"])
def test_exports_with_decimate_target_equal_the_oracle_chain(tmp_path, scene):
    if scene == "bound4":
        t0 = _bound4_trainer()
    else:
        t0 = _train(_garden_trainer(), S.garden_scene(bound=16.0)[2])
    views = _views(96, 96, n=4)
    mvps = torch.stack([m for m, *_ in views])
    clean = M.CleanOptions(min_f=8, min_d=5, visibility_mask_dilation=2, mvps=mvps, H=96, W=96)
    kw = dict(resolution=64, density_thresh=0.5)
    # decimate_target=0 writes exactly what the export without it writes
    M.export_stage0_mesh(t0, str(tmp_path / "plain"), **kw, clean=clean)
    M.export_stage0_mesh(t0, str(tmp_path / "zero"), **kw, clean=clean, decimate_target=0)
    assert (tmp_path / "plain" / "mesh_0.ply").read_bytes() == (tmp_path / "zero" / "mesh_0.ply").read_bytes()
    # mesh_0: visibility -> remove_masked_faces -> clean_mesh(repair=True) -> decimation with optimal placement
    v, f = M.export_stage0_mesh(t0, str(tmp_path / "raw"), **kw)
    cv, cf = O.clean_mesh(*O.remove_masked_faces(*_np(v, f), M.mark_unseen_triangles(v, f, mvps, 96, 96).cpu().numpy(), 2),
                          min_f=8, min_d=5, repair=True)
    target = len(cf) * 2 // 3
    assert target > 100
    ref = D.decimate(cv, cf, target, True)
    out = M.export_stage0_mesh(t0, str(tmp_path / "dec"), **kw, clean=clean, decimate_target=float(target))
    _same(out, ref)
    pv, pf = M.read_ply(tmp_path / "dec" / "mesh_0.ply")
    assert np.array_equal(pv, ref[0]) and np.array_equal(pf, ref[1])
    # without clean=, decimation follows marching cubes directly
    _same(M.export_stage0_mesh(t0, str(tmp_path / "decraw"), **kw, decimate_target=len(f) * 2 // 3), D.decimate(*_np(v, f), len(f) * 2 // 3, True))
    # outer cascades: clean_mesh(repair=False) -> decimation to decimate_target // 2 at midpoints -> visibility -> remove_masked_faces
    raw = M.export_outer_meshes(t0, str(tmp_path / "raw"), env_reso=64)
    plain = M.export_outer_meshes(t0, str(tmp_path / "plain"), env_reso=64, clean=clean)
    zero = M.export_outer_meshes(t0, str(tmp_path / "zero"), env_reso=64, clean=clean, decimate_target=0)
    assert set(plain) == set(zero)
    for cas in plain:
        name = f"mesh_{cas}.ply"
        assert (tmp_path / "plain" / name).read_bytes() == (tmp_path / "zero" / name).read_bytes()
    sizes = [len(O.clean_mesh(*_np(*m), min_f=8, min_d=5, repair=False)[1]) for m in raw.values()]
    dt = max(2 * (max(sizes, default=0) * 2 // 3), 2)
    out = M.export_outer_meshes(t0, str(tmp_path / "dec"), env_reso=64, clean=clean, decimate_target=dt)
    decimated = 0
    for cas, (rv, rf) in raw.items():
        cv, cf = O.clean_mesh(*_np(rv, rf), min_f=8, min_d=5, repair=False)
        if len(cv) and len(cf) > dt // 2:
            cv, cf = D.decimate(cv, cf, dt // 2, False)
            decimated += 1
        if len(cv) and len(cf):
            cvd, cfd = _dev(cv, cf)
            cv, cf = O.remove_masked_faces(cv, cf, M.mark_unseen_triangles(cvd, cfd, mvps, 96, 96).cpu().numpy(), 2)
        path = tmp_path / "dec" / f"mesh_{cas}.ply"
        if len(cv) == 0:
            assert cas not in out and not path.exists()
            continue
        _same(out[cas], (cv, cf))
        pv, pf = M.read_ply(path)
        assert np.array_equal(pv, cv) and np.array_equal(pf, cf)
    assert (decimated >= 1 or not raw) and set(out) <= set(raw)


def test_stage1_trainer_steps_on_the_decimated_meshes(tmp_path):
    t0 = _bound4_trainer()
    v0, f0 = M.export_stage0_mesh(t0, str(tmp_path), resolution=128, density_thresh=0.5, clean=M.CleanOptions(), decimate_target=4000)
    outer = M.export_outer_meshes(t0, str(tmp_path), env_reso=64, clean=M.CleanOptions(), decimate_target=4000)
    assert 0 < f0.shape[0] <= 4000 and all(f.shape[0] <= 2000 for _, f in outer.values())
    # a cascade the export left without a mesh takes the synthetic one of test_gpu_cascades
    sv, sf = _cascade_meshes()
    vs = [v0] + [outer[c][0] if c in outer else sv[c].cuda() for c in range(1, t0.cfg.cascade)]
    fs = [f0] + [outer[c][1] if c in outer else sf[c].cuda() for c in range(1, t0.cfg.cascade)]
    s1 = Stage1Trainer(t0, vs, fs, 64, 64, antialias=True, lr_vert=1e-4, lambda_normal=1e-3)
    views = _views(64, 64)
    for view in views:
        s1.step(*view, use_graph=False)
    torch.cuda.synchronize()
    assert s1.offsets.abs().max().item() > 0
    assert torch.isfinite(s1.vertices).all()
