"""GPU: the mesh clean-up of csrc/meshclean.cu against the CPU oracle (tests/meshclean_oracle.py) -- bit-equal vertices, equal faces -- on
the hand-built meshes of test_meshclean_cpu.py and on marching-cubes meshes of a seeded noisy volume; properties at 512^3; empty and
degenerate inputs; the exports' `clean=` chain against the oracle chain on the uncleaned export."""
import numpy as np
import pytest
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

import meshclean_oracle as O
import test_meshclean_cpu as C
from nerf2mesh_b200 import mesh as M
from nerf2mesh_b200 import synthetic as S
from test_gpu_cascades import _bound4_trainer, _garden_trainer, _views

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


def _same(out, ref):
    v, f = out
    torch.cuda.synchronize()
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and v.shape[1:] == (3,) and f.shape[1:] == (3,)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    assert v.shape == ref[0].shape and np.array_equal(v.view(np.uint32), ref[0].view(np.uint32)), (v.shape, ref[0].shape)
    assert np.array_equal(f, ref[1]), (f.shape, ref[1].shape)


def _check_clean(v, f, info=None, **kw):
    stats = {}
    ref = O.clean_mesh(v, f, stats=stats, **kw)
    _same(M.clean_mesh(*_dev(v, f), info=info, **kw), ref)
    return stats


def _row():
    r = O.merge_radius(np.sqrt(250.0), 100)
    v = np.concatenate([np.array([[0.9 * r * k, 0, 0] for k in range(5)], np.float32), np.array([[3 * k, 5, 0] for k in range(6)], np.float32)])
    return v, np.array([[k, 5 + k, 6 + k] for k in range(5)])


HAND = {
    "bowtie": (C.bowtie, dict(v_pct=0, min_f=0, min_d=0)),
    "bowtie3": (C.bowtie3, dict(v_pct=0, min_f=0, min_d=0)),
    "three_on_edge": (lambda: (np.array([[0, 0, 0], [1, 0, 0], [0.5, 2, 0], [0.5, 0, 0.5], [0.5, -1, 0]], np.float32),
                               np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]])), dict(v_pct=0, min_f=0, min_d=0)),
    "four_equal_on_edge": (lambda: (np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0], [0.5, 0, 1], [0.5, 0, -1]], np.float32),
                                    np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [1, 0, 5]])), dict(v_pct=0, min_f=0, min_d=0)),
    "duplicates": (lambda: (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], np.float32),
                            np.array([[1, 3, 2], [2, 1, 0], [0, 1, 2], [1, 2, 0], [3, 1, 2]])), dict(v_pct=0, min_f=0, min_d=0)),
    "zero_area": (lambda: (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.5, 0, 0], [2, 0, 0]], np.float32),
                           np.array([[0, 1, 2], [0, 3, 1], [1, 4, 3]])), dict(v_pct=0, min_f=0, min_d=0)),
    "row": (_row, dict(v_pct=100, min_f=0, min_d=0, repair=False)),
    "row_repair": (_row, dict(v_pct=100, min_f=0, min_d=0)),
    "diameter": (lambda: C.join(C.strip(0, 0, 6, 80, 10), C.strip(10, 10, 1.5, 4, 2),
                                C.strip(20, 0, 1.5, np.nextafter(np.float32(4), np.float32(0)), 2)), dict(v_pct=0, min_f=0, min_d=5)),
    "face_count": (lambda: C.join(C.strip(0, 0, 1, 1, 10), C.strip(20, 0, 1, 1, 2), C.strip(30, 0, 1, 1, 2)), dict(v_pct=0, min_f=4, min_d=0)),
    "face_count_below": (lambda: (lambda v, f: (v, f[:-1]))(*C.join(C.strip(0, 0, 1, 1, 10), C.strip(20, 0, 1, 1, 2))),
                         dict(v_pct=0, min_f=4, min_d=0)),
    "edge_connected": (C.bowtie, dict(v_pct=0, min_f=3, min_d=0, repair=False)),
    "defaults": (lambda: C.join(C.strip(0, 0, 1, 1, 10), C.bowtie()), dict()),
}


@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_built_cases_equal_the_oracle(name):
    make, kw = HAND[name]
    v, f = make()
    _check_clean(np.asarray(v, np.float32), np.asarray(f), **kw)


@pytest.mark.parametrize("dilation", [0, 1, 2, 7])
def test_dilation_on_a_strip_equals_the_oracle(dilation):
    v, f = C.strip(0, 0, 1, 1, 10)
    mask = np.ones(20, np.int64); mask[10] = 0; mask[19] = 0
    _same(M.remove_masked_faces(*_dev(v, f), torch.from_numpy(mask).cuda(), dilation), O.remove_masked_faces(v, f, mask, dilation))


# ---- marching-cubes meshes of a seeded noisy volume ---------------------------------------------------------------------------------
def noisy_volume(N, seed=0):
    """a sphere of radius 0.6 plus 12 floater blobs of 0.5-3 cells as a signed distance on [-1, 1]^3, with Gaussian noise of 0.7 cells
    within 2 cells of the surface: near-iso samples put marching-cubes vertices close together"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ax = torch.linspace(-1, 1, N, device="cuda")
    x, y, z = ax[:, None, None], ax[None, :, None], ax[None, None, :]
    d = 0.6 - torch.sqrt(x * x + y * y + z * z)
    centres = torch.rand(12, 3, generator=g, device="cuda") * 1.8 - 0.9
    radii = (torch.rand(12, generator=g, device="cuda") * 2.5 + 0.5) * 2 / N
    for c, r in zip(centres, radii):
        d = torch.maximum(d, r - torch.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2))
    h = 2.0 / (N - 1)
    noise = torch.randn(N, N, N, generator=g, device="cuda") * (0.7 * h)
    return torch.where(d.abs() < 2 * h, d + noise, d).contiguous()


def mc_mesh(N, seed=0):
    v, f = M.marching_cubes(noisy_volume(N, seed), 0.0)
    return v / (N - 1.0) * 2 - 1, f


@pytest.mark.parametrize("N", [128, 256])
def test_marching_cubes_meshes_equal_the_oracle(N):
    v, f = mc_mesh(N)
    vn, fn = v.cpu().numpy(), f.cpu().numpy().astype(np.int64)
    info = {}
    stats = _check_clean(vn, fn, info=info)
    for kind in ("merged", "duplicates", "nm_edge_faces", "split_copies", "components_removed"):
        assert stats[kind] > 0, (kind, stats)                                 # every rule is exercised
    assert info["merge_rounds"] >= 2
    _check_clean(vn, fn, repair=False, min_f=0)
    _check_clean(vn, fn, v_pct=3, min_d=0)
    # visibility-style mask: one half-space plus scattered faces, dilated
    c = vn[fn].mean(1)
    mask = ((c[:, 0] > 0.1) | (np.random.default_rng(N).random(len(fn)) < 0.05)).astype(np.uint8)
    for dil in (0, 1, 5):
        _same(M.remove_masked_faces(v, f, torch.from_numpy(mask).cuda(), dil), O.remove_masked_faces(vn, fn, mask, dil))


def test_512_properties():
    v, f = mc_mesh(512, seed=3)
    Fin = f.shape[0]
    info = {}
    vo, fo = M.clean_mesh(v, f, info=info)
    torch.cuda.synchronize()
    vo, fo = vo.cpu().numpy(), fo.cpu().numpy().astype(np.int64)
    vi, fi = v.cpu().numpy(), f.cpu().numpy().astype(np.int64)
    assert 0 < len(fo) < Fin and info["merge_rounds"] >= 2
    # no edge of more than two faces
    a, b = fo.reshape(-1), np.roll(fo, -1, axis=1).reshape(-1)
    _, counts = np.unique(np.minimum(a, b) * len(vo) + np.maximum(a, b), return_counts=True)
    assert counts.max() <= 2
    # every vertex referenced
    assert np.array_equal(np.unique(fo), np.arange(len(vo)))
    # every output vertex sits on an input vertex (leaders and copies keep their positions), and every output face comes from an input
    # face or a split of one: its corners lie, slot by slot, within r of an input face's corners (a merged corner moved to its leader)
    tree = cKDTree(vi.astype(np.float64))
    dist, _ = tree.query(vo.astype(np.float64))
    assert (dist == 0).all()
    r = O.merge_radius(O.bbox_diag(vi), 1) * (1 + 1e-9)
    cin = vi[fi].astype(np.float64)
    cout = vo[fo].astype(np.float64)
    near = cKDTree(cin[:, 0]).query_ball_point(cout[:, 0], r)
    lens = np.array([len(c) for c in near])
    assert (lens > 0).all()
    cand = np.concatenate(near).astype(np.int64)
    owner = np.repeat(np.arange(len(fo)), lens)
    ok = (np.linalg.norm(cin[cand] - cout[owner], axis=2) <= r).all(1)
    assert np.logical_or.reduceat(ok, np.concatenate([[0], np.cumsum(lens)[:-1]])).all()
    # components: edge-connected, each meeting both thresholds (against the output's own diagonal, which is no larger than the one the
    # filter used).  Checked on the clean-up without repair, whose face deletions may split a component.
    vo, fo = (x.cpu().numpy() for x in M.clean_mesh(v, f, repair=False))
    fo = fo.astype(np.int64)
    F = len(fo)
    keys = np.sort(np.stack([fo, np.roll(fo, -1, axis=1)], 2).reshape(-1, 2), 1)
    _, inv = np.unique(keys, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    first = np.full(inv.max() + 1, F); face = np.repeat(np.arange(F), 3)
    np.minimum.at(first, inv, face)
    n, label = connected_components(coo_matrix((np.ones(3 * F), (face, first[inv])), shape=(F, F)), directed=False)
    assert np.bincount(label).min() >= 8
    lo = np.full((n, 3), np.inf); hi = np.full((n, 3), -np.inf)
    for k in range(3):
        np.minimum.at(lo, label, vo[fo[:, k]]); np.maximum.at(hi, label, vo[fo[:, k]])
    assert (np.linalg.norm(hi - lo, axis=1) >= 0.05 * O.bbox_diag(vo) * (1 - 1e-12)).all()


def test_empty_and_degenerate_inputs():
    v, f = C.bowtie()
    vd, fd = _dev(v, f)
    empty_f = torch.empty(0, 3, dtype=torch.int32, device="cuda")
    for out in (M.clean_mesh(vd, empty_f), M.clean_mesh(vd[:0], empty_f), M.remove_masked_faces(vd, empty_f, torch.empty(0, device="cuda"), 3),
                M.remove_masked_faces(vd, fd, torch.ones(4, device="cuda"), 3),             # everything masked
                M.clean_mesh(vd, fd, min_f=100),                                              # every component too small
                M.clean_mesh(vd, fd[[0, 0, 0]], min_f=2, min_d=0),                           # duplicates leave one face: too small
                M.clean_mesh(torch.zeros(3, 3, device="cuda"), fd[:1] * 0 + torch.tensor([0, 1, 2], dtype=torch.int32, device="cuda"))):
        torch.cuda.synchronize()
        assert out[0].shape == (0, 3) and out[1].shape == (0, 3) and out[0].dtype == torch.float32 and out[1].dtype == torch.int32
    # one vertex position for all: the merge radius is 0 and every vertex joins vertex 0
    _check_clean(np.zeros((5, 3), np.float32), np.array([[0, 1, 2], [2, 3, 4]]), min_f=0, min_d=0)


# ---- the exports' clean-up chain ------------------------------------------------------------------------------------------------------
def _train(t0, bricks, steps=3):
    g = torch.Generator().manual_seed(0)
    poses = S.orbit_cameras(100, seed=0)
    for _ in range(steps):
        ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, 1024, g)
        t0.step(ro, rd, S.render_bricks(ro, rd, bricks), torch.rand(1024, 3, generator=g), torch.rand(1024, generator=g), use_graph=False)
    torch.cuda.synchronize()
    return t0


def _np(v, f):
    return v.cpu().numpy(), f.cpu().numpy().astype(np.int64)


@pytest.mark.parametrize("scene", ["bound4", "garden16"])
def test_exports_with_clean_equal_the_oracle_chain(tmp_path, scene):
    if scene == "bound4":
        t0 = _bound4_trainer()
    else:
        t0 = _train(_garden_trainer(), S.garden_scene(bound=16.0)[2])
    views = _views(96, 96, n=4)
    mvps = torch.stack([m for m, *_ in views])
    clean = M.CleanOptions(min_f=8, min_d=5, visibility_mask_dilation=2, mvps=mvps, H=96, W=96)
    # mesh_0: visibility -> remove_masked_faces -> clean_mesh(repair=True)
    v, f = M.export_stage0_mesh(t0, str(tmp_path / "raw"), resolution=128, density_thresh=0.5)
    vc, fc = M.export_stage0_mesh(t0, str(tmp_path / "clean"), resolution=128, density_thresh=0.5, clean=clean)
    assert f.shape[0] > 1000
    unseen = M.mark_unseen_triangles(v, f, mvps, 96, 96).cpu().numpy()
    assert unseen.any() and not unseen.all()
    ref = O.clean_mesh(*O.remove_masked_faces(*_np(v, f), unseen, 2), min_f=8, min_d=5, repair=True)
    _same((vc, fc), ref)
    pv, pf = M.read_ply(tmp_path / "clean" / "mesh_0.ply")
    assert np.array_equal(pv, ref[0]) and np.array_equal(pf, ref[1])
    # without views: clean_mesh alone
    _same(M.export_stage0_mesh(t0, str(tmp_path / "noviews"), resolution=128, density_thresh=0.5, clean=M.CleanOptions()),
          O.clean_mesh(*_np(v, f)))
    # outer cascades: clean_mesh(repair=False) -> visibility -> remove_masked_faces
    raw = M.export_outer_meshes(t0, str(tmp_path / "raw"), env_reso=128)
    out = M.export_outer_meshes(t0, str(tmp_path / "clean"), env_reso=128, clean=clean)
    if scene == "garden16":
        assert len(raw) >= 3
    for cas, (rv, rf) in raw.items():
        cv, cf = O.clean_mesh(*_np(rv, rf), min_f=8, min_d=5, repair=False)
        if len(cv) and len(cf):
            cvd, cfd = _dev(cv, cf)
            m = M.mark_unseen_triangles(cvd, cfd, mvps, 96, 96).cpu().numpy()
            cv, cf = O.remove_masked_faces(cv, cf, m, 2)
        path = tmp_path / "clean" / f"mesh_{cas}.ply"
        if len(cv) == 0:
            assert cas not in out and not path.exists()
            continue
        _same(out[cas], (cv, cf))
        pv, pf = M.read_ply(path)
        assert np.array_equal(pv, cv) and np.array_equal(pf, cf)
    assert set(out) <= set(raw)
