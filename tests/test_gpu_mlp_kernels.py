"""GPU: the stage-0 MLP kernels k_pack_weights, k_mlp_fwd and k_mlp_bwd element by element against the float64 restatement of their
rounding points (tests/mlp_oracle.py).

The kernels are called through their C entry points (n2m_s0_pack_weights, n2m_s0_mlp_fwd, n2m_s0_mlp_bwd) on buffers built here,
never through a trainer step; the test writes M (counters[1]) and the ray-range part boundaries (counters[4..12]) itself.  Rows of
the tile image past M inside the used tiles hold finite junk, tiles past the last hold NaN, `dout` is NaN on every row that is not
owned, and `out` / the denc image start as NaN sentinels.

* Exact probes (mlp_oracle.exact_probes, certified on the CPU): out colours, every denc element and every g_mlp entry equal the
  oracle bit for bit (zeros of either sign count as equal), sigma within the __expf bound, for shading 0 / 1 / 2 and 1 / 2 / 4 / 8
  parts.  Among them: trunc_exp's clamp, the colour clamp's inclusive edge, the specular regulariser on owned rows only, and a
  ReLU unit whose masked gradient overflows fp16.
* Counting probe: identical rows, so that each weight gradient is M times one row's; run at M past every CTA's barrier phases
  and at part tile counts around multiples of the backward's CTA count.
* Dense cases: every element within mlp_oracle.bounds; per-row outputs bit-identical across part counts.
"""
import ctypes

import numpy as np
import pytest
import torch

import mlp_oracle as O
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage0 import S0Params

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module", autouse=True)
def _init():
    call("n2m_s0_init")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _params(shading, lam=0.0):
    p = S0Params()
    p.shading_full = shading
    p.lambda_specular = lam
    return p


class Batch:
    """device buffers of one batch: rows [R, 64] (R <= Mcap), M owned rows, part boundaries"""

    def __init__(self, P, rows, dout, M, bounds=None, Mcap=None, ls=1.0, lam=0.0, seed=0):
        R = rows.shape[0]
        self.M, self.R = M, R
        self.Mcap = Mcap or (R + 127) // 128 * 128 + 256
        self.used = (R + 127) // 128 * 128
        rng = np.random.default_rng(seed)
        img = np.full((self.Mcap, 64), NAN)
        img[:self.used] = O.rh(rng.uniform(-2, 2, (self.used, 64)))       # finite junk in the used tiles past row R
        img[:R] = rows
        self.enc = torch.from_numpy(O.tile_image(img.astype(np.float16))).cuda()
        d = np.full((self.Mcap, 4), NAN, np.float32)
        d[:M] = np.asarray(dout, np.float64)[:M]
        self.dout = torch.from_numpy(d).cuda()
        self.P = torch.from_numpy(np.asarray(P, np.float32)).cuda()
        self.wpack = torch.zeros(O.W_BYTES, dtype=torch.uint8, device="cuda")
        call("n2m_s0_pack_weights", ptr(self.P), ptr(self.wpack), stream())
        self.counters = torch.zeros(16, dtype=torch.int32)
        self.counters[0] = self.counters[1] = M
        self.bounds = list(bounds) if bounds is not None else [M * e // 8 for e in range(9)]
        assert self.bounds[0] == 0 and self.bounds[8] == M and self.bounds == sorted(self.bounds)
        self.counters[4:13] = torch.tensor(self.bounds, dtype=torch.int32)
        self.counters = self.counters.cuda()
        self.ls = torch.tensor([ls] + [0.0] * 7, dtype=torch.float32, device="cuda")
        self.lam = lam

    def fwd(self, shading, nparts=1):
        out = torch.full((self.Mcap, 4), NAN, device="cuda")
        sq = torch.zeros(1, device="cuda")
        p = _params(shading, self.lam)
        for k in range(nparts):
            call("n2m_s0_mlp_fwd", ctypes.byref(p), ptr(self.enc), ptr(self.counters), self.Mcap, ptr(self.wpack), ptr(out), ptr(sq),
                 k, nparts, stream())
        torch.cuda.synchronize()
        return out.cpu().double().numpy(), float(sq.item())

    def bwd(self, shading, nparts=1):
        denc = torch.full((self.Mcap * 64,), NAN, dtype=torch.float16, device="cuda")
        g = torch.zeros(O.P_COUNT, device="cuda")
        p = _params(shading, self.lam)
        for k in range(nparts):
            call("n2m_s0_mlp_bwd", ctypes.byref(p), ptr(self.enc), ptr(self.dout), ptr(self.counters), self.Mcap, ptr(self.wpack),
                 ptr(denc), ptr(g), ptr(self.ls), k, nparts, stream())
        torch.cuda.synchronize()
        return O.untile(denc.cpu().double().numpy(), self.Mcap), g.cpu().double().numpy()

    def check_sentinels(self, out, denc, nparts):
        """rows not owned keep out's NaN; denc rows past M keep NaN with parts (one part writes its whole tiles), and every tile
        past the last used one is untouched"""
        last = (self.M + 127) // 128 * 128           # the rows of the tiles that hold a sample
        assert np.isnan(out[self.M:]).all()
        assert np.isnan(denc[last:]).all()
        tail = denc[self.M:last]
        assert (np.isnan(tail).all() if nparts > 1 else (tail == 0).all())


def _eq(a, b):
    return (a == b) | (np.isnan(a) & np.isnan(b))


# ------------------------------------------------------------------------------------------------------------------------------
# packer
# ------------------------------------------------------------------------------------------------------------------------------
def test_pack_weights_bytes():
    P = np.random.default_rng(0).uniform(-1, 1, O.P_COUNT).astype(np.float32)
    P[:50] *= 1e5                      # past the fp16 range: the packer rounds to inf like __float2half_rn
    b = Batch(P, np.zeros((1, 64)), np.zeros((1, 4)), 1)
    assert (b.wpack.cpu().numpy() == O.pack_weights(P.astype(np.float64))).all()


# ------------------------------------------------------------------------------------------------------------------------------
# exact probes
# ------------------------------------------------------------------------------------------------------------------------------
BOUNDS_190 = [0, 0, 37, 64, 128, 129, 150, 190, 190]          # empty parts, boundaries inside tiles and on tile edges


def _probe_batch(pr):
    R = pr["enc"].shape[0]
    bounds = BOUNDS_190 if pr["M"] == 190 else None
    return Batch(pr["P"], pr["enc"], pr["dout"], pr["M"], bounds=bounds, ls=pr["ls"], lam=pr["lam"], seed=R)


def _check_exact(pr, b, shading, nparts):
    ok, v, c = O.probe_certified(pr, shading)
    assert ok
    M = pr["M"]
    out, sq = b.fwd(shading, nparts)
    assert _eq(out[:M, 1:], v["out"][:M, 1:]).all(), np.argwhere(~_eq(out[:M, 1:], v["out"][:M, 1:]))[:5]
    assert (np.abs(out[:M, 0] - v["out"][:M, 0]) <= O.exp_bound(v["hs"][:M])).all()
    if c["spec_sq"]:
        assert sq == v["spec_sq"], (sq, v["spec_sq"])
    denc, g = b.bwd(shading, nparts)
    b.check_sentinels(out, denc, nparts)
    assert _eq(denc[:M], v["denc"][:M]).all(), np.argwhere(~_eq(denc[:M], v["denc"][:M]))[:5]
    assert _eq(g, v["g"]).all(), [(i, g[i], v["g"][i]) for i in np.flatnonzero(~_eq(g, v["g"]))[:5]]
    assert (denc[:M, 51:] == 0).all()


@pytest.mark.parametrize("nparts", [1, 2, 4, 8])
@pytest.mark.parametrize("shading", [0, 1, 2])
def test_exact_probes(shading, nparts):
    for name, pr in O.exact_probes().items():
        if name == "masked_inf":
            continue
        _check_exact(pr, _probe_batch(pr), shading, nparts)


@pytest.mark.parametrize("nparts", [1, 2, 8])
def test_masked_gradient_overflow_gives_zero_not_nan(nparts):
    """a ReLU unit that is off on every row, whose pre-mask gradient overflows fp16 on the gradient rows: the backward of relu
    selects 0 there (the oracle and torch), where a multiply by the mask would give inf * 0 = NaN in g_mlp and denc"""
    pr = O.exact_probes()["masked_inf"]
    v = O.run(pr["P"], pr["enc"], pr["dout"], 0, pr["M"])
    assert np.abs(v["dH2_acc"][:, pr["inactive_unit"]]).max() > O.OVF
    _check_exact(pr, _probe_batch(pr), 0, nparts)


def test_enc_columns_each_net_does_not_read():
    """junk in enc columns 54..63 changes nothing; columns 3..18 change none of the colour net's outputs or weight gradients,
    columns 19..53 none of the sigma net's"""
    pr = O.exact_probes()["rand0"]
    M = pr["M"]
    rng = np.random.default_rng(5)

    def launch(rows):
        b = Batch(pr["P"], rows, pr["dout"], M, bounds=BOUNDS_190, seed=1)
        out, _ = b.fwd(1, 2)
        denc, g = b.bwd(1, 2)
        return out[:M], denc[:M], g

    base = launch(pr["enc"])
    junk = pr["enc"].copy()
    junk[:, 54:] = O.rh(rng.uniform(-6e4, 6e4, (junk.shape[0], 10)))
    for a, b_ in zip(base, launch(junk)):
        assert _eq(a, b_).all()
    sig = np.r_[O.P_S0:O.P_C0]
    col = np.r_[O.P_C0:O.P_COUNT]
    dens = pr["enc"].copy()
    dens[:, 3:19] = O.rh(rng.uniform(-4, 4, (dens.shape[0], 16)))
    o2 = launch(dens)
    assert _eq(o2[0][:, 1:], base[0][:, 1:]).all() and _eq(o2[2][col], base[2][col]).all()
    assert not _eq(o2[0][:, 0], base[0][:, 0]).all()
    colr = pr["enc"].copy()
    colr[:, 19:54] = O.rh(rng.uniform(-4, 4, (colr.shape[0], 35)))
    o3 = launch(colr)
    assert _eq(o3[0][:, 0], base[0][:, 0]).all() and _eq(o3[2][sig], base[2][sig]).all()
    assert not _eq(o3[0][:, 1:], base[0][:, 1:]).all()


# ------------------------------------------------------------------------------------------------------------------------------
# counting probe: identical rows
# ------------------------------------------------------------------------------------------------------------------------------
def _counting(M, nparts, bounds=None):
    pr = O.exact_probes()["colour_edge"]
    j = int(pr["grad_rows"][0])
    row, d = pr["enc"][j], pr["dout"][j]
    v1 = O.run(pr["P"], row[None], d[None], 0, 1)          # one row's weight-gradient terms
    t = v1["g"]
    # entries whose M-fold sum is exact in fp32 under any order: M |t| <= 2^(lsb(t) + 24)
    exact = (t == 0) | (M * np.abs(t) <= np.exp2(np.minimum(O.lsb_exp(t), 900).astype(np.float64) + 24))
    b = Batch(pr["P"], np.tile(row, (M, 1)), np.tile(d, (M, 1)), M, bounds=bounds, Mcap=(M + 127) // 128 * 128 + 128)
    denc, g = b.bwd(0, nparts)
    want = M * t
    assert (g[exact] == want[exact]).all(), [(i, g[i], want[i]) for i in np.flatnonzero(exact & (g != want))[:5]]
    # the rest: a lost or repeated tile moves a sum by 1 / (tiles) of itself, far past the accumulation bound
    tiles = (M + 127) // 128
    acc = ((tiles + _sms() - 1) // _sms()) * 8 * O.K16 + nparts * _sms() * 2.0 ** -24
    assert (np.abs(g - want) <= acc * np.abs(want)).all()
    assert 1.0 / tiles > 2 * acc
    assert _eq(denc[:M], np.tile(v1["denc"][0], (M, 1))).all()
    return exact.mean()


def test_counting_probe_large_M():
    G = _sms()
    M = 2 * 5 * G * 128 + 77
    frac = _counting(M, 1)
    print(f"\ncounting probe M={M}: {frac:.3f} of the weight-gradient entries exact")
    _counting(M, 2, bounds=[0, M // 8, M // 4, 3 * M // 8, M // 2, 5 * M // 8, 3 * M // 4, 7 * M // 8, M])


@pytest.mark.parametrize("which", ["1", "2", "3", "G-1", "G+1", "2G-1", "2G+1"])
def test_counting_probe_tile_counts(which):
    G = _sms()
    tiles = {"1": 1, "2": 2, "3": 3, "G-1": G - 1, "G+1": G + 1, "2G-1": 2 * G - 1, "2G+1": 2 * G + 1}[which]
    _counting(tiles * 128 - 5, 1)


# ------------------------------------------------------------------------------------------------------------------------------
# dense cases
# ------------------------------------------------------------------------------------------------------------------------------
def _linear_params(seed):
    rng = np.random.default_rng(seed)
    P = np.zeros(O.P_COUNT)
    for off, o, i in O.LAYERS.values():
        P[off:off + o * i] = rng.uniform(-1, 1, o * i) / np.sqrt(i)
    return P.astype(np.float32).astype(np.float64)


def _dense_rows(seed, n):
    rng = np.random.default_rng(seed)
    A = np.zeros((n, 64))
    A[:, :3] = rng.uniform(-1, 1, (n, 3))
    A[:, 3:51] = rng.normal(0, 1.5, (n, 48))
    dvec = rng.normal(0, 1, (n, 3))
    A[:, 51:54] = dvec / np.linalg.norm(dvec, axis=1, keepdims=True)
    return O.rh(A)


def _check_dense(P, rows, dout, M, shading, ls, lam, bounds_list):
    v = O.run(P, rows, dout, shading, M, ls, lam)
    tiles = (rows.shape[0] + 127) // 128
    ref = None
    for nparts, bounds in bounds_list:
        b = Batch(P, rows, dout, M, bounds=bounds, ls=ls, lam=lam, seed=M)
        bd = O.bounds(v, ctas_per_part=nparts * _sms(), tiles_per_cta=(tiles + _sms() - 1) // _sms())
        out, sq = b.fwd(shading, nparts)
        denc, g = b.bwd(shading, nparts)
        b.check_sentinels(out, denc, nparts)
        for got, want, d in ((out[:M], v["out"][:M], bd["out"][:M]), (denc[:M], v["denc"][:M], bd["denc"][:M]), (g, v["g"], bd["g"])):
            assert np.isfinite(got[np.isfinite(d)]).all()
            err = np.abs(got - want)
            assert (err <= d).all(), (np.argwhere(~(err <= d))[:5], err[~(err <= d)][:5], d[~(err <= d)][:5])
        assert abs(sq - v["spec_sq"]) <= bd["spec_sq"]
        if ref is None:
            ref = (out, denc)
        else:            # per-row arithmetic: identical whatever the part count
            assert _eq(out[:M], ref[0][:M]).all() and _eq(denc[:M], ref[1][:M]).all()
    return bd["identical_fraction"]


def _bounds_for(M):
    """part boundaries inside tiles, on tile edges, and empty parts"""
    fix = lambda b: sorted(min(max(x, 0), M) for x in b)
    return [(1, None), (2, fix([0, M // 8, M // 4, M // 3, M // 2, M // 2, 3 * M // 4, 7 * M // 8, M])),
            (4, fix([0, 0, 128 * (M // 256), 128 * (M // 256), M // 2 + 1, M // 2 + 1, M - 1, M, M])),
            (8, [M * e // 8 for e in range(9)])]


@pytest.mark.parametrize("M", [1, 77, 127, 128, 129, 20000 + 77])
@pytest.mark.parametrize("shading", [0, 1])
def test_dense_random_within_bound(M, shading):
    R = M + (17 if M % 128 else 0)
    rows = _dense_rows(M, R)
    rng = np.random.default_rng(M + 1)
    dout = rng.normal(0, 64.0, (R, 4)).astype(np.float32).astype(np.float64)
    _check_dense(_linear_params(M), rows, dout, M, shading, 65536.0, 1e-5, _bounds_for(M))


def test_overflowing_loss_scale_gives_non_finite():
    """upstream gradients at which the oracle overflows fp16: the kernels must produce a non-finite denc or g_mlp entry (that is
    what the step's found_inf check sees), while at 1/2^16 of that scale every output is finite"""
    M = 300
    P = _linear_params(3)
    rows = _dense_rows(3, M)
    dout = np.random.default_rng(4).normal(0, 1, (M, 4))
    big = dout * 2.0 ** 26
    v = O.run(P, rows, big, 1, M)
    assert not (np.isfinite(v["denc"][:, 3:51]).all() and np.isfinite(v["g"]).all())
    b = Batch(P, rows, big, M)
    denc, g = b.bwd(1)
    assert not (np.isfinite(denc[:M, 3:51]).all() and np.isfinite(g).all())
    small = dout * 2.0 ** 10
    v = O.run(P, rows, small, 1, M)
    bd = O.bounds(v, _sms(), 1)
    assert np.isfinite(bd["denc"]).all() and np.isfinite(bd["g"]).all()
    denc, g = Batch(P, rows, small, M).bwd(1)
    assert np.isfinite(denc[:M]).all() and np.isfinite(g).all()


@pytest.mark.parametrize("case", ["lego", "garden"])
def test_trainer_batches_within_bound(case):
    """a Stage0Trainer's own enc_tiles, dout and packed weights after a few steps on the test batches, at loss scale 65536"""
    import cases
    from nerf2mesh_b200 import synthetic as S
    from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer
    mc = cases.march_case({"lego": "lego_converged", "garden": "garden_cascades"}[case])
    N = mc["rays_o"].shape[0]
    cfg = Stage0Config(bound=mc["bound"], num_rays=N, max_samples=N * 256, loss_scale=65536.0)
    tr = Stage0Trainer(cfg, seed=1)
    grid, bits, _ = S.occupancy_regime("converged", H=128, cascades=cfg.cascade, bound=min(mc["bound"], 2.0 ** (cfg.cascade - 1)))
    tr.set_occupancy(bits, grid)
    g = torch.Generator().manual_seed(2)
    gt = torch.rand(N, 4, generator=g)
    bg = torch.rand(N, 3, generator=g)
    for _ in range(3):
        tr.step(mc["rays_o"], mc["rays_d"], gt, bg, mc["noises"], use_graph=False)
    tr.slots[tr.cur].load(mc["rays_o"].cuda(), mc["rays_d"].cuda(), gt.cuda(), bg.cuda(), mc["noises"].cuda())
    tr.loss_acc.zero_()
    for s in ("march", "encode_fwd", "mlp_fwd", "composite_loss"):
        getattr(tr, s)()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    assert M > 128
    used = (M + 127) // 128 * 128
    rows = O.untile(tr.enc_tiles.cpu().double().numpy(), used)[:M]
    dout = tr.dout[:M].cpu().double().numpy()
    P = tr.mlp.cpu().double().numpy()
    frac = _check_dense(P, rows, dout, M, 1, 65536.0, cfg.lambda_specular, _bounds_for(M)[:2])
    print(f"\n{case}: M={M}, rounding points certified identical {frac:.4f}")
