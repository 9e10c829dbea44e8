"""CPU: the float64 restatement of the stage-0 MLP kernels (tests/mlp_oracle.py) against torch float64 autograd, its packer against
the packed layout of mlp_common.cuh / wg.cuh, its exact probes' certificates and coverage, and its error bound against an
independent fp32 simulation of the kernels' arithmetic.  No GPU needed."""
import numpy as np
import pytest
import torch

import mlp_oracle as O
from oracle import train_oracle as T

F32 = np.float32


def _params(seed):
    """nn.Linear default init (U(-1/sqrt(in), 1/sqrt(in))), flat reference layout"""
    rng = np.random.default_rng(seed)
    P = np.zeros(O.P_COUNT)
    for off, o, i in O.LAYERS.values():
        P[off:off + o * i] = rng.uniform(-1, 1, o * i) / np.sqrt(i)
    return P


def _rows(seed, n, scale=1.0):
    rng = np.random.default_rng(seed)
    A = np.zeros((n, 64))
    A[:, :3] = rng.uniform(-1, 1, (n, 3))
    A[:, 3:51] = rng.normal(0, scale, (n, 48))
    d = rng.normal(0, 1, (n, 3))
    A[:, 51:54] = d / np.linalg.norm(d, axis=1, keepdims=True)
    return O.rh(A)


# ------------------------------------------------------------------------------------------------------------------------------
# rounding points off == OracleField(amp=False) under float64 autograd
# ------------------------------------------------------------------------------------------------------------------------------
def _torch_reference(P, A, dout, shading, M, ls, lam):
    field = T.OracleField(1.0, log2_hashmap_size=8).double()
    with torch.no_grad():
        for name, (off, o, i) in O.LAYERS.items():
            mod = {"s": field.sigma_net, "c": field.color_net, "p": field.specular_net}[name[0]]
            mod.net[int(name[1])].weight.copy_(torch.from_numpy(P[off:off + o * i].reshape(o, i)))
    At = torch.from_numpy(A).clone().requires_grad_(True)
    x, hd, hc, d = At[:, 0:3], At[:, 3:19], At[:, 19:51], At[:, 51:54]
    orig = T.grid_encode
    T.grid_encode = lambda x01, emb, *a, **k: hd if emb.shape[1] == 1 else hc       # the encodings are the tile's columns
    try:
        sigma, colour, spec = field(x, d.detach(), {0: "diffuse", 1: "full", 2: "full"}[shading], amp=False)
    finally:
        T.grid_encode = orig
    own = torch.arange(A.shape[0]) < M
    out = torch.cat([sigma[:, None], spec if shading == 2 else colour], 1)
    D = torch.from_numpy(np.nan_to_num(dout)) * own[:, None]
    loss = (out * D).sum() if shading != 2 else (torch.cat([sigma[:, None], colour], 1) * D).sum()
    if shading != 0:
        loss = loss + lam * ls / M * (spec[own] ** 2).sum()
    ws = [m.weight for m in (*field.sigma_net.net, *field.color_net.net, *field.specular_net.net)]
    grads = torch.autograd.grad(loss, [At] + ws, allow_unused=True)
    g = np.concatenate([(gw if gw is not None else torch.zeros_like(w)).reshape(-1).numpy() for gw, w in zip(grads[1:], ws)])
    return out.detach().numpy(), grads[0].numpy(), g


@pytest.mark.parametrize("shading", [0, 1, 2])
def test_unrounded_oracle_is_the_float64_network(shading):
    rng = np.random.default_rng(shading)
    P = _params(3)
    A = _rows(4, 200, scale=2.0)
    A[:5, 3:19] = 0
    # sigma pre-activations at and past trunc_exp's clamp: sigma_net.0 units 0 / 1 read columns 3 / 4, sigma_net.1 = unit 0 - unit 1
    t = np.array([20.0, 15.0, 0.0, -15.0, -20.0])
    A[:5, 3], A[:5, 4] = np.maximum(t, 0), np.maximum(-t, 0)
    s0 = P[O.P_S0:O.P_S0 + 32 * 19].reshape(32, 19)
    s0[:2] = 0
    s0[0, 3] = s0[1, 4] = 1.0
    P[O.P_S1:O.P_S1 + 32] = 0
    P[O.P_S1], P[O.P_S1 + 1] = 1.0, -1.0
    dout = rng.normal(0, 1, (200, 4))
    M = 190
    dout[M:] = np.nan
    v = O.run(P, A, dout, shading, M, loss_scale=8.0, lam_spec=0.05, rnd=False)
    out, denc, g = _torch_reference(P, A, dout, shading, M, 8.0, 0.05)
    np.testing.assert_allclose(v["out"], out, rtol=1e-12, atol=1e-12)
    assert (v["hs"][:5] == t).all()
    denc_ref = np.zeros_like(denc)
    denc_ref[:, :51] = denc[:, :51]                     # the direction has no gradient: denc columns 51.. are zero
    np.testing.assert_allclose(v["denc"], denc_ref, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(v["g"], g, rtol=1e-10, atol=1e-12)
    if shading:
        assert v["clamp_pass"].mean() < 1 and v["clamp_pass"].mean() > 0


def test_unrounded_clamp_is_inclusive():
    """the colour clamp's gradient passes at exactly 0 and 1, like torch.clamp's backward"""
    P = np.zeros(O.P_COUNT)
    A = np.zeros((2, 64))
    dout = np.ones((2, 4))
    v = O.run(P, A, dout, 1, rnd=False)            # every pre-activation 0: feat = sp = 0.5, colour = 1.0 exactly
    assert (v["cs"] == 1.0).all() and v["clamp_pass"].all()
    out, denc, g = _torch_reference(P, A, dout, 1, 2, 1.0, 0.0)
    np.testing.assert_allclose(v["g"], g, rtol=1e-12, atol=1e-15)


# ------------------------------------------------------------------------------------------------------------------------------
# packer
# ------------------------------------------------------------------------------------------------------------------------------
def test_packer_places_every_parameter():
    P = (np.arange(O.P_COUNT) + 0x3C00).astype(np.uint16).view(np.float16).astype(np.float64)     # distinct fp16 values from 1.0 up
    h = O.pack_weights(P).view(np.float16).astype(np.float64)
    seen = np.zeros(h.size, bool)
    where = {"s0": ("s1", lambda o, i: (o, i)), "s1": ("s2", lambda o, i: (o, i)), "c0": ("c1", lambda o, i: (o, i if i < 3 else i + 16)),
             "c1": ("c2", lambda o, i: (o, i)), "c2": ("c3", lambda o, i: (o, i)), "p0": ("p1", lambda o, i: (o, i)),
             "p1": ("p2", lambda o, i: (o, i))}
    for name, (off, nout, nin) in O.LAYERS.items():
        tile, rc = where[name]
        base, rows, _ = O.PACK[tile]
        for o in range(nout):
            for i in range(nin):
                r, c = rc(o, i)
                e = (base + O.tile_off(r, c, rows)) // 2
                assert h[e] == P[off + o * nin + i], (name, o, i)
                assert not seen[e]
                seen[e] = True
    assert seen.sum() == O.P_COUNT
    assert (h[~seen] == 0).all()


def test_tile_image_layout():
    rows = np.arange(256 * 64, dtype=np.float64).reshape(256, 64)
    img = O.tile_image(rows)
    for r, c in [(0, 0), (5, 9), (127, 63), (128, 0), (200, 51)]:
        assert img[(r // 128) * 8192 + O.tile_off(r % 128, c, 128) // 2] == rows[r, c]
    assert (O.untile(img, 256) == rows).all()


# ------------------------------------------------------------------------------------------------------------------------------
# exact probes: certificates and coverage
# ------------------------------------------------------------------------------------------------------------------------------
def test_probe_certificates_and_coverage():
    probes = O.exact_probes()
    cover_g = np.zeros(O.P_COUNT, bool)
    cover_p = np.zeros(O.P_COUNT, bool)
    for name, pr in probes.items():
        for shading in (0, 1):
            ok, v, c = O.probe_certified(pr, shading)
            assert ok, (name, shading)
            assert c["spec_sq"] or shading == 1
            cover_g |= v["g"] != 0
            cover_p |= (v["g"] != 0) & (pr["P"] != 0)
        if not name.startswith("rand"):
            continue
        # random probes: pairwise distinct magnitudes within every weight row, both signs in use
        for lname, (off, o, i) in O.LAYERS.items():
            W = np.abs(pr["P"][off:off + o * i].reshape(o, i))
            for row in W:
                nz = row[row != 0]
                assert len(np.unique(nz)) == len(nz), (name, lname)
        assert (pr["P"] < 0).any() and (pr["P"] > 0).any()
    print(f"\nexact probes: {len(probes)}; weight-gradient entries nonzero in some probe {cover_g.mean():.4f}, "
          f"parameters nonzero where their gradient is {cover_p.mean():.4f}")
    assert cover_g.all(), np.flatnonzero(~cover_g)
    assert cover_p.mean() > 0.65


def test_special_probes_hit_their_edges():
    p = O.exact_probes()
    for t in O.SIGMA_TARGETS:
        pr = p[f"sigma_{t:+.0f}"]
        v = O.run(pr["P"], pr["enc"], pr["dout"], 1, pr["M"])
        assert (v["hs"] == t).all() and v["dOs"][0] != 0
    pr = p["colour_edge"]
    v = O.run(pr["P"], pr["enc"], pr["dout"], 1, pr["M"])
    assert (v["cs"][:, 0] == 1.0).all() and v["clamp_pass"][:, 0].all()
    assert (v["cs"][:, 1] == 1.0 + 2.0 ** -10).all() and not v["clamp_pass"][:, 1].any()
    pr = p["masked_inf"]
    j = pr["inactive_unit"]
    v = O.run(pr["P"], pr["enc"], pr["dout"], 0, pr["M"])
    assert (v["h2"][:, j] == 0).all() and np.abs(v["dH2_acc"][:, j]).max() > O.OVF
    active = v["h2"] > 0
    assert np.isfinite(O.rh(v["dH2_acc"][active])).all()
    assert np.isfinite(v["g"]).all() and np.isfinite(v["denc"]).all()
    pr = p["spec_reg"]
    assert pr["lam"] != 0 and pr["M"] == 2


# ------------------------------------------------------------------------------------------------------------------------------
# the bound against an independent fp32 simulation
# ------------------------------------------------------------------------------------------------------------------------------
class Sim32:
    """The kernels' arithmetic in numpy fp32: each GEMM in k16 steps taken in a random order, each step's sum truncated toward zero
    to fp32; __expf and the fast reciprocal with random errors inside their documented bounds; weight gradients summed per CTA over
    a random split of the tiles, then added in a random order."""

    def __init__(self, seed, ctas):
        self.rng = np.random.default_rng(seed)
        self.ctas = ctas

    def trunc32(self, x):
        y = x.astype(F32)
        over = np.abs(y.astype(np.float64)) > np.abs(x)
        return np.where(over, np.nextafter(y, F32(0)), y)

    def mm(self, X, Wt):
        X, Wt = np.asarray(X, np.float64), np.asarray(Wt, np.float64)
        K = X.shape[1]
        acc = np.zeros((X.shape[0], Wt.shape[1]), F32)
        for s in self.rng.permutation((K + 15) // 16):
            acc = self.trunc32(acc.astype(np.float64) + X[:, 16 * s:16 * s + 16] @ Wt[16 * s:16 * s + 16])
        return acc.astype(np.float64)

    def expf(self, x):
        e = np.exp(x)
        # (ulp - 1) half-ulps of error, then the rounding to fp32: within the documented ulp count
        return (e * (1 + self.rng.uniform(-1, 1, np.shape(x)) * (O.EXP_ULP(x) - 1) * 2.0 ** -24)).astype(F32).astype(np.float64)

    def sig(self, x):
        x = O.rh(x)
        t = (1 + self.expf(-x)).astype(F32).astype(np.float64)
        return O.rh((1 / t) * (1 + self.rng.uniform(-2, 2, np.shape(x)) * O.U32))

    def wgrad(self, d, a):
        n = a.shape[0]
        tiles = np.arange((n + 127) // 128)
        owner = self.rng.integers(0, self.ctas, len(tiles))
        parts = []
        for c in range(self.ctas):
            rows = np.concatenate([np.arange(128 * t, min(128 * t + 128, n)) for t in tiles[owner == c]] + [np.zeros(0, int)])
            if len(rows):
                parts.append(self.mm(d[rows].T, a[rows]))
        tot = np.zeros(parts[0].shape, F32)
        for k in self.rng.permutation(len(parts)):
            tot = (tot + parts[k].astype(F32))
        return tot.astype(np.float64)

    def run(self, P, A, dout, shading, M, ls, lam):
        W = {k: O.rh(w) for k, w in O.padded(P).items()}
        f32 = lambda x: np.asarray(x, F32).astype(np.float64)
        R = A.shape[0]
        own = np.arange(R) < M
        relu_h = lambda x: np.maximum(O.rh(x), 0)
        h1, s1 = relu_h(self.mm(A, W["c1"].T)), relu_h(self.mm(A, W["s1"].T))
        hs = O.rh(self.mm(s1, W["s2"][:1].T)[:, 0])
        sigma = self.expf(hs)
        h2 = relu_h(self.mm(h1, W["c2"].T))
        feat = self.sig(self.mm(h2, W["c3"][:6].T))
        full = shading != 0
        sp = np.zeros((R, 3))
        col = feat[:, :3]
        if full:
            as2 = np.concatenate([A[:, 51:54], feat[:, 3:6]], 1)
            p1 = relu_h(self.mm(as2, W["p1"][:, :6].T))
            sp = self.sig(self.mm(p1, W["p2"][:3].T))
            cs = O.rh(f32(sp + feat[:, :3]))
            col = np.clip(cs, 0, 1)
        out = np.concatenate([sigma[:, None], sp if shading == 2 else col], 1)
        dv = np.where(own[:, None], np.nan_to_num(dout), 0.0)
        spec_reg = f32(f32(2 * lam / M * (1 + self.rng.uniform(-2, 2) * O.U32)) * ls)
        g = dv[:, 1:4]
        if full:
            g = np.where((cs >= 0) & (cs <= 1), g, 0.0)
            dsp = np.where(own[:, None], f32(g + spec_reg * sp), 0.0)
            dO2 = O.rh(f32(f32(dsp * sp) * f32(1 - sp)))
        dOs = O.rh(f32(dv[:, 0] * self.expf(np.clip(hs, -15, 15))))
        dS1 = np.where(s1 > 0, O.rh(self.mm(dOs[:, None], W["s2"][:1])), 0.0)
        dfeat = np.zeros((R, 6))
        dfeat[:, :3] = g
        if full:
            dP1 = np.where(p1 > 0, O.rh(self.mm(dO2, W["p2"][:3])), 0.0)
            dfeat[:, 3:6] = self.mm(dP1, W["p1"][:, :6])[:, 3:6]
        dO = O.rh(f32(f32(dfeat * feat) * f32(1 - feat)))
        dH2 = np.where(h2 > 0, O.rh(self.mm(dO, W["c3"][:6])), 0.0)
        dH1 = np.where(h1 > 0, O.rh(self.mm(dH2, W["c2"])), 0.0)
        denc = O.rh(self.mm(np.concatenate([dS1, dH1], 1), np.concatenate([W["s1"], W["c1"]], 0)))
        gs = {"s0": self.wgrad(dS1, A[:, O.S0_COLS]), "s1": self.wgrad(dOs[:, None], s1), "c0": self.wgrad(dH1, A[:, O.C0_COLS]),
              "c1": self.wgrad(dH2, h1), "c2": self.wgrad(dO, h2)}
        if full:
            gs["p0"] = self.wgrad(dP1, as2)
            gs["p1"] = self.wgrad(dO2, p1)
        return out, denc, O._flat(gs)


@pytest.mark.parametrize("shading", [0, 1])
def test_bound_holds_for_fp32_simulation(shading):
    M, ctas = 700, 4
    P = _params(10 + shading)
    A = _rows(11, M, scale=1.5)
    rng = np.random.default_rng(12)
    dout = rng.normal(0, 64, (M, 4)).astype(F32).astype(np.float64)
    v = O.run(P, A, dout, shading, M, loss_scale=65536.0, lam_spec=1e-5)
    b = O.bounds(v, ctas_per_part=ctas, tiles_per_cta=(M + 127) // 128)
    print(f"\nshading {shading}: rounding points certified identical {b['identical_fraction']:.4f}")
    for seed in range(3):
        out, denc, g = Sim32(seed, ctas).run(P, A, dout, shading, M, 65536.0, 1e-5)
        assert (np.abs(out[:, 1:] - v["out"][:, 1:]) <= b["out"][:, 1:]).all()
        assert (np.abs(out[:, 0] - v["out"][:, 0]) <= b["out"][:, 0]).all()
        assert (np.abs(denc - v["denc"]) <= b["denc"]).all()
        assert (np.abs(g - v["g"]) <= b["g"]).all()
    assert b["identical_fraction"] > 0
