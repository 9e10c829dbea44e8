"""float64 restatement of the stage-0 tensor-core MLP kernels k_pack_weights, k_mlp_fwd and k_mlp_bwd (csrc/mlp_tc.cu,
csrc/mlp_common.cuh), written from the kernels' own rounding points:

  * every GEMM accumulates in fp32 and its output is rounded to fp16 (round_h); ReLU acts on the fp16 value, and the backward mask of
    a ReLU layer is `fp16 activation > 0`, applied as a select after the pre-mask gradient has been rounded to fp16
  * sigmoid_h(a) = round_h(1 / (1 + exp(-round_h(a))));  sigma = exp(round_h(h)) in fp32;  trunc_exp's backward clamps at +-15
  * colour (full shading) = clamp(round_h(sp + feat), 0, 1); its backward passes where 0 <= round_h(sp + feat) <= 1 (inclusive)
  * dOs = round_h(dout.x * exp(clamp(h))), dO2 = round_h(dsp * sp * (1 - sp)), dO = round_h(dfeat * feat * (1 - feat)) are formed in
    fp32; dsp = g + spec_reg * sp on owned rows only, spec_reg = 2 * lambda_specular / M * loss_scale with M = counters[1];
    dfeat[0:3] is the clamped colour gradient, dfeat[3:6] comes straight from the fp32 accumulators of the specular input gradient
  * the specular input is [enc columns 51..53 (direction), feat[3:6]]; shading 0 = diffuse, 1 = full, 2 = specular (forward only:
    out.yzw = sp; the backward treats 2 as full)

Where these differ from torch.autocast(fp16) in the reference (not restated here; the step-level tests cover them): autocast
rounds the ReLU output and its backward mask in the same places, but it runs sigmoid / exp on fp16 tensors with torch's own
transcendental implementations instead of __expf and a fast reciprocal, keeps the fp32 per-sample chain rule in fp16 tensor ops
(GradScaler-scaled fp16 gradients), and rounds dfeat[3:6] to fp16 before the sigmoid backward.

`run(..., rnd=False)` drops every rounding point and is then the float64 network of oracle/train_oracle.OracleField with amp=False.

For the values `run` returns it also reports one of two things:
  * `certify`: whether every value is certified identical to the kernel's.  A GEMM output is exact when all its terms are integer
    multiples of 2^e and sum(|terms|) <= 2^(e+24): then every partial sum is an fp32 value, in any order and under any truncating
    alignment of the tensor core (the weight-gradient sums over all samples and CTAs likewise).  A value that comes from __expf or
    the fast reciprocal must lie farther from every fp16 rounding boundary than that function's documented error: __expf
    2 + floor(1.173 |x|) ulp (CUDA Math API), fast-math division 2 ulp, plus the fp32 roundings of the per-sample chain.
  * `bounds`: a first-order worst-case bound on |kernel - oracle| for every output, from this tensor-core model: products exact,
    each k16 step adds 16 products to the running fp32 sum, and each of those 17 addends may lose every bit below the 24-bit window
    of the largest of them (so a step errs by less than 17 * 2^-23 * sum|terms so far|).  A weight gradient is one such chain of
    k16 steps per CTA over its tiles, then one fp32 atomic add per CTA and part.  A rounding point whose bound interval holds no
    fp16 rounding boundary gets delta = 0, so exactness propagates; otherwise delta + one fp16 ulp.  A mask or clamp whose operand
    interval straddles its edge takes the union of both branches, and a value whose interval reaches 65520 (fp16 overflow) is
    possibly non-finite (delta = inf).
"""
import functools

import numpy as np

F16, F32, F64 = np.float16, np.float32, np.float64
TILE = 128
P_S0, P_S1, P_C0, P_C1, P_C2, P_P0, P_P1, P_COUNT = 0, 608, 640, 2880, 6976, 7360, 7552, 7648
# name -> (flat offset, out, in) of the reference nn.Linear weights [out, in]
LAYERS = {"s0": (P_S0, 32, 19), "s1": (P_S1, 1, 32), "c0": (P_C0, 64, 35), "c1": (P_C1, 64, 64), "c2": (P_C2, 6, 64),
          "p0": (P_P0, 32, 6), "p1": (P_P1, 3, 32)}
# packed tiles (mlp_common.cuh W_*): name -> (byte offset, padded rows = out, padded cols = in)
W_BYTES = 25600
PACK = {"c1": (0, 64, 64), "c2": (8192, 64, 64), "c3": (16384, 16, 64), "s1": (18432, 32, 64), "s2": (22528, 16, 32),
        "p1": (23552, 32, 16), "p2": (24576, 16, 32)}
COL_DIR = 51
C0_COLS = np.r_[0:3, 19:51]            # enc tile column of each color_net.0 input
S0_COLS = np.arange(19)                # enc tile column of each sigma_net.0 input
EXP_ULP = lambda x: 2.0 + np.floor(1.173 * np.abs(x))       # __expf error in ulp (CUDA Math API)
U32 = 2.0 ** -23
K16 = 17 * U32                          # error of one k16 step per unit of sum|terms| (tensor-core model above)
OVF = 65520.0


def map_c1(c):
    return c if c < 3 else c - 16 if 19 <= c < 51 else -1


def map_s1(c):
    return c if c < 19 else -1


def rh(x, on=True):
    """fp16 round-to-nearest-even of float64 values (inf past 65520)"""
    if not on:
        return np.asarray(x, F64)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x, F64).astype(F16).astype(F64)


def layer(P, name):
    off, o, i = LAYERS[name]
    return np.asarray(P[off:off + o * i], F64).reshape(o, i)


def padded(P):
    """the seven packed weight matrices [rows = out (padded), cols = in (padded)], float64"""
    W = {k: np.zeros(v[1:]) for k, v in PACK.items()}
    W["c1"][:, C0_COLS] = layer(P, "c0")
    W["s1"][:, S0_COLS] = layer(P, "s0")
    W["c2"][:] = layer(P, "c1")
    W["c3"][:6] = layer(P, "c2")
    W["s2"][:1] = layer(P, "s1")
    W["p1"][:, :6] = layer(P, "p0")
    W["p2"][:3] = layer(P, "p1")
    return W


def tile_off(r, c, rows):
    """byte offset of element (r, c) of a chunk-major fp16 tile with `rows` rows (wg.cuh)"""
    return (c >> 3) * (rows << 4) + (r >> 3) * 128 + (r & 7) * 16 + (c & 7) * 2


def pack_weights(P):
    """the packer's bytes: fp16 chunk-major tiles of the padded matrices, padding zero -> uint8 [W_BYTES]"""
    out = np.zeros(W_BYTES // 2, F16)
    W = padded(P)
    for name, (base, R, C) in PACK.items():
        r, c = np.meshgrid(np.arange(R), np.arange(C), indexing="ij")
        out[(base + tile_off(r, c, R)) // 2] = W[name].astype(F16)
    return out.view(np.uint8)


def tile_image(rows):
    """[Mcap, 64] rows -> flat tile image [Mcap / 128][8 chunks][128 rows][8 columns]"""
    rows = np.asarray(rows)
    return rows.reshape(-1, TILE, 8, 8).transpose(0, 2, 1, 3).reshape(-1)


def untile(img, n):
    """flat tile image -> its first n (multiple of 128) rows [n, 64]"""
    return np.asarray(img)[: n * 64].reshape(n // TILE, 8, TILE, 8).transpose(0, 2, 1, 3).reshape(n, 64)


def _sigmoid(x):
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-x))


# ----------------------------------------------------------------------------------------------------------------------------------
# forward and backward
# ----------------------------------------------------------------------------------------------------------------------------------
def run(P, enc, dout=None, shading=1, M=None, loss_scale=1.0, lam_spec=0.0, rnd=True):
    """The kernels' arithmetic on rows enc [R, 64] (rows >= M are not owned: no output, zero upstream gradient, no regulariser).
    Returns a dict of every intermediate: *_acc are GEMM outputs before rounding, then `out` [R,4], `spec_sq` (sum over owned rows),
    and with dout: `denc` [R,64] and the flat weight gradient `g` [P_COUNT] (specular layers only with shading != 0)."""
    r = lambda x: rh(x, rnd)
    A = np.asarray(enc, F64)
    R = A.shape[0]
    M = R if M is None else M
    own = np.arange(R) < M
    W = padded(P)
    if rnd:
        W = {k: rh(w) for k, w in W.items()}
    full = shading != 0
    v = dict(A=A, W=W, own=own, M=M, shading=shading, full=full, rnd=rnd, loss_scale=loss_scale, lam_spec=lam_spec)
    v["h1_acc"] = A @ W["c1"].T
    v["h1"] = np.maximum(r(v["h1_acc"]), 0)
    v["s1_acc"] = A @ W["s1"].T
    v["s1"] = np.maximum(r(v["s1_acc"]), 0)
    v["hs_acc"] = v["s1"] @ W["s2"][0]
    v["hs"] = r(v["hs_acc"])
    with np.errstate(over="ignore"):
        v["sigma"] = np.exp(v["hs"])
    v["h2_acc"] = v["h1"] @ W["c2"].T
    v["h2"] = np.maximum(r(v["h2_acc"]), 0)
    v["x_acc"] = v["h2"] @ W["c3"][:6].T
    v["x"] = r(v["x_acc"])
    v["feat"] = r(_sigmoid(v["x"]))
    sp = np.zeros((R, 3))
    colour = v["feat"][:, :3]
    if full:
        v["as2"] = np.concatenate([A[:, COL_DIR:COL_DIR + 3], v["feat"][:, 3:6]], 1)
        v["p1_acc"] = v["as2"] @ W["p1"][:, :6].T
        v["p1"] = np.maximum(r(v["p1_acc"]), 0)
        v["y_acc"] = v["p1"] @ W["p2"][:3].T
        v["y"] = r(v["y_acc"])
        sp = r(_sigmoid(v["y"]))
        v["cs_pre"] = sp + v["feat"][:, :3]
        v["cs"] = r(v["cs_pre"])
        colour = np.clip(v["cs"], 0.0, 1.0)
    v["sp"] = sp
    v["colour"] = colour
    v["out"] = np.concatenate([v["sigma"][:, None], sp if shading == 2 else colour], 1)
    v["spec_sq_terms"] = np.where(own[:, None], sp * sp, 0.0)
    v["spec_sq"] = v["spec_sq_terms"].sum()
    if dout is None:
        return v

    dv = np.where(own[:, None], np.nan_to_num(np.asarray(dout, F64)), 0.0)
    v["dv"] = dv
    dcol = dv[:, 1:4]
    dfeat = np.zeros((R, 6))
    v["spec_reg"] = spec_reg = 2.0 * lam_spec / M * loss_scale if M > 0 else 0.0
    if full:
        v["clamp_pass"] = (v["cs"] >= 0) & (v["cs"] <= 1)
        g = np.where(v["clamp_pass"], dcol, 0.0)
        v["dsp"] = np.where(own[:, None], g + spec_reg * sp, 0.0)
        v["dO2_pre"] = v["dsp"] * sp * (1.0 - sp)
        v["dO2"] = r(v["dO2_pre"])
    else:
        g = dcol
    dfeat[:, :3] = g
    v["hs_clamp"] = np.clip(v["hs"], -15.0, 15.0)
    v["dOs_pre"] = dv[:, 0] * np.exp(v["hs_clamp"])
    v["dOs"] = r(v["dOs_pre"])
    v["dS1_acc"] = v["dOs"][:, None] * W["s2"][0][None, :]
    v["dS1"] = np.where(v["s1"] > 0, r(v["dS1_acc"]), 0.0)
    if full:
        v["dP1_acc"] = v["dO2"] @ W["p2"][:3]
        v["dP1"] = np.where(v["p1"] > 0, r(v["dP1_acc"]), 0.0)
        v["dAs2"] = v["dP1"] @ W["p1"][:, :6]
        dfeat[:, 3:6] = v["dAs2"][:, 3:6]
    v["dfeat"] = dfeat
    v["dO_pre"] = dfeat * v["feat"] * (1.0 - v["feat"])
    v["dO"] = r(v["dO_pre"])
    v["dH2_acc"] = v["dO"] @ W["c3"][:6]
    v["dH2"] = np.where(v["h2"] > 0, r(v["dH2_acc"]), 0.0)
    v["dH1_acc"] = v["dH2"] @ W["c2"]
    v["dH1"] = np.where(v["h1"] > 0, r(v["dH1_acc"]), 0.0)
    v["denc_acc"] = v["dS1"] @ W["s1"] + v["dH1"] @ W["c1"]
    v["denc"] = r(v["denc_acc"])
    gs = {"s0": v["dS1"].T @ A[:, S0_COLS], "s1": v["dOs"][None, :] @ v["s1"], "c0": v["dH1"].T @ A[:, C0_COLS],
          "c1": v["dH2"].T @ v["h1"], "c2": v["dO"].T @ v["h2"]}
    if full:
        gs["p0"] = v["dP1"].T @ v["as2"]
        gs["p1"] = v["dO2"].T @ v["p1"]
    v["g"] = np.zeros(P_COUNT)
    for k, m in gs.items():
        off, o, i = LAYERS[k]
        v["g"][off:off + o * i] = m.reshape(-1)
    return v


# the GEMMs of the backward's weight gradients: layer -> (activation key or columns of A, gradient key), as run() forms them
def _wgrad_operands(v):
    A = v["A"]
    ops = {"s0": (A[:, S0_COLS], v["dS1"]), "s1": (v["s1"], v["dOs"][:, None]), "c0": (A[:, C0_COLS], v["dH1"]),
           "c1": (v["h1"], v["dH2"]), "c2": (v["h2"], v["dO"])}
    if v["full"]:
        ops["p0"] = (v["as2"], v["dP1"])
        ops["p1"] = (v["p1"], v["dO2"])
    return ops


def _flat(parts, default=0.0):
    g = np.full(P_COUNT, default)
    for k, m in parts.items():
        off, o, i = LAYERS[k]
        g[off:off + o * i] = np.asarray(m).reshape(-1)
    return g


# ----------------------------------------------------------------------------------------------------------------------------------
# exact certificates
# ----------------------------------------------------------------------------------------------------------------------------------
_NOBIT = 10 ** 6


def lsb_exp(x):
    """exponent of the lowest set bit of each finite float64 (a huge value for 0)"""
    x = np.asarray(x, F64)
    m, e = np.frexp(x)
    im = np.abs(m * 2.0 ** 53).astype(np.int64)
    low = im & -im
    out = np.where(x != 0, e - 53 + np.log2(np.maximum(low, 1)).astype(np.int64), _NOBIT)
    return out


def grid_exact(X, Y):
    """[n, m] booleans: every fp32 partial sum of X @ Y (X [n,K], Y [K,m]) is exact in any order and alignment: with e the
    lowest set bit over the nonzero terms of an output, sum(|terms|) <= 2^(e+24)"""
    X, Y = np.asarray(X, F64), np.asarray(Y, F64)
    if X.size == 0 or Y.size == 0:
        return np.ones((X.shape[0], Y.shape[1]), bool)
    if not (np.isfinite(X).all() and np.isfinite(Y).all()):
        return np.zeros((X.shape[0], Y.shape[1]), bool)
    lx, ly = lsb_exp(X), lsb_exp(Y)
    e = np.full((X.shape[0], Y.shape[1]), 2 * _NOBIT)
    for k in range(X.shape[1]):                  # lowest bit over the nonzero terms of each output
        e = np.minimum(e, lx[:, k:k + 1] + ly[k:k + 1, :])
    S = np.abs(X) @ np.abs(Y)
    return (S == 0) | (S <= np.exp2(np.minimum(e, 900).astype(F64) + 24))


def f32_exact(x):
    x = np.asarray(x, F64)
    with np.errstate(over="ignore"):
        return x.astype(F32).astype(F64) == x


def rounds_alike(v, eps_rel=0.0, eps_abs=0.0):
    """True where every value within the error band around v rounds to the same fp16 value (no rounding boundary inside)"""
    band = np.abs(v) * eps_rel + eps_abs
    return rh(v - band) == rh(v + band)


def _sig_eps(x):
    """relative error bound of the kernel's 1 / (1 + __expf(-x)) (fp32): __expf, the fp32 add, the fast reciprocal"""
    return EXP_ULP(x) * U32 + 2.0 ** -24 + 2 * U32


def certify(v):
    """Per-value certificates of run(rnd=True): dict of boolean arrays shaped like the outputs (out [R,4] with column 0 = sigma,
    which is never exact and compared within exp_bound, denc [R,64], g [P_COUNT], spec_sq scalar) and `rows` [R] (every per-row
    value of that row certified)."""
    A, W, R = v["A"], v["W"], v["A"].shape[0]
    row = np.ones(R, bool)
    # forward GEMMs (per row): fp32-exact, so rounding to fp16 is deterministic
    row &= grid_exact(A, W["c1"].T).all(1) & grid_exact(A, W["s1"].T).all(1)
    row &= grid_exact(v["s1"], W["s2"][0][:, None]).all(1)
    row &= grid_exact(v["h1"], W["c2"].T).all(1) & grid_exact(v["h2"], W["c3"][:6].T).all(1)
    row &= rounds_alike(_sigmoid(v["x"]), _sig_eps(v["x"])).all(1)
    if v["full"]:
        row &= grid_exact(v["as2"], W["p1"][:, :6].T).all(1) & grid_exact(v["p1"], W["p2"][:3].T).all(1)
        row &= rounds_alike(_sigmoid(v["y"]), _sig_eps(v["y"])).all(1)
        row &= (f32_exact(v["cs_pre"]) | rounds_alike(v["cs_pre"], 2.0 ** -24)).all(1)
    spec_ok = bool(grid_exact(v["spec_sq_terms"].reshape(1, -1), np.ones((v["spec_sq_terms"].size, 1)))[0, 0])
    if "dv" not in v:
        return dict(rows=row, spec_sq=spec_ok)
    # per-sample chain (fp32) and the backward GEMMs
    dv = v["dv"]
    row &= f32_exact(dv).all(1)
    eps = EXP_ULP(v["hs_clamp"]) * U32 + 2.0 ** -24
    row &= rounds_alike(v["dOs_pre"], eps)
    row &= grid_exact(v["dOs"][:, None], W["s2"][0][None, :]).all(1)
    if v["full"]:
        # spec_reg: 2 lambda / M by the fast division (2 ulp), times the loss scale; dsp = g + spec_reg sp, two products
        sp = v["sp"]
        band = np.abs(v["spec_reg"] * sp * sp * (1 - sp)) * (2 * U32 + 2.0 ** -24) + np.abs(v["dO2_pre"]) * 4 * 2.0 ** -24
        exact = (v["spec_reg"] == 0) & f32_exact(v["dsp"] * sp) & f32_exact(v["dO2_pre"])
        row &= (exact | rounds_alike(v["dO2_pre"], eps_abs=band)).all(1)
        row &= grid_exact(v["dO2"], W["p2"][:3]).all(1) & grid_exact(v["dP1"], W["p1"][:, :6]).all(1)
    exact = f32_exact(v["dfeat"] * v["feat"]) & f32_exact(v["dO_pre"])      # else two fp32 roundings
    row &= (exact | rounds_alike(v["dO_pre"], 2 * 2.0 ** -24)).all(1)
    row &= grid_exact(v["dO"], W["c3"][:6]).all(1) & grid_exact(v["dH2"], W["c2"]).all(1)
    row &= grid_exact(np.concatenate([v["dS1"], v["dH1"]], 1), np.concatenate([W["s1"], W["c1"]], 0)).all(1)
    # weight gradients: sums over every row of the batch (all CTAs, all parts)
    g = {k: grid_exact(d.T, a) for k, (a, d) in _wgrad_operands(v).items()}
    return dict(rows=row, spec_sq=spec_ok, g=_flat(g, default=1.0).astype(bool))


def exp_bound(h, dh=0.0):
    """|__expf(h') - exp(h)| for |h' - h| <= dh"""
    e = np.exp(np.minimum(h + dh, 80))
    return np.exp(h) * np.expm1(dh) + e * EXP_ULP(np.abs(h) + dh) * U32


# ----------------------------------------------------------------------------------------------------------------------------------
# error bounds (dense inputs)
# ----------------------------------------------------------------------------------------------------------------------------------
_BIG = 1e300


def _mm(a, b):
    """a @ b for non-negative bound matrices, with inf * 0 = 0"""
    y = np.where(np.isinf(a), _BIG, a) @ np.where(np.isinf(b), _BIG, b)
    return np.where(y >= 1e250, np.inf, y)


def _gemm_delta(X, dX, Wt, ksteps):
    """bound on |kernel - exact| of X @ Wt (fp16 operands X with error dX, exact weights Wt [K, N]) under the tensor-core model"""
    aW = np.abs(Wt)
    return _mm(dX, aW) + ksteps * K16 * _mm(np.abs(X) + dX, aW)


def _round_delta(pre, d):
    """rounding point: delta 0 where no fp16 rounding boundary lies within pre +- d, else d + one fp16 ulp; inf past the overflow"""
    with np.errstate(invalid="ignore", over="ignore"):
        same = (d == 0) | (np.isfinite(d) & (rh(pre - d) == rh(pre + d)) & np.isfinite(rh(pre)))
        mag = np.abs(pre) + d
        ulp = np.exp2(np.floor(np.log2(np.maximum(mag, 2.0 ** -14))) - 10)
        out = np.where(same, 0.0, d + ulp)
        return np.where(mag >= OVF, np.inf, out)


def _relu_delta(act, d):
    """ReLU is 1-Lipschitz: delta passes, except where the unit is off across the whole interval"""
    return np.where(act + d <= 0, 0.0, d)


def _mask_delta(act, dact, grad, dgrad):
    """select(act > 0, grad): union of both branches where act +- dact straddles 0"""
    amb = (act - dact <= 0) & (act + dact > 0)
    off = (act <= 0) & ~amb
    return np.where(off, 0.0, np.where(amb, np.abs(np.nan_to_num(grad, posinf=_BIG, neginf=_BIG)) + dgrad, dgrad))


def bounds(v, ctas_per_part, tiles_per_cta):
    """delta of every output of run(rnd=True, dout given): dict(out [R,4], denc [R,64], g [P_COUNT], spec_sq, certified fractions).
    ctas_per_part: the number of CTAs that flush weight gradients (all parts together); tiles_per_cta: the most tiles one CTA
    accumulates (sets the length of its k16 chain, 8 steps per tile)."""
    A, W, R, full = v["A"], v["W"], v["A"].shape[0], v["full"]
    z = np.zeros_like(A)
    st = {}
    d_h1 = _round_delta(v["h1_acc"], _gemm_delta(A, z, W["c1"].T, 4))
    d_h1 = _relu_delta(v["h1"], d_h1)
    d_s1 = _relu_delta(v["s1"], _round_delta(v["s1_acc"], _gemm_delta(A, z, W["s1"].T, 4)))
    d_hs = _round_delta(v["hs_acc"], _gemm_delta(v["s1"], d_s1, W["s2"][:1].T, 2)[:, 0])
    d_sigma = exp_bound(v["hs"], d_hs)
    d_h2 = _relu_delta(v["h2"], _round_delta(v["h2_acc"], _gemm_delta(v["h1"], d_h1, W["c2"].T, 4)))
    d_x = _round_delta(v["x_acc"], _gemm_delta(v["h2"], d_h2, W["c3"][:6].T, 4))
    s = _sigmoid(v["x"])
    d_feat = _round_delta(s, d_x / 4 + s * _sig_eps(np.abs(v["x"]) + d_x))
    d_sp = np.zeros((R, 3))
    d_col = d_feat[:, :3]
    if full:
        d_as2 = np.concatenate([np.zeros((R, 3)), d_feat[:, 3:6]], 1)
        d_p1 = _relu_delta(v["p1"], _round_delta(v["p1_acc"], _gemm_delta(v["as2"], d_as2, W["p1"][:, :6].T, 1)))
        d_y = _round_delta(v["y_acc"], _gemm_delta(v["p1"], d_p1, W["p2"][:3].T, 2))
        sy = _sigmoid(v["y"])
        d_sp = _round_delta(sy, d_y / 4 + sy * _sig_eps(np.abs(v["y"]) + d_y))
        d_cs = _round_delta(v["cs_pre"], d_sp + d_feat[:, :3] + np.abs(v["cs_pre"]) * 2.0 ** -24)
        d_col = d_cs
    d_out = np.concatenate([d_sigma[:, None], d_sp if v["shading"] == 2 else d_col], 1)
    sq = np.where(v["own"][:, None], 2 * np.abs(v["sp"]) * d_sp + d_sp ** 2, 0.0)
    n_terms = int(v["own"].sum()) * 3
    d_spec = sq.sum() + (n_terms + ctas_per_part) * 2.0 ** -24 * (np.abs(v["spec_sq_terms"]).sum() + sq.sum())
    st["fwd_points"] = [d_h1, d_s1, d_hs, d_h2, d_x, d_feat] + ([d_p1, d_y, d_sp, d_cs] if full else [])
    res = dict(out=d_out, spec_sq=d_spec)
    if "dv" not in v:
        return res

    dv = v["dv"]
    f32e = 2.0 ** -24
    # trunc_exp backward: the clamp is 1-Lipschitz
    d_e = exp_bound(v["hs_clamp"], d_hs)
    d_dOs = _round_delta(v["dOs_pre"], np.abs(dv[:, 0]) * d_e + np.abs(v["dOs_pre"]) * f32e)
    d_dS1 = _mask_delta(v["s1"], d_s1, rh(v["dS1_acc"]), _round_delta(v["dS1_acc"], _gemm_delta(v["dOs"][:, None], d_dOs[:, None],
                                                                                                      W["s2"][:1], 1)))
    d_dfeat = np.zeros((R, 6))
    if full:
        sp = v["sp"]
        dcol = dv[:, 1:4]
        amb = ((v["cs"] - d_cs < 0) & (v["cs"] + d_cs >= 0)) | ((v["cs"] - d_cs <= 1) & (v["cs"] + d_cs > 1))
        d_g = np.where(amb, np.abs(dcol), 0.0)
        d_dfeat[:, :3] = d_g
        sr = abs(v["spec_reg"])
        d_dsp = np.where(v["own"][:, None], d_g + sr * d_sp + sr * np.abs(sp) * (2 * U32 + f32e) + (np.abs(v["dsp"]) + d_g) * f32e, 0.0)
        dsig = sp * (1 - sp)
        d_dO2 = _round_delta(v["dO2_pre"], d_dsp * (dsig + d_sp) + np.abs(v["dsp"]) * d_sp + np.abs(v["dO2_pre"]) * 3 * f32e)
        d_dP1 = _mask_delta(v["p1"], d_p1, rh(v["dP1_acc"]), _round_delta(v["dP1_acc"], _gemm_delta(v["dO2"], d_dO2, W["p2"][:3], 1)))
        d_dAs2 = _gemm_delta(v["dP1"], d_dP1, W["p1"][:, :6], 2)
        d_dfeat[:, 3:6] = d_dAs2[:, 3:6]
    feat = v["feat"]
    fsig = feat * (1 - feat)
    d_dO = _round_delta(v["dO_pre"], d_dfeat * (fsig + d_feat) + np.abs(v["dfeat"]) * d_feat + np.abs(v["dO_pre"]) * 3 * f32e)
    d_dH2 = _mask_delta(v["h2"], d_h2, rh(v["dH2_acc"]), _round_delta(v["dH2_acc"], _gemm_delta(v["dO"], d_dO, W["c3"][:6], 1)))
    d_dH1 = _mask_delta(v["h1"], d_h1, rh(v["dH1_acc"]), _round_delta(v["dH1_acc"], _gemm_delta(v["dH2"], d_dH2, W["c2"], 4)))
    X = np.concatenate([v["dS1"], v["dH1"]], 1)
    dX = np.concatenate([d_dS1, d_dH1], 1)
    d_denc = _round_delta(v["denc_acc"], _gemm_delta(X, dX, np.concatenate([W["s1"], W["c1"]], 0), 6))
    res["denc"] = d_denc
    # weight gradients: first-order propagation plus the CTA chains and the atomics
    dact = {"s0": np.zeros((R, 19)), "s1": d_s1, "c0": np.zeros((R, 35)), "c1": d_h1, "c2": d_h2}
    dgrad = {"s0": d_dS1, "s1": d_dOs[:, None], "c0": d_dH1, "c1": d_dH2, "c2": d_dO}
    if full:
        dact["p0"] = d_as2
        dact["p1"] = d_p1
        dgrad["p0"] = d_dP1
        dgrad["p1"] = d_dO2
    acc = tiles_per_cta * 8 * K16 + ctas_per_part * f32e
    dg = {}
    for k, (a, d) in _wgrad_operands(v).items():
        aa, ad = np.abs(a), np.abs(d)
        prop = _mm(dgrad[k].T, aa) + _mm(ad.T, dact[k]) + _mm(dgrad[k].T, dact[k])
        dg[k] = prop + acc * _mm((ad + dgrad[k]).T, aa + dact[k])
    res["g"] = _flat(dg)
    pts = st["fwd_points"] + [d_dOs, d_dS1, d_dO, d_dH2, d_dH1, d_denc] + ([d_dO2, d_dP1] if full else [])
    res["identical_fraction"] = float(np.mean(np.concatenate([np.ravel(p) == 0 for p in pts])))
    return res


# ----------------------------------------------------------------------------------------------------------------------------------
# exact probes: dyadic weights and inputs with few bits each, sparse rows, power-of-two upstream gradients
# ----------------------------------------------------------------------------------------------------------------------------------
MAGS = np.array([1.0, 1.25, 1.5, 1.75, 0.5, 0.625, 0.75, 0.875])     # 3-bit mantissas, pairwise distinct
NNZ = {"s0": 4, "s1": 8, "c0": 4, "c1": 5, "c2": 6, "p0": 3, "p1": 6}


def _sparse(rng, o, i, nnz):
    """[o, i]: nnz entries per row, pairwise distinct magnitudes in a row, random signs, scaled by 2^-round(log2(nnz))"""
    W = np.zeros((o, i))
    scale = 2.0 ** -round(np.log2(nnz))
    for r in range(o):
        k = rng.choice(i, size=min(nnz, i), replace=False)
        W[r, k] = rng.permutation(MAGS)[:len(k)] * scale * rng.choice([-1.0, 1.0], len(k))
    return W


def probe_params(rng):
    P = np.zeros(P_COUNT)
    for k, (off, o, i) in LAYERS.items():
        P[off:off + o * i] = _sparse(rng, o, i, NNZ[k]).reshape(-1)
    return P


def probe_rows(rng, idx):
    """[len(idx), 64] fp16-exact rows: columns 0..53 sparse dyadic with 3-bit mantissas, 54..63 finite junk (no weight reads them)"""
    n = len(idx)
    A = np.where(rng.random((n, 64)) < 0.6, rng.choice(MAGS, (n, 64)) * rng.choice([-1.0, 1.0], (n, 64)), 0.0)
    A[:, 54:] = rh(rng.uniform(-300, 300, (n, 10)))
    return A


def probe_dout(rng, idx):
    """[len(idx), 4] powers of two with random signs"""
    n = len(idx)
    return np.exp2(rng.integers(-2, 3, (n, 4))) * rng.choice([-1.0, 1.0], (n, 4))


def _certified_rows(P, A, D, M, ls, lam):
    ok = np.ones(A.shape[0], bool)
    for shading in (0, 1):
        ok &= certify(run(P, A, D, shading, M, ls, lam))["rows"]
    return ok


def make_probe(seed, R, M=None, lam=0.0, ls=1.0, P=None, row_fn=probe_rows, dout_fn=probe_dout, max_grad_rows=None,
               first=()):
    """A probe of R rows (rows >= M not owned) whose every output is certified for shading 0, 1 and 2: rows are drawn until each one's
    forward and backward certify, then upstream gradients are kept on as many rows as leave every weight-gradient sum exact (the
    others get dout = 0).  Returns dict(P, enc [R,64], dout [R,4] (NaN on rows not owned), M, ls, lam)."""
    rng = np.random.default_rng(seed)
    M = R if M is None else M
    P = probe_params(rng) if P is None else P
    A = row_fn(rng, np.arange(R))
    D = dout_fn(rng, np.arange(R))
    for _ in range(50):
        bad = ~_certified_rows(P, A, D, M, ls, lam)
        if not bad.any():
            break
        A[bad] = row_fn(rng, np.flatnonzero(bad))
    else:
        raise AssertionError("probe rows do not certify")
    # a row's weight-gradient terms do not depend on other rows' upstream gradients: select rows on the terms of the full run
    ops = [_wgrad_operands(run(P, A, D, s, M, ls, lam)) for s in (0, 1)]
    keep = np.zeros(R, bool)
    order = list(first) + [j for j in rng.permutation(min(M, R)) if j not in first]
    for j in order:
        if max_grad_rows is not None and keep.sum() >= max_grad_rows:
            break
        keep[j] = True
        rows_ = np.flatnonzero(keep)
        if not all(grid_exact(d[rows_].T, a[rows_]).all() for o in ops for a, d in o.values()):
            keep[j] = False
    Dk = np.where(keep[:, None], D, 0.0)
    assert all(certify(run(P, A, Dk, s, M, ls, lam))["g"].all() for s in (0, 1)), "weight gradients do not certify"
    Dk[M:] = np.nan
    return dict(P=P, enc=A, dout=Dk, M=M, ls=ls, lam=lam, grad_rows=np.flatnonzero(keep))


def probe_certified(pr, shading):
    v = run(pr["P"], pr["enc"], pr["dout"], shading, pr["M"], pr["ls"], pr["lam"])
    c = certify(v)
    return bool(c["rows"].all() and c["g"].all()), v, c


def _set(P, name, W):
    off, o, i = LAYERS[name]
    P[off:off + o * i] = np.asarray(W, F64).reshape(-1)


SIGMA_TARGETS = (-20.0, -15.0, 0.0, 15.0, 20.0)


def sigma_clamp_probe(t, seed=100):
    """sigma pre-activation t on every row (trunc_exp's backward clamps at +-15): sigma_net.0 units 0 / 1 read enc columns 3 / 4
    alone, sigma_net.1 = unit 0 - unit 1, enc columns 3 / 4 = max(t, 0) / max(-t, 0); dout.x scaled so that dOs is of order one"""
    rng = np.random.default_rng(seed)
    P = probe_params(rng)
    s0 = layer(P, "s0").copy()
    s0[0] = 0; s0[0, 3] = 1.0
    s0[1] = 0; s0[1, 4] = 1.0
    _set(P, "s0", s0)
    s1 = np.zeros((1, 32)); s1[0, 0], s1[0, 1] = 1.0, -1.0
    _set(P, "s1", s1)

    def rows(rng, idx):
        A = probe_rows(rng, idx)
        A[:, 3], A[:, 4] = max(t, 0.0), max(-t, 0.0)
        return A

    def dout(rng, idx):
        D = probe_dout(rng, idx)
        D[:, 0] = np.sign(D[:, 0]) * np.exp2(-np.round(np.clip(t, -15, 15) / np.log(2)))
        return D
    return make_probe(seed, 40, P=P, row_fn=rows, dout_fn=dout, first=[0])


def colour_edge_probe(seed=200):
    """sp + feat = 1.0 exactly in channel 0 (both sigmoids at 0.5: the clamp's gradient passes) and the next fp16 above 1.0 in channel
    1 (sp = 0.5 + 2^-10: it must not): color_net.2 rows 0..2 zero; specular_net.0 unit 0 reads the direction's x (= 1) alone;
    specular_net.1 row 0 zero, row 1 = 2^-8 on unit 0"""
    rng = np.random.default_rng(seed)
    P = probe_params(rng)
    c2 = layer(P, "c2").copy(); c2[:3] = 0; _set(P, "c2", c2)
    p0 = layer(P, "p0").copy(); p0[0] = 0; p0[0, 0] = 1.0; _set(P, "p0", p0)
    p1 = layer(P, "p1").copy(); p1[0] = 0; p1[1] = 0; p1[1, 0] = 2.0 ** -8; _set(P, "p1", p1)

    def rows(rng, idx):
        A = probe_rows(rng, idx)
        A[:, COL_DIR] = 1.0
        return A
    return make_probe(seed, 60, P=P, row_fn=rows)


def spec_reg_probe(seed=300):
    """the specular regulariser: lambda_specular != 0 with two owned rows of a 128-row tile (rows 2..127 hold finite activations and
    no upstream gradient: they must add nothing)"""
    for s in range(seed, seed + 50):
        try:
            return make_probe(s, 128, M=2, lam=2.0 ** -6, ls=2.0 ** 4)
        except AssertionError:
            continue
    raise AssertionError("no certified specular-regulariser probe")


def masked_inf_probe(seed=400):
    """color_net.1 unit j inactive on every row (its weights <= 0 on non-negative inputs) with color_net.2[0, j] = 2^14 and
    dout.y = +-64, so that unit j's pre-mask gradient overflows fp16 on the gradient rows while every active unit stays finite:
    the mask must give 0 there (threshold_backward is a select), not inf * 0 = NaN"""
    rng = np.random.default_rng(seed)
    P = probe_params(rng)
    j = 7
    c1 = layer(P, "c1").copy(); c1[j] = -np.abs(c1[j]); c1[j, 0] = -1.0; _set(P, "c1", c1)
    c2 = layer(P, "c2").copy(); c2[:, j] = 0; c2[0, j] = 2.0 ** 14; _set(P, "c2", c2)

    def dout(rng, idx):
        D = probe_dout(rng, idx)
        D[:, 1] = 64.0 * np.sign(D[:, 1])
        return D
    pr = make_probe(seed, 64, P=P, dout_fn=dout)
    pr["inactive_unit"] = j
    return pr


@functools.lru_cache(maxsize=None)
def exact_probes(n_random=32):
    """name -> probe: random sparse probes of 190 rows, and the special probes above"""
    out = {f"rand{s}": make_probe(s, 190) for s in range(n_random)}
    for t in SIGMA_TARGETS:
        out[f"sigma_{t:+.0f}"] = sigma_clamp_probe(t)
    out["colour_edge"] = colour_edge_probe()
    out["spec_reg"] = spec_reg_probe()
    out["masked_inf"] = masked_inf_probe()
    return out
