"""oracle/raymarching_oracle.py -- TEST INFRASTRUCTURE ONLY (never imported by the product).

CPU restatement (numpy, float32) of the reference's ray-marching / compositing kernels,
vectorised over rays.  Each function cites the reference lines it follows.

Pinning: the reference has no tests or golden vectors; this oracle is
pinned against outputs of the reference's own CUDA kernels (oracle/_ref) stored
under tests/golden/ (see tests/golden/make_golden.py and tests/test_oracle_golden.py).
Arithmetic notes: the reference is built with -use_fast_math, i.e. FMA contraction, approximate
reciprocal and ex2, flush-to-zero.  numpy cannot reproduce MUFU.RCP / MUFU.EX2 bit-for-bit, so this
oracle matches the CUDA paths to a few ulp in t and agrees on sample counts for all but
boundary-grazing rays; the bit-exact gate is the GPU test against oracle/_ref.
"""
import numpy as np

F = np.float32
SQRT3 = F(1.7320508075688772)


def _fma(a, b, c):
    """float32 fused multiply-add emulated through float64 (exact product, one rounding to
    double, one to float -- differs from a true fma only in rare double-rounding cases)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F)


def _clamp(x, lo, hi):
    return np.fmin(F(hi), np.fmax(F(lo), x)).astype(F)   # fminf/fmaxf ignore NaN


def _spread3(v):
    v = v.astype(np.uint64)
    v = (v * 0x00010001) & 0xFF0000FF
    v = (v * 0x00000101) & 0x0F00F00F
    v = (v * 0x00000011) & 0xC30C30C3
    v = (v * 0x00000005) & 0x49249249
    return v.astype(np.uint32)


def morton3D(coords):
    """raymarching.cu:56-71, :214-226."""
    c = np.asarray(coords).astype(np.uint32)
    return (_spread3(c[..., 0]) | (_spread3(c[..., 1]) << np.uint32(1)) | (_spread3(c[..., 2]) << np.uint32(2))).astype(np.int32)


def morton3D_invert(indices):
    """raymarching.cu:73-81, :237-254."""
    def compact(x):
        x = x.astype(np.uint32) & np.uint32(0x49249249)
        x = (x | (x >> np.uint32(2))) & np.uint32(0xc30c30c3)
        x = (x | (x >> np.uint32(4))) & np.uint32(0x0f00f00f)
        x = (x | (x >> np.uint32(8))) & np.uint32(0xff0000ff)
        x = (x | (x >> np.uint32(16))) & np.uint32(0x0000ffff)
        return x
    i = np.asarray(indices).astype(np.uint32)
    return np.stack([compact(i), compact(i >> np.uint32(1)), compact(i >> np.uint32(2))], -1).astype(np.int32)


def packbits(grid, thresh):
    """raymarching.cu:268-289: bit i of byte n <-> grid.flat[8n+i] > thresh."""
    g = np.asarray(grid, F).reshape(-1, 8)
    bits = (g > F(thresh)).astype(np.uint8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(-1).astype(np.uint8)


def flatten_rays(rays, M):
    """raymarching.cu:303-319."""
    res = np.zeros(M, np.int32)
    for n, (off, cnt) in enumerate(np.asarray(rays)):
        res[off:off + cnt] = n
    return res


def near_far_from_aabb(rays_o, rays_d, aabb, min_near):
    """raymarching.cu:92-145 (slab test; miss => both FLT_MAX)."""
    o = np.asarray(rays_o, F).reshape(-1, 3)
    d = np.asarray(rays_d, F).reshape(-1, 3)
    aabb = np.asarray(aabb, F)
    with np.errstate(divide="ignore", invalid="ignore"):
        rd = (F(1) / d).astype(F)
        t0 = ((aabb[:3] - o) * rd).astype(F)
        t1 = ((aabb[3:] - o) * rd).astype(F)
    swap = t0 > t1
    lo = np.where(swap, t1, t0)
    hi = np.where(swap, t0, t1)
    near, far = lo[:, 0].copy(), hi[:, 0].copy()
    miss = np.zeros(len(o), bool)
    for a in (1, 2):
        m = (near > hi[:, a]) | (lo[:, a] > far)
        miss |= m
        upd = ~miss
        near = np.where(upd & (lo[:, a] > near), lo[:, a], near)
        far = np.where(upd & (hi[:, a] < far), hi[:, a], far)
    near = np.where(near < F(min_near), F(min_near), near)
    fmax = np.finfo(F).max
    near = np.where(miss, fmax, near).astype(F)
    far = np.where(miss, fmax, far).astype(F)
    return near, far


def sph_from_ray(rays_o, rays_d, radius):
    """raymarching.cu:163-198."""
    o = np.asarray(rays_o, F).reshape(-1, 3)
    d = np.asarray(rays_d, F).reshape(-1, 3)
    A = (d * d).sum(-1)
    B = (o * d).sum(-1)
    C = (o * o).sum(-1) - F(radius) * F(radius)
    t = (-B + np.sqrt(B * B - A * C)) / A
    p = o + t[:, None] * d
    theta = np.arctan2(np.sqrt(p[:, 0] ** 2 + p[:, 2] ** 2), p[:, 1])
    phi = np.arctan2(p[:, 2], p[:, 0])
    return np.stack([2 * theta / np.pi - 1, phi / np.pi], -1).astype(F)


# ------------------------------------------------------------------------------------------------
# marcher
# ------------------------------------------------------------------------------------------------
def _frexp_exp(x):
    _, e = np.frexp(x.astype(F))
    return e.astype(np.int32)


def _probe(t, o, d, bits, bound, contract, dt_gamma, dt_min, dt_max, C, H):
    """One loop-iteration head of the marcher (raymarching.cu:397-432), vectorised."""
    bound = F(bound)
    x = _clamp(_fma(t, d[:, 0], o[:, 0]), -bound, bound)
    y = _clamp(_fma(t, d[:, 1], o[:, 1]), -bound, bound)
    z = _clamp(_fma(t, d[:, 2], o[:, 2]), -bound, bound)
    dt = _clamp((t * F(dt_gamma)).astype(F), dt_min, dt_max)
    mx = np.maximum(np.abs(x), np.maximum(np.abs(y), np.abs(z)))
    lvl_pos = np.minimum(C - 1, np.maximum(0, _frexp_exp(mx)))                       # :42-47
    lvl_dt = np.minimum(C - 1, np.maximum(0, _frexp_exp((dt * F(H) * F(0.5)).astype(F))))   # :49-54
    level = np.maximum(lvl_pos, lvl_dt).astype(np.int32)
    mip_bound = np.minimum(np.ldexp(F(1), level).astype(F), bound)
    mip_rbound = (F(1) / mip_bound).astype(F)
    cx, cy, cz = x, y, z
    outer = np.zeros(len(t), bool)
    if contract:
        outer = mx > 1
        with np.errstate(divide="ignore", invalid="ignore"):
            s = ((F(2) - F(1) / mx) / mx).astype(F)                                   # :415
        cx = np.where(outer, cx * s, cx).astype(F)
        cy = np.where(outer, cy * s, cy).astype(F)
        cz = np.where(outer, cz * s, cz).astype(F)

    def cell(c):                                                                      # :422-424
        v = (np.float64(0.5) * _fma(c, mip_rbound, F(1)).astype(np.float64) * np.float64(H)).astype(F)
        return _clamp(v, 0.0, H - 1).astype(np.int32)
    nx, ny, nz = cell(cx), cell(cy), cell(cz)
    H3 = F(H * H * H)
    mort = morton3D(np.stack([nx, ny, nz], -1)).astype(np.uint32)
    index = (level.astype(F) * H3 + mort.astype(F)).astype(np.uint32)                 # :426 (float math)
    occ = (bits[index // 8] >> (index % 8).astype(np.uint8)) & 1
    emit = (occ == 1) | outer
    return dict(cx=cx, cy=cy, cz=cz, dt=dt, nx=nx, ny=ny, nz=nz, mip_bound=mip_bound, emit=emit)


def _hop(t, p, d, rd, rH, dt_gamma, dt_min, dt_max):
    """Skip to the voxel exit (raymarching.cu:452-464)."""
    def axis(n, c, dd, rdd):
        a = (n.astype(F) + F(0.5)).astype(F)
        a = (a + F(0.5) * np.copysign(F(1), dd)).astype(F)
        b = (a * rH).astype(F)
        b2 = (b * F(2) - F(1)).astype(F)
        with np.errstate(invalid="ignore", over="ignore"):
            return (_fma(b2, p["mip_bound"], -c) * rdd).astype(F)
    tx = axis(p["nx"], p["cx"], d[:, 0], rd[:, 0])
    ty = axis(p["ny"], p["cy"], d[:, 1], rd[:, 1])
    tz = axis(p["nz"], p["cz"], d[:, 2], rd[:, 2])
    with np.errstate(invalid="ignore"):
        tt = (t + np.fmax(F(0), np.fmin(tx, np.fmin(ty, tz)))).astype(F)
    t = t.copy()
    active = np.ones(len(t), bool)
    while active.any():
        dt = _clamp((t * F(dt_gamma)).astype(F), dt_min, dt_max)
        t = np.where(active, (t + dt).astype(F), t)
        with np.errstate(invalid="ignore"):
            active &= t < tt
    return t


def march_rays_train(rays_o, rays_d, bound, contract, density_bitfield, C, H, nears, fars, noises,
                     dt_gamma=0.0, max_steps=1024):
    """raymarching.cu:338-475 + wrapper raymarching.py:184-245 (noises passed in explicitly).
    Returns xyzs [M,3], dirs [M,3], ts [M,2], rays [N,2] with ray-order (deterministic) offsets."""
    o = np.asarray(rays_o, F).reshape(-1, 3)
    d = np.asarray(rays_d, F).reshape(-1, 3)
    bits = np.asarray(density_bitfield, np.uint8)
    nears = np.asarray(nears, F)
    fars = np.asarray(fars, F)
    noises = np.asarray(noises, F)
    N = len(o)
    with np.errstate(divide="ignore"):
        rd = (F(1) / d).astype(F)
    rH = F(1) / F(H)
    dt_min = F(F(2) * SQRT3 / F(max_steps))
    dt_max = F(F(2) * SQRT3 * F(bound) / F(H))
    t = _fma(_clamp((nears * F(dt_gamma)).astype(F), dt_min, dt_max), noises, nears)          # :389-390
    step = np.zeros(N, np.int64)
    buf = np.zeros((N, max_steps, 5), F)         # per-ray (cx, cy, cz, t_after, dt)
    with np.errstate(invalid="ignore"):
        alive = (t < fars) & (step < max_steps)
    while alive.any():
        idx = np.nonzero(alive)[0]
        p = _probe(t[idx], o[idx], d[idx], bits, bound, contract, dt_gamma, dt_min, dt_max, C, H)
        em = p["emit"]
        # occupied: emit a sample and advance by dt
        ie = idx[em]
        t_new = (t[ie] + p["dt"][em]).astype(F)
        buf[ie, step[ie]] = np.stack([p["cx"][em], p["cy"][em], p["cz"][em], t_new, p["dt"][em]], -1)
        t[ie] = t_new
        step[ie] += 1
        # empty: hop to the voxel exit
        ih = idx[~em]
        if len(ih):
            ph = {k: v[~em] for k, v in p.items()}
            t[ih] = _hop(t[ih], ph, d[ih], rd[ih], rH, dt_gamma, dt_min, dt_max)
        with np.errstate(invalid="ignore"):
            alive = (t < fars) & (step < max_steps)
    counts = step.astype(np.int32)
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32) if N else np.zeros(0, np.int32)
    M = int(counts.sum())
    sel = np.arange(max_steps)[None, :] < counts[:, None]            # ray-major == offset order
    flat = buf[sel]
    xyzs = np.ascontiguousarray(flat[:, :3])
    ts = np.ascontiguousarray(flat[:, 3:5])
    dirs = np.repeat(d, counts, axis=0).astype(F)
    rays = np.stack([offsets, counts], -1).astype(np.int32)
    return xyzs, dirs, ts, rays


def march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, contract, density_bitfield,
               C, H, nears, fars, noises, dt_gamma=0.0, max_steps=1024):
    """Inference marcher, raymarching.cu:713-828."""
    o_all = np.asarray(rays_o, F).reshape(-1, 3)
    d_all = np.asarray(rays_d, F).reshape(-1, 3)
    ra = np.asarray(rays_alive)[:n_alive]
    o, d = o_all[ra], d_all[ra]
    bits = np.asarray(density_bitfield, np.uint8)
    rd = (F(1) / (d + F(1e-10))).astype(F)                                             # :744
    rH = F(1) / F(H)
    dt_min = F(F(2) * SQRT3 / F(max_steps))
    dt_max = F(F(2) * SQRT3 * F(bound) / F(H))
    t = np.asarray(rays_t, F)[ra].copy()
    far = np.asarray(fars, F)[ra]
    t = _fma(_clamp((t * F(dt_gamma)).astype(F), dt_min, dt_max), np.asarray(noises, F)[:n_alive], t)
    xyzs = np.zeros((n_alive * n_step, 3), F)
    dirs = np.zeros((n_alive * n_step, 3), F)
    ts = np.zeros((n_alive * n_step, 2), F)
    step = np.zeros(n_alive, np.int64)
    with np.errstate(invalid="ignore"):
        alive = (t < far) & (step < n_step)
    while alive.any():
        idx = np.nonzero(alive)[0]
        p = _probe(t[idx], o[idx], d[idx], bits, bound, contract, dt_gamma, dt_min, dt_max, C, H)
        em = p["emit"]
        ie = idx[em]
        j = ie * n_step + step[ie]
        xyzs[j] = np.stack([p["cx"][em], p["cy"][em], p["cz"][em]], -1)
        dirs[j] = d[ie]
        t[ie] = (t[ie] + p["dt"][em]).astype(F)
        ts[j, 0] = t[ie]
        ts[j, 1] = p["dt"][em]
        step[ie] += 1
        ih = idx[~em]
        if len(ih):
            ph = {k: v[~em] for k, v in p.items()}
            t[ih] = _hop(t[ih], ph, d[ih], rd[ih], rH, dt_gamma, dt_min, dt_max)
        with np.errstate(invalid="ignore"):
            alive = (t < far) & (step < n_step)
    return xyzs, dirs, ts


# ------------------------------------------------------------------------------------------------
# compositing
# ------------------------------------------------------------------------------------------------
def _alpha(sigma, dt, alpha_mode):
    if alpha_mode:
        return F(sigma)
    return F(F(1) - np.exp(-F(sigma) * F(dt), dtype=F))


def composite_rays_train_forward(sigmas, rgbs, ts, rays, T_thresh=1e-4, alpha_mode=False):
    """raymarching.cu:501-578."""
    sigmas = np.asarray(sigmas, F); rgbs = np.asarray(rgbs, F).reshape(-1, 3); ts = np.asarray(ts, F).reshape(-1, 2)
    rays = np.asarray(rays)
    M, N = len(sigmas), len(rays)
    weights = np.zeros(M, F)
    weights_sum = np.zeros(N, F); depth = np.zeros(N, F); image = np.zeros((N, 3), F)
    for n in range(N):
        off, cnt = int(rays[n, 0]), int(rays[n, 1])
        if cnt == 0 or off + cnt > M:
            continue
        T = F(1); acc = np.zeros(3, F); ws = F(0); dd = F(0)
        for j in range(off, off + cnt):
            a = _alpha(sigmas[j], ts[j, 1], alpha_mode)
            w = F(a * T)
            weights[j] = w
            acc = (acc + w * rgbs[j]).astype(F)
            ws = F(ws + w)
            dd = F(dd + w * ts[j, 0])
            T = F(T * (F(1) - a))
            if T < T_thresh:
                break
        weights_sum[n] = ws; depth[n] = dd; image[n] = acc
    return weights, weights_sum, depth, image


def composite_rays_train_backward(grad_weights, grad_weights_sum, grad_depth, grad_image, sigmas, rgbs, ts, rays,
                                  weights_sum, depth, image, T_thresh=1e-4, alpha_mode=False):
    """raymarching.cu:605-694."""
    sigmas = np.asarray(sigmas, F); rgbs = np.asarray(rgbs, F).reshape(-1, 3); ts = np.asarray(ts, F).reshape(-1, 2)
    rays = np.asarray(rays)
    M, N = len(sigmas), len(rays)
    g_sig = np.zeros(M, F); g_rgb = np.zeros((M, 3), F)
    for n in range(N):
        off, cnt = int(rays[n, 0]), int(rays[n, 1])
        if cnt == 0 or off + cnt > M:
            continue
        T = F(1); acc = np.zeros(3, F); ws = F(0); dd = F(0)
        for j in range(off, off + cnt):
            a = _alpha(sigmas[j], ts[j, 1], alpha_mode)
            w = F(a * T)
            acc = (acc + w * rgbs[j]).astype(F)
            ws = F(ws + w)
            dd = F(dd + w * ts[j, 0])
            T = F(T * (F(1) - a))
            g_rgb[j] = grad_image[n] * w
            scale = F(1) / (F(1) - a) if alpha_mode else ts[j, 1]
            g_sig[j] = scale * (
                np.dot(grad_image[n], T * rgbs[j] - (image[n] - acc)) +
                (grad_weights_sum[n] + grad_weights[j]) * (T - (weights_sum[n] - ws)) +
                grad_depth[n] * (T * ts[j, 0] - (depth[n] - dd)))
            if T < T_thresh:
                break
    return g_sig, g_rgb


def composite_rays(n_alive, n_step, rays_alive, rays_t, sigmas, rgbs, ts, weights_sum, depth, image,
                   T_thresh=1e-2, alpha_mode=False):
    """raymarching.cu:842-924 (in place on copies; returns the updated arrays)."""
    rays_alive = np.array(rays_alive).copy(); rays_t = np.array(rays_t, F).copy()
    weights_sum = np.array(weights_sum, F).copy(); depth = np.array(depth, F).copy(); image = np.array(image, F).copy()
    sigmas = np.asarray(sigmas, F); rgbs = np.asarray(rgbs, F).reshape(-1, 3); ts = np.asarray(ts, F).reshape(-1, 2)
    for n in range(n_alive):
        idx = int(rays_alive[n])
        ws = weights_sum[idx]; d = depth[idx]; c = image[idx].copy(); t = F(0)
        k = 0
        while k < n_step:
            j = n * n_step + k
            if ts[j, 0] == 0:
                break
            a = _alpha(sigmas[j], ts[j, 1], alpha_mode)
            T = F(F(1) - ws)
            w = F(a * T)
            ws = F(ws + w)
            t = ts[j, 0]
            d = F(d + w * t)
            c = (c + w * rgbs[j]).astype(F)
            if T < T_thresh:
                break
            k += 1
        if k < n_step:
            rays_alive[n] = -1
        else:
            rays_t[idx] = t
        weights_sum[idx] = ws; depth[idx] = d; image[idx] = c
    return rays_alive, rays_t, weights_sum, depth, image
