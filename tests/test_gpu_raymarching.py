"""GPU parity: nerf2mesh_b200.raymarching (through the C ABI) vs the reference's own CUDA kernels
(oracle/_ref) on identical inputs.  Bar: bit-exact sample counts, M, and per-ray sample values
(integers AND floats -- the arithmetic is reproduced op for op); composite is bit-exact too."""
import numpy as np
import pytest
import torch

import cases
import refcall
import refreplay
from nerf2mesh_b200 import raymarching as rm

pytestmark = pytest.mark.gpu


def cu(x):
    return x.cuda() if torch.is_tensor(x) else x


@pytest.mark.parametrize("name", cases.MARCH_CASES)
def test_near_far_bit_exact(ref_raymarching, name):
    c = cases.march_case(name)
    ro, rd, aabb = cu(c["rays_o"]), cu(c["rays_d"]), cu(c["aabb"])
    # add degenerate rays: axis-parallel (zero components) and guaranteed misses
    ro = torch.cat([ro, torch.tensor([[0.0, 0.0, 3.0], [5.0, 5.0, 5.0], [0.2, 0.1, 0.0]], device="cuda")])
    rd = torch.cat([rd, torch.tensor([[0.0, 0.0, -1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], device="cuda")])
    n0, f0 = refcall.near_far(ref_raymarching, ro, rd, aabb, c["min_near"])
    n1, f1 = rm.near_far_from_aabb(ro, rd, aabb, c["min_near"])
    assert torch.equal(n0, n1) and torch.equal(f0, f1)


@pytest.mark.parametrize("name", cases.MARCH_CASES)
def test_march_rays_train_bit_exact(ref_raymarching, name):
    c = cases.march_case(name)
    ro, rd, bits, aabb = cu(c["rays_o"]), cu(c["rays_d"]), cu(c["bits"]), cu(c["aabb"])
    nears, fars = rm.near_far_from_aabb(ro, rd, aabb, c["min_near"])
    noises = cu(c["noises"])

    def summary(mod):        # the reference's outputs in ray order, as digests (bit-exact comparison)
        x0, d0, t0, r0 = refcall.march_train(mod, ro, rd, bits, c["bound"], c["contract"], c["dt_gamma"],
                                             c["max_steps"], c["C"], c["H"], nears, fars, noises)
        out = {"M": np.array(x0.shape[0]), "counts": r0[:, 1].cpu().numpy()}
        for a, nm in ((x0, "xyzs"), (d0, "dirs"), (t0, "ts")):
            out[nm] = refreplay.digest(refcall.by_ray(a, r0))
        return out
    ref = ref_raymarching.summary(summary)
    # ours, with the wrapper's RNG replaced by the same noises: call the C ABI protocol directly
    from nerf2mesh_b200._lib import call, ptr, stream
    N = ro.shape[0]
    for use_slab in (True, False):
        counter = torch.zeros(1, dtype=torch.int32, device="cuda")
        rays = torch.empty(N, 2, dtype=torch.int32, device="cuda")
        tbuf = torch.empty(N * c["max_steps"] * 2, device="cuda") if use_slab else None
        args = (ptr(ro), ptr(rd), ptr(bits), c["bound"], int(c["contract"]), c["dt_gamma"], c["max_steps"], N,
                c["C"], c["H"], ptr(nears), ptr(fars))
        call("n2m_march_rays_train", *args, None, None, None, ptr(rays), ptr(counter), ptr(noises), ptr(tbuf), stream())
        M = int(counter.item())
        assert M == int(ref["M"]), f"M differs: {M} vs {int(ref['M'])}"
        assert M > 0
        # counts bit-exact; our offsets are the exclusive scan in ray order
        assert np.array_equal(rays[:, 1].cpu().numpy(), ref["counts"])
        cnt = rays[:, 1].long()
        assert torch.equal(rays[:, 0].long(), torch.cumsum(cnt, 0) - cnt)
        x1 = torch.zeros(M, 3, device="cuda"); d1 = torch.zeros(M, 3, device="cuda"); t1 = torch.zeros(M, 2, device="cuda")
        call("n2m_march_rays_train", *args, ptr(x1), ptr(d1), ptr(t1), ptr(rays), ptr(counter), ptr(noises), ptr(tbuf), stream())
        torch.cuda.synchronize()
        for b, nm in ((x1, "xyzs"), (d1, "dirs"), (t1, "ts")):
            assert refreplay.digest(refcall.by_ray(b, rays)) == ref[nm], f"{nm} differ (slab={use_slab})"


def test_march_wrapper_matches_abi():
    c = cases.march_case("lego_converged")
    ro, rd, bits, aabb = cu(c["rays_o"]), cu(c["rays_d"]), cu(c["bits"]), cu(c["aabb"])
    nears, fars = rm.near_far_from_aabb(ro, rd, aabb, c["min_near"])
    xyzs, dirs, ts, rays = rm.march_rays_train(ro, rd, c["bound"], c["contract"], bits, c["C"], c["H"], nears, fars,
                                               False, c["dt_gamma"], c["max_steps"])
    M = xyzs.shape[0]
    assert M == int(rays[:, 1].sum()) and dirs.shape == (M, 3) and ts.shape == (M, 2) and rays.dtype == torch.int32
    assert (ts[:, 1] > 0).all() and (xyzs.abs() <= c["bound"]).all()
    flat = rm.flatten_rays(rays, M)
    assert torch.equal(dirs, rd[flat.long()])
    # empty input
    e = torch.zeros(0, 3, device="cuda")
    x, d, t, r = rm.march_rays_train(e, e, 1.0, False, bits, 1, 128, torch.zeros(0, device="cuda"), torch.zeros(0, device="cuda"))
    assert x.shape == (0, 3) and r.shape == (0, 2)


@pytest.mark.parametrize("alpha_mode", [False, True])
@pytest.mark.parametrize("T_thresh", [1e-4, 1e-2])
def test_composite_train_bit_exact(ref_raymarching, alpha_mode, T_thresh):
    c = cases.composite_case()
    sig = cu(c["sigmas"]); rgb = cu(c["rgbs"]); ts = cu(c["ts"]); rays = cu(c["rays"])
    if alpha_mode:
        sig = (sig / sig.max()).clamp(0, 0.999)
    w0, ws0, d0, i0 = refcall.composite_fwd(ref_raymarching, sig, rgb, ts, rays, T_thresh, alpha_mode)
    w1, ws1, d1, i1 = rm.composite_rays_train(sig, rgb, ts, rays, T_thresh, alpha_mode)
    for a, b in ((w0, w1), (ws0, ws1), (d0, d1), (i0, i1)):
        assert torch.equal(a, b)
    gw, gws, gd, gi = cu(c["grad_weights"]), cu(c["grad_weights_sum"]), cu(c["grad_depth"]), cu(c["grad_image"])
    gs0, gr0 = refcall.composite_bwd(ref_raymarching, gw, gws, gd, gi, sig, rgb, ts, rays, ws0, d0, i0, T_thresh, alpha_mode)
    sig_r = sig.clone().requires_grad_(True); rgb_r = rgb.clone().requires_grad_(True)
    w, ws, d, im = rm.composite_rays_train(sig_r, rgb_r, ts, rays, T_thresh, alpha_mode)
    torch.autograd.backward([w, ws, d, im], [gw, gws, gd, gi])
    assert torch.equal(sig_r.grad, gs0) and torch.equal(rgb_r.grad, gr0)


def test_composite_rays_beyond_M_zeroed(ref_raymarching):
    """rays whose slice exceeds M produce zeros (raymarching.cu:521-528)."""
    c = cases.composite_case(N=16)
    sig = cu(c["sigmas"]); rgb = cu(c["rgbs"]); ts = cu(c["ts"]); rays = cu(c["rays"]).clone()
    rays[-1, 1] += 1000
    w0, ws0, d0, i0 = refcall.composite_fwd(ref_raymarching, sig, rgb, ts, rays, 1e-4, False)
    w1, ws1, d1, i1 = rm.composite_rays_train(sig, rgb, ts, rays, 1e-4, False)
    assert torch.equal(ws0, ws1) and torch.equal(i0, i1) and torch.equal(w0, w1)
    assert ws1[-1] == 0


@pytest.mark.parametrize("name", ["lego_converged", "garden_cascades", "contract"])
def test_inference_loop_bit_exact(ref_raymarching, name):
    """The eval loop of renderer.py:764-802 driven with both backends on identical sigmas/rgbs."""
    c = cases.march_case(name)
    ro, rd, bits, aabb = cu(c["rays_o"]), cu(c["rays_d"]), cu(c["bits"]), cu(c["aabb"])
    N = ro.shape[0]
    nears, fars = rm.near_far_from_aabb(ro, rd, aabb, c["min_near"])

    def field(xyzs):       # deterministic stand-in for the network
        s = (xyzs.sum(-1) * 37.0).sin().abs() * 30.0
        return s, (xyzs * 0.5 + 0.5).clamp(0, 1)

    def loop(mod):           # mod: the reference extension, or None for ours
        ws = torch.zeros(N, device="cuda"); depth = torch.zeros(N, device="cuda"); image = torch.zeros(N, 3, device="cuda")
        alive = torch.arange(N, dtype=torch.int32, device="cuda"); rays_t = nears.clone()
        step = 0
        trace = []
        while step < 256:
            n_alive = alive.shape[0]
            if n_alive <= 0:
                break
            n_step = max(min(N // n_alive, 8), 1)
            if mod is not None:
                M = n_alive * n_step
                xyzs = torch.zeros(M, 3, device="cuda"); dirs = torch.zeros(M, 3, device="cuda"); ts = torch.zeros(M, 2, device="cuda")
                noises = torch.zeros(n_alive, device="cuda")
                mod.march_rays(n_alive, n_step, alive, rays_t, ro, rd, c["bound"], c["contract"], c["dt_gamma"],
                               c["max_steps"], c["C"], c["H"], bits, nears, fars, xyzs, dirs, ts, noises)
                s, col = field(xyzs)
                mod.composite_rays(n_alive, n_step, 1e-2, False, alive, rays_t, s, col, ts, ws, depth, image)
            else:
                xyzs, dirs, ts = rm.march_rays(n_alive, n_step, alive, rays_t, ro, rd, c["bound"], c["contract"], bits,
                                               c["C"], c["H"], nears, fars, False, c["dt_gamma"], c["max_steps"])
                s, col = field(xyzs)
                rm.composite_rays(n_alive, n_step, alive, rays_t, s, col, ts, ws, depth, image, 1e-2, False)
            trace.append((xyzs.clone(), ts.clone()))
            alive = alive[alive >= 0]
            step += n_step
        # every round's samples and the final buffers, as digests (bit-exact comparison)
        out = {"rounds": np.array(len(trace))}
        for i, (x, t) in enumerate(trace):
            out[f"x{i}"] = refreplay.digest(x); out[f"t{i}"] = refreplay.digest(t)
        for nm, a in (("ws", ws), ("depth", depth), ("image", image), ("rays_t", rays_t)):
            out[nm] = refreplay.digest(a)
        return out

    ref = ref_raymarching.summary(loop)
    ours = loop(None)
    assert int(ours["rounds"]) == int(ref["rounds"])
    for k in ours:
        if k != "rounds":
            assert ours[k] == ref[k], k


def test_packbits_morton_flatten_exact(ref_raymarching):
    g = torch.Generator().manual_seed(0)
    grid = torch.rand(2, 64 ** 3, generator=g).cuda() * 2 - 0.5
    grid[0, :100] = -1.0
    for thresh in (0.0, 0.37, 10.0):
        b0 = torch.empty(grid.numel() // 8, dtype=torch.uint8, device="cuda")
        ref_raymarching.packbits(grid, grid.numel() // 8, thresh, b0)
        b1 = rm.packbits(grid, thresh)
        assert torch.equal(b0, b1)
        # in-place variant + unaligned view
        buf = torch.zeros(grid.numel() // 8 + 8, dtype=torch.uint8, device="cuda")
        out = rm.packbits(grid, thresh, buf[1:1 + grid.numel() // 8])
        assert torch.equal(out, b0)
    coords = torch.randint(0, 128, (5000, 3), generator=g, dtype=torch.int32).cuda()
    i0 = torch.empty(5000, dtype=torch.int32, device="cuda")
    ref_raymarching.morton3D(coords, 5000, i0)
    i1 = rm.morton3D(coords)
    assert torch.equal(i0, i1)
    c1 = rm.morton3D_invert(i1)
    assert torch.equal(c1, coords)
    c0 = torch.empty(5000, 3, dtype=torch.int32, device="cuda")
    ref_raymarching.morton3D_invert(i0, 5000, c0)
    assert torch.equal(c0, c1)
    cnt = torch.randint(0, 50, (300,), generator=g)
    off = torch.cumsum(cnt, 0) - cnt
    rays = torch.stack([off, cnt], -1).int().cuda()
    M = int(cnt.sum())
    f0 = torch.zeros(M, dtype=torch.int32, device="cuda")
    ref_raymarching.flatten_rays(rays, 300, M, f0)
    assert torch.equal(f0, rm.flatten_rays(rays, M))


def test_sph_from_ray_close(ref_raymarching):
    ro, rd = cases.rays(500, seed=9)
    ro, rd = ro.cuda() * 0.2, rd.cuda()
    c0 = torch.empty(500, 2, device="cuda")
    ref_raymarching.sph_from_ray(ro, rd, 4.0, 500, c0)
    c1 = rm.sph_from_ray(ro, rd, 4.0)
    assert torch.allclose(c0, c1, atol=1e-6, rtol=0)
