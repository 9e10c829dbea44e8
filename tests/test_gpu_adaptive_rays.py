"""GPU: the adaptive ray count of stage 0 (Stage0Config.adaptive_num_rays, the reference's --adaptive_num_rays of the `-O` preset).

After every march the device computes the next batch's ray count exactly as the reference's Trainer.train_step does
(nerf/utils.py:795-797: num_rays = int(round((num_points / M) * num_rays))) and every later kernel reads the count from device memory.
Checked here: the rule itself against Python, the n / M sequence and one step's loss, image and gradients against the unmodified
reference trainer over the reference kernels, that rows past n have no effect, that every launch mode gives the same sequence, the
clamp / capacity accounting, and (with two GPUs) per-rank counts under NCCL data parallelism."""
import os
import socket

import pytest
import torch

import test_gpu_reference_parity as RP
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200.stage0 import MLP_LAYOUT, Stage0Config, Stage0Trainer

pytestmark = pytest.mark.gpu


def _expected(P, M, n, max_rays):
    """the reference's rule (utils.py:797) with this project's clamp to [1, max_rays]; M == 0 keeps n"""
    if M == 0:
        return n
    return min(max(int(round((P / M) * n)), 1), max_rays)


# ------------------------------------------------------------------------------------------------
# 1. the rule on the device
# ------------------------------------------------------------------------------------------------
def test_rule_on_the_device_matches_python():
    """Rays that all cross the full-occupancy cube along the same line march the same count c each, rays pointing away march none: the
    march then has M = (hitting rays among the first n) * c, and num_points is chosen to give exact .5 ties, requests that round to 0
    (clamped to 1), requests above max_rays (clamped and counted) and M == 0."""
    max_rays = 256
    cfg = Stage0Config(bound=1.0, dt_gamma=0.0, num_rays=64, max_samples=max_rays * 1024, adaptive_num_rays=True, max_rays=max_rays)
    tr = Stage0Trainer(cfg, seed=0)
    tr.set_occupancy(torch.full_like(tr.density_bitfield, 255))
    dev = "cuda"

    def load(hit, tilt=0.0):
        ro = torch.tensor([0.0, 0.0, -3.0], device=dev).repeat(max_rays, 1)
        rd = torch.tensor([0.0, tilt, 1.0], device=dev).repeat(max_rays, 1)
        rd[~hit.to(dev)] = torch.tensor([0.0, 0.0, -1.0], device=dev)
        tr.slots[tr.cur].load(ro, rd, torch.zeros(max_rays, 4, device=dev), torch.zeros(max_rays, 3, device=dev),
                              torch.zeros(max_rays, device=dev))

    def march(n, P):
        tr.ray_ctl[0] = n
        tr.cfg.num_points = P
        tr.march()
        torch.cuda.synchronize()
        return int(tr.counters[0].item()), int(tr.counters[16].item()), int(tr.ray_ctl[0].item())

    for tilt in [i / 64 for i in range(16)]:                    # a ray whose count c is even: the ties below are then exact
        load(torch.ones(max_rays, dtype=torch.bool), tilt)
        c, n_rec, _ = march(1, 1000)
        if c % 2 == 0:
            break
    assert c > 100 and n_rec == 1 and c % 2 == 0, c
    tr.check_rays()
    cases_ = []
    for n in (1, 2, 4, 8, 64, 128, 256):                        # powers of two: P / (n c) * n == fl(P / c), so P = c k + c / 2 ties
        for k in (0, 1, 2, 3, 10, 255):
            cases_.append((n, c * k + c // 2))
        cases_ += [(n, c * 7 + 1), (n, c * 7 - 1), (n, 1)]
    for n in (3, 5, 100, 255, 200):
        cases_ += [(n, P) for P in (1, c, 3 * c // 2, 2 ** 18, 12345, c * n * 3 + 7)]
    ties = 0
    for n, P in cases_:
        M, n_rec, nxt = march(n, P)
        assert n_rec == n and M == n * c, (n, P, M)
        assert nxt == _expected(P, M, n, max_rays), (n, P, M, nxt)
        ties += (P / M) * n % 1 == 0.5
    assert ties >= 20
    # rays >= n are not marched, whatever they hold; M counts the active hitting rays only
    hit = torch.arange(max_rays) % 3 == 0
    load(hit, tilt)
    M, _, nxt = march(100, 2 ** 18)
    assert M == int(hit[:100].sum()) * c and nxt == _expected(2 ** 18, M, 100, max_rays)
    # clamp accounting
    clamped, largest, _ = tr.check_rays()
    want = [int(round((P / (n * c)) * n)) for n, P in cases_] + [int(round((2 ** 18 / M) * 100))]
    assert clamped == sum(w > max_rays for w in want) > 0 and largest == max(want)
    # M == 0: the count stays
    load(torch.zeros(max_rays, dtype=torch.bool))
    for n in (1, 77, 256):
        M, n_rec, nxt = march(n, 2 ** 18)
        assert M == 0 and n_rec == n and nxt == n
    assert tr.check_rays() == (0, 0, 256)


# ------------------------------------------------------------------------------------------------
# helpers: a warmed-up state, batches of max_rays rows
# ------------------------------------------------------------------------------------------------
def _warm_state(name, steps=40):
    c = RP.CASES[name]
    grid, bits, bricks = RP._scene(c)
    tr = RP._make_ours(c, bits, grid)
    RP._warm_up(tr, c, bricks, steps)
    return c, bricks, tr.export_reference_state()


def _adaptive(c, state, num_rays=4096, max_rays=16384, **kw):
    cfg = Stage0Config(bound=c["bound"], dt_gamma=c["dt_gamma"], num_rays=num_rays, max_samples=4096 * c["cap"],
                       lambda_entropy=c["lambda_entropy"], lambda_tv=c.get("lambda_tv", 1e-8), adaptive_num_rays=True,
                       max_rays=max_rays, **kw)
    tr = Stage0Trainer(cfg, seed=3)
    tr.load_reference_state(state)
    tr.use_cam_near_far = c["cam_nf"]
    return tr


def _pool(c, bricks, rows, seed):
    """`rows` rays of the case's cameras with their ground truth and camera near / far, on the device"""
    g = torch.Generator().manual_seed(seed)
    poses = S.orbit_cameras(100, radius=c["radius"], seed=seed)
    ro, rd, _, _ = S.sample_rays(poses, S.lego_intrinsics(), 800, 800, rows, g)
    gt = RP._gt(c, ro, rd, bricks)
    cnf = RP._cam_nf(c, ro)
    return ro.cuda(), rd.cuda(), gt.cuda(), (cnf.cuda() if cnf is not None else None)


# ------------------------------------------------------------------------------------------------
# 2. sequence parity with the reference trainer
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lego", "garden"])
def test_sequence_matches_reference_trainer(name):
    ref_stage, ns = RP._ref_stack()
    c, bricks, state = _warm_state(name)
    tr = _adaptive(c, state)
    max_rays = tr.N
    rt = RP._ref_trainer(ref_stage, ns, c, state, True)
    rt.opt.adaptive_num_rays, rt.opt.num_rays, rt.opt.num_points = True, 4096, 2 ** 18
    seq = []
    for step in range(32):
        ro, rd, gt, cnf = _pool(c, bricks, max_rays, 500 + step)
        n = rt.opt.num_rays
        assert int(tr.ray_ctl[0].item()) == n, (step, n)
        # the reference takes the first n rows; its two draws (bg in train_step, noises in march_rays_train) go into our first n rows
        seed = 7000 + step
        torch.manual_seed(seed)
        bg_n = torch.rand(n, 3, device="cuda"); noises_n = torch.rand(n, device="cuda")
        bg = torch.full((max_rays, 3), float("nan"), device="cuda"); bg[:n] = bg_n
        noises = torch.full((max_rays,), float("nan"), device="cuda"); noises[:n] = noises_n
        data = dict(rays_o=ro[:n].contiguous(), rays_d=rd[:n].contiguous(), index=[0], images=gt[:n].contiguous())
        if cnf is not None:
            data["cam_near_far"] = cnf[:n].contiguous()
        res = {}
        ren = rt.model.render

        def spy(*a, **k):
            out = ren(*a, **k)
            res.update(M=int(out["num_points"]), image=out["image"].detach())
            return out
        rt.model.render = spy
        try:
            torch.manual_seed(seed)
            _, _, loss_ref = rt.train_step(dict(data))           # forward only: the march does not depend on the parameters
        finally:
            rt.model.render = ren
        tr.step(ro, rd, gt, bg, noises, cam_near_far=cnf, use_graph=step > 0)
        torch.cuda.synchronize()
        assert int(tr.counters[16].item()) == n and int(tr.counters[0].item()) == res["M"], (step, n, res["M"])
        assert int(tr.ray_ctl[0].item()) == rt.opt.num_rays, step
        if step == 0:                                            # same parameters on both sides: loss and image as well
            loss_ours = tr.read_loss()
            assert abs(loss_ours - loss_ref.item()) <= 1e-3 * abs(loss_ref.item()), (loss_ours, loss_ref.item())
            assert (tr.image[:n] - res["image"]).abs().max().item() <= 1e-3 * res["image"].abs().max().item()
        seq.append((n, res["M"]))
    ns_ = [n for n, _ in seq]
    assert len(set(ns_)) > 2, seq                                # the count really moves
    assert any(n != 4096 and n != max_rays for n in ns_), seq


@pytest.mark.parametrize("name", ["lego", "garden"])
def test_adapted_step_matches_reference_gradients(name):
    """one step at an adapted count n (not num_rays, not max_rays): loss, image and the reference-format gradients against the
    reference's fp16 and fp32 runs, with the tolerances of test_fused_step_matches_reference_cuda_path except for the MLP weights'
    noise factor (see below)"""
    ref_stage, ns = RP._ref_stack()
    c, bricks, state = _warm_state(name)
    tr = _adaptive(c, state)
    n = 3001
    ro, rd, gt, cnf = _pool(c, bricks, tr.N, 77)
    seed = 4242
    torch.manual_seed(seed)
    bg_n = torch.rand(n, 3, device="cuda"); noises_n = torch.rand(n, device="cuda")
    data = dict(rays_o=ro[:n].contiguous(), rays_d=rd[:n].contiguous(), index=[0], images=gt[:n].contiguous())
    if cnf is not None:
        data["cam_near_far"] = cnf[:n].contiguous()
    scale = 65536.0
    for _ in range(16):
        r16a = RP._ref_step(RP._ref_trainer(ref_stage, ns, c, state, True, scale), data, seed)
        if all(torch.isfinite(g).all().item() for g in r16a["grads"].values()):
            break
        scale *= 0.5
    r16b = RP._ref_step(RP._ref_trainer(ref_stage, ns, c, state, True, scale), data, seed)
    r32 = RP._ref_step(RP._ref_trainer(ref_stage, ns, c, state, False), data, seed)
    if c.get("lambda_tv", 1e-8) == 0:
        for run in (r16a, r16b):
            run["grads"] = {k: v / scale for k, v in run["grads"].items()}
    tr.opt_state[0] = scale
    bg = torch.full((tr.N, 3), float("nan"), device="cuda"); bg[:n] = bg_n
    noises = torch.full((tr.N,), float("nan"), device="cuda"); noises[:n] = noises_n
    tr.slots[tr.cur].load(ro, rd, gt, bg, noises, cnf)
    tr._fill_params(True, c["alpha"])
    tr.ray_ctl[0] = n
    tr.forward_backward()
    torch.cuda.synchronize()
    assert int(tr.counters[16].item()) == n and int(tr.counters[0].item()) == r16a["M"] and tr.counters[2].item() == 0
    assert tr.opt_state[3].item() == 0
    assert torch.equal(tr.rays[:n, 1], r16a["rays"][:, 1])
    loss = tr.read_loss()
    assert abs(loss - r16a["loss"]) <= 1e-3 * abs(r16a["loss"]), (loss, r16a["loss"])
    for key, ours in (("image", tr.image[:n]), ("ws", tr.weights_sum[:n]), ("depth", tr.depth[:n])):
        assert RP._cmp(ours, r16a[key])["max_err_of_scale"] <= 1e-3, key
    g = tr.export_reference_grads()
    for nm in ["encoder.embeddings", "encoder_color.embeddings"] + [k for k, _ in MLP_LAYOUT]:
        ga, gb, g32 = r16a["grads"][nm], r16b["grads"][nm], r32["grads"][nm]
        vs32 = RP._cmp(g[nm], g32)
        if nm == "encoder.embeddings":
            assert vs32["rel_l2"] <= 1e-2 and vs32["cos"] > 0.9999, (nm, vs32)
            continue
        ref_noise = RP._cmp(ga, g32)
        floor = max(ref_noise["rel_l2"], RP._cmp(gb, ga)["rel_l2"])
        vs16 = RP._cmp(g[nm], ga)
        # both sides round the per-sample MLP gradients to fp16 independently, so each is about as far from the fp32 gradient as the
        # other, and how far depends on the state.  The warm-up is not bit-reproducible (atomic order), and over warmed-up garden
        # states at this n the colour-net weights measured 0.0017-0.0032 (reference) against 0.0019-0.0040 (ours), our step itself
        # bit-identical from run to run; ours / reference reached 2.5.  A wrong ray count or part boundary moves these by 1e-1 or more
        assert vs32["rel_l2"] <= 2.5 * ref_noise["rel_l2"] + 1e-3, (nm, vs32, ref_noise)
        assert vs16["rel_l2"] <= 2.5 * floor + 1e-3, (nm, vs16, floor)
        assert vs16["cos"] > 0.9999 or vs16["cos"] >= ref_noise["cos"] - 1e-3, (nm, vs16, ref_noise)


# ------------------------------------------------------------------------------------------------
# 3. rows past n have no effect
# ------------------------------------------------------------------------------------------------
def test_inactive_rows_have_no_effect():
    c, bricks, state = _warm_state("lego", steps=24)
    n = 2900
    ad = _adaptive(c, state, num_rays=n, max_rays=8192)
    fx = Stage0Trainer(Stage0Config(bound=c["bound"], dt_gamma=c["dt_gamma"], num_rays=n, max_samples=4096 * c["cap"]), seed=3)
    fx.load_reference_state(state)
    ro, rd, gt, _ = _pool(c, bricks, 8192, 31)
    g = torch.Generator(device="cuda").manual_seed(5)
    bg = torch.rand(8192, 3, device="cuda", generator=g); noises = torch.rand(8192, device="cuda", generator=g)
    nan = float("nan")
    pad = lambda t: torch.cat([t[:n], torch.full_like(t[n:], nan)])          # noqa: E731
    ad.slots[ad.cur].load(pad(ro), pad(rd), pad(gt), pad(bg), pad(noises))
    fx.slots[fx.cur].load(ro[:n], rd[:n], gt[:n], bg[:n], noises[:n])
    for t in (ad, fx):
        t._fill_params(True, True)
        t.forward_backward()
    torch.cuda.synchronize()
    assert int(ad.counters[16].item()) == n
    assert torch.equal(ad.counters[:16], fx.counters[:16])
    M = int(fx.counters[1].item())
    assert torch.equal(ad.rays[:n], fx.rays) and torch.equal(ad.recs[:M], fx.recs[:M])
    la, lf = ad.read_loss(), fx.read_loss()
    assert abs(la - lf) <= 1e-5 * abs(lf), (la, lf)
    for a, b in ((ad.image[:n], fx.image), (ad.weights_sum[:n], fx.weights_sum), (ad.depth[:n], fx.depth)):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6)
    ga, gf = ad.export_reference_grads(), fx.export_reference_grads()
    for k in gf:
        assert torch.isfinite(ga[k]).all(), k
        d = (ga[k] - gf[k]).double().norm() / max(gf[k].double().norm().item(), 1e-30)
        assert d <= 1e-4, (k, d.item())
    # the optimizer step sees no non-finite gradient and leaves finite parameters (a first Adam step moves every parameter by
    # +-lr whatever the gradient's size, so the two trainers' parameters are not compared here: their gradients are, above)
    assert ad.opt_state[3].item() == 0
    ad.adam()
    torch.cuda.synchronize()
    assert ad.opt_state[3].item() == 0 and ad.opt_state[2].item() == 1
    for k, v in ad.export_reference_state().items():
        if v.is_floating_point():
            assert torch.isfinite(v).all(), k


# ------------------------------------------------------------------------------------------------
# 4. every launch mode gives the same sequence
# ------------------------------------------------------------------------------------------------
def test_launch_modes_agree():
    c, bricks, state = _warm_state("lego", steps=24)
    max_rays = 16384
    batches = []
    for i in range(8):
        ro, rd, gt, _ = _pool(c, bricks, max_rays, 900 + i)
        g = torch.Generator(device="cuda").manual_seed(i)
        batches.append((ro, rd, gt, torch.rand(max_rays, 3, device="cuda", generator=g), torch.rand(max_rays, device="cuda", generator=g)))

    def run(use_graph=True, prefetch=None, nparts=1, fused_fwd=False):
        tr = _adaptive(c, state, max_rays=max_rays)
        tr.nparts, tr.fused_fwd = nparts, fused_fwd
        if prefetch:
            tr.prefetch_at = prefetch
        ns_, losses = [], []
        for i, b in enumerate(batches):
            nxt = batches[i + 1] if prefetch and i + 1 < len(batches) else None
            tr.step(*b, use_graph=use_graph, next_batch=nxt)
            torch.cuda.synchronize()
            ns_.append(int(tr.counters[16].item()))
            losses.append(tr.read_loss())
        return ns_, losses

    base_n, base_l = run(use_graph=False)
    assert len(set(base_n)) > 1, base_n
    for kw in (dict(), dict(prefetch="optimizer"), dict(prefetch="start"), dict(nparts=2), dict(nparts=4), dict(nparts=8),
               dict(fused_fwd=True), dict(prefetch="start", nparts=4, use_graph=False)):
        n_, l_ = run(**kw)
        assert n_ == base_n, (kw, n_, base_n)
        for i, (a, b) in enumerate(zip(l_, base_l)):          # summation order only; Adam amplifies it over the steps
            assert abs(a - b) <= (1e-3 if i < 3 else 1e-2) * abs(b), (kw, i, l_, base_l)


def test_dropped_prefetch_keeps_the_sequence():
    """A prefetched batch has been marched already, so its scan has written the count after it; dropping it (check_capacity,
    check_rays, render and density_volume do) must put the count back.  With drops in the middle of the run, every prefetch mode gives
    the sequence of the run without prefetch, and the same clamp report.  The evaluation render of all samples works in chunks of
    num_rays, so it does not overflow the sample slab sized for num_rays."""
    c, bricks, state = _warm_state("lego", steps=24)
    max_rays = 16384
    batches = []
    for i in range(10):
        ro, rd, gt, _ = _pool(c, bricks, max_rays, 950 + i)
        g = torch.Generator(device="cuda").manual_seed(50 + i)
        batches.append((ro, rd, gt, torch.rand(max_rays, 3, device="cuda", generator=g), torch.rand(max_rays, device="cuda", generator=g)))
    ro_e, rd_e, _, _ = _pool(c, bricks, 12000, 99)

    def run(prefetch):
        tr = _adaptive(c, state, max_rays=max_rays)
        if prefetch:
            tr.prefetch_at = prefetch
        ns_, reports = [], []
        for i, b in enumerate(batches):
            nxt = batches[i + 1] if prefetch and i + 1 < len(batches) else None
            tr.step(*b, next_batch=nxt)
            ns_.append(int(tr.counters[16].item()))
            if i in (2, 5):
                reports.append(tr.check_capacity())
            if i == 3:
                reports.append(tr.check_rays())
            if i == 4:
                tr.render(ro_e, rd_e)
            if i == 7:
                tr.render(ro_e, rd_e, early_stop=False)
                reports.append(tr.check_capacity(grow=False))
        reports.append(tr.check_rays())
        return ns_, reports

    # reports: check_capacity after steps 2 and 5 and after the all-samples render, check_rays after step 3 and at the end.  The
    # capacity reports' largest M also sees the staged marches, so only their overflow counts are compared
    base_n, base_r = run(None)
    assert len(set(base_n)) > 1 and all(base_r[k][0] == 0 for k in (0, 2, 3)), (base_n, base_r)
    for prefetch in ("optimizer", "start"):
        n_, r_ = run(prefetch)
        assert n_ == base_n, (prefetch, n_, base_n)
        assert [r_[k][0] for k in (0, 2, 3)] == [0, 0, 0] and (r_[1], r_[4]) == (base_r[1], base_r[4]), (prefetch, r_, base_r)


# ------------------------------------------------------------------------------------------------
# 5. accounting
# ------------------------------------------------------------------------------------------------
def test_clamp_empty_grid_and_capacity_accounting():
    c, bricks, state = _warm_state("lego", steps=8)
    ro, rd, gt, _ = _pool(c, bricks, 8192, 3)
    bg = torch.rand(8192, 3, device="cuda"); noises = torch.rand(8192, device="cuda")
    # a huge num_points pins n at max_rays; every step's request is clamped
    tr = _adaptive(c, state, num_rays=1024, max_rays=8192, num_points=2 ** 30)
    for _ in range(5):
        tr.step(ro, rd, gt, bg, noises)
    torch.cuda.synchronize()
    assert int(tr.counters[16].item()) == 8192
    clamped, largest, nxt = tr.check_rays()
    assert clamped == 5 and largest > 8192 and nxt == 8192
    assert tr.check_rays()[:2] == (0, 0)
    # an empty bitfield marches nothing: the count stays
    tr = _adaptive(c, state, num_rays=1500, max_rays=8192)
    tr.set_occupancy(torch.zeros_like(tr.density_bitfield))
    for _ in range(3):
        tr.step(ro, rd, gt, bg, noises)
    torch.cuda.synchronize()
    assert int(tr.counters[0].item()) == 0 and int(tr.counters[16].item()) == 1500 and tr.check_rays() == (0, 0, 1500)
    assert all(torch.isfinite(v).all() for v in tr.export_reference_state().values() if v.is_floating_point())
    # a sample overflow is still reported by check_capacity (and the slab grows)
    tr = Stage0Trainer(Stage0Config(bound=1.0, num_rays=1024, max_samples=1024 * 8, adaptive_num_rays=True, max_rays=8192), seed=3)
    tr.load_reference_state(state)
    tr.step(ro, rd, gt, bg, noises, use_graph=False)
    over, max_m = tr.check_capacity()
    assert over == 1 and max_m > 1024 * 8 and tr.Mcap >= max_m


# ------------------------------------------------------------------------------------------------
# 6. data parallel: each rank adapts its own count
# ------------------------------------------------------------------------------------------------
def _dp_worker(rank, world, port, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, "tests"))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from nerf2mesh_b200 import synthetic as S_
    from nerf2mesh_b200.parallel import GradSync
    grid, bits, bricks = S_.occupancy_regime("converged")
    max_rays = 4096
    batches = []
    for i in range(6):
        g = torch.Generator().manual_seed(100 * rank + i)
        ro, rd, _, _ = S_.sample_rays(S_.orbit_cameras(100, seed=rank), S_.lego_intrinsics(), 800, 800, max_rays, g)
        batches.append((ro, rd, S_.render_bricks(ro, rd, bricks), torch.rand(max_rays, 3, generator=g), torch.rand(max_rays, generator=g)))
    out = {}
    for mode in ("single", "nccl"):
        cfg = Stage0Config(bound=1.0, num_rays=512, max_samples=512 * 256, adaptive_num_rays=True, max_rays=max_rays, num_points=2 ** 15)
        tr = Stage0Trainer(cfg, seed=0)
        tr.set_occupancy(bits, grid)
        sync = GradSync(tr) if mode == "nccl" else None
        seq = []
        for i, b in enumerate(batches):
            tr.step(*b, grad_sync=sync, use_graph=i > 0)
            torch.cuda.synchronize()
            seq.append(int(tr.counters[16].item()))
        out[mode] = seq
        dist.barrier()
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_ranks_adapt_their_own_count():
    """NCCL grad_sync: the march does not depend on the parameters, so each rank's count sequence equals a single-GPU run of its own
    batches (the first step shares the parameters, so the second step's count already differs between ranks with different batches)"""
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = dict(q.get(timeout=600) for _ in range(2))
    [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    for r in range(2):
        assert res[r]["nccl"] == res[r]["single"], (r, res[r])
    assert res[0]["nccl"] != res[1]["nccl"]
