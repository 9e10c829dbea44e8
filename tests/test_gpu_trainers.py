"""Two stage-0 trainers in one process: constructing a trainer must not change what another trainer's step computes (no launch reads
state that a constructor or a setter of one trainer sets for the whole process).  Tolerances: those of the other two-run stage-0
comparisons (loss 1e-5 relative, gradients 1e-4 of the tensor's largest entry: fp32 atomic summation order)."""
import pytest
import torch

import cases
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200.stage0 import Stage0Config, Stage0Trainer

pytestmark = pytest.mark.gpu

N = 96


def make(seed, lambda_tv):
    tr = Stage0Trainer(Stage0Config(bound=1.0, num_rays=N, max_samples=N * 256, lambda_tv=lambda_tv), seed=seed)
    grid, bits, bricks = S.occupancy_regime("converged")
    tr.set_occupancy(bits, grid)
    return tr, bricks


def test_second_trainer_leaves_the_first_trainers_step_alone():
    """Trainer A's forward + backward on a fixed batch from a fixed state, before and after trainer B is constructed.  The TV weight is
    large enough for the TV gradient to be a visible part of the density-table gradient, and the TV pass must count every sample
    (counters[3] + counters[15] == M) both times, so a TV evaluation that went missing cannot hide behind the random-point fallback."""
    tr, bricks = make(seed=0, lambda_tv=1e-2)
    ro, rd = cases.rays(N, seed=3)
    gt = S.render_bricks(ro, rd, bricks)
    g = torch.Generator().manual_seed(5)
    bg, noises = torch.rand(N, 3, generator=g), torch.rand(N, generator=g)
    init = tr.export_reference_state()

    def run():
        tr.load_reference_state(init)
        tr.gtable.zero_(); tr.g_mlp.zero_()
        tr.rays_o.copy_(ro); tr.rays_d.copy_(rd); tr.gt.copy_(gt); tr.bg.copy_(bg); tr.noises.copy_(noises)
        tr.forward_backward()
        torch.cuda.synchronize()
        M = int(tr.counters[1].item())
        assert M > 0 and int(tr.counters[3].item()) + int(tr.counters[15].item()) == M
        return tr.read_loss(), tr.export_reference_grads()

    loss_a, g_a = run()
    make(seed=1, lambda_tv=1e-8)             # trainer B
    loss_b, g_b = run()
    assert abs(loss_b - loss_a) <= 1e-5 * abs(loss_a), (loss_a, loss_b)
    for name in g_a:
        a, r = g_b[name].double(), g_a[name].double()
        assert (a - r).abs().max().item() <= 1e-4 * r.abs().max().item() + 1e-12, name
