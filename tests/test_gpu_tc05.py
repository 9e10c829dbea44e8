"""Pins the wgmma descriptor conventions of csrc/wg.cuh against torch.matmul: one
128 x N x K GEMM (two m64 wgmma halves) with each operand K-major or MN-major (all four combinations the fused MLP
kernels use: forward, dgrad, wgrad)."""
import pytest
import torch

from nerf2mesh_b200 import _lib
from nerf2mesh_b200._lib import P, U, I, call, ptr, stream

pytestmark = pytest.mark.gpu

from profiles.probes import call as probe_call


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("N,K", [(64, 64), (16, 64), (48, 64), (64, 48), (32, 16), (64, 128)])
def test_umma_matches_matmul(a_mn, b_mn, N, K):
    g = torch.Generator().manual_seed(N * 131 + K + a_mn * 7 + b_mn)
    A = (torch.randn(128, K, generator=g) * 0.5).half()      # logical A [M=128, K]
    B = (torch.randn(N, K, generator=g) * 0.5).half()        # logical B [N, K]
    ref = A.float() @ B.float().t()
    Ap = (A.t().contiguous() if a_mn else A).cuda()          # MN-major: stored [K, M]
    Bp = (B.t().contiguous() if b_mn else B).cuda()          # MN-major: stored [K, N]
    D = torch.full((128, N), float("nan"), device="cuda")
    probe_call("n2m_tc_probe", ptr(Ap), ptr(Bp), ptr(D), N, K, a_mn, b_mn, stream())
    torch.cuda.synchronize()
    err = (D.cpu() - ref).abs().max().item()
    assert err <= 1e-3 * ref.abs().max().item(), f"max err {err}"
