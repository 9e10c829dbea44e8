"""GPU: the scatter (n2m_s0_encode_bwd) gives the same gradient table in both of its launch forms, beside the TV pass (n2m_s0_tv).

The per-slot form (k_s0_encode_bwd) runs one 128-thread walker per CTA on every SM; the whole-SM form (k_s0_scatter_walkers) runs 8
walkers per 1024-thread CTA, one CTA per SM, on 1/nparts of the SMs.  The form is forced through n2m_s0_set_scatter_form on marched
batches, whole batch and two ray-range parts, each time with the TV pass on a forked stream into the same table: the table must be within
the fp32 summation-order bound of test_gpu_grid_passes.py of the float64 oracle entry by entry, the two forms within the sum of their
bounds of each other, found_inf clear and the TV sample counts (counters[3], [15]) identical.
"""
import pytest
import torch

from nerf2mesh_b200._lib import call
from test_gpu_grid_passes import LAM, LS, Bufs, ScatterRef, TVRef, _forked, marched, random_cot

pytestmark = pytest.mark.gpu

FORMS = {"per_slot": 1, "whole_sm": 2}


def within(gpu, ref, tol, what):
    """|gpu - ref| <= tol entry by entry (an entry whose exact sum is 0 may cancel to a tiny nonzero in one summation order)"""
    err = (gpu.double().cpu() - ref).abs()
    assert (err <= tol).all(), f"{what}: {int((err > tol).sum())} entries beyond the bound, worst {float((err - tol).max()):.3e}"


@pytest.fixture
def forced_form():
    yield lambda form: call("n2m_s0_set_scatter_form", FORMS[form])
    call("n2m_s0_set_scatter_form", 0)


@pytest.mark.parametrize("name", ["converged4096", "garden_cascades", "contract"])
def test_scatter_forms_agree_beside_tv(name, forced_form):
    g, x, bounds = marched(name)
    M = len(x)
    cot = random_cot(M, 4)
    b = Bufs(g, x, cot, bounds, lambda_tv=LAM, loss_scale=LS)
    sref, tref = ScatterRef(g, x, cot), TVRef(g, x, b.tab_d, LAM, LS)
    ref = sref.ref.clone()
    tol = sref.tol()
    ref[:, 0] += tref.ref
    tol[:, 0] += tref.tol()
    out = {}
    main = torch.cuda.current_stream()
    side = _forked(8)[7]
    for form in FORMS:
        forced_form(form)
        for nparts in (1, 2):
            b.gt.zero_()
            b.set_bounds(b.bounds)                      # fresh counters: the TV pass adds its sample counts into [3] and [15]
            side.wait_stream(main)
            with torch.cuda.stream(side):
                b.tv()
            b.scatter(nparts)
            main.wait_stream(side)
            assert b.found_inf() == 0
            c = b.counters_d.cpu()
            assert (int(c[3]), int(c[15])) == (tref.n_in, tref.n_out), (form, nparts)
            gt = b.gt.cpu()
            within(gt[:, :3], ref, tol, f"{name} {form} nparts={nparts}")
            out[(form, nparts)] = gt[:, :3].double()
    for nparts in (1, 2):
        err = (out[("per_slot", nparts)] - out[("whole_sm", nparts)]).abs()
        assert (err <= 2 * tol).all(), f"{name}: the forms differ beyond the bound, nparts={nparts}"
