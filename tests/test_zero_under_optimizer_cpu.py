"""CPU: with deferred zeroing, a single-GPU step zeroes the other gradient table on a side stream forked after the forward and
backward launches, underneath the optimizer sweep, and joins it before the step ends (the CUDA layer mocked out)."""
import types

import nerf2mesh_b200.stage0 as S0
import torch


def test_other_gradient_table_is_zeroed_under_the_optimizer(monkeypatch):
    log = []
    cur = {"s": "main"}
    monkeypatch.setattr(S0, "call", lambda name, *a: log.append((cur["s"], name)))
    monkeypatch.setattr(S0, "ptr", lambda t: 0)
    monkeypatch.setattr(S0, "stream", lambda: 0)

    class FakeStream:
        def __init__(self, name):
            self.name = name

        def wait_stream(self, o):
            log.append((self.name, "wait " + o.name))

        def wait_event(self, e):
            pass

    streams = iter(f"side{i}" for i in range(100))

    class Ctx:
        def __init__(self, s):
            self.s = s

        def __enter__(self):
            self.prev, cur["s"] = cur["s"], self.s.name

        def __exit__(self, *a):
            cur["s"] = self.prev
            return False

    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream(cur["s"]))
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream(next(streams)))
    monkeypatch.setattr(torch.cuda, "stream", lambda s: Ctx(s))

    class T:
        def __init__(self, name=None):
            self.name = name

        def zero_(self):
            log.append((cur["s"], "zero " + str(self.name)))
            return self

        def __getitem__(self, k):
            return self

        def data_ptr(self):
            return 0

    tr = object.__new__(S0.Stage0Trainer)
    tr.cfg = types.SimpleNamespace(lambda_tv=1e-8, eps=1e-15, num_levels=16)
    slot = types.SimpleNamespace(**{k: T() for k in ("rays_o", "rays_d", "gt", "bg", "noises", "rays", "counters", "tbuf", "recs",
                                                     "cam_nf")}, has_alpha=True)
    tr.slots, tr.cur = [slot, slot], 0
    for k in ("table", "offsets", "enc_tiles", "opt_state", "wpack", "out", "dout", "image", "weights_sum", "depth", "denc_tiles",
              "color_master", "m_table", "v_table", "mlp", "m_mlp", "v_mlp", "loss_acc"):
        setattr(tr, k, T())
    tr.gtables, tr.g_mlps, tr._zero_stream = [T("g0"), T("g1")], [T()], None
    tr.params = S0.S0Params(); tr.Mcap, tr.N, tr.rows, tr.parity, tr.device = 128, 4, 160, 0, "cpu"
    tr._tv_stream, tr._part_streams, tr._adam_stream = None, [], None
    tr.fused_fwd, tr.tv_fallback_points, tr._graphs, tr.adaptive = False, 1000, {}, False
    tr.defer_zero, tr.nparts = True, 2

    for run in (lambda: tr._compute_then_adam(), lambda: (tr._compute_sg(), tr._adam_sg())):
        log.clear()
        run()
        names = [n for _, n in log]
        zero = names.index("zero g1")                       # the other parity, never the table this step accumulates into
        assert "zero g0" not in names
        side = log[zero][0]
        assert side != "main"
        last_scatter = max(i for i, n in enumerate(names) if n == "n2m_s0_encode_bwd")
        fork = log.index((side, "wait main"))
        assert last_scatter < fork < zero < names.index("n2m_s0_adam_head")
        assert ("main", "n2m_s0_adam_tables_keep") in log and "n2m_s0_adam_tables" not in names
        assert log.index(("main", "wait " + side)) > names.index("n2m_s0_adam_tables_keep")     # joined within the step
