"""CPU: the host side of the adaptive ray count (Stage0Config.adaptive_num_rays) with the CUDA layer mocked -- which pointers reach the
march and the composite, the prefetch ordering it needs, config validation, and the C-ABI bindings of the two changed entry points."""
import os
import re
import types

import pytest
import torch

import nerf2mesh_b200.stage0 as S0

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_arg_count(name):
    src = open(os.path.join(ROOT, "include", "n2m_b200_fused.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", src)
    return len([a for a in m.group(1).split(",") if a.strip()])


def test_bindings_match_the_header():
    for name in ("n2m_s0_march", "n2m_s0_composite_loss"):
        assert len(S0._lib.SIGNATURES[name]) == _header_arg_count(name), name


def test_config_defaults_and_validation():
    c = S0.Stage0Config()
    assert not c.adaptive_num_rays and c.num_points == 2 ** 18 and c.max_rays == c.num_rays == 4096
    assert c.max_samples == 4096 * 128
    c = S0.Stage0Config(num_rays=1024, adaptive_num_rays=True)
    assert c.max_rays == 4096 and c.max_samples == 1024 * 128          # the sample capacity still follows num_rays
    assert S0.Stage0Config(num_rays=1024, adaptive_num_rays=True, max_rays=1024).max_rays == 1024
    with pytest.raises(ValueError):
        S0.Stage0Config(num_rays=1024, adaptive_num_rays=True, max_rays=512)
    with pytest.raises(ValueError):
        S0.Stage0Config(adaptive_num_rays=True, num_points=0)


@pytest.fixture
def mocked(monkeypatch):
    calls = []
    monkeypatch.setattr(S0, "call", lambda name, *a: calls.append((name, a)))
    monkeypatch.setattr(S0, "stream", lambda: 0)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return calls


def _trainer(adaptive):
    cfg = S0.Stage0Config(num_rays=128, max_steps=16, log2_hashmap_size=10, adaptive_num_rays=adaptive, num_points=5000)
    return S0.Stage0Trainer(cfg, device="cpu")


def test_adaptive_pointers_reach_march_and_composite(mocked):
    calls = mocked
    tr = _trainer(True)
    assert tr.N == 512 and tr.slots[0].rays_o.shape[0] == 512 and tr.image.shape[0] == 512
    assert tr.counters.numel() == 17 and tr.ray_ctl.tolist() == [128, 0, 0, 0]
    calls.clear()
    tr.march()
    tr.composite_loss(1, 2)
    (n1, a1), (n2, a2) = calls
    assert n1 == "n2m_s0_march" and a1[-3] == tr.ray_ctl.data_ptr() and a1[-2] == 5000 and a1[7] == 512
    assert n2 == "n2m_s0_composite_loss" and a2[-4] == tr.counters.data_ptr() + 4 * 16 and a2[-3:-1] == (1, 2)
    # evaluation rendering marches and composites every row of its chunks
    calls.clear()
    tr._render_all_samples(torch.zeros(600, 3), torch.ones(600, 3))
    marches = [a for n, a in calls if n == "n2m_s0_march"]
    composites = [a for n, a in calls if n == "n2m_s0_composite_loss"]
    assert len(marches) == len(composites) == 5      # 600 rays in chunks of num_rays = 128: the sample slab is sized for num_rays
    assert all(a[-3] is None and a[-2] == 0 for a in marches)
    assert all(a[-4] is None for a in composites)


def test_fixed_mode_passes_null(mocked):
    calls = mocked
    tr = _trainer(False)
    assert not tr.adaptive and tr.ray_ctl is None and tr.N == 128
    calls.clear()
    tr.march()
    tr.composite_loss()
    (_, a1), (_, a2) = calls
    assert a1[-3] is None and a1[-2] == 0 and a2[-4] is None
    assert tr.check_rays() == (0, 128, 128)


def test_check_rays_reads_and_resets_the_control_block(mocked):
    tr = _trainer(True)
    tr.ray_ctl.copy_(torch.tensor([300, 3, 9000, 0], dtype=torch.int32))
    assert tr.check_rays() == (3, 9000, 300)
    assert tr.ray_ctl.tolist() == [300, 0, 0, 0]


def test_start_prefetch_waits_for_the_current_march(monkeypatch):
    """prefetch_at == "start" in adaptive mode: the side stream's march of the next batch reads the count the current march writes, so it
    waits for an event recorded on the main stream right after that march (the start mark alone comes before it)"""
    log = []
    cur = {"s": "main"}

    class FakeStream:
        def __init__(self, name): self.name = name
        def wait_stream(self, o): log.append((self.name, "wait_stream", o.name))
        def wait_event(self, e): log.append((self.name, "wait_event", e.tag))
        def synchronize(self): pass

    class FakeEvent:
        n = 0
        def __init__(self): FakeEvent.n += 1; self.tag = None
        def record(self, s=None):
            self.tag = f"ev{FakeEvent.n}"
            log.append((s.name if s is not None else cur["s"], "record", self.tag))

    class Ctx:
        def __init__(self, s): self.s = s
        def __enter__(self): self.prev = cur["s"]; cur["s"] = self.s.name
        def __exit__(self, *a): cur["s"] = self.prev; return False

    streams = {"main": FakeStream("main")}
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: streams.setdefault(cur["s"], FakeStream(cur["s"])))
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: streams.setdefault("side", FakeStream("side")))
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: FakeEvent())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: Ctx(s))

    def trainer(mode, adaptive):
        tr = object.__new__(S0.Stage0Trainer)
        tr.adaptive = adaptive
        tr.ray_ctl, tr._ray_ctl_undo = torch.tensor([7, 0, 0, 0], dtype=torch.int32), torch.zeros(4, dtype=torch.int32)
        tr.prefetch_at, tr.defer_zero, tr.parity, tr.cur, tr.global_step, tr.device = mode, True, 0, 0, 0, "cpu"
        tr._prefetched, tr._side, tr._ev_done, tr._ev_march = None, None, [None, None], [None, None]
        tr.params = S0.S0Params(); tr.params.shading_full = 1; tr.params.gt_has_alpha = 1
        slot = types.SimpleNamespace(has_alpha=True, load=lambda *a: log.append((cur["s"], "load", None)))
        tr.slots = [slot, slot]
        tr._run = lambda name, fn, g: log.append((cur["s"], "run", name))
        return tr

    batch = (None,) * 4
    tr = trainer("start", True)
    tr.step(*batch, next_batch=batch)
    i_march = log.index(("main", "run", "march"))
    after = next(e for e in log[i_march + 1:] if e[0] == "main" and e[1] == "record")
    assert log.index(after) < log.index(("main", "run", "compute+adam"))       # recorded right after the march
    side_waits = [e[2] for e in log if e[0] == "side" and e[1] == "wait_event"]
    assert after[2] in side_waits
    assert log.index(("side", "wait_event", after[2])) < log.index(("side", "run", "march"))
    assert tr._ray_ctl_undo.tolist() == [7, 0, 0, 0]                            # saved for a drop_prefetch() before the staged march
    # the next step consumes the prefetched march (no march on main): the side stream orders the following march after it
    log.clear()
    tr.step(*batch, next_batch=batch)
    assert ("main", "run", "march") not in log
    assert sum(1 for e in log if e[0] == "side" and e[1] == "wait_event") == 2       # previous reader of the slot, start mark
    # optimizer mode: the mid mark after the compute already orders it; fixed mode: nothing extra
    for mode, adaptive, waits in (("optimizer", True, 2), ("start", False, 1)):
        log.clear(); streams.pop("side", None)
        tr = trainer(mode, adaptive)
        tr.step(*batch, next_batch=batch)
        assert sum(1 for e in log if e[0] == "side" and e[1] == "wait_event") == waits, (mode, adaptive)


def test_dropped_prefetch_restores_the_control_block(mocked):
    """the side-stream march of a prefetched batch saves the control block before it runs; dropping that batch (check_capacity,
    check_rays, render, density_volume) puts the block back, so the next march takes the count the reference would"""
    tr = _trainer(True)
    tr._side = types.SimpleNamespace(synchronize=lambda: None)
    tr.ray_ctl.copy_(torch.tensor([900, 2, 5000, 0], dtype=torch.int32))          # written by the staged march
    tr._ray_ctl_undo.copy_(torch.tensor([700, 1, 4000, 0], dtype=torch.int32))    # as it was before it
    tr._prefetched, tr.cur = 1, 0
    tr.drop_prefetch()
    assert tr.ray_ctl.tolist() == [700, 1, 4000, 0] and tr.cur == 1 and tr._prefetched is None
    tr.ray_ctl.copy_(torch.tensor([900, 2, 5000, 0], dtype=torch.int32))
    tr.drop_prefetch()                                                              # nothing staged: nothing restored
    assert tr.ray_ctl.tolist() == [900, 2, 5000, 0]
    tr._prefetched = 0
    assert tr.check_rays() == (1, 4000, 700)                                        # check_rays drops the staged batch first
    assert tr.ray_ctl.tolist() == [700, 0, 0, 0]
