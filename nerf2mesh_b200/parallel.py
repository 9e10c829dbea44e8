"""Multi-GPU data parallelism for the fused stage-0 step: rays are sharded across ranks (one process
per GPU, each rank draws its own batch), every rank holds a full replica of the tables / MLPs, and the
only exchange per step is one all-reduce of the flat gradient buffers (hash-table gradients + MLP
gradients) plus the 4-byte found_inf flag, NCCL over NVLink / NVSwitch.  The reference has no working
multi-GPU path (its DDP scaffolding is unreachable)."""
import torch
import torch.distributed as dist


class GradSync:
    """Averages the loss-scaled gradients of a Stage0Trainer-like object (attributes gtable, g_mlp,
    opt_state) over the default process group; found_inf is OR-ed so every rank skips the same steps."""

    def __init__(self, trainer, group=None):
        if getattr(trainer, "ind_dim", 0):
            raise ValueError("data-parallel training with appearance codes (ind_dim > 0) is not supported")
        self.t = trainer
        self.group = group
        self.world = dist.get_world_size(group)
        self.backend = dist.get_backend(group)

    def buffers(self):
        return [self.t.gtable, self.t.g_mlp]

    def __call__(self):
        if self.world == 1:
            return
        for buf in self.buffers():
            if self.backend == "nccl":
                dist.all_reduce(buf, op=dist.ReduceOp.AVG, group=self.group)
            else:       # gloo (CPU tests) has no AVG
                dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group)
                buf.div_(self.world)
        dist.all_reduce(self.t.opt_state[3:4], op=dist.ReduceOp.MAX, group=self.group)

    def bytes_per_step(self):
        return sum(b.numel() * b.element_size() for b in self.buffers()) + 4


# ------------------------------------------------------------------------------------------------
# fused reduce-scatter + Adam + all-gather over NVLink peer memory (csrc/dp.cu)
# ------------------------------------------------------------------------------------------------
import ctypes  # noqa: E402

from . import _lib  # noqa: E402
from ._lib import F, P, U, call, ptr, stream  # noqa: E402

_lib.register({
    "n2m_ipc_export": [P, P, ctypes.POINTER(ctypes.c_uint64)],
    "n2m_ipc_open": [P, ctypes.POINTER(ctypes.c_void_p)],
    "n2m_ipc_close": [P],
    "n2m_dp_ctx_fill": [P, U, U, U, U, P, P, P, P, P, P, P, P],
    "n2m_dp_barrier": [P, P],
    "n2m_dp_adam": [P, U, U, U, U, P, P, P, P, P, P, P, P, P, P, F, P],
    "n2m_dp_adam_nvls": [P, P, P, U, U, U, U, P, P, P, P, P, P, P, P, P, P, F, P],
})
_lib.lib.n2m_dp_ctx_bytes.restype = ctypes.c_uint32


def slice_rows(rows, world):
    """Rows owned by one rank: ceil(rows / world) rounded up to a multiple of 4 (csrc/dp.cu slice_rows(): the float2
    colour moments follow `per` density moments in the slice-sized m / v arrays and must stay 8-byte aligned)."""
    return ((rows + world - 1) // world + 3) // 4 * 4


class PeerAdam:
    """Sharded optimizer for data-parallel training of a Stage0Trainer: each rank owns rows
    [r*per, (r+1)*per), per = ceil(R/W) rounded up to 4, of the hash tables.  After the backward pass one kernel per rank reads its
    slice of every peer's gradient table over NVLink, applies Adam to the slice and stores the refreshed table
    entries into every peer's table (include/n2m_b200_fused.h, "Data-parallel optimizer").  Replaces
    GradSync + Stage0Trainer.adam(); the fp32 colour masters and Adam moments exist only for the owned slice."""

    fused = True

    def __init__(self, trainer, group=None):
        if getattr(trainer, "ind_dim", 0):
            raise ValueError("data-parallel training with appearance codes (ind_dim > 0) is not supported")
        t = self.t = trainer
        self.group = group
        self.world = W = dist.get_world_size(group)
        self.rank = r = dist.get_rank(group)
        assert W <= 8, "PeerAdam supports up to 8 ranks (one NVSwitch domain)"
        dev = t.device
        R = t.rows
        self.per = per = slice_rows(R, W)
        lo, hi = min(R, r * per), min(R, (r + 1) * per)
        # two gradient-buffer parities (peers may still be reading parity p while parity p^1 is being zeroed): the trainer already owns
        # two tables; the MLP gradient vector gets its second copy here
        assert t.parity == 0
        t.gtables = [t.gtables[0], t.gtables[1]]
        t.g_mlps = [t.g_mlps[0], torch.zeros_like(t.g_mlps[0])]
        self.flags = torch.zeros(16, dtype=torch.int32, device=dev)
        self.epoch = torch.zeros(1, dtype=torch.int32, device=dev)
        # slice-sized optimizer state, initialised from the replicated parameters
        self.cm = torch.zeros(per, 2, device=dev)
        self.cm[: hi - lo].copy_(t.color_master[lo:hi])
        self.m = torch.zeros(per * 3, device=dev)
        self.v = torch.zeros(per * 3, device=dev)
        torch.cuda.synchronize()

        bufs = {"gtab0": t.gtables[0], "gtab1": t.gtables[1], "table": t.table, "gmlp0": t.g_mlps[0], "gmlp1": t.g_mlps[1],
                "opt": t.opt_state, "flags": self.flags}
        mine = {}
        for k, b in bufs.items():
            h = ctypes.create_string_buffer(64)
            off = ctypes.c_uint64(0)
            call("n2m_ipc_export", ptr(b), ctypes.cast(h, ctypes.c_void_p), ctypes.byref(off))
            mine[k] = (bytes(h.raw), int(off.value))
        everyone = [None] * W
        dist.all_gather_object(everyone, mine, group=group)
        self._opened = {}
        ptrs = {k: [0] * W for k in bufs}
        for p in range(W):
            for k in bufs:
                if p == r:
                    ptrs[k][p] = bufs[k].data_ptr()
                    continue
                hb, off = everyone[p][k]
                base = self._opened.get((p, hb))
                if base is None:
                    out = ctypes.c_void_p()
                    hbuf = ctypes.create_string_buffer(hb, 64)
                    call("n2m_ipc_open", ctypes.cast(hbuf, ctypes.c_void_p), ctypes.byref(out))
                    base = out.value
                    self._opened[(p, hb)] = base
                ptrs[k][p] = base + off

        def arr(k):
            a = (ctypes.c_void_p * W)(*ptrs[k])
            return ctypes.cast(a, ctypes.c_void_p), a          # keep `a` alive

        keep = []
        args = []
        for k in ("gtab0", "gtab1", "table", "gmlp0", "gmlp1", "opt", "flags"):
            c, a = arr(k); keep.append(a); args.append(c)
        nbytes = int(_lib.lib.n2m_dp_ctx_bytes())
        host = ctypes.create_string_buffer(nbytes)
        call("n2m_dp_ctx_fill", ctypes.cast(host, ctypes.c_void_p), W, r, R, t.n_mlp, *args, ptr(self.epoch))
        self.ctx = torch.frombuffer(bytearray(host.raw), dtype=torch.uint8).to(dev)
        torch.cuda.synchronize()
        dist.barrier(group=group)
        # from here on trainer.color_master is stale (the masters live in the per-rank slices): exports must gather them
        t._color_master_provider = self.gather_color_master

    zero_inside = False        # False: the trainer zeroes the next-parity gradient buffers on a side stream under the step (Stage0Trainer.step)

    def run(self, parity):
        """Enqueue barrier -> reduce-scatter + Adam + all-gather -> barrier for gradient parity `parity`."""
        t = self.t
        nxt = parity ^ 1
        zi = self.zero_inside
        call("n2m_dp_adam", ptr(self.ctx), parity, self.world, t.rows, t.n_mlp, ptr(self.cm), ptr(self.m), ptr(self.v),
             ptr(t.mlp), ptr(t.m_mlp), ptr(t.v_mlp), ptr(t.wpack), ptr(t.gtables[nxt]) if zi else None, ptr(t.g_mlps[nxt]) if zi else None,
             ptr(t.opt_state), t.cfg.eps, stream())

    def nvlink_bytes_per_step(self):
        W = self.world
        return int((W - 1) * self.per * (16 + 8) + (W - 1) * self.t.n_mlp * 4)

    def gather_color_master(self):
        """Full fp32 colour master table (for export): all-gather of the slices."""
        parts = [torch.zeros_like(self.cm) for _ in range(self.world)]
        dist.all_gather(parts, self.cm, group=self.group)
        return torch.cat(parts)[: self.t.rows]


class NvlsAdam(PeerAdam):
    """PeerAdam with the gradient reduce-scatter done INSIDE the NVSwitch and the table all-gather as multicast stores
    (csrc/dp.cu k_dp_adam_tables_mc: multimem.ld_reduce / multimem.st on multicast addresses).  The buffers the peers touch (both
    gradient-table parities, the working table, the MLP gradient vectors, the barrier flags) are re-allocated as
    torch.distributed._symmetric_memory tensors -- PyTorch does the VMM / multicast-object plumbing, the data path is this repo's
    kernel.  Raises when the fabric / driver offers no multicast (callers fall back to PeerAdam, then to NCCL)."""

    def __init__(self, trainer, group=None):
        if getattr(trainer, "ind_dim", 0):
            raise ValueError("data-parallel training with appearance codes (ind_dim > 0) is not supported")
        import torch.distributed._symmetric_memory as symm_mem
        t = self.t = trainer
        self.group = group
        pg = group if group is not None else dist.group.WORLD
        self.world = W = dist.get_world_size(group)
        self.rank = r = dist.get_rank(group)
        assert W <= 8, "one NVSwitch domain"
        dev = t.device
        R = t.rows
        self.per = per = slice_rows(R, W)
        lo, hi = min(R, r * per), min(R, (r + 1) * per)
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                symm_mem.enable_symm_mem_for_group(pg.group_name)      # needed by older torch; a deprecated no-op in newer ones
            except Exception:      # noqa: BLE001
                pass

        def sym(src):
            buf = symm_mem.empty(tuple(src.shape), dtype=src.dtype, device=dev)
            buf.copy_(src)
            return buf, symm_mem.rendezvous(buf, pg)

        assert t.parity == 0
        gt0, h_gt0 = sym(t.gtables[0])
        gt1, h_gt1 = sym(t.gtables[1])
        table, h_tab = sym(t.table)
        gm0, h_gm0 = sym(t.g_mlps[0])
        gm1, h_gm1 = sym(torch.zeros_like(t.g_mlps[0]))
        flags, h_fl = sym(torch.zeros(16, dtype=torch.int32, device=dev))
        mc = [int(h_gt0.multicast_ptr), int(h_gt1.multicast_ptr), int(h_tab.multicast_ptr)]
        if not all(mc):
            raise RuntimeError("symmetric memory without multicast support (no NVLS on this fabric / driver)")
        self.mc_gtab, self.mc_table = mc[:2], mc[2]
        self._handles = (h_gt0, h_gt1, h_tab, h_gm0, h_gm1, h_fl)
        # the trainer now works on the symmetric buffers
        t.gtables, t.table = [gt0, gt1], table
        t.g_mlps = [gm0, gm1]
        t._graphs = {}
        self.flags = flags
        self.epoch = torch.zeros(1, dtype=torch.int32, device=dev)
        self.cm = torch.zeros(per, 2, device=dev)
        self.cm[: hi - lo].copy_(t.color_master[lo:hi])
        self.m = torch.zeros(per * 3, device=dev)
        self.v = torch.zeros(per * 3, device=dev)

        def arr(vals):
            a = (ctypes.c_void_p * W)(*[int(v) for v in vals])
            return ctypes.cast(a, ctypes.c_void_p), a

        keep, args = [], []
        for h in (h_gt0, h_gt1, h_tab, h_gm0, h_gm1):
            c, a = arr(list(h.buffer_ptrs)); keep.append(a); args.append(c)
        c, a = arr([t.opt_state.data_ptr()] * W); keep.append(a); args.append(c)          # peers never read opt_state (found_inf goes through the flags)
        c, a = arr(list(h_fl.buffer_ptrs)); keep.append(a); args.append(c)
        nbytes = int(_lib.lib.n2m_dp_ctx_bytes())
        host = ctypes.create_string_buffer(nbytes)
        call("n2m_dp_ctx_fill", ctypes.cast(host, ctypes.c_void_p), W, r, R, t.n_mlp, *args, ptr(self.epoch))
        self.ctx = torch.frombuffer(bytearray(host.raw), dtype=torch.uint8).to(dev)
        torch.cuda.synchronize()
        dist.barrier(group=group)
        t._color_master_provider = self.gather_color_master

    def run(self, parity):
        t = self.t
        nxt = parity ^ 1
        zi = self.zero_inside
        call("n2m_dp_adam_nvls", ptr(self.ctx), ctypes.c_void_p(self.mc_gtab[parity]), ctypes.c_void_p(self.mc_table), parity, self.world,
             t.rows, t.n_mlp, ptr(self.cm), ptr(self.m), ptr(self.v), ptr(t.mlp), ptr(t.m_mlp), ptr(t.v_mlp), ptr(t.wpack),
             ptr(t.gtables[nxt]) if zi else None, ptr(t.g_mlps[nxt]) if zi else None, ptr(t.opt_state), t.cfg.eps, stream())

    def nvlink_bytes_per_step(self):
        return int(self.per * (16 + 8) + (self.world - 1) * self.t.n_mlp * 4)


def make_grad_sync(trainer, mode="auto", group=None):
    """Data-parallel optimizer for `trainer`: 'nvls' (in-switch reduce + multicast all-gather), 'peer' (P2P loads / stores over NVLink),
    'nccl' (all-reduce + replicated Adam) or 'auto' = the one moving the fewest bytes at this world size that every rank can set up.
    Collective: all ranks must call it with the same mode.  Returns (sync, mode_used)."""
    # per rank the in-switch reduce-scatter sends 16 B x rows whatever W is, P2P loads 16 B x rows x (W-1)/W each way, and the
    # multicast all-gather 8 B x rows / W instead of 8 B x rows x (W-1)/W: the byte counts cross at W = 4
    W = dist.get_world_size(group)
    order = {"auto": ["nvls", "peer", "nccl"] if W > 4 else ["peer", "nccl"], "nvls": ["nvls", "peer", "nccl"],
             "peer": ["peer", "nccl"], "nccl": ["nccl"]}[mode]
    for m in order:
        if m == "nccl":
            return GradSync(trainer, group), "nccl"
        ok = torch.ones(1, device=trainer.device)
        sync = None
        try:
            sync = NvlsAdam(trainer, group) if m == "nvls" else PeerAdam(trainer, group)
        except Exception as e:      # noqa: BLE001
            import sys
            print(f"[rank {dist.get_rank(group)}] {m} data-parallel optimizer unavailable ({str(e)[:200]})", file=sys.stderr)
            ok.zero_()
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
        if ok.item() == 1:
            return sync, m
        del sync
    raise RuntimeError("unreachable")
