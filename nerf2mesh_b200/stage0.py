"""Fused stage-0 train path: host side (allocation, CUDA-graph capture, import/export of
reference-format parameters).  All arithmetic runs in libn2m_b200.so (include/n2m_b200_fused.h).

`Stage0Trainer` owns the model state in the library's native layout (interleaved hash tables, packed
tensor-core weights, flat gradient / Adam buffers) and exposes

    loss = trainer.step(rays_o, rays_d, gt, bg_color)        # one full optimizer step

which is the fused equivalent of one iteration of the reference's Trainer.train_one_epoch
(nerf/utils.py:1152-1182: zero_grad, train_step -> NeRFRenderer.render, scaler.scale(loss).backward(),
post_train_step TV gradient, scaler.step(optimizer), scaler.update(), lr_scheduler.step()).
`load_reference_state` / `export_reference_state` convert to and from the reference checkpoint's
parameter names (encoder.embeddings, sigma_net.net.0.weight, ...).
"""
import ctypes
import math
from ctypes import c_float, c_uint32

import numpy as np
import torch

from . import _lib
from ._lib import F, I, P, U, call, ptr, stream
from .gridencoder.grid import level_offsets


class S0Params(ctypes.Structure):
    _fields_ = [(n, c_float) for n in ("bound", "grid_bound", "inv_2gb", "dt_gamma", "min_near", "T_thresh", "S",
                                       "lambda_mask", "lambda_specular", "lambda_tv", "lambda_entropy")] + \
               [(n, c_uint32) for n in ("contract", "max_steps", "cascades", "grid_size", "num_levels", "base_res",
                                        "shading_full", "gt_has_alpha", "ind_dim")]


PP = ctypes.POINTER(S0Params)

_lib.register({
    "n2m_s0_init": [],
    "n2m_s0_set_serial_march": [I],
    "n2m_s0_set_scatter_form": [I],
    "n2m_s0_tv": [PP, P, P, U, P, P, P, P, P, P, P],
    "n2m_s0_tv_random": [PP, P, P, P, P, P, U, P, P],
    "n2m_s0_pack_weights": [P, P, P],
    "n2m_s0_pack_tables": [P, P, U, P, P, P],
    "n2m_s0_unpack_tables": [P, P, U, P, P, P],
    "n2m_s0_unpack_grads": [P, U, P, P, P, P],
    "n2m_s0_march": [PP, P, P, P, P, P, P, U, P, P, P, P, U, P, U, P],
    "n2m_s0_encode_fwd": [PP, P, P, U, P, P, P, P, P, U, U, P],
    "n2m_s0_encode_points": [PP, P, P, P, U, P, P, P, P],
    "n2m_s0_grid_points": [U, U, U, F, P, P, P],
    "n2m_s0_grid_update": [P, U, F, P, P],
    "n2m_s0_packbits_dev": [P, U, P, F, P, P],
    "n2m_s0_mlp_fwd": [PP, P, P, U, P, P, P, U, U, P],
    "n2m_s0_composite_loss": [PP, P, P, P, P, U, U, P, P, P, P, P, P, P, P, P, U, U, P],
    "n2m_s0_mlp_bwd": [PP, P, P, P, U, P, P, P, P, U, U, P],
    "n2m_s0_encode_bwd": [PP, P, P, U, P, P, P, P, P, P, P, U, U, P],
    "n2m_s0_adam_head": [P, P, P],
    "n2m_s0_adam_tables": [P, P, P, P, P, U, P, F, P],
    "n2m_s0_adam_tables_keep": [P, P, P, P, P, U, P, F, P],
    "n2m_s0_adam_mlp": [P, P, P, P, P, P, F, P],
    "n2m_s0_adam_post": [P, P],
    "n2m_mark_untrained_grid": [P, U, P, U, P, F, P, F, U, U, P, P, P],
    "n2m_s0_fwd_fused": [PP, P, P, U, P, P, P, P, P, P, P, P, P],
    "n2m_s0_render_begin": [PP, P, P, P, P, U, P, P, P, P, P, P, P, P],
    "n2m_s0_render_rounds": [PP, P, P, P, U, P, U, P, P, P, P, P, P, P, U, P, P, P, P, P, P, P],
    "n2m_s0_render_finish": [P, P, P, F, U, P],
    "n2m_s0_ema_update": [P, P, P, P, P, P, U, F, P],
    "n2m_s0_ema_swap": [P, P, P, P, P, P, U, P, P],
    "n2m_s0_encode_fwd_codes": [PP, P, P, U, P, P, P, P, P, P, P, U, U, P],
    "n2m_s0_encode_points_codes": [PP, P, P, P, U, P, P, P, P, P],
    "n2m_s0_fwd_fused_codes": [PP, P, P, U, P, P, P, P, P, P, P, P, P, P, P],
    "n2m_s0_render_rounds_codes": [PP, P, P, P, U, P, U, P, P, P, P, P, P, P, U, P, P, P, P, P, P, P, P],
    "n2m_s0_mlp_bwd_codes": [PP, P, P, P, U, P, P, P, P, P, U, U, P],
    "n2m_s0_code_grad": [PP, P, P, U, P, P, P, P, P, U, U, P],
    "n2m_s0_code_grad_row": [PP, P, U, P, P, P, P],
    "n2m_s0_pack_code_weights": [P, U, P, P],
    "n2m_s0_adam_codes_head": [P, U, P, P],
    "n2m_s0_adam_codes": [P, P, P, P, U, U, P, P, F, P],
    "n2m_s0_codes_ema_update": [P, P, U, F, P],
    "n2m_s0_codes_ema_swap": [P, P, U, U, P, P],
})
_lib.lib.n2m_s0_wpack_bytes.restype = c_uint32
_lib.lib.n2m_s0_mlp_param_count.restype = c_uint32

# flat MLP parameter vector: (reference parameter name, shape)
MLP_LAYOUT = [
    ("sigma_net.net.0.weight", (32, 19)), ("sigma_net.net.1.weight", (1, 32)),
    ("color_net.net.0.weight", (64, 35)), ("color_net.net.1.weight", (64, 64)), ("color_net.net.2.weight", (6, 64)),
    ("specular_net.net.0.weight", (32, 6)), ("specular_net.net.1.weight", (3, 32)),
]
# per-image appearance codes (include/n2m_b200_fused.h "Per-image appearance codes"): widest code the 64-column tile image has room for
MAX_IND_DIM = 10


class Stage0Config:
    """The operator arguments the reference passes down from `opt`."""

    def __init__(self, bound=1.0, contract=False, dt_gamma=0.0, max_steps=1024, grid_size=128, min_near=0.05,
                 T_thresh=1e-4, num_levels=16, base_resolution=16, log2_hashmap_size=19, lambda_mask=0.1,
                 lambda_specular=1e-5, lambda_tv=1e-8, lambda_entropy=0.0, lr=1e-2, eps=1e-15, max_samples=None, num_rays=4096,
                 loss_scale=65536.0, adaptive_num_rays=False, num_points=2 ** 18, max_rays=None, ind_dim=0, ind_num=500):
        self.real_bound = float(bound)
        self.contract = bool(contract)
        self.bound = 2.0 if contract else float(bound)          # renderer.py:74-80
        self.cascade = 1 + math.ceil(math.log2(self.bound))     # renderer.py:82
        self.dt_gamma, self.max_steps, self.grid_size, self.min_near = float(dt_gamma), int(max_steps), int(grid_size), float(min_near)
        self.T_thresh = float(T_thresh)
        self.num_levels, self.base_resolution, self.log2_hashmap_size = int(num_levels), int(base_resolution), int(log2_hashmap_size)
        desired = 2048 * self.bound                             # network.py:66,71
        self.per_level_scale = float(np.exp2(np.log2(desired / base_resolution) / (num_levels - 1)))
        self.lambda_mask, self.lambda_specular, self.lambda_tv = float(lambda_mask), float(lambda_specular), float(lambda_tv)
        self.lambda_entropy = float(lambda_entropy)          # main.py --lambda_entropy (garden recipe: 1e-3)
        self.lr, self.eps = float(lr), float(eps)
        self.num_rays = int(num_rays)
        # --adaptive_num_rays (main.py:68-69,129-135): after every step the next batch takes round(num_points / M * n) rays, decided
        # on the device by the march (include/n2m_b200_fused.h ray_ctl).  The first step takes num_rays; the per-ray buffers are max_rays
        # wide and every step() is handed max_rays rows, of which the trainer uses the first n.
        self.adaptive_num_rays = bool(adaptive_num_rays)
        self.num_points = int(num_points)
        self.max_rays = (int(max_rays) if max_rays else 4 * self.num_rays) if self.adaptive_num_rays else self.num_rays
        if self.adaptive_num_rays and self.num_points <= 0:
            raise ValueError(f"num_points must be positive, got {self.num_points}")
        if self.adaptive_num_rays and self.max_rays < self.num_rays:
            raise ValueError(f"max_rays ({self.max_rays}) must be at least num_rays ({self.num_rays})")
        # sample capacity of the per-step buffers.  The reference allocates exactly M samples per step (raymarching.py:232-238)
        # and never drops a ray; here a step whose M exceeds the capacity renders the rays that do not fit (the LAST rays of the
        # batch) as background without gradient -- counted on the device (counters[13], [14]); Stage0Trainer.check_capacity()
        # reports / grows the slab, training loops call it at every density-grid update.
        self.max_samples = int(max_samples) if max_samples else self.num_rays * 128
        self.max_samples = (self.max_samples + 127) // 128 * 128
        self.loss_scale = float(loss_scale)
        # --ind_dim / --ind_num (main.py:94-95): a learned code per training image, appended to color_net's input
        # (renderer.py:97-104, network.py:72,159-166).  The code columns share the colour net's 64-column first GEMM with the features,
        # so at most MAX_IND_DIM of them fit.
        self.ind_dim, self.ind_num = int(ind_dim), int(ind_num)
        if not 0 <= self.ind_dim <= MAX_IND_DIM:
            raise ValueError(f"ind_dim must be in [0, {MAX_IND_DIM}], got {self.ind_dim}")
        if self.ind_num < 1:
            raise ValueError(f"ind_num must be at least 1, got {self.ind_num}")


class _Slot:
    """Buffers tied to one batch of rays: inputs, ray (offset, count) table, sample records."""

    def __init__(self, N, Mc, max_steps, dev):
        self.rays_o = torch.zeros(N, 3, device=dev); self.rays_d = torch.zeros(N, 3, device=dev)
        self.gt = torch.zeros(N, 4, device=dev); self.bg = torch.zeros(N, 3, device=dev)
        self.noises = torch.zeros(N, device=dev)
        self.rays = torch.zeros(N, 2, dtype=torch.int32, device=dev)
        self.counters = torch.zeros(17, dtype=torch.int32, device=dev)    # include/n2m_b200_fused.h: [4..12] part boundaries, [16] n
        self.tbuf = torch.empty(N * max_steps * 2, device=dev)
        self.recs = torch.zeros(Mc, 4, device=dev)
        self.cam_nf = torch.zeros(N, 2, device=dev)                      # per-ray (near, far) clamp, renderer.py:689-691
        self.ray_img = torch.zeros(N, dtype=torch.int32, device=dev)     # image index of every ray (appearance codes only)
        self.has_alpha = True

    def load_index(self, index):
        """The batch's image indices (data['index']): an int for the whole batch, or an int32 [N] tensor, one per ray."""
        if isinstance(index, int):
            self.ray_img.fill_(index)
        else:
            self.ray_img.copy_(index, non_blocking=True)

    def load(self, rays_o, rays_d, gt, bg, noises=None, cam_near_far=None):
        N = self.rays_o.shape[0]
        if gt.shape[-1] == 3:
            self.gt.view(-1)[: N * 3].view(N, 3).copy_(gt, non_blocking=True)       # packed [N,3] at the front
            self.has_alpha = False
        else:
            self.gt.copy_(gt, non_blocking=True)
            self.has_alpha = True
        self.rays_o.copy_(rays_o, non_blocking=True); self.rays_d.copy_(rays_d, non_blocking=True)
        self.bg.copy_(bg, non_blocking=True)
        if noises is not None:
            self.noises.copy_(noises, non_blocking=True)
        if cam_near_far is not None:
            self.cam_nf.copy_(cam_near_far, non_blocking=True)


class Stage0Trainer:
    # adaptive ray count (Stage0Config.adaptive_num_rays): the device-resident control block the march reads and rewrites
    adaptive = False
    ray_ctl = None
    # per-image appearance codes (Stage0Config.ind_dim > 0): the parameter block `ind` [64 D code columns of color_net.0 | ind_num D codes]
    # (include/n2m_b200_fused.h "Per-image appearance codes") with its gradient g_ind and Adam moments m_ind / v_ind
    ind_dim = 0
    ind_num = 0
    _ray_ctl_undo = None        # ray_ctl as it was before the side-stream march of a prefetched batch (see drop_prefetch)

    def __init__(self, cfg: Stage0Config, device="cuda", seed=0):
        self.cfg = cfg
        self.device = torch.device(device)
        dev = self.device
        call("n2m_s0_init")
        c = cfg
        offs = level_offsets(3, c.num_levels, c.per_level_scale, c.base_resolution, c.log2_hashmap_size, False)
        self.offsets = torch.from_numpy(offs).to(dev)
        self._offsets_host = [int(v) for v in offs]
        self.rows = int(offs[-1])
        R = self.rows
        self.n_mlp = int(_lib.lib.n2m_s0_mlp_param_count())
        # ---- model state (native layout) ----
        self.table = torch.zeros(R, 2, dtype=torch.float32, device=dev)          # 8-byte entries {f32, half2}
        self.color_master = torch.zeros(R, 2, dtype=torch.float32, device=dev)
        self.gtables = [torch.zeros(R, 4, dtype=torch.float32, device=dev), torch.zeros(R, 4, dtype=torch.float32, device=dev)]
        self.parity = 0                     # which gradient table the current step accumulates into (see defer_zero / PeerAdam)
        self.m_table = torch.zeros(R * 3, dtype=torch.float32, device=dev)
        self.v_table = torch.zeros(R * 3, dtype=torch.float32, device=dev)
        self.mlp = torch.zeros(self.n_mlp, dtype=torch.float32, device=dev)
        self.g_mlps = [torch.zeros_like(self.mlp)]
        self.m_mlp = torch.zeros_like(self.mlp); self.v_mlp = torch.zeros_like(self.mlp)
        self.wpack = torch.zeros(int(_lib.lib.n2m_s0_wpack_bytes()), dtype=torch.uint8, device=dev)
        if c.ind_dim:
            self.ind_dim, self.ind_num = c.ind_dim, c.ind_num
            self.ind = torch.zeros((64 + c.ind_num) * c.ind_dim, dtype=torch.float32, device=dev)
            self.g_ind = torch.zeros_like(self.ind)
            self.m_ind = torch.zeros_like(self.ind); self.v_ind = torch.zeros_like(self.ind)
        self.opt_state = torch.zeros(8, dtype=torch.float32, device=dev)
        self.opt_state[0] = c.loss_scale
        self.opt_state[4] = c.lr
        # ---- scene state ----
        self.density_grid = torch.zeros(c.cascade, c.grid_size ** 3, device=dev)
        self.density_bitfield = torch.zeros(c.cascade * c.grid_size ** 3 // 8, dtype=torch.uint8, device=dev)
        b = c.real_bound
        self.aabb = torch.tensor([-b, -b, -b, b, b, b], dtype=torch.float32, device=dev)
        # ---- per-batch buffers: two slots, so the (parameter-independent) march of batch i+1 can run on a side
        # stream while batch i is in encode / MLP / scatter / Adam ----
        N, Mc = c.max_rays, c.max_samples
        self.N, self.Mcap = N, Mc
        if c.adaptive_num_rays:
            self.adaptive = True
            self.ray_ctl = torch.tensor([c.num_rays, 0, 0, 0], dtype=torch.int32, device=dev)     # include/n2m_b200_fused.h ray_ctl
            self._ray_ctl_undo = torch.zeros_like(self.ray_ctl)
        self.slots = [_Slot(N, Mc, c.max_steps, dev) for _ in range(2)]
        self.cur = 0
        self._prefetched = None                 # slot index holding an already staged + marched batch
        self._side = None
        self._ev_march = [None, None]
        self._ev_done = [None, None]
        # ---- per-step buffers shared by both slots (consumed within the step) ----
        self.enc_tiles = torch.zeros(Mc * 64, dtype=torch.float16, device=dev)
        self.denc_tiles = torch.zeros(Mc * 64, dtype=torch.float16, device=dev)
        self.out = torch.zeros(Mc, 4, device=dev)
        self.dout = torch.zeros(Mc, 4, device=dev)
        self.image = torch.zeros(N, 3, device=dev); self.weights_sum = torch.zeros(N, device=dev); self.depth = torch.zeros(N, device=dev)
        self.loss_acc = torch.zeros(4, device=dev)          # [0] rgb(+mask) loss, [1] sum |spec|^2
        # explicit-point evaluation (density-grid update, density volume): positions and their count
        self._pts = torch.zeros(Mc, 3, device=dev)
        self._pcount = torch.zeros(4, dtype=torch.int32, device=dev)
        self.params = S0Params()
        self._fill_params(shading_full=True, gt_has_alpha=True)
        self.fused_fwd = False              # True: gather + MLP forward as one warp-specialised launch (whole batch: needs nparts == 1)
        self.use_cam_near_far = False       # clamp (near, far) with the per-ray values in the slot's cam_nf (--enable_cam_near_far)
        self._tv_stream = None              # the TV launch runs on its own stream, overlapped with the MLP kernels
        self.nparts = 1                     # ray-range parts run as concurrent chains on forked streams (1, 2, 4 or 8)
        self._part_streams = []
        self._adam_stream = None
        self.tv_fallback_points = 1000000   # GridEncoder.grad_total_variation's random-point fallback (grid.py:172,181-183)
        # EMA of the parameters (Trainer(ema_decay=0.95), main.py:241): shadow buffers are allocated by enable_ema()
        self.ema_decay = None
        self.ema_num_updates = 0
        self._ema = None
        self._ema_swapped = False
        self._color_master_provider = None  # PeerAdam: the fp32 colour masters live in per-rank slices (parallel.py)
        # single GPU: the gradient table of step i is zeroed on a side stream under the optimizer of step i+1 (which accumulates into
        # the other parity) instead of by the optimizer kernel: 16 of its 112 bytes per row leave the optimizer's sweep
        self.defer_zero = True
        self._zero_stream = None
        # step(next_batch=...): where the next batch's march (issue-bound, a few MB of traffic) is released on the side stream --
        # "optimizer": underneath the optimizer stage (HBM-bound table sweep, or the NVLink-bound data-parallel exchange), on a
        # high-priority stream so that its blocks are dispatched ahead of the sweep's; "start": underneath the forward pass
        self.prefetch_at = "optimizer"
        self.global_step = 0
        self._graphs = {}
        self.reset_parameters(seed)

    # the gradient buffers of the CURRENT parity under their historical names
    @property
    def gtable(self):
        return self.gtables[self.parity]

    @gtable.setter
    def gtable(self, t):
        self.gtables[self.parity] = t

    @property
    def g_mlp(self):
        return self.g_mlps[min(self.parity, len(self.g_mlps) - 1)]

    @g_mlp.setter
    def g_mlp(self, t):
        self.g_mlps[min(self.parity, len(self.g_mlps) - 1)] = t

    @property
    def fused_bwd(self):
        """Always False: the per-sample backward is two launches, k_mlp_bwd (two tiles in flight per SM beside a weight-gradient
        warpgroup) and then the hash-grid scatter k_s0_encode_bwd.  The one-launch MLP-backward + scatter kernel was slower on every
        workload on the H100 and has been removed; setting the flag to a true value raises ValueError, a false value is accepted."""
        return False

    @fused_bwd.setter
    def fused_bwd(self, on):
        if on:
            raise ValueError("fused_bwd: the fused MLP-backward + scatter kernel was removed; the backward is k_mlp_bwd followed by "
                             "k_s0_encode_bwd")

    # current slot's buffers under their historical names
    rays_o = property(lambda self: self.slots[self.cur].rays_o)
    rays_d = property(lambda self: self.slots[self.cur].rays_d)
    gt = property(lambda self: self.slots[self.cur].gt)
    bg = property(lambda self: self.slots[self.cur].bg)
    noises = property(lambda self: self.slots[self.cur].noises)
    rays = property(lambda self: self.slots[self.cur].rays)
    counters = property(lambda self: self.slots[self.cur].counters)
    tbuf = property(lambda self: self.slots[self.cur].tbuf)
    recs = property(lambda self: self.slots[self.cur].recs)

    # -------------------------------------------------------------------------------------------
    def _fill_params(self, shading_full, gt_has_alpha):
        c, p = self.cfg, self.params
        p.bound, p.grid_bound = c.real_bound, c.bound
        p.inv_2gb = float(np.float32(1.0) / np.float32(2.0 * c.bound))
        p.dt_gamma, p.min_near, p.T_thresh = c.dt_gamma, c.min_near, c.T_thresh
        p.S = float(np.float32(np.log2(c.per_level_scale)))
        p.lambda_mask, p.lambda_specular, p.lambda_tv = c.lambda_mask, c.lambda_specular, c.lambda_tv
        p.lambda_entropy = c.lambda_entropy
        p.contract, p.max_steps, p.cascades, p.grid_size = int(c.contract), c.max_steps, c.cascade, c.grid_size
        p.num_levels, p.base_res = c.num_levels, c.base_resolution
        p.shading_full, p.gt_has_alpha = int(shading_full), int(gt_has_alpha)
        p.ind_dim = self.ind_dim

    def params_with(self, **fields):
        """A copy of `params` with `fields` overridden, e.g. params_with(shading_full=0) for sigma-only evaluation."""
        p = S0Params()
        ctypes.memmove(ctypes.byref(p), ctypes.byref(self.params), ctypes.sizeof(S0Params))
        for name, value in fields.items():
            setattr(p, name, value)
        return p

    def reset_parameters(self, seed=0):
        """Reference initialisation: embeddings U(-1e-4, 1e-4) (grid.py:144-146), nn.Linear default
        (kaiming_uniform(a=sqrt(5)) == U(-1/sqrt(fan_in), 1/sqrt(fan_in)))."""
        g = torch.Generator().manual_seed(seed)
        state = {"encoder.embeddings": torch.rand(self.rows, 1, generator=g) * 2e-4 - 1e-4,
                 "encoder_color.embeddings": torch.rand(self.rows, 2, generator=g) * 2e-4 - 1e-4}
        for name, (o, i) in MLP_LAYOUT:
            if name == "color_net.net.0.weight":
                i += self.ind_dim                   # the code columns are inputs of the same nn.Linear (network.py:72)
            k = 1.0 / math.sqrt(i)
            state[name] = (torch.rand(o, i, generator=g) * 2 - 1) * k
        if self.ind_dim:
            state["individual_codes"] = torch.randn(self.ind_num, self.ind_dim, generator=g) * 0.1     # renderer.py:101-102
        self.load_reference_state(state)

    def load_reference_state(self, state):
        dev = self.device
        ed = state["encoder.embeddings"].to(dev, torch.float32).contiguous()
        ec = state["encoder_color.embeddings"].to(dev, torch.float32).contiguous()
        assert ed.shape == (self.rows, 1) and ec.shape == (self.rows, 2)
        call("n2m_s0_pack_tables", ptr(ed), ptr(ec), self.rows, ptr(self.table), ptr(self.color_master), stream())
        D = self.ind_dim
        c0 = state["color_net.net.0.weight"]
        if tuple(c0.shape) != (64, 35 + D):
            raise ValueError(f"color_net.net.0.weight has shape {tuple(c0.shape)}, the model (ind_dim = {D}) expects {(64, 35 + D)}")
        flat = torch.cat([(state[n][:, :35] if n == "color_net.net.0.weight" else state[n]).to(dev, torch.float32).reshape(-1)
                          for n, _ in MLP_LAYOUT])
        assert flat.numel() == self.n_mlp
        self.mlp.copy_(flat)
        call("n2m_s0_pack_weights", ptr(self.mlp), ptr(self.wpack), stream())
        if D:
            codes = state["individual_codes"]
            if tuple(codes.shape) != (self.ind_num, D):
                raise ValueError(f"individual_codes has shape {tuple(codes.shape)}, the model expects {(self.ind_num, D)}")
            self.ind.copy_(torch.cat([c0[:, 35:].to(dev, torch.float32).reshape(-1), codes.to(dev, torch.float32).reshape(-1)]))
            call("n2m_s0_pack_code_weights", ptr(self.ind), D, ptr(self.wpack), stream())
        if "density_bitfield" in state:
            self.density_bitfield.copy_(state["density_bitfield"].to(dev))
        if "density_grid" in state:
            self.density_grid.copy_(state["density_grid"].to(dev))
        torch.cuda.synchronize()

    def export_reference_state(self):
        ed = torch.empty(self.rows, 1, device=self.device); ec = torch.empty(self.rows, 2, device=self.device)
        # under PeerAdam the fp32 colour masters are sharded over the ranks: gather them (a collective -- every rank must call)
        cm = self.color_master if self._color_master_provider is None else self._color_master_provider().contiguous()
        call("n2m_s0_unpack_tables", ptr(self.table), ptr(cm), self.rows, ptr(ed), ptr(ec), stream())
        # the complete stage-0 `NeRFNetwork.state_dict()` key set (renderer.py:92-117, grid.py:135-140, network.py:66-75): loads
        # into the reference model with strict=True (no individual codes / SDF variance in the default recipes)
        state = {"encoder.embeddings": ed, "encoder_color.embeddings": ec,
                 "encoder.offsets": self.offsets.clone(), "encoder_color.offsets": self.offsets.clone(),
                 "aabb_train": self.aabb.clone(), "aabb_infer": self.aabb.clone(),
                 "density_grid": self.density_grid.clone(), "density_bitfield": self.density_bitfield.clone()}
        o = 0
        for name, shp in MLP_LAYOUT:
            n = shp[0] * shp[1]
            state[name] = self.mlp[o:o + n].view(shp).clone(); o += n
        if self.ind_dim:
            self._with_codes(state, self.ind)
        return state

    def _with_codes(self, tensors, ind):
        """Reference layout of an `ind` block (parameters, gradients or EMA shadow) merged into `tensors`: the code columns appended to
        color_net.net.0.weight ([64, 35 + D]) and individual_codes [ind_num, D] (renderer.py:102)."""
        D = self.ind_dim
        key = "color_net.net.0.weight"
        tensors[key] = torch.cat([tensors[key], ind[:64 * D].view(64, D)], dim=1)
        tensors["individual_codes"] = ind[64 * D:].view(self.ind_num, D).clone()
        return tensors

    def _codes_table(self):
        """Device address of the code table [ind_num, D] (row 0: the code the reference evaluates with, renderer.py:702-703)."""
        return self.ind.data_ptr() + 4 * 64 * self.ind_dim

    def save_reference_checkpoint(self, path, epoch=0, stats=None, best=False, full=False):
        """A checkpoint in the schema `Trainer.save_checkpoint` writes and `Trainer.load_checkpoint` reads (nerf/utils.py:1345-1381,
        1407-1473): epoch / global_step / stats / stage / mean_density / model (+ 'ema' when `full`).  `best=True` stores the EMA
        parameters as the model, as the reference does for its best checkpoint (utils.py:1389-1401)."""
        mean = getattr(self, "mean_density", None)
        state = {"epoch": int(epoch), "global_step": int(self.global_step), "stage": 0,
                 "stats": stats or {"loss": [], "valid_loss": [], "results": [], "checkpoints": [], "best_result": None},
                 "mean_density": float(mean.item()) if mean is not None else 0.0}
        if full and self._ema is not None:
            state["ema"] = {k: ([t.cpu() for t in v] if isinstance(v, list) else v) for k, v in self.ema_state_dict().items()}
        if best:
            self.ema_apply()
        state["model"] = {k: v.cpu() for k, v in self.export_reference_state().items()}
        if best:
            self.ema_restore()
        torch.save(state, path)
        return state

    # -------------------------------------------------------------------------------------------
    # EMA (torch_ema.ExponentialMovingAverage as the reference's Trainer uses it)
    # -------------------------------------------------------------------------------------------
    def enable_ema(self, decay=0.95):
        """Trainer(ema_decay=0.95) (main.py:241; utils.py:544-545): shadow parameters start as a copy of the parameters."""
        if self._color_master_provider is not None:
            raise NotImplementedError("EMA with the sharded PeerAdam optimizer: use GradSync, or keep the EMA on one rank")
        self.ema_decay, self.ema_num_updates, self._ema_swapped = float(decay), 0, False
        st = self.export_reference_state()
        self._ema = {"d": st["encoder.embeddings"].reshape(-1).contiguous(), "c": st["encoder_color.embeddings"].contiguous(),
                     "mlp": self.mlp.clone()}
        if self.ind_dim:
            self._ema["ind"] = self.ind.clone()

    def ema_update(self):
        """`self.ema.update()` -- the reference calls it once per EPOCH (utils.py:1213-1214), not per step.  torch_ema's warm-up:
        decay = min(decay, (1 + num_updates) / (10 + num_updates)) with num_updates incremented first."""
        assert self._ema is not None and not self._ema_swapped
        self.ema_num_updates += 1
        decay = min(self.ema_decay, (1 + self.ema_num_updates) / (10 + self.ema_num_updates))
        e = self._ema
        call("n2m_s0_ema_update", ptr(self.table), ptr(self.color_master), ptr(self.mlp), ptr(e["d"]), ptr(e["c"]), ptr(e["mlp"]),
             self.rows, 1.0 - decay, stream())
        if self.ind_dim:
            call("n2m_s0_codes_ema_update", ptr(self.ind), ptr(e["ind"]), self.ind.numel(), 1.0 - decay, stream())

    def _ema_swap(self):
        e = self._ema
        call("n2m_s0_ema_swap", ptr(self.table), ptr(self.color_master), ptr(self.mlp), ptr(e["d"]), ptr(e["c"]), ptr(e["mlp"]),
             self.rows, ptr(self.wpack), stream())
        if self.ind_dim:        # after the swap above, whose repack zeroes the code columns
            call("n2m_s0_codes_ema_swap", ptr(self.ind), ptr(e["ind"]), self.ind_dim, self.ind_num, ptr(self.wpack), stream())
        self._ema_swapped = not self._ema_swapped

    def ema_apply(self):
        """`ema.store(); ema.copy_to()` (utils.py:1250-1252): evaluate / export with the averaged parameters.  In place: the live
        parameters are parked in the shadow buffers until ema_restore()."""
        if self._ema is not None and not self._ema_swapped:
            self._ema_swap()

    def ema_restore(self):
        """`ema.restore()` (utils.py:1340-1341)."""
        if self._ema is not None and self._ema_swapped:
            self._ema_swap()

    def ema_state_dict(self):
        """torch_ema's state_dict() for a 'full' checkpoint (utils.py:1364-1365): shadow parameters in model.parameters() order
        (encoder, sigma_net, encoder_color, color_net, specular_net: nerf/network.py:66-75)."""
        assert self._ema is not None and not self._ema_swapped
        e = self._ema
        mlps, o = {}, 0
        for name, shp in MLP_LAYOUT:
            n = shp[0] * shp[1]
            mlps[name] = e["mlp"][o:o + n].view(shp).clone(); o += n
        order = ["encoder.embeddings", "sigma_net.net.0.weight", "sigma_net.net.1.weight", "encoder_color.embeddings",
                 "color_net.net.0.weight", "color_net.net.1.weight", "color_net.net.2.weight",
                 "specular_net.net.0.weight", "specular_net.net.1.weight"]
        tensors = {"encoder.embeddings": e["d"].view(-1, 1).clone(), "encoder_color.embeddings": e["c"].clone(), **mlps}
        if self.ind_dim:
            # individual_codes is a parameter of the renderer itself, registered before the network's modules (renderer.py:102)
            self._with_codes(tensors, e["ind"])
            order = ["individual_codes"] + order
        return {"decay": self.ema_decay, "num_updates": self.ema_num_updates, "shadow_params": [tensors[k] for k in order],
                "collected_params": None}

    def export_reference_grads(self):
        """Current (un-scaled) gradients in reference layout -- for parity tests; call before the optimizer."""
        gd = torch.empty(self.rows, 1, device=self.device); gc = torch.empty(self.rows, 2, device=self.device)
        call("n2m_s0_unpack_grads", ptr(self.gtable), self.rows, ptr(self.opt_state), ptr(gd), ptr(gc), stream())
        grads = {"encoder.embeddings": gd, "encoder_color.embeddings": gc}
        g = self.g_mlp / self.opt_state[0]
        o = 0
        for name, shp in MLP_LAYOUT:
            n = shp[0] * shp[1]
            grads[name] = g[o:o + n].view(shp).clone(); o += n
        if self.ind_dim:
            self._with_codes(grads, self.g_ind / self.opt_state[0])
        return grads

    def mark_untrained_grid(self, poses, intrinsics, cam_near_far=None):
        """NeRFRenderer.mark_untrained_grid (renderer.py:985-1071): density-grid cells outside every training camera's frustum (or
        outside the AABB) become -1 and are never updated again.  poses [B,4,4] camera-to-world, intrinsics [4] or [B,4]
        (fx, fy, cx, cy), cam_near_far [B,2] optional.  Returns the number of marked cells as a device tensor (no host sync)."""
        dev = self.device
        poses = torch.as_tensor(poses, dtype=torch.float32).to(dev).contiguous()
        intr = torch.as_tensor(intrinsics, dtype=torch.float32).to(dev).reshape(-1, 4).contiguous()
        near = None if cam_near_far is None else torch.as_tensor(cam_near_far, dtype=torch.float32).to(dev)[:, 0].contiguous()
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        c = self.cfg
        call("n2m_mark_untrained_grid", ptr(poses), poses.shape[0], ptr(intr), intr.shape[0], ptr(near), c.min_near, ptr(self.aabb),
             c.bound, c.cascade, c.grid_size, ptr(self.density_grid), ptr(count), stream())
        return count

    def set_occupancy(self, density_bitfield, density_grid=None):
        self.density_bitfield.copy_(density_bitfield.to(self.device))
        if density_grid is not None:
            self.density_grid.copy_(density_grid.to(self.device))

    # -------------------------------------------------------------------------------------------
    # the stages (all asynchronous on the current stream)
    # -------------------------------------------------------------------------------------------
    def _pp(self):
        return ctypes.byref(self.params)

    def march(self, all_rays=False):
        """`all_rays`: march every row of the buffers whatever the adaptive ray count (evaluation)."""
        adaptive = self.adaptive and not all_rays
        call("n2m_s0_march", self._pp(), ptr(self.rays_o), ptr(self.rays_d), ptr(self.aabb),
             ptr(self.slots[self.cur].cam_nf) if self.use_cam_near_far else None, ptr(self.density_bitfield),
             ptr(self.noises), self.N, ptr(self.rays), ptr(self.counters), ptr(self.tbuf), ptr(self.recs), self.Mcap,
             ptr(self.ray_ctl) if adaptive else None, self.cfg.num_points if adaptive else 0, stream())

    def encode_fwd(self, part=0, nparts=1):
        if self.ind_dim:
            call("n2m_s0_encode_fwd_codes", self._pp(), ptr(self.recs), ptr(self.counters), self.Mcap, ptr(self.rays_o), ptr(self.rays_d),
                 ptr(self.table), ptr(self.offsets), self._codes_table(), ptr(self.slots[self.cur].ray_img), ptr(self.enc_tiles), part,
                 nparts, stream())
            return
        call("n2m_s0_encode_fwd", self._pp(), ptr(self.recs), ptr(self.counters), self.Mcap, ptr(self.rays_o), ptr(self.rays_d),
             ptr(self.table), ptr(self.offsets), ptr(self.enc_tiles), part, nparts, stream())

    def encode_points(self, pp, pts, dirs, counters, cap, enc_tiles, code_row=0):
        """The hash-grid gather of explicit points pts [cap,3] (dirs nullable; counters[1] points) into tile images with parameter block
        `pp`; with appearance codes every point reads code row `code_row` (stage 1: the view's image; evaluation and the bake: 0)."""
        if self.ind_dim:
            call("n2m_s0_encode_points_codes", pp, ptr(pts), ptr(dirs), ptr(counters), cap, ptr(self.table), ptr(self.offsets),
                 self.ind.data_ptr() + 4 * self.ind_dim * (64 + int(code_row)), ptr(enc_tiles), stream())
        else:
            call("n2m_s0_encode_points", pp, ptr(pts), ptr(dirs), ptr(counters), cap, ptr(self.table), ptr(self.offsets), ptr(enc_tiles),
                 stream())

    def mlp_fwd(self, part=0, nparts=1):
        call("n2m_s0_mlp_fwd", self._pp(), ptr(self.enc_tiles), ptr(self.counters), self.Mcap, ptr(self.wpack), ptr(self.out),
             self.loss_acc.data_ptr() + 4, part, nparts, stream())

    def composite_loss(self, part=0, nparts=1, all_rays=False):
        active = self.counters.data_ptr() + 4 * 16 if self.adaptive and not all_rays else None      # counters[16]: the batch's n
        call("n2m_s0_composite_loss", self._pp(), ptr(self.out), ptr(self.recs), ptr(self.rays), ptr(self.counters), self.N, self.Mcap,
             ptr(self.gt), ptr(self.bg), ptr(self.opt_state), ptr(self.dout), ptr(self.image), ptr(self.weights_sum), ptr(self.depth),
             ptr(self.loss_acc), active, part, nparts, stream())

    def mlp_bwd(self, part=0, nparts=1):
        if self.ind_dim:
            call("n2m_s0_mlp_bwd_codes", self._pp(), ptr(self.enc_tiles), ptr(self.dout), ptr(self.counters), self.Mcap, ptr(self.wpack),
                 ptr(self.denc_tiles), ptr(self.g_mlp), ptr(self.g_ind), ptr(self.opt_state), part, nparts, stream())
            self.code_grad(part, nparts)
            return
        call("n2m_s0_mlp_bwd", self._pp(), ptr(self.enc_tiles), ptr(self.dout), ptr(self.counters), self.Mcap, ptr(self.wpack),
             ptr(self.denc_tiles), ptr(self.g_mlp), ptr(self.opt_state), part, nparts, stream())

    def code_grad(self, part=0, nparts=1, all_rays=False):
        """Gradient of the appearance codes: the code columns of denc_tiles summed per ray into its image's code row."""
        active = self.counters.data_ptr() + 4 * 16 if self.adaptive and not all_rays else None      # counters[16]: the batch's n
        call("n2m_s0_code_grad", self._pp(), ptr(self.rays), ptr(self.counters), self.N, ptr(self.denc_tiles),
             ptr(self.slots[self.cur].ray_img), self.g_ind.data_ptr() + 4 * 64 * self.ind_dim, ptr(self.opt_state), active, part, nparts,
             stream())

    def fwd_fused(self):
        if self.ind_dim:
            call("n2m_s0_fwd_fused_codes", self._pp(), ptr(self.recs), ptr(self.counters), self.Mcap, ptr(self.rays_o), ptr(self.rays_d),
                 ptr(self.table), ptr(self.offsets), self._codes_table(), ptr(self.slots[self.cur].ray_img), ptr(self.wpack),
                 ptr(self.enc_tiles), ptr(self.out), self.loss_acc.data_ptr() + 4, stream())
            return
        call("n2m_s0_fwd_fused", self._pp(), ptr(self.recs), ptr(self.counters), self.Mcap, ptr(self.rays_o), ptr(self.rays_d),
             ptr(self.table), ptr(self.offsets), ptr(self.wpack), ptr(self.enc_tiles), ptr(self.out), self.loss_acc.data_ptr() + 4, stream())

    def encode_bwd(self, part=0, nparts=1):
        call("n2m_s0_encode_bwd", self._pp(), ptr(self.recs), ptr(self.counters), self.Mcap, ptr(self.rays_o), ptr(self.rays_d),
             ptr(self.denc_tiles), ptr(self.table), ptr(self.offsets), ptr(self.gtables[self.parity]), ptr(self.opt_state),
             part, nparts, stream())

    def tv(self):
        """TV gradient of the density table at the step's samples (utils.py:801-823) + the random-point fallback of the TV calls that
        got no sample (grid.py:181-183; exits at once when every group is populated)"""
        call("n2m_s0_tv", self._pp(), ptr(self.recs), ptr(self.counters), self.Mcap, ptr(self.rays_o), ptr(self.rays_d),
             ptr(self.table), ptr(self.offsets), ptr(self.gtables[self.parity]), ptr(self.opt_state), stream())
        self.tv_random()

    def tv_random(self, dump=None):
        if self.cfg.lambda_tv > 0 and self.tv_fallback_points > 0:
            call("n2m_s0_tv_random", self._pp(), ptr(self.counters), ptr(self.table), ptr(self.offsets), ptr(self.gtables[self.parity]),
                 ptr(self.opt_state), int(self.tv_fallback_points), ptr(dump), stream())

    def adam(self, keep_grads=False, between=None):
        """Optimizer stage: head -> [table rows || MLP parameters + weight repack] -> GradScaler update.  The MLP branch
        (three tiny launches) runs on a forked stream underneath the 0.7 GB table sweep.  `keep_grads`: do not zero the gradient
        table (the caller zeroes it off the critical path, see `defer_zero`).  `between`: callable run after the parameter updates and
        before the GradScaler update -- further parameter groups of the same optimizer step (stage 1: the vertex offsets)."""
        main = torch.cuda.current_stream()
        if self.ind_dim:
            call("n2m_s0_adam_codes_head", ptr(self.g_ind), self.g_ind.numel(), ptr(self.opt_state), stream())
        call("n2m_s0_adam_head", ptr(self.g_mlp), ptr(self.opt_state), stream())
        if self._adam_stream is None:
            self._adam_stream = torch.cuda.Stream(device=self.device)
        side = self._adam_stream
        side.wait_stream(main)
        with torch.cuda.stream(side):
            call("n2m_s0_adam_mlp", ptr(self.mlp), ptr(self.g_mlp), ptr(self.m_mlp), ptr(self.v_mlp), ptr(self.wpack),
                 ptr(self.opt_state), self.cfg.eps, stream())
            if self.ind_dim:        # after adam_mlp, whose weight repack zeroes the code columns
                call("n2m_s0_adam_codes", ptr(self.ind), ptr(self.g_ind), ptr(self.m_ind), ptr(self.v_ind), self.ind_dim, self.ind_num,
                     ptr(self.wpack), ptr(self.opt_state), self.cfg.eps, stream())
        call("n2m_s0_adam_tables_keep" if keep_grads else "n2m_s0_adam_tables", ptr(self.table), ptr(self.color_master), ptr(self.gtable),
             ptr(self.m_table), ptr(self.v_table), self.rows, ptr(self.opt_state), self.cfg.eps, stream())
        if between is not None:
            between()
        main.wait_stream(side)
        call("n2m_s0_adam_post", ptr(self.opt_state), stream())

    def forward_backward(self):
        """march -> encode (|| TV) -> MLP -> composite+loss -> MLP backward -> scatter; gradients stay in
        gtable / g_mlp (loss-scaled)."""
        self.march()
        self._compute()

    def _compute(self):
        """Everything after the march for the current slot.

        * `nparts` > 1: the batch is cut into ray-range parts (include/n2m_b200_fused.h "Ray-range parts"); the chain
          gather -> MLP -> composite -> MLP backward -> scatter of every part runs on its own stream, so the
          latency-bound tensor-core MLP kernels of one part share the SMs with the memory-bound gather / scatter
          kernels of another.
        * with lambda_tv > 0 the TV-gradient kernel (memory bound, independent of the MLPs) runs on a forked stream as well.
        All forks are joined before returning (and they are graph-capturable: fork/join by events only)."""
        self.loss_acc.zero_()
        main = torch.cuda.current_stream()
        P_ = int(self.nparts)
        fork_tv = self.cfg.lambda_tv > 0

        def launch_tv():
            if fork_tv:
                if self._tv_stream is None:
                    self._tv_stream = torch.cuda.Stream(device=self.device)
                self._tv_stream.wait_stream(main)
                with torch.cuda.stream(self._tv_stream):
                    self.tv()

        if self.fused_fwd and P_ > 1:
            raise RuntimeError("fused_fwd works on the whole batch: set nparts = 1")
        if P_ <= 1:
            if self.fused_fwd:
                launch_tv()
                self.fwd_fused()
            else:
                self.encode_fwd()
                launch_tv()
                self.mlp_fwd()
            self.composite_loss()
            self.mlp_bwd()
            self.encode_bwd()
        else:
            # independent chains, one stream per part
            launch_tv()
            while len(self._part_streams) < P_ - 1:
                self._part_streams.append(torch.cuda.Stream(device=self.device))
            streams = [main] + self._part_streams[:P_ - 1]
            for st in streams[1:]:
                st.wait_stream(main)
            for k, st in enumerate(streams):
                with torch.cuda.stream(st):
                    self.encode_fwd(k, P_)
                    self.mlp_fwd(k, P_)
                    self.composite_loss(k, P_)
                    self.mlp_bwd(k, P_)
                    self.encode_bwd(k, P_)
            for st in streams[1:]:
                main.wait_stream(st)
        if fork_tv:
            main.wait_stream(self._tv_stream)

    def _under_zeroing(self, fn, zero_mlp=False):
        """Run `fn` while the gradient table of the OTHER parity (and with `zero_mlp` its MLP gradient) is zeroed on a side stream
        underneath; joined before returning."""
        main = torch.cuda.current_stream()
        if self._zero_stream is None:
            self._zero_stream = torch.cuda.Stream(device=self.device)
        side = self._zero_stream
        side.wait_stream(main)
        with torch.cuda.stream(side):
            self.gtables[self.parity ^ 1].zero_()
            if zero_mlp:
                self.g_mlps[(self.parity ^ 1) % len(self.g_mlps)].zero_()
        fn()
        main.wait_stream(side)

    def _compute_dp(self):
        """`_compute` for the fused data-parallel optimizers: the gradient buffers of the OTHER parity (consumed by every peer in the
        previous step's reduce, which ended with a barrier) are zeroed underneath this step's forward / backward."""
        self._under_zeroing(self._compute, zero_mlp=True)

    def _compute_then_adam(self):
        """forward + backward + optimizer of one step (single GPU).  With `defer_zero` the gradient table the PREVIOUS step used is
        zeroed on a side stream underneath this step's optimizer sweep, and this step's optimizer leaves its own table for the next
        step to clean."""
        self._compute()
        self._adam_sg()

    def _compute_sg(self):
        """`_compute` of a single-GPU step whose optimizer is launched separately (see `prefetch_at`)."""
        self._compute()

    def _adam_sg(self):
        """The optimizer of a single-GPU step.  With `defer_zero` the other gradient table is zeroed underneath it, not underneath the
        forward and backward.  Forked at the start of the step, the 97.6 MB zeroing (23,906 blocks) filled the SMs first: in the
        graph-replayed lego step the gathers and TV started 76 us into the step instead of 2 us.  Beside the optimizer's table sweep
        it shares HBM with another stream and delays no latency-bound kernel.  On an H100 80GB HBM3 (700 W) this took bench.py's lego
        step from 287.7-289.1 to 299.8-301.1 M samples/s and the garden step from 370.2-372.9 to 385.8-386.2."""
        if not self.defer_zero:
            self.adam()
            return
        self._under_zeroing(lambda: self.adam(keep_grads=True))

    # -------------------------------------------------------------------------------------------
    def _graph(self, name, fn):
        """Capture-once CUDA graph of `fn` for the current (slot, shading, alpha) configuration."""
        # only what the captured launches actually depend on goes into the key (fewer captures)
        if name == "march":
            key = (name, self.cur, bool(self.use_cam_near_far))
        elif name in ("adam", "peer_adam"):
            key = (name, self.parity)
        else:
            key = (name, self.cur, self.parity, int(self.params.shading_full), int(self.params.gt_has_alpha), int(self.nparts),
                   bool(self.fused_fwd), int(self.tv_fallback_points), bool(self.defer_zero))
        g = self._graphs.get(key)
        if g is None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                fn()
            self._graphs[key] = g
        return g

    def _run(self, name, fn, use_graph):
        if use_graph:
            self._graph(name, fn).replay()
        else:
            fn()

    def step(self, rays_o=None, rays_d=None, gt=None, bg_color=None, noises=None, shading="full", lr=None, use_graph=True,
             grad_sync=None, next_batch=None, cam_near_far=None, index=None, next_index=None):
        """One optimizer step on the batch (rays_o, rays_d, gt, bg_color[, noises]).

        * tensors given: copied into the step buffers first (pinned host -> async H2D);
          with rays_o=None the buffers of the current slot are used as they are.
        * `cam_near_far` [N,2]: per-ray (near, far) clamp (used when `use_cam_near_far` is set; renderer.py:689-691).
        * `next_batch=(rays_o, rays_d, gt, bg[, noises[, cam_near_far]])`: the NEXT step's batch; its H2D copy and its march
          (which do not depend on the parameters) are enqueued on a side stream and overlap this step's
          compute.  The following step() call must then pass that same batch (its copy and march are skipped).
        * `grad_sync`: callable run between backward and optimizer (data-parallel gradient all-reduce).
        * adaptive ray count (`cfg.adaptive_num_rays`): every batch has `max_rays` (= self.N) rows; the step uses the first n, the count
          the previous march left in `ray_ctl[0]` (recorded in the slot's counters[16]); rows >= n are never read.
        * `index` (appearance codes, `cfg.ind_dim > 0`: required with a batch, rejected without codes): the reference's data['index'],
          the training image of the batch (an int) or of every ray (an int32 [N] tensor, random_image_batch).  It is staged with the batch
          (persistent per-slot buffer: graph replays read it); `next_index` goes with `next_batch`.  Indices on the host are range-checked;
          a device tensor is not (a check would synchronise, as n2m_s0_gen_rays does not check its indices either).
        No host sync happens here; read `loss_acc` / `counters` afterwards."""
        self._check_index(index, "index")
        self._check_index(next_index, "next_index")
        if self.ind_dim and grad_sync is not None:
            raise ValueError("data-parallel training with appearance codes (ind_dim > 0) is not supported")
        if self.ind_dim and next_batch is not None and next_index is None:
            raise ValueError("next_index is required with next_batch when the model has appearance codes (ind_dim > 0)")
        main = torch.cuda.current_stream()
        if self._prefetched is not None:
            self.cur = self._prefetched
            self._prefetched = None
            main.wait_event(self._ev_march[self.cur])
            marched = True
        else:
            if rays_o is not None:
                if self.ind_dim and index is None:
                    raise ValueError("index is required when the model has appearance codes (ind_dim > 0)")
                self.slots[self.cur].load(rays_o, rays_d, gt, bg_color, noises, cam_near_far)
            if index is not None:
                self.slots[self.cur].load_index(index)
            marched = False
        if lr is not None:
            self.opt_state[4:5].fill_(float(lr))
        key = (shading == "full", self.slots[self.cur].has_alpha)
        if key != (bool(self.params.shading_full), bool(self.params.gt_has_alpha)):
            self._fill_params(*key)

        ev_start = ev_mid = None
        split = next_batch is not None and self.prefetch_at == "optimizer"
        if next_batch is not None:
            # the prefetch below must come after whatever is already queued on this stream (e.g. set_occupancy), but NOT after
            # this step's own compute: mark the spot now, enqueue the compute first (the GPU starts on it while the host is
            # still enqueueing the prefetch -- matters when the caller synchronises every step), the prefetch afterwards
            ev_start = torch.cuda.Event(); ev_start.record(main)

        def mid():
            nonlocal ev_mid
            if split:
                ev_mid = torch.cuda.Event(); ev_mid.record(main)

        ev_marched = None
        if not marched:
            self._run("march", self.march, use_graph)
            if next_batch is not None and self.adaptive and not split:
                # the next batch's march reads the ray count this march's scan writes (ray_ctl[0])
                ev_marched = torch.cuda.Event(); ev_marched.record(main)
        if grad_sync is None:
            if split:
                self._run("compute_sg", self._compute_sg, use_graph)
                mid()
                self._run("adam_sg", self._adam_sg, use_graph)
            else:
                self._run("compute+adam", self._compute_then_adam, use_graph)
            if self.defer_zero:
                self.parity ^= 1           # the next step accumulates into the other gradient table
        elif getattr(grad_sync, "fused", False):
            # data parallel, sharded optimizer fused with its collective over NVLink peer memory (parallel.PeerAdam / NvlsAdam)
            self._run("compute", self._compute_dp, use_graph)
            mid()
            p = self.parity
            self._run("peer_adam", lambda: grad_sync.run(p), use_graph)
            self.parity ^= 1
        else:
            # data parallel: [forward+backward] -> gradient all-reduce (NCCL) -> [optimizer]
            self._run("compute", self._compute, use_graph)
            mid()
            grad_sync()
            self._run("adam", self.adam, use_graph)
        ev = torch.cuda.Event(); ev.record(main)
        self._ev_done[self.cur] = ev
        self.global_step += 1
        if next_batch is not None:
            # side stream: stage the next batch into the other slot (at once) and march it (underneath the optimizer stage)
            nxt = 1 - self.cur
            if self._side is None:
                self._side = torch.cuda.Stream(device=self.device, priority=-1 if self.prefetch_at == "optimizer" else 0)
            side = self._side
            if self._ev_done[nxt] is not None:
                side.wait_event(self._ev_done[nxt])              # slot `nxt` was last read by the previous step
            side.wait_event(ev_start)
            if ev_marched is not None:
                side.wait_event(ev_marched)
            keep = self.cur
            with torch.cuda.stream(side):
                self.slots[nxt].load(*next_batch)
                if self.ind_dim:
                    self.slots[nxt].load_index(next_index)
                if ev_mid is not None:
                    side.wait_event(ev_mid)
                if self.adaptive:
                    self._ray_ctl_undo.copy_(self.ray_ctl)          # a dropped prefetch restores it (drop_prefetch)
                self.cur = nxt
                self._run("march", self.march, use_graph)
                self.cur = keep
                ev = torch.cuda.Event(); ev.record(side)
                self._ev_march[nxt] = ev
            self._prefetched = nxt


    def _check_index(self, index, what):
        if index is None:
            return
        if not self.ind_dim:
            raise ValueError(f"{what} given, but the model has no appearance codes (ind_dim = 0)")
        if isinstance(index, bool) or not isinstance(index, (int, torch.Tensor)):
            raise ValueError(f"{what} must be an int or an int32 tensor of one index per ray, got {type(index).__name__}")
        if isinstance(index, torch.Tensor):
            if index.dtype != torch.int32 or index.shape != (self.N,):
                raise ValueError(f"{what} must be an int32 tensor of shape ({self.N},), got {index.dtype} {tuple(index.shape)}")
            if index.device.type != "cpu":
                return                      # not checked on the device: see step()
            lo, hi = (int(index.min()), int(index.max())) if index.numel() else (0, 0)
        else:
            lo = hi = index
        if lo < 0 or hi >= self.ind_num:
            raise ValueError(f"{what} out of range [0, {self.ind_num}): [{lo}, {hi}]")

    # -------------------------------------------------------------------------------------------
    # density grid / bitfield update and evaluation rendering
    # -------------------------------------------------------------------------------------------
    def update_density_grid(self, decay=0.95, density_thresh=10.0, generator=None, shard_group=None):
        """NeRFRenderer.update_extra_state (renderer.py:1074-1149): evaluate the density field at one jittered
        point per grid cell and cascade (hash gather + sigma_net on tensor cores), grid = max(grid * decay, sigma),
        threshold = min(mean(clamp(grid, 0)), density_thresh), repack the bitfield.  Everything stays on the
        device (the reference syncs for `mean_density.item()`).
        With `step(next_batch=...)` a batch whose march is already staged on the side stream keeps the samples of the previous
        bitfield (the update then takes effect one step later than in the reference); call `drop_prefetch()` first for the
        reference's exact order.
        `generator`: CUDA generator of the per-cell jitter (default: the global one, as the reference).
        `shard_group` (data parallel, identical replicas): every rank evaluates 1/W of the cells of each cascade and the grid rows are
        all-gathered (NCCL; 8 MB per cascade) -- the 2.1 M - 10.5 M density evaluations per call divide by W.  All ranks must pass
        generators in the same state; the result is then bit-identical to the replicated update."""
        c = self.cfg
        H, cells = c.grid_size, c.grid_size ** 3
        dev = self.device
        W, rank = 1, 0
        if shard_group is not None:
            import torch.distributed as dist
            W, rank = dist.get_world_size(shard_group), dist.get_rank(shard_group)
            if generator is None:
                raise ValueError("a sharded density-grid update needs a generator that is in the same state on every rank")
            if cells % W:
                raise ValueError(f"grid cells ({cells}) not divisible by the world size ({W})")
        lo, hi = rank * (cells // W), (rank + 1) * (cells // W)
        pparams = self.params_with(shading_full=0)           # sigma only: skip the specular rounds
        pp = ctypes.byref(pparams)
        for cas in range(c.cascade):
            bound = float(min(2 ** cas, c.bound))
            row = self.density_grid[cas]
            noise = torch.rand(cells, 3, device=dev, generator=generator)      # == torch.rand_like(cas_xyzs) of the reference (renderer.py:1110)
            for first in range(lo, hi, self.Mcap):
                cnt = min(self.Mcap, hi - first)
                call("n2m_s0_grid_points", H, first, cnt, bound, ptr(noise), ptr(self._pts), stream())
                self._pcount.fill_(cnt)
                call("n2m_s0_encode_points", pp, ptr(self._pts), None, ptr(self._pcount), self.Mcap, ptr(self.table),
                     ptr(self.offsets), ptr(self.enc_tiles), stream())
                call("n2m_s0_mlp_fwd", pp, ptr(self.enc_tiles), ptr(self._pcount), self.Mcap, ptr(self.wpack), ptr(self.out),
                     None, 0, 1, stream())
                call("n2m_s0_grid_update", ptr(self.out), cnt, float(decay), row.data_ptr() + 4 * first, stream())
            if W > 1:
                dist.all_gather_into_tensor(row, row[lo:hi].clone(), group=shard_group)
        self.mean_density = self.density_grid.clamp(min=0).mean().reshape(1)
        if self._side is not None:
            # a prefetched march on the side stream may still be reading the bitfield
            torch.cuda.current_stream().wait_stream(self._side)
        call("n2m_s0_packbits_dev", ptr(self.density_grid), self.density_bitfield.numel(), ptr(self.mean_density),
             float(density_thresh), ptr(self.density_bitfield), stream())

    @torch.no_grad()
    def density_volume(self, resolution=512, density_thresh=10.0):
        """The marching-cubes input of NeRFRenderer.export_stage0 (renderer.py:480-513): sigma on the regular grid linspace(-1, 1, R)^3
        (x-major), multiplied by the occupancy mask of cascade 0 (density_grid > min(mean_density, density_thresh), nearest-neighbour
        up-sampled) so that empty / untrained regions stay empty; for R == grid_size the density grid itself, re-mapped from Morton order.
        Returns a float32 [R, R, R] tensor on the device (the mesh extraction that follows in the reference is CPU library code)."""
        self.drop_prefetch()
        dev, c = self.device, self.cfg
        R, H = int(resolution), c.grid_size
        from . import raymarching as rm
        coords = rm.morton3D_invert(torch.arange(H ** 3, dtype=torch.int32, device=dev)).long()
        grid0 = torch.zeros(H, H, H, device=dev)
        grid0[tuple(coords.T)] = self.density_grid[0]
        if R == H:
            return torch.nan_to_num(grid0, 0)
        mean = getattr(self, "mean_density", None)
        thresh = min(float(mean.item()), density_thresh) if mean is not None else density_thresh
        pparams = self.params_with(shading_full=0)
        pp = ctypes.byref(pparams)
        lin = torch.linspace(-1, 1, R, device=dev)
        sig = torch.empty(R ** 3, device=dev)
        per = max(1, self.Mcap // (R * R))                # x-slabs per chunk
        for x0 in range(0, R, per):
            x1 = min(R, x0 + per)
            xx, yy, zz = torch.meshgrid(lin[x0:x1], lin, lin, indexing="ij")
            pts = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1).contiguous()
            n = pts.shape[0]
            self._pcount.fill_(n)
            call("n2m_s0_encode_points", pp, ptr(pts), None, ptr(self._pcount), self.Mcap, ptr(self.table), ptr(self.offsets),
                 ptr(self.enc_tiles), stream())
            call("n2m_s0_mlp_fwd", pp, ptr(self.enc_tiles), ptr(self._pcount), self.Mcap, ptr(self.wpack), ptr(self.out), None, 0, 1,
                 stream())
            sig[x0 * R * R: x1 * R * R] = self.out[:n, 0]
        mask = torch.nn.functional.interpolate(grid0[None, None], size=[R] * 3, mode="nearest")[0, 0] > thresh
        return torch.nan_to_num(sig.view(R, R, R) * mask, 0)

    RENDER_SCHEDULE = (8, 8, 16, 16, 32, 64, 128, 256, 512)          # slab widths per round (sum >= max_steps = 1024)

    @torch.no_grad()
    def render(self, rays_o, rays_d, bg_color=1.0, shading="full", early_stop=True, chunk=262144, cam_near_far=None):
        """Forward-only rendering of arbitrarily many rays, no perturbation.  Returns (image [R,3], weights_sum [R], depth [R]) on the device.

        `early_stop` (default): NeRFRenderer.render's inference branch (renderer.py:749-802) with the alive-ray bookkeeping on the device
        (csrc/render.cu): per chunk of `chunk` rays one host call enqueues RENDER_SCHEDULE rounds of march -> gather -> MLPs -> slab
        compositor + survivor compaction; rays stop at T < T_thresh, so samples behind the first surfaces are never evaluated.  One
        read-back per chunk checks that no ray is left alive (else further rounds run); bench.py's `psnr.eval_render` times it
        against the all-samples path on an 800 x 800 view.  `render_rounds` / `render_rows` afterwards: rounds of the last chunk, sample rows evaluated in total.
        `early_stop=False`: every ray's samples are marched up front and evaluated with the training kernels in chunks of `num_rays`
        (the compositor stops at T_thresh, the gather / MLP work behind it is spent)."""
        self.drop_prefetch()
        if not early_stop:
            return self._render_all_samples(rays_o, rays_d, bg_color, shading)
        dev = self.device
        R = rays_o.shape[0]
        rays_o = rays_o.to(dev, torch.float32).contiguous(); rays_d = rays_d.to(dev, torch.float32).contiguous()
        img = torch.empty(R, 3, device=dev); ws = torch.empty(R, device=dev); dep = torch.empty(R, device=dev)
        if R == 0:
            return img, ws, dep
        chunk = int(min(max(chunk, 32), max(R, 32)))
        rb = getattr(self, "_render_buf", None)
        if rb is None or rb["chunk"] < chunk:
            cap = ((chunk * 16 + 127) // 128) * 128                                   # sample rows per round (160 B each)
            rb = self._render_buf = dict(
                chunk=chunk, cap=cap, rays_t=torch.empty(chunk, device=dev), rays_far=torch.empty(chunk, device=dev),
                alive=torch.empty(2 * chunk, dtype=torch.int32, device=dev), ctl=torch.zeros(16, dtype=torch.int32, device=dev),
                recs=torch.empty(cap, 4, device=dev), enc=torch.empty(cap * 64, dtype=torch.float16, device=dev),
                out=torch.empty(cap, 4, device=dev))
        rb["params"] = self.params_with(shading_full=int(shading == "full"))        # the parameter block of this call's launches
        pp = ctypes.byref(rb["params"])
        sched = (ctypes.c_uint32 * len(self.RENDER_SCHEDULE))(*self.RENDER_SCHEDULE)
        more = (ctypes.c_uint32 * 2)(512, 512)
        bg_t = bg_color.to(dev, torch.float32).contiguous() if torch.is_tensor(bg_color) else None
        cnf = cam_near_far.to(dev, torch.float32).contiguous() if cam_near_far is not None else None
        rows_total = 0
        for a in range(0, R, chunk):
            n = min(chunk, R - a)
            ro, rd = rays_o[a:a + n], rays_d[a:a + n]
            io, wo, do = img[a:a + n], ws[a:a + n], dep[a:a + n]
            call("n2m_s0_render_begin", pp, ptr(ro), ptr(rd), ptr(self.aabb), ptr(cnf[a:a + n]) if cnf is not None else None, n,
                 ptr(rb["rays_t"]), ptr(rb["rays_far"]), ptr(rb["alive"]), ptr(rb["ctl"]), ptr(wo), ptr(do), ptr(io), stream())

            def rounds(widths):
                if self.ind_dim:        # evaluation uses code 0 (renderer.py:702-703)
                    call("n2m_s0_render_rounds_codes", pp, ptr(ro), ptr(rd), ptr(self.density_bitfield), n, widths, len(widths),
                         ptr(rb["rays_t"]), ptr(rb["rays_far"]), ptr(rb["alive"]), ptr(rb["ctl"]), ptr(rb["recs"]), ptr(rb["enc"]),
                         ptr(rb["out"]), rb["cap"], ptr(self.table), ptr(self.offsets), ptr(self.wpack), self._codes_table(), ptr(wo),
                         ptr(do), ptr(io), stream())
                    return
                call("n2m_s0_render_rounds", pp, ptr(ro), ptr(rd), ptr(self.density_bitfield), n, widths, len(widths), ptr(rb["rays_t"]),
                     ptr(rb["rays_far"]), ptr(rb["alive"]), ptr(rb["ctl"]), ptr(rb["recs"]), ptr(rb["enc"]), ptr(rb["out"]), rb["cap"],
                     ptr(self.table), ptr(self.offsets), ptr(self.wpack), ptr(wo), ptr(do), ptr(io), stream())

            rounds(sched)
            guard = 0
            ctl = rb["ctl"].tolist()                           # the one read-back per chunk; further rounds only if rays are left
            while ctl[10] > 0:
                rounds(more)
                ctl = rb["ctl"].tolist()
                guard += 1
                if guard > 4096:
                    raise RuntimeError("render: rays do not terminate")
            rows_total += ctl[13]
            call("n2m_s0_render_finish", ptr(io), ptr(wo), ptr(bg_t[a:a + n]) if bg_t is not None else None,
                 float(bg_color) if bg_t is None else 0.0, n, stream())
        self.render_rounds, self.render_rows = ctl[12], rows_total          # diagnostics: rounds of the last chunk, rows evaluated in all
        return img, ws, dep

    @torch.no_grad()
    def _render_all_samples(self, rays_o, rays_d, bg_color=1.0, shading="full"):
        R = rays_o.shape[0]
        img = torch.empty(R, 3, device=self.device); ws = torch.empty(R, device=self.device); dep = torch.empty(R, device=self.device)
        key = (shading == "full", False)
        self._fill_params(*key)
        slot = self.slots[self.cur]
        zeros3 = torch.zeros(self.N, 3, device=self.device)
        bg = torch.full((self.N, 3), float(bg_color), device=self.device) if not torch.is_tensor(bg_color) else None
        C = self.cfg.num_rays           # rays per chunk: the sample slab is sized for num_rays, also when the buffers are max_rays wide
        for a in range(0, R, C):
            b = min(R, a + C)
            n = b - a
            ro = torch.zeros(self.N, 3, device=self.device); rd = torch.ones(self.N, 3, device=self.device)
            ro[:n] = rays_o[a:b]; rd[:n] = rays_d[a:b]
            if n < self.N:
                ro[n:] = 1e6            # padding rays miss the volume
            if bg is None:
                bgc = torch.ones(self.N, 3, device=self.device); bgc[:n] = bg_color[a:b]
            slot.load(ro, rd, zeros3, bg if bg is not None else bgc, torch.zeros(self.N, device=self.device))
            if self.ind_dim:
                slot.load_index(0)              # evaluation uses code 0 (renderer.py:702-703)
            self.loss_acc.zero_()
            self.march(all_rays=True); self.encode_fwd(); self.mlp_fwd(); self.composite_loss(all_rays=True)
            img[a:b] = self.image[:n]; ws[a:b] = self.weights_sum[:n]; dep[a:b] = self.depth[:n]
        return img, ws, dep

    def check_capacity(self, grow=True, headroom=1.25):
        """(host sync) -> (overflowed steps since the last call, largest M seen).  With `grow` the per-step sample buffers are
        re-allocated for headroom * max M (and the captured graphs dropped) when a step overflowed."""
        self.drop_prefetch()
        torch.cuda.synchronize()
        over = sum(int(s.counters[13].item()) for s in self.slots)
        max_m = max(int(s.counters[14].item()) for s in self.slots)
        for s_ in self.slots:
            s_.counters[13:15] = 0
        if over and grow:
            new_cap = (int(max_m * headroom) + 127) // 128 * 128
            if new_cap > self.Mcap:
                self._resize_samples(new_cap)
        return over, max_m

    def check_rays(self):
        """(host sync) adaptive ray count -> (steps whose requested count was clamped to max_rays since the last call, largest count
        requested since the last call, ray count of the next march).  Without adaptive mode (0, num_rays, num_rays), no sync.
        Drops a prefetched batch first, as check_capacity() does: its staged march has counted a request of a step not yet run."""
        if not self.adaptive:
            return 0, self.N, self.N
        self.drop_prefetch()
        torch.cuda.synchronize()
        nxt, clamped, largest = (int(v) for v in self.ray_ctl[:3].tolist())
        self.ray_ctl[1:3] = 0
        return clamped, largest, nxt

    def _resize_samples(self, Mc):
        dev = self.device
        self.Mcap = self.cfg.max_samples = int(Mc)
        for s_ in self.slots:
            s_.recs = torch.zeros(Mc, 4, device=dev)
        self.enc_tiles = torch.zeros(Mc * 64, dtype=torch.float16, device=dev)
        self.denc_tiles = torch.zeros(Mc * 64, dtype=torch.float16, device=dev)
        self.out = torch.zeros(Mc, 4, device=dev)
        self.dout = torch.zeros(Mc, 4, device=dev)
        self._pts = torch.zeros(Mc, 3, device=dev)
        self._graphs = {}

    def drop_prefetch(self):
        """Forget a batch staged by `next_batch=` (e.g. when the caller changes its batch sequence).  With the adaptive ray count the
        dropped march has already written the count after its own batch and counted its request: the control block is put back as it
        was before that march, so the next step takes the count the reference would and the clamp counts stay those of the steps run."""
        if self._side is not None:
            self._side.synchronize()
        if self._prefetched is not None:
            if self.adaptive:
                self.ray_ctl.copy_(self._ray_ctl_undo)
            self.cur = self._prefetched      # keep the slot alternation in phase (graphs are captured per slot)
        self._prefetched = None

    def read_loss(self):
        """(host sync) loss of the last step as the reference reports it: rgb/mask part + specular regulariser."""
        acc = self.loss_acc.tolist()
        M = max(int(self.counters[1].item()), 1)
        loss = acc[0]
        if self.params.shading_full and self.cfg.lambda_specular > 0:
            loss += self.cfg.lambda_specular * acc[1] / M
        if self.cfg.lambda_entropy > 0:
            # acc[2]: sum of the entropies of the weights the compositor touched; every other entry of `weights` is 0,
            # clamped to 1e-5 by the loss (utils.py:729)
            w0 = 1e-5
            h0 = -w0 * math.log2(w0) - (1 - w0) * math.log2(1 - w0)
            touched = acc[3]
            loss += self.cfg.lambda_entropy * ((acc[2] + (M - touched) * h0) / M)
        return loss
