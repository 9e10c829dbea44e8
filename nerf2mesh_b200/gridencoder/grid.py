"""Drop-in `gridencoder` backed by libn2m_b200.so (sm_90a).

Mirrors reference gridencoder/grid.py:24-192: `grid_encode` autograd Function (same positional
arguments), `GridEncoder` module (same constructor, parameter/buffer names `embeddings`,
`offsets`, same init U(-1e-4, 1e-4)), `grad_total_variation`.  The kernel-side layout is the
reference's ([L, B, C] level-major output, permuted here), the half-precision rule is the
reference's (table cast to fp16 iff autocast is on and C is even, grid.py:45-46).
"""
import numpy as np
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.amp import custom_bwd, custom_fwd

from .._lib import call, ptr, stream

_gridtype_to_id = {"hash": 0, "tiled": 1}
_interp_to_id = {"linear": 0, "smoothstep": 1}


def _check(t, name, floating=True):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")
    if floating and t.dtype not in (torch.float32, torch.float16, torch.float64):
        raise RuntimeError(f"{name} must be a floating tensor")
    if not floating and t.dtype != torch.int32:
        raise RuntimeError(f"{name} must be an int tensor")


def _dtype_id(t):
    if t.dtype == torch.float32:
        return 0
    if t.dtype == torch.float16:
        return 1
    raise RuntimeError("embeddings must be float32 or float16")


class _grid_encode(Function):
    @staticmethod
    @custom_fwd(device_type="cuda")
    def forward(ctx, inputs, embeddings, offsets, per_level_scale, base_resolution,
                calc_grad_inputs=False, gridtype=0, align_corners=False, interpolation=0, max_level=None):
        # inputs [B, D] float32 in [0, 1]; embeddings [rows, C]; offsets int32 [L+1]  ->  [B, L*C]
        inputs = inputs.float().contiguous()
        B, D = inputs.shape
        L = offsets.shape[0] - 1
        C = embeddings.shape[1]
        S = float(np.log2(per_level_scale))
        H = int(base_resolution)
        max_level = L if max_level is None else min(int(max_level), L)

        if torch.is_autocast_enabled() and C % 2 == 0:
            embeddings = embeddings.to(torch.half)
        embeddings = embeddings.contiguous()
        _check(inputs, "inputs"); _check(embeddings, "embeddings"); _check(offsets, "offsets", floating=False)

        outputs = torch.empty(L, B, C, device=inputs.device, dtype=embeddings.dtype)
        if max_level < L:
            outputs.zero_()
        dy_dx = None
        if calc_grad_inputs:
            dy_dx = torch.empty(B, L * D * C, device=inputs.device, dtype=embeddings.dtype)
            if max_level < L:
                dy_dx.zero_()

        call("n2m_grid_encode_forward", ptr(inputs), ptr(embeddings), ptr(offsets), ptr(outputs),
             B, D, C, L, max_level, S, H, ptr(dy_dx), int(gridtype), int(bool(align_corners)),
             int(interpolation), _dtype_id(embeddings), stream())

        outputs = outputs.permute(1, 0, 2).reshape(B, L * C)
        ctx.save_for_backward(inputs, embeddings, offsets, dy_dx)
        ctx.dims = (B, D, C, L, S, H, int(gridtype), int(interpolation), max_level)
        ctx.align_corners = bool(align_corners)
        return outputs

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, grad):
        inputs, embeddings, offsets, dy_dx = ctx.saved_tensors
        B, D, C, L, S, H, gridtype, interpolation, max_level = ctx.dims
        grad = grad.to(embeddings.dtype).view(B, L, C).permute(1, 0, 2).contiguous()   # [L, B, C]
        grad_embeddings = torch.zeros_like(embeddings)
        grad_inputs = torch.zeros_like(inputs, dtype=embeddings.dtype) if dy_dx is not None else None
        call("n2m_grid_encode_backward", ptr(grad), ptr(inputs), ptr(embeddings), ptr(offsets),
             ptr(grad_embeddings), B, D, C, L, max_level, S, H, ptr(dy_dx), ptr(grad_inputs),
             gridtype, int(ctx.align_corners), interpolation, _dtype_id(embeddings), stream())
        if grad_inputs is not None:
            grad_inputs = grad_inputs.to(inputs.dtype)
        return grad_inputs, grad_embeddings, None, None, None, None, None, None, None, None


grid_encode = _grid_encode.apply


def level_offsets(input_dim, num_levels, per_level_scale, base_resolution, log2_hashmap_size, align_corners):
    """Row offsets of every level, each level padded to a multiple of 8 rows (grid.py:124-134)."""
    offsets, offset = [], 0
    max_params = 2 ** log2_hashmap_size
    for i in range(num_levels):
        resolution = int(np.ceil(base_resolution * per_level_scale ** i))
        side = resolution if align_corners else resolution + 1
        rows = min(max_params, side ** input_dim)
        rows = int(np.ceil(rows / 8) * 8)
        offsets.append(offset)
        offset += rows
    offsets.append(offset)
    return np.array(offsets, dtype=np.int32)


class GridEncoder(nn.Module):
    def __init__(self, input_dim=3, num_levels=16, level_dim=2, per_level_scale=2, base_resolution=16,
                 log2_hashmap_size=19, desired_resolution=None, gridtype="hash", align_corners=False,
                 interpolation="linear"):
        super().__init__()
        if desired_resolution is not None:
            per_level_scale = np.exp2(np.log2(desired_resolution / base_resolution) / (num_levels - 1))
        self.input_dim = input_dim
        self.num_levels = num_levels
        self.level_dim = level_dim
        self.per_level_scale = per_level_scale
        self.log2_hashmap_size = log2_hashmap_size
        self.base_resolution = base_resolution
        self.output_dim = num_levels * level_dim
        self.gridtype = gridtype
        self.gridtype_id = _gridtype_to_id[gridtype]
        self.interpolation = interpolation
        self.interp_id = _interp_to_id[interpolation]
        self.align_corners = align_corners
        self.max_params = 2 ** log2_hashmap_size

        offsets = level_offsets(input_dim, num_levels, per_level_scale, base_resolution,
                                log2_hashmap_size, align_corners)
        self.register_buffer("offsets", torch.from_numpy(offsets))
        self.n_params = int(offsets[-1]) * level_dim
        self.embeddings = nn.Parameter(torch.empty(int(offsets[-1]), level_dim))
        self.reset_parameters()

    def reset_parameters(self):
        self.embeddings.data.uniform_(-1e-4, 1e-4)

    def __repr__(self):
        top = int(round(self.base_resolution * self.per_level_scale ** (self.num_levels - 1)))
        return (f"GridEncoder: input_dim={self.input_dim} num_levels={self.num_levels} "
                f"level_dim={self.level_dim} resolution={self.base_resolution} -> {top} "
                f"per_level_scale={self.per_level_scale:.4f} params={tuple(self.embeddings.shape)} "
                f"gridtype={self.gridtype} align_corners={self.align_corners} "
                f"interpolation={self.interpolation}")

    def forward(self, inputs, bound=1, max_level=None):
        # inputs [..., input_dim] in [-bound, bound] -> [..., num_levels * level_dim]
        inputs = (inputs + bound) / (2 * bound)
        prefix = list(inputs.shape[:-1])
        inputs = inputs.view(-1, self.input_dim)
        outputs = grid_encode(inputs, self.embeddings, self.offsets, self.per_level_scale,
                              self.base_resolution, inputs.requires_grad, self.gridtype_id,
                              self.align_corners, self.interp_id, max_level)
        return outputs.view(prefix + [self.output_dim])

    @torch.amp.autocast("cuda", enabled=False)
    def grad_total_variation(self, weight=1e-7, inputs=None, bound=1, B=1000000):
        """Add the TV-regulariser gradient at the cells visited by `inputs` into embeddings.grad,
        in place (grid.py:170-192; called from Trainer.post_train_step, utils.py:801-823)."""
        D = self.input_dim
        C = self.embeddings.shape[1]
        L = self.offsets.shape[0] - 1
        S = float(np.log2(self.per_level_scale))
        H = int(self.base_resolution)
        if inputs is None or inputs.size(0) == 0:
            inputs = torch.rand(B, self.input_dim, device=self.embeddings.device)
        else:
            inputs = (inputs + bound) / (2 * bound)
            inputs = inputs.view(-1, self.input_dim)
            B = inputs.shape[0]
        if self.embeddings.grad is None:
            raise ValueError("grad is None, should be called after loss.backward() and before optimizer.step()!")
        inputs = inputs.float().contiguous()
        call("n2m_grad_total_variation", ptr(inputs), ptr(self.embeddings.data), ptr(self.embeddings.grad),
             ptr(self.offsets), float(weight), B, D, C, L, S, H, self.gridtype_id,
             int(bool(self.align_corners)), stream())
