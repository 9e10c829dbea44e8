"""Drop-in `shencoder` backed by libn2m_b200.so (sm_90a).

Mirrors reference shencoder/sphere_harmonics.py:14-89: `sh_encode(inputs, degree,
calc_grad_inputs)` and the `SHEncoder` module (normalises the direction, degree 1..8)."""
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.amp import custom_bwd, custom_fwd

from .._lib import call, ptr, stream


class _sh_encoder(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, inputs, degree, calc_grad_inputs=False):
        # inputs [B, 3] float in [-1, 1] -> [B, degree^2]
        if not inputs.is_cuda:
            raise RuntimeError("inputs must be a CUDA tensor")
        inputs = inputs.float().contiguous()
        B, input_dim = inputs.shape
        output_dim = degree ** 2
        outputs = torch.empty(B, output_dim, dtype=inputs.dtype, device=inputs.device)
        dy_dx = torch.empty(B, input_dim * output_dim, dtype=inputs.dtype, device=inputs.device) \
            if calc_grad_inputs else None
        call("n2m_sh_encode_forward", ptr(inputs), ptr(outputs), B, input_dim, int(degree), ptr(dy_dx), stream())
        ctx.save_for_backward(inputs, dy_dx)
        ctx.dims = (B, input_dim, int(degree))
        return outputs

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, grad):
        inputs, dy_dx = ctx.saved_tensors
        if dy_dx is None:
            return None, None, None
        grad = grad.float().contiguous()
        B, input_dim, degree = ctx.dims
        grad_inputs = torch.zeros_like(inputs)
        call("n2m_sh_encode_backward", ptr(grad), ptr(inputs), B, input_dim, degree, ptr(dy_dx),
             ptr(grad_inputs), stream())
        return grad_inputs, None, None


sh_encode = _sh_encoder.apply


class SHEncoder(nn.Module):
    def __init__(self, input_dim=3, degree=4):
        super().__init__()
        self.input_dim = input_dim
        self.degree = degree
        self.output_dim = degree ** 2
        assert self.input_dim == 3, "SH encoder only support input dim == 3"
        assert self.degree > 0 and self.degree <= 8, "SH encoder only supports degree in [1, 8]"

    def __repr__(self):
        return f"SHEncoder: input_dim={self.input_dim} degree={self.degree}"

    def forward(self, inputs, size=1):
        # inputs [..., 3] in [-size, size] -> [..., degree^2]
        inputs = inputs / size
        inputs = inputs / torch.norm(inputs, dim=-1, keepdim=True)
        prefix = list(inputs.shape[:-1])
        inputs = inputs.reshape(-1, self.input_dim)
        outputs = sh_encode(inputs, self.degree, inputs.requires_grad)
        return outputs.reshape(prefix + [self.output_dim])
