"""Batch sampling on the device: the stage-0 training branch of `NeRFDataset.collate` (nerf/provider.py:300-331) and
`get_rays` (nerf/utils.py:236-290) for random (image, pixel) pairs, with the pose / image set resident in HBM (the
reference's `--preload`).  One kernel (`n2m_s0_gen_rays`, include/n2m_b200_fused.h) replaces the ~15 small torch
kernels and the [H*W] meshgrid the reference builds per step."""
import ctypes

import torch

from . import _lib
from ._lib import P, U, call, ptr, stream

_lib.register({"n2m_s0_gen_rays": [P, U, P, U, U, P, P, P, U, U, P, P, P, P]})


class DeviceRaySampler:
    def __init__(self, poses, intrinsics, H, W, images=None, device="cuda"):
        """poses [B,4,4] float (camera-to-world, the reference's convention after its loaders), intrinsics (fx, fy, cx, cy),
        images uint8 [B,H,W,3|4] or None."""
        self.device = torch.device(device)
        self.poses = torch.as_tensor(poses, dtype=torch.float32).to(self.device).contiguous()
        self.H, self.W = int(H), int(W)
        self._intr = (ctypes.c_float * 4)(*[float(v) for v in intrinsics])
        self.images = None
        if images is not None:
            images = torch.as_tensor(images)
            assert images.dtype == torch.uint8 and images.shape[:3] == (self.poses.shape[0], self.H, self.W) and images.shape[3] in (3, 4)
            self.images = images.to(self.device).contiguous()

    def draw_indices(self, N, generator=None):
        """provider.py:303 (image per ray) and utils.py:271 (pixel per ray): torch.randint on the device."""
        img = torch.randint(0, self.poses.shape[0], (N,), device=self.device, generator=generator, dtype=torch.int32)
        pix = torch.randint(0, self.H * self.W, (N,), device=self.device, generator=generator, dtype=torch.int32)
        return img, pix

    def sample(self, N, img_idx=None, pix_idx=None, generator=None, out=None):
        """-> rays_o [N,3], rays_d [N,3] (unnormalised), gt [N,C] float in [0,1] (None without images), all on the device.
        `out=(rays_o, rays_d, gt)` writes into existing contiguous device tensors."""
        if img_idx is None:
            img_idx, pix_idx = self.draw_indices(N, generator)
        img_idx = img_idx.to(self.device, torch.int32).contiguous(); pix_idx = pix_idx.to(self.device, torch.int32).contiguous()
        C = 0 if self.images is None else int(self.images.shape[3])
        if out is None:
            rays_o = torch.empty(N, 3, device=self.device); rays_d = torch.empty(N, 3, device=self.device)
            gt = torch.empty(N, C, device=self.device) if C else None
        else:
            rays_o, rays_d, gt = out
        call("n2m_s0_gen_rays", ptr(self.poses), int(self.poses.shape[0]), ctypes.cast(self._intr, ctypes.c_void_p), self.H, self.W,
             ptr(img_idx), ptr(pix_idx), ptr(self.images) if C else None, C, N, ptr(rays_o), ptr(rays_d),
             ptr(gt) if (C and gt is not None) else None, stream())
        return rays_o, rays_d, gt
