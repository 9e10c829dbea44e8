"""Drop-in `raymarching` operators backed by libn2m_b200.so (sm_90a).

Mirrors the reference's Python operator surface (reference: raymarching/raymarching.py:19-386):
same callable names, argument order, defaults, dtypes, shapes and zero-init contracts, so that
`nerf/renderer.py` works unmodified (call sites renderer.py:688,711,717,741,776,796,1020,1100,1142).
Deliberate differences:
  * every kernel runs on torch's CURRENT stream (the reference uses the legacy default stream);
  * `march_rays_train` returns ray offsets in ray order (deterministic), the reference's come
    from an atomic counter; per-ray sample sets and counts are bit-identical;
  * native errors surface as RuntimeError with the library's message.
"""
import torch
from torch.autograd import Function
from torch.amp import custom_bwd, custom_fwd

from .. import _lib
from .._lib import call, ptr, stream

__all__ = [
    "near_far_from_aabb", "sph_from_ray", "morton3D", "morton3D_invert", "packbits",
    "flatten_rays", "march_rays_train", "composite_rays_train", "march_rays", "composite_rays",
]


def _cuda(t):
    return t if t.is_cuda else t.cuda()


def _rays(t):
    return _cuda(t).float().contiguous().view(-1, 3)


# ----------------------------------------------------------------------------------------------
# utils
# ----------------------------------------------------------------------------------------------
class _near_far_from_aabb(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, rays_o, rays_d, aabb, min_near=0.2):
        """rays_o/d [N,3], aabb [6] -> nears, fars [N] (raymarching.py:19-49)."""
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        aabb = _cuda(aabb).float().contiguous()
        N = rays_o.shape[0]
        nears = torch.empty(N, dtype=torch.float32, device=rays_o.device)
        fars = torch.empty(N, dtype=torch.float32, device=rays_o.device)
        call("n2m_near_far_from_aabb", ptr(rays_o), ptr(rays_d), ptr(aabb), N, float(min_near),
             ptr(nears), ptr(fars), stream())
        return nears, fars


near_far_from_aabb = _near_far_from_aabb.apply


class _sph_from_ray(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, rays_o, rays_d, radius):
        """rays -> (theta, phi) in [-1,1] on the bounding sphere, [N,2] (raymarching.py:52-80)."""
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        N = rays_o.shape[0]
        coords = torch.empty(N, 2, dtype=torch.float32, device=rays_o.device)
        call("n2m_sph_from_ray", ptr(rays_o), ptr(rays_d), float(radius), N, ptr(coords), stream())
        return coords


sph_from_ray = _sph_from_ray.apply


class _morton3D(Function):
    @staticmethod
    def forward(ctx, coords):
        """coords int [N,3] -> Morton indices int32 [N] (raymarching.py:82-103)."""
        coords = _cuda(coords).int().contiguous()
        N = coords.shape[0]
        indices = torch.empty(N, dtype=torch.int32, device=coords.device)
        call("n2m_morton3D", ptr(coords), N, ptr(indices), stream())
        return indices


morton3D = _morton3D.apply


class _morton3D_invert(Function):
    @staticmethod
    def forward(ctx, indices):
        """Morton indices int [N] -> coords int32 [N,3] (raymarching.py:105-125)."""
        indices = _cuda(indices).int().contiguous()
        N = indices.shape[0]
        coords = torch.empty(N, 3, dtype=torch.int32, device=indices.device)
        call("n2m_morton3D_invert", ptr(indices), N, ptr(coords), stream())
        return coords


morton3D_invert = _morton3D_invert.apply


class _packbits(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, grid, thresh, bitfield=None):
        """grid float [C, H^3] -> bitfield uint8 [C*H^3/8], bit i of byte n = grid[8n+i] > thresh
        (raymarching.py:128-154).  Writes into `bitfield` when given (renderer.py:1142)."""
        grid = _cuda(grid).float().contiguous()
        C, H3 = grid.shape[0], grid.shape[1]
        N = C * H3 // 8
        if bitfield is None:
            bitfield = torch.empty(N, dtype=torch.uint8, device=grid.device)
        call("n2m_packbits", ptr(grid), N, float(thresh), ptr(bitfield), stream())
        return bitfield


packbits = _packbits.apply


class _flatten_rays(Function):
    @staticmethod
    def forward(ctx, rays, M):
        """rays int32 [N,2] (offset,count) -> ray id per sample, int32 [M] (raymarching.py:157-178)."""
        rays = _cuda(rays).contiguous()
        N = rays.shape[0]
        res = torch.zeros(M, dtype=torch.int32, device=rays.device)
        call("n2m_flatten_rays", ptr(rays), N, int(M), ptr(res), stream())
        return res


flatten_rays = _flatten_rays.apply


# ----------------------------------------------------------------------------------------------
# train
# ----------------------------------------------------------------------------------------------


# (t, dt) slab of the two-call march protocol: N * max_steps float2.  Allocated per call through torch's caching allocator (so that
# concurrent callers on different streams never share it) and only while it stays below this budget -- with --adaptive_num_rays N can
# reach 10^5-10^6 rays; beyond the budget the native side re-walks the rays in the second call instead (k_march_train_rewalk).
SLAB_BUDGET_BYTES = 512 << 20


def _tbuf(device, n_floats):
    if n_floats * 4 > SLAB_BUDGET_BYTES:
        return None
    return torch.empty(n_floats, dtype=torch.float32, device=device)


class _march_rays_train(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, rays_o, rays_d, bound, contract, density_bitfield, C, H, nears, fars,
                perturb=False, dt_gamma=0, max_steps=1024):
        """Occupancy-grid marching for training (raymarching.py:181-245).

        Returns xyzs [M,3], dirs [M,3] (unnormalised), ts [M,2] = (t after the step, dt),
        rays int32 [N,2] = (offset, count).  One device->host sync for M, like the reference.
        """
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        density_bitfield = _cuda(density_bitfield).contiguous()
        nears = _cuda(nears).float().contiguous()
        fars = _cuda(fars).float().contiguous()
        N = rays_o.shape[0]
        dev = rays_o.device

        counter = torch.zeros(1, dtype=torch.int32, device=dev)
        if perturb:
            noises = torch.rand(N, dtype=torch.float32, device=dev)
        else:
            noises = torch.zeros(N, dtype=torch.float32, device=dev)
        rays = torch.empty(N, 2, dtype=torch.int32, device=dev)
        tbuf = _tbuf(dev, max(N, 1) * int(max_steps) * 2)

        args = (ptr(rays_o), ptr(rays_d), ptr(density_bitfield), float(bound), int(bool(contract)),
                float(dt_gamma), int(max_steps), N, int(C), int(H), ptr(nears), ptr(fars))
        # pass 1: count + (t, dt) slab + deterministic offsets
        call("n2m_march_rays_train", *args, None, None, None, ptr(rays), ptr(counter), ptr(noises),
             ptr(tbuf), stream())
        M = int(counter.item())

        xyzs = torch.zeros(M, 3, dtype=torch.float32, device=dev)
        dirs = torch.zeros(M, 3, dtype=torch.float32, device=dev)
        ts = torch.zeros(M, 2, dtype=torch.float32, device=dev)
        # pass 2: parallel regeneration of the samples from the slab
        if M > 0:
            call("n2m_march_rays_train", *args, ptr(xyzs), ptr(dirs), ptr(ts), ptr(rays), ptr(counter),
                 ptr(noises), ptr(tbuf), stream())
        return xyzs, dirs, ts, rays


march_rays_train = _march_rays_train.apply


class _composite_rays_train(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, sigmas, rgbs, ts, rays, T_thresh=1e-4, alpha_mode=False):
        """Front-to-back compositing with early termination (raymarching.py:248-283).

        Returns weights [M], weights_sum [N], depth [N], image [N,3]."""
        sigmas = sigmas.float().contiguous()
        rgbs = rgbs.float().contiguous()
        ts = ts.float().contiguous()
        rays = rays.contiguous()
        M, N = sigmas.shape[0], rays.shape[0]
        dev = sigmas.device
        weights = torch.zeros(M, dtype=torch.float32, device=dev)     # tails past the break stay 0
        weights_sum = torch.empty(N, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        image = torch.empty(N, 3, dtype=torch.float32, device=dev)
        call("n2m_composite_rays_train_forward", ptr(sigmas), ptr(rgbs), ptr(ts), ptr(rays), M, N,
             float(T_thresh), int(bool(alpha_mode)), ptr(weights), ptr(weights_sum), ptr(depth),
             ptr(image), stream())
        ctx.save_for_backward(sigmas, rgbs, ts, rays, weights_sum, depth, image)
        ctx.dims = (M, N, float(T_thresh), bool(alpha_mode))
        return weights, weights_sum, depth, image

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, grad_weights, grad_weights_sum, grad_depth, grad_image):
        sigmas, rgbs, ts, rays, weights_sum, depth, image = ctx.saved_tensors
        M, N, T_thresh, alpha_mode = ctx.dims
        grad_weights = grad_weights.float().contiguous()
        grad_weights_sum = grad_weights_sum.float().contiguous()
        grad_depth = grad_depth.float().contiguous()
        grad_image = grad_image.float().contiguous()
        grad_sigmas = torch.zeros_like(sigmas)
        grad_rgbs = torch.zeros_like(rgbs)
        call("n2m_composite_rays_train_backward", ptr(grad_weights), ptr(grad_weights_sum),
             ptr(grad_depth), ptr(grad_image), ptr(sigmas), ptr(rgbs), ptr(ts), ptr(rays),
             ptr(weights_sum), ptr(depth), ptr(image), M, N, T_thresh, int(alpha_mode),
             ptr(grad_sigmas), ptr(grad_rgbs), stream())
        return grad_sigmas, grad_rgbs, None, None, None, None


composite_rays_train = _composite_rays_train.apply


# ----------------------------------------------------------------------------------------------
# inference
# ----------------------------------------------------------------------------------------------
class _march_rays(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, contract,
                density_bitfield, C, H, near, far, perturb=False, dt_gamma=0, max_steps=1024):
        """March every alive ray for at most n_step samples (raymarching.py:311-359).

        Returns xyzs/dirs [n_alive*n_step,3], ts [n_alive*n_step,2], zero where a ray ran out."""
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        dev = rays_o.device
        M = int(n_alive) * int(n_step)
        xyzs = torch.zeros(M, 3, dtype=torch.float32, device=dev)
        dirs = torch.zeros(M, 3, dtype=torch.float32, device=dev)
        ts = torch.zeros(M, 2, dtype=torch.float32, device=dev)
        if perturb:
            noises = torch.rand(n_alive, dtype=torch.float32, device=dev)
        else:
            noises = torch.zeros(n_alive, dtype=torch.float32, device=dev)
        call("n2m_march_rays", int(n_alive), int(n_step), ptr(rays_alive), ptr(rays_t), ptr(rays_o),
             ptr(rays_d), float(bound), int(bool(contract)), float(dt_gamma), int(max_steps), int(C),
             int(H), ptr(density_bitfield), ptr(near), ptr(far), ptr(xyzs), ptr(dirs), ptr(ts),
             ptr(noises), stream())
        return xyzs, dirs, ts


march_rays = _march_rays.apply


class _composite_rays(Function):
    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, n_alive, n_step, rays_alive, rays_t, sigmas, rgbs, ts, weights_sum, depth, image,
                T_thresh=1e-2, alpha_mode=False):
        """Accumulate one slab into weights_sum/depth/image in place; dead rays get
        rays_alive[n] = -1 (raymarching.py:362-386).  Returns ()."""
        sigmas = sigmas.float().contiguous()
        rgbs = rgbs.float().contiguous()
        call("n2m_composite_rays", int(n_alive), int(n_step), float(T_thresh), int(bool(alpha_mode)),
             ptr(rays_alive), ptr(rays_t), ptr(sigmas), ptr(rgbs), ptr(ts), ptr(weights_sum),
             ptr(depth), ptr(image), stream())
        return tuple()


composite_rays = _composite_rays.apply
