"""Stage-1 mesh operators with the call surface of `nvdiffrast.torch` as the reference uses it (nerf/renderer.py:126-128, 856-901):

    glctx = RasterizeCudaContext()
    rast, rast_db = rasterize(glctx, pos, tri, (h, w))          # pos [1,V,4] clip space, tri [F,3] int32 -> rast [1,h,w,4]
    out, out_db   = interpolate(attr, rast, tri)                 # attr [1,V,A] -> [1,h,w,A], differentiable w.r.t. attr and rast
    img           = antialias(color, rast, pos, tri, pos_gradient_boost=1.0)   # color [1,h,w,C]; differentiable w.r.t. color and pos

over the sm_90a kernels of csrc/raster.cu and csrc/antialias.cu (C ABI: include/n2m_b200_raster.h).
`rast[..., :] = (u, v, z/w, triangle_id + 1)`.
`rasterize` and `interpolate` are differentiable as nvdiffrast's are: the gradient of interpolate w.r.t. rast's (u, v) goes on
through rasterize's (u, v) gradient to pos (clip x, y, w; z/w and the triangle id carry none).  rast stays a plain tensor: interpolate
applies both steps of that chain rule in its backward, for a rast that rasterize made from a pos that requires grad.  That is the path of the reference's
--enable_offset_nerf_grad (renderer.py:877-879: `xyzs` not detached); in its default composition the only differentiable use of rast is
interpolate(ones) for the mask, whose (u, v) gradient is exactly zero.
Not provided: image-space derivative outputs (`rast_db`, `out_db` are None: the reference ignores them, renderer.py:860-863).
No CPU fallback: tensors must live on a CUDA device.
"""
import torch

from . import _lib
from ._lib import F, P, U, call, ptr, stream

_lib.register({
    "n2m_rasterize": [P, U, P, U, U, U, P, P, P, P],
    "n2m_interpolate_forward": [P, U, U, P, P, U, P, P],
    "n2m_interpolate_backward": [P, P, P, U, U, U, P, P],
    "n2m_interpolate_backward_rast": [P, P, P, P, U, U, P, P],
    "n2m_rasterize_backward": [P, U, P, P, P, U, U, P, P],
    "n2m_compact_covered": [P, P, P, U, U, P, P, P, P, P],
    "n2m_antialias_topology": [P, U, P, P, U, P],
    "n2m_antialias_forward": [P, P, P, P, P, P, U, U, U, U, P, P],
    "n2m_antialias_backward": [P, P, P, P, P, P, U, U, U, U, P, F, P, P, P],
})
_lib.lib.n2m_antialias_topology_slots.argtypes = [U]
_lib.lib.n2m_antialias_topology_slots.restype = U


class RasterizeCudaContext:
    """Scratch owner (visibility buffer + large-triangle queue), the counterpart of dr.RasterizeCudaContext / RasterizeGLContext."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self._vis = None
        self._queue = None

    def scratch(self, num_pixels, num_tris):
        if self._vis is None or self._vis.numel() < num_pixels:
            self._vis = torch.empty(num_pixels, dtype=torch.int64, device=self.device)
        if self._queue is None or self._queue.numel() < num_tris + 1:
            self._queue = torch.empty(num_tris + 1, dtype=torch.int32, device=self.device)
        return self._vis, self._queue


RasterizeGLContext = RasterizeCudaContext        # the reference picks either (renderer.py:126-128); both map to the CUDA kernels


def rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    """dr.rasterize: pos [1,V,4] float32 clip space (or [V,4]), tri [F,3] int32, resolution (h, w) -> (rast [1,h,w,4], None).
    Differentiable w.r.t. pos through the (u, v) channels of rast, as nvdiffrast is, with the gradient applied where the reference
    differentiates rast: `interpolate` (see _Interpolate).  rast itself is a plain tensor that can be read as data."""
    if ranges is not None:
        raise NotImplementedError("range mode is not used by the reference")
    if not pos.is_cuda:
        raise RuntimeError("rasterize: pos must be a CUDA tensor (nerf2mesh_b200 has no CPU path)")
    if pos.dim() == 3:
        if pos.shape[0] != 1:
            raise NotImplementedError("instanced mode with minibatch > 1 is not used by the reference")
        pos = pos[0]
    pos_g = pos.float().contiguous()
    pos = pos_g.detach()
    tri = tri.int().contiguous()
    h, w = int(resolution[0]), int(resolution[1])
    vis, queue = glctx.scratch(h * w, tri.shape[0])
    rast = torch.empty(1, h, w, 4, device=pos.device, dtype=torch.float32)
    call("n2m_rasterize", ptr(pos), pos.shape[0], ptr(tri), tri.shape[0], h, w, ptr(vis), ptr(queue), ptr(rast), stream())
    if pos_g.requires_grad and torch.is_grad_enabled():
        rast._n2m_raster_src = (pos_g, tri)          # the (u, v) of rast are a function of pos: interpolate differentiates through them
    return rast, None


class _Interpolate(torch.autograd.Function):
    """out = interpolate(attr, rast); pos (optional) is the clip-space input rast was rasterized from: the gradient w.r.t. rast's (u, v)
    (n2m_interpolate_backward_rast) goes on through dr.rasterize's backward (n2m_rasterize_backward) to pos -- the chain rule through rast
    evaluated inside one node, so that rast stays a plain tensor"""

    @staticmethod
    def forward(ctx, attr, rast, tri, pos, raster_tri):
        V, A = attr.shape
        n = rast.shape[0] * rast.shape[1] * rast.shape[2]
        out = torch.empty(*rast.shape[:3], A, device=attr.device, dtype=torch.float32)
        call("n2m_interpolate_forward", ptr(attr), V, A, ptr(rast), ptr(tri), n, ptr(out), stream())
        ctx.save_for_backward(attr, rast, tri, pos, raster_tri)
        ctx.dims = (V, A, n)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        attr, rast, tri, pos, raster_tri = ctx.saved_tensors
        V, A, n = ctx.dims
        grad_out = grad_out.float().contiguous()
        g = gp = None
        if ctx.needs_input_grad[0]:
            g = torch.zeros(V, A, device=grad_out.device, dtype=torch.float32)
            call("n2m_interpolate_backward", ptr(grad_out), ptr(rast), ptr(tri), n, V, A, ptr(g), stream())
        if pos is not None and ctx.needs_input_grad[3]:
            gr = torch.empty_like(rast)
            call("n2m_interpolate_backward_rast", ptr(grad_out), ptr(attr), ptr(rast), ptr(tri), n, A, ptr(gr), stream())
            gp = torch.zeros_like(pos)
            call("n2m_rasterize_backward", ptr(pos), pos.shape[0], ptr(raster_tri), ptr(rast), ptr(gr), rast.shape[1], rast.shape[2], ptr(gp),
                 stream())
        return g, None, None, gp, None


def interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
    """dr.interpolate: attr [1,V,A] (or [V,A]) float32, rast [1,h,w,4], tri [F,3] -> (out [1,h,w,A], None)."""
    if not attr.is_cuda:
        raise RuntimeError("interpolate: attr must be a CUDA tensor")
    a = attr[0] if attr.dim() == 3 else attr
    if a.shape[-1] < 1 or a.shape[-1] > 4:
        raise RuntimeError("interpolate: 1..4 attributes per vertex are supported")
    src = getattr(rast, "_n2m_raster_src", None)
    pos, raster_tri = src if src is not None else (None, None)
    out = _Interpolate.apply(a.float().contiguous(), rast.contiguous(), tri.int().contiguous(), pos, raster_tri)
    return out, None


class TopologyHash:
    """Edge -> opposing-vertex hash of a triangle mesh (dr.antialias_construct_topology_hash): keys [slots] int64, opp [slots,2] int32."""

    def __init__(self, tri):
        tri = tri.int().contiguous()
        if not tri.is_cuda:
            raise RuntimeError("antialias: tri must be a CUDA tensor")
        self.slots = int(_lib.lib.n2m_antialias_topology_slots(tri.shape[0]))
        self.keys = torch.empty(self.slots, dtype=torch.int64, device=tri.device)
        self.opp = torch.empty(self.slots, 2, dtype=torch.int32, device=tri.device)
        call("n2m_antialias_topology", ptr(tri), tri.shape[0], ptr(self.keys), ptr(self.opp), self.slots, stream())
        self.tri = tri                   # keeps the indexed storage alive: its address cannot be reused while this hash is cached


def antialias_construct_topology_hash(tri):
    return TopologyHash(tri)


_topology_cache = {}


def _topology_for(tri):
    """one cached hash per int32 triangle tensor (the reference's mesh changes only at re-meshing; the library caches the same way);
    tensors that had to be converted are temporaries whose address may be recycled: their hash is built per call"""
    if tri.dtype != torch.int32 or not tri.is_contiguous():
        return TopologyHash(tri)
    key = (tri.data_ptr(), tuple(tri.shape), tri._version, tri.device.index)
    th = _topology_cache.get(key)
    if th is None:
        if len(_topology_cache) >= 4:
            _topology_cache.clear()
        th = _topology_cache[key] = TopologyHash(tri)
    return th


class _Antialias(torch.autograd.Function):
    @staticmethod
    def forward(ctx, color, rast, pos, tri, th, boost):
        n, h, w, C = color.shape
        out = torch.empty_like(color)
        call("n2m_antialias_forward", ptr(color), ptr(rast), ptr(pos), ptr(tri), ptr(th.keys), ptr(th.opp), th.slots, h, w, C, ptr(out), stream())
        ctx.save_for_backward(color, rast, pos, tri)
        ctx.th, ctx.boost = th, float(boost)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        color, rast, pos, tri = ctx.saved_tensors
        th = ctx.th
        n, h, w, C = color.shape
        grad_out = grad_out.float().contiguous()
        need_c, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        gc = torch.empty_like(color) if need_c else None
        gp = torch.zeros_like(pos) if need_p else None
        if need_c or need_p:
            call("n2m_antialias_backward", ptr(color), ptr(rast), ptr(pos), ptr(tri), ptr(th.keys), ptr(th.opp), th.slots, h, w, C,
                 ptr(grad_out), ctx.boost, ptr(gc), ptr(gp), stream())
        return gc, None, gp, None, None, None


def antialias(color, rast, pos, tri, topology_hash=None, pos_gradient_boost=1.0):
    """dr.antialias: color [1,h,w,C] (C = 1..4), rast [1,h,w,4], pos [1,V,4] (or [V,4]) clip space, tri [F,3] int32 -> [1,h,w,C];
    differentiable w.r.t. color and pos (clip-space x, y, w of the silhouette edges' vertices)."""
    if not (color.is_cuda and rast.is_cuda and pos.is_cuda):
        raise RuntimeError("antialias: tensors must live on a CUDA device (nerf2mesh_b200 has no CPU path)")
    if color.dim() != 4 or color.shape[0] != 1 or color.shape[:3] != rast.shape[:3]:
        raise RuntimeError("antialias: color must be [1,h,w,C] with the resolution of rast")
    if not 1 <= color.shape[-1] <= 4:
        raise RuntimeError("antialias: 1..4 channels are supported")
    squeeze = pos.dim() == 2
    p = pos if squeeze else pos[0]
    th = topology_hash if topology_hash is not None else _topology_for(tri)
    tri = th.tri
    out = _Antialias.apply(color.float().contiguous(), rast.contiguous(), p.float().contiguous(), tri, th, pos_gradient_boost)
    return out


def compact_covered(rast, xyz, dirs, cap=None):
    """Covered pixels of `rast` ([1,h,w,4]) with their interpolated positions `xyz` [h*w,3] and view directions `dirs` [h*w,3]:
    -> (count [1] int32 on the device, pixel index [cap] int32, points [cap,3], dirs [cap,3]); no host synchronisation."""
    n = rast.shape[1] * rast.shape[2]
    cap = int(cap or n)
    dev = rast.device
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    pix = torch.empty(cap, dtype=torch.int32, device=dev)
    pts = torch.zeros(cap, 3, device=dev); pd = torch.zeros(cap, 3, device=dev)
    call("n2m_compact_covered", ptr(rast), ptr(xyz.contiguous()), ptr(dirs.contiguous()), n, cap, ptr(counter), ptr(pix), ptr(pts), ptr(pd), stream())
    return counter, pix, pts, pd
