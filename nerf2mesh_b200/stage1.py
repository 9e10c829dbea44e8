"""Stage-1 texture step: host side of csrc/raster.cu + csrc/stage1.cu (C ABI include/n2m_b200_raster.h).

`Stage1Trainer` is the fused equivalent of one stage-1 iteration of the reference restricted to the appearance model
(NeRFRenderer.render_stage1, nerf/renderer.py:806-935; Trainer.train_step stage-1 branch, nerf/utils.py:703-716;
the optimizer step of utils.py:1163-1177): rasterize the mesh at ssaa x the image resolution, evaluate the colour
MLPs (`self.rgb`, network.py:170-189) on the covered pixels with the tensor-core kernels of stage 0, average the
super-samples, mix the background, MSE loss, backward into color_net / specular_net / encoder_color, Adam.  It shares
the model state (hash tables, MLP weights, optimizer moments, GradScaler state) with a Stage0Trainer.

`antialias=True` inserts dr.antialias on (rgbs, alphas) as the reference does (renderer.py:886-887; csrc/antialias.cu) and leaves the
image-loss gradient w.r.t. the vertices in `vertex_gradient()` -- the quantity the reference's vertex optimizer consumes.
`lr_vert > 0` also trains the vertex offsets as the reference's default stage 1 does (`vertices_offsets`, renderer.py:160,180: an Adam
group with lr_vert; regularisers lambda_lap * laplacian_smooth_loss (uniform) + lambda_offsets * mean(sum(offsets^2)), utils.py:750-779).
Not built: re-meshing (`refine_and_decimate`, CPU mesh libraries) and the pytorch3d regularisers that are off by
default (lambda_normal, lambda_edgelen).
"""
import ctypes

import torch

from . import _lib
from ._lib import F, I, P, U, call, ptr, stream
from . import raster as dr
from . import texture  # noqa: F401  (the stage-1 export, texture.export_stage1; binds include/n2m_b200_texture.h)

_lib.register({
    "n2m_s1_points": [P, P, P, P, U, U, U, U, P, P, P, P, P, P],
    "n2m_s1_loss": [P, P, P, U, P, U, U, U, F, P, P, P, P, P, P],
    "n2m_s1_rgba": [P, P, U, P, P],
    "n2m_s1_loss_aa": [P, P, U, P, U, U, U, F, P, P, P, P, P, P],
    "n2m_s1_dout": [P, P, U, P, P],
    "n2m_s1_vert_check": [P, U, P, P],
    "n2m_s1_vert_step": [P, P, P, U, P, P, P, P, P, P, P, U, F, F, F, F, P, P, P, P],
})


class Stage1Trainer:
    def __init__(self, t0, vertices, triangles, h0, w0, ssaa=2, max_points=None, lambda_mask=0.1, antialias=False, pos_gradient_boost=1.0,
                 lr_vert=0.0, lambda_lap=0.001, lambda_offsets=0.1):
        assert ssaa in (1, 2), "the ssaa average equals the reference's bilinear down-scale only at factors 1 and 2"
        self.t0 = t0
        dev = t0.device
        self.vertices = vertices.to(dev, torch.float32).contiguous()
        self.triangles = triangles.to(dev, torch.int32).contiguous()
        self.h0, self.w0, self.ssaa = int(h0), int(w0), int(ssaa)
        self.h, self.w = self.h0 * ssaa, self.w0 * ssaa
        n = self.h * self.w
        self.cap = ((int(max_points) if max_points else n) + 127) // 128 * 128
        self.lambda_mask = float(lambda_mask)
        self.glctx = dr.RasterizeCudaContext(dev)
        self.inv = torch.empty(n, dtype=torch.int32, device=dev)
        self.pts = torch.zeros(self.cap, 3, device=dev); self.pdirs = torch.zeros(self.cap, 3, device=dev)
        self.recs = torch.zeros(self.cap, 4, device=dev)
        self.counters = torch.zeros(16, dtype=torch.int32, device=dev)
        self.enc_tiles = torch.zeros(self.cap * 64, dtype=torch.float16, device=dev)
        self.denc_tiles = torch.zeros(self.cap * 64, dtype=torch.float16, device=dev)
        self.out = torch.zeros(self.cap, 4, device=dev); self.dout = torch.zeros(self.cap, 4, device=dev)
        Q = self.h0 * self.w0
        self.image = torch.zeros(Q, 3, device=dev); self.weights_sum = torch.zeros(Q, device=dev)
        self.loss_acc = torch.zeros(4, device=dev)
        self.rast = None
        self.antialias = bool(antialias)
        self.pos_gradient_boost = float(pos_gradient_boost)
        if self.antialias:
            self.topology = dr.TopologyHash(self.triangles)               # once per mesh
            self.rgba = torch.zeros(n, 4, device=dev); self.aa = torch.zeros(n, 4, device=dev)
            self.d_aa = torch.zeros(n, 4, device=dev); self.g_rgba = torch.zeros(n, 4, device=dev)
            self.grad_vclip = torch.zeros(self.vertices.shape[0], 4, device=dev)
        self.vclip = None
        self.mvp = None
        self._graphs, self._warm = {}, False
        # vertex offsets (main.py:49,84-85 defaults: lr_vert 1e-4, lambda_lap 1e-3, lambda_offsets 0.1); 0 = vertices fixed
        self.lr_vert, self.lambda_lap, self.lambda_offsets = float(lr_vert), float(lambda_lap), float(lambda_offsets)
        if self.lr_vert > 0:
            if not self.antialias:
                raise ValueError("the image loss reaches the vertices through dr.antialias only: lr_vert > 0 needs antialias=True")
            V = self.vertices.shape[0]
            self.base_vertices = self.vertices.clone()
            self.offsets = torch.zeros(V, 3, device=dev)
            self.m_vert = torch.zeros(V, 3, device=dev); self.v_vert = torch.zeros(V, 3, device=dev)
            self.vert_state = torch.zeros(4, device=dev)                  # [0] Adam step count of this group, [1] current lr_vert
            self.vert_scratch = torch.zeros(6 * V, device=dev)
            self.grad_offsets = torch.zeros(V, 3, device=dev)             # total gradient of the last step (diagnostic / tests)
        # the specular regulariser and TV are stage-0 losses (utils.py:726,735-738)
        self.params = t0.params_with(lambda_specular=0.0, lambda_tv=0.0)

    def _pp(self):
        return ctypes.byref(self.params)

    def forward(self, mvp, rays_d, shading="full"):
        """rasterize -> surface points -> colour MLPs; leaves per-point colours in `out`, the pixel -> point map in `inv`."""
        t0 = self.t0
        self.params.shading_full = int(shading == "full")
        mvp = mvp.to(t0.device, torch.float32).contiguous()
        vclip = (torch.nn.functional.pad(self.vertices, (0, 1), value=1.0) @ mvp.T).contiguous()           # renderer.py:858
        self.vclip, self.mvp = vclip, mvp
        self.rast, _ = dr.rasterize(self.glctx, vclip[None], self.triangles, (self.h, self.w))
        call("n2m_s1_points", ptr(self.rast), ptr(self.vertices), ptr(self.triangles), ptr(rays_d), self.h, self.w, self.ssaa, self.cap,
             ptr(self.counters), ptr(self.inv), ptr(self.pts), ptr(self.pdirs), ptr(self.recs), stream())
        call("n2m_s0_encode_points", self._pp(), ptr(self.pts), ptr(self.pdirs), ptr(self.counters), self.cap, ptr(t0.table),
             ptr(t0.offsets), ptr(self.enc_tiles), stream())
        call("n2m_s0_mlp_fwd", self._pp(), ptr(self.enc_tiles), ptr(self.counters), self.cap, ptr(t0.wpack), ptr(self.out), None, 0, 1,
             stream())
        if self.antialias:
            n = self.h * self.w
            th = self.topology
            call("n2m_s1_rgba", ptr(self.out), ptr(self.inv), n, ptr(self.rgba), stream())
            call("n2m_antialias_forward", ptr(self.rgba), ptr(self.rast), ptr(self.vclip), ptr(self.triangles), ptr(th.keys), ptr(th.opp),
                 th.slots, self.h, self.w, 4, ptr(self.aa), stream())

    def loss_backward(self, gt, bg):
        t0 = self.t0
        self.loss_acc.zero_()
        if self.antialias:
            n = self.h * self.w
            th = self.topology
            call("n2m_s1_loss_aa", ptr(self.aa), ptr(gt), gt.shape[-1], ptr(bg), self.h0, self.w0, self.ssaa, self.lambda_mask,
                 ptr(t0.opt_state), ptr(self.d_aa), ptr(self.image), ptr(self.weights_sum), ptr(self.loss_acc), stream())
            self.grad_vclip.zero_()
            call("n2m_antialias_backward", ptr(self.rgba), ptr(self.rast), ptr(self.vclip), ptr(self.triangles), ptr(th.keys), ptr(th.opp),
                 th.slots, self.h, self.w, 4, ptr(self.d_aa), self.pos_gradient_boost, ptr(self.g_rgba), ptr(self.grad_vclip), stream())
            call("n2m_s1_dout", ptr(self.g_rgba), ptr(self.inv), n, ptr(self.dout), stream())
        else:
            call("n2m_s1_loss", ptr(self.out), ptr(self.inv), ptr(gt), gt.shape[-1], ptr(bg), self.h0, self.w0, self.ssaa, self.lambda_mask,
                 ptr(t0.opt_state), ptr(self.dout), ptr(self.image), ptr(self.weights_sum), ptr(self.loss_acc), stream())
        call("n2m_s0_mlp_bwd", self._pp(), ptr(self.enc_tiles), ptr(self.dout), ptr(self.counters), self.cap, ptr(t0.wpack),
             ptr(self.denc_tiles), ptr(t0.g_mlp), ptr(t0.opt_state), 0, 1, stream())
        call("n2m_s0_encode_bwd", self._pp(), ptr(self.recs), ptr(self.counters), self.cap, ptr(self.pts), ptr(self.pdirs),
             ptr(self.denc_tiles), ptr(t0.table), ptr(t0.offsets), ptr(t0.gtables[t0.parity]), ptr(t0.opt_state), 0, 1, stream())

    def step(self, mvp, rays_d, gt, bg, shading="full", lr=None, use_graph=False):
        """One optimizer step on one view: mvp [4,4], rays_d [h0*w0,3] (unnormalised), gt [h0*w0, 3 or 4], bg [h0*w0,3].
        `use_graph`: the step is captured once per view (keyed by the addresses of its device-resident tensors, which must then stay
        valid and in place -- the dataset of a stage-1 run is a fixed set of views) and replayed as one CUDA graph: ~17 launches and a
        handful of torch ops leave the host's critical path (the eager step is host-bound at this size)."""
        t0 = self.t0
        if lr is not None:
            t0.opt_state[4:5].fill_(float(lr))
        rays_d, gt, bg = rays_d.contiguous(), gt.contiguous(), bg.contiguous()
        if self.lr_vert > 0:
            self.vert_state[1:2].fill_(self.lr_vert)
        if not use_graph or not self._warm:
            self._step_body(mvp, rays_d, gt, bg, shading)
            self._warm = True                         # lazily created buffers / streams exist now: later steps may be captured
        else:
            if not (mvp.is_cuda and mvp.dtype == torch.float32 and mvp.is_contiguous()):
                raise RuntimeError("use_graph: mvp must be a contiguous float32 CUDA tensor that stays in place (the graph is keyed by its address)")
            key = (mvp.data_ptr(), rays_d.data_ptr(), gt.data_ptr(), bg.data_ptr(), int(gt.shape[-1]), shading, int(t0.parity))
            g = self._graphs.get(key)
            if g is None:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._step_body(mvp, rays_d, gt, bg, shading)
                self._graphs[key] = (g, mvp, rays_d, gt, bg)          # keeps the captured addresses alive
                g = self._graphs[key]
            g[0].replay()
        t0.global_step += 1

    def _step_body(self, mvp, rays_d, gt, bg, shading):
        self.forward(mvp, rays_d, shading)
        self.loss_backward(gt, bg)
        if self.lr_vert > 0:
            call("n2m_s1_vert_check", ptr(self.grad_vclip), self.vertices.shape[0], ptr(self.t0.opt_state), stream())
            self.t0.adam(between=self._vertex_step)
        else:
            self.t0.adam()

    def _vertex_step(self):
        """the `vertices_offsets` group of the optimizer step: regularisers (evaluated on the offsets before the update, as autograd does),
        Adam, vertices = base + offsets"""
        V = self.vertices.shape[0]
        th = self.topology
        if self.lambda_offsets > 0:
            self.loss_acc[0:1].add_(self.lambda_offsets * (self.offsets * self.offsets).sum(1).mean())          # utils.py:764-776
        call("n2m_s1_vert_step", ptr(self.grad_vclip), ptr(self.mvp), ptr(th.keys), th.slots, ptr(self.base_vertices), ptr(self.offsets),
             ptr(self.m_vert), ptr(self.v_vert), ptr(self.vertices), ptr(self.vert_scratch), ptr(self.grad_offsets), V, self.lambda_lap,
             self.lambda_offsets, -1.0, self.t0.cfg.eps, ptr(self.t0.opt_state), ptr(self.vert_state), ptr(self.loss_acc), stream())

    def vertex_gradient(self):
        """d loss / d vertices [V,3] of the last `loss_backward` (through dr.antialias and the projection of renderer.py:858; the
        gradient the reference accumulates on `vertices_offsets`), unscaled.  Valid when the step's found_inf flag is clear."""
        if not self.antialias:
            raise RuntimeError("vertex gradients flow through dr.antialias only: construct Stage1Trainer(antialias=True)")
        return (self.grad_vclip @ self.mvp[:, :3]) / self.t0.opt_state[0]

    def read_loss(self):
        return float(self.loss_acc[0].item())
