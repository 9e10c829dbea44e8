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
`offset_nerf_grad=True` (needs lr_vert > 0) is the reference's --enable_offset_nerf_grad (renderer.py:877-879; main.py:62, on whenever
--sdf is set, main.py:149): the surface points are not detached, so the image loss also reaches the vertices through the colour field --
the colour-net and colour-grid input gradient of every covered super-sample, through contract() in unbounded scenes, then
dr.interpolate and dr.rasterize's (u, v) (n2m_s1_offset_grad, after the MLP backward).  `vertex_gradient()` is then the sum of both paths.
`refine=True` adds the error-guided mesh refinement of the reference's stage 1 (opt.refine, main.py:129-136): every step also adds each
low-res pixel's loss and a hit to the face that pixel sees (update_triangles_errors, renderer.py:893-903,923-943, fused into the loss
kernels) in `face_errors` / `face_counts`; `refine_mask()` turns them into the decimate / refine face mask of refine_and_decimate
(renderer.py:217-240), and after the caller re-meshes on the CPU (decimate_and_refine_mesh, pymeshlab) `replace_mesh()` restarts the step on
the new mesh (renderer.py:287-292, utils.py:1209-1210).

Unbounded scenes (bound > 1): `vertices` / `triangles` may be equal-length lists of per-cascade meshes (mesh.load_stage0_meshes), which the
trainer concatenates with index offsets as the reference does (renderer.py:130-157, `v_cumsum` / `f_cumsum`); every kernel of the step then
runs on the concatenated mesh, and `cascade_mesh(cas)` returns one cascade for the export.  Refinement looks at cascade 0 only
(renderer.py:223-225) and `replace_mesh` replaces cascade 0, rebasing the outer cascades on their current vertices (:258-285).  With
Stage0Config(contract=True) the surface points are contracted before the colour field is queried (n2m_s1_points_contract).
`render()` is render_stage1 at inference (eval_step / test_step, utils.py:853,882): the forward part of the step on buffers of its own, then
n2m_s1_render_compose -> image, weights_sum, depth, in shading 'diffuse', 'specular' or 'full'.
`lambda_normal` / `lambda_edgelen` (need lr_vert > 0) add the reference's two pytorch3d regularisers of the vertex-offset group
(utils.py:759-769): lambda_normal * mesh_normal_consistency + lambda_edgelen * mesh_edge_loss over the concatenated mesh of all cascades,
one walk over the edge hash per step (n2m_s1_vert_step_reg).  The normal term needs a mesh without non-manifold edges (the reference
repairs them before stage 1 and after every re-mesh, meshutils.py:172-175,211-214), and both need faces of three distinct vertices: such
meshes raise ValueError at construction and in replace_mesh.  Not built: SDF mode's all-ones refinement mask.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import F, I, P, U, call, ptr, stream
from . import raster as dr
from . import texture  # noqa: F401  (the stage-1 export, texture.export_stage1; binds include/n2m_b200_texture.h)

_lib.register({
    "n2m_s1_points": [P, P, P, P, U, U, U, U, P, P, P, P, P, P],
    "n2m_s1_points_contract": [P, P, P, P, U, U, U, U, P, P, P, P, P, U, P],
    "n2m_s1_loss": [P, P, P, U, P, U, U, U, F, P, P, P, P, P, P],
    "n2m_s1_rgba": [P, P, U, P, P],
    "n2m_s1_loss_aa": [P, P, U, P, U, U, U, F, P, P, P, P, P, P],
    "n2m_s1_loss_err": [P, P, P, U, P, U, U, U, F, P, P, P, P, P, P, P, P, U, P],
    "n2m_s1_loss_aa_err": [P, P, U, P, U, U, U, F, P, P, P, P, P, P, P, P, U, P],
    "n2m_s1_dout": [P, P, U, P, P],
    "n2m_s1_vert_check": [P, U, P, P],
    "n2m_s1_vert_step": [P, P, P, U, P, P, P, P, P, P, P, U, F, F, F, F, P, P, P, P],
    "n2m_s1_offset_grad": [P, P, P, P, P, P, U, U, P, P, P, P, P, P, P, P],
    "n2m_s1_vert_step_world": [P, P, P, P, U, P, P, P, P, P, P, P, U, F, F, F, F, P, P, P, P],
    "n2m_s1_render_compose": [P, P, P, U, U, U, P, P, P, P],
    "n2m_s1_mesh_reg_setup": [P, U, P, U, P, P, P],
    "n2m_s1_mesh_reg": [P, P, U, U, U, P, F, F, P, P, P],
    "n2m_s1_vert_step_reg": [P, P, P, P, P, U, U, U, P, P, P, P, P, P, P, U, F, F, F, F, F, F, P, P, P, P],
})

# shading -> n2m_s0_params.shading_full of the forward MLP launch ('specular': the specular term alone, evaluation only)
SHADING_MODES = {"diffuse": 0, "full": 1, "specular": 2}


def bg_image(bg_color, q, device):
    """bg_color (a scalar, or a tensor [q,3]) as the contiguous float32 [q,3] device tensor the compose kernel reads"""
    if torch.is_tensor(bg_color):
        bg = bg_color.to(device, torch.float32).reshape(-1, 3).contiguous()
        if bg.shape[0] != q:
            raise ValueError(f"bg_color: {bg.shape[0]} rows for {q} pixels")
        return bg
    return torch.full((q, 3), float(bg_color), device=device)


class Stage1Trainer:
    v_cumsum = f_cumsum = ()            # per-cascade vertex / face offsets, set by _set_cascades

    _index = 0                  # appearance-code row of the current step's view (t0.ind_dim > 0)

    def __init__(self, t0, vertices, triangles, h0, w0, ssaa=2, max_points=None, lambda_mask=0.1, antialias=False, pos_gradient_boost=1.0,
                 lr_vert=0.0, lambda_lap=0.001, lambda_offsets=0.1, refine=False, offset_nerf_grad=False, lambda_normal=0.0, lambda_edgelen=0.0):
        assert ssaa in (1, 2), "the ssaa average equals the reference's bilinear down-scale only at factors 1 and 2"
        self.t0 = t0
        dev = t0.device
        self._set_cascades(*_cascade_lists(vertices, triangles))
        self.contract = bool(getattr(t0.cfg, "contract", False))
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
            self.rgba = torch.zeros(n, 4, device=dev); self.aa = torch.zeros(n, 4, device=dev)
            self.d_aa = torch.zeros(n, 4, device=dev); self.g_rgba = torch.zeros(n, 4, device=dev)
        self.vclip = None
        self.mvp = None
        self._graphs, self._warm = {}, False
        self._render_cache, self._render_th = {}, None       # render(): buffers per (h0, w0), the edge hash of a non-antialiased trainer
        # vertex offsets (main.py:49,84-85 defaults: lr_vert 1e-4, lambda_lap 1e-3, lambda_offsets 0.1); 0 = vertices fixed
        self.lr_vert, self.lambda_lap, self.lambda_offsets = float(lr_vert), float(lambda_lap), float(lambda_offsets)
        if self.lr_vert > 0:
            if not self.antialias:
                raise ValueError("the image loss reaches the vertices through dr.antialias only: lr_vert > 0 needs antialias=True")
            self.vert_state = torch.zeros(4, device=dev)                  # [0] Adam step count of this group, [1] current lr_vert
        # --enable_offset_nerf_grad (main.py:62; on with --sdf, main.py:149): the image loss also reaches the vertices through the colour field
        self.offset_nerf_grad = bool(offset_nerf_grad)
        if self.offset_nerf_grad and not self.lr_vert > 0:
            raise ValueError("offset_nerf_grad trains the vertex offsets: it needs lr_vert > 0 (and with it antialias=True)")
        # mesh regularisers of the vertex offsets (main.py:86-87, off by default; the reference's recipes use lambda_normal 1e-3 .. 1e-1)
        self.lambda_normal, self.lambda_edgelen = float(lambda_normal), float(lambda_edgelen)
        if not (self.lambda_normal >= 0 and self.lambda_edgelen >= 0):
            raise ValueError("lambda_normal and lambda_edgelen must be >= 0")
        self.mesh_reg = self.lambda_normal > 0 or self.lambda_edgelen > 0
        if self.mesh_reg and not self.lr_vert > 0:
            raise ValueError("lambda_normal / lambda_edgelen regularise the vertex offsets: they need lr_vert > 0 (and with it antialias=True)")
        self.refine = bool(refine)
        self._mesh_buffers()
        # the specular regulariser and TV are stage-0 losses (utils.py:726,735-738)
        self.params = t0.params_with(lambda_specular=0.0, lambda_tv=0.0)

    def _set_cascades(self, vertices, triangles):
        """the concatenated mesh of the per-cascade lists: faces offset by the vertices of the cascades before them; v_cumsum / f_cumsum
        (host ints) delimit cascade c as vertices[v_cumsum[c]:v_cumsum[c+1]], triangles[f_cumsum[c]:f_cumsum[c+1]].  No face links two
        cascades, so the edge hash of the antialias / Laplacian kernels never does either: both act on each cascade on its own."""
        dev = self.t0.device
        self.v_cumsum, self.f_cumsum = [0], [0]
        vs, fs = [], []
        for v, f in zip(vertices, triangles):
            off = self.v_cumsum[-1]
            vs.append(v.to(dev, torch.float32)); fs.append(f.to(dev, torch.int32) + off if off else f.to(dev, torch.int32))
            self.v_cumsum.append(self.v_cumsum[-1] + int(v.shape[0])); self.f_cumsum.append(self.f_cumsum[-1] + int(f.shape[0]))
        self.vertices = (vs[0] if len(vs) == 1 else torch.cat(vs)).contiguous()
        self.triangles = (fs[0] if len(fs) == 1 else torch.cat(fs)).contiguous()

    @property
    def cascades(self):
        return len(self.v_cumsum) - 1

    def cascade_mesh(self, cas):
        """(vertices [Vc,3], triangles [Fc,3]) of cascade `cas` as it is now (base + offsets), triangles indexing its own vertices: the mesh the
        export bakes and the one a refinement writes back as mesh_{cas}_updated.ply"""
        v0, v1 = self.v_cumsum[cas], self.v_cumsum[cas + 1]
        f0, f1 = self.f_cumsum[cas], self.f_cumsum[cas + 1]
        return self.vertices[v0:v1], self.triangles[f0:f1] - v0

    def _mesh_buffers(self):
        """(re)allocate everything sized by the mesh, for self.vertices / self.triangles: the edge hash, the clip-space vertex gradient,
        the vertex-offset group (base = vertices, zero offsets and moments), the mesh regularisers' edge / pair counts and the per-face
        error accumulators"""
        dev = self.t0.device
        V, Fn = self.vertices.shape[0], self.triangles.shape[0]
        if self.antialias:
            self.topology = dr.TopologyHash(self.triangles)               # once per mesh
            self.grad_vclip = torch.zeros(V, 4, device=dev)
        if self.mesh_reg:
            # E (unique edges) and P (edges with two faces): the means' denominators, launch constants of every step on this mesh
            self.mesh_edges, self.mesh_pairs = self._check_mesh_reg(self.topology, "Stage1Trainer")
        if self.lr_vert > 0:
            self.base_vertices = self.vertices.clone()
            self.offsets = torch.zeros(V, 3, device=dev)
            self.m_vert = torch.zeros(V, 3, device=dev); self.v_vert = torch.zeros(V, 3, device=dev)
            # [6V] the Laplacian's two [V,3] vectors, + [3V] the mesh regularisers' gradient
            self.vert_scratch = torch.zeros((9 if self.mesh_reg else 6) * V, device=dev)
            self.grad_offsets = torch.zeros(V, 3, device=dev)             # total gradient of the last step (diagnostic / tests)
        if self.offset_nerf_grad:
            self.grad_vworld = torch.zeros(V, 3, device=dev)              # colour-field path, world space, loss-scaled
        if self.refine:
            # triangles_errors / triangles_errors_cnt (renderer.py:163-164): summed per-pixel loss and pixel count per face
            self.face_errors = torch.zeros(Fn, device=dev); self.face_counts = torch.zeros(Fn, device=dev)

    def _check_mesh_reg(self, th, where):
        """(E, P) of the mesh of edge hash `th` for the mesh regularisers; ValueError for faces with a repeated vertex index (pytorch3d
        would pair such a face with itself) and, with lambda_normal > 0, for edges of three or more faces (the hash keeps two)"""
        E, P, nonmanifold, repeated = mesh_reg_counts(th)
        if repeated:
            raise ValueError(f"{where}: {repeated} faces with a repeated vertex index: lambda_normal / lambda_edgelen need faces of three "
                             "distinct vertices")
        if self.lambda_normal > 0 and nonmanifold:
            raise ValueError(f"{where}: {nonmanifold} non-manifold edges (three or more faces): lambda_normal needs a mesh without; repair "
                             "them first, as the reference does before stage 1 and after every re-mesh")
        return E, P

    def _pp(self):
        return ctypes.byref(self.params)

    def forward(self, mvp, rays_d, shading="full"):
        """rasterize -> surface points -> colour MLPs; leaves per-point colours in `out`, the pixel -> point map in `inv`."""
        t0 = self.t0
        if shading == "specular":
            raise ValueError("shading 'specular' is for render() only: the step trains with 'diffuse' or 'full'")
        self.params.shading_full = int(shading == "full")
        mvp = mvp.to(t0.device, torch.float32).contiguous()
        vclip = (torch.nn.functional.pad(self.vertices, (0, 1), value=1.0) @ mvp.T).contiguous()           # renderer.py:858
        self.vclip, self.mvp = vclip, mvp
        self.rast, _ = dr.rasterize(self.glctx, vclip[None], self.triangles, (self.h, self.w))
        pts_args = (ptr(self.rast), ptr(self.vertices), ptr(self.triangles), ptr(rays_d), self.h, self.w, self.ssaa, self.cap, ptr(self.counters),
                    ptr(self.inv), ptr(self.pts), ptr(self.pdirs), ptr(self.recs))
        if self.contract:               # the colour field of an unbounded scene is queried at contract(x) (renderer.py:25-32)
            call("n2m_s1_points_contract", *pts_args, 1, stream())
        else:
            call("n2m_s1_points", *pts_args, stream())
        t0.encode_points(self._pp(), self.pts, self.pdirs, self.counters, self.cap, self.enc_tiles, self._index)
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
        # refinement: the same loss kernels also scatter each pixel's loss into the face it sees (utils.py:720-721)
        err = (ptr(self.rast), ptr(self.face_errors), ptr(self.face_counts), self.triangles.shape[0]) if self.refine else ()
        if self.antialias:
            n = self.h * self.w
            th = self.topology
            call("n2m_s1_loss_aa_err" if self.refine else "n2m_s1_loss_aa", ptr(self.aa), ptr(gt), gt.shape[-1], ptr(bg), self.h0, self.w0,
                 self.ssaa, self.lambda_mask, ptr(t0.opt_state), ptr(self.d_aa), ptr(self.image), ptr(self.weights_sum), ptr(self.loss_acc),
                 *err, stream())
            self.grad_vclip.zero_()
            call("n2m_antialias_backward", ptr(self.rgba), ptr(self.rast), ptr(self.vclip), ptr(self.triangles), ptr(th.keys), ptr(th.opp),
                 th.slots, self.h, self.w, 4, ptr(self.d_aa), self.pos_gradient_boost, ptr(self.g_rgba), ptr(self.grad_vclip), stream())
            call("n2m_s1_dout", ptr(self.g_rgba), ptr(self.inv), n, ptr(self.dout), stream())
        else:
            call("n2m_s1_loss_err" if self.refine else "n2m_s1_loss", ptr(self.out), ptr(self.inv), ptr(gt), gt.shape[-1], ptr(bg), self.h0,
                 self.w0, self.ssaa, self.lambda_mask, ptr(t0.opt_state), ptr(self.dout), ptr(self.image), ptr(self.weights_sum),
                 ptr(self.loss_acc), *err, stream())
        if t0.ind_dim:
            # appearance codes: the view's code row (renderer.py:845-852) gets the summed input gradient of all the view's points
            call("n2m_s0_mlp_bwd_codes", self._pp(), ptr(self.enc_tiles), ptr(self.dout), ptr(self.counters), self.cap, ptr(t0.wpack),
                 ptr(self.denc_tiles), ptr(t0.g_mlp), ptr(t0.g_ind), ptr(t0.opt_state), 0, 1, stream())
            call("n2m_s0_code_grad_row", self._pp(), ptr(self.counters), self.cap, ptr(self.denc_tiles),
                 t0.g_ind.data_ptr() + 4 * t0.ind_dim * (64 + self._index), ptr(t0.opt_state), stream())
        else:
            call("n2m_s0_mlp_bwd", self._pp(), ptr(self.enc_tiles), ptr(self.dout), ptr(self.counters), self.cap, ptr(t0.wpack),
                 ptr(self.denc_tiles), ptr(t0.g_mlp), ptr(t0.opt_state), 0, 1, stream())
        call("n2m_s0_encode_bwd", self._pp(), ptr(self.recs), ptr(self.counters), self.cap, ptr(self.pts), ptr(self.pdirs),
             ptr(self.denc_tiles), ptr(t0.table), ptr(t0.offsets), ptr(t0.gtables[t0.parity]), ptr(t0.opt_state), 0, 1, stream())
        if self.offset_nerf_grad:
            # d loss / d xyzs of every point (colour-net input + colour-grid input gradient, through contract()) -> the vertices, through
            # dr.interpolate (grad_vworld) and dr.rasterize's (u, v) (grad_vclip, beside the antialias gradient)
            self.grad_vworld.zero_()
            call("n2m_s1_offset_grad", self._pp(), ptr(self.rast), ptr(self.vertices), ptr(self.vclip), ptr(self.triangles), ptr(self.inv),
                 self.h, self.w, ptr(self.pts), ptr(self.denc_tiles), ptr(t0.table), ptr(t0.offsets), ptr(self.grad_vclip),
                 ptr(self.grad_vworld), ptr(t0.opt_state), stream())

    def step(self, mvp, rays_d, gt, bg, shading="full", lr=None, use_graph=False, index=None):
        """One optimizer step on one view: mvp [4,4], rays_d [h0*w0,3] (unnormalised), gt [h0*w0, 3 or 4], bg [h0*w0,3].
        `index` (appearance codes, t0.cfg.ind_dim > 0: required, rejected otherwise): the view's image, data['index'] (utils.py:711);
        the view's points read its code and the step trains that code (its own Adam group, as in stage 0).
        `use_graph`: the step is captured once per view (keyed by the addresses of its device-resident tensors, which must then stay
        valid and in place -- the dataset of a stage-1 run is a fixed set of views) and replayed as one CUDA graph: ~17 launches and a
        handful of torch ops leave the host's critical path (the eager step is host-bound at this size)."""
        t0 = self.t0
        self._index = self._check_index(index)
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
            key = (mvp.data_ptr(), rays_d.data_ptr(), gt.data_ptr(), bg.data_ptr(), int(gt.shape[-1]), shading, int(t0.parity), self._index)
            g = self._graphs.get(key)
            if g is None:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._step_body(mvp, rays_d, gt, bg, shading)
                self._graphs[key] = (g, mvp, rays_d, gt, bg)          # keeps the captured addresses alive
                g = self._graphs[key]
            g[0].replay()
        t0.global_step += 1

    def _check_index(self, index):
        t0 = self.t0
        if not t0.ind_dim:
            if index is not None:
                raise ValueError("index given, but the model has no appearance codes (ind_dim = 0)")
            return 0
        if index is None:
            raise ValueError("index is required when the model has appearance codes (ind_dim > 0)")
        if isinstance(index, bool) or not isinstance(index, int):
            raise ValueError(f"index must be an int (the view's image), got {type(index).__name__}")
        if not 0 <= index < t0.ind_num:
            raise ValueError(f"index {index} out of range [0, {t0.ind_num})")
        return index

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
        if self.mesh_reg:               # + lambda_normal * mesh_normal_consistency + lambda_edgelen * mesh_edge_loss (utils.py:759-769)
            call("n2m_s1_vert_step_reg", ptr(self.grad_vclip), ptr(self.grad_vworld) if self.offset_nerf_grad else None, ptr(self.mvp),
                 ptr(th.keys), ptr(th.opp), th.slots, self.mesh_edges, self.mesh_pairs, ptr(self.base_vertices), ptr(self.offsets),
                 ptr(self.m_vert), ptr(self.v_vert), ptr(self.vertices), ptr(self.vert_scratch), ptr(self.grad_offsets), V, self.lambda_lap,
                 self.lambda_offsets, self.lambda_normal, self.lambda_edgelen, -1.0, self.t0.cfg.eps, ptr(self.t0.opt_state),
                 ptr(self.vert_state), ptr(self.loss_acc), stream())
            return
        rest = (ptr(self.mvp), ptr(th.keys), th.slots, ptr(self.base_vertices), ptr(self.offsets), ptr(self.m_vert), ptr(self.v_vert),
                ptr(self.vertices), ptr(self.vert_scratch), ptr(self.grad_offsets), V, self.lambda_lap, self.lambda_offsets, -1.0,
                self.t0.cfg.eps, ptr(self.t0.opt_state), ptr(self.vert_state), ptr(self.loss_acc), stream())
        if self.offset_nerf_grad:
            call("n2m_s1_vert_step_world", ptr(self.grad_vclip), ptr(self.grad_vworld), *rest)
        else:
            call("n2m_s1_vert_step", ptr(self.grad_vclip), *rest)

    def vertex_gradient(self):
        """d loss / d vertices [V,3] of the last `loss_backward` (through dr.antialias and the projection of renderer.py:858, plus with
        offset_nerf_grad the colour-field path through dr.interpolate / dr.rasterize; the gradient the reference accumulates on
        `vertices_offsets`), unscaled.  Valid when the step's found_inf flag is clear."""
        if not self.antialias:
            raise RuntimeError("vertex gradients flow through dr.antialias only: construct Stage1Trainer(antialias=True)")
        g = self.grad_vclip @ self.mvp[:, :3]
        if self.offset_nerf_grad:
            g = g + self.grad_vworld
        return g / self.t0.opt_state[0]

    def read_loss(self):
        return float(self.loss_acc[0].item())

    @torch.no_grad()
    def render(self, mvp, rays_d, h0=None, w0=None, bg_color=1.0, shading="full", antialias=True):
        """render_stage1 at inference (renderer.py:816-921; eval_step / test_step, utils.py:853,882): mvp [4,4], rays_d [h0*w0,3] (the
        low-res per-pixel directions, unnormalised, as step() takes them), bg_color a scalar or [h0*w0,3], shading 'diffuse' / 'specular' /
        'full'.  Returns (image [h0*w0,3], weights_sum [h0*w0], depth [h0*w0]) on the device; depth is the mean over the super-samples of
        alpha * z/w (:889,:900).  h0, w0 default to the trainer's; any other resolution works.

        The pipeline of forward() at ssaa * (h0, w0) -- rasterize, surface points (contracted when cfg.contract), gather, colour MLPs,
        with `antialias` (the reference always antialiases here) n2m_s1_rgba + dr.antialias -- then n2m_s1_render_compose.  It runs on
        buffers of its own per (h0, w0), with a point cap of every super-sample, and leaves the step's buffers, the optimizer state and the
        captured step graphs untouched.  The EMA is the caller's: t0.ema_apply() / t0.ema_restore() around the call."""
        if shading not in SHADING_MODES:
            raise ValueError(f"shading must be one of {sorted(SHADING_MODES)}")
        t0 = self.t0
        dev = t0.device
        h0 = self.h0 if h0 is None else int(h0)
        w0 = self.w0 if w0 is None else int(w0)
        Q = h0 * w0
        rays_d = rays_d.to(dev, torch.float32).contiguous()
        if tuple(rays_d.shape) != (Q, 3):
            raise ValueError(f"rays_d must be [{Q},3] for a {h0}x{w0} render")
        bg = bg_image(bg_color, Q, dev)
        rb = self._render_buffers(h0, w0)
        h, w = rb["h"], rb["w"]
        params = type(self.params)()
        ctypes.memmove(ctypes.byref(params), ctypes.byref(self.params), ctypes.sizeof(params))
        params.shading_full = SHADING_MODES[shading]
        pp = ctypes.byref(params)
        mvp = mvp.to(dev, torch.float32).contiguous()
        vclip = (torch.nn.functional.pad(self.vertices, (0, 1), value=1.0) @ mvp.T).contiguous()            # as forward()
        rast, _ = dr.rasterize(rb["glctx"], vclip[None], self.triangles, (h, w))
        rb["rast"] = rast
        call("n2m_s1_points_contract", ptr(rast), ptr(self.vertices), ptr(self.triangles), ptr(rays_d), h, w, self.ssaa, rb["cap"],
             ptr(rb["counters"]), ptr(rb["inv"]), ptr(rb["pts"]), ptr(rb["pdirs"]), ptr(rb["recs"]), int(self.contract), stream())
        t0.encode_points(pp, rb["pts"], rb["pdirs"], rb["counters"], rb["cap"], rb["enc_tiles"], 0)     # inference: code 0 (renderer.py:849-850)
        call("n2m_s0_mlp_fwd", pp, ptr(rb["enc_tiles"]), ptr(rb["counters"]), rb["cap"], ptr(t0.wpack), ptr(rb["out"]), None, 0, 1, stream())
        call("n2m_s1_rgba", ptr(rb["out"]), ptr(rb["inv"]), h * w, ptr(rb["rgba"]), stream())
        img = rb["rgba"]
        if antialias:
            th = self._render_topology()
            if "aa" not in rb:
                rb["aa"] = torch.empty(h * w, 4, device=dev)
            call("n2m_antialias_forward", ptr(rb["rgba"]), ptr(rast), ptr(vclip), ptr(self.triangles), ptr(th.keys), ptr(th.opp), th.slots,
                 h, w, 4, ptr(rb["aa"]), stream())
            img = rb["aa"]
        image = torch.empty(Q, 3, device=dev); weights_sum = torch.empty(Q, device=dev); depth = torch.empty(Q, device=dev)
        call("n2m_s1_render_compose", ptr(img), ptr(rast), ptr(bg), h0, w0, self.ssaa, ptr(image), ptr(weights_sum), ptr(depth), stream())
        return image, weights_sum, depth

    def _render_buffers(self, h0, w0):
        """render()'s buffers for a (h0, w0) render, made on first use and cached: its own rasterizer scratch (the step's graphs hold the
        addresses of the trainer's), point buffers with room for every super-sample, the (r, g, b, alpha) image"""
        rb = self._render_cache.get((h0, w0))
        if rb is None:
            dev = self.t0.device
            h, w = h0 * self.ssaa, w0 * self.ssaa
            n = h * w
            cap = (n + 127) // 128 * 128
            rb = self._render_cache[(h0, w0)] = dict(
                h=h, w=w, cap=cap, glctx=dr.RasterizeCudaContext(dev), inv=torch.empty(n, dtype=torch.int32, device=dev),
                pts=torch.zeros(cap, 3, device=dev), pdirs=torch.zeros(cap, 3, device=dev), recs=torch.zeros(cap, 4, device=dev),
                counters=torch.zeros(16, dtype=torch.int32, device=dev), enc_tiles=torch.zeros(cap * 64, dtype=torch.float16, device=dev),
                out=torch.zeros(cap, 4, device=dev), rgba=torch.empty(n, 4, device=dev))
        return rb

    def _render_topology(self):
        """the edge hash of the current mesh for render()'s antialias: the step's when it antialiases, else one built on first use (and
        again after replace_mesh)"""
        if self.antialias:
            return self.topology
        th = self._render_th
        if th is None or th.tri is not self.triangles:
            th = self._render_th = dr.TopologyHash(self.triangles)
        return th

    def refine_mask(self):
        """refine_and_decimate's face mask (renderer.py:217-240, not SDF) over the faces of cascade 0 (:223-225; with one mesh, all faces):
        mean error per face seen since the last reset, thresholds = the 90th / 50th percentiles over the seen faces (numpy's default 'linear'
        method in float32, as np.percentile computes them for the float32 errors).  Returns (mask [f_cumsum[1]] float32: 2 = refine
        (error > 90th), 1 = decimate (error < 50th), 0 = keep or unseen, (thresh_refine, thresh_decimate)).  ValueError when no face of
        cascade 0 has been seen."""
        if not self.refine:
            raise RuntimeError("refine_mask: construct Stage1Trainer(refine=True)")
        f1 = self.f_cumsum[1] if self.f_cumsum else None                  # None (no cascade bookkeeping): every face
        cnt = self.face_counts[:f1]
        seen = cnt > 0
        errors = self.face_errors[:f1].clone()
        errors[seen] = errors[seen] / cnt[seen]
        vals = torch.sort(errors[seen]).values
        if vals.numel() == 0:
            raise ValueError("refine_mask: no face has been seen since the mesh was (re)set")
        t_refine, t_decimate = _percentile_f32(vals, 90), _percentile_f32(vals, 50)
        mask = torch.zeros_like(errors)
        mask[(errors > t_refine) & seen] = 2
        mask[(errors < t_decimate) & seen] = 1
        return mask, (float(t_refine), float(t_decimate))

    def replace_mesh(self, vertices, triangles, reset_optimizer=True):
        """Restart the step on a new mesh (the tail of refine_and_decimate, renderer.py:287-292, and the new optimizer of utils.py:1209-1210):
        vertices [V,3] float, triangles [F,3] integer.  The vertices become the base of zero vertex offsets with zero Adam state; everything
        sized by the mesh is reallocated, the face errors restart from zero and the captured per-view graphs are dropped (they hold the old
        buffers' addresses).  reset_optimizer: also zero the shared Stage0Trainer's Adam moments and step count in place (a fresh
        torch.optim.Adam; its own captured graphs stay valid), keeping the GradScaler state as the reference keeps its scaler.  The
        reference also restarts its LambdaLR here (utils.py:1211): the schedule is the caller's (`step(lr=...)`), so the caller restarts it.
        On a trainer of several cascades the new mesh replaces cascade 0 and every outer cascade takes its current vertices (base + offsets)
        as its new base (renderer.py:258-285); v_cumsum / f_cumsum are rebuilt."""
        if not (torch.is_tensor(vertices) and torch.is_tensor(triangles)):
            raise ValueError("replace_mesh: vertices and triangles must be tensors")
        if vertices.dim() != 2 or vertices.shape[1] != 3 or not vertices.is_floating_point() or vertices.shape[0] == 0:
            raise ValueError("replace_mesh: vertices must be a float tensor [V,3], V >= 1")
        if triangles.dim() != 2 or triangles.shape[1] != 3 or triangles.dtype not in _INT_DTYPES or triangles.shape[0] == 0:
            raise ValueError("replace_mesh: triangles must be an integer tensor [F,3], F >= 1")
        V = int(vertices.shape[0])
        if int(triangles.min()) < 0 or int(triangles.max()) >= V:
            raise ValueError(f"replace_mesh: triangles index outside the vertices (0..{V - 1})")
        if not bool(torch.isfinite(vertices).all()):
            raise ValueError("replace_mesh: vertices must be finite")
        if self.mesh_reg:               # checked before anything changes; the outer cascades passed already and no face links two cascades
            self._check_mesh_reg(dr.TopologyHash(triangles.to(self.t0.device, torch.int32)), "replace_mesh")
        outer = [self.cascade_mesh(cas) for cas in range(1, self.cascades)]
        self._graphs.clear()
        self._warm = False
        self._set_cascades([vertices] + [v.clone() for v, _ in outer], [triangles] + [f for _, f in outer])
        self.rast = self.vclip = self.mvp = None
        if self.lr_vert > 0:
            self.vert_state[0:1].zero_()
        self._mesh_buffers()
        if reset_optimizer:
            t0 = self.t0
            for buf in (t0.m_table, t0.v_table, t0.m_mlp, t0.v_mlp) + ((t0.m_ind, t0.v_ind) if t0.ind_dim else ()):
                buf.zero_()
            t0.opt_state[2:3].zero_()


_INT_DTYPES = (torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64)


def mesh_reg_counts(th):
    """(E unique edges, P edges with exactly two faces, edges with more than two faces, faces with a repeated vertex index) of the mesh
    th.tri over its edge hash `th` (dr.TopologyHash): n2m_s1_mesh_reg_setup, which reads the four counts back to the host"""
    scratch = torch.empty(th.slots + 4, dtype=torch.int32, device=th.tri.device)
    counts = (ctypes.c_uint32 * 4)()
    call("n2m_s1_mesh_reg_setup", ptr(th.tri), th.tri.shape[0], ptr(th.keys), th.slots, ptr(scratch), counts, stream())
    return tuple(int(c) for c in counts)


def _cascade_lists(vertices, triangles):
    """(vertices, triangles) as equal-length lists of per-cascade tensors: a single tensor is a list of one"""
    if torch.is_tensor(vertices) and torch.is_tensor(triangles):
        return [vertices], [triangles]
    vertices, triangles = list(vertices), list(triangles)
    if len(vertices) == 0 or len(vertices) != len(triangles):
        raise ValueError("vertices and triangles: one tensor each, or equal-length non-empty lists of per-cascade tensors")
    return vertices, triangles


def _percentile_f32(sorted_vals, q):
    """np.percentile(x, q) (method 'linear') of a float32 tensor x given sorted: numpy keeps the float32 dtype throughout -- q / 100,
    the virtual index (n - 1) * q, its fraction and the two-sided lerp are all float32 operations."""
    n = sorted_vals.numel()
    qf = np.float32(q) / np.float32(100)
    vi = np.float32(n - 1) * qf
    if vi >= n - 1:                                       # past the last index: the maximum (numpy's index -1, gamma against -1)
        lo = hi = n - 1
        gamma = vi - np.float32(-1)
    else:
        lo = int(np.floor(vi)); hi = lo + 1
        gamma = vi - np.float32(lo)
    a, b = sorted_vals[lo], sorted_vals[hi]
    t = torch.tensor(float(gamma), dtype=torch.float32, device=sorted_vals.device)
    d = b - a
    if gamma >= 0.5:
        return b - d * (1 - t)
    return a + d * t
