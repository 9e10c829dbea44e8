"""Generate tests/golden/*.npz by running the UNMODIFIED reference CUDA kernels (oracle/_ref,
built from the reference tree by oracle/build_ref.py) on a GPU:

    python tests/golden/make_golden.py OUT_DIR          # writes OUT_DIR/*.npz
    cp OUT_DIR/*.npz tests/golden/

Inputs are regenerated from seeds by tests/cases.py (identical on every machine); only the
reference's OUTPUTS are stored.  The CPU tests pin oracle/ against these vectors; the GPU tests
check nerf2mesh_b200 against them as well as against the reference kernels' recorded outputs
(tests/refreplay.py)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases      # noqa: E402
import refcall    # noqa: E402
from oracle.build_ref import load_ref   # noqa: E402


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    rm = load_ref("_ref_raymarching"); ge = load_ref("_ref_gridencoder"); sh = load_ref("_ref_shencoder")
    cu = lambda t: t.cuda()

    # ---- raymarching -------------------------------------------------------------------------
    for name in cases.MARCH_CASES:
        c = cases.march_case(name)
        ro, rd, bits, aabb = cu(c["rays_o"]), cu(c["rays_d"]), cu(c["bits"]), cu(c["aabb"])
        nears, fars = refcall.near_far(rm, ro, rd, aabb, c["min_near"])
        xyzs, dirs, ts, rays = refcall.march_train(rm, ro, rd, bits, c["bound"], c["contract"], c["dt_gamma"],
                                                   c["max_steps"], c["C"], c["H"], nears, fars, cu(c["noises"]))
        x = refcall.by_ray(xyzs, rays); t = refcall.by_ray(ts, rays)
        keep = min(len(x), 4096)
        np.savez_compressed(os.path.join(out_dir, f"march_{name}.npz"), nears=nears.cpu().numpy(), fars=fars.cpu().numpy(),
                            counts=rays[:, 1].cpu().numpy(), xyzs_head=x[:keep], ts_head=t[:keep],
                            xyzs_sum=x.astype(np.float64).sum(0), ts_sum=t.astype(np.float64).sum(0))
    # ---- compositing --------------------------------------------------------------------------
    c = cases.composite_case()
    sig, rgb, ts, rays = cu(c["sigmas"]), cu(c["rgbs"]), cu(c["ts"]), cu(c["rays"])
    out = {}
    for T in (1e-4, 1e-2):
        w, ws, d, im = refcall.composite_fwd(rm, sig, rgb, ts, rays, T, False)
        gs, gr = refcall.composite_bwd(rm, cu(c["grad_weights"]), cu(c["grad_weights_sum"]), cu(c["grad_depth"]), cu(c["grad_image"]),
                                       sig, rgb, ts, rays, ws, d, im, T, False)
        for k, v in dict(w=w, ws=ws, d=d, im=im, gs=gs, gr=gr).items():
            out[f"{k}_{T}"] = v.cpu().numpy()
    np.savez_compressed(os.path.join(out_dir, "composite.npz"), **out)
    # ---- grid encoder -------------------------------------------------------------------------
    for name in cases.GRID_CASES:
        c = cases.grid_case(name)
        inputs, emb, offsets = cu(c["inputs"]), cu(c["embeddings"]), cu(c["offsets"])
        o, dy = refcall.grid_fwd(ge, inputs, emb, offsets, c["S"], c["H"], c["L"], c["gridtype"], c["align"], c["interp"], True)
        g = torch.Generator().manual_seed(2)
        grad = torch.randn(c["L"], c["B"], c["C"], generator=g).cuda().to(emb.dtype)
        gemb, ginp = refcall.grid_bwd(ge, grad, inputs, emb, offsets, c["S"], c["H"], c["L"], c["gridtype"], c["align"], c["interp"], dy)
        nz = gemb.float().abs().sum(-1).nonzero().flatten()
        extra = {}
        if not c["half"]:
            gtv = torch.zeros_like(emb)
            ge.grad_total_variation(inputs, emb, gtv, offsets, 1e-3, c["B"], c["D"], c["C"], c["L"], c["S"], c["H"], c["gridtype"], c["align"])
            nzt = gtv.abs().sum(-1).nonzero().flatten()
            extra = dict(tv_rows=nzt.cpu().numpy(), tv_vals=gtv[nzt].cpu().numpy())
        np.savez_compressed(os.path.join(out_dir, f"grid_{name}.npz"), outputs=o.float().cpu().numpy(), dy_dx=dy.float().cpu().numpy(),
                            gemb_rows=nz.cpu().numpy(), gemb_vals=gemb[nz].float().cpu().numpy(), ginp=ginp.float().cpu().numpy(), **extra)
    # ---- SH ----------------------------------------------------------------------------------
    v = cu(cases.sh_case())
    out = {}
    for deg in range(1, 9):
        o, dy = refcall.sh_fwd(sh, v, deg, True)
        out[f"o{deg}"] = o.cpu().numpy(); out[f"dy{deg}"] = dy.cpu().numpy()
    np.savez_compressed(os.path.join(out_dir, "sh.npz"), **out)
    torch.cuda.synchronize()
    print("golden written to", out_dir, sorted(os.listdir(out_dir)))


if __name__ == "__main__":
    import tempfile
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "n2m_golden"))
