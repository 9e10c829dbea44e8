"""oracle/ref_stage.py -- TEST / BASELINE INFRASTRUCTURE, NOT PRODUCT.

Runs the reference's OWN, UNMODIFIED Python model code (nerf/network.py NeRFNetwork + nerf/renderer.py NeRFRenderer,
encoding.py, activation.py, and -- for the "ref" backend -- its operator wrappers raymarching/raymarching.py,
gridencoder/grid.py, shencoder/sphere_harmonics.py) on a GPU machine that need not hold the reference tree:

* `stage()` (called by __graft_entry__.build() where the reference tree is present, see N2M_REFERENCE_ROOT) copies those
  files byte for byte into the git-ignored directory oracle/_ref/py/ -- the same treatment as the
  compiled reference kernels in oracle/_ref/*.so.  Nothing is committed to the repository.
* `load(backend)` imports the staged `nerf` package with
    backend="ref" : the staged reference wrappers over the reference's compiled kernels (oracle/_ref/_ref_*.so, made
                    importable under the names the wrappers try first: `_raymarching_mob`, `_gridencoder`, `_shencoder`,
                    raymarching.py:9-12, grid.py:9-12, sphere_harmonics.py:9-12) -- the reference CUDA path itself;
    backend="ours": `nerf2mesh_b200.install()` -- the drop-in proof: the unmodified model code over this repo's operators.
  Modules the renderer / trainer import at module scope but stage 0 never touches (nvdiffrast, mcubes, trimesh, xatlas,
  pymeshlab, matplotlib, imageio, tensorboardX, pytorch3d, torch_ema, lpips, torch_scatter) are stubbed when absent.
  Each call returns a FRESH copy of the module tree, so "ref" and "ours" can live side by side in one process.
* `default_opt(**overrides)`: the argparse defaults of main.py:12-131 plus the `-O` switches (main.py:129-136) that matter
  for the model (fp16, cuda_ray, ...), as a namespace.
"""
import importlib
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("N2M_REFERENCE_ROOT", "/root/reference")
PY = os.path.join(HERE, "_ref", "py")

FILES = [
    "nerf/network.py", "nerf/renderer.py", "nerf/utils.py", "encoding.py", "activation.py", "meshutils.py",
    "raymarching/__init__.py", "raymarching/raymarching.py",
    "gridencoder/__init__.py", "gridencoder/grid.py",
    "shencoder/__init__.py", "shencoder/sphere_harmonics.py",
]

STUBS = ["nvdiffrast", "nvdiffrast.torch", "mcubes", "trimesh", "xatlas", "pymeshlab", "matplotlib", "matplotlib.pyplot",
         "imageio", "tensorboardX", "pytorch3d", "pytorch3d.structures", "pytorch3d.loss", "torch_ema", "lpips",
         "torch_scatter", "dearpygui", "dearpygui.dearpygui"]

_OWN = ["nerf", "nerf.network", "nerf.renderer", "nerf.utils", "encoding", "activation", "meshutils",
        "raymarching", "raymarching.raymarching", "gridencoder", "gridencoder.grid", "shencoder", "shencoder.sphere_harmonics",
        "_raymarching_mob", "_gridencoder", "_shencoder"]


def staged():
    return all(os.path.exists(os.path.join(PY, f)) for f in FILES)


def stage(force=False):
    """Copy the reference's Python files into oracle/_ref/py/ (only where the reference tree exists)."""
    if not os.path.isdir(REF):
        return staged()
    for f in FILES:
        src, dst = os.path.join(REF, f), os.path.join(PY, f)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if force or not os.path.exists(dst) or os.path.getmtime(src) > os.path.getmtime(dst):
            shutil.copy2(src, dst)
    init = os.path.join(PY, "nerf", "__init__.py")      # the reference's `nerf` is a namespace-style package without __init__
    if not os.path.exists(init) and not os.path.exists(os.path.join(REF, "nerf", "__init__.py")):
        open(init, "w").close()
    return True


class _Anything:
    """Attribute sink for stubbed third-party modules: any attribute is a dummy class / callable."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Anything()


def _stub(name):
    m = types.ModuleType(name)

    def _getattr(attr):
        if attr.startswith("__"):
            raise AttributeError(attr)
        return _Anything

    m.__getattr__ = _getattr
    m.__path__ = []
    parent, _, child = name.rpartition(".")
    if parent and parent in sys.modules:
        setattr(sys.modules[parent], child, m)
    return m


def load(backend="ref"):
    """-> namespace(nerf_network, nerf_renderer, raymarching, gridencoder, encoding) of a fresh import of the staged tree."""
    assert backend in ("ref", "ours")
    if not staged():
        raise FileNotFoundError(f"{PY}: reference Python files not staged (run __graft_entry__.build() where the reference tree exists)")
    import torch  # noqa: F401
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in _OWN}
    for name in STUBS:
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except Exception:
                if name == "torch_ema":       # a working restatement, so that Trainer(ema_decay=...) runs (oracle/torch_ema_port.py)
                    from . import torch_ema_port
                    sys.modules[name] = torch_ema_port
                else:
                    sys.modules[name] = _stub(name)
    path_before = list(sys.path)
    try:
        if backend == "ref":
            from .build_ref import load_ref
            sys.modules["_raymarching_mob"] = load_ref("_ref_raymarching")
            sys.modules["_gridencoder"] = load_ref("_ref_gridencoder")
            sys.modules["_shencoder"] = load_ref("_ref_shencoder")
            sys.path.insert(0, PY)
        else:
            import nerf2mesh_b200
            nerf2mesh_b200.install()
            # only nerf/, encoding.py, activation.py, meshutils.py may resolve from the staged tree: the operator packages
            # are already in sys.modules (ours), so `import raymarching` never reaches the staged wrappers
            sys.path.insert(0, PY)
        for pkg in ("raymarching", "gridencoder", "shencoder"):
            importlib.import_module(pkg)
        net = importlib.import_module("nerf.network")
        ren = importlib.import_module("nerf.renderer")
        out = types.SimpleNamespace(backend=backend, network=net, renderer=ren, NeRFNetwork=net.NeRFNetwork,
                                    raymarching=sys.modules["raymarching"], gridencoder=sys.modules["gridencoder"],
                                    encoding=sys.modules["encoding"])
        try:
            out.utils = importlib.import_module("nerf.utils")
        except Exception as e:      # noqa: BLE001  (optional: Trainer needs more of the stubs to behave)
            out.utils, out.utils_error = None, repr(e)
        out._mods = {k: sys.modules[k] for k in _OWN if k in sys.modules}
        out.context = lambda: _Context(out._mods)
        out.make_model = lambda opt: _make_model(out, opt)
    finally:
        sys.path[:] = path_before
        for k in _OWN:
            sys.modules.pop(k, None)
        sys.modules.update(saved)
    return out


class _Context:
    """Temporarily re-installs one loaded tree's modules in sys.modules: the reference resolves `from gridencoder import
    GridEncoder` lazily inside encoding.get_encoder (encoding.py:93-95), i.e. when a model is constructed."""

    def __init__(self, mods):
        self.mods = mods

    def __enter__(self):
        self.saved = {k: sys.modules.get(k) for k in _OWN}
        for k in _OWN:
            sys.modules.pop(k, None)
        sys.modules.update(self.mods)

    def __exit__(self, *exc):
        for k in _OWN:
            sys.modules.pop(k, None)
        sys.modules.update({k: v for k, v in self.saved.items() if v is not None})
        return False


def _make_model(ns, opt):
    with ns.context():
        return ns.NeRFNetwork(opt)


def default_opt(**over):
    """main.py:12-131 defaults + what `-O` switches on (main.py:129-136) + cuda_ray forced (main.py:127)."""
    o = dict(
        O=True, stage=0, fp16=True, sdf=False, tcnn=False, progressive_level=False, cuda_ray=True, preload=True,
        bound=2.0, scale=-1, offset=[0, 0, 0], min_near=0.05, iters=30000, lr=1e-2, lr_vert=1e-4, pos_gradient_boost=1,
        max_steps=1024, update_extra_interval=16, max_ray_batch=4096, grid_size=128, mark_untrained=True, dt_gamma=1 / 256,
        density_thresh=10, diffuse_step=1000, diffuse_only=False, background="random", enable_offset_nerf_grad=False,
        num_rays=4096, adaptive_num_rays=True, num_points=2 ** 18, lambda_density=0, lambda_entropy=0, lambda_tv=1e-8,
        lambda_depth=0.1, lambda_specular=1e-5, lambda_eikonal=0.1, lambda_rgb=1, lambda_mask=0.1, wo_smooth=False,
        lambda_lpips=0, lambda_offsets=0.1, lambda_lap=0.001, lambda_normal=0, lambda_edgelen=0, contract=False, patch_size=1,
        trainable_density_grid=False, color_space="srgb", ind_dim=0, ind_num=500, mcubes_reso=512, env_reso=256,
        decimate_target=3e5, mesh_visibility_culling=True, visibility_mask_dilation=5, clean_min_f=8, clean_min_d=5, ssaa=2,
        texture_size=4096, refine=True, refine_size=0.01, refine_decimate_ratio=0.1, refine_remesh_size=0.02, gui=False,
        random_image_batch=True, enable_cam_near_far=False, enable_cam_center=False, test=False, workspace="workspace",
        seed=0, ckpt="latest", data_format="nerf",
    )
    o.update(over)
    return types.SimpleNamespace(**o)


if __name__ == "__main__":
    print("staged" if stage(force="--force" in sys.argv) else "reference tree not present and nothing staged", PY)
