"""oracle/build_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT.

Builds the UNMODIFIED reference CUDA extensions (raymarching / gridencoder /
shencoder) from the sources where they lie under the reference tree
(``N2M_REFERENCE_ROOT``) into ``oracle/_ref/`` so that bench.py's ``ref_cuda``
leg can run the reference's own kernels beside ours on the same GPU, and so
that the GPU parity tests can record their outputs (tests/refreplay.py).

Nothing is copied into the repo: the sources are compiled in place
(``<reference>/<ext>/src/*.cu|cpp``), only the resulting ``.so`` files are
written to ``oracle/_ref/`` (git-ignored).
Flags are the reference's own (``raymarching/backend.py:10-23``): -O3
-std=c++17 -use_fast_math and the half-operator -U defines; the arch is forced
to sm_90a because the reference pins none.

Usage:  python oracle/build_ref.py            # builds what is missing
        python oracle/build_ref.py --force
"""
import os
import sys
import shutil
import glob

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("N2M_REFERENCE_ROOT", "/root/reference")

EXTS = [
    # (module name, reference dir, sources)
    ("_ref_raymarching", "raymarching", ["raymarching.cu", "bindings.cpp"]),
    ("_ref_gridencoder", "gridencoder", ["gridencoder.cu", "bindings.cpp"]),
    ("_ref_shencoder", "shencoder", ["shencoder.cu", "bindings.cpp"]),
]

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
    "-U__CUDA_NO_HALF2_OPERATORS__",
    "-use_fast_math",
    "-gencode", "arch=compute_90a,code=sm_90a",
]
C_FLAGS = ["-O3", "-std=c++17"]


def built(name):
    return bool(glob.glob(os.path.join(OUT, name + "*.so")))


def build(force=False, verbose=False):
    if not os.path.isdir(REF):
        return False  # GPU box: only the prebuilt files are used
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))
    from torch.utils.cpp_extension import load
    for name, d, srcs in EXTS:
        if built(name) and not force:
            continue
        bdir = os.path.join("/tmp", "n2m_refbuild", name)
        os.makedirs(bdir, exist_ok=True)
        load(name=name,
             sources=[os.path.join(REF, d, "src", s) for s in srcs],
             extra_cflags=C_FLAGS, extra_cuda_cflags=NVCC_FLAGS,
             build_directory=bdir, verbose=verbose, is_python_module=False)
        so = os.path.join(bdir, name + ".so")
        shutil.copy2(so, os.path.join(OUT, name + ".so"))
    return True


def load_ref(name):
    """Import a prebuilt reference extension from oracle/_ref (tests/bench only)."""
    import importlib.util
    import torch  # noqa: F401  (libtorch symbols must be loaded first)
    path = os.path.join(OUT, name + ".so")
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built" if ok else "reference tree not present; nothing built",
          sorted(os.listdir(OUT)) if os.path.isdir(OUT) else [])
