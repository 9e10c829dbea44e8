"""ctypes binding of libn2m_b200.so (the C ABI declared in include/n2m_b200.h).

There is NO fallback: if the shared library is missing or a symbol is absent the import
fails loudly -- the product path never routes through the oracle or any CPU code.
"""
import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_uint32, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libn2m_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: build it with `python -m nerf2mesh_b200.build` "
        "(nvcc, sm_90a). nerf2mesh_b200 has no CPU / PyTorch fallback.")

lib = ctypes.CDLL(LIB_PATH)

P = c_void_p
U = c_uint32
F = c_float
I = c_int

# name -> argtypes (restype is int unless listed in _RESTYPES)
SIGNATURES = {
    "n2m_near_far_from_aabb": [P, P, P, U, F, P, P, P],
    "n2m_sph_from_ray": [P, P, F, U, P, P],
    "n2m_morton3D": [P, U, P, P],
    "n2m_morton3D_invert": [P, U, P, P],
    "n2m_packbits": [P, U, F, P, P],
    "n2m_flatten_rays": [P, U, U, P, P],
    "n2m_march_rays_train": [P, P, P, F, I, F, U, U, U, U, P, P, P, P, P, P, P, P, P, P],
    "n2m_composite_rays_train_forward": [P, P, P, P, U, U, F, I, P, P, P, P, P],
    "n2m_composite_rays_train_backward": [P, P, P, P, P, P, P, P, P, P, P, U, U, F, I, P, P, P],
    "n2m_march_rays": [U, U, P, P, P, P, F, I, F, U, U, U, P, P, P, P, P, P, P, P],
    "n2m_composite_rays": [U, U, F, I, P, P, P, P, P, P, P, P, P],
    "n2m_grid_encode_forward": [P, P, P, P, U, U, U, U, U, F, U, P, U, I, U, I, P],
    "n2m_grid_encode_backward": [P, P, P, P, P, U, U, U, U, U, F, U, P, P, U, I, U, I, P],
    "n2m_grad_total_variation": [P, P, P, P, F, U, U, U, U, F, U, U, I, P],
    "n2m_sh_encode_forward": [P, P, U, U, U, P, P],
    "n2m_sh_encode_backward": [P, P, U, U, U, P, P, P],
}
_RESTYPES = {
    "n2m_last_error": (c_char_p, []),
    "n2m_version": (c_int, []),
    "n2m_launch_count": (c_uint64, []),
}

# fused / optimizer entry points (include/n2m_b200_fused.h) are registered by fused.py


def _bind(name, argtypes, restype=c_int):
    fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
    fn.argtypes = argtypes
    fn.restype = restype
    return fn


for _n, _a in SIGNATURES.items():
    _bind(_n, _a)
for _n, (_r, _a) in _RESTYPES.items():
    _bind(_n, _a, _r)


def register(signatures):
    """Bind additional entry points (used by the fused path)."""
    for n, a in signatures.items():
        _bind(n, a)
        SIGNATURES[n] = a


def last_error():
    return lib.n2m_last_error().decode("utf-8", "replace")


def launch_count():
    return int(lib.n2m_launch_count())


def check(rc):
    if rc != 0:
        raise RuntimeError(last_error())


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    check(getattr(lib, name)(*args))


def require_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    return t
