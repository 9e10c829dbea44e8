"""ctypes binding of libn2m_probes.so: the wgmma layout probe (csrc/tc_probe.cu).  Test and profiling infrastructure -- not part of the product library libn2m_b200.so."""
import ctypes
import os

from nerf2mesh_b200 import _lib        # loads libn2m_b200.so first (the probes resolve n2m::fail / launch counters from it)
from nerf2mesh_b200._lib import I, P, U, check

PATH = os.path.join(os.path.dirname(os.path.abspath(_lib.__file__)), "libn2m_probes.so")
lib = ctypes.CDLL(PATH, mode=ctypes.RTLD_GLOBAL)
for _n, _a in {"n2m_tc_probe": [P, P, P, U, U, I, I, P]}.items():
    _f = getattr(lib, _n); _f.argtypes = _a; _f.restype = ctypes.c_int


def call(name, *args):
    check(getattr(lib, name)(*args))
