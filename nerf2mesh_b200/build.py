"""Build libn2m_b200.so (sm_90a only) in-tree with nvcc.

    python -m nerf2mesh_b200.build [--force] [--verbose]

The library has no torch / python dependency: plain CUDA runtime (static cudart), C ABI
declared in include/n2m_b200.h.  Objects are cached under nerf2mesh_b200/csrc/_obj and rebuilt
when a source or header is newer.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(HERE, "libn2m_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

SOURCES = ["raymarching.cu", "gridencoder.cu", "shencoder.cu", "stage0.cu", "mlp_tc.cu", "fused.cu", "render.cu", "mcubes.cu", "cascade.cu", "meshclean.cu", "decimate.cu", "atlas.cu", "raster.cu", "antialias.cu", "stage1.cu", "texture.cu", "grid_aux.cu", "optim.cu", "dp.cu"]
# micro-benchmarks and the wgmma layout probe: test / profiling infrastructure, kept OUT of the product library
PROBE_SOURCES = ["tc_probe.cu"]
PROBE_LIB = os.path.join(HERE, "libn2m_probes.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    # same numerics contract as the reference build (raymarching/backend.py:16-21):
    "-use_fast_math",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
    "-I", INCLUDE,
]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return hs


def build(force=False, verbose=False):
    lib = _build(SOURCES, LIB, [], force, verbose)
    # the probes resolve the error / launch-count plumbing from the product library (rpath $ORIGIN)
    _build(PROBE_SOURCES, PROBE_LIB, ["-L", HERE, "-ln2m_b200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"], force, verbose)
    return lib


def _build(sources, LIB, link_extra, force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = [s for s in sources if os.path.exists(os.path.join(CSRC, s))]
    hdrs = _headers()
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        objs.append(obj)
        stale = force or _newer(src, obj) or any(_newer(h, obj) for h in hdrs)
        if stale:
            jobs.append([NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stdout + r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for out in ex.map(run, jobs):
                if verbose and out.strip():
                    print(out)
    if jobs or force or not os.path.exists(LIB) or any(_newer(o, LIB) for o in objs):
        run([NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + link_extra)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
