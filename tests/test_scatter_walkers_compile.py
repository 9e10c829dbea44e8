"""CPU: the compile-time budget of the whole-SM scatter kernel k_s0_scatter_walkers (csrc/stage0.cu).

No spill or stack frame (local-memory round trips beside the L2-bound REDs), and at most 56 registers, so that a 1024-thread CTA
launches and the per-slot kernel beside it in the library keeps its own budget (tests/test_grid_pass_compile.py).
"""
import os
import re
import subprocess

from nerf2mesh_b200 import build as B


def test_scatter_walkers_fit_the_register_cap_without_spills(tmp_path):
    src = os.path.join(B.CSRC, "stage0.cu")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "stage0.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    props = [i for i, l in enumerate(lines) if "Function properties for" in l and "k_s0_scatter_walkers" in l]
    assert len(props) == 1, "\n".join(lines)
    i = props[0]
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
    assert m and (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (0, 0, 0), lines[i + 1]
    m = re.search(r"Used (\d+) registers", lines[i + 2])
    assert m and int(m.group(1)) <= 56, lines[i + 2]
