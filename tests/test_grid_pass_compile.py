"""CPU: the compile-time budget of the hash-grid scatter / TV kernel k_s0_encode_bwd (csrc/stage0.cu).

Both instantiations (feature-gradient scatter and TV) read only the gradient columns of the level group they visit and keep them in
registers; a spill or a local-memory array would put per-thread local-memory round trips beside the L2-bound REDs of every level.
Compiles stage0.cu with the library's nvcc flags plus -Xptxas -v; no GPU needed.
"""
import os
import re
import subprocess

from nerf2mesh_b200 import build as B


def test_encode_bwd_has_no_spills_and_no_stack_frame(tmp_path):
    src = os.path.join(B.CSRC, "stage0.cu")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "stage0.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = (r.stdout + r.stderr).splitlines()
    props = [i for i, l in enumerate(lines) if "Function properties for" in l and "k_s0_encode_bwd" in l]
    assert len(props) == 2, "\n".join(lines)
    for i in props:
        frame = lines[i + 1]
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", frame)
        assert m, frame
        assert (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (0, 0, 0), lines[i] + "\n" + frame
