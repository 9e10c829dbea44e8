"""CPU: the compile-time budget of the stand-alone MLP backward kernel k_mlp_bwd (csrc/mlp_tc.cu).

The kernel runs three warpgroups at __launch_bounds__(384, 1), i.e. at most 168 registers per thread.  Spilled accumulators
or wgmma issues that ptxas serialises or fences (advisories C7510-C7519) put local-memory round trips or stalls into the
latency-bound chain of tensor-core rounds, so the build must have neither.  Compiles mlp_tc.cu with the library's nvcc flags
plus -Xptxas -v; no GPU needed.
"""
import os
import re
import subprocess

from nerf2mesh_b200 import build as B


def _ptxas_report(tmp_path):
    src = os.path.join(B.CSRC, "mlp_tc.cu")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "mlp_tc.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return (r.stdout + r.stderr).splitlines()


def test_mlp_bwd_has_no_spills_and_no_wgmma_advisories(tmp_path):
    lines = _ptxas_report(tmp_path)
    props = [i for i, l in enumerate(lines) if "Function properties for" in l and "k_mlp_bwd" in l]
    assert len(props) == 1, "\n".join(lines)
    frame = lines[props[0] + 1]
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", frame)
    assert m, frame
    assert (int(m.group(2)), int(m.group(3))) == (0, 0), frame
    advisories = [l for l in lines if re.search(r"\(C751\d\)", l) and "k_mlp_bwd" in l]
    assert not advisories, "\n".join(advisories)
