"""Recorded outputs of the reference CUDA extensions (oracle/_ref), so that the parity tests run where the
reference cannot be built.

`Replay(name, module, nodeid)` stands in for one reference extension inside one test.  Every call of a
binding mutates some of its tensor arguments (the reference's kernels write into caller-allocated outputs):
  * with the built extension and N2M_RECORD_GOLDEN=<directory>, the call runs and the arguments it changed
    are recorded, keyed by test id and call index; `save_all()` writes them to <directory>/ref_<name>.npz,
    which is copied to tests/golden/;
  * otherwise the recorded values are copied into the same arguments, so the test compares the project's
    kernels against what the reference computed on the same seeded inputs.
Inputs are generated from seeds on the CPU (tests/cases.py), so a recording matches its replay exactly.  Recordings are keyed
by "<test file name>::<test name with parameters>".

Where the outputs are too large to store, a test records a `summary()` instead: a few small arrays and SHA-256 digests of
the reference's outputs, against which a bit-exact comparison is exactly as strict, or a fixed, seeded sample of an output
too large to store.  A test without a recording runs against the built extension itself (`live`), and fails where it is not
built: a renamed test or parameter must be recorded again."""
import hashlib
import os

import pytest

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD = os.environ.get("N2M_RECORD_GOLDEN")
_recorded = {}          # name -> {key: array}
_loaded = {}


def _key(nodeid, idx, arg):
    return f"{hashlib.sha1(nodeid.encode()).hexdigest()[:16]}_{idx}_{arg}"


def _golden(name):
    """the recordings of one extension: tests/golden/ref_<name>.npz, split into ref_<name>_<part>.npz where one file would be large"""
    if name not in _loaded:
        _loaded[name] = {}
        for f in sorted(os.listdir(GOLDEN)):
            if f == f"ref_{name}.npz" or (f.startswith(f"ref_{name}_") and f.endswith(".npz")):
                with np.load(os.path.join(GOLDEN, f)) as z:
                    _loaded[name].update({k: z[k] for k in z.files})
    return _loaded[name]


def digest(a):
    """SHA-256 of an array's dtype, shape and bytes (equal digests <=> bit-identical arrays)"""
    a = np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a)
    return hashlib.sha256(f"{a.dtype}{a.shape}".encode() + a.tobytes()).hexdigest()


def _recorded_here(name, nodeid):
    prefix = hashlib.sha1(nodeid.encode()).hexdigest()[:16] + "_"
    return any(k.startswith(prefix) for k in _golden(name))


class Replay:
    def __init__(self, name, module, nodeid):
        self._name, self._mod, self._nodeid, self._n = name, module, nodeid, 0
        if RECORD:
            self._mode = "record"
        elif _recorded_here(name, nodeid):
            self._mode = "replay"
        elif module is not None:
            self._mode = "live"
        else:
            pytest.fail(f"no recorded reference outputs for {nodeid} in tests/golden/ref_{name}*.npz and the reference extensions are "
                        "not built: record them with N2M_RECORD_GOLDEN=<directory>")

    def summary(self, compute):
        """compute(module) -> dict of small arrays (digests as strings), from the extension or from the recording"""
        idx = self._n
        self._n += 1
        if self._mode == "replay":
            g = _golden(self._name)
            pre = _key(self._nodeid, idx, "s_")
            return {k[len(pre):]: (str(v) if v.dtype.kind == "U" else v) for k, v in g.items() if k.startswith(pre)}
        out = compute(self._mod)
        if self._mode == "record":
            rec = _recorded.setdefault(self._name, {})
            for k, v in out.items():
                rec[_key(self._nodeid, idx, "s_" + k)] = np.asarray(v)
        return out

    def __getattr__(self, fn):
        if self._mode == "live":
            return getattr(self._mod, fn)

        def call(*args):
            idx = self._n
            self._n += 1
            tens = [(i, a) for i, a in enumerate(args) if isinstance(a, torch.Tensor)]
            if self._mode == "record":
                before = [a.clone() for _, a in tens]
                out = getattr(self._mod, fn)(*args)
                torch.cuda.synchronize()
                rec = _recorded.setdefault(self._name, {})
                for (i, a), b in zip(tens, before):
                    now = a.detach().cpu().numpy()
                    if now.tobytes() != b.cpu().numpy().tobytes():
                        rec[_key(self._nodeid, idx, i)] = now
                return out
            g = _golden(self._name)
            for i, a in tens:
                k = _key(self._nodeid, idx, i)
                if k in g:
                    a.copy_(torch.from_numpy(g[k]).to(a.device))
            return None
        return call


def save_all():
    os.makedirs(RECORD, exist_ok=True)
    for name, rec in _recorded.items():
        np.savez_compressed(os.path.join(RECORD, f"ref_{name}.npz"), **rec)
