"""Generate tests/golden/psamask_ref_digests.json: SHA-256 digests of the reference's own psa_mask kernels
(lib/psa/src/{cpu,gpu}, compiled into oracle/_ref/ by oracle/build.py) on the seeded inputs of
tests/test_oracle_cpu.py::test_psamask_oracle_matches_compiled_reference (CPU kernel) and
tests/test_validate_path_gpu.py::test_psamask_bit_identical_to_the_references_cuda_kernel (CUDA kernel).

    python tests/golden/make_psamask_digests.py      # needs oracle/_ref built; the CUDA part needs a GPU
"""
import hashlib
import importlib.util
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests import psamask_cases as pc  # noqa: E402


def _ext(prefix):
    d = os.path.join(ROOT, "oracle", "_ref")
    for f in sorted(os.listdir(d)):
        if f.startswith(prefix) and f.endswith(".so"):
            spec = importlib.util.spec_from_file_location(prefix, os.path.join(d, f))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            return mod
    raise SystemExit("oracle/_ref/%s*.so not built" % prefix)


def sha(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def run(ext, device, cases):
    out = {}
    for key, t, (n, h, w, mh, mw), x, g in cases:
        o = torch.zeros((n, h * w, h, w), device=device)
        ext.psamask_forward(t, torch.from_numpy(x).to(device), o, n, h, w, mh, mw, (mh - 1) // 2, (mw - 1) // 2)
        gi = torch.zeros((n, mh * mw, h, w), device=device)
        ext.psamask_backward(t, torch.from_numpy(g).to(device), gi, n, h, w, mh, mw, (mh - 1) // 2, (mw - 1) // 2)
        out[key] = {"out": sha(o), "din": sha(gi)}
    return out


def main():
    path = os.path.join(HERE, "psamask_ref_digests.json")
    res = json.load(open(path)) if os.path.exists(path) else {}
    res["cpu"] = run(_ext("psamask_ref_cpu"), "cpu", pc.cpu_cases())
    if torch.cuda.is_available():
        res["gpu"] = run(_ext("psamask_ref_gpu"), "cuda", pc.gpu_cases())
    json.dump(res, open(path, "w"), indent=1, sort_keys=True)
    print(path)


if __name__ == "__main__":
    main()
