"""Writes tests/golden/tail_x8.npz: inputs and outputs of the x8 fused tail entry points (semseg_upsample_ce_fwd / _bwd)
on seeded inputs, the vectors `tests/test_zoom_gpu.py::test_zoom8_matches_the_x8_kernel_golden` holds the zoom-8 instance
of the templated kernels to, bit for bit.

    python tests/golden/make_tail_x8_golden.py [--lib path/to/libsemseg_b200.so] [--out tests/golden/tail_x8.npz]

The committed file was written on an H100 with the library of commit 5b5f3cd, whose kernels were x8-only. Needs a GPU.
"""
import argparse
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

# (N, h, w, C, pitch): a padded pitch at 21 classes, and 150 classes over two 128-column forward CTAs
CASES = {"c21": (2, 9, 13, 21, 24), "c150": (1, 5, 17, 150, 152)}
GRAD = 0.4


def case_inputs(n, h, w, c, pitch, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    ho, wo = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    logits = torch.randn((n, h, w, pitch), generator=g) * 3
    t = torch.randint(0, c, (n, ho, wo), generator=g)
    t[torch.rand((n, ho, wo), generator=g) < 0.05] = 255
    odd = torch.rand((n, ho, wo), generator=g) < 0.003
    t[odd] = torch.where(torch.rand((n, ho, wo), generator=g)[odd] < 0.5, c + 3, -2)
    return logits, t


def main():
    import torch
    from semseg_b200 import _lib
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=_lib.LIB_PATH)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "tail_x8.npz"))
    args = ap.parse_args()
    lib = ctypes.CDLL(args.lib)
    for name in ("semseg_upsample_ce_workspace_floats", "semseg_upsample_ce_fwd", "semseg_upsample_ce_bwd_workspace_floats",
                 "semseg_upsample_ce_bwd"):
        res, argt = _lib.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, argt
    p = lambda t: ctypes.c_void_p(t.data_ptr())          # noqa: E731
    out = {}
    for k, (key, (n, h, w, c, pitch)) in enumerate(CASES.items()):
        ho, wo = 8 * (h - 1) + 1, 8 * (w - 1) + 1
        logits_cpu, t_cpu = case_inputs(n, h, w, c, pitch, seed=10 + k)
        logits, t = logits_cpu.cuda()[..., :c], t_cpu.cuda()
        grad = torch.tensor([GRAD], device="cuda")
        ws = torch.empty((lib.semseg_upsample_ce_workspace_floats(n, ho, wo),), device="cuda")
        info = torch.empty(2, device="cuda")
        amax = torch.empty((n, ho, wo), dtype=torch.int64, device="cuda")
        lse = torch.empty((n, ho, wo), device="cuda")
        assert lib.semseg_upsample_ce_fwd(p(logits), pitch, n, h, w, c, p(t), ho, wo, 255, p(ws), p(info), p(amax),
                                          p(lse), None) == 0
        wsb = torch.empty((lib.semseg_upsample_ce_bwd_workspace_floats(n, ho, w, c),), device="cuda")
        dl = torch.empty((n, h, w, c), device="cuda")
        assert lib.semseg_upsample_ce_bwd(p(logits), pitch, n, h, w, c, p(t), ho, wo, 255, p(lse), p(info), p(grad),
                                          p(wsb), p(dl), None) == 0
        torch.cuda.synchronize()
        out.update({key + "_logits": logits_cpu.numpy(), key + "_target": t_cpu.numpy().astype(np.int16),
                    key + "_info": info.cpu().numpy(), key + "_argmax": amax.cpu().numpy().astype(np.int16),
                    key + "_lse": lse.cpu().numpy(), key + "_dlogits": dl.cpu().numpy()})
    np.savez_compressed(args.out, **out)
    print("wrote", args.out, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
