"""Writes tests/golden/psa_attend_default.json: SHA-256 digests of what the window + softmax fused PSA attention entry
points (semseg_psa_attend modes 0 and 1, semseg_psa_attend_bwd_attn) compute on the seeded operands of
tests/psa_attend_cases.py, in bf16 and bf16x3, for psa_type 0 and 1. `tests/test_psa_variants_gpu.py` holds the default
form of the kernels to these digests, bit for bit, through the original entry points and the `_ex` ones.

    python tests/golden/make_psa_attend_golden.py [--lib path/to/libsemseg_b200.so] [--out path.json]

The committed file was written on an H100 with the library of commit 707f71f, whose kernels knew only the window form
with softmax. Needs a GPU.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    import torch
    from semseg_b200 import _lib
    from tests import psa_attend_cases as pc
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=_lib.LIB_PATH)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "psa_attend_default.json"))
    args = ap.parse_args()
    lib = ctypes.CDLL(args.lib)
    for name in ("semseg_psa_attend", "semseg_psa_attend_bwd_attn", "semseg_last_error"):
        res, argt = _lib.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, argt
    p = lambda t: ctypes.c_void_p(t.data_ptr())                                              # noqa: E731
    lo = lambda t: ctypes.c_void_p(t.data_ptr() + 2 * t.stride(0) if t.dim() == 5 else 0)   # noqa: E731
    c, scale = pc.C, pc.SCALE
    out = {}
    for k, (key, geom) in enumerate(pc.CASES.items()):
        n, h, w, mh, mw = geom
        for split_form in (False, True):
            attn, feat, dout = (t.cuda() for t in pc.operands(geom, 100 + k, split_form))
            for psa_type in (0, 1):
                stats = torch.empty((n, h * w, 2), device="cuda")
                y = torch.empty_like(feat)
                dfeat = torch.empty_like(feat)
                dattn = torch.empty_like(attn)
                assert lib.semseg_psa_attend(0, psa_type, p(attn), mh * mw, p(feat), lo(feat), c, p(stats), p(y), lo(y), c,
                                             n, h, w, mh, mw, c, scale, None) == 0, lib.semseg_last_error()
                assert lib.semseg_psa_attend(1, psa_type, p(attn), mh * mw, p(dout), lo(dout), c, p(stats), p(dfeat),
                                             lo(dfeat), c, n, h, w, mh, mw, c, scale, None) == 0, lib.semseg_last_error()
                assert lib.semseg_psa_attend_bwd_attn(psa_type, p(attn), mh * mw, p(stats), p(feat), lo(feat), c, p(y),
                                                      lo(y), c, p(dout), lo(dout), c, p(dattn), n, h, w, mh, mw, c, scale,
                                                      None) == 0, lib.semseg_last_error()
                torch.cuda.synchronize()
                tag = "%s/t%d/%s" % (key, psa_type, "bf16x3" if split_form else "bf16")
                out[tag] = {"out": pc.digest(y), "stats": pc.digest(stats), "dfeat": pc.digest(dfeat),
                            "dattn": pc.digest(dattn)}
    with open(args.out, "w") as fh:
        json.dump({"device": torch.cuda.get_device_name(0), "digests": out}, fh, indent=1, sort_keys=True)
    print("wrote", args.out, len(out), "entries")


if __name__ == "__main__":
    main()
