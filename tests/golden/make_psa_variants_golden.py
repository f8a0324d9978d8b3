"""Generate the PSANet variant fixtures tests/golden/psanet50_65_<variant>.npz from the REAL reference (hszhao/semseg),
for the PSA options the main fixture (psanet50_65.npz: psa_type 2, windowed mask, softmax) does not cover: compact mode
and psa_softmax=False.

    python tests/golden/make_psa_variants_golden.py          # minutes: four PSANet50 on CPU

As tests/golden/make_golden.py does, it copies the reference to a scratch dir and runs this file again with `--worker` in
a subprocess whose PYTHONPATH holds ONLY that copy, so `model.psanet` is the reference's own module. The worker writes what
`_ref_worker.run_model` writes (losses, train argmax, gradient norms and heads, sampled eval logits, a running mean) plus
`wsum/<parameter>` = (sum |w|, sum w) of the freshly seeded variant. PSANet50, 65 x 65 input, 150 classes, the seed-321
input of the main fixture; the mask sized as tool/train.py:63-70 sizes it (compact: 5 x 5, windowed: 9 x 9).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SEMSEG_REFERENCE", "/root/reference")
SCRATCH = "/tmp/semseg_ref_copy"

# tag -> (psa_type, compact, psa_softmax)
VARIANTS = {
    "psanet50_65_t2_compact": (2, True, True),           # collect (identity) and distribute (transposed) dense forms
    "psanet50_65_t2_nosoftmax": (2, False, False),
    "psanet50_65_t1_compact_nosoftmax": (1, True, False),
    "psanet50_65_t0_compact": (0, True, True),
}
WSUM_KEYS = ["layer0.0.weight", "psa.reduce.0.weight", "psa.attention.3.weight", "psa.attention_p.3.weight",
             "psa.proj.0.weight", "cls.0.weight"]
GRAD_KEYS = ["psa.reduce.0.weight", "psa.attention.3.weight", "psa.proj.1.weight"]


def mask_size(compact, size=65, shrink=2):
    """tool/train.py:63-70 for a square crop: h of the shrunk feature map (compact) or 2h - 1 (windowed)."""
    h = (size - 1) // (8 * shrink) + 1
    return h if compact else 2 * h - 1


def worker():
    import numpy as np
    import torch
    import _ref_worker as rw                           # tests/golden, this file's directory (sys.path[0])
    from model.psanet import PSANet
    for tag, (psa_type, compact, softmax) in VARIANTS.items():
        mask = mask_size(compact)
        torch.manual_seed(0)
        m = PSANet(layers=50, classes=150, zoom_factor=8, dropout=0.0, psa_type=psa_type, compact=compact,
                   shrink_factor=2, mask_h=mask, mask_w=mask, normalization_factor=1.0, psa_softmax=softmax,
                   pretrained=False)
        sd = m.state_dict()
        wsum = {"wsum/" + k: np.array(v, dtype=np.float64) for k, v in rw.checksum({k: sd[k] for k in WSUM_KEYS
                                                                                   if k in sd}).items()}
        x, y = rw.synth(2, 65, 65, 150, seed=321)
        rw.run_model(m, x, y, tag, GRAD_KEYS + (["psa.attention_p.3.weight"] if psa_type == 2 else []))
        path = os.path.join(rw.OUT, tag + ".npz")
        res = dict(np.load(path))
        res.update(wsum)
        np.savez_compressed(path, **res)


def main():
    if not os.path.isdir(REF):
        sys.exit("reference tree not found at %s" % REF)
    if not os.path.isdir(SCRATCH):
        shutil.copytree(REF, SCRATCH, ignore=shutil.ignore_patterns(".git"))
    env = dict(os.environ)
    env["PYTHONPATH"] = SCRATCH
    env["GOLDEN_OUT"] = HERE
    subprocess.check_call([sys.executable, os.path.abspath(__file__), "--worker"], cwd=SCRATCH, env=env)


if __name__ == "__main__":
    worker() if "--worker" in sys.argv[1:] else main()
