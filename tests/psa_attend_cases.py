"""Seeded operands of the fused PSA attention entry points (semseg_psa_attend, semseg_psa_attend_bwd_attn), shared by
tests/golden/make_psa_attend_golden.py, which stored the digests of what the window + softmax kernels computed on them,
and by the GPU test that replays those digests."""
import hashlib

import torch

C = 512
SCALE = 1.0 / 3.0
# (N, H, W, mH, mW). On a 132-SM H100 the first three run 8-row forward tiles and the last 64-row forward and 128-row
# logit-gradient tiles; every case ends in a partial tile. Masks smaller than 2H-1 x 2W-1 in all but the first.
CASES = {
    "n2_13x13_m25": (2, 13, 13, 25, 25),
    "n1_9x12_m9x7": (1, 9, 12, 9, 7),
    "n1_20x23_m15x11": (1, 20, 23, 15, 11),
    "n2_66x66_m17": (2, 66, 66, 17, 17),
}


def split(x):
    """fp32 -> split activation [2, ...]: hi = bf16(x), lo = bf16(x - hi)."""
    hi = x.to(torch.bfloat16)
    return torch.stack([hi, (x - hi.float()).to(torch.bfloat16)])


def operands(geom, seed, split_form, a_cols=None):
    """(attn fp32 [N,H,W,a_cols], feat, dout) on the CPU; feat / dout plain bf16 or split. a_cols defaults to mH*mW."""
    n, h, w, mh, mw = geom
    g = torch.Generator().manual_seed(seed)
    attn = torch.randn((n, h, w, a_cols or mh * mw), generator=g) * 2
    feat = torch.relu(torch.randn((n, h, w, C), generator=g))
    dout = torch.randn((n, h, w, C), generator=g)
    if split_form:
        return attn, split(feat), split(dout)
    return attn, feat.to(torch.bfloat16), dout.to(torch.bfloat16)


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()
