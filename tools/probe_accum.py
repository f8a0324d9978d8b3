"""Accumulation-error probe: tensor-core fp32 accumulation vs an fp64 reference on bf16-exact operands, as a function
of the number of sequential MMA steps (K / 16). Output feeds DESIGN.md §4 (why long-K convs are K-sliced in bf16x3)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from semseg_b200 import ops

torch.backends.cudnn.allow_tf32 = False
g = torch.Generator(device="cuda").manual_seed(0)
for cin, k in [(64, 1), (256, 1), (1024, 1), (4096, 1), (512, 3), (4096, 3)]:
    n, h, w, cout = 2, 30, 30, 64
    x = torch.randn((n, h, w, cin), device="cuda", generator=g).to(torch.bfloat16)
    wt = (torch.randn((cout, cin, k, k), device="cuda", generator=g) / (cin * k * k) ** 0.5).to(torch.bfloat16).float()
    for positive in (False, True):
        xx = x.abs() if positive else x
        ww = wt.abs() if positive else wt
        y, _ = ops.conv_fprop(xx, ops.pack_weights(ww).wf, cout, ops.conv_taps(k, 1), epi=ops.EPI_F32)
        ref = F.conv2d(xx.double().permute(0, 3, 1, 2), ww.double(), padding=k // 2).permute(0, 2, 3, 1)
        ref32 = F.conv2d(xx.float().permute(0, 3, 1, 2), ww, padding=k // 2).permute(0, 2, 3, 1)
        e = ((y.double() - ref).norm() / ref.norm()).item()
        e32 = ((ref32.double() - ref).norm() / ref.norm()).item()
        bias = ((y.double() - ref) * ref.sign()).sum().item() / ref.abs().sum().item()
        print("K=%6d steps=%5d %s: tensor core rel %.2e (signed bias %.2e) | cuDNN fp32 rel %.2e" %
              (cin * k * k, cin * k * k // 16, "pos" if positive else "rnd", e, bias, e32), flush=True)
