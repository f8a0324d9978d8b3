"""Accumulation-error probe: tensor-core fp32 accumulation vs an fp64 reference on bf16-exact operands, as a function
of the number of sequential MMA steps (K / 16). Output feeds DESIGN.md §4 (why long-K convs are K-sliced in bf16x3, and
why the FP8 convs promote their accumulation)."""
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

# e4m3 leg: the FP8 conv (semseg_b200/fp8.py) with and without promotion (each 128-channel K block's tensor-core partial
# added into an fp32 accumulator, or one tensor-core accumulation chain over all of K), against fp64 on the same
# e4m3-exact operands. Scale 1, shift 0, no ReLU: the bf16 output rounding (2^-9 relative) is the floor of both.
for cin, k in [(128, 1), (1024, 1), (4096, 1), (512, 3), (2048, 3), (4096, 3)]:
    n, h, w, cout = 2, 30, 30, 128
    for positive in (False, True):
        x = torch.randn((n, h, w, cin), device="cuda", generator=g)
        wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) / (cin * k * k) ** 0.5
        if positive:
            x, wt = x.abs(), wt.abs()
        xb = x.to(torch.bfloat16)
        qs = 448.0 / float(xb.float().abs().max())
        x8 = ops.fp8_quantize(xb, qs)
        wf8, sw = ops.fp8_pack_weights(wt)
        xd = x8.float().double() / qs
        wd = (wf8.float().double().permute(1, 2, 0).reshape(cout, cin, k, k) * sw.double()[:, None, None, None])
        ref = F.conv2d(xd.permute(0, 3, 1, 2), wd, padding=k // 2).permute(0, 2, 3, 1)
        scale = (sw / qs).contiguous()
        zero = torch.zeros(cout, device="cuda")
        res = []
        for promote in (True, False):
            y, _ = ops.conv_fprop_e4m3(x8, wf8.contiguous(), cout, ops.conv_taps(k, 1), scale=scale, shift=zero,
                                       promote=promote)
            e = ((y.double() - ref).norm() / ref.norm()).item()
            bias = ((y.double() - ref) * ref.sign()).sum().item() / ref.abs().sum().item()
            res.append((e, bias))
        print("e4m3 K=%6d %s: promoted rel %.2e (signed bias %.2e) | unpromoted rel %.2e (signed bias %.2e)" %
              (cin * k * k, "pos" if positive else "rnd", res[0][0], res[0][1], res[1][0], res[1][1]), flush=True)
