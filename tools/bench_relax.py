"""Training-step cost of boundary label relaxation on the native tail against the default loss and the ATen tail.

Four arms run bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on copies of one seeded PSPNet50, the default `bf16` mode, one GPU:
  * ce         : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * relax_b1   : semseg_b200.losses.BoundaryRelaxationLoss(border=1) on the native tail, graphed;
  * relax_b2   : the same at border 2;
  * torch_relax: the border-1 loss written in PyTorch with a multi-hot [N, C, H, W] target (one-hot, max-pool,
                 logsumexp) under a BoundaryRelaxationLoss subclass, the route such a criterion takes without the native
                 form: the ATen tail (F.interpolate -> criterion -> max), eager.
Workloads: ADE20K-shaped (473x473, 150 classes, 16 images) and Cityscapes-shaped (713x713, 19 classes, 8 images), with
bench.py's synthetic images and labels constant on 24 x 24 tiles (bench.py's per-pixel random labels would make every
pixel a boundary pixel). The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the
warm-up (eager calls and, for the graphed arms, the capture) and is timed with CUDA events. Then the relaxation kernels
alone (label sets + forward + reduce, rows + cols) against the plain tail's on the head's fp32 NHWC logits, timed with
CUDA events over `--kernel-iters` calls each. Prints one JSON line per workload and arm, and per workload for the
kernels: the GPU, its power limit and SM clock (read in the same process). Not part of bench.py's contract.
"""
import argparse
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs, ops  # noqa: E402
from semseg_b200.losses import BoundaryRelaxationLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchRelaxLoss(BoundaryRelaxationLoss):
    """BoundaryRelaxationLoss written in PyTorch under another type: the network takes the ATen tail, eagerly."""

    def forward(self, logits, target):
        c = logits.shape[1]
        valid = (target != self.ignore_index) & (target >= 0) & (target < c)
        t = torch.where(valid, target, torch.zeros_like(target))
        onehot = F.one_hot(t, c).permute(0, 3, 1, 2).float() * valid.unsqueeze(1)
        s = F.max_pool2d(onehot, 2 * self.border + 1, stride=1, padding=self.border) > 0
        pix = torch.logsumexp(logits, 1) - torch.logsumexp(logits.masked_fill(~s, float("-inf")), 1)
        return (pix * valid).sum() / valid.sum().clamp(min=1)


ARMS = {
    "ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
    "relax_b1": lambda: BoundaryRelaxationLoss(border=1),
    "relax_b2": lambda: BoundaryRelaxationLoss(border=2),
    "torch_relax": lambda: TorchRelaxLoss(border=1),
}


def _blocky_labels(n, size, classes, dev, block=24):
    """Labels constant on block x block tiles with 5 % of the pixels ignored: a label map with interior pixels and
    boundaries, unlike bench.py's per-pixel random labels (where every pixel is a boundary pixel)."""
    g = torch.Generator().manual_seed(100)
    nb = -(-size // block)
    y = torch.randint(0, classes, (n, nb, nb), generator=g)
    y = y.repeat_interleave(block, 1).repeat_interleave(block, 2)[:, :size, :size].contiguous()
    y[torch.rand((n, size, size), generator=g) < 0.05] = 255
    return y.to(dev)


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _kernels(n, size, classes, y, iters):
    """ms per call of the tail kernels alone at the network's head shape (zoom 8)."""
    h = (size - 1) // 8 + 1
    g = torch.Generator(device="cuda").manual_seed(0)
    logits = torch.randn((n, h, h, classes), device="cuda", generator=g) * 3
    one = torch.ones(1, device="cuda")
    out = {}
    info, _, lse = ops.upsample_ce_fwd(logits, y, 255)
    out["ce_fwd_ms"] = _time(lambda: ops.upsample_ce_fwd(logits, y, 255), iters)
    out["ce_bwd_ms"] = _time(lambda: ops.upsample_ce_bwd(logits, y, 255, lse, info, one), iters)
    for border in (1, 2, 4):
        info, _, lse, sets, lq = ops.upsample_ce_relax_fwd(logits, y, 255, None, border)
        out["relax_b%d_fwd_ms" % border] = _time(lambda: ops.upsample_ce_relax_fwd(logits, y, 255, None, border), iters)
        out["relax_b%d_bwd_ms" % border] = _time(lambda: ops.upsample_ce_relax_bwd(logits, lse, sets, lq, info, one),
                                                 iters)
        valid = (y != 255) & (y >= 0) & (y < classes)
        tag = sets[:y.numel()].view_as(y)
        out["relax_b%d_boundary_share" % border] = round(float((tag >= classes).sum()) / float(valid.sum()), 4)
    return {k: round(v, 3) if isinstance(v, float) and k.endswith("ms") else v for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    ap.add_argument("--kernel-iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_relax measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    arms = args.arms.split(",")
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for wl in args.workloads.split(","):
        size, classes, n = (int(v) for v in wl.split(":"))
        torch.manual_seed(0)
        base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
        x, _ = bench.synth_batch(n, size, classes, 100)
        x, y = x.to(dev), _blocky_labels(n, size, classes, dev)
        runs = {arm: dict(ms=[]) for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:          # a fresh copy per window: one arm's graph memory pool is held at a time
                model = copy.deepcopy(base).to(dev)
                model.criterion = ARMS[arm]()
                opt = bench.build_optimizer(model, "psp")

                def step():
                    _, main_loss, aux_loss = model(x, y)
                    loss = main_loss + 0.4 * aux_loss
                    opt.zero_grad()
                    loss.backward()
                    opt.step()

                for _ in range(n_warm):
                    step()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
                runs[arm]["ms"].append(e0.elapsed_time(e1) / args.steps)
                runs[arm]["kernels"] = graphs.launches_per_step(model)
                del model, opt, step
                torch.cuda.empty_cache()
        wname = "PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU" % (size, size, classes, n)
        for arm in arms:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload=wname, arm=arm, steps=args.steps,
                                  ms_per_step=[round(v, 2) for v in ms], img_per_s=round(n / (min(ms) / 1e3), 2),
                                  kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        print(json.dumps(dict(info, workload=wname, arm="kernels", **_kernels(n, size, classes, y, args.kernel_iters))),
              flush=True)
        del runs, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
