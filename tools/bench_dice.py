"""Training-step cost of the Dice (+ cross-entropy) loss on the native tail against the default loss and the ATen tail.

Three arms run bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on copies of one seeded PSPNet50, the default `bf16` mode, one GPU:
  * ce        : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * dice_ce   : semseg_b200.losses.DiceLoss(ignore_index=255, ce_weight=1) on the native tail, graphed;
  * torch_dice: the same loss written in PyTorch (full-resolution softmax and one-hot target) as a DiceLoss subclass,
                so the network takes the ATen tail (F.interpolate -> criterion -> max), eager.
Workloads: ADE20K-shaped (473x473, 150 classes, 16 images) and Cityscapes-shaped (713x713, 19 classes, 2 and 8
images). The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up (eager
calls and, for the graphed arms, the capture) and is timed with CUDA events. Prints one JSON line per workload and arm:
the GPU, its power limit and SM clock (read in the same process), ms/step of every round, and the kernels per graphed
step. Not part of bench.py's contract.
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
from semseg_b200 import graphs  # noqa: E402
from semseg_b200.losses import DiceLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchDice(DiceLoss):
    """DiceLoss written in PyTorch under another type: the network takes the ATen tail and runs eagerly."""

    def forward(self, logits, target):
        c = logits.shape[1]
        valid = (target != self.ignore_index) & (target >= 0) & (target < c)
        t = torch.where(valid, target, torch.zeros_like(target))
        p = torch.softmax(logits, dim=1) * valid.unsqueeze(1)
        hot = F.one_hot(t, c).permute(0, 3, 1, 2).to(p.dtype) * valid.unsqueeze(1)
        inter = (p * hot).sum((0, 2, 3))
        n = hot.sum((0, 2, 3))
        s = p.sum((0, 2, 3)) + n
        dice = (2 * inter + self.smooth) / (s + self.smooth).clamp_min(self.eps)
        loss = ((1 - dice) * (n > 0)).sum() / c
        ce = F.cross_entropy(logits, torch.where(valid, target, torch.full_like(target, -100)), ignore_index=-100)
        return loss + self.ce_weight * ce


ARMS = {
    "ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
    "dice_ce": lambda: DiceLoss(ignore_index=255, ce_weight=1.0),
    "torch_dice": lambda: TorchDice(ignore_index=255, ce_weight=1.0),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:2,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dice measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    arms = args.arms.split(",")
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for wl in args.workloads.split(","):
        size, classes, n = (int(v) for v in wl.split(":"))
        torch.manual_seed(0)
        base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
        x, y = bench.synth_batch(n, size, classes, 100)
        x, y = x.to(dev), y.to(dev)
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
        for arm in arms:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload="PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU" % (
                size, size, classes, n), arm=arm, steps=args.steps, ms_per_step=[round(v, 2) for v in ms],
                img_per_s=round(n / (min(ms) / 1e3), 2),
                kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        del runs, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
