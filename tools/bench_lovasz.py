"""Training-step cost of the Lovász-Softmax (+ cross-entropy) loss on the native tail against the default loss and
Berman's PyTorch statement on the ATen tail.

Three arms run bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on copies of one seeded PSPNet50, the default `bf16` mode, one GPU:
  * ce           : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * lovasz_ce    : semseg_b200.losses.LovaszSoftmaxLoss(ignore_index=255, ce_weight=1) on the native tail, graphed;
  * torch_lovasz : the same loss as Berman's lovasz_softmax code writes it (full-resolution softmax, then per class a
                   torch.sort of every pixel's error, a cumsum and a dot product) plus F.cross_entropy, as a
                   LovaszSoftmaxLoss subclass, so the network takes the ATen tail (F.interpolate -> criterion), eager.
Workloads: ADE20K-shaped (473x473, 150 classes, 16 images) and Cityscapes-shaped (713x713, 19 classes, 2 and 8
images). The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up and is
timed with CUDA events. Prints one JSON line per workload and arm: the GPU, its power limit and SM clock (read in the
same process), ms/step of every round, the peak memory of the timed window (the larger of the allocated peak and the reserved
memory, which holds the graph pools), the kernels per graphed step and
the number of classes present in the batch's target. Not part of bench.py's contract.
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
from semseg_b200.losses import LovaszSoftmaxLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


def _lovasz_grad(gt_sorted):
    gts = gt_sorted.sum()
    intersection = gts - gt_sorted.cumsum(0)
    union = gts + (1 - gt_sorted).cumsum(0)
    jaccard = 1.0 - intersection / union
    jaccard[1:] = jaccard[1:] - jaccard[:-1]
    return jaccard


class TorchLovasz(LovaszSoftmaxLoss):
    """Berman's lovasz_softmax (classes='present', per_image=False) plus CE, under another type: the network takes the
    ATen tail and runs eagerly."""

    def forward(self, logits, target):
        c = logits.shape[1]
        valid = (target != self.ignore_index) & (target >= 0) & (target < c)
        probas = torch.softmax(logits, dim=1).permute(0, 2, 3, 1).reshape(-1, c)[valid.reshape(-1)]
        labels = target.reshape(-1)[valid.reshape(-1)]
        losses = []
        for k in range(c):
            fg = (labels == k).float()
            if fg.sum() == 0:
                continue
            errors = (fg - probas[:, k]).abs()
            errors_sorted, perm = torch.sort(errors, 0, descending=True)
            losses.append(torch.dot(errors_sorted, _lovasz_grad(fg[perm])))
        loss = torch.stack(losses).mean()
        ce = F.cross_entropy(logits, torch.where(valid, target, torch.full_like(target, -100)), ignore_index=-100)
        return loss + self.ce_weight * ce


ARMS = {
    "ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
    "lovasz_ce": lambda: LovaszSoftmaxLoss(ignore_index=255, ce_weight=1.0),
    "torch_lovasz": lambda: TorchLovasz(ignore_index=255, ce_weight=1.0),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:2,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lovasz measures on a GPU; there is no CPU arm"
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
        present = int(torch.unique(y[(y >= 0) & (y < classes)]).numel())
        runs = {arm: dict(ms=[], peak=[]) for arm in arms}
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
                torch.cuda.reset_peak_memory_stats(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
                runs[arm]["ms"].append(e0.elapsed_time(e1) / args.steps)
                # the graphed arms' memory lives in their graph pools: reserved, not in the allocated peak
                runs[arm]["peak"].append(max(torch.cuda.max_memory_allocated(dev), torch.cuda.memory_reserved(dev))
                                         / 2 ** 30)
                runs[arm]["kernels"] = graphs.launches_per_step(model)
                del model, opt, step
                torch.cuda.empty_cache()
        for arm in arms:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload="PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU" % (
                size, size, classes, n), arm=arm, steps=args.steps, ms_per_step=[round(v, 2) for v in ms],
                img_per_s=round(n / (min(ms) / 1e3), 2), peak_gib=round(max(runs[arm]["peak"]), 2),
                present_classes=present, kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        del runs, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
