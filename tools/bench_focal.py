"""Training-step cost of the focal loss on the native tail against the default loss and the ATen tail.

Four arms run bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on copies of one seeded PSPNet50, the default `bf16` mode, one GPU:
  * ce            : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * focal         : semseg_b200.losses.FocalLoss(gamma=2, ignore_index=255) on the native tail, graphed;
  * focal_weighted: the same with class weights, native, graphed;
  * torch_focal   : the weighted focal loss written in PyTorch (log_softmax, gather, pow) under a FocalLoss subclass,
                    the route such a criterion takes without the native form: the ATen tail (F.interpolate ->
                    criterion -> max), eager.
The class weights are fixed seeded positive values in [0.5, 1.5). Workloads: ADE20K-shaped (473x473, 150 classes, 16
images) and Cityscapes-shaped (713x713, 19 classes, 2 and 8 images). The arms alternate over `--rounds` rounds; each
timed window of `--steps` steps follows the warm-up (eager calls and, for the graphed arms, the capture) and is timed
with CUDA events. Prints one JSON line per workload and arm: the GPU, its power limit and SM clock (read in the same
process), ms/step of every round, and the kernels per graphed step. Not part of bench.py's contract.
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
from semseg_b200.losses import FocalLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchFocalLoss(FocalLoss):
    """FocalLoss written in PyTorch under another type: the network takes the ATen tail and runs eagerly."""

    def forward(self, logits, target):
        valid = target != self.ignore_index
        t = torch.where(valid, target, torch.zeros_like(target))
        logp_t = F.log_softmax(logits, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
        pix = torch.pow(1.0 - logp_t.exp(), self.gamma) * -logp_t
        if self.weight is not None:
            pix = pix * self.weight[t]
        return (pix * valid).sum() / valid.sum().clamp(min=1)


def _class_weights(classes, dev):
    g = torch.Generator().manual_seed(1234)
    return (torch.rand(classes, generator=g) + 0.5).to(dev)


ARMS = {
    "ce": lambda w: nn.CrossEntropyLoss(ignore_index=255),
    "focal": lambda w: FocalLoss(gamma=2.0, ignore_index=255),
    "focal_weighted": lambda w: FocalLoss(gamma=2.0, weight=w, ignore_index=255),
    "torch_focal": lambda w: TorchFocalLoss(gamma=2.0, weight=w, ignore_index=255),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:2,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_focal measures on a GPU; there is no CPU arm"
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
        weight = _class_weights(classes, dev)
        runs = {arm: dict(ms=[]) for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:          # a fresh copy per window: one arm's graph memory pool is held at a time
                model = copy.deepcopy(base).to(dev)
                model.criterion = ARMS[arm](weight.clone())
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
