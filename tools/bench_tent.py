"""Cost of a TENT test-time adaptation step (semseg_b200.adapt.Tent) against the full training step.

Three arms on copies of one seeded PSPNet50, the default `bf16` mode, one GPU, PSPNet50 473x473, 150 classes, 16 images:
  * train_ce    : bench.py's training step (model(input, target) with nn.CrossEntropyLoss(ignore_index=255),
                  loss = main + 0.4 aux, zero_grad, backward, SGD with the reference's 8 parameter groups), graphed;
  * tent        : one Tent call (steps=1): forward, backward and FusedSGD step of the BatchNorm gamma / beta on the
                  fused upsample + entropy tail, graphed; no weight gradient is computed;
  * tent_torch  : the same Tent step with the entropy written in PyTorch (log_softmax, exp, sum) under an EntropyLoss
                  subclass: the fused gate refuses it, so the network takes the ATen tail (F.interpolate -> criterion)
                  and runs eagerly.
The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up (eager calls and, for
the graphed arms, the capture) and is timed with CUDA events. Prints one JSON line per arm: the GPU, its power limit and
SM clock (read in the same process), ms/step of every round, img/s of the best round and the kernels per graphed step.
Not part of bench.py's contract.
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

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402
from semseg_b200.adapt import Tent  # noqa: E402
from semseg_b200.losses import EntropyLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchEntropyLoss(EntropyLoss):
    """EntropyLoss written in PyTorch under another type: the network takes the ATen tail and runs eagerly."""

    def forward(self, logits, target):
        c = logits.shape[1]
        lab = (target != self.ignore_index) & (target >= 0) & (target < c)
        unl = target == self.ignore_index
        t = torch.where(lab, target, torch.zeros_like(target))
        logp = torch.log_softmax(logits, dim=1)
        ce = -logp.gather(1, t.unsqueeze(1)).squeeze(1)
        ent = -(logp.exp() * logp).sum(1)
        return (self.ce_weight * (ce * lab).sum() / lab.sum().clamp(min=1) +
                self.ent_weight * (ent * unl).sum() / unl.sum().clamp(min=1))


ARMS = ("train_ce", "tent", "tent_torch")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=3, help="windows per arm, the arms alternating")
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tent measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    arms = args.arms.split(",")
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    size, classes, n = args.size, args.classes, args.images
    torch.manual_seed(0)
    base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
    x, y = bench.synth_batch(n, size, classes, 100)
    x, y = x.to(dev), y.to(dev)
    runs = {arm: dict(ms=[]) for arm in arms}
    for _ in range(args.rounds):
        for arm in arms:              # a fresh copy per window: one arm's graph memory pool is held at a time
            model = copy.deepcopy(base).to(dev)
            if arm == "train_ce":
                model.criterion = nn.CrossEntropyLoss(ignore_index=255)
                opt = bench.build_optimizer(model, "psp")

                def step():
                    _, main_loss, aux_loss = model(x, y)
                    loss = main_loss + 0.4 * aux_loss
                    opt.zero_grad()
                    loss.backward()
                    opt.step()
            else:
                tent = Tent(model, lr=1e-3, momentum=0.9)
                if arm == "tent_torch":
                    model.criterion = TorchEntropyLoss(ignore_index=255, ent_weight=1.0, ce_weight=0.0)

                def step():
                    tent(x)

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
            del model, step
            opt = tent = None
            torch.cuda.empty_cache()
    for arm in arms:
        ms = runs[arm]["ms"]
        print(json.dumps(dict(info, workload="PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU" % (
            size, size, classes, n), arm=arm, steps=args.steps, ms_per_step=[round(v, 2) for v in ms],
            img_per_s=round(n / (min(ms) / 1e3), 2), kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)


if __name__ == "__main__":
    main()
