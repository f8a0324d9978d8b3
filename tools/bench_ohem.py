"""Training-step cost of OHEM cross-entropy: the native OHEM tail against the default loss and a torch OHEM module.

Three arms run bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on copies of one seeded PSPNet50, the default `bf16` mode, one GPU:
  * ce        : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * ohem      : semseg_b200.losses.OhemCrossEntropyLoss(thresh=0.7, min_kept=100000) on the native tail, graphed;
  * torch_ohem: the same loss written in PyTorch (softmax, gather, sort, masked mean), as a user would write it; the
                network takes the ATen tail (F.interpolate -> criterion -> max) and runs eagerly.
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
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402
from semseg_b200.losses import OhemCrossEntropyLoss  # noqa: E402


class TorchOhemCrossEntropy(nn.Module):
    """The OHEM contract of semseg_b200.losses written in PyTorch: what the network ran before the native form."""

    def __init__(self, ignore_index=255, thresh=0.7, min_kept=100000):
        super(TorchOhemCrossEntropy, self).__init__()
        self.ignore_index, self.thresh, self.min_kept = ignore_index, thresh, min_kept

    def forward(self, logits, target):
        valid = (target != self.ignore_index).view(-1)
        nll = F.cross_entropy(logits, target, ignore_index=self.ignore_index, reduction="none").view(-1)
        t = target.clone()
        t[t == self.ignore_index] = 0
        pt = F.softmax(logits, dim=1).gather(1, t.unsqueeze(1)).view(-1)[valid]
        pt, order = pt.sort()
        kth = pt[min(self.min_kept, pt.numel() - 1)]
        kept = pt < torch.clamp(kth, min=self.thresh)
        return nll[valid][order][kept].mean()


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in q.stdout.strip().split(",")] if q.stdout.strip() else []
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = (vals + ["unknown"] * 3)[:3]
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = info["sm_clock"] = "unknown"
    return info


ARMS = {
    "ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
    "ohem": lambda: OhemCrossEntropyLoss(ignore_index=255, thresh=0.7, min_kept=100000),
    "torch_ohem": lambda: TorchOhemCrossEntropy(ignore_index=255, thresh=0.7, min_kept=100000),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:2,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ohem measures on a GPU; there is no CPU arm"
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
