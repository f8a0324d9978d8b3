"""Training-step cost of the RMI loss (with its BCE term) on the native tail against the default loss and the ATen tail.

Three arms run bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on copies of one seeded PSPNet50, the default `bf16` mode, one GPU:
  * ce       : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * rmi      : semseg_b200.losses.RMILoss(ignore_index=255) (bce_weight 0.5) on the native tail, graphed;
  * torch_rmi: the same loss written in PyTorch the way the paper's code writes it (full-resolution sigmoid and one-hot
               maps, 4x4 average pooling, nine shifted views, float64 9x9 algebra) as an RMILoss subclass, so the
               network takes the ATen tail (F.interpolate -> criterion -> max), eager.
Workload: ADE20K-shaped (473x473, 150 classes, 16 images) by default. The arms alternate over `--rounds` rounds; each
timed window of `--steps` steps follows the warm-up (eager calls and, for the graphed arms, the capture) and is timed
with CUDA events. Prints one JSON line per workload and arm: the GPU, its power limit and SM clock (read in the same
process), ms/step of every round, peak memory, and the kernels per graphed step. Not part of bench.py's contract.
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
from semseg_b200.losses import RMILoss  # noqa: E402
from tests.rmi_oracle import rmi_literal  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchRMI(RMILoss):
    """RMILoss written in PyTorch under another type: the network takes the ATen tail and runs eagerly."""

    def forward(self, logits, target):
        return rmi_literal(logits, target, self.ignore_index, self.bce_weight, self.pos_alpha,
                           self.ce_weight).to(logits.dtype)


ARMS = {
    "ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
    "rmi": lambda: RMILoss(ignore_index=255),
    "torch_rmi": lambda: TorchRMI(ignore_index=255),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rmi measures on a GPU; there is no CPU arm"
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
                torch.cuda.reset_peak_memory_stats(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
                runs[arm]["ms"].append(e0.elapsed_time(e1) / args.steps)
                runs[arm]["kernels"] = graphs.launches_per_step(model)
                runs[arm]["peak_gb"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)
                del model, opt, step
                torch.cuda.empty_cache()
        for arm in arms:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload="PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU" % (
                size, size, classes, n), arm=arm, steps=args.steps, ms_per_step=[round(v, 2) for v in ms],
                img_per_s=round(n / (min(ms) / 1e3), 2),
                peak_memory_gb=runs[arm]["peak_gb"], kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        del runs, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
