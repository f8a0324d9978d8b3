"""Training-step cost of pixel-wise knowledge distillation from a frozen PSPNet101 teacher on the native tail.

Arms, each running bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on a fresh copy of one seeded PSPNet50 student, the default `bf16` mode, one GPU:
  * ce          : nn.CrossEntropyLoss(ignore_index=255) on the native tail, the step replayed from CUDA graphs;
  * kd_output   : semseg_b200.losses.DistillationLoss(teacher, T=4, at='output') on the native tail, teacher forward
                  and KL term graphed with the step;
  * kd_logits   : the same with at='logits' (the KL of the 1/8-resolution maps);
  * torch_kd    : the 'output' loss written in PyTorch as a DistillationLoss subclass: the network takes the eager
                  route (F.interpolate of both maps -> log_softmax, KL, cross-entropy), eager;
  * teacher_fwd : the teacher's eval forward alone (under no_grad), per step of the same batch.
Workloads: ADE20K-shaped (473x473, 150 classes, 16 images) and Cityscapes-shaped (713x713, 19 classes, 2 and 8
images). The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up (eager
calls and, for the graphed arms, the capture) and is timed with CUDA events. Prints one JSON line per workload and arm:
the GPU, its power limit and SM clock (read in the same process), ms/step of every round, the peak memory of the
window and the kernels per graphed step. Not part of bench.py's contract.
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
from semseg_b200 import functional as SF  # noqa: E402
from semseg_b200.losses import DistillationLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchKD(DistillationLoss):
    """DistillationLoss written in PyTorch under another type: the network takes the eager route."""

    def forward(self, logits, target, teacher_logits=None):
        valid = (target != self.ignore_index) & (target >= 0) & (target < logits.shape[1])
        ce = F.cross_entropy(logits, torch.where(valid, target, torch.full_like(target, -100)), ignore_index=-100)
        if teacher_logits is None:
            return ce
        t = self.temperature
        lp = F.log_softmax(logits / t, dim=1)
        lq = F.log_softmax(teacher_logits / t, dim=1)
        kl = F.kl_div(lp, lq, reduction="sum", log_target=True) / (lp.numel() // lp.shape[1])
        return self.ce_weight * ce + self.kd_weight * t * t * kl


ARMS = {
    "ce": lambda teacher: nn.CrossEntropyLoss(ignore_index=255),
    "kd_output": lambda teacher: DistillationLoss(teacher, temperature=4.0, at="output"),
    "kd_logits": lambda teacher: DistillationLoss(teacher, temperature=4.0, at="logits"),
    "torch_kd": lambda teacher: TorchKD(teacher, temperature=4.0),
    "teacher_fwd": None,
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:2,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_kd measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    arms = args.arms.split(",")
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for wl in args.workloads.split(","):
        size, classes, n = (int(v) for v in wl.split(":"))
        torch.manual_seed(0)
        base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
        torch.manual_seed(1)
        teacher = PSPNet(layers=101, classes=classes, zoom_factor=8, pretrained=False).to(dev).eval()
        x, y = bench.synth_batch(n, size, classes, 100)
        x, y = x.to(dev), y.to(dev)
        runs = {arm: dict(ms=[], peak=[]) for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:          # a fresh copy per window: one arm's graph memory pool is held at a time
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats(dev)
                if arm == "teacher_fwd":
                    model = opt = None

                    def step():
                        with torch.no_grad(), SF.network_mode(False, False):
                            teacher._eval_logits_nhwc(x)
                else:
                    model = copy.deepcopy(base).to(dev)
                    model.criterion = ARMS[arm](teacher)
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
                runs[arm]["peak"].append(torch.cuda.max_memory_allocated(dev) / 2 ** 30)
                runs[arm]["kernels"] = graphs.launches_per_step(model) if model is not None else None
                del model, opt, step
        for arm in arms:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload="PSPNet50 student, PSPNet101 teacher, %dx%d, %d classes, %d images, "
                                  "bf16, one GPU" % (size, size, classes, n), arm=arm, steps=args.steps,
                                  ms_per_step=[round(v, 2) for v in ms],
                                  peak_gib=round(max(runs[arm]["peak"]), 2),
                                  kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        del runs, base, teacher
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
