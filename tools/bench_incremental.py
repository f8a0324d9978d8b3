"""Training-step cost of class-incremental training (losses.IncrementalLoss, MiB's unbiased cross-entropy and
distillation) on the native tail, at ADE20K 100-50's split: a PSPNet50 student of 150 classes grown from a 100-class
network of the previous step.

Arms, each running bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the
reference's 8 parameter groups) on a fresh copy of one seeded PSPNet50 student, the default `bf16` mode, one GPU:
  * ce          : nn.CrossEntropyLoss(ignore_index=255) on the native tail, graphed;
  * kd          : losses.DistillationLoss from a 150-class PSPNet50 teacher (T = 1, at='output'), graphed;
  * incremental : losses.IncrementalLoss from the 100-class PSPNet50 teacher (kd_weight 10, at='output'), graphed;
  * torch_mib   : the same losses written in PyTorch as an IncrementalLoss subclass: the network takes the eager route
                  (F.interpolate of both maps -> logsumexp over the class subsets, softmax of the teacher), eager.
The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up (eager calls and,
for the graphed arms, the capture) and is timed with CUDA events. Prints one JSON line per arm with the GPU, its power
limit and SM clock (read in the same process), ms/step and img/s of every round and the peak memory of the window.
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
from semseg_b200.incremental import expand_classifier  # noqa: E402
from semseg_b200.losses import DistillationLoss, IncrementalLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchMiB(IncrementalLoss):
    """IncrementalLoss written in PyTorch under another type: the network takes the eager route."""

    def forward(self, logits, target, teacher_logits=None):
        c, c_old = logits.shape[1], self.c_old
        valid = (target != self.ignore_index) & (target >= 0) & (target < c)
        tc = torch.where(valid, target, torch.zeros_like(target))
        lse_all = torch.logsumexp(logits, 1)
        lse_old = torch.logsumexp(logits[:, :c_old], 1)
        s_t = logits.gather(1, tc.unsqueeze(1)).squeeze(1)
        pix = torch.where(tc < c_old, lse_all - lse_old, lse_all - s_t)
        ce = torch.where(valid, pix, torch.zeros_like(pix)).sum() / valid.sum().clamp(min=1)
        if teacher_logits is None:
            return ce
        q = torch.softmax(self.alpha * teacher_logits, 1)
        lse_b = torch.logsumexp(torch.cat([logits[:, :1], logits[:, c_old:]], 1), 1)
        k = q[:, 0] * (lse_b - lse_all) + (q[:, 1:] * (logits[:, 1:c_old] - lse_all.unsqueeze(1))).sum(1)
        return self.ce_weight * ce + self.kd_weight * (-k / c_old).mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--old", type=int, default=100, help="classes of the previous step")
    ap.add_argument("--classes", type=int, default=150, help="classes after this step")
    ap.add_argument("--arms", default="ce,kd,incremental,torch_mib")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_incremental measures on a GPU; there is no CPU arm"
    from semseg_b200.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    arms = args.arms.split(",")
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    torch.manual_seed(0)
    old = PSPNet(layers=50, classes=args.old, zoom_factor=8, pretrained=False).to(dev).eval()
    base = expand_classifier(copy.deepcopy(old).train(), args.classes - args.old)
    torch.manual_seed(1)
    kd_teacher = PSPNet(layers=50, classes=args.classes, zoom_factor=8, pretrained=False).to(dev).eval()
    crits = {
        "ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
        "kd": lambda: DistillationLoss(kd_teacher),
        "incremental": lambda: IncrementalLoss(old),
        "torch_mib": lambda: TorchMiB(old),
    }
    x, y = bench.synth_batch(args.images, args.size, args.classes, 100)
    x, y = x.to(dev), y.to(dev)
    runs = {arm: dict(ms=[], peak=[]) for arm in arms}
    for _ in range(args.rounds):
        for arm in arms:              # a fresh copy per window: one arm's graph memory pool is held at a time
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            model = copy.deepcopy(base)
            model.criterion = crits[arm]()
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
            del model, opt, step
    for arm in arms:
        ms = runs[arm]["ms"]
        print(json.dumps(dict(info, workload="PSPNet50 %d -> %d classes, %dx%d, %d images, bf16, one GPU" % (
            args.old, args.classes, args.size, args.size, args.images), arm=arm, steps=args.steps,
            ms_per_step=[round(v, 2) for v in ms], img_per_s=[round(args.images * 1e3 / v, 2) for v in ms],
            peak_gib=round(max(runs[arm]["peak"]), 2))), flush=True)


if __name__ == "__main__":
    main()
