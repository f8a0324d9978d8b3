"""Training-step cost of mean-teacher training on the native tail: an optim.ModelEMA of the student as the teacher of
the distillation and pseudo-label losses, updated after every optimizer step.

Arms, each running bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, FusedSGD with the
reference's 8 parameter groups) on a fresh copy of one seeded PSPNet50 student, the default `bf16` mode, one GPU; the
first half of every batch is labelled, the second half unlabelled (an all-ignore target):
  * ce          : nn.CrossEntropyLoss(ignore_index=255) on the native tail, graphed;
  * kd_frozen   : losses.DistillationLoss from a frozen PSPNet50 teacher (T = 1), graphed;
  * kd_ema      : losses.DistillationLoss(ema.module) + ema.update(model) after the step, graphed;
  * pl_ema      : losses.PseudoLabelLoss(ema.module, threshold=0.95) + ema.update(model), graphed;
  * torch_pl    : the pseudo-label loss written in PyTorch as a PseudoLabelLoss subclass with a
                  torch.optim.swa_utils.AveragedModel teacher (get_ema_multi_avg_fn, buffers averaged) updated by its
                  update_parameters: the network takes the eager route (F.interpolate of both maps, softmax, masked CE);
  * ema_update  : ema.update(model) alone (the Python call included: it bounds the rate when nothing else runs), and
  * ema_launch  : the bare semseg_ema_multi launch update issues, both timed with CUDA events over the window; bytes =
                  12 per fp32 element (read shadow and source, write shadow), reported against the 3.35 TB/s H100 SXM
                  data-sheet HBM3 bandwidth.
Workloads: ADE20K-shaped (473x473, 150 classes, 16 images) and Cityscapes-shaped (713x713, 19 classes, 2 and 8
images). The arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up (eager
calls and, for the graphed arms, the capture). Prints one JSON line per workload and arm: the GPU, its power limit and
SM clock (read in the same process), ms/step of every round, the peak memory of the window and the kernels per graphed
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
from semseg_b200 import graphs, ops  # noqa: E402
from semseg_b200.losses import DistillationLoss, PseudoLabelLoss  # noqa: E402
from semseg_b200.optim import ModelEMA  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

HBM_DATASHEET_TBS = 3.35      # H100 SXM5 80 GB data sheet


class TorchPL(PseudoLabelLoss):
    """PseudoLabelLoss written in PyTorch under another type: the network takes the eager route."""

    def forward(self, logits, target, teacher_logits=None):
        c = logits.shape[1]
        lab = (target != self.ignore_index) & (target >= 0) & (target < c)
        ce = F.cross_entropy(logits, torch.where(lab, target, torch.full_like(target, -100)), ignore_index=-100)
        if teacher_logits is None:
            return ce
        unl = target == self.ignore_index
        conf, yhat = torch.softmax(teacher_logits, dim=1).max(1)
        keep = unl & (conf >= self.threshold)
        pl = F.cross_entropy(logits, torch.where(keep, yhat, torch.full_like(yhat, -100)), ignore_index=-100,
                             reduction="sum") / unl.sum().clamp(min=1)
        return self.ce_weight * ce + self.pl_weight * pl


ARMS = ("ce", "kd_frozen", "kd_ema", "pl_ema", "torch_pl", "ema_update", "ema_launch")


def _arm(arm, base, frozen, dev):
    """(model, step closure) of one arm on a fresh copy of `base`."""
    model = copy.deepcopy(base).to(dev)
    opt = bench.build_optimizer(model, "psp", kind="fused")
    after = None
    if arm == "ce":
        model.criterion = nn.CrossEntropyLoss(ignore_index=255)
    elif arm == "kd_frozen":
        model.criterion = DistillationLoss(frozen)
    elif arm in ("kd_ema", "pl_ema", "ema_update", "ema_launch"):
        ema = ModelEMA(model, decay=0.999)
        model.criterion = (DistillationLoss(ema.module) if arm == "kd_ema" else
                           PseudoLabelLoss(ema.module, threshold=0.95))
        after = lambda: ema.update(model)                                    # noqa: E731
        if arm in ("ema_update", "ema_launch"):
            n = sum(t.numel() for t in list(ema.module.parameters()) + list(ema.module.buffers())
                    if t.dtype == torch.float32)
            if arm == "ema_launch":
                ema.update(model)                  # builds the item table; then the bare launch, as update issues it
                table = ema._table[2]
                return model, lambda: ops.ema_multi(*table, ema.decay), 12 * n
            return model, after, 12 * n
    else:
        from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn
        avg = AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(0.999), use_buffers=True)
        avg.module.eval()
        model.criterion = TorchPL(avg.module, threshold=0.95)
        after = lambda: avg.update_parameters(model)                         # noqa: E731

    def step():
        _, main_loss, aux_loss = model(x_dev[0], x_dev[1])
        loss = main_loss + 0.4 * aux_loss
        opt.zero_grad()
        loss.backward()
        opt.step()
        if after is not None:
            after()
    return model, step, None


x_dev = [None, None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:2,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mean_teacher measures on a GPU; there is no CPU arm"
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
        frozen = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).to(dev).eval()
        x, y = bench.synth_batch(n, size, classes, 100)
        y[n // 2:] = 255                                   # the unlabelled half of the batch
        x_dev[0], x_dev[1] = x.to(dev), y.to(dev)
        runs = {arm: dict(ms=[], peak=[]) for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:          # a fresh copy per window: one arm's graph memory pool is held at a time
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats(dev)
                model, step, nbytes = _arm(arm, base, frozen, dev)
                for _ in range(n_warm):
                    step()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                runs[arm]["ms"].append(ms)
                runs[arm]["peak"].append(torch.cuda.max_memory_allocated(dev) / 2 ** 30)
                runs[arm]["kernels"] = graphs.launches_per_step(model) if nbytes is None else None
                if nbytes is not None:
                    runs[arm].setdefault("tbs", []).append(nbytes / (ms * 1e-3) / 1e12)
                    runs[arm]["bytes"] = nbytes
                del model, step
        for arm in arms:
            r = runs[arm]
            out = dict(info, workload="PSPNet50 student, %dx%d, %d classes, %d images (half unlabelled), bf16, one GPU"
                       % (size, size, classes, n), arm=arm, steps=args.steps,
                       ms_per_step=[round(v, 4 if arm.startswith("ema_") else 2) for v in r["ms"]],
                       peak_gib=round(max(r["peak"]), 2), kernels_per_graphed_step=r["kernels"])
            if "tbs" in r:
                out.update(bytes=r["bytes"], tb_per_s=[round(v, 3) for v in r["tbs"]],
                           of_datasheet_3_35_tbs=[round(v / HBM_DATASHEET_TBS, 3) for v in r["tbs"]])
            print(json.dumps(out), flush=True)
        del runs, base, frozen
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
