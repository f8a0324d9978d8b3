"""Training-step cost of CutMix / ClassMix mean-teacher training on the native tail (losses.MixPseudoLabelLoss).

Arms, each running bench.py's step (model(input, target), loss = main + 0.4 aux, zero_grad, backward, FusedSGD with the
reference's 8 parameter groups, then ema.update(model)) on a fresh copy of one seeded PSPNet50 student with an
optim.ModelEMA teacher, the default `bf16` mode, one GPU; the first half of every batch is labelled, the second half
unlabelled (an all-ignore target):
  * pl_ema        : losses.PseudoLabelLoss(ema.module, threshold=0.95), the teacher on the student's input, graphed;
  * cutmix_ema    : losses.MixPseudoLabelLoss(ema.module, mix='cutmix', threshold=0.95), graphed;
  * classmix_ema  : the same with mix='classmix', graphed;
  * torch_cutmix / torch_classmix: the same two mixes written in PyTorch under another type, so the network takes the
                    eager ATen route: the box on the host, or F.interpolate of the teacher's logits, argmax and a
                    per-image class draw; torch.where for the input, target and teacher maps; the pseudo-label loss in
                    PyTorch (softmax, masked cross-entropy).
Workloads: ADE20K-shaped (473x473, 150 classes, 16 images) and Cityscapes-shaped (713x713, 19 classes, 8 images). The
arms alternate over `--rounds` rounds; each timed window of `--steps` steps follows the warm-up (eager calls and, for
the graphed arms, the capture). Prints one JSON line per workload and arm: the GPU, its power limit and SM clock (read
in the same process), ms/step of every round, the peak memory of the window and the kernels per graphed step. Not part
of bench.py's contract.
"""
import argparse
import copy
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402
from semseg_b200.losses import MixPseudoLabelLoss, PseudoLabelLoss  # noqa: E402
from semseg_b200.optim import ModelEMA  # noqa: E402
from tools.bench_mean_teacher import TorchPL  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


class TorchMix(MixPseudoLabelLoss):
    """MixPseudoLabelLoss written in PyTorch under another type: the network takes the eager route."""

    forward = TorchPL.forward

    def mix_batch(self, x, y, u, t_logits, zoom):
        n, _, hh, ww = x.shape
        uc = u.cpu()
        mask = torch.zeros((n, hh, ww), dtype=torch.bool, device=x.device)
        if self.mix == 'cutmix':
            for i in range(n):
                if float(uc[i, 0]) >= self.p:
                    continue
                u1, u2, u3, u4 = (float(v) for v in uc[i, 1:5])
                a = (self.area[0] + (self.area[1] - self.area[0]) * u1) * hh * ww
                rho = self.ratio[0] + (self.ratio[1] - self.ratio[0]) * u2
                bw = min(ww, max(1, math.floor(math.sqrt(a / rho))))
                bh = min(hh, max(1, math.floor(math.sqrt(a * rho))))
                x0 = min(ww - bw, math.floor(u4 * (ww - bw + 1)))
                y0 = min(hh - bh, math.floor(u3 * (hh - bh + 1)))
                mask[i, y0:y0 + bh, x0:x0 + bw] = True
        else:
            amap = F.interpolate(t_logits.permute(0, 3, 1, 2), size=(hh, ww), mode='bilinear',
                                 align_corners=True).argmax(1)
            for i in range(n):
                if float(uc[i, 0]) >= self.p:
                    continue
                j = (i + 1) % n
                present = amap[j].unique()
                order = torch.argsort(u[j, 5 + present], stable=True)
                mask[i] = torch.isin(amap[j], present[order[:(present.numel() + 1) // 2]])
        xm = torch.where(mask.unsqueeze(1), x.roll(-1, 0), x)
        s = 8 // zoom
        ym = torch.where(mask[:, ::s, ::s], y.roll(-1, 0), y)
        self._last['mix'] = {'mask': mask.to(torch.uint8), 'target': ym, 'uniforms': u}
        return xm, ym, mask.to(torch.uint8)


ARMS = ("pl_ema", "cutmix_ema", "classmix_ema", "torch_cutmix", "torch_classmix")


def _arm(arm, base, dev):
    """(model, step closure) of one arm on a fresh copy of `base`."""
    model = copy.deepcopy(base).to(dev)
    opt = bench.build_optimizer(model, "psp", kind="fused")
    ema = ModelEMA(model, decay=0.999)
    if arm == "pl_ema":
        model.criterion = PseudoLabelLoss(ema.module, threshold=0.95)
    else:
        mix = arm.split("_")[1 if arm.startswith("torch") else 0]
        cls = TorchMix if arm.startswith("torch") else MixPseudoLabelLoss
        model.criterion = cls(ema.module, mix=mix, threshold=0.95)

    def step():
        _, main_loss, aux_loss = model(x_dev[0], x_dev[1])
        loss = main_loss + 0.4 * aux_loss
        opt.zero_grad()
        loss.backward()
        opt.step()
        ema.update(model)
    return model, step


x_dev = [None, None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16,713:19:8", help="size:classes:images, comma separated")
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mix measures on a GPU; there is no CPU arm"
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
        y[n // 2:] = 255                                   # the unlabelled half of the batch
        x_dev[0], x_dev[1] = x.to(dev), y.to(dev)
        runs = {arm: dict(ms=[], peak=[]) for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:          # a fresh copy per window: one arm's graph memory pool is held at a time
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats(dev)
                model, step = _arm(arm, base, dev)
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
                runs[arm]["kernels"] = graphs.launches_per_step(model)
                del model, step
        for arm in arms:
            r = runs[arm]
            print(json.dumps(dict(info, workload="PSPNet50 student, %dx%d, %d classes, %d images (half unlabelled), "
                                  "bf16, one GPU" % (size, size, classes, n), arm=arm, steps=args.steps,
                                  ms_per_step=[round(v, 2) for v in r["ms"]], peak_gib=round(max(r["peak"]), 2),
                                  kernels_per_graphed_step=r["kernels"])), flush=True)
        del runs, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
