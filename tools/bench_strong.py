"""Cost of the strong view of mean-teacher training (augment.StrongAugment, csrc/strong.cu).

1. The kernel (both launches) on ADE20K-shaped (16x3x473x473) and Cityscapes-shaped (16x3x713x713) batches with
   UniMatch's defaults and one fixed draw, against the same chain written with torchvision.transforms.v2.functional on
   the GPU, one image at a time, with the same draws (tests/strong_oracle.py's `params`). CUDA events over `--iters`
   calls after a warm-up. Achieved GB/s is the kernel's algorithmic bytes over its time: every pixel read and written
   once by strong_apply (24 B), plus one read (12 B) by strong_stats for each image contrast applies to; the halo
   re-reads of blurred tiles are not counted. The largest difference between the two outputs is reported too.
2. The graphed PSPNet50 step (bench.py's step plus ema.update) with losses.MixPseudoLabelLoss(mix='cutmix') and an
   optim.ModelEMA teacher, without and with `strong=StrongAugment()`, the two arms alternating over `--rounds` rounds.

Prints one JSON line per measurement with the GPU, its power limit and SM clock, read in the same process. Not part of
bench.py's contract.
"""
import argparse
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402
from semseg_b200.augment import StrongAugment  # noqa: E402
from semseg_b200.losses import MixPseudoLabelLoss  # noqa: E402
from semseg_b200.optim import ModelEMA  # noqa: E402
from tests.strong_oracle import params  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402


def _opts(s):
    return dict(brightness=s.brightness, contrast=s.contrast, saturation=s.saturation, hue=s.hue,
                p_jitter=s.p_jitter, p_gray=s.p_gray, p_blur=s.p_blur, sigma=s.sigma)


def torchvision_chain(x, u, s):
    """The chain with torchvision.transforms.v2.functional, one image at a time, on x's device."""
    import torchvision.transforms.v2.functional as TF
    fns = {"brightness": TF.adjust_brightness, "contrast": TF.adjust_contrast, "saturation": TF.adjust_saturation,
           "hue": TF.adjust_hue}
    mean = torch.tensor(s.mean, device=x.device).view(3, 1, 1)
    std = torch.tensor(s.std, device=x.device).view(3, 1, 1)
    out = x.clone()
    for n, un in enumerate(u.cpu().numpy()):
        prm = params(un, **_opts(s))
        if not (prm['ops'] or prm['gray'] or prm['r']):
            continue
        v = ((x[n] * std + mean) / 255).clamp(0, 1)
        for name, f in prm['ops']:
            v = fns[name](v, f)
        if prm['gray']:
            v = TF.rgb_to_grayscale(v, num_output_channels=3)
        if prm['r']:
            v = TF.gaussian_blur(v, [2 * prm['r'] + 1] * 2, [prm['sigma']] * 2)
        out[n] = (255 * v - mean) / std
    return out


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_bench(info, iters, dev):
    s = StrongAugment()
    for size in (473, 713):
        n = 16
        g = torch.Generator(device=dev).manual_seed(size)
        x = torch.randn((n, 3, size, size), device=dev, generator=g)
        u = torch.rand((n, 12), device=dev, generator=g)
        prms = [params(un, **_opts(s)) for un in u.cpu().numpy()]
        n_contrast = sum(any(name == "contrast" for name, _ in p['ops']) for p in prms)
        hw = size * size
        nbytes = n * hw * 24 + n_contrast * hw * 12
        ms = _time(lambda: s(x, u), iters)
        rec = dict(info, workload="strong view, %dx3x%dx%d fp32, UniMatch defaults, one draw" % (n, size, size),
                   arm="kernel", ms=round(ms, 4), algorithmic_mb=round(nbytes / 1e6, 1),
                   achieved_gb_s=round(nbytes / ms / 1e6, 1), images_contrast=n_contrast,
                   images_blurred=sum(p['r'] > 0 for p in prms), images_copied=sum(
                       not (p['ops'] or p['gray'] or p['r']) for p in prms))
        try:
            import torchvision  # noqa: F401
        except ImportError:
            rec["torchvision"] = "not installed"
        else:
            ms_tv = _time(lambda: torchvision_chain(x, u, s), max(2, iters // 20))
            rec.update(torchvision_ms=round(ms_tv, 3), speedup=round(ms_tv / ms, 1),
                       max_abs_diff=float((s(x, u) - torchvision_chain(x, u, s)).abs().max()))
        print(json.dumps(rec), flush=True)


def step_bench(info, args, dev):
    from model.pspnet import PSPNet
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for wl in args.workloads.split(","):
        size, classes, n = (int(v) for v in wl.split(":"))
        torch.manual_seed(0)
        base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
        x, y = bench.synth_batch(n, size, classes, 100)
        y[n // 2:] = 255                                   # the unlabelled half of the batch
        x, y = x.to(dev), y.to(dev)
        runs = {arm: dict(ms=[]) for arm in ("cutmix_ema", "cutmix_ema_strong")}
        for _ in range(args.rounds):
            for arm in runs:
                torch.cuda.empty_cache()
                model = copy.deepcopy(base).to(dev)
                opt = bench.build_optimizer(model, "psp", kind="fused")
                ema = ModelEMA(model, decay=0.999)
                model.criterion = MixPseudoLabelLoss(ema.module, mix='cutmix', threshold=0.95,
                                                     strong=StrongAugment() if arm.endswith("strong") else None)

                def step():
                    _, main_loss, aux_loss = model(x, y)
                    opt.zero_grad()
                    (main_loss + 0.4 * aux_loss).backward()
                    opt.step()
                    ema.update(model)
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
                del model, opt, ema, step
        for arm, r in runs.items():
            print(json.dumps(dict(info, workload="PSPNet50 student, %dx%d, %d classes, %d images (half unlabelled), "
                                  "bf16, one GPU" % (size, size, classes, n), arm=arm, steps=args.steps,
                                  ms_per_step=[round(v, 2) for v in r["ms"]],
                                  kernels_per_graphed_step=r["kernels"])), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200, help="timed kernel calls")
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--workloads", default="473:150:16", help="size:classes:images of the step, comma separated")
    ap.add_argument("--skip-step", action="store_true", help="measure the kernel only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_strong measures on a GPU; there is no CPU arm"
    dev = torch.device("cuda", 0)
    info = _gpu_info()
    kernel_bench(info, args.iters, dev)
    if not args.skip_step:
        step_bench(info, args, dev)


if __name__ == "__main__":
    main()
