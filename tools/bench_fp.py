"""Cost of the feature-perturbation stream of mean-teacher training (losses.PseudoLabelLoss / MixPseudoLabelLoss
fp_weight > 0, UniMatch's FP; csrc/bn.cu fp_fork / fp_fold).

1. The fork and the fold alone at the layer4 shape of the step below (16 x 60 x 60 x 2048, plain bf16), CUDA events over
   `--iters` calls after a warm-up. Bytes from shapes: each reads N images once and writes 2N (fork) or reads 2N and
   writes N (fold), 3 N h w C 2 bytes, plus the [N, C] fp32 scale; achieved GB/s against the 3.35 TB/s data sheet.
2. The second tail call (the FP term: the mixed pseudo-label forward and backward with ce_weight 0 on the perturbed
   logits, [16, 60, 60, 150] -> 473 x 473) under torch.profiler in a run of its own: device time of its kernels per call.
3. The graphed PSPNet50 step (bench.py's step plus ema.update) with MixPseudoLabelLoss(mix='cutmix', strong=...) and an
   optim.ModelEMA teacher, 16 images of which 8 all-ignore, at fp_weight 0 and 0.5, the arms alternating over
   `--rounds` rounds. By FLOPs from shapes the FP stream adds about 408 of the 1022.8 GFLOP step (the cls 3x3 conv,
   4096 -> 512 at 60 x 60, doubled in fprop, dgrad and wgrad): about 1.4x. The JSON line states the measured ratio.

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
from semseg_b200 import functional as SF  # noqa: E402
from semseg_b200 import graphs, ops  # noqa: E402
from semseg_b200.augment import StrongAugment  # noqa: E402
from semseg_b200.losses import MixPseudoLabelLoss  # noqa: E402
from semseg_b200.optim import ModelEMA  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

HBM_TB_S = 3.35
FLOP_RATIO = (1022.8 + 407.7) / 1022.8           # step FLOPs with / without the FP stream, from shapes


def _time(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_bench(info, iters, dev, n=16, h=60, w=60, c=2048):
    g = torch.Generator(device=dev).manual_seed(0)
    f = torch.randn((n, h, w, c), device=dev, generator=g).to(torch.bfloat16)
    d = torch.randn((2 * n, h, w, c), device=dev, generator=g).to(torch.bfloat16)
    s = (torch.rand((n, c), device=dev, generator=g) < 0.5).float().mul_(2.0)
    nbytes = 3 * n * h * w * c * 2 + n * c * 4
    for name, fn in (("fork", lambda: ops.fp_fork(f, s)), ("fold", lambda: ops.fp_fold(d, s))):
        ms = _time(fn, iters)
        gb_s = nbytes / ms / 1e6
        print(json.dumps(dict(info, workload="fp_%s, layer4 %dx%dx%dx%d bf16" % (name, n, h, w, c), arm=name,
                              ms=round(ms, 4), algorithmic_mb=round(nbytes / 1e6, 1), achieved_gb_s=round(gb_s, 1),
                              share_of_hbm_data_sheet=round(gb_s / (HBM_TB_S * 1e3), 3))), flush=True)


def tail_profile(info, dev, n=16, h=60, w=60, classes=150, iters=10):
    from torch.profiler import ProfilerActivity, profile
    size = 8 * (h - 1) + 1
    g = torch.Generator(device=dev).manual_seed(1)
    s_fp = torch.randn((n, h, w, classes), device=dev, generator=g).requires_grad_(True)
    t = torch.randn((n, h, w, classes), device=dev, generator=g) * 3
    y = torch.randint(0, classes, (n, size, size), device=dev, generator=g)
    y[n // 2:] = 255
    mask = torch.zeros((n, size, size), dtype=torch.uint8, device=dev)
    mask[:, 100:300, 150:400] = 1
    # the criterion only supplies the options here: its teacher is not run
    crit = MixPseudoLabelLoss(_net(classes).eval(), mix='cutmix', threshold=0.95, fp_weight=0.5)

    def call():
        loss, _ = SF.upsample_fp(s_fp, y, 8, crit, t, mask)
        (gs,) = torch.autograd.grad(loss, s_fp)
        return gs
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            kern[e.name] = kern.get(e.name, 0.0) + e.device_time / 1e3 / iters
    print(json.dumps(dict(info, workload="second tail call (FP term, mixed pseudo-label fwd + bwd), %dx%dx%dx%d -> "
                          "%dx%d" % (n, h, w, classes, size, size), arm="fp_tail_profiled",
                          ms_per_call=round(sum(kern.values()), 3),
                          kernels_ms={k[:60]: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])})),
          flush=True)


def _net(classes):
    from model.pspnet import PSPNet
    torch.manual_seed(0)
    return PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()


def step_bench(info, args, dev):
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    size, classes, n = 473, 150, 16
    base = _net(classes)
    x, y = bench.synth_batch(n, size, classes, 100)
    y[n // 2:] = 255                                   # the unlabelled half of the batch
    x, y = x.to(dev), y.to(dev)
    runs = {w: dict(ms=[]) for w in (0.0, 0.5)}
    for _ in range(args.rounds):
        for fp_weight, r in runs.items():
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            model = copy.deepcopy(base).to(dev)
            opt = bench.build_optimizer(model, "psp", kind="fused")
            ema = ModelEMA(model, decay=0.999)
            model.criterion = MixPseudoLabelLoss(ema.module, mix='cutmix', threshold=0.95, strong=StrongAugment(),
                                                 fp_weight=fp_weight)

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
            r["ms"].append(e0.elapsed_time(e1) / args.steps)
            r["kernels"] = graphs.launches_per_step(model)
            r["peak_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
            del model, opt, ema, step
    for fp_weight, r in runs.items():
        print(json.dumps(dict(info, workload="PSPNet50 student, %dx%d, %d classes, %d images (half unlabelled), cutmix + "
                              "strong, EMA teacher, bf16, one GPU" % (size, size, classes, n),
                              arm="fp_weight=%g" % fp_weight, steps=args.steps,
                              ms_per_step=[round(v, 2) for v in r["ms"]], peak_gb=r["peak_gb"],
                              kernels_per_graphed_step=r["kernels"])), flush=True)
    ratio = min(runs[0.5]["ms"]) / min(runs[0.0]["ms"])
    print(json.dumps(dict(info, workload="step time ratio fp_weight 0.5 / 0", measured_ratio=round(ratio, 3),
                          flop_ratio_from_shapes=round(FLOP_RATIO, 3))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200, help="timed kernel calls")
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    ap.add_argument("--skip-step", action="store_true", help="measure the kernels and the tail call only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fp measures on a GPU; there is no CPU arm"
    dev = torch.device("cuda", 0)
    info = _gpu_info()
    kernel_bench(info, args.iters, dev)
    tail_profile(info, dev)
    if not args.skip_step:
        step_bench(info, args, dev)


if __name__ == "__main__":
    main()
