"""Cost of the Gated CRF loss (semseg_b200.losses.GatedCRFLoss) against plain cross-entropy.

For each class count (`--classes`, default 21 and 150) on copies of one seeded PSPNet50 (bf16, one GPU, 473x473, 16
images, a scribble-like target with ~2 % of the pixels labelled):
  * step arms, graphed and alternated over `--rounds` rounds, timed with CUDA events: bench.py's training step with
    nn.CrossEntropyLoss (ce), GatedCRFLoss(at='output') (crf_output) and GatedCRFLoss(at='logits') (crf_logits), with
    torch.cuda.max_memory_allocated over each arm's copy, warm-up, capture and timed steps;
  * the CRF kernels alone (ops.gated_crf_fwd / gated_crf_bwd at the network's logits and image shapes, radius 5), timed
    with CUDA events over `--kernel-iters` calls, with their share of the FP32 bound: one stencil pass is
    P ((2r+1)^2 - 1) C FMAs, at the 67 TFLOP/s data-sheet FP32 rate;
  * the published PyTorch unfold formulation (tests/gatedcrf_oracle.py's crf_unfold in fp32, forward and backward) at
    at='logits' on the whole batch and at='output' on one image; out of memory is reported as such.
Prints one JSON line per measurement with the GPU name, power limit and SM clock read in the same process.
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
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs, ops  # noqa: E402
from semseg_b200.losses import GatedCRFLoss  # noqa: E402
from tests.gatedcrf_oracle import crf_unfold, grid_rgb  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

FP32_PEAK = 67e12
ARMS = ("ce", "crf_output", "crf_logits")


def _scribbles(y, seed=0):
    g = torch.Generator(device=y.device).manual_seed(seed)
    keep = torch.rand(y.shape, device=y.device, generator=g) < 0.02
    return torch.where(keep, y, torch.full_like(y, 255))


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--classes", default="21,150")
    ap.add_argument("--radius", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gatedcrf measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    size, n, r = args.size, args.images, args.radius
    h = (size - 1) // 8 + 1
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for classes in (int(c) for c in args.classes.split(",")):
        workload = "PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU, radius %d" % (size, size, classes, n, r)
        torch.manual_seed(0)
        base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
        x, y = bench.synth_batch(n, size, classes, 100)
        x, y = x.to(dev), _scribbles(y.to(dev))
        runs = {arm: dict(ms=[], peak=0) for arm in ARMS}
        for _ in range(args.rounds):
            for arm in ARMS:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()      # the peak spans the copy, warm-up, capture and timed steps
                model = copy.deepcopy(base).to(dev)
                model.criterion = (nn.CrossEntropyLoss(ignore_index=255) if arm == "ce" else
                                   GatedCRFLoss(crf_weight=0.1, radius=r, at=arm[4:]))
                opt = bench.build_optimizer(model, "psp")

                def step():
                    _, main_loss, aux_loss = model(x, y)
                    loss = main_loss + 0.4 * aux_loss
                    opt.zero_grad()
                    loss.backward()
                    opt.step()
                for _ in range(n_warm):
                    step()
                runs[arm]["ms"].append(_time(step, args.steps))
                runs[arm]["peak"] = max(runs[arm]["peak"], torch.cuda.max_memory_allocated())
                runs[arm]["kernels"] = graphs.launches_per_step(model)
                del model, step, opt
                torch.cuda.empty_cache()
        for arm in ARMS:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload=workload, arm=arm, ms_per_step=[round(v, 2) for v in ms],
                                  img_per_s=round(n / (min(ms) / 1e3), 2), peak_gb=round(runs[arm]["peak"] / 1e9, 2),
                                  kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        del base
        torch.cuda.empty_cache()

        # the CRF kernels alone, at the network's shapes
        g = torch.Generator(device=dev).manual_seed(1)
        logits = torch.randn((n, h, h, classes), device=dev, generator=g) * 3
        for at, zoom, stride in (("output", 8, 1), ("logits", 1, 8)):
            lse = None
            if at == "output":
                tgt = torch.zeros((n, size, size), dtype=torch.int64, device=dev)
                lse = ops.upsample_ce_fwd(logits, tgt, 255, want_argmax=False, zoom=8)[2]
            crit = GatedCRFLoss(radius=r, at=at)
            cfg = (r, crit.sigma_xy, crit.sigma_rgb, crit.mean, crit.std)
            _, s, crf_lse = ops.gated_crf_fwd(logits, lse, x, zoom, stride, *cfg)
            dl = torch.zeros_like(logits)
            gout = torch.ones((), device=dev)
            fwd_ms = _time(lambda: ops.gated_crf_fwd(logits, crf_lse if lse is not None else None, x, zoom, stride,
                                                     *cfg), args.kernel_iters)
            bwd_ms = _time(lambda: ops.gated_crf_bwd(logits, crf_lse, x, s, 0.1, gout, dl, zoom, stride, *cfg),
                           args.kernel_iters)
            grid = zoom * (h - 1) + 1
            flops = 2.0 * n * grid * grid * ((2 * r + 1) ** 2 - 1) * classes
            print(json.dumps(dict(info, workload=workload, measure="crf_kernels", at=at, fwd_ms=round(fwd_ms, 3),
                                  bwd_ms=round(bwd_ms, 3), stencil_gflop=round(flops / 1e9, 1),
                                  fwd_share_of_fp32_bound=round(flops / FP32_PEAK / (fwd_ms / 1e3), 3),
                                  bwd_share_of_fp32_bound=round(flops / FP32_PEAK / (bwd_ms / 1e3), 3))), flush=True)

        # the published PyTorch unfold formulation, fp32, forward + backward
        for at, imgs in (("logits", n), ("output", 1)):
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            crit = GatedCRFLoss(radius=r)
            try:
                s8 = logits[:imgs].permute(0, 3, 1, 2).contiguous().requires_grad_(True)
                stride = 8 if at == "logits" else 1
                rgb = grid_rgb(x[:imgs], stride).float()

                def unfold_step():
                    grid_l = s8 if at == "logits" else F.interpolate(s8, size=(size, size), mode="bilinear",
                                                                    align_corners=True)
                    loss = crf_unfold(grid_l, rgb, r, crit.sigma_xy, crit.sigma_rgb, dtype=torch.float32)
                    s8.grad = None
                    loss.backward()
                ms = round(_time(unfold_step, 3), 2)
                peak = round(torch.cuda.max_memory_allocated() / 1e9, 2)
            except torch.OutOfMemoryError:
                ms, peak = "out of memory", None
            print(json.dumps(dict(info, workload=workload, measure="pytorch_unfold", at=at, images=imgs,
                                  ms_fwd_bwd=ms, peak_gb=peak)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
