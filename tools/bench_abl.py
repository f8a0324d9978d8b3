"""Cost of the Active Boundary Loss (semseg_b200.losses.ActiveBoundaryLoss) and of Boundary IoU.

For each workload (`--workloads`, default 473:16:21, 473:16:150 and 713:8:19 as size:images:classes) on copies of one
seeded PSPNet50 (bf16, one GPU, zoom 8) and a scene-like target (blocks of 32 x 32 pixels with ignored stripes):
  * step arms, graphed and alternated over `--rounds` rounds, timed with CUDA events: bench.py's training step with
    nn.CrossEntropyLoss (ce) and ActiveBoundaryLoss() (abl), with torch.cuda.max_memory_allocated over each arm;
  * the ABL kernels alone (ops.abl_fwd / abl_bwd at the network's logits shape, zoom 8), CUDA events over
    `--kernel-iters` calls, and the distance transform's two kernels under torch.profiler;
  * the published form on the same batch: the same loss written in PyTorch (fp32, on the GPU) with the distance
    transform from scipy on the host and the threshold search as a host loop, forward and backward;
  * boundaryIoUGPU on the argmax and target against the paper's per-class cv2 erosion loop on the host.
Prints one JSON line per measurement with the GPU name, power limit and SM clock read in the same process.
Not part of bench.py's contract.
"""
import argparse
import copy
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from scipy import ndimage  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs, ops  # noqa: E402
from semseg_b200.losses import ActiveBoundaryLoss  # noqa: E402
from semseg_b200.metrics import boundaryIoUGPU  # noqa: E402
from tests import abl_oracle as O  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

ARMS = ("ce", "abl")


def _scene_target(n, size, classes, seed):
    g = torch.Generator().manual_seed(seed)
    cells = torch.randint(0, classes, (n, size // 32 + 1, size // 32 + 1), generator=g)
    y = cells.repeat_interleave(32, 1).repeat_interleave(32, 2)[:, :size, :size].contiguous()
    y[:, ::97, :] = 255
    return y


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


def _published_abl(up, target, crit):
    """The loss as the published code computes it, in fp32: scipy's EDT per image on the host, a host threshold loop."""
    n, c, H, W = up.shape
    t = target
    b = t == crit.ignore_index
    b[:, :-1] |= t[:, :-1] != t[:, 1:]
    b[:, :, :-1] |= t[:, :, :-1] != t[:, :, 1:]
    bh = b.cpu().numpy()
    dist = np.stack([ndimage.distance_transform_edt(~bh[k]) for k in range(n)]).astype(np.float32)
    D = torch.from_numpy(np.maximum(dist - 1.0, 0.0)).to(up.device)
    lp = torch.log_softmax(up, 1)
    p = lp.exp()
    k = torch.zeros((n, H, W), device=up.device)
    k[:, :-1] += (p[:, :, :-1] * (lp[:, :, :-1] - lp[:, :, 1:])).sum(1)
    k[:, :, :-1] += (p[..., :-1] * (lp[..., :-1] - lp[..., 1:])).sum(1)
    k = k.detach()
    eps, max_n = 1e-5, crit.max_n_ratio * H * W
    while (k > eps).sum().item() > max_n:
        eps *= 1.2
    B = F.max_pool2d((k > eps).float()[:, None], 3, 1, 1)[:, 0] > 0
    Dp = F.pad(D[:, None], (1, 1, 1, 1), value=float("inf"))[:, 0]
    stack = torch.stack([Dp[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W] for dy, dx in O.NEIGHBOURS] + [D], 1)
    direction = stack.argmin(1)
    sel = B & (direction != 8)
    pad = F.pad(lp.detach(), (1, 1, 1, 1), mode="replicate")
    z = torch.stack([(pad[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W].exp() *
                      (pad[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W] - lp)).sum(1) for dy, dx in O.NEIGHBOURS], 1)
    zs, ds, ws = z.permute(0, 2, 3, 1)[sel], direction[sel], (D.clamp(max=crit.max_clip_dist) / crit.max_clip_dist)[sel]
    y = torch.full_like(zs, crit.label_smoothing / 8).scatter(1, ds[:, None], 1 - crit.label_smoothing)
    return (-(y * torch.log_softmax(zs, 1)).sum(1) * ws).mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workloads", default="473:16:21,473:16:150,713:8:19")
    ap.add_argument("--kernel-iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_abl measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for spec in args.workloads.split(","):
        size, n, classes = (int(v) for v in spec.split(":"))
        h = (size - 1) // 8 + 1
        workload = "PSPNet50 %dx%d, %d classes, %d images, bf16, one GPU" % (size, size, classes, n)
        torch.manual_seed(0)
        base = PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()
        x, _ = bench.synth_batch(n, size, classes, 100)
        x, y = x.to(dev), _scene_target(n, size, classes, 100).to(dev)
        runs = {arm: dict(ms=[], peak=0) for arm in ARMS}
        pred = None
        for _ in range(args.rounds):
            for arm in ARMS:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                model = copy.deepcopy(base).to(dev)
                model.criterion = nn.CrossEntropyLoss(ignore_index=255) if arm == "ce" else ActiveBoundaryLoss()
                opt = bench.build_optimizer(model, "psp")

                def step():
                    nonlocal pred
                    pred, main_loss, aux_loss = model(x, y)
                    loss = main_loss + 0.4 * aux_loss
                    opt.zero_grad()
                    loss.backward()
                    opt.step()
                for _ in range(n_warm):
                    step()
                runs[arm]["ms"].append(_time(step, args.steps))
                runs[arm]["peak"] = max(runs[arm]["peak"], torch.cuda.max_memory_allocated())
                runs[arm]["kernels"] = graphs.launches_per_step(model)
                del model, opt
                torch.cuda.empty_cache()
        for arm in ARMS:
            ms = runs[arm]["ms"]
            print(json.dumps(dict(info, workload=workload, arm=arm, ms_per_step=[round(v, 2) for v in ms],
                                  img_per_s=round(n / (min(ms) / 1e3), 2), peak_gb=round(runs[arm]["peak"] / 1e9, 2),
                                  kernels_per_graphed_step=runs[arm]["kernels"])), flush=True)
        pred = pred.clone()
        del base
        torch.cuda.empty_cache()

        # the ABL kernels alone, at the network's logits shape
        crit = ActiveBoundaryLoss()
        cfg = (crit.max_n_ratio, crit.max_clip_dist, crit.label_smoothing)
        g = torch.Generator(device=dev).manual_seed(1)
        logits = torch.randn((n, h, h, classes), device=dev, generator=g) * 3
        _, _, lse = ops.upsample_ce_fwd(logits, y, 255, want_argmax=False, zoom=8)
        ainfo, state = ops.abl_fwd(logits, lse, y, 255, 8, *cfg)
        dl = torch.zeros_like(logits)
        gout = torch.ones((), device=dev)
        fwd_ms = _time(lambda: ops.abl_fwd(logits, lse, y, 255, 8, *cfg), args.kernel_iters)
        bwd_ms = _time(lambda: ops.abl_bwd(logits, lse, state, ainfo, 1.0, gout, dl, 8), args.kernel_iters)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                ops.abl_fwd(logits, lse, y, 255, 8, *cfg)
            torch.cuda.synchronize()
        per_kernel = {}
        for e in prof.key_averages():
            if "abl_" in e.key:
                name = e.key.split("(")[0].split("::")[-1].replace("void ", "")
                per_kernel[name] = round(e.device_time_total / 1e3 / 3, 3)
        print(json.dumps(dict(info, workload=workload, measure="abl_kernels", fwd_ms=round(fwd_ms, 3),
                              bwd_ms=round(bwd_ms, 3), selected=int(ainfo[1].item()),
                              fwd_ms_per_kernel=per_kernel)), flush=True)

        # the published form: PyTorch on the GPU, scipy's EDT and the threshold loop on the host
        s8 = logits.permute(0, 3, 1, 2).contiguous().requires_grad_(True)

        def published():
            up = F.interpolate(s8, size=(size, size), mode="bilinear", align_corners=True)
            loss = _published_abl(up, y, crit)
            s8.grad = None
            loss.backward()
        torch.cuda.reset_peak_memory_stats()
        pub_ms = _time(published, 3)
        print(json.dumps(dict(info, workload=workload, measure="published_form", ms_fwd_bwd=round(pub_ms, 2),
                              peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))), flush=True)
        del s8
        torch.cuda.empty_cache()

        # Boundary IoU: one kernel pair against the per-class cv2 loop on the host
        biou_ms = _time(lambda: boundaryIoUGPU(pred, y, classes), args.kernel_iters)
        t0 = time.perf_counter()
        pc, tc = pred.cpu().numpy(), y.cpu().numpy()
        ref = O.biou_counts_cv2(pc, tc, classes, 255, O.band_width(size, size))
        cv2_ms = (time.perf_counter() - t0) * 1e3
        inter, union, target = boundaryIoUGPU(pred, y, classes)
        same = bool(np.array_equal(inter.cpu().numpy(), ref[0]) and np.array_equal(target.cpu().numpy(), ref[2]))
        print(json.dumps(dict(info, workload=workload, measure="boundary_iou", gpu_ms=round(biou_ms, 3),
                              cv2_host_ms=round(cv2_ms, 1), counts_equal=same)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
