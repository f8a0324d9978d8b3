"""Cost of the relation term of losses.DistillationLoss (relation_weight > 0; csrc/relation.cu).

1. The kernels alone at (B, h, w, pool) = (16, 60, 60, 2), (2, 90, 90, 2) and (16, 60, 60, 1), plain bf16 operands:
   forward (nodes of both networks + fused KL + reduce) and backward (KL backward + nodes backward), CUDA events over
   windows of at least `--window` seconds. FLOPs from shapes: forward 4 B^2 M^2 C (the S and T GEMMs), backward
   10 B^2 M^2 C (each of the two channel-half CTAs of an owner recomputes S and T: 2 x 4, plus the G X_j GEMM: 2).
   The share is of the 989 TFLOP/s dense BF16 data-sheet rate: tensor-core compute bounds these kernels (their bytes
   are a few MB against GFLOPs).
2. The same term in PyTorch (fp32) on the same GPU at the first shape, forward + backward: the per-pair loop form of
   the paper's code and the batched form with [B M, B M] maps; time and torch.cuda.max_memory_allocated.
3. The graphed PSPNet50 KD step (bench.py's step, 473^2, 150 classes, 16 images) with a PSPNet101 teacher at
   relation_weight 0 and 1, the arms alternating over `--rounds` rounds.

Every comparison runs at least twice with the arms alternating. Prints one JSON line per measurement with the GPU, its
power limit and SM clock, read in the same process. Not part of bench.py's contract.
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
from semseg_b200 import graphs, ops  # noqa: E402
from semseg_b200.losses import DistillationLoss  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

BF16_TFLOPS = 989.0
C = 512


def _time(fn, window_s):
    """ms per call over a window of at least window_s seconds (after a warm-up)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    iters = max(3, int(window_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _features(b, h, w, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.relu(torch.randn((b, h, w, C), device=dev, generator=g)).to(torch.bfloat16)


def kernel_bench(info, args, dev):
    for b, h, w, pool in ((16, 60, 60, 2), (2, 90, 90, 2), (16, 60, 60, 1)):
        fs, ft = _features(b, h, w, dev, 1), _features(b, h, w, dev, 2)
        m = ops.relation_grid(h, w, pool)
        xs, arg, inv = ops.relation_nodes(fs, pool, False, student=True)
        xt = ops.relation_nodes(ft, pool, False)[0]
        loss, lse = ops.relation_kl_fwd(xs, xt, 1.0)
        g = torch.ones((1,), device=dev)
        dn = ops.relation_kl_bwd(xs, xt, 1.0, lse, g)

        def fwd():
            a = ops.relation_nodes(fs, pool, False, student=True)[0]
            ops.relation_kl_fwd(a, ops.relation_nodes(ft, pool, False)[0], 1.0)

        def bwd():
            ops.relation_nodes_bwd(fs, pool, arg, inv, ops.relation_kl_bwd(xs, xt, 1.0, lse, g))
        arms = {"forward": (fwd, 4), "backward": (bwd, 10)}
        res = {k: [] for k in arms}
        for _ in range(2):
            for k, (fn, _) in arms.items():
                res[k].append(_time(fn, args.window))
        for k, (_, mult) in arms.items():
            flop = mult * b * b * m * m * C
            ms = min(res[k])
            tf = flop / ms / 1e9
            print(json.dumps(dict(info, workload="relation %s, B=%d %dx%d pool %d (M=%d), bf16" % (k, b, h, w, pool, m),
                                  arm=k, ms=[round(v, 3) for v in res[k]], gflop_from_shapes=round(flop / 1e9, 1),
                                  achieved_tflop_s=round(tf, 1), share_of_bf16_dense_data_sheet=round(tf / BF16_TFLOPS, 3),
                                  bound="tensor-core compute")), flush=True)
        del xs, xt, arg, inv, lse, dn, loss


def _torch_loop(fs, ft, tau, pool):
    b = fs.shape[0]
    xs = torch.nn.functional.normalize(torch.nn.functional.max_pool2d(fs, pool, pool, ceil_mode=True).flatten(2), dim=1)
    xt = torch.nn.functional.normalize(torch.nn.functional.max_pool2d(ft, pool, pool, ceil_mode=True).flatten(2), dim=1)
    m = xs.shape[2]
    total = 0.0
    for i in range(b):
        for j in range(b):
            ls = torch.log_softmax(xs[i].T @ xs[j] / tau, dim=1)
            lt = torch.log_softmax(xt[i].T @ xt[j] / tau, dim=1)
            total = total + (lt.exp() * (lt - ls)).sum()
    return total * tau * tau / (b * b * m)


def _torch_batched(fs, ft, tau, pool):
    b = fs.shape[0]
    xs = torch.nn.functional.normalize(torch.nn.functional.max_pool2d(fs, pool, pool, ceil_mode=True).flatten(2), dim=1)
    xt = torch.nn.functional.normalize(torch.nn.functional.max_pool2d(ft, pool, pool, ceil_mode=True).flatten(2), dim=1)
    m = xs.shape[2]
    xs = xs.permute(0, 2, 1).reshape(b * m, -1)
    xt = xt.permute(0, 2, 1).reshape(b * m, -1)
    ls = torch.log_softmax((xs @ xs.T / tau).view(b * m, b, m), dim=2)
    lt = torch.log_softmax((xt @ xt.T / tau).view(b * m, b, m), dim=2)
    return (lt.exp() * (lt - ls)).sum() * tau * tau / (b * b * m)


def torch_bench(info, args, dev, b=16, h=60, w=60, pool=2):
    g = torch.Generator(device=dev).manual_seed(3)
    fs = torch.relu(torch.randn((b, C, h, w), device=dev, generator=g)).requires_grad_(True)
    ft = torch.relu(torch.randn((b, C, h, w), device=dev, generator=g))
    arms = {"pytorch per-pair loop": _torch_loop, "pytorch batched": _torch_batched}
    res = {k: dict(ms=[]) for k in arms}
    for _ in range(2):
        for k, fn in arms.items():
            def call():
                fs.grad = None
                fn(fs, ft, 1.0, pool).backward()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            res[k]["ms"].append(_time(call, args.window))
            res[k]["peak_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    for k, r in res.items():
        print(json.dumps(dict(info, workload="relation forward + backward in PyTorch fp32, B=%d %dx%d pool %d" %
                              (b, h, w, pool), arm=k, ms=[round(v, 2) for v in r["ms"]], peak_gb=r["peak_gb"])),
              flush=True)


def _net(layers, classes):
    from semseg_b200.pspnet import PSPNet
    torch.manual_seed(0)
    return PSPNet(layers=layers, classes=classes, zoom_factor=8, pretrained=False)


def step_bench(info, args, dev):
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    size, classes, n = 473, 150, 16
    base = _net(50, classes).train()
    teacher = _net(101, classes).to(dev).eval()
    x, y = bench.synth_batch(n, size, classes, 100)
    x, y = x.to(dev), y.to(dev)
    runs = {w: dict(ms=[]) for w in (0.0, 1.0)}
    for _ in range(args.rounds):
        for weight, r in runs.items():
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            model = copy.deepcopy(base).to(dev)
            opt = bench.build_optimizer(model, "psp", kind="fused")
            model.criterion = DistillationLoss(teacher, temperature=1.0, relation_weight=weight)

            def step():
                _, main_loss, aux_loss = model(x, y)
                opt.zero_grad()
                (main_loss + 0.4 * aux_loss).backward()
                opt.step()
            for _ in range(n_warm):
                step()
            r["ms"].append(_time(step, args.window))
            r["kernels"] = graphs.launches_per_step(model)
            r["peak_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
            del model, opt, step
    for weight, r in runs.items():
        print(json.dumps(dict(info, workload="graphed PSPNet50 KD step, PSPNet101 teacher, %dx%d, %d classes, %d images, "
                              "bf16, one GPU" % (size, size, classes, n), arm="relation_weight=%g" % weight,
                              ms_per_step=[round(v, 2) for v in r["ms"]], peak_gb=r["peak_gb"],
                              kernels_per_graphed_step=r["kernels"])), flush=True)
    print(json.dumps(dict(info, workload="step time ratio relation_weight 1 / 0",
                          measured_ratio=round(min(runs[1.0]["ms"]) / min(runs[0.0]["ms"]), 3))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per step arm, the arms alternating")
    ap.add_argument("--skip-step", action="store_true", help="measure the kernels and the PyTorch forms only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_relation measures on a GPU; there is no CPU arm"
    dev = torch.device("cuda", 0)
    info = _gpu_info()
    kernel_bench(info, args, dev)
    torch_bench(info, args, dev)
    if not args.skip_step:
        step_bench(info, args, dev)


if __name__ == "__main__":
    main()
