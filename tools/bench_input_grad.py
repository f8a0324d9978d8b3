"""Input-gradient cost: the eval-mode attack iteration against the stock cuDNN path, and what dx adds to a training step.

Attack iteration (PGD / SegPGD style): `model.eval()`, frozen parameters, `x.requires_grad_()`,
`F.cross_entropy(model(x), y, ignore_index=255).backward()`, then a sign step on x. Arms: this package (`bf16`) and
oracle.torch_oracle.Oracle with the same seeded weights on cuDNN (fp32 NCHW, torch's default TF32 settings), for
PSPNet50 at 473x473 and PSANet50 at 465x465, 150 classes, 16 images by default.
Training step: bench.py's step (main + 0.4 aux, SGD), graphed, with and without x.requires_grad.
The arms run alternately, `--rounds` times `--steps` iterations each, timed with CUDA events. Prints one JSON line with
the GPU, its power limit and SM clock (read in the same process). `--profile-kernel` instead times the stem dgrad kernel
with torch.profiler over one attack iteration of PSPNet50.
"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in q.stdout.strip().split(",")]
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = (vals + ["unknown"] * 3)[:3]
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = info["sm_clock"] = "unknown"
    return info


def _nets(arch, classes):
    from model.pspnet import PSPNet
    from model.psanet import PSANet
    torch.manual_seed(0)
    if arch == "psp":
        return PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False), 473, {}
    return PSANet(layers=50, classes=classes, zoom_factor=8, psa_type=2, mask_h=59, mask_w=59,
                  pretrained=False), 465, dict(psa_type=2, mask_h=59, mask_w=59)


def _timed(fn, steps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _attack_arms(arch, args, dev):
    from oracle.torch_oracle import Oracle
    model, size, okw = _nets(arch, args.classes)
    model = model.to(dev).eval()
    for p in model.parameters():
        p.requires_grad_(False)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    orc = Oracle(sd, arch=arch, layers=50, classes=args.classes, **okw).eval()
    x0, y = bench.synth_batch(args.batch, size, args.classes, 100)
    x0, y = x0.to(dev), y.to(dev)
    state = {"ours": x0.clone(), "cudnn": x0.clone()}
    fwd = {"ours": model, "cudnn": orc.forward}

    def it(name):
        def run():
            x = state[name].requires_grad_(True)
            F.cross_entropy(fwd[name](x), y, ignore_index=255).backward()
            with torch.no_grad():
                state[name] = (x + (1.0 / 255) * x.grad.sign()).detach()
        return run
    return {"%s_attack_%s" % (arch, k): it(k) for k in fwd}


def _train_arms(args, dev):
    from model.pspnet import PSPNet
    torch.manual_seed(0)
    base = PSPNet(layers=50, classes=args.classes, zoom_factor=8, pretrained=False).to(dev).train()
    x, y = bench.synth_batch(args.batch, 473, args.classes, 100)
    x, y = x.to(dev), y.to(dev)
    arms = {}
    for want_dx in (False, True):
        m = copy.deepcopy(base)
        opt = bench.build_optimizer(m, "psp")

        def run(m=m, opt=opt, want_dx=want_dx):
            xi = x.clone().requires_grad_(want_dx)
            _, ml, al = m(xi, y)
            opt.zero_grad()
            (ml + 0.4 * al).backward()
            opt.step()
        arms["psp_train_%s" % ("with_dx" if want_dx else "no_dx")] = (run, m)
    return arms


def profile_kernel(args, dev):
    from torch.profiler import ProfilerActivity, profile
    run = _attack_arms("psp", args, dev)["psp_attack_ours"]
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        if "stem_dgrad" in e.key or "im2col" in e.key or "phases" in e.key:
            rows[e.key] = {"calls": e.count, "us_per_call": e.device_time_total / max(e.count, 1)}
    print(json.dumps(dict(_gpu_info(), workload="PSPNet50 473x473, %d images, bf16, eval attack iteration" % args.batch,
                          kernels=rows)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed iterations per round and arm")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--profile-kernel", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_input_grad measures on a GPU"
    dev = torch.device("cuda", 0)
    if args.profile_kernel:
        return profile_kernel(args, dev)
    rounds, kernels = {}, {}
    # one group of arms at a time (fp32 oracle activations of 16 images are large), alternating within the group
    for group in ("psp", "psa", "train"):
        if group == "train":
            train = _train_arms(args, dev)
            arms = {k: v[0] for k, v in train.items()}
        else:
            arms = _attack_arms(group, args, dev)
        for name, fn in arms.items():              # eager warm-up, and graph capture of the training arms
            for _ in range(2 + (graphs.WARMUP_CALLS + 1 if group == "train" else 0)):
                fn()
        for name in arms:
            rounds[name] = []
        for _ in range(args.rounds):
            for name, fn in arms.items():
                rounds[name].append(_timed(fn, args.steps))
        if group == "train":
            kernels = {k: graphs.launches_per_step(v[1]) for k, v in train.items()}
            del train
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(dict(_gpu_info(), batch=args.batch, classes=args.classes, precision="bf16",
                          steps_per_round=args.steps, ms_per_iteration=rounds, kernels_per_graphed_step=kernels)),
          flush=True)


if __name__ == "__main__":
    main()
