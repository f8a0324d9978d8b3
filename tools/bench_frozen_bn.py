"""Training-step throughput with frozen BatchNorm against the same step with batch statistics.

Frozen BN is the fine-tuning recipe `model.train()`, then `.eval()` on every BatchNorm layer: the layers normalise with
their running statistics, do not update them, and still pass gradients (DESIGN.md §1, §4). Both arms run bench.py's step
(tool/train.py:267-276: model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the reference's
8 parameter groups) on the same workload: PSPNet50 473x473, 150 classes, 16 images by default, one GPU, the default
`bf16` mode, CUDA graphs as the package uses them by default.

The arms are two copies of one seeded model. The frozen copy first gets the running statistics of one batch (a
no-grad batch-statistics forward with momentum 1), as a network fine-tuned from a checkpoint has meaningful statistics;
with the constructor's (0, 1) statistics a frozen BN normalises nothing. After the warm-up (eager calls and the graph
capture of each arm), the arms are timed alternately, `--rounds` times `--steps` steps each, with CUDA events. Prints
one JSON line: the GPU and its power limit (read in the same process), img/s and ms/step of every round of both arms,
and the losses of the last timed frozen step. `--dump-outputs DIR` also writes that step's prediction and losses as
DIR/<name>.npy (bench.py's format). Not part of bench.py's contract (that one measures the batch-statistics step).
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
import torch.nn as nn  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit"] = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = "unknown"
    return info


def _bns(model):
    return [m for m in model.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per round and arm")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3, help="eager steps per arm before the graph warm-up")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--layers", type=int, default=50)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_frozen_bn measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    base = PSPNet(layers=args.layers, classes=args.classes, zoom_factor=8, pretrained=False).to(dev).train()
    x, y = bench.synth_batch(args.batch, args.size, args.classes, 100)
    x, y = x.to(dev), y.to(dev)
    arms = {"batch_stats": copy.deepcopy(base), "frozen_bn": copy.deepcopy(base)}
    frozen = arms["frozen_bn"]
    moms = [m.momentum for m in _bns(frozen)]
    for m in _bns(frozen):
        m.momentum = 1.0
    with torch.no_grad():
        frozen(x, y)                               # running statistics of one batch
    for m, mom in zip(_bns(frozen), moms):
        m.momentum = mom
        m.eval()
    opts = {k: bench.build_optimizer(m, "psp") for k, m in arms.items()}
    last = {}

    def step(name):
        out, main_loss, aux_loss = arms[name](x, y)
        loss = main_loss + 0.4 * aux_loss
        opts[name].zero_grad()
        loss.backward()
        opts[name].step()
        last[name] = dict(prediction=out, main_loss=main_loss, aux_loss=aux_loss, loss=loss)

    def timed(name):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            step(name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    n_warm = max(3, args.warmup) + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for name in arms:
        for _ in range(n_warm):
            step(name)
    rounds = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name in arms:                          # alternating: batch statistics, frozen, batch statistics, ...
            ms = timed(name)
            rounds[name].append({"img_per_s": args.batch * args.steps / (ms / 1e3), "ms_per_step": ms / args.steps})
    if args.dump_outputs:
        bench.dump_outputs(args.dump_outputs, {k: v.detach().float().cpu().numpy()
                                               for k, v in last["frozen_bn"].items()})
    out = dict(_gpu_info(), workload="PSPNet%d %dx%d, %d classes, %d images, bf16, one GPU" % (
        args.layers, args.size, args.size, args.classes, args.batch), steps_per_round=args.steps,
        kernels_per_graphed_step={k: graphs.launches_per_step(m) for k, m in arms.items()}, rounds=rounds,
        frozen_last_losses={k: last["frozen_bn"][k].item() for k in ("main_loss", "aux_loss")})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
