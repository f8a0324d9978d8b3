"""Cost of the dual-stream perturbation of mean-teacher training (losses.PseudoLabelLoss / MixPseudoLabelLoss
streams=2, UniMatch's two strong views of every image in one student pass).

The graphed PSPNet50 mean-teacher step (bench.py's step plus ema.update) at 473 x 473 with 150 classes, on
MixPseudoLabelLoss(mix='cutmix', strong=StrongAugment(), fp_weight=0.25) and an optim.ModelEMA teacher, N images of
which half all-ignore, at streams=1 and streams=2, the arms alternating over `--rounds` rounds in one process. Per arm:
ms per step, images per second of the N-image batch, torch.cuda.max_memory_allocated and the native kernels per graphed
step. N = 8 runs first; N = 16 runs only when twice N = 8's dual-stream peak fits the card's memory with a 10 % margin
(activations grow with the batch), else the JSON line says it does not fit.

Expected from shapes, not measured here: the student's backbone, heads and tail do 2N images and the teacher stays at N,
so a dual step costs roughly 1.6-2x a single one. Prints one JSON line per measurement with the GPU, its power limit
and SM clock, read in the same process. Not part of bench.py's contract.
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
from tools.bench_ohem import _gpu_info  # noqa: E402


def _net(classes):
    from model.pspnet import PSPNet
    torch.manual_seed(0)
    return PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False).train()


def step_bench(info, args, dev, n, size=473, classes=150):
    """{streams: {'ms': [per round], 'peak_gb', 'kernels'}} of the two arms at batch n."""
    n_warm = 3 + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    base = _net(classes)
    x, y = bench.synth_batch(n, size, classes, 100)
    y[n // 2:] = 255                                   # the unlabelled half of the batch
    x, y = x.to(dev), y.to(dev)
    runs = {s: dict(ms=[]) for s in (1, 2)}
    for _ in range(args.rounds):
        for streams, r in runs.items():
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            model = copy.deepcopy(base).to(dev)
            opt = bench.build_optimizer(model, "psp", kind="fused")
            ema = ModelEMA(model, decay=0.999)
            model.criterion = MixPseudoLabelLoss(ema.module, mix='cutmix', threshold=0.95, strong=StrongAugment(),
                                                 ce_weight=0.5, pl_weight=0.25, fp_weight=0.25, streams=streams)

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
    for streams, r in runs.items():
        print(json.dumps(dict(info, workload="PSPNet50 student, %dx%d, %d classes, %d images (half unlabelled), cutmix + "
                              "strong + fp_weight 0.25, EMA teacher, bf16, one GPU, graphed" % (size, size, classes, n),
                              arm="streams=%d" % streams, n=n, steps=args.steps,
                              ms_per_step=[round(v, 2) for v in r["ms"]],
                              images_per_s=[round(n * 1e3 / v, 1) for v in r["ms"]], peak_gb=r["peak_gb"],
                              kernels_per_graphed_step=r["kernels"])), flush=True)
    print(json.dumps(dict(info, workload="step time ratio streams 2 / 1, %d images" % n,
                          measured_ratio=round(min(runs[2]["ms"]) / min(runs[1]["ms"]), 3),
                          expected_from_shapes="1.6-2 (not measured)")), flush=True)
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8, help="timed steps per window")
    ap.add_argument("--rounds", type=int, default=2, help="windows per arm, the arms alternating")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dual measures on a GPU; there is no CPU arm"
    dev = torch.device("cuda", 0)
    info = _gpu_info()
    runs = step_bench(info, args, dev, 8)
    total_gb = torch.cuda.get_device_properties(dev).total_memory / 1e9
    need_gb = 2 * runs[2]["peak_gb"]
    if need_gb <= 0.9 * total_gb:
        step_bench(info, args, dev, 16)
    else:
        print(json.dumps(dict(info, workload="16 images, streams=2", fits=False, peak_gb_at_8=runs[2]["peak_gb"],
                              estimate_gb_at_16=round(need_gb, 1), card_gb=round(total_gb, 1))), flush=True)


if __name__ == "__main__":
    main()
