"""Training-step throughput at every zoom factor: the native tail against the ATen tail.

`zoom_factor` (1, 2, 4 or 8) sets the resolution the losses are taken at: the 1/8-resolution logits are upsampled xZ and
the target is downsampled to that size by the trainer (tool/train.py:262-266). Two arms run bench.py's step
(tool/train.py:267-276: model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD with the reference's
8 parameter groups) on PSPNet50 473x473, 150 classes, one GPU, the default `bf16` mode:
  * native: the fused upsample + cross-entropy + argmax kernels of csrc/tail.cu, the step replayed from CUDA graphs;
  * aten  : the same network whose criterion is a trivial subclass of nn.CrossEntropyLoss, which keeps the ATen tail
            (F.interpolate -> CrossEntropyLoss -> max) and with it the eager step.
Both arms are copies of one seeded model per zoom factor and run at 16 and at 2 images per step. The target is a seeded
label map without ignored pixels, downsampled as the trainer does, with ~5 % of its pixels then set to 255 (interpolating
255 into class ids would give labels >= classes, on which ATen's nll_loss asserts). After the warm-up (eager calls and,
for the native arm, the graph capture) `--steps` steps are timed with CUDA events. Prints one JSON line per zoom factor
and arm: the GPU and its power limit (read in the same process), img/s and ms/step at each batch size, and the kernels per
graphed step. Not part of bench.py's contract (that one measures zoom 8).
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
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402


class ATenCrossEntropy(nn.CrossEntropyLoss):
    """nn.CrossEntropyLoss under another type: the network keeps the ATen tail."""


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit"] = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = "unknown"
    return info


def zoom_batch(n, size, classes, zoom, seed, dev):
    """Input [n, 3, size, size] and the target at zoom `zoom`, built as tool/train.py:262-266 builds it."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, 3, size, size), generator=g)
    y = torch.randint(0, classes, (n, size, size), generator=g)
    if zoom != 8:
        h = int((y.size()[1] - 1) / 8 * zoom + 1)
        w = int((y.size()[2] - 1) / 8 * zoom + 1)
        y = F.interpolate(y.unsqueeze(1).float(), size=(h, w), mode='bilinear', align_corners=True).squeeze(1).long()
    y[torch.rand(y.shape, generator=g) < 0.05] = 255
    return x.to(dev), y.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per zoom factor, batch size and arm")
    ap.add_argument("--warmup", type=int, default=3, help="eager steps per arm before the graph warm-up")
    ap.add_argument("--batches", default="16,2", help="images per step, comma separated")
    ap.add_argument("--zooms", default="1,2,4,8")
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--layers", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_zoom measures on a GPU; there is no CPU arm"
    from model.pspnet import PSPNet

    dev = torch.device("cuda", 0)
    info = _gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    n_warm = max(3, args.warmup) + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    for zoom in (int(z) for z in args.zooms.split(",")):
        torch.manual_seed(0)
        base = PSPNet(layers=args.layers, classes=args.classes, zoom_factor=zoom, pretrained=False).train()
        results = {"native": {}, "aten": {}}
        kernels = {}
        for n in batches:
            x, y = zoom_batch(n, args.size, args.classes, zoom, 100, dev)
            for arm in results:
                model = copy.deepcopy(base).to(dev)
                if arm == "aten":
                    model.criterion = ATenCrossEntropy(ignore_index=255)
                opt = bench.build_optimizer(model, "psp")

                def step():
                    _, main_loss, aux_loss = model(x, y)
                    loss = main_loss + 0.4 * aux_loss
                    opt.zero_grad()
                    loss.backward()
                    opt.step()

                for _ in range(n_warm):
                    step()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1)
                results[arm]["batch%d" % n] = {"img_per_s": n * args.steps / (ms / 1e3), "ms_per_step": ms / args.steps}
                kernels.setdefault(arm, {})["batch%d" % n] = graphs.launches_per_step(model)
                del model, opt
                torch.cuda.empty_cache()
        for arm, r in results.items():
            print(json.dumps(dict(info, zoom=zoom, arm=arm, workload="PSPNet%d %dx%d, %d classes, bf16, one GPU" % (
                args.layers, args.size, args.size, args.classes), steps=args.steps, results=r,
                kernels_per_graphed_step=kernels[arm])), flush=True)


if __name__ == "__main__":
    main()
