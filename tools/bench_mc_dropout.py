"""Cost of Monte Carlo dropout in the sliding-window predictor (semseg_b200/inference.py, mc_draws > 0;
csrc/window.cu's semseg_window_scores_mc).

At two shapes, seeded networks in eval mode with dropout 0.1, one image, flip on:
  * Cityscapes: PSPNet101, 19 classes, 1024 x 2048 image, crop 713, scale 1.0;
  * ADE20K: PSPNet50, 150 classes, 512 x 683 image, crop 473, scale 1.0;
it times one predictor call (host clock around work that ends in a device synchronise, arms alternated over `--rounds`
rounds after a warm-up round: median and range) for the deterministic predictor, the native MC predictor at
T in {4, 8, 20}, and the ATen path (the same network behind a wrapper the predictor does not recognise) at the same T.
It also times the MC scores kernel alone against T launches of window_scores on the same per-draw logits (CUDA events),
and states the bytes and FLOPs of the MC head per crop batch, computed from the shapes.
Prints one JSON line per shape with the GPU name and power limit read in the same process. Not part of bench.py.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from semseg_b200 import ops  # noqa: E402
from semseg_b200.inference import SlidingWindowPredictor, crop_origins  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]
SHAPES = {"cityscapes": dict(layers=101, classes=19, h=1024, w=2048, crop=713),
          "ade20k": dict(layers=50, classes=150, h=512, w=683, crop=473)}
DRAWS = (4, 8, 20)


class _Foreign(torch.nn.Module):
    """The same network behind a module the predictor does not recognise: the ATen path."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x)


def _events(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def head_cost(g, hn, wn, classes, crop, draws):
    """Bytes and FLOPs of the MC head for one batch of g crops (2g images with their mirrors) over `draws` draws, bf16
    feature: the masked 512-channel feature (read + write), the 1x1 classifier, its fp32 logits (write, then read by
    the scores kernel) and the scores kernel's fp32 output [g, classes + 1, crop, crop]."""
    px = 2 * g * hn * wn
    feat = draws * px * 512 * 2 * 2
    conv_flops = draws * 2 * px * 512 * classes
    logits = draws * px * classes * 4 * 2
    out = g * (classes + 1) * crop * crop * 4
    return {"bytes": feat + logits + out, "flops": conv_flops, "feature_bytes": feat, "logit_bytes": logits,
            "score_bytes": out}


def bench_shape(name, cfg, rounds, iters):
    classes, crop, h, w = cfg["classes"], cfg["crop"], cfg["h"], cfg["w"]
    torch.manual_seed(0)
    net = PSPNet(layers=cfg["layers"], classes=classes, zoom_factor=8, dropout=0.1, pretrained=False).cuda().eval()
    image = (np.random.default_rng(0).random((h, w, 3)) * 255).astype(np.float32)
    g = len(crop_origins(h, crop)) * len(crop_origins(w, crop))
    make = lambda m, t=0: SlidingWindowPredictor(m, classes, crop, crop, MEAN, STD, max_batch=2 * g,  # noqa: E731
                                                 mc_draws=t)
    arms = {"deterministic": make(net)}
    for t in DRAWS:
        arms["native_T%d" % t] = make(net, t)
    for t in DRAWS:
        arms["aten_T%d" % t] = make(_Foreign(net), t)
    times = {k: [] for k in arms}
    with torch.no_grad():
        for r in range(rounds + 1):                      # round 0 warms every arm up
            for k, p in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = p(image, w, [1.0], return_scores=False)
                if len(out) == 3:
                    out[2].cpu()
                torch.cuda.synchronize()
                if r:
                    times[k].append((time.perf_counter() - t0) * 1e3)
    rec = {"bench": "mc_dropout", "shape": name, "arch": "PSPNet%d" % cfg["layers"], "classes": classes,
           "image": [h, w], "crop": crop, "scale": 1.0, "flip": True, "crops": g, "rounds": rounds,
           "call_ms_median": {k: round(float(np.median(v)), 2) for k, v in times.items()},
           "call_ms_range": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()}}
    det = float(np.median(times["deterministic"]))
    rec["over_deterministic"] = {k: round(float(np.median(v)) / det, 3) for k, v in times.items()}
    rec["aten_over_native"] = {t: round(float(np.median(times["aten_T%d" % t])) /
                                        float(np.median(times["native_T%d" % t])), 2) for t in DRAWS}
    # the kernel alone, on the network's own per-draw logits of the batch
    hn = (crop - 1) // 8 + 1
    x = torch.randn((2 * g, 3, crop, crop), device="cuda") * 50
    kern = {}
    for t in DRAWS:
        logits = net._mc_eval_logits_nhwc(x, t)
        mc_out = torch.empty((g, classes + 1, crop, crop), device="cuda")
        plain = torch.empty((g, classes, crop, crop), device="cuda")

        def plain_all():
            for k in range(t):
                ops.window_scores(logits[k], True, plain)

        fns = {"window_scores_mc": lambda: ops.window_scores_mc(logits, True, mc_out), "window_scores_xT": plain_all}
        for fn in fns.values():
            _events(fn, 2)
        ms = {k: [] for k in fns}
        for _ in range(3):
            for k, fn in fns.items():
                ms[k].append(_events(fn, iters))
        kern["T%d" % t] = {k: round(min(v), 3) for k, v in ms.items()}
        kern["T%d" % t]["head"] = head_cost(g, hn, hn, classes, crop, t)
        del logits
    rec["kernel_ms"] = kern
    rec.update(_gpu_info())
    print(json.dumps(rec), flush=True)
    del arms, net
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--rounds", type=int, default=3, help="timed predictor rounds per arm, alternated")
    ap.add_argument("--iters", type=int, default=10, help="kernel launches per timed window")
    ap.add_argument("--only", default=",".join(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mc_dropout needs a CUDA device")
    torch.cuda.set_device(0)
    for name in args.only.split(","):
        bench_shape(name, SHAPES[name], args.rounds, args.iters)


if __name__ == "__main__":
    main()
