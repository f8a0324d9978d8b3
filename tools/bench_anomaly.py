"""Cost of anomaly segmentation (semseg_b200/anomaly.py, csrc/anomaly.cu, the stats variant of csrc/window.cu).

  * the scores kernel: ops.window_scores against ops.window_scores_stats (two more channels) on 8 flipped 713 x 713
    crops, at 19 and 150 classes, the two alternated, CUDA events;
  * one SlidingWindowPredictor image at Cityscapes shape (1024 x 2048, 19 classes, crop 713, seeded PSPNet50 in eval
    mode), single scale and the six-scale set, with anomaly=None, AnomalyScorer('maxlogit') and AnomalyScorer('sml'),
    the arms alternated over `--rounds` rounds: median and range per arm;
  * the SML post-processing alone (ops.anomaly_sml) at 1024 x 2048;
  * AnomalyMeter.compute() over `--maps` synthetic 1024 x 2048 maps (ties, 10 % void), against sklearn's
    roc_auc_score + average_precision_score on the host over `--host-maps` of them, with the per-pixel rate ratio.
Everything is timed with CUDA events or a host clock around work that ends in a device synchronise, after a warm-up.
Prints one JSON line per measurement with the GPU name, power limit and SM clock read in the same process.
Not part of bench.py's contract.
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
from semseg_b200.anomaly import AnomalyMeter, AnomalyScorer  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

SIX_SCALES = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75]
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def _emit(rec, info):
    rec.update(info)
    print(json.dumps(rec), flush=True)


def _events(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_kernel(info, iters):
    for C in (19, 150):
        g, crop = 8, 713
        h = (crop - 1) // 8 + 1
        gen = torch.Generator(device="cuda").manual_seed(C)
        logits = torch.randn((2 * g, h, h, C), device="cuda", generator=gen) * 4
        plain = torch.empty((g, C, crop, crop), device="cuda")
        stats = torch.empty((g, C + 2, crop, crop), device="cuda")
        arms = {"window_scores": lambda: ops.window_scores(logits, True, plain),
                "window_scores_stats": lambda: ops.window_scores(logits, True, stats, stats=True)}
        for fn in arms.values():
            _events(fn, 3)
        times = {k: [] for k in arms}
        for _ in range(3):
            for k, fn in arms.items():
                times[k].append(_events(fn, iters))
        _emit({"bench": "window_scores", "classes": C, "crops": g, "crop": crop, "flip": True,
               "ms": {k: round(min(v), 4) for k, v in times.items()},
               "ms_all": {k: [round(t, 4) for t in v] for k, v in times.items()},
               "stats_over_plain": round(min(times["window_scores_stats"]) / min(times["window_scores"]), 4)}, info)


def bench_predictor(info, rounds):
    from semseg_b200 import inference
    from tests import util
    classes, crop, h, w = 19, 713, 1024, 2048
    model = util.build_pspnet(50, classes=classes).cuda().eval()
    image = (np.random.default_rng(0).random((h, w, 3)) * 255).astype(np.float32)
    make = lambda a=None: inference.SlidingWindowPredictor(model, classes, crop, crop, MEAN, STD,  # noqa: E731
                                                             max_batch=16, anomaly=a)
    fit = AnomalyScorer("sml").fit(make(), [image], w, [1.0])
    arms = {"none": make(), "maxlogit": make(AnomalyScorer("maxlogit")),
            "sml": make(AnomalyScorer("sml", statistics=fit.statistics))}
    for name, scales in (("single", [1.0]), ("six", SIX_SCALES)):
        for p in arms.values():
            p(image, w, scales, return_scores=False)
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, p in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = p(image, w, scales, return_scores=False)
                if len(out) == 3:
                    out[2].cpu()
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) * 1e3)
        _emit({"bench": "predictor", "shape": [h, w], "classes": classes, "crop": crop, "scales": scales,
               "ms_median": {k: round(float(np.median(v)), 1) for k, v in times.items()},
               "ms_range": {k: [round(min(v), 1), round(max(v), 1)] for k, v in times.items()},
               "rounds": rounds, "set": name}, info)


def bench_sml(info, iters):
    h, w, classes = 1024, 2048, 19
    rng = np.random.default_rng(1)
    coarse = rng.integers(0, classes, (h // 32 + 1, w // 32 + 1))
    pred = torch.from_numpy(np.kron(coarse, np.ones((32, 32), np.int64))[:h, :w]).cuda()
    total = torch.zeros((classes + 2, h, w), dtype=torch.float64, device="cuda")
    total[classes] = torch.randn((h, w), dtype=torch.float64, device="cuda") * 2 + 8
    sc = AnomalyScorer("sml", statistics=(np.full(classes, 8.0), np.full(classes, 2.0)))
    _events(lambda: sc.score_map(total, pred), 3)
    ms = [_events(lambda: sc.score_map(total, pred), iters) for _ in range(3)]
    _emit({"bench": "sml_postprocess", "shape": [h, w], "defaults": repr(sc), "ms": round(min(ms), 3),
           "ms_all": [round(t, 3) for t in ms]}, info)


def bench_meter(info, maps, host_maps):
    from sklearn.metrics import average_precision_score, roc_auc_score
    h, w = 1024, 2048
    meter = AnomalyMeter()
    gen = torch.Generator(device="cuda").manual_seed(2)
    host = []
    for k in range(maps):
        s = torch.round(torch.randn((h, w), device="cuda", generator=gen) * 100) / 100      # ties
        y = (torch.rand((h, w), device="cuda", generator=gen) < 0.02 + 0.3 * (s > 1.5)).to(torch.uint8)
        y[torch.rand((h, w), device="cuda", generator=gen) < 0.1] = 255
        meter.update(s, y)
        if k < host_maps:
            host.append((s.cpu().numpy().ravel(), y.cpu().numpy().ravel()))
    meter.compute()                                          # warm-up
    torch.cuda.synchronize()
    t = []
    for _ in range(2):
        t0 = time.perf_counter()
        res = meter.compute()
        t.append(time.perf_counter() - t0)
    s = np.concatenate([a for a, _ in host])
    y = np.concatenate([b for _, b in host])
    keep = y != 255
    t0 = time.perf_counter()
    roc_auc_score(y[keep], s[keep])
    average_precision_score(y[keep], s[keep])
    t_host = time.perf_counter() - t0
    rate_dev = meter.count / min(t)
    rate_host = s.size / t_host
    _emit({"bench": "meter_compute", "maps": maps, "pixels": meter.count, "s": round(min(t), 3),
           "s_all": [round(v, 3) for v in t], "result": res, "sklearn_maps": host_maps, "sklearn_pixels": int(s.size),
           "sklearn_s": round(t_host, 3), "pixels_per_s_device": round(rate_dev), "pixels_per_s_sklearn": round(rate_host),
           "rate_ratio": round(rate_dev / rate_host, 1)}, info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="launches per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="alternated predictor rounds")
    ap.add_argument("--maps", type=int, default=100, help="1024 x 2048 maps in the meter")
    ap.add_argument("--host-maps", type=int, default=2, help="maps scored by sklearn on the host")
    ap.add_argument("--only", default="kernel,predictor,sml,meter")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    info = _gpu_info()
    parts = args.only.split(",")
    if "kernel" in parts:
        bench_kernel(info, args.iters)
    if "sml" in parts:
        bench_sml(info, args.iters)
    if "meter" in parts:
        bench_meter(info, args.maps, args.host_maps)
    if "predictor" in parts:
        bench_predictor(info, args.rounds)


if __name__ == "__main__":
    main()
