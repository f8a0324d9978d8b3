"""Cost of the dense CRF (semseg_b200.densecrf.DenseCRF, csrc/densecrf.cu) at the evaluation shapes users run.

For ADE20K (512 x 683, 150 classes) and Cityscapes (1024 x 2048, 19 classes), on two seeded images (noisy colour
regions, and a smooth scene-like layout whose flat areas make the splat's per-vertex runs long) and softmax scores of
random logits, with the default parameters (pos 3 / 3, bi 10 / 80 / 13):
  * the lattice build (both kernels, ops.densecrf_build including its one host read of V), V of each kernel, and one
    build's device time per kernel family from torch.profiler (after the timed runs);
  * the per-iteration time of each kernel alone (mean field with only that kernel's weight, (t(k) - t(0)) / k);
  * the whole CRF (build + mean field) at 5 and 10 iterations, and torch.cuda.max_memory_allocated over it;
  * one SlidingWindowPredictor image (seeded PSPNet50 in eval mode, crop 473 / 713, one scale, the noisy image) with
    and without crf, the two arms alternated over `--rounds` rounds: median and range of each and of their difference;
  * the float64 numpy lattice of tests/densecrf_oracle.py at a reduced size (`--oracle-size`), for scale.
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
from semseg_b200.densecrf import DenseCRF  # noqa: E402
from tools.bench_ohem import _gpu_info  # noqa: E402

SHAPES = {"ade20k": (512, 683, 150, 473), "cityscapes": (1024, 2048, 19, 713)}


def _image(h, w, kind="noisy", seed=0):
    """noisy: six colour regions with per-pixel noise of std 10 (pixels spread over many appearance vertices).
    smooth: a scene-like layout of large flat areas (a sky gradient over the top third, a uniform road band at the
    bottom, a few flat blocks between) with noise of std 1, so that many pixels share a vertex and the splat's runs
    are long, as in sky and road regions of natural images."""
    rng = np.random.default_rng(seed)
    yy, xx = np.indices((h, w))
    if kind == "noisy":
        region = ((xx * 7 // w) + 3 * (yy * 5 // h)) % 6
        palette = rng.uniform(0, 255, (6, 3))
        return np.clip(palette[region] + rng.normal(0, 10, (h, w, 3)), 0, 255).astype(np.float32)
    img = np.empty((h, w, 3))
    t = (yy / max(h - 1, 1))[..., None]
    img[:] = (1 - t) * np.array([90, 150, 230]) + t * np.array([180, 210, 245])          # sky gradient
    mid = (yy >= h // 3) & (yy < 2 * h // 3)
    img[mid] = rng.uniform(0, 255, (5, 3))[(xx[mid] * 5) // w]                           # flat blocks
    img[yy >= 2 * h // 3] = [100, 100, 105]                                              # road
    return np.clip(img + rng.normal(0, 1, (h, w, 3)), 0, 255).astype(np.float32)


def _probs(C, h, w, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.softmax(2 * torch.randn((C, h, w), device="cuda", generator=g), 0)


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


def _host_time(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def _host_time_once(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def _build_split(img_dev):
    """Device time of one build per kernel family (torch.profiler, after the timed runs): the radix sort's hist / scan /
    scatter passes and each dcrf_* kernel."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.densecrf_build(img_dev, 3.0, 80.0, 13.0)
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        name = e.key
        for fam in ("segsort_hist", "segsort_scan", "segsort_scatter", "dcrf_keys", "dcrf_gather_hi", "dcrf_unique_count",
                    "dcrf_scan_tiles", "dcrf_unique_write", "dcrf_neighbours", "dcrf_splat", "dcrf_blur", "dcrf_slice"):
            if fam in name and t > 0:
                split[fam] = round(split.get(fam, 0.0) + t / 1e3, 3)
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="timed repetitions per measurement")
    ap.add_argument("--shapes", default="ade20k,cityscapes")
    ap.add_argument("--oracle-size", type=int, nargs=2, default=(64, 86))
    ap.add_argument("--no-predictor", action="store_true")
    ap.add_argument("--rounds", type=int, default=8, help="alternated predictor calls per arm")
    args = ap.parse_args()
    info = _gpu_info()
    torch.cuda.set_device(0)

    def emit(rec):
        rec.update(info)
        print(json.dumps(rec), flush=True)

    for name, kind in ((n, k) for n in args.shapes.split(",") for k in ("noisy", "smooth")):
        h, w, C, crop = SHAPES[name]
        img = _image(h, w, kind)
        img_dev = torch.from_numpy(img).cuda()
        probs = _probs(C, h, w)
        hwc = probs.permute(1, 2, 0).contiguous()
        flat = hwc.view(h * w, C)
        build_ms = _host_time(lambda: ops.densecrf_build(img_dev, 3.0, 80.0, 13.0), args.iters)
        lattice, V = ops.densecrf_build(img_dev, 3.0, 80.0, 13.0)
        split = _build_split(img_dev)
        rec = {"shape": name, "image": kind, "h": h, "w": w, "classes": C, "build_ms": round(build_ms, 3), "V_smoothness": V[0],
               "V_appearance": V[1], "V_bound": [3 * h * w, 6 * h * w], "build_kernels_ms": split}
        k = 5
        t0 = _time(lambda: ops.densecrf_meanfield(lattice, (h, w), V, flat, 1e-5, 0, 3.0, 10.0), args.iters)
        ts = _time(lambda: ops.densecrf_meanfield(lattice, (h, w), V, flat, 1e-5, k, 3.0, 0.0), args.iters)
        ta = _time(lambda: ops.densecrf_meanfield(lattice, (h, w), V, flat, 1e-5, k, 0.0, 10.0), args.iters)
        tb = _time(lambda: ops.densecrf_meanfield(lattice, (h, w), V, flat, 1e-5, k, 3.0, 10.0), args.iters)
        rec.update({"init_update_ms": round(t0, 3), "smoothness_iter_ms": round((ts - t0) / k, 3),
                    "appearance_iter_ms": round((ta - t0) / k, 3), "both_iter_ms": round((tb - t0) / k, 3)})
        for iters in (5, 10):
            crf = DenseCRF(iterations=iters)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            ms = _host_time(lambda: crf(img, probs), args.iters)
            rec["crf_%d_ms" % iters] = round(ms, 3)
            rec["crf_%d_peak_gb" % iters] = round((torch.cuda.max_memory_allocated() - base) / 1e9, 3)
        del lattice
        emit(rec)

        if not args.no_predictor and kind == "noisy":
            from semseg_b200 import inference
            from tests import util
            model = util.build_pspnet(50, classes=C).cuda().eval()
            mean = [0.485 * 255, 0.456 * 255, 0.406 * 255]
            std = [0.229 * 255, 0.224 * 255, 0.225 * 255]
            rec = {"shape": name, "predictor_crop": crop, "scales": [1.0], "rounds": args.rounds}
            arms = {"plain": inference.SlidingWindowPredictor(model, C, crop, crop, mean, std, max_batch=8),
                    "crf": inference.SlidingWindowPredictor(model, C, crop, crop, mean, std, max_batch=8,
                                                            crf=DenseCRF())}
            times = {a: [] for a in arms}
            for a, p in arms.items():
                p(img, max(h, w), [1.0])                        # warm-up
            for _ in range(args.rounds):                        # the two arms alternated, one call each per round
                for a, p in arms.items():
                    times[a].append(_host_time_once(lambda: p(img, max(h, w), [1.0])))
            for a, ts in times.items():
                rec[a + "_ms_median"] = round(float(np.median(ts)), 2)
                rec[a + "_ms_range"] = [round(min(ts), 2), round(max(ts), 2)]
            diffs = [c - p for c, p in zip(times["crf"], times["plain"])]
            rec["crf_minus_plain_ms_median"] = round(float(np.median(diffs)), 2)
            rec["crf_minus_plain_ms_range"] = [round(min(diffs), 2), round(max(diffs), 2)]
            del model, arms
            torch.cuda.empty_cache()
            emit(rec)

    from tests import densecrf_oracle as O
    oh, ow = args.oracle_size
    img = _image(oh, ow)
    prob = O.softmax(np.random.default_rng(0).normal(0, 2, (oh * ow, 19)))
    t = time.perf_counter()
    O.crf(img, prob, iterations=5)
    emit({"oracle_numpy_lattice": [oh, ow], "classes": 19, "iterations": 5,
          "ms": round((time.perf_counter() - t) * 1e3, 1)})


if __name__ == "__main__":
    main()
