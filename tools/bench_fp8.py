"""FP8 (e4m3) inference vs bf16 on the same card in one call (semseg_b200/fp8.py). Prints one JSON line with the GPU and
its power limit and:
  convs          : kernel time of single eval convs (conv + folded BN + ReLU), bf16 vs e4m3 at config5 / ade20k feature
                   shapes, as achieved TFLOP/s (2*M*Cin*Cout*taps / time) and as a share of the H100 SXM data-sheet dense
                   rate (989 TFLOP/s bf16, 1979 TFLOP/s FP8); the e4m3 time excludes quantising the input
  presets        : images/s of tools/bench_inference.py's network_only arm (the network calls of all crops of six scales
                   with flip, no finish) and device_finish_batched arm (SlidingWindowPredictor), bf16 and FP8 alternated,
                   --repeats times each
  calibrate_freeze_s : one calibrate() batch plus freeze() of PSPNet101
Not part of bench.py's contract (that one measures the training step)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from semseg_b200 import inference, ops  # noqa: E402
from semseg_b200.fp8 import Fp8Eval  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402

PRESETS = {   # tools/bench_inference.py's presets
    "config5": dict(layers=101, classes=19, crop=713, height=1024, width=2048, base_size=2048),
    "ade20k": dict(layers=50, classes=150, crop=473, height=512, width=683, base_size=512),
}
SCALES = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75]
MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
PEAK = {"bf16": 989.0, "e4m3": 1979.0}


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unknown"
    return info


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def bench_convs(iters):
    # (label, N, H, W, Cin, Cout, k, dilation): config5 crops at 713 -> 90x90 features, 16 crops per call; ade20k 473 ->
    # 60x60, 16 per call
    cases = [("config5 cls.0 3x3 4096->512", 16, 90, 90, 4096, 512, 3, 1),
             ("config5 layer4 conv2 3x3 d4 512->512", 16, 90, 90, 512, 512, 3, 4),
             ("config5 layer3 conv1 1x1 1024->256", 16, 90, 90, 1024, 256, 1, 1),
             ("config5 layer4 conv3 1x1 512->2048", 16, 90, 90, 512, 2048, 1, 1),
             ("ade20k cls.0 3x3 4096->512", 16, 60, 60, 4096, 512, 3, 1),
             ("ade20k layer3 conv2 3x3 d2 256->256", 16, 60, 60, 256, 256, 3, 2)]
    out = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for label, n, h, w, cin, cout, k, dil in cases:
        x = torch.randn((n, h, w, cin), device="cuda", generator=g).to(torch.bfloat16)
        wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) / (cin * k * k) ** 0.5
        scale = torch.ones(cout, device="cuda")
        shift = torch.zeros(cout, device="cuda")
        taps = ops.conv_taps(k, dil)
        wf = ops.pack_weights(wt, need_dgrad=False).wf
        wf8, sw = ops.fp8_pack_weights(wt)
        x8 = ops.fp8_quantize(x, 448.0 / float(x.float().abs().max()))
        t16 = _time(lambda: ops.conv_fprop(x, wf, cout, taps, epi=ops.EPI_AFFINE, relu=True, scale=scale,
                                           shift=shift), iters)
        t8 = _time(lambda: ops.conv_fprop_e4m3(x8, wf8, cout, taps, scale=sw, shift=shift, relu=True), iters)
        flop = 2.0 * n * h * w * cin * cout * k * k
        out.append({"conv": label, "bf16_ms": round(t16 * 1e3, 4), "e4m3_ms": round(t8 * 1e3, 4),
                    "bf16_tflops": round(flop / t16 / 1e12, 1), "e4m3_tflops": round(flop / t8 / 1e12, 1),
                    "bf16_share_of_datasheet": round(flop / t16 / 1e12 / PEAK["bf16"], 3),
                    "e4m3_share_of_datasheet": round(flop / t8 / 1e12 / PEAK["e4m3"], 3)})
    return out


def _network_only(net, image_hw, crop, max_batch):
    """The network calls of every crop of every scale (flip doubles each batch), no crop extraction and no finish."""
    h0, w0 = image_hw
    x = torch.zeros((max_batch // 2, 3, crop, crop), device="cuda")
    with torch.no_grad():
        for s in SCALES:
            h, w = int(h0 * s + 0.5), int(w0 * s + 0.5)
            n = (len(inference.crop_origins(max(h, crop), crop)) * len(inference.crop_origins(max(w, crop), crop)))
            for g0 in range(0, n, max_batch // 2):
                part = x[:min(max_batch // 2, n - g0)]
                net._eval_logits_nhwc(torch.cat([part, part.flip(3)], 0))


def bench_preset(name, repeats, max_batch):
    c = PRESETS[name]
    torch.manual_seed(0)
    model = PSPNet(layers=c["layers"], classes=c["classes"], zoom_factor=8, pretrained=False).cuda().eval()
    rng = np.random.default_rng(0)
    image = rng.integers(0, 256, (c["height"], c["width"], 3)).astype(np.float32)
    q = Fp8Eval(model)
    q.calibrate(((torch.from_numpy(image[:c["crop"], :c["crop"]]).cuda().permute(2, 0, 1)[None] -
                  torch.tensor(MEAN, device="cuda")[:, None, None]) / torch.tensor(STD, device="cuda")[:, None, None]))
    q.freeze()
    nets = {"bf16": model, "fp8": q}
    preds = {k: inference.SlidingWindowPredictor(v, c["classes"], c["crop"], c["crop"], MEAN, STD, max_batch=max_batch)
             for k, v in nets.items()}
    res = {"network_only": {"bf16": [], "fp8": []}, "device_finish_batched": {"bf16": [], "fp8": []}}
    for k in nets:                                            # warm-up of every shape
        _network_only(nets[k], image.shape[:2], c["crop"], max_batch)
        preds[k](image, c["base_size"], SCALES)
    for _ in range(repeats):
        for k in ("bf16", "fp8"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _network_only(nets[k], image.shape[:2], c["crop"], max_batch)
            torch.cuda.synchronize()
            res["network_only"][k].append(1.0 / (time.perf_counter() - t0))
            t0 = time.perf_counter()
            preds[k](image, c["base_size"], SCALES)
            torch.cuda.synchronize()
            res["device_finish_batched"][k].append(1.0 / (time.perf_counter() - t0))
    a, _ = preds["bf16"](image, c["base_size"], SCALES)
    b, _ = preds["fp8"](image, c["base_size"], SCALES)
    out = {arm: {k: {"images_per_s": [round(v, 3) for v in vals], "median": round(float(np.median(vals)), 3),
                     "min": round(min(vals), 3), "max": round(max(vals), 3)}
                 for k, vals in d.items()} for arm, d in res.items()}
    for arm in out:
        out[arm]["fp8_speedup_median"] = round(out[arm]["fp8"]["median"] / out[arm]["bf16"]["median"], 3)
        # the slowest FP8 repeat against the fastest bf16 one: > 1 means no overlap of the two spreads
        out[arm]["fp8_min_over_bf16_max"] = round(out[arm]["fp8"]["min"] / out[arm]["bf16"]["max"], 3)
    out["argmax_agreement_fp8_vs_bf16"] = round(float((a.argmax(2) == b.argmax(2)).mean()), 4)
    return out


def bench_calibrate_freeze():
    torch.manual_seed(0)
    model = PSPNet(layers=101, classes=19, zoom_factor=8, pretrained=False).cuda().eval()
    x = torch.randn((8, 3, 713, 713), device="cuda")
    Fp8Eval(model).calibrate(x[:1])                           # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    q = Fp8Eval(model)
    q.calibrate(x)
    q.freeze()
    torch.cuda.synchronize()
    return round(time.perf_counter() - t0, 3)


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--conv-iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a CUDA device")
    out = _gpu_info()
    out["convs"] = bench_convs(args.conv_iters)
    out["presets"] = {p: bench_preset(p, args.repeats, args.max_batch) for p in ("config5", "ade20k")}
    out["calibrate_freeze_s"] = bench_calibrate_freeze()
    out.update(_gpu_info())                                   # read again after the runs: the same card
    print(json.dumps(out))


if __name__ == "__main__":
    main()
