"""Multi-scale sliding-window inference throughput (SURVEY §8 f3): one synthetic image, six scales {0.5 ... 1.75}, flip.
Defaults = BASELINE config 5 (`--preset config5`: PSPNet101, 713 crop, 19 classes, 1024x2048 image, base 2048);
`--preset ade20k` = PSPNet50, 473 crop, 150 classes, a 512x683 image, base 512. Arms through the SAME eval-mode network:
  reference_procedure_serial : one crop + its mirror per model call and the host-side cv2 / numpy finish of
                               tool/test.py:122-199 (the reference's procedure, driven by this package's network)
  reference_finish_batched   : crops batched (`--max-batch`), host-side finish (bit-identical scores)
  device_finish_batched      : crops batched, everything after the network on the native kernels of csrc/window.cu
                               (upsample + softmax + flip average, overlap accumulation, resize + add; the default)
  aten_finish_batched        : the same device finish as ATen ops (F.interpolate / softmax / flip / per-crop canvas
                               updates / F.interpolate), forced by hiding the network behind a plain nn.Module
  network_only               : the per-scale image resize and the same network calls, no crops and no finish
The three device arms run alternately, one image each, `--repeats` times. Prints one JSON line with the GPU and its
power limit, images/s of every arm, the share of each device-finish arm's time spent outside the network calls
(1 - network_only / arm: crop extraction and the finish), and the largest score difference between the native and the
ATen finish. Not part of bench.py's contract (that one measures the training step).
"""
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

from semseg_b200 import inference  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402

PRESETS = {
    # BASELINE config 5: PSPNet101, 713 crop, 19 classes, a 1024x2048 image, base 2048 (the defaults below)
    "config5": dict(layers=101, classes=19, crop=713, height=1024, width=2048, base_size=2048),
    # ADE20K (configs 2 / 3): PSPNet50, 473 crop, 150 classes, a 512x683 image, base 512
    "ade20k": dict(layers=50, classes=150, crop=473, height=512, width=683, base_size=512),
}


class _Foreign(torch.nn.Module):
    """The network behind a module the engine does not recognise: the engine finishes with ATen ops."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x)


class _NetworkOnly(inference.SlidingWindowPredictor):
    """The per-scale image resize and the network calls (logits up to the classifier, same batches) of every scale, no
    crop extraction and no finish. Construct with _Foreign(model)."""

    def scale_on_device(self, image, out_h, out_w):
        ch, cw = self.crop_h, self.crop_w
        img_h, img_w = image.shape[:2]
        full_h, full_w = max(img_h, ch), max(img_w, cw)
        n = len(inference.crop_origins(full_h, ch, self.stride_rate)) * len(inference.crop_origins(full_w, cw,
                                                                                               self.stride_rate))
        per_call = self.max_batch // 2 if self.flip else self.max_batch
        x = torch.zeros((min(n, per_call), 3, ch, cw), device=self.device)
        with torch.no_grad():
            for g0 in range(0, n, per_call):
                part = x[:min(per_call, n - g0)]
                self.model.net._eval_logits_nhwc(torch.cat([part, part.flip(3)], 0) if self.flip else part)
                self.forward_calls += 1
        return 0.0


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit"] = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = "unknown"
    return info


def main():
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--preset", choices=sorted(PRESETS))
    ap = argparse.ArgumentParser(parents=[pre])
    ap.add_argument("--layers", type=int, default=101)
    ap.add_argument("--classes", type=int, default=19)
    ap.add_argument("--crop", type=int, default=713)
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--base-size", type=int, default=2048)
    ap.add_argument("--scales", type=float, nargs="+", default=[0.5, 0.75, 1.0, 1.25, 1.5, 1.75])
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=1)
    preset = pre.parse_known_args()[0].preset
    if preset:
        ap.set_defaults(**PRESETS[preset])
    args = ap.parse_args()
    torch.manual_seed(0)
    model = PSPNet(layers=args.layers, classes=args.classes, zoom_factor=8, pretrained=False).cuda().eval()
    rng = np.random.default_rng(0)
    image = (rng.random((args.height, args.width, 3)) * 255).astype(np.float32)
    mean = [0.485 * 255, 0.456 * 255, 0.406 * 255]
    std = [0.229 * 255, 0.224 * 255, 0.225 * 255]
    out = {"workload": "PSPNet%d eval, %d classes, %dx%d image, base %d, crop %d, scales %s, flip" % (
        args.layers, args.classes, args.height, args.width, args.base_size, args.crop, args.scales), "preset": preset}
    out.update(_gpu_info())
    results = {}

    def engine(name, mb):
        cls = _NetworkOnly if name == "network_only" else inference.SlidingWindowPredictor
        net = _Foreign(model) if name in ("aten_finish_batched", "network_only") else model
        eng = cls(net, args.classes, args.crop, args.crop, mean, std, max_batch=mb)
        exact = name.startswith("reference")
        eng(image, args.base_size, args.scales[:1] if exact else args.scales, exact=exact, return_scores=False)  # warm-up
        torch.cuda.synchronize()
        eng.forward_calls = 0
        return eng

    def timed(name, eng):
        t0 = time.perf_counter()
        _, amax = eng(image, args.base_size, args.scales, exact=name.startswith("reference"), return_scores=False)
        torch.cuda.synchronize()
        results[name] = amax
        return time.perf_counter() - t0

    def report(name, eng, times, mb):
        dt = sum(times) / len(times)
        out[name] = {"seconds_per_image": dt, "images_per_sec": 1.0 / dt, "seconds_per_image_min": min(times),
                     "model_calls_per_image": eng.forward_calls // len(times), "max_batch": mb}

    # the device arms alternate, one image each, so drift on a shared host hits them alike
    arms = {n: engine(n, args.max_batch) for n in ("device_finish_batched", "aten_finish_batched", "network_only")}
    times = {n: [] for n in arms}
    for _ in range(args.repeats):
        for n, eng in arms.items():
            times[n].append(timed(n, eng))
    for n, eng in arms.items():
        report(n, eng, times[n], args.max_batch)
    net_dt = out["network_only"]["seconds_per_image"]
    for n in ("device_finish_batched", "aten_finish_batched"):
        out[n]["share_outside_network_calls"] = 1.0 - net_dt / out[n]["seconds_per_image"]
    native_scores, native_amax = arms["device_finish_batched"](image, args.base_size, args.scales)
    aten_scores, aten_amax = arms["aten_finish_batched"](image, args.base_size, args.scales)
    out["max_abs_score_diff_native_vs_aten"] = float(np.abs(native_scores - aten_scores).max())
    out["argmax_mismatch_native_vs_aten"] = float((native_amax != aten_amax).mean())
    out["speedup_native_vs_aten_finish"] = (out["aten_finish_batched"]["seconds_per_image"] /
                                            out["device_finish_batched"]["seconds_per_image"])
    del native_scores, aten_scores
    for name, mb in (("reference_finish_batched", args.max_batch),    # batched network calls, host cv2 / numpy finish
                     ("reference_procedure_serial", 2)):               # one crop (+ mirror) per call, host finish
        eng = engine(name, mb)
        report(name, eng, [timed(name, eng)], mb)
    ref = results["reference_procedure_serial"]
    out["argmax_identical_reference_finish"] = bool(np.array_equal(results["reference_finish_batched"], ref))
    out["argmax_mismatch_device_finish"] = float((results["device_finish_batched"] != ref).mean())
    out["speedup_vs_reference_procedure"] = (out["reference_procedure_serial"]["seconds_per_image"] /
                                             out["device_finish_batched"]["seconds_per_image"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
