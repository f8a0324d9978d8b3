"""Accuracy evidence for FP8 inference (semseg_b200/fp8.py) without a dataset: train PSPNet50 from scratch on a seeded
procedural segmentation task (textured random shapes of K classes on a textured background, colour and noise), calibrate
FP8 on 32 training images, and report mIoU through SlidingWindowPredictor for bf16, bf16x3 and FP8 on held-out images.
Prints one JSON line with the GPU and its power limit. The acceptance gate of the FP8 mode is
|mIoU(FP8) - mIoU(bf16)| <= 0.5 points (DESIGN §8)."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from semseg_b200 import precision  # noqa: E402
from semseg_b200.fp8 import Fp8Eval  # noqa: E402
from semseg_b200.inference import SlidingWindowPredictor  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402

MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]


def make_batch(n, size, classes, gen):
    """n images [n, 3, size, size] in 0..255 and labels [n, size, size] (int64): a striped background (class 0) and
    3-6 ellipses / rectangles of random classes, each class with its own colour, stripe direction and frequency."""
    dev = gen.device
    yy, xx = torch.meshgrid(torch.arange(size, device=dev, dtype=torch.float32),
                            torch.arange(size, device=dev, dtype=torch.float32), indexing="ij")
    cg = torch.Generator(device=dev).manual_seed(1234)                       # the class palette is fixed
    colour = torch.rand((classes, 3), device=dev, generator=cg) * 200 + 28
    freq = torch.rand((classes,), device=dev, generator=cg) * 0.5 + 0.15
    angle = torch.rand((classes,), device=dev, generator=cg) * math.pi
    label = torch.zeros((n, size, size), dtype=torch.int64, device=dev)
    for i in range(n):
        for _ in range(int(torch.randint(3, 7, (1,), device=dev, generator=gen))):
            c = int(torch.randint(1, classes, (1,), device=dev, generator=gen))
            cy, cx = (torch.rand(2, device=dev, generator=gen) * size).tolist()
            ry, rx = (torch.rand(2, device=dev, generator=gen) * size * 0.25 + size * 0.08).tolist()
            if bool(torch.rand(1, device=dev, generator=gen) < 0.5):
                m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1
            else:
                m = ((yy - cy).abs() <= ry) & ((xx - cx).abs() <= rx)
            label[i][m] = c
    a = angle[label]
    stripe = torch.sin((xx * torch.cos(a) + yy * torch.sin(a)) * freq[label])
    img = colour[label].permute(0, 3, 1, 2) * (0.75 + 0.25 * stripe[:, None])
    img = img + torch.randn(img.shape, device=dev, generator=gen) * 12
    jitter = (torch.rand((n, 3, 1, 1), device=dev, generator=gen) - 0.5) * 40      # per-image colour shift
    return (img + jitter).clamp(0, 255), label


def normalise(img):
    m = torch.tensor(MEAN, device=img.device)[:, None, None]
    s = torch.tensor(STD, device=img.device)[:, None, None]
    return (img - m) / s


def miou(pred, label, classes):
    hist = np.bincount(label.ravel() * classes + pred.ravel(), minlength=classes * classes).reshape(classes, classes)
    inter = np.diag(hist)
    union = hist.sum(0) + hist.sum(1) - inter
    return float(np.mean(inter[union > 0] / union[union > 0]))


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
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--classes", type=int, default=6)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--crop", type=int, default=129)
    ap.add_argument("--test-images", type=int, default=24)
    ap.add_argument("--test-size", type=int, default=257)
    ap.add_argument("--lr", type=float, default=0.01)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_accuracy needs a CUDA device")
    out = _gpu_info()
    torch.manual_seed(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    model = PSPNet(layers=50, classes=args.classes, zoom_factor=8, pretrained=False).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=args.lr, momentum=0.9, weight_decay=1e-4)
    model.train()
    t0 = time.perf_counter()
    losses = []
    for step in range(args.steps):
        for grp in opt.param_groups:
            grp["lr"] = args.lr * (1 - step / args.steps) ** 0.9
        img, lab = make_batch(args.batch, args.crop, args.classes, gen)
        _, main_loss, aux_loss = model(normalise(img), lab)
        loss = main_loss + 0.4 * aux_loss
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        if step % 100 == 0 or step == args.steps - 1:
            losses.append(round(float(main_loss.detach()), 4))
    torch.cuda.synchronize()
    out["train_s"] = round(time.perf_counter() - t0, 1)
    out["train_main_loss_every_100_steps"] = losses
    model.eval()
    q = Fp8Eval(model)
    cal_img, _ = make_batch(32, args.crop, args.classes, gen)                   # 32 training-distribution images
    for k in range(0, 32, 8):
        q.calibrate(normalise(cal_img[k:k + 8]))
    q.freeze()
    test_gen = torch.Generator(device="cuda").manual_seed(99)                  # held out: another seed
    timg, tlab = make_batch(args.test_images, args.test_size, args.classes, test_gen)
    timg = timg.permute(0, 2, 3, 1).cpu().numpy()
    tlab = tlab.cpu().numpy()
    res = {}
    for arm, net, mode in (("bf16", model, "bf16"), ("bf16x3", model, "bf16x3"), ("fp8", q, "bf16")):
        pred = SlidingWindowPredictor(net, args.classes, args.crop, args.crop, MEAN, STD)
        preds = []
        with precision.mode(mode):
            for i in range(args.test_images):
                _, p = pred(timg[i], args.test_size, [1.0])
                preds.append(p)
        res[arm] = np.stack(preds)
        out["miou_" + arm] = round(100 * miou(res[arm], tlab, args.classes), 3)
    out["miou_fp8_minus_bf16_points"] = round(out["miou_fp8"] - out["miou_bf16"], 3)
    out["pixel_agreement_fp8_vs_bf16"] = round(float((res["fp8"] == res["bf16"]).mean()), 5)
    out["gate_abs_diff_le_0.5_points"] = abs(out["miou_fp8_minus_bf16_points"]) <= 0.5
    out.update(_gpu_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
