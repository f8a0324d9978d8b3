"""Accuracy evidence for boundary label relaxation (losses.BoundaryRelaxationLoss) without a dataset, on the procedural
segmentation task of tools/fp8_accuracy.py (textured random shapes of K classes on a textured background).

The training labels have noisy boundaries, the way hand-drawn polygons do: each label map is resampled (nearest) through
a smooth random displacement field of up to `--jitter` pixels, so a band around every object boundary carries the
neighbouring class. The images and the evaluation labels are clean. Three arms train a PSPNet50 from the same seed on
the same batches for the same number of steps:
  * ce       : nn.CrossEntropyLoss(ignore_index=255);
  * relax_b1 : BoundaryRelaxationLoss(border=1);
  * relax_b2 : BoundaryRelaxationLoss(border=2).
Each is scored on held-out images through SlidingWindowPredictor: mIoU and the Boundary IoU (metrics.boundaryIoUGPU,
dilation ratio 0.02). Prints one JSON line with the GPU and its power limit."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from semseg_b200.inference import SlidingWindowPredictor  # noqa: E402
from semseg_b200.losses import BoundaryRelaxationLoss  # noqa: E402
from semseg_b200.metrics import boundaryIoUGPU, intersectionAndUnionGPU  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402
from tools.fp8_accuracy import MEAN, STD, _gpu_info, make_batch, normalise  # noqa: E402


def jitter_labels(lab, amplitude, gen):
    """lab [n, H, W] int64 resampled through a smooth random displacement of at most `amplitude` pixels."""
    n, h, w = lab.shape
    coarse = (torch.rand((n, 2, max(h // 16, 2), max(w // 16, 2)), device=lab.device, generator=gen) * 2 - 1)
    disp = F.interpolate(coarse, size=(h, w), mode="bicubic", align_corners=True).clamp_(-1, 1) * amplitude
    yy, xx = torch.meshgrid(torch.arange(h, device=lab.device, dtype=torch.float32),
                            torch.arange(w, device=lab.device, dtype=torch.float32), indexing="ij")
    gx = (xx + disp[:, 0]) / (w - 1) * 2 - 1
    gy = (yy + disp[:, 1]) / (h - 1) * 2 - 1
    out = F.grid_sample(lab[:, None].float(), torch.stack([gx, gy], -1), mode="nearest", padding_mode="border",
                        align_corners=True)
    return out[:, 0].round().long()


def train(model, steps, lr, batch, crop, classes, gen, jitter):
    opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)
    model.train()
    losses, noisy = [], []
    for step in range(steps):
        for grp in opt.param_groups:
            grp["lr"] = lr * (1 - step / steps) ** 0.9
        img, lab = make_batch(batch, crop, classes, gen)
        noisy_lab = jitter_labels(lab, jitter, gen)
        noisy.append(float((noisy_lab != lab).float().mean()))
        _, main_loss, aux_loss = model(normalise(img), noisy_lab)
        loss = main_loss + 0.4 * aux_loss
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        if step % 100 == 0 or step == steps - 1:
            losses.append(round(float(main_loss.detach()), 4))
    torch.cuda.synchronize()
    return losses, float(np.mean(noisy))


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--classes", type=int, default=6)
    ap.add_argument("--steps", type=int, default=600)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--crop", type=int, default=129)
    ap.add_argument("--lr", type=float, default=0.01)
    ap.add_argument("--jitter", type=float, default=3.0, help="largest label displacement in pixels")
    ap.add_argument("--test-images", type=int, default=24)
    ap.add_argument("--test-size", type=int, default=257)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("relax_accuracy needs a CUDA device")
    K = args.classes
    out = _gpu_info()
    out.update(classes=K, steps=args.steps, jitter_px=args.jitter)
    test_gen = torch.Generator(device="cuda").manual_seed(99)                  # held out: another seed
    timg, tlab = make_batch(args.test_images, args.test_size, K, test_gen)
    timg = timg.permute(0, 2, 3, 1).cpu().numpy()
    arms = {"ce": lambda: nn.CrossEntropyLoss(ignore_index=255),
            "relax_b1": lambda: BoundaryRelaxationLoss(border=1),
            "relax_b2": lambda: BoundaryRelaxationLoss(border=2)}
    for arm, crit in arms.items():
        t0 = time.perf_counter()
        torch.manual_seed(0)
        model = PSPNet(layers=50, classes=K, zoom_factor=8, pretrained=False).cuda()
        model.criterion = crit()
        gen = torch.Generator(device="cuda").manual_seed(0)                    # the same batches for every arm
        out["%s_main_loss_every_100_steps" % arm], out["noisy_label_share"] = train(
            model, args.steps, args.lr, args.batch, args.crop, K, gen, args.jitter)
        out["%s_train_s" % arm] = round(time.perf_counter() - t0, 1)
        model.eval()
        pred = SlidingWindowPredictor(model, K, args.crop, args.crop, MEAN, STD)
        preds = torch.from_numpy(np.stack([pred(timg[i], args.test_size, [1.0])[1]
                                           for i in range(args.test_images)])).long().cuda()
        inter, union, _ = intersectionAndUnionGPU(preds.clone(), tlab, K)
        b_inter, b_union, _ = boundaryIoUGPU(preds, tlab, K)
        out["miou_" + arm] = round(100 * float((inter / union.clamp(min=1)).mean()), 2)
        out["boundary_iou_" + arm] = round(100 * float((b_inter / b_union.clamp(min=1)).mean()), 2)
        del model, pred
        torch.cuda.empty_cache()
    out["noisy_label_share"] = round(out["noisy_label_share"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
