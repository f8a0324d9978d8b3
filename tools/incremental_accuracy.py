"""Accuracy evidence for class-incremental training (losses.IncrementalLoss, MiB) without a dataset, on the procedural
segmentation task of tools/fp8_accuracy.py (textured random shapes of K classes on a textured background).

Step 1 trains a PSPNet50 on classes {0..k-1}: the labels of the future classes k..K-1 are background (0) in its data.
Step 2 adds k..K-1 with incremental.expand_classifier; its data labels only the new classes, the old ones are set to 0.
From the same expanded network two arms train step 2 for the same number of steps:
  * mib      : losses.IncrementalLoss(step-1 network) (unbiased cross-entropy + unbiased distillation);
  * finetune : plain nn.CrossEntropyLoss, which learns that old-class pixels are background and forgets.
Each is scored on held-out, fully labelled images through SlidingWindowPredictor: mIoU over the old classes (0..k-1,
the background included, as MiB reports them), the new ones and all. Prints one JSON line with the GPU and its power
limit."""
import argparse
import copy
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from semseg_b200.incremental import expand_classifier  # noqa: E402
from semseg_b200.inference import SlidingWindowPredictor  # noqa: E402
from semseg_b200.losses import IncrementalLoss  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402
from tools.fp8_accuracy import MEAN, STD, _gpu_info, make_batch, normalise  # noqa: E402


def per_class_iou(pred, label, classes):
    hist = np.bincount(label.ravel() * classes + pred.ravel(), minlength=classes * classes).reshape(classes, classes)
    inter = np.diag(hist)
    union = hist.sum(0) + hist.sum(1) - inter
    return np.where(union > 0, inter / np.maximum(union, 1), np.nan)


def train(model, steps, lr, batch, crop, classes, gen, relabel):
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=lr, momentum=0.9, weight_decay=1e-4)
    model.train()
    losses = []
    for step in range(steps):
        for grp in opt.param_groups:
            grp["lr"] = lr * (1 - step / steps) ** 0.9
        img, lab = make_batch(batch, crop, classes, gen)
        _, main_loss, aux_loss = model(normalise(img), relabel(lab))
        loss = main_loss + 0.4 * aux_loss
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        if step % 100 == 0 or step == steps - 1:
            losses.append(round(float(main_loss.detach()), 4))
    torch.cuda.synchronize()
    return losses


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--classes", type=int, default=6, help="K, all classes (the background included)")
    ap.add_argument("--old", type=int, default=4, help="k, the classes of step 1")
    ap.add_argument("--steps1", type=int, default=1000)
    ap.add_argument("--steps2", type=int, default=500)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--crop", type=int, default=129)
    ap.add_argument("--lr1", type=float, default=0.01)
    ap.add_argument("--lr2", type=float, default=0.005)
    ap.add_argument("--kd-weight", type=float, default=10.0)
    ap.add_argument("--test-images", type=int, default=24)
    ap.add_argument("--test-size", type=int, default=257)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("incremental_accuracy needs a CUDA device")
    K, k = args.classes, args.old
    assert 2 <= k < K <= 256
    out = _gpu_info()
    out.update(classes=K, old=k, steps1=args.steps1, steps2=args.steps2, kd_weight=args.kd_weight)
    torch.manual_seed(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    t0 = time.perf_counter()
    step1 = PSPNet(layers=50, classes=k, zoom_factor=8, pretrained=False).cuda()
    out["step1_main_loss_every_100_steps"] = train(step1, args.steps1, args.lr1, args.batch, args.crop, K, gen,
                                                   lambda y: torch.where(y >= k, torch.zeros_like(y), y))
    step1.eval()
    # a network that has run graphed training steps holds its CUDA graphs, which do not deep-copy: the student is a fresh
    # network with the step-1 weights
    expanded = PSPNet(layers=50, classes=k, zoom_factor=8, pretrained=False).cuda()
    expanded.load_state_dict(step1.state_dict())
    expanded = expand_classifier(expanded, K - k)
    new_only = lambda y: torch.where(y < k, torch.zeros_like(y), y)       # noqa: E731
    models = {}
    for arm in ("mib", "finetune"):
        m = copy.deepcopy(expanded)
        m.criterion = IncrementalLoss(step1, kd_weight=args.kd_weight) if arm == "mib" else \
            nn.CrossEntropyLoss(ignore_index=255)
        g2 = torch.Generator(device="cuda").manual_seed(1)                  # the same step-2 batches for both arms
        out["step2_%s_main_loss_every_100_steps" % arm] = train(m, args.steps2, args.lr2, args.batch, args.crop, K,
                                                                 g2, new_only)
        models[arm] = m.eval()
    out["train_s"] = round(time.perf_counter() - t0, 1)
    test_gen = torch.Generator(device="cuda").manual_seed(99)                  # held out: another seed
    timg, tlab = make_batch(args.test_images, args.test_size, K, test_gen)
    timg = timg.permute(0, 2, 3, 1).cpu().numpy()
    tlab = tlab.cpu().numpy()
    for arm, net in [("step1", step1)] + list(models.items()):
        c = k if arm == "step1" else K
        pred = SlidingWindowPredictor(net, c, args.crop, args.crop, MEAN, STD)
        preds = np.stack([pred(timg[i], args.test_size, [1.0])[1] for i in range(args.test_images)])
        iou = per_class_iou(preds, np.where(tlab >= c, 0, tlab) if arm == "step1" else tlab, c)
        out["miou_old_" + arm] = round(100 * float(np.nanmean(iou[:k])), 2)
        if arm != "step1":
            out["miou_new_" + arm] = round(100 * float(np.nanmean(iou[k:])), 2)
            out["miou_all_" + arm] = round(100 * float(np.nanmean(iou)), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
