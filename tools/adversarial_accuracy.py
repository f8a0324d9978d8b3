"""Robustness evidence for the attacks and PGD adversarial training (semseg_b200/adversarial.py, losses.AdversarialLoss)
without a dataset: train PSPNet50 from scratch on fp8_accuracy's seeded procedural segmentation task twice, with plain
cross-entropy and with PGD adversarial training (K = 3 iterations, eps = --at-eps, alpha = 2.5 eps / K), then report on
held-out images the clean mIoU and the mIoU under FGSM, PGD-10 and SegPGD-10 (alpha = eps / 4, random start) at eps 2,
4 and 8 (0-255 pixel units). The attacks run on whole images (no sliding window). Prints one JSON line with the GPU and
its power limit, read in the same process."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from fp8_accuracy import MEAN, STD, _gpu_info, make_batch, miou, normalise  # noqa: E402
from semseg_b200.adversarial import PGDAttack  # noqa: E402
from semseg_b200.losses import AdversarialLoss  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402


def train(args, adversarial):
    torch.manual_seed(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    model = PSPNet(layers=50, classes=args.classes, zoom_factor=8, pretrained=False).cuda()
    if adversarial:
        k = args.at_steps
        model.criterion = AdversarialLoss(PGDAttack(args.at_eps, 2.5 * args.at_eps / k, k, mean=MEAN, std=STD))
    opt = torch.optim.SGD(model.parameters(), lr=args.lr, momentum=0.9, weight_decay=1e-4)
    model.train()
    t0 = time.perf_counter()
    losses = []
    for step in range(args.steps):
        for grp in opt.param_groups:
            grp["lr"] = args.lr * (1 - step / args.steps) ** 0.9
        img, lab = make_batch(args.batch, args.crop, args.classes, gen)
        _, main_loss, aux_loss = model(normalise(img), lab)
        opt.zero_grad(set_to_none=True)
        (main_loss + 0.4 * aux_loss).backward()
        opt.step()
        if step % 100 == 0 or step == args.steps - 1:
            losses.append(round(float(main_loss.detach()), 4))
    torch.cuda.synchronize()
    return model.eval(), round(time.perf_counter() - t0, 1), losses


def evaluate(model, x, y, classes, chunk):
    """mIoU (points) of the model's argmax on the normalised batch x against y, clean and under each attack."""
    attacks = {"clean": None}
    for eps in (2, 4, 8):
        attacks["fgsm_eps%d" % eps] = PGDAttack(eps, eps, 1, random_start=False, mean=MEAN, std=STD)
        attacks["pgd10_eps%d" % eps] = PGDAttack(eps, eps / 4, 10, mean=MEAN, std=STD)
        attacks["segpgd10_eps%d" % eps] = PGDAttack(eps, eps / 4, 10, kind="segpgd", mean=MEAN, std=STD)
    out = {}
    for name, atk in attacks.items():
        torch.manual_seed(5)
        preds = []
        for k in range(0, x.shape[0], chunk):
            xb, yb = x[k:k + chunk], y[k:k + chunk]
            if atk is not None:
                xb = atk(model, xb, yb)
            with torch.no_grad():
                preds.append(model(xb).argmax(1).cpu().numpy())
        out[name] = round(100 * miou(np.concatenate(preds), y.cpu().numpy(), classes), 2)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--classes", type=int, default=6)
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--crop", type=int, default=129)
    ap.add_argument("--test-images", type=int, default=32)
    ap.add_argument("--lr", type=float, default=0.01)
    ap.add_argument("--at-eps", type=float, default=4.0)
    ap.add_argument("--at-steps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adversarial_accuracy needs a CUDA device")
    out = dict(_gpu_info(), classes=args.classes, steps=args.steps, batch=args.batch, crop=args.crop,
               at_eps=args.at_eps, at_steps=args.at_steps)
    test_gen = torch.Generator(device="cuda").manual_seed(99)                  # held out: another seed
    timg, tlab = make_batch(args.test_images, args.crop, args.classes, test_gen)
    x = normalise(timg).contiguous()
    for name, adv in (("clean_training", False), ("pgd_at", True)):
        model, secs, losses = train(args, adv)
        out[name] = dict(train_s=secs, train_main_loss_every_100_steps=losses,
                         miou=evaluate(model, x, tlab, args.classes, 16))
        del model
        torch.cuda.empty_cache()
    out.update(_gpu_info())
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
