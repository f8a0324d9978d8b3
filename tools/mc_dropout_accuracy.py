"""Accuracy evidence for Monte Carlo dropout (SlidingWindowPredictor(mc_draws=T)) without a dataset: train PSPNet50
with Dropout2d p = 0.1 (`--dropout` for another rate) on the seeded procedural task of tools/fp8_accuracy.py, then score
held-out images with the deterministic predictor and with MC dropout (T = `--draws`, default 20), and report for each:
mIoU, NLL of the ground truth under the predicted scores, 15-bin ECE of the max score (computed on the host here), and
the misclassification AUROC (label = prediction != ground truth; the task has no void pixels) through AnomalyMeter,
scored by 1 - MSP for both, and by H[p_bar] and the mutual information for MC. Prints one JSON line with the GPU and
its power limit. There is no gate: last-layer MC dropout at a small rate may change little."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from semseg_b200.anomaly import AnomalyMeter  # noqa: E402
from semseg_b200.inference import SlidingWindowPredictor  # noqa: E402
from semseg_b200.pspnet import PSPNet  # noqa: E402
from tools.fp8_accuracy import MEAN, STD, _gpu_info, make_batch, miou, normalise  # noqa: E402


def ece(conf, correct, bins=15):
    """Expected calibration error over `bins` equal-width confidence bins (fp64 on the host)."""
    edges = np.linspace(0.0, 1.0, bins + 1)
    idx = np.clip(np.digitize(conf, edges[1:-1], right=True), 0, bins - 1)
    count = np.bincount(idx, minlength=bins).astype(np.float64)
    s_conf = np.bincount(idx, weights=conf, minlength=bins)
    s_acc = np.bincount(idx, weights=correct.astype(np.float64), minlength=bins)
    keep = count > 0
    return float(np.sum(np.abs(s_acc[keep] - s_conf[keep])) / conf.size)


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--classes", type=int, default=6)
    ap.add_argument("--dropout", type=float, default=0.1)
    ap.add_argument("--draws", type=int, default=20)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--crop", type=int, default=129)
    ap.add_argument("--test-images", type=int, default=24)
    ap.add_argument("--test-size", type=int, default=257)
    ap.add_argument("--lr", type=float, default=0.01)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mc_dropout_accuracy needs a CUDA device")
    out = _gpu_info()
    out.update(dropout=args.dropout, draws=args.draws, steps=args.steps, classes=args.classes)
    torch.manual_seed(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    model = PSPNet(layers=50, classes=args.classes, zoom_factor=8, dropout=args.dropout, pretrained=False).cuda()
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
        if step % 500 == 0 or step == args.steps - 1:
            losses.append(round(float(main_loss.detach()), 4))
    torch.cuda.synchronize()
    out["train_s"] = round(time.perf_counter() - t0, 1)
    out["train_main_loss"] = losses
    model.eval()
    test_gen = torch.Generator(device="cuda").manual_seed(99)                  # held out: another seed
    timg, tlab = make_batch(args.test_images, args.test_size, args.classes, test_gen)
    timg = timg.permute(0, 2, 3, 1).cpu().numpy()
    tlab = tlab.cpu().numpy()
    torch.manual_seed(1)
    for arm, draws in (("det", 0), ("mc", args.draws)):
        pred = SlidingWindowPredictor(model, args.classes, args.crop, args.crop, MEAN, STD, mc_draws=draws)
        meters = {k: AnomalyMeter() for k in (("msp", "entropy", "mi") if draws else ("msp",))}
        preds, confs, nll = [], [], []
        t0 = time.perf_counter()
        for i in range(args.test_images):
            res = pred(timg[i], args.test_size, [1.0])
            scores, p = res[0], res[1]
            y = tlab[i]
            preds.append(p)
            conf = scores.max(2)
            confs.append(conf.ravel())
            py = np.take_along_axis(scores, y[..., None], 2)[..., 0]
            nll.append(-np.log(np.maximum(py, 1e-12)).ravel())
            wrong = torch.from_numpy((p != y).astype(np.uint8)).cuda()
            meters["msp"].update(torch.from_numpy(1.0 - conf).cuda(), wrong)
            if draws:
                meters["entropy"].update(res[2][0], wrong)
                meters["mi"].update(res[2][1], wrong)
        out[arm + "_s"] = round(time.perf_counter() - t0, 1)
        preds = np.stack(preds)
        correct = (preds == tlab).ravel()
        out[arm + "_miou"] = round(100 * miou(preds, tlab, args.classes), 3)
        out[arm + "_nll"] = round(float(np.concatenate(nll).mean()), 5)
        out[arm + "_ece15"] = round(ece(np.concatenate(confs), correct), 5)
        out[arm + "_pixel_error"] = round(float(1.0 - correct.mean()), 5)
        for k, m in meters.items():
            out["%s_misclass_auroc_%s" % (arm, k)] = round(float(m.compute()["auroc"]), 5)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
