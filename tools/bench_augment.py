"""Time the GPU batch augmentation (semseg_b200/augment.py) and the loader-fed training loop it is for.

1. Kernel time per batch (CUDA events, warmed up) at the ADE20K shape (16 images 512x683 -> 473^2) and the Cityscapes
   shape (8 images 1024x2048 -> 713^2), with the achieved bytes/s from the byte count below.
2. The training loop fed by a DataLoader (2 and 8 workers, pin_memory=True) over seeded synthetic JPEG / PNG pairs
   encoded in memory at start-up (smooth images, 512x683), driving bench.py's graphed PSPNet50 step (150 classes,
   bf16) at 16 and at 2 images per step through either
     cpu: the reference chain in the workers (cv2 on float32, tests/augment_oracle.py with the reference's draws), or
     gpu: ToUint8 in the workers, `collate`, and TrainAugment in the main process.
   The two arms alternate over two rounds. img/s counts images the step consumed.
The card's name and power limit and the host CPU model and count are read in the same process.

    python tools/bench_augment.py [--steps 12] [--warmup 4] [--rounds 2]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from semseg_b200 import ops  # noqa: E402
from semseg_b200.augment import ToUint8, TrainAugment, collate  # noqa: E402
from tests.augment_oracle import augment_one  # noqa: E402

MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def platform():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    cpu = "?"
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                cpu = line.split(":", 1)[1].strip()
                break
    except OSError:
        pass
    return {"gpu": q[0] if q else "?", "cpu": cpu, "cpu_count": os.cpu_count(),
            "cpus_usable": len(os.sched_getaffinity(0))}


def smooth_pair(rng, h, w, classes=150):
    lo = rng.integers(0, 256, (h // 32 + 2, w // 32 + 2, 3)).astype(np.uint8)
    img = cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC)
    img = np.clip(img.astype(np.int16) + rng.integers(-3, 4, img.shape), 0, 255).astype(np.uint8)
    lab = rng.integers(0, classes, (h // 16 + 1, w // 16 + 1)).repeat(16, 0).repeat(16, 1)[:h, :w].astype(np.uint8)
    return img, lab


# ------------------------------------------------------------------------------------------------ 1. kernel time
def kernel_time(n, h, w, crop, iters=50):
    rng = np.random.default_rng(0)
    samples = [smooth_pair(rng, h, w) for _ in range(n)]
    aug = TrainAugment(crop, [0.5, 2.0], [-10, 10], MEAN, STD, 255)
    batch = collate(samples)
    params = aug.draw_params(batch.sizes(), random.Random(0))
    # every stage on, as the slowest draw
    params = [p._replace(angle=p.angle if p.angle is not None else 5.0, blur=True) for p in params]
    descs = aug.descriptors(batch, params)
    table = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    data = batch.data.cuda()
    for _ in range(5):
        ops.augment(data, descs, table, crop, crop, MEAN, STD, 255)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.augment(data, descs, table, crop, crop, MEAN, STD, 255)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    written = n * crop * crop * (3 * 4 + 8)
    read = n * h * w * 4                                         # upper bound: every source byte once
    return {"shape": "%dx%dx%d -> %d^2" % (n, h, w, crop), "kernel_ms": round(ms, 4),
            "written_MB": round(written / 1e6, 2), "read_MB_max": round(read / 1e6, 2),
            "GB_per_s": round((written + read) / ms / 1e6, 1)}


# ------------------------------------------------------------------------------------------------ 2. loader-fed loop
class EncodedData(torch.utils.data.Dataset):
    """SemData's decode (cv2.imdecode, BGR -> RGB, np.float32 image, grayscale label) over in-memory JPEG / PNG pairs."""

    def __init__(self, pairs, transform, length):
        self.pairs, self.transform, self.length = pairs, transform, length

    def __len__(self):
        return self.length

    def __getitem__(self, i):
        jpg, png = self.pairs[i % len(self.pairs)]
        image = cv2.imdecode(jpg, cv2.IMREAD_COLOR)
        image = cv2.cvtColor(image, cv2.COLOR_BGR2RGB)
        image = np.float32(image)
        label = cv2.imdecode(png, cv2.IMREAD_GRAYSCALE)
        return self.transform(image, label)


class CpuChain:
    """The reference's train_transform in a worker: draws from the worker's `random`, cv2 chain, ToTensor, Normalize."""

    def __init__(self, crop):
        self.aug = TrainAugment(crop, [0.5, 2.0], [-10, 10], MEAN, STD, 255)

    def __call__(self, image, label):
        p = self.aug.draw_params([label.shape])[0]
        return augment_one(image.astype(np.uint8), label, p, self.aug.crop_h, self.aug.crop_w, MEAN, STD, 255)


def make_model():
    from semseg_b200.pspnet import PSPNet
    torch.manual_seed(0)
    model = PSPNet(layers=50, classes=150, zoom_factor=8, dropout=0.1, pretrained=False,
                   criterion=nn.CrossEntropyLoss(ignore_index=255)).cuda().train()
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    return model, opt


def loop(model, opt, pairs, arm, bs, workers, steps, warmup, crop):
    n_items = bs * (steps + warmup)
    if arm == "cpu":
        ds = EncodedData(pairs, CpuChain(crop), n_items)
        dl = torch.utils.data.DataLoader(ds, batch_size=bs, shuffle=True, num_workers=workers, pin_memory=True,
                                         drop_last=True)
        aug = None
    else:
        ds = EncodedData(pairs, ToUint8(), n_items)
        dl = torch.utils.data.DataLoader(ds, batch_size=bs, shuffle=True, num_workers=workers, pin_memory=True,
                                         drop_last=True, collate_fn=collate)
        aug = TrainAugment(crop, [0.5, 2.0], [-10, 10], MEAN, STD, 255)
    t0 = None
    for i, batch in enumerate(dl):
        if i == warmup:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        if aug is None:
            x, y = batch
            x, y = x.cuda(non_blocking=True), y.cuda(non_blocking=True)
        else:
            x, y = aug(batch)
        _, ml, al = model(x, y)
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
    torch.cuda.synchronize()
    return bs * steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--skip-loop", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = False
    info = platform()
    print(json.dumps({"platform": info}), flush=True)
    for n, h, w, crop in ((16, 512, 683, 473), (8, 1024, 2048, 713)):
        print(json.dumps({"kernel": kernel_time(n, h, w, crop)}), flush=True)
    if args.skip_loop:
        return
    rng = np.random.default_rng(1)
    pairs = []
    for _ in range(args.pairs):
        img, lab = smooth_pair(rng, 512, 683)
        jpg = cv2.imencode(".jpg", cv2.cvtColor(img, cv2.COLOR_RGB2BGR), [cv2.IMWRITE_JPEG_QUALITY, 90])[1]
        png = cv2.imencode(".png", lab)[1]
        pairs.append((jpg, png))
    models = {bs: make_model() for bs in (16, 2)}
    results = {}
    for r in range(args.rounds):
        for bs in (16, 2):
            for workers in (2, 8):
                for arm in ("cpu", "gpu"):
                    ips = loop(*models[bs], pairs, arm, bs, workers, args.steps, args.warmup, 473)
                    results.setdefault("bs%d_w%d_%s" % (bs, workers, arm), []).append(round(ips, 1))
                    print(json.dumps({"round": r, "bs": bs, "workers": workers, "arm": arm, "img_s": round(ips, 1)}),
                          flush=True)
    print(json.dumps({"loop_img_s": results, "platform": info}), flush=True)


if __name__ == "__main__":
    main()
