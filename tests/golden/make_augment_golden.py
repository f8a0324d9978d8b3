"""Generate tests/golden/augment.npz from the REAL reference transforms (util/transform.py of hszhao/semseg).

Run once where the reference tree and cv2 exist (the reference does not exist on the GPU box):
    python tests/golden/make_augment_golden.py
Each case seeds `random`, runs the reference's train_transform chain (RandScale, RandRotate, RandomGaussianBlur,
RandomHorizontalFlip, Crop('rand', padding=mean), ToTensor, Normalize) on a seeded uint8 image / label pair and stores
the inputs, the outputs, the parameters the chain drew and a digest of `random.getstate()` afterwards. Seeds are picked
so that the cases cover every stage on and off, padding on one and on both axes, cv2's copy shortcut, an aspect ratio
and rotations at +-10 degrees.
"""
import collections
import collections.abc
import hashlib
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("SEMSEG_REFERENCE", "/root/reference")

MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]
IGNORE = 255

# (h, w), (crop_h, crop_w), scale, aspect_ratio, rotate, wanted (rotated, blurred, flipped)
CASES = [
    ((60, 80), (49, 49), [0.5, 2.0], None, [-10, 10], (1, 1, 1)),
    ((60, 80), (49, 49), [0.5, 2.0], None, [-10, 10], (0, 0, 0)),
    ((70, 50), (49, 49), [0.5, 2.0], None, [-10, 10], (1, 0, 1)),
    ((50, 70), (49, 49), [0.5, 2.0], None, [-10, 10], (0, 1, 0)),
    ((53, 37), (49, 41), [1.0, 1.008], None, [-10, 10], (1, 1, 0)),      # copy shortcut; padding on the width only
    ((30, 40), (49, 49), [0.5, 0.6], None, [-10, 10], (1, 1, 1)),        # padding on both axes
    ((64, 64), (49, 49), [0.5, 2.0], [0.5, 2.0], [-10, 10], (1, 0, 0)),  # aspect ratio
    ((60, 80), (49, 49), [0.5, 2.0], None, [9.999, 10.0], (1, 1, 1)),    # +10 degrees
    ((60, 80), (49, 49), [0.5, 2.0], None, [-10.0, -9.999], (1, 0, 1)),  # -10 degrees
    ((90, 60), (65, 41), [0.5, 2.0], None, [-10, 10], (0, 1, 1)),        # non-square crops
    ((50, 130), (41, 65), [0.75, 0.8], None, [-10, 10], (1, 1, 0)),      # padding on the height only
    ((30, 40), (49, 49), [1.9, 2.0], None, [-10, 10], (1, 1, 1)),        # upscaling
]


def source(seed, h, w):
    """Smooth seeded RGB image plus a blocky label (values 0..20 and a few 255)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3), np.uint8)
    for c in range(3):
        f = rng.uniform(0.05, 0.3, 2)
        v = 127.5 + 100 * np.sin(f[0] * yy + rng.uniform(0, 6)) * np.cos(f[1] * xx) + rng.normal(0, 12, (h, w))
        img[..., c] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    lab = (rng.integers(0, 21, (h // 8 + 1, w // 8 + 1)).repeat(8, 0).repeat(8, 1)[:h, :w]).astype(np.uint8)
    lab[rng.random((h, w)) < 0.02] = IGNORE
    return img, lab


def main():
    sys.path.insert(0, ROOT)
    if not hasattr(collections, "Iterable"):
        collections.Iterable = collections.abc.Iterable          # util/transform.py:67,79,118,171
    sys.path.insert(0, REF)
    from util import transform
    from semseg_b200.augment import TrainAugment

    out = {"mean": np.array(MEAN, np.float64), "std": np.array(STD, np.float64)}
    for k, ((h, w), crop, scale, ar, rot, want) in enumerate(CASES):
        aug = TrainAugment(list(crop), scale, rot, MEAN, STD, IGNORE, aspect_ratio=ar)
        seed = 1000 * k
        while True:
            p = aug.draw_params([(h, w)], random.Random(seed))[0]
            if (p.angle is not None, p.blur, p.flip) == tuple(map(bool, want)):
                break
            seed += 1
        img, lab = source(seed, h, w)
        chain = transform.Compose([
            transform.RandScale(scale, aspect_ratio=ar),
            transform.RandRotate(rot, padding=MEAN, ignore_label=IGNORE),
            transform.RandomGaussianBlur(),
            transform.RandomHorizontalFlip(),
            transform.Crop(list(crop), crop_type='rand', padding=MEAN, ignore_label=IGNORE),
            transform.ToTensor(),
            transform.Normalize(mean=MEAN, std=STD)])
        random.seed(seed)
        ti, tl = chain(np.float32(img), lab)
        state = hashlib.sha256(repr(random.getstate()).encode()).hexdigest()
        out["case%d_img_in" % k] = img
        out["case%d_lab_in" % k] = lab
        out["case%d_img" % k] = ti.numpy()
        out["case%d_lab" % k] = tl.numpy().astype(np.uint8)
        out["case%d_cfg" % k] = np.array([seed, crop[0], crop[1], scale[0], scale[1],
                                          ar[0] if ar else np.nan, ar[1] if ar else np.nan, rot[0], rot[1]], np.float64)
        out["case%d_params" % k] = np.array([p.fx, p.fy, np.nan if p.angle is None else p.angle, p.blur, p.flip,
                                             p.h_off, p.w_off], np.float64)
        out["case%d_state" % k] = np.array(state)
        print("case %d: seed %d %dx%d -> crop %s, params %s" % (k, seed, h, w, crop, p))
    np.savez_compressed(os.path.join(HERE, "augment.npz"), **out)


if __name__ == "__main__":
    main()
