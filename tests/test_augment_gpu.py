"""GPU tier of the batch augmentation (semseg_b200/augment.py, csrc/augment.cu): the kernel against the goldens of the
reference's util/transform.py and against cv2 live at ADE20K and Cityscapes sizes, validation mode, determinism,
batch independence, no host synchronisation, and a graphed PSPNet50 training step fed from it."""
import random

import numpy as np
import pytest
import torch

from semseg_b200.augment import AugParams, TrainAugment, ValAugment, collate, resized_size
from tests import util
from tests.test_augment_cpu import MEAN, STD, golden_cases

pytestmark = pytest.mark.gpu

IMG_TOL = 1e-5          # normalised units (~6e-4 of a grey level)

try:
    import cv2  # noqa: F401
    from tests import augment_oracle
except ImportError:     # the golden cases below still run
    augment_oracle = None
needs_cv2 = pytest.mark.skipif(augment_oracle is None, reason="cv2 is not installed: live comparison skipped")


def smooth_pair(rng, h, w, classes=150):
    """Seeded smooth RGB image (a JPEG-like photo, not noise) and a blocky label with some ignore pixels."""
    lo = rng.integers(0, 256, (h // 32 + 2, w // 32 + 2, 3)).astype(np.float32)
    yy = np.linspace(0, lo.shape[0] - 1.001, h)
    xx = np.linspace(0, lo.shape[1] - 1.001, w)
    y0, x0 = yy.astype(int), xx.astype(int)
    fy, fx = (yy - y0)[:, None, None], (xx - x0)[None, :, None]
    img = (lo[y0][:, x0] * (1 - fy) * (1 - fx) + lo[y0 + 1][:, x0] * fy * (1 - fx) + lo[y0][:, x0 + 1] * (1 - fy) * fx
           + lo[y0 + 1][:, x0 + 1] * fy * fx) + rng.normal(0, 4, (h, w, 3))
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    lab = rng.integers(0, classes, (h // 16 + 1, w // 16 + 1)).repeat(16, 0).repeat(16, 1)[:h, :w].astype(np.uint8)
    lab[rng.random((h, w)) < 0.01] = 255
    return img, lab


def check(aug, samples, params):
    gi, gl = aug.apply(samples, params)
    oi, ol = augment_oracle.augment_batch(samples, params, aug.crop_h, aug.crop_w, aug.mean, aug.std, aug.ignore_label)
    gi, gl = gi.cpu(), gl.cpu()
    assert gl.dtype == torch.int64 and gi.dtype == torch.float32
    assert torch.equal(gl, ol), int((gl != ol).sum())
    err = float((gi - oi).abs().max())
    assert err <= IMG_TOL, err
    return err


def test_kernel_reproduces_goldens():
    worst = 0.0
    for img, lab, aug, p, oi, ol, *_ in golden_cases():
        gi, gl = aug.apply([(img, lab)], [p])
        assert np.array_equal(gl[0].cpu().numpy(), ol)
        err = float(np.abs(gi[0].cpu().numpy() - oi).max())
        worst = max(worst, err)
        assert err <= IMG_TOL, err
    print("goldens: max |image error| %.3g" % worst)


@needs_cv2
@pytest.mark.parametrize("rot, blur, flip", [(r, b, f) for r in (0, 1) for b in (0, 1) for f in (0, 1)])
@pytest.mark.parametrize("shape", ["ade", "cityscapes"])
def test_live_cv2_at_dataset_sizes(shape, rot, blur, flip):
    if shape == "ade":
        n, (h, w), crop = 16, (512, 683), 473
    else:
        n, (h, w), crop = 4, (1024, 2048), 713
    rng = np.random.default_rng((shape == "ade") * 8 + rot * 4 + blur * 2 + flip)
    samples = [smooth_pair(rng, h, w) for _ in range(n)]
    aug = TrainAugment(crop, [0.5, 2.0], [-10, 10], MEAN, STD, 255)
    r = random.Random(rot * 4 + blur * 2 + flip)
    params = [p._replace(angle=(p.angle if p.angle is not None else r.uniform(-10, 10)) if rot else None,
                         blur=bool(blur), flip=bool(flip)) for p in aug.draw_params([(h, w)] * n, r)]
    err = check(aug, samples, params)
    print("%s rot %d blur %d flip %d: max |image error| %.3g" % (shape, rot, blur, flip, err))


@needs_cv2
def test_scales_padding_and_crop_shapes():
    rng = np.random.default_rng(7)
    samples = [smooth_pair(rng, 120, 170) for _ in range(4)]
    for crop, f, ang in [((97, 65), 0.5, 7.5), ((97, 65), 2.0, -10.0), ((65, 97), 0.3, 4.0), ((150, 65), 0.45, None),
                         ((60, 85), 0.5, None), ((240, 340), 2.0, 10.0)]:
        aug = TrainAugment(list(crop), [0.1, 3.0], [-10, 10], MEAN, STD, 255)
        rh, rw = resized_size(120, 170, f, f)
        params = []
        for k in range(4):
            ph, pw = max(rh, crop[0]), max(rw, crop[1])
            params.append(AugParams(f, f, ang, k % 2 == 0, k // 2 == 1, (k * 7) % (ph - crop[0] + 1),
                                    (k * 13) % (pw - crop[1] + 1)))
        check(aug, samples, params)


@needs_cv2
def test_validation_mode():
    rng = np.random.default_rng(8)
    samples = [smooth_pair(rng, h, w) for h, w in ((512, 683), (400, 300), (473, 473), (300, 700))]
    v = ValAugment(473, MEAN, STD, 255)
    gi, gl = v(samples)
    for k, (img, lab) in enumerate(samples):
        h, w = lab.shape
        ph, pw = max(h, 473), max(w, 473)
        p = AugParams(1.0, 1.0, None, False, False, int((ph - 473) / 2), int((pw - 473) / 2))
        oi, ol = augment_oracle.augment_one(img, lab, p, 473, 473, MEAN, STD, 255)
        assert torch.equal(gl[k].cpu(), ol)
        assert float((gi[k].cpu() - oi).abs().max()) <= IMG_TOL


def test_deterministic_and_independent_of_the_batch():
    rng = np.random.default_rng(9)
    samples = [smooth_pair(rng, 200 + 17 * k, 260 - 9 * k) for k in range(6)]
    aug = TrainAugment(193, [0.5, 2.0], [-10, 10], MEAN, STD, 255)
    a = aug(samples, random.Random(1))
    b = aug(collate(samples), random.Random(1))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    params = aug.draw_params([s[1].shape for s in samples], random.Random(1))
    for k in (0, 3, 5):
        one = aug.apply([samples[k]], [params[k]])
        assert torch.equal(one[0][0], a[0][k]) and torch.equal(one[1][0], a[1][k])


def test_no_host_synchronisation():
    rng = np.random.default_rng(10)
    batch = collate([smooth_pair(rng, 512, 683) for _ in range(4)]).pin_memory()
    aug = TrainAugment(473, [0.5, 2.0], [-10, 10], MEAN, STD, 255)
    aug(batch, random.Random(0))                   # first call: module load outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for s in range(3):
            x, y = aug(batch, random.Random(s))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert x.shape == (4, 3, 473, 473) and y.shape == (4, 473, 473)


@needs_cv2
def test_graphed_training_step_fed_from_augment():
    """A graphed PSPNet50 step on TrainAugment's tensors equals the step on the cv2 oracle's tensors for the same draws.
    The learning rate is 0, so every step starts from the same weights in both runs: at 65^2 and 2 images, training
    amplifies any input difference (a 1e-6 perturbation moves per-parameter gradients by percents, DESIGN §4), so
    only steps from equal weights are comparable. Even then, a random-init network in training mode at this size turns
    the one-bf16-ulp input flips that a 1e-6 image difference causes into loss changes of up to 0.8 % (measured on an
    H100; steps without such a flip are bit-identical), so the losses are held to 2e-2."""
    import copy
    from semseg_b200 import graphs
    rng = np.random.default_rng(11)
    pool = [smooth_pair(rng, 90, 110, classes=21) for _ in range(6)]
    aug = TrainAugment(65, [0.5, 2.0], [-10, 10], MEAN, STD, 255)
    draws = random.Random(4)
    feeds = []
    for s in range(graphs.WARMUP_CALLS + 3):
        samples = [pool[(2 * s) % 6], pool[(2 * s + 1) % 6]]
        params = aug.draw_params([p[1].shape for p in samples], draws)
        x, y = aug.apply(samples, params)
        ox, oy = augment_oracle.augment_batch(samples, params, 65, 65, MEAN, STD, 255)
        feeds.append(((x, y), (ox.cuda(), oy.cuda())))
    base = util.build_pspnet(50, 21).cuda().train()
    losses = []
    for which in (0, 1):
        model = copy.deepcopy(base)
        opt = torch.optim.SGD(model.parameters(), lr=0.0, momentum=0.9, weight_decay=1e-4)
        out = []
        for f in feeds:
            x, y = f[which]
            _, ml, al = model(x, y)
            opt.zero_grad()
            (ml + 0.4 * al).backward()
            opt.step()
            out.append((ml.item(), al.item()))
        assert graphs.launches_per_step(model) > 100          # the step was captured and replayed
        losses.append(out)
    print("losses (augment, oracle):", losses)
    for (a, b), (c, d) in zip(*losses):
        assert abs(a - c) <= 2e-2 * abs(c) and abs(b - d) <= 2e-2 * abs(d), losses
