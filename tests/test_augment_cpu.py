"""CPU tier of the GPU batch augmentation (semseg_b200/augment.py, csrc/augment.cu): the host-side draws and geometry
against the reference chain and cv2, the cv2 oracle against the goldens of the real util/transform.py, argument
validation in Python and in the C entry point, the descriptor layout, and the collated batch object."""
import ctypes
import hashlib
import math
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from semseg_b200 import _lib
from semseg_b200.augment import (AugBatch, AugParams, ToUint8, TrainAugment, ValAugment, collate, resized_size,
                                 rotation_inverse)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "augment.npz")
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def golden_cases():
    """[(img, lab, TrainAugment, AugParams, out_img, out_lab, seed, state digest)] from tests/golden/augment.npz."""
    g = np.load(GOLDEN)
    out, k = [], 0
    while "case%d_cfg" % k in g:
        seed, ch, cw, s0, s1, a0, a1, r0, r1 = g["case%d_cfg" % k].tolist()
        ar = None if math.isnan(a0) else [a0, a1]
        aug = TrainAugment([int(ch), int(cw)], [s0, s1], [r0, r1], MEAN, STD, 255, aspect_ratio=ar)
        fx, fy, ang, blur, flip, ho, wo = g["case%d_params" % k].tolist()
        p = AugParams(fx, fy, None if math.isnan(ang) else ang, bool(blur), bool(flip), int(ho), int(wo))
        out.append((g["case%d_img_in" % k], g["case%d_lab_in" % k], aug, p, g["case%d_img" % k],
                    g["case%d_lab" % k].astype(np.int64), int(seed), str(g["case%d_state" % k])))
        k += 1
    return out


def test_goldens_cover_every_stage():
    cases = golden_cases()
    assert len(cases) == 12
    stages = {(p.angle is not None, p.blur, p.flip) for _, _, _, p, *_ in cases}
    assert len(stages) >= 6 and all(any(s[i] for s in stages) and any(not s[i] for s in stages) for i in range(3))
    shortcut = [resized_size(*img.shape[:2], p.fx, p.fy) == img.shape[:2] for img, _, _, p, *_ in cases]
    assert any(shortcut)
    assert any(p.fx != p.fy for _, _, _, p, *_ in cases)
    assert max(p.angle for _, _, _, p, *_ in cases if p.angle is not None) > 9.99
    assert min(p.angle for _, _, _, p, *_ in cases if p.angle is not None) < -9.99


def test_draw_params_consume_random_as_the_reference_chain():
    """Same parameters as the reference chain drew, and the same generator state afterwards (digest of getstate())."""
    for img, _, aug, p, _, _, seed, state in golden_cases():
        rng = random.Random(seed)
        got = aug.draw_params([img.shape[:2]], rng)[0]
        assert got == p
        assert hashlib.sha256(repr(rng.getstate()).encode()).hexdigest() == state
        # the module-level generator is the default
        random.seed(seed)
        assert aug.draw_params([img.shape[:2]])[0] == p
        assert hashlib.sha256(repr(random.getstate()).encode()).hexdigest() == state


def test_oracle_reproduces_goldens_bit_for_bit():
    pytest.importorskip("cv2")
    from tests.augment_oracle import augment_one
    for img, lab, aug, p, oi, ol, *_ in golden_cases():
        ti, tl = augment_one(img, lab, p, aug.crop_h, aug.crop_w, MEAN, STD, 255)
        assert np.array_equal(ti.numpy(), oi)
        assert np.array_equal(tl.numpy(), ol)


def test_resized_size_and_inverse_matrix_equal_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = random.Random(3)
    cases = [(5, 3, 0.5, 0.5), (7, 9, 0.5, 0.5), (37, 53, 1.004, 1.004), (10, 10, 0.25, 0.35), (6, 2, 0.75, 1.25)]
    cases += [(rng.randint(1, 300), rng.randint(1, 300), rng.uniform(0.3, 2.2), rng.uniform(0.3, 2.2)) for _ in range(300)]
    for h, w, fx, fy in cases:
        try:
            want = cv2.resize(np.zeros((h, w), np.uint8), None, fx=fx, fy=fy).shape
        except cv2.error:
            with pytest.raises(ValueError):
                resized_size(h, w, fx, fy)
            continue
        assert resized_size(h, w, fx, fy) == want, (h, w, fx, fy)
    for _ in range(200):
        h, w, ang = rng.randint(1, 2000), rng.randint(1, 2000), rng.uniform(-10, 10)
        ref = cv2.invertAffineTransform(cv2.getRotationMatrix2D((w / 2, h / 2), ang, 1)).reshape(-1)
        assert rotation_inverse(h, w, ang) == ref.tolist()


def _label_map(h, w, angle):
    """The kernel's fixed-point INTER_NEAREST warp (csrc/augment.cu warp_fixed, round_delta 512, >> 10), in numpy:
    flat source index per destination pixel, -1 outside."""
    m = rotation_inverse(h, w, angle)
    x = np.arange(w, dtype=np.float64)
    y = np.arange(h, dtype=np.float64)
    adelta = np.rint(m[0] * x * 1024).astype(np.int64)
    bdelta = np.rint(m[3] * x * 1024).astype(np.int64)
    x0 = np.rint((m[1] * y + m[2]) * 1024).astype(np.int64) + 512
    y0 = np.rint((m[4] * y + m[5]) * 1024).astype(np.int64) + 512
    X = (x0[:, None] + adelta[None, :]) >> 10
    Y = (y0[:, None] + bdelta[None, :]) >> 10
    ok = (X >= 0) & (X < w) & (Y >= 0) & (Y < h)
    return np.where(ok, Y * w + X, -1)


def test_fixed_point_label_map_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = random.Random(5)
    for h, w, ang in [(41, 65, 10.0), (65, 41, -10.0), (473, 473, 3.3)] + \
            [(rng.randint(2, 300), rng.randint(2, 300), rng.uniform(-10, 10)) for _ in range(40)]:
        idx = np.arange(h * w, dtype=np.float32).reshape(h, w)
        mat = cv2.getRotationMatrix2D((w / 2, h / 2), ang, 1)
        ref = cv2.warpAffine(idx, mat, (w, h), flags=cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT, borderValue=-1)
        assert np.array_equal(_label_map(h, w, ang), ref.astype(np.int64)), (h, w, ang)


def test_nearest_resize_rule_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = random.Random(6)
    for _ in range(60):
        h, w, f = rng.randint(2, 200), rng.randint(2, 200), rng.uniform(0.3, 2.2)
        rh, rw = resized_size(h, w, f, f)
        idx = np.arange(h * w, dtype=np.float32).reshape(h, w)
        ref = cv2.resize(idx, None, fx=f, fy=f, interpolation=cv2.INTER_NEAREST).astype(np.int64)
        ys = np.minimum(np.floor(np.arange(rh) * (1.0 / f)).astype(np.int64), h - 1)
        xs = np.minimum(np.floor(np.arange(rw) * (1.0 / f)).astype(np.int64), w - 1)
        if (rh, rw) == (h, w):
            ys, xs = np.arange(h), np.arange(w)
        assert np.array_equal(ys[:, None] * w + xs[None, :], ref), (h, w, f)


def test_constructor_validation_mirrors_the_reference():
    ok = dict(crop=[65, 65], scale=[0.5, 2.0], rotate=[-10, 10], mean=MEAN, std=STD)
    TrainAugment(**ok)
    for bad in (dict(scale=[2.0, 0.5]), dict(scale=[0, 1]), dict(rotate=[10, -10]), dict(crop=[0, 65]),
                dict(crop=[65.0, 65]), dict(mean=[1, 2])):
        with pytest.raises(RuntimeError):
            TrainAugment(**{**ok, **bad})
    with pytest.raises(RuntimeError):
        TrainAugment(**ok, aspect_ratio=[2, 1])
    with pytest.raises(RuntimeError):
        TrainAugment(**ok, ignore_label=255.0)
    with pytest.raises(ValueError):
        TrainAugment(**{**ok, "scale": [0.5]})
    with pytest.raises(ValueError):
        TrainAugment(**{**ok, "std": [1, 0, 1]})
    ValAugment(65, MEAN, STD)


def test_input_validation():
    img, lab = np.zeros((8, 9, 3), np.uint8), np.zeros((8, 9), np.uint8)
    collate([(img, lab)])
    for bad in ((img.astype(np.float32), lab), (img, lab.astype(np.int64)), (img[..., :2], lab), (img, lab[:4]),
                (img[..., 0], lab)):
        with pytest.raises(ValueError):
            collate([bad])
    with pytest.raises(ValueError):
        collate([])
    with pytest.raises(ValueError):           # the reference crashes inside cv2 on an empty scaled image
        TrainAugment(4, [0.01, 0.02], [-10, 10], MEAN, STD).draw_params([(8, 9)], random.Random(0))
    t = ToUint8()
    i8, l8 = t(np.float32(np.arange(24).reshape(2, 4, 3)), np.ones((2, 4), np.uint8))
    assert i8.dtype == np.uint8 and l8.dtype == np.uint8 and i8.ravel().tolist() == list(range(24))
    with pytest.raises(ValueError):
        t(np.full((2, 4, 3), 0.5, np.float32), np.ones((2, 4), np.uint8))
    with pytest.raises(ValueError):
        t(np.zeros((2, 4), np.float32), np.ones((2, 4), np.uint8))


def test_val_params_are_centred():
    v = ValAugment([5, 7], MEAN, STD)
    assert v.draw_params([(9, 4), (3, 12)]) == [AugParams(1.0, 1.0, None, False, False, 2, 0),
                                                 AugParams(1.0, 1.0, None, False, False, 0, 2)]


def test_collate_and_pin_memory(monkeypatch):
    rng = np.random.default_rng(0)
    samples = [(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), rng.integers(0, 256, (h, w), dtype=np.uint8))
               for h, w in ((5, 7), (3, 2), (11, 4))]
    b = collate(samples)
    assert isinstance(b, AugBatch) and len(b) == 3 and b.sizes() == [(5, 7), (3, 2), (11, 4)]
    assert b.data.dtype == torch.uint8 and b.data.dim() == 1 and b.data.numel() == sum(4 * h * w for h, w in b.sizes())
    for (img, lab), (h, w, io, lo) in zip(samples, b.header.tolist()):
        assert np.array_equal(b.data[io:io + 3 * h * w].numpy().reshape(h, w, 3), img)
        assert np.array_equal(b.data[lo:lo + h * w].numpy().reshape(h, w), lab)
    pinned = []
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: pinned.append(self) or self.clone())
    p = b.pin_memory()
    assert isinstance(p, AugBatch) and pinned == [b.data] and p.header is b.header
    assert torch.equal(p.data, b.data)
    # what DataLoader(pin_memory=True) does with a batch it does not know
    from torch.utils.data._utils.pin_memory import pin_memory
    assert isinstance(pin_memory(b), AugBatch) and len(pinned) == 2


def test_descriptor_layout_matches_header():
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "semseg_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(semseg_augment_desc), offsetof(semseg_augment_desc, h),
         offsetof(semseg_augment_desc, scale_y), offsetof(semseg_augment_desc, m), offsetof(semseg_augment_desc, rotate),
         offsetof(semseg_augment_desc, pad_top), offsetof(semseg_augment_desc, off_x),
         offsetof(semseg_augment_desc, reserved));
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        v = list(map(int, subprocess.check_output([exe]).split()))
    D = _lib.AugmentDesc
    assert v == [ctypes.sizeof(D), D.h.offset, D.scale_y.offset, D.m.offset, D.rotate.offset, D.pad_top.offset,
                 D.off_x.offset, D.reserved.offset]


def test_entry_point_validates_before_any_cuda_call():
    lib = _lib.load()
    P = ctypes.c_void_p(16)
    m3, s3 = (ctypes.c_float * 3)(*MEAN), (ctypes.c_float * 3)(*STD)

    def desc(**kw):
        d = _lib.AugmentDesc()
        d.img_off, d.lab_off, d.h, d.w, d.rh, d.rw = 0, 300, 10, 10, 10, 10
        d.pad_top = d.pad_left = 0
        for k, v in kw.items():
            setattr(d, k, v)
        return (_lib.AugmentDesc * 1)(d)

    def call(d, n=1, ch=8, cw=8, nbytes=400, std=s3, data=P):
        return lib.semseg_augment(data, nbytes, d, P, n, ch, cw, m3, std, 255, P, P, None)

    err = lambda: lib.semseg_last_error()      # noqa: E731
    assert call(desc(), data=None) == -1 and b"null pointer" in err()
    assert call(desc(), n=0) == -1 and b"batch" in err()
    assert call(desc(), ch=0) == -1 and b"crop" in err()
    assert call(desc(), nbytes=0) == -1 and b"empty data" in err()
    assert call(desc(), std=(ctypes.c_float * 3)(1, 0, 1)) == -1 and b"std[1]" in err()
    assert call(desc(rh=0)) == -1 and b"size" in err()
    assert call(desc(), nbytes=399) == -1 and b"label" in err()
    assert call(desc(img_off=101)) == -1 and b"image" in err()
    assert call(desc(lab_off=-1)) == -1 and b"label" in err()
    assert call(desc(rh=12, scale_y=0.0, scale_x=1.0)) == -1 and b"resize step" in err()
    assert call(desc(blur=2)) == -1 and b"flags" in err()
    assert call(desc(), ch=14) == -1 and b"padding" in err()          # pad_top must be (14 - 10) / 2
    assert call(desc(off_y=3)) == -1 and b"crop offset" in err()        # padded 10, crop 8: offsets 0..2
    assert call(desc(off_x=-1)) == -1 and b"crop offset" in err()
