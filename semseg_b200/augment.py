"""Training-batch augmentation on the GPU: tool/train.py:194-212's transform chains as one native launch per batch.

The reference augments each sample in a DataLoader worker with cv2 on float32 images (util/transform.py):
RandScale -> RandRotate -> RandomGaussianBlur -> RandomHorizontalFlip -> Crop('rand') -> ToTensor -> Normalize. Here
the workers only decode (`ToUint8` as the dataset's transform) and pack the batch into one uint8 buffer (`collate`);
`TrainAugment` draws the random parameters on the host in the reference's order and runs the whole chain in
`csrc/augment.cu`, producing what the DataLoader handed the trainer: fp32 NCHW images and int64 labels on the current
CUDA device and stream. `ValAugment` is the validation chain (centre Crop, ToTensor, Normalize) on the same kernel.

Semantics are cv2's (checked against cv2 4.13 by tests/test_augment_*.py): resized size round-half-even(W*fx) x
round-half-even(H*fy) with cv2's copy when it equals the source size, INTER_LINEAR / INTER_NEAREST resize, warpAffine
in cv2's 10-bit fixed point about (w/2, h/2) with border mean / ignore_label, 5x5 sigma-0 Gaussian with reflect-101
borders, horizontal flip, padding (mean / ignore_label, half leading) and crop, then (x - mean) / std in fp32.
Random draws happen in the calling process, from `rng` (default: the `random` module): a DataLoader worker's
`random.seed` no longer affects augmentation.

`StrongAugment` is the strong view of mean-teacher training (colour jitter, grayscale, Gaussian blur of an already
normalised batch, csrc/strong.cu), drawn on the device and made inside the student's forward.
"""
import collections.abc
import ctypes
import math
import numbers
import random

import numpy as np
import torch

from . import _lib, ops

__all__ = ["AugParams", "AugBatch", "ToUint8", "collate", "TrainAugment", "ValAugment", "StrongAugment",
           "resized_size", "rotation_inverse"]

AugParams = collections.namedtuple("AugParams", "fx fy angle blur flip h_off w_off")
AugParams.__doc__ = """One sample's draws: resize factors, rotation angle in degrees (None: not rotated), blur and flip
flags, crop offsets in the padded frame."""


def resized_size(h, w, fx, fy):
    """(rh, rw) of cv2.resize(src, None, fx=fx, fy=fy): saturate_cast<int> of the double products, i.e. round half to
    even. Raises ValueError on an empty result, where cv2 itself would fail."""
    rh, rw = round(h * fy), round(w * fx)
    if rh <= 0 or rw <= 0:
        raise ValueError("scaling %dx%d by (fy=%r, fx=%r) gives an empty %dx%d image" % (h, w, fy, fx, rh, rw))
    return rh, rw


def rotation_inverse(h, w, angle):
    """cv2.invertAffineTransform(cv2.getRotationMatrix2D((w / 2, h / 2), angle, 1)) in double, without cv2: the map from
    the rotated image back to its source that cv2.warpAffine applies."""
    a = angle * (math.pi / 180)
    alpha, beta = math.cos(a), math.sin(a)
    cx, cy = w / 2, h / 2
    m = [alpha, beta, (1 - alpha) * cx - beta * cy, -beta, alpha, beta * cx + (1 - alpha) * cy]
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22, a12, a21 = m[4] * d, m[0] * d, -m[1] * d, -m[3] * d
    b1 = -a11 * m[2] - a12 * m[5]
    b2 = -a21 * m[2] - a22 * m[5]
    return [a11, a12, b1, a21, a22, b2]


class ToUint8:
    """Dataset transform (`SemData(..., transform=ToUint8())`): the decoded float32 RGB image back to uint8 (exact: the
    values are decoded integers) and the label as uint8, both as contiguous numpy arrays for `collate`."""

    def __call__(self, image, label):
        image, label = np.asarray(image), np.asarray(label)
        if image.ndim != 3 or image.shape[2] != 3:
            raise ValueError("ToUint8: expected an HxWx3 RGB image, got shape %s" % (image.shape,))
        if label.ndim != 2 or label.shape != image.shape[:2]:
            raise ValueError("ToUint8: label shape %s does not match image %s" % (label.shape, image.shape))
        img8 = image.astype(np.uint8)
        if image.dtype != np.uint8 and not np.array_equal(img8, image):
            raise ValueError("ToUint8: image values are not integers in [0, 255]")
        lab8 = label.astype(np.uint8)
        if label.dtype != np.uint8 and not np.array_equal(lab8, label):
            raise ValueError("ToUint8: label values are not integers in [0, 255]")
        return np.ascontiguousarray(img8), np.ascontiguousarray(lab8)


class AugBatch:
    """A collated batch: `data` uint8 [bytes] holding every image (RGB HWC) and label (HW) back to back, `header` int64
    [N, 4] rows (h, w, image offset, label offset). `pin_memory()` pins the data, so `DataLoader(pin_memory=True)`
    hands the main process a pinned batch."""

    def __init__(self, data, header):
        self.data = data
        self.header = header

    def __len__(self):
        return int(self.header.shape[0])

    def sizes(self):
        return [(int(h), int(w)) for h, w in self.header[:, :2].tolist()]

    def pin_memory(self, device=None):
        return AugBatch(self.data.pin_memory(), self.header)


def _check_pair(image, label):
    if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
        raise ValueError("augmentation takes uint8 HxWx3 RGB images (use ToUint8 as the dataset transform)")
    if not isinstance(label, np.ndarray) or label.dtype != np.uint8 or label.shape != image.shape[:2]:
        raise ValueError("augmentation takes uint8 HxW labels of the image's size")


def collate(samples):
    """DataLoader `collate_fn`: pack [(uint8 image, uint8 label), ...] into one AugBatch."""
    if len(samples) == 0:
        raise ValueError("collate: empty batch")
    header = np.zeros((len(samples), 4), dtype=np.int64)
    off = 0
    for i, (image, label) in enumerate(samples):
        _check_pair(image, label)
        h, w = label.shape
        header[i] = (h, w, off, off + 3 * h * w)
        off += 4 * h * w
    data = torch.empty(off, dtype=torch.uint8)
    buf = data.numpy()
    for (image, label), (h, w, io, lo) in zip(samples, header.tolist()):
        buf[io:lo] = image.reshape(-1)
        buf[lo:lo + h * w] = label.reshape(-1)
    return AugBatch(data, torch.from_numpy(header))


def _is_pair(x):
    return isinstance(x, collections.abc.Iterable) and len(x) == 2 and all(isinstance(v, numbers.Number) for v in x)


def _crop_size(crop):
    if isinstance(crop, int) and crop > 0:
        return crop, crop
    if isinstance(crop, collections.abc.Iterable) and len(crop) == 2 and all(isinstance(v, int) for v in crop) \
            and crop[0] > 0 and crop[1] > 0:
        return int(crop[0]), int(crop[1])
    raise RuntimeError("crop size error.\n")


def _channels(v, what):
    if not (isinstance(v, (list, tuple)) and len(v) == 3 and all(isinstance(x, numbers.Number) for x in v)):
        raise RuntimeError("%s should be a list of 3 numbers\n" % what)
    return [float(x) for x in v]


class _Augment:
    """Shared launch: descriptor table -> one non-blocking upload of the batch -> semseg_augment."""

    def __init__(self, crop, mean, std, ignore_label):
        self.crop_h, self.crop_w = _crop_size(crop)
        self.mean = _channels(mean, "mean")
        self.std = _channels(std, "std")
        if any(s == 0 for s in self.std):
            raise ValueError("std must be non-zero")
        if not isinstance(ignore_label, int):
            raise RuntimeError("ignore_label should be an integer number\n")
        self.ignore_label = ignore_label

    def _padded(self, rh, rw):
        return max(rh, self.crop_h), max(rw, self.crop_w)

    def descriptors(self, batch, params):
        """ctypes array of semseg_augment_desc for an AugBatch and one AugParams per sample."""
        descs = (_lib.AugmentDesc * len(batch))()
        for d, (h, w, io, lo), p in zip(descs, batch.header.tolist(), params):
            rh, rw = resized_size(h, w, p.fx, p.fy)
            d.img_off, d.lab_off, d.h, d.w, d.rh, d.rw = io, lo, h, w, rh, rw
            d.scale_x, d.scale_y = 1.0 / p.fx, 1.0 / p.fy
            if p.angle is not None:
                d.m[:] = rotation_inverse(rh, rw, p.angle)
                d.rotate = 1
            d.blur, d.flip = int(p.blur), int(p.flip)
            d.pad_top, d.pad_left = max(self.crop_h - rh, 0) // 2, max(self.crop_w - rw, 0) // 2
            d.off_y, d.off_x = p.h_off, p.w_off
        return descs

    def apply(self, batch, params):
        """Run the chain on `batch` (an AugBatch or a list of (image, label) pairs) with explicit per-sample AugParams.
        -> (input fp32 [N,3,ch,cw], target int64 [N,ch,cw]) on the current CUDA device and stream."""
        if not isinstance(batch, AugBatch):
            batch = collate(batch)
        descs = self.descriptors(batch, params)
        device = torch.device("cuda", torch.cuda.current_device())
        # both uploads are asynchronous: the descriptor table from pinned memory, the batch as the loader pinned it
        table = torch.empty(ctypes.sizeof(descs), dtype=torch.uint8, pin_memory=True)
        ctypes.memmove(table.data_ptr(), descs, ctypes.sizeof(descs))
        table_dev = table.to(device, non_blocking=True)
        data_dev = batch.data.to(device, non_blocking=True)
        return ops.augment(data_dev, descs, table_dev, self.crop_h, self.crop_w, self.mean, self.std,
                           self.ignore_label)


class TrainAugment(_Augment):
    """tool/train.py:194-201's train_transform on the GPU. Arguments are the reference constructors': crop = Crop's
    size, scale / aspect_ratio = RandScale's, rotate / rotate_p = RandRotate's (padding = mean), mean / std = Normalize's
    (and the padding value), ignore_label = RandRotate's and Crop's. blur / flip False leave that transform out of the
    chain (neither draws). `aug(batch, rng=random)` -> (input fp32 [N,3,ch,cw], target int64 [N,ch,cw]) on the current
    CUDA device and stream, without synchronising the host."""

    def __init__(self, crop, scale, rotate, mean, std, ignore_label=255, aspect_ratio=None, rotate_p=0.5, blur=True,
                 flip=True):
        if not (isinstance(scale, collections.abc.Iterable) and len(scale) == 2):
            raise ValueError("scale must be a pair [min, max]")
        if not (_is_pair(scale) and 0 < scale[0] < scale[1]):
            raise RuntimeError("segtransform.RandScale() scale param error.\n")
        if aspect_ratio is not None and not (_is_pair(aspect_ratio) and 0 < aspect_ratio[0] < aspect_ratio[1]):
            raise RuntimeError("segtransform.RandScale() aspect_ratio param error.\n")
        if not (isinstance(rotate, collections.abc.Iterable) and len(rotate) == 2):
            raise ValueError("rotate must be a pair [min, max]")
        if not (_is_pair(rotate) and rotate[0] < rotate[1]):
            raise RuntimeError("segtransform.RandRotate() scale param error.\n")
        super().__init__(crop, mean, std, ignore_label)
        self.scale, self.aspect_ratio, self.rotate = list(scale), aspect_ratio, list(rotate)
        self.rotate_p, self.blur, self.flip = rotate_p, bool(blur), bool(flip)

    def draw_params(self, sizes, rng=random):
        """Per-sample parameters for source sizes [(h, w), ...], drawn from `rng` exactly as the reference chain draws
        them from `random` (RandScale, RandRotate, RandomGaussianBlur, RandomHorizontalFlip, Crop's two randints)."""
        out = []
        for h, w in sizes:
            s = self.scale[0] + (self.scale[1] - self.scale[0]) * rng.random()
            ar = 1.0
            if self.aspect_ratio is not None:
                ar = math.sqrt(self.aspect_ratio[0] + (self.aspect_ratio[1] - self.aspect_ratio[0]) * rng.random())
            fx, fy = s * ar, s / ar
            rh, rw = resized_size(h, w, fx, fy)
            angle = None
            if rng.random() < self.rotate_p:
                angle = self.rotate[0] + (self.rotate[1] - self.rotate[0]) * rng.random()
            blur = self.blur and rng.random() < 0.5
            flip = self.flip and rng.random() < 0.5
            ph, pw = self._padded(rh, rw)
            h_off = rng.randint(0, ph - self.crop_h)
            w_off = rng.randint(0, pw - self.crop_w)
            out.append(AugParams(fx, fy, angle, blur, flip, h_off, w_off))
        return out

    def __call__(self, batch, rng=random):
        if not isinstance(batch, AugBatch):
            batch = collate(batch)
        return self.apply(batch, self.draw_params(batch.sizes(), rng))


class ValAugment(_Augment):
    """tool/train.py:209-212's val_transform (centre Crop with mean / ignore_label padding, ToTensor, Normalize) on the
    same kernel with every random stage off. `aug(batch)` -> (input, target) as TrainAugment."""

    def __init__(self, crop, mean, std, ignore_label=255):
        super().__init__(crop, mean, std, ignore_label)

    def draw_params(self, sizes, rng=None):
        out = []
        for h, w in sizes:
            ph, pw = self._padded(h, w)
            out.append(AugParams(1.0, 1.0, None, False, False, int((ph - self.crop_h) / 2), int((pw - self.crop_w) / 2)))
        return out

    def __call__(self, batch):
        if not isinstance(batch, AugBatch):
            batch = collate(batch)
        return self.apply(batch, self.draw_params(batch.sizes()))


def _number(name, v):
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise TypeError("%s must be a number, got %r" % (name, v))
    v = float(v)
    if not math.isfinite(v):
        raise ValueError("%s must be finite, got %r" % (name, v))
    return v


class StrongAugment:
    """The strong view of weak-to-strong mean-teacher training (FixMatch, UniMatch, U2PL, CutMix-Seg): colour jitter,
    random grayscale and Gaussian blur of a normalised fp32 NCHW batch on the GPU, in two launches of csrc/strong.cu,
    without a host synchronisation (so it runs inside a captured training step). The defaults are UniMatch's strong
    pipeline; `mean` / `std` are the normalisation the batch carries (the trainer's, tool/train.py:189-192), and the view
    is computed on the de-normalised image. Give it to a teacher criterion (losses.DistillationLoss, PseudoLabelLoss,
    MixPseudoLabelLoss: `strong=`) and the teacher sees the batch while the student sees its strong view.

    Each image n has its own uniforms u[n, 0..11], one torch.rand(N, 12) on the device's default CUDA generator (`draw`).
    Per image (include/semseg_b200.h semseg_strong_augment states it exactly):

        v      = clamp((x std_c + mean_c) / 255, 0, 1)       only when some operation applies; else x is copied bit for bit
        jitter iff u0 < p_jitter: factors b in [max(0, 1 - brightness), 1 + brightness] by u1, contrast c by u2,
               saturation s by u3 alike, hue in [-hue, hue] by u4 (each lo + (hi - lo) u in fp64, rounded once to fp32);
               a strength of 0 skips its operation (torchvision's None); the order is ascending (u5..u8, index) in
               place of torchvision's randperm(4). Each is torchvision.transforms.v2.functional's float form:
               brightness clamp(b v), contrast clamp(c v + (1 - c) mean(gray(v))), saturation clamp(s v + (1 - s)
               gray(v)), hue through torchvision's HSV conversion; gray = 0.2989 r + 0.587 g + 0.114 b
        gray   iff u9 < p_gray: every channel becomes gray(v)
        blur   iff u10 < p_blur: sigma = sigma_lo + (sigma_hi - sigma_lo) u11, r = ceil(3 sigma), the true Gaussian of
               torchvision's gaussian_blur(v, [2r+1]*2, [sigma]*2) with reflect padding. UniMatch blurs with PIL's box
               approximation of a Gaussian; this is the exact one. PIL's uint8 rounding between operations is not
               reproduced either: the chain stays in fp32.
        x_s    = (255 v - mean_c) / std_c

    The operations move no pixel, so labels stay valid. There is no gradient through the view: an input with
    requires_grad raises. `strong(x, u=None)` -> the view (u = strong.draw(x) when None), a new tensor; the input is a
    CUDA fp32 [N, 3, H, W] tensor with H, W > ceil(3 sigma_hi). Under DistributedDataParallel each rank draws its own
    view (multi-GPU runs have not been made)."""

    def __init__(self, brightness=0.5, contrast=0.5, saturation=0.5, hue=0.25, p_jitter=0.8, p_gray=0.2, p_blur=0.5,
                 sigma=(0.1, 2.0), mean=(0.485 * 255, 0.456 * 255, 0.406 * 255),
                 std=(0.229 * 255, 0.224 * 255, 0.225 * 255)):
        for name, v in (("brightness", brightness), ("contrast", contrast), ("saturation", saturation), ("hue", hue)):
            v = _number(name, v)
            if v < 0.0:
                raise ValueError("%s must be >= 0, got %r" % (name, v))
            setattr(self, name, v)
        if self.hue > 0.5:
            raise ValueError("hue must be <= 0.5, got %r" % self.hue)
        for name, v in (("p_jitter", p_jitter), ("p_gray", p_gray), ("p_blur", p_blur)):
            v = _number(name, v)
            if not 0.0 <= v <= 1.0:
                raise ValueError("%s must lie in [0, 1], got %r" % (name, v))
            setattr(self, name, v)
        if not isinstance(sigma, (tuple, list)) or len(sigma) != 2:
            raise TypeError("sigma must be a pair (lo, hi), got %r" % (sigma,))
        lo, hi = _number("sigma", sigma[0]), _number("sigma", sigma[1])
        if not 0.0 < lo <= hi <= 5.0:
            raise ValueError("sigma must satisfy 0 < lo <= hi <= 5, got %r" % (sigma,))
        self.sigma = (lo, hi)
        for name, v in (("mean", mean), ("std", std)):
            if not isinstance(v, (tuple, list)) or len(v) != 3:
                raise ValueError("%s must hold 3 numbers, got %r" % (name, v))
            setattr(self, name, tuple(_number(name, c) for c in v))
        if any(s <= 0.0 for s in self.std):
            raise ValueError("std must be > 0, got %r" % (self.std,))

    def key(self):
        """The options as a tuple: what a captured training step bakes in."""
        return (self.brightness, self.contrast, self.saturation, self.hue, self.p_jitter, self.p_gray, self.p_blur,
                self.sigma, self.mean, self.std)

    def extra_repr(self):
        return "brightness=%g, contrast=%g, saturation=%g, hue=%g, p_jitter=%g, p_gray=%g, p_blur=%g, sigma=(%g, %g)" \
               ", mean=(%g, %g, %g), std=(%g, %g, %g)" % ((self.brightness, self.contrast, self.saturation, self.hue,
                                                           self.p_jitter, self.p_gray, self.p_blur) + self.sigma +
                                                          self.mean + self.std)

    def __repr__(self):
        return "StrongAugment(%s)" % self.extra_repr()

    def _check(self, x):
        if not torch.is_tensor(x):
            raise TypeError("StrongAugment: the input must be a tensor, got %s" % type(x).__name__)
        if x.requires_grad:
            raise RuntimeError("StrongAugment: there is no gradient through the strong view; the input must not "
                               "require grad")
        if not x.is_cuda or x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise TypeError("StrongAugment: the input must be a CUDA fp32 [N, 3, H, W] tensor, got %s %s on %s" %
                            (x.dtype, tuple(x.shape), x.device))
        r = math.ceil(3.0 * self.sigma[1])
        if x.shape[2] <= r or x.shape[3] <= r:
            raise ValueError("StrongAugment: a %dx%d image needs H, W > ceil(3 sigma_hi) = %d" % (x.shape[2], x.shape[3],
                                                                                                  r))

    def draw(self, x, views=1):
        """The uniforms of `views` views of `x`: fp32 [views * N, 12] from one torch.rand on x's device, view-major."""
        self._check(x)
        return torch.rand((views * x.shape[0], 12), device=x.device)

    def __call__(self, x, u=None):
        self._check(x)
        if u is None:
            u = self.draw(x)
        if not (torch.is_tensor(u) and u.dtype == torch.float32 and u.device == x.device and u.dim() == 2 and
                u.shape[0] == x.shape[0] and u.shape[1] >= 12 and u.stride(1) == 1):
            raise ValueError("StrongAugment: uniforms must be fp32 [%d, >= 12] on %s" % (x.shape[0], x.device))
        return ops.strong_augment(x.contiguous(), u, self.brightness, self.contrast, self.saturation, self.hue,
                                  self.p_jitter, self.p_gray, self.p_blur, self.sigma, self.mean, self.std)
