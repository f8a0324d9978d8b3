"""Dense CRF refinement of segmentation scores at test time (Krähenbühl & Koltun, NeurIPS 2011), on the device.

`DenseCRF` is what users otherwise run through `pydensecrf` on the host, one image at a time: `DenseCRF2D` with
`addPairwiseGaussian(sxy=pos_xy_std, compat=pos_weight)` and `addPairwiseBilateral(sxy=bi_xy_std, srgb=bi_rgb_std,
compat=bi_weight)`, the unary of `unary_from_softmax(probs, clip)` and `inference(iterations)`. The defaults are the ones
of the pydensecrf README example. For one image with pixel positions p_i, RGB colours I_i in 0..255 and probabilities
P[c, i]:
    U[c, i]   = -log(max(P[c, i], clip))
    k_s(i, j) = exp(-|p_i - p_j|^2 / 2 pos_xy_std^2)
    k_a(i, j) = exp(-|p_i - p_j|^2 / 2 bi_xy_std^2 - |I_i - I_j|^2 / 2 bi_rgb_std^2)
each filter summed over all j (j = i included) and symmetrically normalised, K~ v = n * K (n * v) with
n = (K 1 + 1e-20)^-1/2, and Potts mean field from Q0 = softmax(-U):
    Q <- softmax_c(-U + pos_weight K~_s Q + bi_weight K~_a Q)     (`iterations` times).
K is approximated on a permutohedral lattice (Adams, Baek & Davis 2010), as pydensecrf does; csrc/densecrf.cu holds the
kernels and include/semseg_b200.h the C contract. The result is deterministic: two runs give the same bits.
"""
import math

import numpy as np
import torch

from . import _lib
from . import ops

__all__ = ["DenseCRF"]


def _number(name, value, positive):
    if isinstance(value, bool) or not isinstance(value, (int, float, np.integer, np.floating)):
        raise TypeError("DenseCRF: %s must be a number, got %r" % (name, value))
    v = float(value)
    if not math.isfinite(v) or (v <= 0.0 if positive else v < 0.0):
        raise ValueError("DenseCRF: %s must be finite and %s, got %r" % (name, "positive" if positive else ">= 0", value))
    return v


class DenseCRF:
    """crf(image, probs) -> refined marginals Q, fp32 [C, h, w] on the device.

    image: HWC RGB in 0..255, float32 (as util/dataset.py decodes it) or uint8, a numpy array or a CUDA tensor.
    probs: class probabilities, a CUDA fp32 or fp64 [C, h, w] tensor. There is no CPU fallback: CPU tensors raise
    SemsegError."""

    def __init__(self, iterations=5, pos_weight=3.0, pos_xy_std=3.0, bi_weight=10.0, bi_xy_std=80.0, bi_rgb_std=13.0,
                 clip=1e-5):
        if isinstance(iterations, bool) or not isinstance(iterations, (int, np.integer)):
            raise TypeError("DenseCRF: iterations must be an int, got %r" % (iterations,))
        if iterations < 0:
            raise ValueError("DenseCRF: iterations must be >= 0, got %d" % iterations)
        self.iterations = int(iterations)
        self.pos_weight = _number("pos_weight", pos_weight, False)
        self.pos_xy_std = _number("pos_xy_std", pos_xy_std, True)
        self.bi_weight = _number("bi_weight", bi_weight, False)
        self.bi_xy_std = _number("bi_xy_std", bi_xy_std, True)
        self.bi_rgb_std = _number("bi_rgb_std", bi_rgb_std, True)
        c = _number("clip", clip, True)
        if not (float(np.finfo(np.float32).tiny) <= c < 1.0):   # the kernels take log max(p, clip) in fp32
            raise ValueError("DenseCRF: clip must lie in [FLT_MIN, 1) = [1.18e-38, 1), got %r" % (clip,))
        self.clip = c

    def __repr__(self):
        return ("DenseCRF(iterations=%d, pos_weight=%g, pos_xy_std=%g, bi_weight=%g, bi_xy_std=%g, bi_rgb_std=%g, "
                "clip=%g)" % (self.iterations, self.pos_weight, self.pos_xy_std, self.bi_weight, self.bi_xy_std,
                              self.bi_rgb_std, self.clip))

    def _image(self, image, hw, device):
        if isinstance(image, np.ndarray):
            if image.dtype not in (np.float32, np.uint8):
                raise TypeError("DenseCRF: image must be float32 or uint8, got %s" % image.dtype)
            t = torch.from_numpy(np.ascontiguousarray(image))
        elif isinstance(image, torch.Tensor):
            if image.dtype not in (torch.float32, torch.uint8):
                raise TypeError("DenseCRF: image must be float32 or uint8, got %s" % image.dtype)
            if not image.is_cuda:
                raise _lib.SemsegError("DenseCRF needs a CUDA image tensor or a numpy array (no CPU fallback)")
            t = image
        else:
            raise TypeError("DenseCRF: image must be a numpy array or a CUDA tensor, got %s" % type(image).__name__)
        if t.dim() != 3 or t.shape[2] != 3 or tuple(t.shape[:2]) != hw:
            raise ValueError("DenseCRF: image must be HWC [%d, %d, 3] like probs, got %s" % (hw + (tuple(t.shape),)))
        return t.to(device, non_blocking=True).float().contiguous()

    def refine_hwc(self, image, probs_hwc):
        """The refined marginals fp32 [h, w, C] of class-contiguous fp32 probabilities [h, w, C] on the device (the
        layout the kernels use; SlidingWindowPredictor hands its scores over in it)."""
        h, w, C = probs_hwc.shape
        img = self._image(image, (h, w), probs_hwc.device)
        lattice, V = ops.densecrf_build(img, self.pos_xy_std, self.bi_xy_std, self.bi_rgb_std)
        Q = ops.densecrf_meanfield(lattice, (h, w), V, probs_hwc.reshape(h * w, C), self.clip, self.iterations,
                                   self.pos_weight, self.bi_weight)
        return Q.view(h, w, C)

    def __call__(self, image, probs):
        if not isinstance(probs, torch.Tensor):
            raise TypeError("DenseCRF: probs must be a CUDA tensor [C, h, w], got %s" % type(probs).__name__)
        if probs.dtype not in (torch.float32, torch.float64):
            raise TypeError("DenseCRF: probs must be float32 or float64, got %s" % probs.dtype)
        if probs.dim() != 3 or min(probs.shape) < 1:
            raise ValueError("DenseCRF: probs must be a non-empty [C, h, w] tensor, got %s" % (tuple(probs.shape),))
        if not probs.is_cuda:
            raise _lib.SemsegError("DenseCRF needs CUDA probabilities (no CPU fallback)")
        hwc = probs.permute(1, 2, 0).float().contiguous()
        return self.refine_hwc(image, hwc).permute(2, 0, 1).contiguous()
