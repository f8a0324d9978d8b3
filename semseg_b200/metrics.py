"""Device-side evaluation metrics of the training / validation loop (SURVEY §8 f4).

`intersectionAndUnionGPU` has the signature, return values and in-place side effect of the reference's helper
(util/util.py:55-67, used at tool/train.py:286 and :375) but is ONE kernel with integer shared-memory histograms
instead of a masked write, a boolean-mask gather and three `torch.histc` passes. Replace the import in tool/train.py:21
by `from semseg_b200.metrics import intersectionAndUnionGPU`.

`boundaryIoUGPU` has the same call shape and returns the Boundary IoU counts (Cheng et al., CVPR 2021): region IoU
hardly moves when only object boundaries improve, the band counts do.
"""
import ctypes
import math

import torch

from . import _lib

from . import ops

__all__ = ["intersectionAndUnionGPU", "boundaryIoUGPU"]


def intersectionAndUnionGPU(output, target, K, ignore_index=255):
    """output, target: int64 CUDA tensors of the same shape (N, N*L or N*H*W), class ids in [0, K).
    Returns (area_intersection, area_union, area_target): float32 [K] tensors on the device. Like the reference,
    `output` is overwritten with `ignore_index` wherever `target == ignore_index`."""
    assert output.dim() in [1, 2, 3]
    assert output.shape == target.shape
    if not (output.is_cuda and target.is_cuda):
        raise _lib.SemsegError("intersectionAndUnionGPU needs CUDA tensors (no CPU fallback); use the reference's "
                               "numpy intersectionAndUnion on the host")
    assert output.dtype == torch.int64 and target.dtype == torch.int64
    lib = _lib.load()
    out_flat = output.view(-1)                  # a view: the masking below is visible to the caller, as in the reference
    tgt_flat = target.reshape(-1)
    counts = torch.empty((3, int(K)), dtype=torch.int32, device=output.device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(output.device).cuda_stream)
    _lib.check(lib.semseg_iou_hist(ctypes.c_void_p(out_flat.data_ptr()), ctypes.c_void_p(tgt_flat.data_ptr()),
                                   out_flat.numel(), int(K), int(ignore_index), 1,
                                   ctypes.c_void_p(counts.data_ptr()), stream), "semseg_iou_hist")
    c = counts.float()
    return c[0], c[1] + c[2] - c[0], c[2]


def boundaryIoUGPU(output, target, K, ignore_index=255, dilation_ratio=0.02):
    """output, target: int64 CUDA tensors [N, H, W], class ids in [0, K). Returns (area_intersection, area_union,
    area_target) of the Boundary IoU: float32 [K] tensors on the device, summable over batches like
    intersectionAndUnionGPU's. With the band width d = max(1, round(dilation_ratio * sqrt(H^2 + W^2))), a pixel of class
    c lies in its map's band if its (2d+1)^2 window holds a pixel of another label or reaches outside the image (in the
    target, ignore_index is a label of its own); this is the paper's per-class mask, padded by 1, 3x3-eroded d times and
    subtracted from the mask. Over the pixels whose target is not ignore_index:
        I_c = #(target == output == c, both in their band),  T_c = #(target c in band),
        U_c = T_c + #(output c in band) - I_c.
    `output` is not modified. The window is separable: two passes of integer minima / maxima, then integer histograms."""
    if output.dim() != 3 or output.shape != target.shape:
        raise ValueError("boundaryIoUGPU: output and target [N, H, W] expected, got %s and %s" %
                         (tuple(output.shape), tuple(target.shape)))
    if not (output.is_cuda and target.is_cuda):
        raise _lib.SemsegError("boundaryIoUGPU needs CUDA tensors (no CPU fallback)")
    if output.dtype != torch.int64 or target.dtype != torch.int64:
        raise TypeError("boundaryIoUGPU: int64 output and target expected, got %s and %s" % (output.dtype, target.dtype))
    h, w = output.shape[1], output.shape[2]
    d = max(1, round(float(dilation_ratio) * math.sqrt(h * h + w * w)))
    c = ops.boundary_iou_hist(output, target, K, ignore_index, d).float()
    return c[0], c[1] + c[2] - c[0], c[2]
