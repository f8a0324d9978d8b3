"""Batched multi-scale sliding-window inference (SURVEY §8 f3) — drop-in for the evaluation helpers of the reference.

The reference (tool/test.py:122-199, mirrored in tool/demo.py:106-181) pushes ONE crop (+ its mirror) through the
network per call: at base size 2048 / crop 713 / six scales that is 81 crops = 162 serial forward passes and 81
device→host copies of a [classes, 713, 713] score map per image, with the accumulation done by numpy on the host.
Here every crop of a scale goes through the network in batches and mirroring / softmax / flip-averaging /
accumulation / normalisation by the overlap count stay on the device. Two ways to finish:
  * exact=True — each scale's score map goes to the host once and the reference's own last steps (cv2 INTER_LINEAR
    resize to the image size, numpy sum over scales, argmax) run there. Crop grid, padding, normalisation, flip
    averaging, float64 accumulation order and the resizes are the reference's, so for a network whose per-image output
    does not depend on what else is in the batch (true for this package's kernels: every tile belongs to one image) the
    scores are bit-identical to the serial procedure.
  * exact=False (default) — the per-scale resize (same half-pixel bilinear sampling as cv2.INTER_LINEAR, fp64 weights),
    the sum over scales and the argmax also run on the device; only the result crosses PCIe. At 1024x2048 x 19 classes
    the host steps of the reference procedure (float64 [h, w, classes] arrays through cv2 and numpy) cost several times
    the network itself. Scores agree with the exact path to ~1e-7.
    When the model is this package's PSPNet / PSANet (eval mode, CUDA, crop = 8(h'-1)+1, at most 256 classes, any zoom
    factor) everything after the network runs on the native kernels of csrc/window.cu: one kernel turns the 1/8
    resolution logits of a batch into flip-averaged softmax scores (the upsampled [2G, classes, crop, crop] logits never
    exist), one gathers a scale's crops into its overlap-normalised fp64 canvas (bit-identical to the ATen loop), and
    one resizes the canvas and adds it into the running total. Any other model runs the ATen steps below.
    At zoom factor Z < 8 the model's output is the logits upsampled xZ, and the ATen steps upsample that again by 8/Z
    to the crop. The native kernel upsamples the 1/8-resolution logits x8 straight to the crop instead. The two are
    equal up to fp32 rounding: the xZ grid nests in the x8 grid (align_corners), the xZ result is bilinear on every
    cell of its grid, and bilinear interpolation reproduces a bilinear function exactly.
`net_process` / `scale_process` keep the reference's signatures and return types (and the exact arithmetic);
`SlidingWindowPredictor` is the object form that also covers the per-image scale loop.

The engine is device-agnostic torch glue around `model(batch)`; the arithmetic that matters (the network) is the CUDA
path of this package when `model` is a semseg_b200 PSPNet / PSANet in eval mode.
"""
import math

import cv2
import numpy as np
import torch
import torch.nn.functional as F

from . import ops

__all__ = ["crop_origins", "scaled_size", "net_process", "scale_process", "SlidingWindowPredictor"]


def crop_origins(extent, crop, stride_rate=2 / 3):
    """Start offsets of the crops along one axis: they advance by ceil(crop * stride_rate) and the last one is pulled
    back so that it ends at the border (tool/test.py:158-173)."""
    stride = int(math.ceil(crop * stride_rate))
    count = int(math.ceil(float(extent - crop) / stride) + 1)
    return [min(k * stride + crop, extent) - crop for k in range(count)]


def scaled_size(h, w, long_size):
    """(new_h, new_w): long side = long_size, short side rounded (tool/test.py:187-193)."""
    if h > w:
        return long_size, round(long_size / float(h) * w)
    return round(long_size / float(w) * h), long_size


def _model_device(model):
    p = next(iter(model.parameters()), None)
    return p.device if p is not None else torch.device("cpu")


def _native_net(model, classes, crop_h, crop_w, device):
    """The semseg_b200 PSPNet / PSANet behind `model` when its scores can be finished by csrc/window.cu, else None."""
    from .psanet import PSANet
    from .pspnet import PSPNet
    if isinstance(model, torch.nn.DataParallel):
        if len(model.device_ids) > 1:
            return None
        model = model.module
    # any zoom factor: the scores kernel upsamples the 1/8-resolution logits x8 (see the module docstring)
    if not (type(model) in (PSPNet, PSANet) and not model.training and device.type == "cuda"
            and (crop_h - 1) % 8 == 0 and (crop_w - 1) % 8 == 0 and classes <= 256):
        return None
    return model


class SlidingWindowPredictor:
    """model: eval-mode network mapping [B, 3, crop_h, crop_w] -> [B, classes, h', w'] logits."""

    def __init__(self, model, classes, crop_h, crop_w, mean, std=None, stride_rate=2 / 3, flip=True, max_batch=32):
        self.model, self.classes = model, int(classes)
        self.crop_h, self.crop_w = int(crop_h), int(crop_w)
        self.mean = [float(m) for m in mean]
        self.std = None if std is None else [float(s) for s in std]
        self.stride_rate, self.flip = stride_rate, bool(flip)
        self.max_batch = max(2 if flip else 1, int(max_batch))
        self.device = _model_device(model)
        self.forward_calls = 0          # model invocations so far (the reference makes one per crop)

    # ------------------------------------------------------------------------------------------- device side
    def _normalised(self, image_hwc):
        """float32 HWC numpy -> normalised float32 CHW tensor on the model's device ((x - mean) / std in fp32, the
        same two roundings as the reference's in-place sub_/div_, tool/test.py:124-129)."""
        t = torch.from_numpy(np.ascontiguousarray(image_hwc)).to(self.device, non_blocking=True).float()
        t = t.permute(2, 0, 1)
        t = t - torch.tensor(self.mean, dtype=torch.float32, device=self.device).view(3, 1, 1)
        if self.std is not None:
            t = t / torch.tensor(self.std, dtype=torch.float32, device=self.device).view(3, 1, 1)
        return t.contiguous()

    def _scores(self, crops, net=None):
        """[G, 3, ch, cw] normalised crops -> [G, classes, ch, cw] flip-averaged softmax scores (fp32). With `net` (see
        _native_net) the scores kernel writes each batch's scores straight into the result from the 1/8-resolution
        logits."""
        per_call = self.max_batch // 2 if self.flip else self.max_batch
        if net is not None:
            out = torch.empty((crops.shape[0], self.classes) + tuple(crops.shape[2:]), dtype=torch.float32,
                              device=crops.device)
            with torch.no_grad():
                for g0 in range(0, crops.shape[0], per_call):
                    part = crops[g0:g0 + per_call]
                    logits = net._eval_logits_nhwc(torch.cat([part, part.flip(3)], 0) if self.flip else part)
                    self.forward_calls += 1
                    ops.window_scores(logits, self.flip, out[g0:g0 + part.shape[0]])
            return out
        outs = []
        with torch.no_grad():
            for g0 in range(0, crops.shape[0], per_call):
                part = crops[g0:g0 + per_call]
                batch = torch.cat([part, part.flip(3)], 0) if self.flip else part
                logits = self.model(batch)
                self.forward_calls += 1
                if logits.shape[2:] != batch.shape[2:]:
                    logits = F.interpolate(logits, tuple(batch.shape[2:]), mode="bilinear", align_corners=True)
                prob = F.softmax(logits.float(), dim=1)
                if self.flip:
                    n = part.shape[0]
                    prob = (prob[:n] + prob[n:].flip(3)) / 2
                outs.append(prob)
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    # ------------------------------------------------------------------------------------------- one scale
    def _scale_canvas(self, image, net=None):
        """Overlap-normalised scores of one rescaled image, un-padded: float64 [classes, img_h, img_w] on the device
        (tool/test.py:148-176: padding, crop grid, accumulation in grid order, division by the crop count). With `net`
        the scores and the accumulation run on the native kernels (contiguous result, same bits as the loop)."""
        ch, cw = self.crop_h, self.crop_w
        img_h, img_w = image.shape[:2]
        extra_h, extra_w = max(ch - img_h, 0), max(cw - img_w, 0)
        top, left = extra_h // 2, extra_w // 2
        if extra_h or extra_w:
            image = cv2.copyMakeBorder(image, top, extra_h - top, left, extra_w - left, cv2.BORDER_CONSTANT,
                                       value=self.mean)
        full_h, full_w = image.shape[:2]
        ys, xs = crop_origins(full_h, ch, self.stride_rate), crop_origins(full_w, cw, self.stride_rate)
        windows = [(y0, x0) for y0 in ys for x0 in xs]
        x = self._normalised(image)
        crops = torch.stack([x[:, y0:y0 + ch, x0:x0 + cw] for y0, x0 in windows], 0)
        scores = self._scores(crops, net)
        if net is not None:
            return ops.window_accumulate(scores, ys, xs, (full_h, full_w), top, left, (img_h, img_w))
        canvas = torch.zeros((self.classes, full_h, full_w), dtype=torch.float64, device=self.device)
        hits = np.zeros((full_h, full_w), dtype=np.float64)
        for k, (y0, x0) in enumerate(windows):          # grid order = the reference's accumulation order
            canvas[:, y0:y0 + ch, x0:x0 + cw] += scores[k]
            hits[y0:y0 + ch, x0:x0 + cw] += 1
        canvas /= torch.from_numpy(hits).to(self.device)
        return canvas[:, top:top + img_h, left:left + img_w]

    def scale(self, image, out_h, out_w):
        """Scores float64 [out_h, out_w, classes] of one (already rescaled) float32 HWC image — scale_process,
        tool/test.py:148-178, with the reference's own final step (cv2 INTER_LINEAR on the host): bit-identical to the
        serial procedure; one device->host copy per scale."""
        host = self._scale_canvas(image).permute(1, 2, 0).contiguous().cpu().numpy()
        return cv2.resize(host, (out_w, out_h), interpolation=cv2.INTER_LINEAR)

    def scale_on_device(self, image, out_h, out_w):
        """Same scores as `scale`, float64 [classes, out_h, out_w], resized on the device (bilinear, half-pixel centres,
        no anti-aliasing = cv2.INTER_LINEAR's sampling; cv2 rounds its interpolation weights to fp32, so the two agree
        to ~1e-7, not bit for bit)."""
        canvas = self._scale_canvas(image)
        return F.interpolate(canvas[None], size=(out_h, out_w), mode="bilinear", align_corners=False)[0]

    # ------------------------------------------------------------------------------------------- one image
    def __call__(self, image, base_size, scales, exact=False, return_scores=True):
        """(scores float64 [h, w, classes] or None, argmax int64 [h, w]) of a float32 HWC image: the body of the
        evaluation loop, tool/test.py:186-199.

        exact=True  : every step as in the reference (host cv2 resize of each scale's score map, numpy accumulation):
                      bit-identical to the serial procedure, but the host works on [h, w, classes] float64 arrays.
        exact=False : score maps are resized, summed over the scales and arg-maxed on the device; only the result
                      crosses PCIe (the argmax, plus the scores when return_scores)."""
        h, w = image.shape[:2]
        total = np.zeros((h, w, self.classes), dtype=np.float64) if exact else \
            torch.zeros((self.classes, h, w), dtype=torch.float64, device=self.device)
        net = None if exact else _native_net(self.model, self.classes, self.crop_h, self.crop_w, self.device)
        for s in scales:
            new_h, new_w = scaled_size(h, w, round(s * base_size))
            resized = cv2.resize(image, (new_w, new_h), interpolation=cv2.INTER_LINEAR)
            if exact:
                total += self.scale(resized, h, w)
            elif net is not None:
                ops.window_resize_add(self._scale_canvas(resized, net), total)     # resize + add in one pass
            else:
                total += self.scale_on_device(resized, h, w)
        total /= len(scales)
        if exact:
            return total, np.argmax(total, axis=2)
        amax = total.argmax(0).cpu().numpy()
        return (total.permute(1, 2, 0).contiguous().cpu().numpy() if return_scores else None), amax


def net_process(model, image, mean, std=None, flip=True):
    """Reference signature (tool/test.py:122): softmax scores float32 [h, w, classes] of one HWC float32 crop."""
    h, w = image.shape[:2]
    p = SlidingWindowPredictor(model, 0, h, w, mean, std, flip=flip)
    x = p._normalised(image)
    return p._scores(x[None])[0].permute(1, 2, 0).float().cpu().numpy()


def scale_process(model, image, classes, crop_h, crop_w, h, w, mean, std=None, stride_rate=2 / 3, max_batch=32):
    """Reference signature (tool/test.py:148) plus `max_batch`: scores float64 [h, w, classes] of one rescaled image."""
    return SlidingWindowPredictor(model, classes, crop_h, crop_w, mean, std, stride_rate, True, max_batch).scale(image, h, w)
