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
With an `anomaly` scorer (anomaly.AnomalyScorer) the exact=False finishes carry two more channels through the same
steps: the flip-averaged max logit (ML) and logsumexp (LSE) of each crop's upsampled logits (csrc/window.cu's
stats variant of the scores kernel, or torch amax / logsumexp in the ATen finish). The C score channels and the argmax
are the same bits as without a scorer; the scorer turns ML, LSE or the scores into a per-pixel anomaly map.
With `mc_draws` = T > 0 the predictor does Monte Carlo dropout (Gal & Ghahramani 2016; Kendall et al. 2017): every
crop batch is scored under T dropout draws and the exact=False finish carries one more channel, the mean sample entropy
E[H], through the same accumulation and resize. On the native path the network runs once per batch up to cls[2] and
each draw is one masked 1x1 classifier (PSPNet._mc_eval_logits_nhwc); csrc/window.cu's MC variant of the scores kernel
upsamples, soft-maxes, flip-averages and draw-averages them (the [T, 2G, classes, crop, crop] logits never exist).
Any other model runs T forwards per batch with its dropout modules in training mode and the ATen steps. Both paths
take the same Dropout2d masks in the same order, so one seed gives both the same draws.
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
    from .fp8 import Fp8Eval
    from .psanet import PSANet
    from .pspnet import PSPNet
    if isinstance(model, Fp8Eval):      # the FP8 forward of its PSPNet / PSANet (semseg_b200/fp8.py)
        inner = _native_net(model.model, classes, crop_h, crop_w, device)
        return model if inner is not None else None
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

    def __init__(self, model, classes, crop_h, crop_w, mean, std=None, stride_rate=2 / 3, flip=True, max_batch=32,
                 crf=None, anomaly=None, mc_draws=0):
        """crf: None, or a densecrf.DenseCRF run on the scale-averaged scores before the argmax (both finishes); the
        returned scores are then its marginals.
        anomaly: None, or an anomaly.AnomalyScorer; __call__ then also returns its fp32 [h, w] CUDA anomaly map
        (exact=False only; not together with crf).
        mc_draws: 0 (deterministic), or T in 1..128 Monte Carlo dropout draws per crop; __call__ then returns the
        predictive mean and an uncertainty map (exact=False only; not with crf, anomaly or an Fp8Eval model; the model
        must hold a dropout layer with p > 0)."""
        from .anomaly import AnomalyScorer
        from .densecrf import DenseCRF
        from .fp8 import Fp8Eval
        if isinstance(mc_draws, bool) or not isinstance(mc_draws, (int, np.integer)):
            raise TypeError("SlidingWindowPredictor: mc_draws must be an int, got %s" % type(mc_draws).__name__)
        if not 0 <= int(mc_draws) <= 128:
            raise ValueError("SlidingWindowPredictor: mc_draws must be in 0..128 (0 = off), got %d" % mc_draws)
        self.mc_draws = int(mc_draws)
        if self.mc_draws:
            if crf is not None or anomaly is not None:
                raise ValueError("SlidingWindowPredictor: mc_draws cannot be combined with crf or anomaly")
            if isinstance(model, Fp8Eval):
                raise ValueError("SlidingWindowPredictor: mc_draws does not support an Fp8Eval model")
            if not any(isinstance(m, torch.nn.modules.dropout._DropoutNd) and m.p > 0 for m in model.modules()):
                raise ValueError("SlidingWindowPredictor: mc_draws needs a model with a dropout layer of p > 0")
        if crf is not None and not isinstance(crf, DenseCRF):
            raise TypeError("SlidingWindowPredictor: crf must be None or a DenseCRF, got %s" % type(crf).__name__)
        if anomaly is not None and not isinstance(anomaly, AnomalyScorer):
            raise TypeError("SlidingWindowPredictor: anomaly must be None or an AnomalyScorer, got %s"
                            % type(anomaly).__name__)
        if crf is not None and anomaly is not None:
            raise ValueError("SlidingWindowPredictor: crf and anomaly cannot be combined")
        self.crf, self.anomaly = crf, anomaly
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

    def _scores(self, crops, net=None, stats=False, mc=False):
        """[G, 3, ch, cw] normalised crops -> [G, classes, ch, cw] flip-averaged softmax scores (fp32). With `net` (see
        _native_net) the scores kernel writes each batch's scores straight into the result from the 1/8-resolution
        logits. With `stats` two more channels follow the scores: the flip-averaged max and logsumexp over the classes
        of the upsampled logits. With `mc` the scores are the mean over self.mc_draws dropout draws and one more
        channel follows them: the mean flip-averaged sample entropy."""
        per_call = self.max_batch // 2 if self.flip else self.max_batch
        if mc and net is None:
            return self._mc_scores_aten(crops, per_call)
        if net is not None:
            out = torch.empty((crops.shape[0], self.classes + (1 if mc else 2 if stats else 0)) + tuple(crops.shape[2:]),
                              dtype=torch.float32, device=crops.device)
            with torch.no_grad():
                for g0 in range(0, crops.shape[0], per_call):
                    part = crops[g0:g0 + per_call]
                    batch = torch.cat([part, part.flip(3)], 0) if self.flip else part
                    if mc:
                        logits = net._mc_eval_logits_nhwc(batch, self.mc_draws)
                        self.forward_calls += 1
                        ops.window_scores_mc(logits, self.flip, out[g0:g0 + part.shape[0]])
                        continue
                    logits = net._eval_logits_nhwc(batch)
                    self.forward_calls += 1
                    ops.window_scores(logits, self.flip, out[g0:g0 + part.shape[0]], stats)
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
                if stats:
                    lf = logits.float()
                    extra = torch.stack([lf.amax(1), torch.logsumexp(lf, 1)], 1)
                if self.flip:
                    n = part.shape[0]
                    prob = (prob[:n] + prob[n:].flip(3)) / 2
                    if stats:
                        extra = (extra[:n] + extra[n:].flip(3)) * 0.5
                if stats:
                    prob = torch.cat([prob, extra], 1)
                outs.append(prob)
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def _mc_scores_aten(self, crops, per_call):
        """The `mc` scores of _scores for any model: self.mc_draws forwards per batch with every dropout module of the
        model in training mode (each module's own mode restored afterwards, also on an error), then the ATen steps:
        upsample, softmax, sample entropy log S - sum_c q_c (v_c - max), flip average, draw mean."""
        drops = [m for m in self.model.modules() if isinstance(m, torch.nn.modules.dropout._DropoutNd)]
        modes = [m.training for m in drops]
        outs = []
        try:
            for m in drops:
                m.train()
            with torch.no_grad():
                for g0 in range(0, crops.shape[0], per_call):
                    part = crops[g0:g0 + per_call]
                    n = part.shape[0]
                    batch = torch.cat([part, part.flip(3)], 0) if self.flip else part
                    acc = None
                    for _ in range(self.mc_draws):
                        logits = self.model(batch)
                        self.forward_calls += 1
                        if logits.shape[2:] != batch.shape[2:]:
                            logits = F.interpolate(logits, tuple(batch.shape[2:]), mode="bilinear", align_corners=True)
                        lf = logits.float()
                        prob = F.softmax(lf, dim=1)
                        d = lf - lf.amax(1, keepdim=True)
                        ent = torch.logsumexp(d, 1) - (prob * d).sum(1)
                        sample = torch.cat([prob, ent[:, None]], 1)
                        if self.flip:
                            sample = (sample[:n] + sample[n:].flip(3)) * 0.5
                        acc = sample if acc is None else acc + sample
                    outs.append(acc * (1.0 / self.mc_draws))
        finally:
            for m, mode in zip(drops, modes):
                m.train(mode)
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    # ------------------------------------------------------------------------------------------- one scale
    def _scale_canvas(self, image, net=None, stats=False, mc=False):
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
        scores = self._scores(crops, net, stats, mc)
        if net is not None:
            return ops.window_accumulate(scores, ys, xs, (full_h, full_w), top, left, (img_h, img_w))
        canvas = torch.zeros((scores.shape[1], full_h, full_w), dtype=torch.float64, device=self.device)
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

    def scale_on_device(self, image, out_h, out_w, stats=False, mc=False):
        """Same scores as `scale`, float64 [classes, out_h, out_w], resized on the device (bilinear, half-pixel centres,
        no anti-aliasing = cv2.INTER_LINEAR's sampling; cv2 rounds its interpolation weights to fp32, so the two agree
        to ~1e-7, not bit for bit)."""
        canvas = self._scale_canvas(image, stats=stats, mc=mc)
        return F.interpolate(canvas[None], size=(out_h, out_w), mode="bilinear", align_corners=False)[0]

    # ------------------------------------------------------------------------------------------- one image
    def _stats_total(self, image, base_size, scales, mc=False):
        """The exact=False finish with the two statistics channels: (total fp64 [classes + 2, h, w] on the device, the
        scale average of the scores, ML and LSE; argmax int64 [h, w] of its score channels). With `mc` the one MC
        dropout channel instead: total [classes + 1, h, w], the predictive mean and the mean sample entropy E[H]."""
        h, w = image.shape[:2]
        total = torch.zeros((self.classes + (1 if mc else 2), h, w), dtype=torch.float64, device=self.device)
        net = _native_net(self.model, self.classes, self.crop_h, self.crop_w, self.device)
        stats = not mc
        for s in scales:
            new_h, new_w = scaled_size(h, w, round(s * base_size))
            resized = cv2.resize(image, (new_w, new_h), interpolation=cv2.INTER_LINEAR)
            if net is not None:
                ops.window_resize_add(self._scale_canvas(resized, net, stats=stats, mc=mc), total)
            else:
                total += self.scale_on_device(resized, h, w, stats=stats, mc=mc)
        total /= len(scales)
        return total, total[:self.classes].argmax(0)

    def __call__(self, image, base_size, scales, exact=False, return_scores=True):
        """(scores float64 [h, w, classes] or None, argmax int64 [h, w]) of a float32 HWC image: the body of the
        evaluation loop, tool/test.py:186-199.

        exact=True  : every step as in the reference (host cv2 resize of each scale's score map, numpy accumulation):
                      bit-identical to the serial procedure, but the host works on [h, w, classes] float64 arrays.
        exact=False : score maps are resized, summed over the scales and arg-maxed on the device; only the result
                      crosses PCIe (the argmax, plus the scores when return_scores).
        With a `crf`, the scale-averaged scores are refined by it on the device before the argmax, in both finishes,
        and the scores returned are its marginals (float64 [h, w, classes]).
        With an `anomaly` scorer the result is (scores, argmax, anomaly map fp32 [h, w] on the device); scores and
        argmax are the same bits as without it. exact=True raises ValueError then.
        With mc_draws = T > 0 the result is (scores, argmax, uncertainty): scores the MC predictive mean p_bar (float64
        [h, w, classes], or None), argmax its argmax, uncertainty fp32 [2, h, w] on the device: channel 0 the predictive
        entropy H[p_bar] = -sum_c p_bar log p_bar (0 log 0 = 0), channel 1 the mutual information H[p_bar] - E[H[p]]
        (not clamped), both in nats. Every sample the predictor averages (T draws x the crop and its mirror x the
        overlapping crops x the scales) enters p_bar and E[H] with the same weight, so the mutual information is the
        Jensen gap over all of them: zero only where a pixel sees one sample (T = 1, no flip, one crop, one scale).
        exact=True raises ValueError then."""
        if self.mc_draws:
            if exact:
                raise ValueError("SlidingWindowPredictor: exact=True does not support mc_draws")
            total, pred = self._stats_total(image, base_size, scales, mc=True)
            pbar = total[:self.classes]
            hbar = -torch.special.xlogy(pbar, pbar).sum(0)
            uncertainty = torch.stack([hbar, hbar - total[self.classes]]).float()
            scores = pbar.permute(1, 2, 0).contiguous().cpu().numpy() if return_scores else None
            return scores, pred.cpu().numpy(), uncertainty
        if self.anomaly is not None:
            if exact:
                raise ValueError("SlidingWindowPredictor: exact=True does not support an anomaly scorer")
            total, pred = self._stats_total(image, base_size, scales)
            amap = self.anomaly.score_map(total, pred)
            scores = total[:self.classes].permute(1, 2, 0).contiguous().cpu().numpy() if return_scores else None
            return scores, pred.cpu().numpy(), amap
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
        if self.crf is not None:
            # the CRF works on class-contiguous fp32 scores on the device; exact=True sends its host total there once
            scores = torch.from_numpy(total).to(self.device) if exact else total.permute(1, 2, 0)
            q = self.crf.refine_hwc(image, scores.float().contiguous())
            amax = q.argmax(2).cpu().numpy()
            return (q.double().cpu().numpy() if exact or return_scores else None), amax
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
