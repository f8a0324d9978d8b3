"""Anomaly (out-of-distribution) segmentation on sliding-window predictions, and its pixel-level metrics.

`AnomalyScorer` turns what inference.SlidingWindowPredictor computes for an image into a per-pixel anomaly score,
higher = more anomalous. Let p be the scale-averaged probabilities, y their argmax (first maximum), and ML / LSE the
max / logsumexp (max + log sum exp(v - max)) over the classes of each crop's bilinearly upsampled logits, flip-averaged
as (a + a_mirror) * 0.5, then overlap-averaged, resized and scale-averaged exactly as a probability channel is:
  * "msp"      : 1 - max_c p_c;
  * "maxlogit" : -ML;
  * "energy"   : -LSE;
  * "sml"      : -T(S), S = (ML - mean_y) / std_y: the standardized max logit (Jung et al., ICCV 2021) as defined here,
                 with T boundary suppression followed by dilated smoothing. mean_c / std_c are the mean and population
                 standard deviation of ML over the fit pixels predicted as c; a class with fewer than 2 fit pixels or a
                 zero std uses those of all fit pixels. Suppression runs iterations i = 0 .. n-1 at width
                 r_i = r0 - i floor(r0 / n): a pixel whose (2 r_i + 1)^2 window, clipped to the image, holds another
                 prediction takes the mean of S over the non-boundary pixels of its clipped 3x3 neighbourhood (keeping
                 its value if there are none), every iteration reading the previous one's map. Smoothing is
                 sum g(a,b) S(p + d (a,b)) / sum g(a,b) over a, b in [-k/2, k/2], g = exp(-(a^2 + b^2) / 2 sigma^2),
                 taps outside the image dropped and the weights renormalised over the rest. fp64, emitted as fp32.
                 No parity with the published code is claimed: its padding conventions are not reproduced.
The post-processing, the class moments and the metrics run on csrc/anomaly.cu; ML and LSE come from the stats variant
of csrc/window.cu's scores kernel.

`AnomalyMeter` accumulates CUDA score maps and labels (1 = anomaly, 0 = inlier, ignore_index = void) and computes
AUROC, AP and FPR at 95 % TPR on the device (one radix sort, integer cumulative counts; sklearn's roc_auc_score and
average_precision_score, ties grouped).
"""
import math

import torch

from . import ops

__all__ = ["AnomalyScorer", "AnomalyMeter"]

KINDS = ("msp", "maxlogit", "energy", "sml")
_MAX_PIXELS = 2 ** 31 - 1          # the radix sort's limit on one segment


def _int_option(name, v):
    if isinstance(v, bool) or not isinstance(v, int):
        raise TypeError("AnomalyScorer: %s must be an int, got %s" % (name, type(v).__name__))
    return v


class AnomalyScorer:
    """Per-pixel anomaly scores of SlidingWindowPredictor(anomaly=...). The defaults are the Cityscapes setting reported
    for SML; `boundary_iterations=0` turns suppression off and `smooth_kernel=1` smoothing. `statistics`: None, or
    (mean, std), each [classes] (the result of `fit`, saved by the user)."""

    def __init__(self, kind="sml", statistics=None, boundary_width=4, boundary_iterations=4, smooth_kernel=7,
                 smooth_sigma=1.0, smooth_dilation=6):
        if kind not in KINDS:
            raise ValueError("AnomalyScorer: kind must be one of %s, got %r" % (", ".join(KINDS), kind))
        self.kind = kind
        self.boundary_width = _int_option("boundary_width", boundary_width)
        self.boundary_iterations = _int_option("boundary_iterations", boundary_iterations)
        self.smooth_kernel = _int_option("smooth_kernel", smooth_kernel)
        self.smooth_dilation = _int_option("smooth_dilation", smooth_dilation)
        if isinstance(smooth_sigma, bool) or not isinstance(smooth_sigma, (int, float)):
            raise TypeError("AnomalyScorer: smooth_sigma must be a number, got %s" % type(smooth_sigma).__name__)
        self.smooth_sigma = float(smooth_sigma)
        if self.boundary_iterations < 0:
            raise ValueError("AnomalyScorer: boundary_iterations must be >= 0")
        if self.boundary_iterations > 0 and self.boundary_width < 1:
            raise ValueError("AnomalyScorer: boundary_width must be >= 1 when boundary_iterations > 0")
        if self.smooth_kernel < 1 or self.smooth_kernel % 2 == 0 or self.smooth_kernel > 63:
            raise ValueError("AnomalyScorer: smooth_kernel must be odd and in 1..63, got %d" % self.smooth_kernel)
        if not (self.smooth_sigma > 0 and math.isfinite(self.smooth_sigma)):
            raise ValueError("AnomalyScorer: smooth_sigma must be finite and > 0")
        if self.smooth_dilation < 1:
            raise ValueError("AnomalyScorer: smooth_dilation must be >= 1")
        self.statistics = None if statistics is None else self._check_statistics(statistics)

    def __repr__(self):
        return ("AnomalyScorer(kind=%r, boundary_width=%d, boundary_iterations=%d, smooth_kernel=%d, smooth_sigma=%g, "
                "smooth_dilation=%d, fitted=%s)" % (self.kind, self.boundary_width, self.boundary_iterations,
                                                    self.smooth_kernel, self.smooth_sigma, self.smooth_dilation,
                                                    self.statistics is not None))

    @staticmethod
    def _check_statistics(statistics):
        try:
            mean, std = statistics
        except (TypeError, ValueError):
            raise TypeError("AnomalyScorer: statistics must be a (mean, std) pair") from None
        mean = torch.as_tensor(mean, dtype=torch.float64).detach().cpu().clone()
        std = torch.as_tensor(std, dtype=torch.float64).detach().cpu().clone()
        if mean.dim() != 1 or mean.shape != std.shape or mean.numel() == 0:
            raise ValueError("AnomalyScorer: statistics must be two 1-D [classes] sequences of equal length")
        if not (bool(torch.isfinite(mean).all()) and bool(torch.isfinite(std).all()) and bool((std > 0).all())):
            raise ValueError("AnomalyScorer: statistics must be finite, with every std > 0")
        return mean, std

    # ------------------------------------------------------------------------------------------- fitting
    def fit(self, predictor, images, base_size, scales):
        """Run `predictor` (a SlidingWindowPredictor, exact=False finish) over the float32 HWC `images` and set
        `self.statistics` = (mean, std), fp64 [classes] CPU tensors: per predicted class, the mean and population std
        of ML over the fit pixels (moments summed on the device). Returns self."""
        classes = predictor.classes
        moments = torch.zeros((3, classes), dtype=torch.float64, device=predictor.device)
        for image in images:
            total, pred = predictor._stats_total(image, base_size, scales)
            ops.anomaly_class_moments(pred, total[classes].contiguous(), moments)
        self.statistics = self.statistics_from_moments(moments.cpu())
        return self

    @staticmethod
    def statistics_from_moments(moments):
        """(mean, std) fp64 [C] of the fp64 [3, C] moments (sum ML, sum ML^2, count): population std, and the all-pixel
        mean / std for a class with fewer than 2 pixels or a zero std."""
        s, s2, n = (moments[i].double() for i in range(3))
        total = float(n.sum())
        if total < 2:
            raise ValueError("AnomalyScorer.fit: fewer than 2 fit pixels")
        g_mean = float(s.sum()) / total
        g_std = math.sqrt(max(float(s2.sum()) / total - g_mean * g_mean, 0.0))
        if not g_std > 0:
            raise ValueError("AnomalyScorer.fit: the max logit has zero variance over the fit pixels")
        safe = n.clamp(min=1)
        mean = s / safe
        std = (s2 / safe - mean * mean).clamp(min=0).sqrt()
        fallback = (n < 2) | (std == 0)
        mean = torch.where(fallback, torch.full_like(mean, g_mean), mean)
        std = torch.where(fallback, torch.full_like(std, g_std), std)
        return mean, std

    # ------------------------------------------------------------------------------------------- scoring
    def score_map(self, total, pred):
        """fp32 [h, w] CUDA anomaly map of a predictor's statistics total (fp64 [classes + 2, h, w]: the scale-averaged
        scores, ML, LSE) and its argmax `pred` (int64 [h, w])."""
        classes = total.shape[0] - 2
        if self.kind == "msp":
            return (1.0 - total[:classes].amax(0)).float()
        if self.kind == "maxlogit":
            return (-total[classes]).float()
        if self.kind == "energy":
            return (-total[classes + 1]).float()
        if self.statistics is None:
            raise ValueError("AnomalyScorer: kind='sml' needs statistics: pass them or call fit() first")
        mean, std = self.statistics
        if mean.numel() != classes:
            raise ValueError("AnomalyScorer: statistics have %d classes, the predictor %d" % (mean.numel(), classes))
        return ops.anomaly_sml(total[classes].contiguous(), pred, mean.to(total.device), std.to(total.device),
                               self.boundary_width,
                               self.boundary_iterations, self.smooth_kernel, self.smooth_sigma, self.smooth_dilation)


class AnomalyMeter:
    """Pixel-level AUROC, AP and FPR at 95 % TPR of anomaly maps. `update(score, label)` keeps a CUDA score map (compared
    in fp32) and its same-shaped int64 or uint8 CUDA label (1 = anomaly, 0 = inlier, ignore_index = void) on the device;
    `compute()` -> {"auroc", "ap", "fpr95", "positives", "negatives"}. Nothing crosses to the host before compute()."""

    def __init__(self, ignore_index=255):
        self.ignore_index = int(ignore_index)
        self.reset()

    def reset(self):
        self._scores, self._labels, self.count = [], [], 0

    def update(self, score, label):
        if not (torch.is_tensor(score) and torch.is_tensor(label)):
            raise TypeError("AnomalyMeter.update: score and label must be tensors")
        if not (score.is_cuda and label.is_cuda):
            raise ValueError("AnomalyMeter.update: score and label must be CUDA tensors")
        if not score.is_floating_point():
            raise TypeError("AnomalyMeter.update: score must be a floating-point tensor, got %s" % score.dtype)
        if label.dtype not in (torch.int64, torch.uint8):
            raise TypeError("AnomalyMeter.update: label must be int64 or uint8, got %s" % label.dtype)
        if score.shape != label.shape:
            raise ValueError("AnomalyMeter.update: score %s and label %s differ in shape"
                             % (tuple(score.shape), tuple(label.shape)))
        n = score.numel()
        if self.count + n > _MAX_PIXELS:
            raise ValueError("AnomalyMeter.update: more than 2^31 - 1 pixels in all (%d stored, %d more)"
                             % (self.count, n))
        self._scores.append(score.detach().to(torch.float32).reshape(-1).clone())
        self._labels.append(label.detach().reshape(-1).clone())
        self.count += n

    def compute(self):
        if self.count == 0:
            raise ValueError("AnomalyMeter.compute: no pixels")
        score = self._scores[0] if len(self._scores) == 1 else torch.cat(self._scores)
        dtypes = {l.dtype for l in self._labels}
        if len(dtypes) == 1:
            label = self._labels[0] if len(self._labels) == 1 else torch.cat(self._labels)
        else:
            label = torch.cat([l.to(torch.int64) for l in self._labels])
        out, info = ops.anomaly_metrics(score, label, self.ignore_index)
        auroc, ap, fpr95 = out.cpu().tolist()
        positives, negatives, errors = info.cpu().tolist()
        if errors & 1:
            raise ValueError("AnomalyMeter.compute: a label other than 0, 1 or ignore_index (%d)" % self.ignore_index)
        if errors & 2:
            raise ValueError("AnomalyMeter.compute: a non-finite score on a non-void pixel")
        if positives == 0 or negatives == 0:
            raise ValueError("AnomalyMeter.compute: needs anomaly and inlier pixels (%d positives, %d negatives)"
                             % (positives, negatives))
        return {"auroc": auroc, "ap": ap, "fpr95": fpr95, "positives": positives, "negatives": negatives}
