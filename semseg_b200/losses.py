"""Loss modules the networks accept as `criterion` besides nn.CrossEntropyLoss.

OhemCrossEntropyLoss is online hard-pixel mining: only the pixels the network is least sure of are trained on. With
the network's fused tail (functional.upsample_ce) it runs inside the same kernels as the default loss, graphed at every
zoom factor; called as a module (validate(), or the network's tail when the fused one does not apply) it runs the
zoom-1 form of those kernels on an NHWC copy of the logits. DiceLoss, the soft Dice loss alone or plus cross-entropy,
LovaszSoftmaxLoss, the Lovász-Softmax loss alone or plus cross-entropy, and FocalLoss, the softmax focal loss with
optional class weights, run the same way, and so does RMILoss, the Region Mutual Information loss with its BCE term. DistillationLoss adds a
pixel-wise distillation term from a teacher network that the student's training forward runs, and PseudoLabelLoss a
confidence-masked pseudo-label term on the unlabelled pixels; the teacher is a frozen network or the mean teacher of an
optim.ModelEMA. MixPseudoLabelLoss is that pseudo-label loss with CutMix or ClassMix: the teacher labels the clean
batch, the student learns on the mixed one. Each of the three teacher criteria takes `strong=` (augment.StrongAugment):
the student then learns on a strongly perturbed view of the batch the teacher sees. The two pseudo-label criteria take
`fp_weight=` too: UniMatch's feature perturbation, a second pass of the context module and classifier on the student's
channel-dropped layer4 features that learns the same pseudo-labels, and `streams=2`: UniMatch's dual-stream
perturbation, two strong views of every image, each with its own draws, in one student pass.
"""
import math

import torch
from torch import nn


class OhemCrossEntropyLoss(nn.Module):
    """Pixel OHEM cross-entropy, the sort-based definition of the HRNet / OCR code bases, for logits [N, C, H, W] and
    target [N, H, W]:

        valid = target != ignore_index and 0 <= target < C     (other out-of-range targets are skipped)
        p_t   = softmax(logits)[target],  nll = -log_softmax(logits)[target]        per valid pixel
        k     = min(min_kept, n_valid - 1)
        thr   = max(thresh, k-th smallest p_t over the valid pixels (0-based))
        kept  = valid and p_t < thr                                                  (strict)
        loss  = mean of nll over the kept pixels

    With no valid or no kept pixel the loss is 0 and every gradient is 0 (the fused tail's convention; torch's mean over
    nothing would be nan). The selection is exact: the k-th value is found by a radix select on the device, without a
    host synchronisation. Under DistributedDataParallel each rank mines its own pixels.

    `weight` (a 1-D float tensor of one weight per class, as nn.CrossEntropyLoss's) weights each kept pixel's nll by its
    target class's weight, as HRNet's OhemCrossEntropy does: the selection on p_t is unchanged and unweighted, and the
    loss is the plain mean of w_t * nll over the kept pixels (not divided by the sum of the weights). It is registered
    as a buffer like nn.CrossEntropyLoss's (moved by .cuda() / .to(), saved in the state_dict); without it there is no
    buffer. The native tail needs it contiguous fp32 on the logits' device.

    CUDA fp32 logits with at most 256 classes only: there is no CPU or library fallback."""

    def __init__(self, ignore_index=255, thresh=0.7, min_kept=100000, weight=None):
        super(OhemCrossEntropyLoss, self).__init__()
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        if isinstance(min_kept, bool) or not isinstance(min_kept, int):
            raise TypeError("min_kept must be an int, got %r" % (min_kept,))
        thresh = float(thresh)
        if not 0.0 <= thresh <= 1.0:
            raise ValueError("thresh must lie in [0, 1], got %r" % thresh)
        if not 0 <= min_kept < 2 ** 31:
            raise ValueError("min_kept must be a non-negative 32-bit int, got %r" % min_kept)
        if weight is not None:
            if not torch.is_tensor(weight) or not weight.is_floating_point():
                raise TypeError("weight must be a floating-point tensor or None, got %r" % (weight,))
            if weight.dim() != 1 or weight.numel() == 0:
                raise ValueError("weight must be 1-D with one entry per class, got shape %s" % (tuple(weight.shape),))
        self.ignore_index, self.thresh, self.min_kept = ignore_index, thresh, min_kept
        self.register_buffer("weight", weight)

    def extra_repr(self):
        s = "ignore_index=%d, thresh=%g, min_kept=%d" % (self.ignore_index, self.thresh, self.min_kept)
        return s if self.weight is None else s + ", weight=[%d]" % self.weight.numel()

    def forward(self, logits, target):
        from . import functional as SF
        if logits.dim() != 4 or target.dim() != 3 or target.shape != logits.shape[:1] + logits.shape[2:]:
            raise ValueError("OhemCrossEntropyLoss: logits [N, C, H, W] and target [N, H, W] expected, got %s and %s" %
                             (tuple(logits.shape), tuple(target.shape)))
        if logits.shape[1] > 256:
            raise ValueError("OhemCrossEntropyLoss: at most 256 classes (got %d); no fallback" % logits.shape[1])
        if not (logits.is_cuda and target.is_cuda):
            raise RuntimeError("OhemCrossEntropyLoss runs on the native CUDA kernels only (no CPU fallback); got %s, %s"
                               % (logits.device, target.device))
        if logits.dtype != torch.float32 or target.dtype != torch.int64:
            raise TypeError("OhemCrossEntropyLoss: fp32 logits and int64 target expected, got %s and %s" %
                            (logits.dtype, target.dtype))
        w = self.weight
        if w is not None and not (w.numel() == logits.shape[1] and w.dtype == torch.float32 and w.is_contiguous()
                                  and w.device == logits.device):
            raise ValueError("OhemCrossEntropyLoss: weight must be contiguous fp32 [%d] on %s (no fallback), got %s "
                             "[%d] on %s" % (logits.shape[1], logits.device, w.dtype, w.numel(), w.device))
        loss, _ = SF.upsample_ce(logits.permute(0, 2, 3, 1).contiguous(), target, self.ignore_index, 1, criterion=self)
        return loss


def _non_negative(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise TypeError("%s must be a number, got %r" % (name, v))
    v = float(v)
    if not (math.isfinite(v) and v >= 0.0):
        raise ValueError("%s must be finite and >= 0, got %r" % (name, v))
    return v


class DiceLoss(nn.Module):
    """Soft Dice loss from logits, optionally plus cross-entropy, for logits [N, C, H, W] and target [N, H, W]:

        valid  = target != ignore_index and 0 <= target < C     (other out-of-range targets are skipped)
        p      = softmax(logits) over C
        n_c    = #{valid pixels with target c},  I_c = sum over valid pixels of p_c [target = c]
        S_c    = sum over valid pixels of p_c, plus n_c
        dice_c = (2 I_c + smooth) / max(S_c + smooth, eps)
        loss   = (1/C) sum over the classes with n_c > 0 of (1 - dice_c) + ce_weight * CE

    CE is the mean cross-entropy over the valid pixels. The sums run over every pixel of every image of the call (per
    rank under DistributedDataParallel). Classes without a pixel add 0 but still count in 1/C. With no valid pixel the
    loss is 0 and every gradient is 0. This is segmentation_models_pytorch's DiceLoss(mode='multiclass',
    from_logits=True, smooth, eps, ignore_index), plus the CE term.

    With the network's fused tail (functional.upsample_ce) it runs inside the tail's kernels, graphed at every zoom
    factor; called as a module (validate()) it runs their zoom-1 form on an NHWC copy of the logits. CUDA fp32 logits
    with at most 256 classes only: there is no CPU or library fallback."""

    def __init__(self, ignore_index=255, smooth=0.0, eps=1e-7, ce_weight=0.0):
        super(DiceLoss, self).__init__()
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        self.ignore_index = ignore_index
        self.smooth = _non_negative("smooth", smooth)
        self.eps = _non_negative("eps", eps)
        self.ce_weight = _non_negative("ce_weight", ce_weight)

    def extra_repr(self):
        return "ignore_index=%d, smooth=%g, eps=%g, ce_weight=%g" % (self.ignore_index, self.smooth, self.eps,
                                                                      self.ce_weight)

    def forward(self, logits, target):
        from . import functional as SF
        if logits.dim() != 4 or target.dim() != 3 or target.shape != logits.shape[:1] + logits.shape[2:]:
            raise ValueError("DiceLoss: logits [N, C, H, W] and target [N, H, W] expected, got %s and %s" %
                             (tuple(logits.shape), tuple(target.shape)))
        if logits.shape[1] > 256:
            raise ValueError("DiceLoss: at most 256 classes (got %d); no fallback" % logits.shape[1])
        if not (logits.is_cuda and target.is_cuda):
            raise RuntimeError("DiceLoss runs on the native CUDA kernels only (no CPU fallback); got %s, %s"
                               % (logits.device, target.device))
        if logits.dtype != torch.float32 or target.dtype != torch.int64:
            raise TypeError("DiceLoss: fp32 logits and int64 target expected, got %s and %s" %
                            (logits.dtype, target.dtype))
        loss, _ = SF.upsample_ce(logits.permute(0, 2, 3, 1).contiguous(), target, self.ignore_index, 1, criterion=self)
        return loss


def _check_native_logits(name, logits, target):
    if logits.dim() != 4 or target.dim() != 3 or target.shape != logits.shape[:1] + logits.shape[2:]:
        raise ValueError("%s: logits [N, C, H, W] and target [N, H, W] expected, got %s and %s" %
                         (name, tuple(logits.shape), tuple(target.shape)))
    if logits.shape[1] > 256:
        raise ValueError("%s: at most 256 classes (got %d); no fallback" % (name, logits.shape[1]))
    if not (logits.is_cuda and target.is_cuda):
        raise RuntimeError("%s runs on the native CUDA kernels only (no CPU fallback); got %s, %s"
                           % (name, logits.device, target.device))
    if logits.dtype != torch.float32 or target.dtype != torch.int64:
        raise TypeError("%s: fp32 logits and int64 target expected, got %s and %s" % (name, logits.dtype, target.dtype))


class FocalLoss(nn.Module):
    """Softmax focal loss (Lin et al., ICCV 2017), for logits [N, C, H, W] and target [N, H, W]:

        valid = target != ignore_index and 0 <= target < C     (other out-of-range targets are skipped)
        p     = softmax(logits) over C,  p_t = p[target],  q = 1 - p_t,  nll = -log p_t
        l     = w_t * q^gamma * nll                             per valid pixel (w_t = 1 without `weight`)
        loss  = sum of l over the valid pixels / n_valid

    The mean is over the valid pixel count, not over the sum of the weights: a zero-weight class lowers the loss and
    leaves the denominator alone. q^gamma follows torch.pow (0^0 = 1), so gamma = 0 is the (weighted) cross-entropy
    summed and divided by n_valid; gamma is any finite float >= 0. With no valid pixel the loss is 0 and every gradient
    is 0. Under DistributedDataParallel each rank averages over its own pixels.

    `weight` is a 1-D float tensor of one weight per class, registered as a buffer like nn.CrossEntropyLoss's (moved by
    .cuda() / .to(), saved in the state_dict; without it there is no buffer). It gets no gradient. The native tail needs
    it contiguous fp32 on the logits' device and reads it on the device at every launch.

    With the network's fused tail (functional.upsample_ce) it runs inside the tail's kernels, graphed at every zoom
    factor; called as a module (validate()) it runs their zoom-1 form on an NHWC copy of the logits. CUDA fp32 logits
    with at most 256 classes only: there is no CPU or library fallback."""

    def __init__(self, gamma=2.0, weight=None, ignore_index=255):
        super(FocalLoss, self).__init__()
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        if weight is not None:
            if not torch.is_tensor(weight) or not weight.is_floating_point():
                raise TypeError("weight must be a floating-point tensor or None, got %r" % (weight,))
            if weight.dim() != 1 or weight.numel() == 0:
                raise ValueError("weight must be 1-D with one entry per class, got shape %s" % (tuple(weight.shape),))
        self.gamma = _non_negative("gamma", gamma)
        self.ignore_index = ignore_index
        self.register_buffer("weight", weight)

    def extra_repr(self):
        s = "gamma=%g, ignore_index=%d" % (self.gamma, self.ignore_index)
        return s if self.weight is None else s + ", weight=[%d]" % self.weight.numel()

    def forward(self, logits, target):
        from . import functional as SF
        _check_native_logits("FocalLoss", logits, target)
        w = self.weight
        if w is not None and not (w.numel() == logits.shape[1] and w.dtype == torch.float32 and w.is_contiguous()
                                  and w.device == logits.device):
            raise ValueError("FocalLoss: weight must be contiguous fp32 [%d] on %s (no fallback), got %s [%d] on %s" %
                             (logits.shape[1], logits.device, w.dtype, w.numel(), w.device))
        loss, _ = SF.upsample_ce(logits.permute(0, 2, 3, 1).contiguous(), target, self.ignore_index, 1, criterion=self)
        return loss


class _TeacherLoss(nn.Module):
    """What the criteria that learn from a teacher network share: the teacher, held outside the module tree, and
    `run_teacher`, its forward inside the student's training forward.

    `teacher` is a PSPNet or PSANet of this package, in eval mode, on the input's device, with the student's number of
    classes: a frozen network, or the `module` of an optim.ModelEMA (a mean teacher). It is held, not owned: it is not a
    submodule, so it stays out of the student's state_dict, modules(), .cuda() / .to(), convert_sync_batchnorm and DDP's
    buffer broadcast. It runs inside the student's training forward, before the student's stem, under torch.no_grad() in
    the student's precision mode, on the folded eval kernels; the criterion never modifies its parameters, running
    statistics or training flag, and no gradient reaches it or, through it, the input (with x.requires_grad, x.grad is
    the student's). A ModelEMA shadow changes after every `ema.update`: its operand slabs are re-packed at the top of
    every teacher forward (in one launch, part of the captured training step), and the graphed step is keyed on its
    tensors' addresses, not their versions, so it is captured once and replays each step with the current shadow.

    `strong` (an augment.StrongAugment, default None) gives the student a strong view of the batch: per training forward
    its uniforms are drawn after any mix draw and before the teacher forward, the teacher runs on the batch, and the
    student, both heads' losses and any mixing see the view (the targets are unchanged: the view moves no pixel).
    `last_strong()` returns {'image': the view before any mixing, 'uniforms': its draws} of the latest training forward,
    graphed or eager, as views that stay valid until the next forward. There is no gradient through the view: an input
    with requires_grad raises. strong=None changes nothing."""

    def __init__(self, teacher, ignore_index, strong=None):
        super(_TeacherLoss, self).__init__()
        from .augment import StrongAugment
        from .pspnet import PSPNet
        from .psanet import PSANet
        if not isinstance(teacher, (PSPNet, PSANet)):
            raise TypeError("teacher must be a semseg_b200 PSPNet or PSANet, got %s" % type(teacher).__name__)
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        if strong is not None and not isinstance(strong, StrongAugment):
            raise TypeError("strong must be an augment.StrongAugment or None, got %s" % type(strong).__name__)
        self.ignore_index = ignore_index
        self.strong = strong
        self._strong_state = None
        self.__dict__['_teacher'] = teacher      # held outside the module tree (see the class docstring)

    @property
    def teacher(self):
        return self.__dict__['_teacher']

    def __setattr__(self, name, value):
        # nn.Module.__setattr__ would register a module value as a child, past the read-only property
        if name in ('teacher', '_teacher'):
            raise AttributeError("%s: the teacher is fixed at construction; build a new criterion" %
                                 type(self).__name__)
        super(_TeacherLoss, self).__setattr__(name, value)

    def _strong_repr(self):
        return "" if self.strong is None else ", strong=%r" % (self.strong,)

    def last_strong(self):
        """{'image', 'uniforms'} of the latest training forward's strong view (None before the first one, or without
        `strong`)."""
        return None if self._strong_state is None else dict(self._strong_state)

    def strong_view(self, x, u):
        """The student's view of `x` from `strong.draw`'s uniforms `u`; remembered for last_strong()."""
        xs = self.strong(x, u)
        self._strong_state = {'image': xs, 'uniforms': u}
        return xs

    def run_teacher(self, x, classes):
        """The teacher's detached fp32 NHWC 1/8-resolution logits of the input batch `x` (NCHW), for a student with
        `classes` classes."""
        from . import functional as SF
        from . import graphs
        name = type(self).__name__
        teacher = self.teacher
        # the network and every layer whose mode changes the forward (the teacher's own criterion, a module that the
        # networks' default argument shares with every other network, does not take part)
        if teacher.training or any(m.training for m in teacher.modules()
                                   if isinstance(m, (nn.modules.batchnorm._BatchNorm, nn.modules.dropout._DropoutNd))):
            raise RuntimeError("%s: the teacher must be in eval mode (call teacher.eval())" % name)
        dev = next(teacher.parameters()).device
        if dev != x.device:
            raise RuntimeError("%s: the teacher is on %s, the input on %s (move the teacher yourself)" %
                               (name, dev, x.device))
        tc = teacher.cls[4].out_channels
        if tc != classes:
            raise ValueError("%s: the teacher has %d classes, the student %d" % (name, tc, classes))
        if getattr(teacher, "_sb_ema_shadow", False):
            # a mean teacher changes every step: its slabs are re-packed here, inside the captured step while capturing
            SF.prepack(teacher, force=graphs.capturing(), dgrad=False)
        with torch.no_grad(), SF.network_mode(False, False):
            return teacher._eval_logits_nhwc(x.detach())

    def _teacher_logits_nhwc(self, logits, teacher_logits):
        if teacher_logits.shape != logits.shape or teacher_logits.dtype != torch.float32 or \
                teacher_logits.device != logits.device:
            raise ValueError("%s: teacher_logits must be fp32 %s on %s like the logits, got %s %s on %s" %
                             (type(self).__name__, tuple(logits.shape), logits.device, teacher_logits.dtype,
                              tuple(teacher_logits.shape), teacher_logits.device))
        return teacher_logits.detach().permute(0, 2, 3, 1).contiguous()


class DistillationLoss(_TeacherLoss):
    """Pixel-wise knowledge distillation from a teacher network, plus cross-entropy. With s, t the student and
    teacher logits at the KD resolution, T the temperature, p = softmax(s/T) and q = softmax(t/T) over the classes and P
    the number of pixels at the KD resolution over all images of the call:

        KL   = (1/P) sum_pixels sum_c q_c (log q_c - log p_c)        (every pixel; the target plays no part)
        main = ce_weight * CE(student xZ, target; ignore_index, mean over valid pixels) + kd_weight * T^2 * KL
        aux  = plain CE of the aux head (ignore_index); the teacher has no aux counterpart, ce_weight does not scale it
        d main / d s_c at the KD resolution, KD part = kd_weight * T * (p_c - q_c) / P

    at='output': s and t after the same bilinear xZ upsample (align_corners) that the CE term uses, i.e. at the target's
    size; at='logits': the raw 1/8-resolution maps (as structured KD / CIRKD distil them). "Valid" is as in the other
    criteria: target != ignore_index and 0 <= target < C. Under DistributedDataParallel each rank holds its own teacher
    and averages over its own pixels.

    `teacher` is a frozen PSPNet or PSANet of this package or the `module` of an optim.ModelEMA, with the rules of
    _TeacherLoss (eval mode, the input's device, the student's classes; held outside the module tree; never modified).

    With the network's fused tail (functional.upsample_ce) it runs inside the tail's kernels, teacher forward and KL
    term graphed at every zoom factor. Called as a module, forward(logits, target, teacher_logits=None) takes NCHW logits
    at the target size: without teacher_logits it returns the student's mean cross-entropy (the validation loss
    validate() logs), with them (the same shape) `main` computed at that size. It runs the zoom-1 kernels on NHWC copies.
    CUDA fp32 logits with at most 256 classes only: there is no CPU or library fallback."""

    def __init__(self, teacher, temperature=1.0, kd_weight=1.0, ce_weight=1.0, ignore_index=255, at='output',
                 strong=None):
        super(DistillationLoss, self).__init__(teacher, ignore_index, strong)
        if not isinstance(at, str):
            raise TypeError("at must be 'output' or 'logits', got %r" % (at,))
        if at not in ('output', 'logits'):
            raise ValueError("at must be 'output' or 'logits', got %r" % (at,))
        temperature = _non_negative("temperature", temperature)
        if temperature <= 0.0:
            raise ValueError("temperature must be > 0, got %r" % temperature)
        self.temperature = temperature
        self.kd_weight = _non_negative("kd_weight", kd_weight)
        self.ce_weight = _non_negative("ce_weight", ce_weight)
        self.at = at

    def extra_repr(self):
        return "teacher=%s, temperature=%g, kd_weight=%g, ce_weight=%g, ignore_index=%d, at=%r" % (
            type(self.teacher).__name__, self.temperature, self.kd_weight, self.ce_weight, self.ignore_index,
            self.at) + self._strong_repr()

    def forward(self, logits, target, teacher_logits=None):
        from . import functional as SF
        _check_native_logits("DistillationLoss", logits, target)
        s = logits.permute(0, 2, 3, 1).contiguous()
        if teacher_logits is None:
            loss, _ = SF.upsample_ce(s, target, self.ignore_index, 1)
            return loss
        t = self._teacher_logits_nhwc(logits, teacher_logits)
        loss, _ = SF.upsample_ce(s, target, self.ignore_index, 1, criterion=self, teacher_logits=t)
        return loss


class PseudoLabelLoss(_TeacherLoss):
    """Confidence-masked pseudo-label cross-entropy from a teacher network (the self-training loss of FixMatch-style
    segmentation, UniMatch and U2PL), plus cross-entropy on the labelled pixels. With s, t the student and teacher
    logits after the same bilinear xZ upsample (align_corners) that the CE term uses, per output pixel:

        L    = {target in [0, C), target != ignore_index}       labelled pixels
        U    = {target == ignore_index}                          unlabelled pixels (an unlabelled image: all ignore)
        yhat = argmax_c t_c (first maximum, as torch.argmax),    conf = softmax(t)_yhat = 1 / sum_c exp(t_c - t_yhat)
        main = ce_weight (1/|L|) sum_L (lse(s) - s_target) + pl_weight (1/|U|) sum_{U, conf >= threshold} (lse(s) - s_yhat)
        aux  = plain CE of the aux head on L (ce_weight does not scale it)

    The pseudo-label term is averaged over |U|, every unlabelled pixel, not over the confident ones: UniMatch's
    normalisation, so that a teacher that grows more confident does not change the weight of each pixel. A term whose set
    is empty is 0 with an exactly zero gradient; a target outside [0, C) that is not ignore_index belongs to neither set.
    threshold 0 (or below) trains on every unlabelled pixel, a threshold above 1 on none. The mask and yhat are
    constants: no gradient flows through the teacher. Under DistributedDataParallel each rank averages over its own
    pixels.

    `teacher` is a frozen PSPNet or PSANet of this package or the `module` of an optim.ModelEMA (a mean teacher), with
    the rules of _TeacherLoss. It sees the student's input batch.

    With the network's fused tail (functional.upsample_ce) it runs inside the tail's kernels, teacher forward included,
    graphed at every zoom factor. Called as a module, forward(logits, target, teacher_logits=None) takes NCHW logits at the
    target size: without teacher_logits it returns the mean cross-entropy over L (the validation loss validate() logs),
    with them (the same shape) `main` computed at that size. CUDA fp32 logits with at most 256 classes only: there is no
    CPU or library fallback.

    `fp_weight` > 0 adds UniMatch's feature perturbation (Yang et al., CVPR 2023, its "FP" stream): the context module
    and classifier run a second time on the student's layer4 features after a channel dropout, and that prediction learns
    the same pseudo-labels. Per training forward of a PSPNet / PSANet, with f the student's layer4 output (of whatever
    the student sees: its strong view, mixed):

        u    = torch.rand(N, 2048) on the default CUDA generator, after the mix and strong draws, before the teacher
        s    = [u < 1 - fp_dropout] / (1 - fp_dropout)        per (image, channel); fp_dropout = 0 gives s = 1
        the context module and cls run once on cat(f, f * s) (2N images: every BatchNorm there takes batch statistics
        over the 2N, running statistics are updated once; cls's Dropout2d draws for all 2N) -> s_main, s_fp
        main = the main above of s_main + fp_weight (1/|U|) sum_{U, conf >= threshold} (lse(s_fp) - s_fp[yhat])
        aux, pred: unchanged (of the aux head and of s_main)

    U, yhat and conf are the pseudo-label term's (with mixing: the mixed target and the teacher map of each pixel's
    source image); labelled pixels get no FP term. The gradient reaching f is d[:N] + s * d[N:]; none flows through s or
    the teacher. `last_fp()` returns {'uniforms': u, 'scale': s} of the latest training forward, graphed or eager (None
    before the first one, and with fp_weight 0). fp_weight = 0 (the default) runs no draw and no second stream: the
    forward is the one without the option. validate(), eval mode and the teacher's forward never run the stream.
    UniMatch's (loss_x + 0.5 loss_s + 0.5 loss_fp) / 2 with one strong stream is ce_weight=0.5, pl_weight=0.25,
    fp_weight=0.25. Under DistributedDataParallel SyncBatchNorm sees 2N images per rank in the context module and cls
    (multi-GPU runs have not been made).

    `streams=2` is UniMatch's dual-stream perturbation: every image gets two strong views, each with its own draws, and
    both learn the same pseudo-labels. It needs `strong` (two views without it would be the same images; the CutMix /
    ClassMix criterion takes it without, its two mixes differ). Per training forward of a PSPNet / PSANet with input x
    [N,3,H,W] and target y, rows [0, N) of every [2N, .] draw belonging to stream 1 and rows [N, 2N) to stream 2:

        draws  in the one-stream order on the default CUDA generator, before the teacher: the mix uniforms
               torch.rand(2N, 5 [+ C]) (MixPseudoLabelLoss), the strong uniforms torch.rand(2N, 12), the FP uniforms
               torch.rand(N, 2048) (fp_weight > 0)
        teacher once, on the unmixed x (N images)
        view_k = mix_k(strong_k(x)), y_k = mix_k(y): each stream's strong view from its own uniform rows, each stream
                 mixed within itself (image n's partner is that stream's view of image (n + 1) mod N; ClassMix takes the
                 one teacher argmax and selects classes from the stream's own rows); without mixing y_k = y
        the whole student runs once on cat(view_1, view_2) (2N images: every BatchNorm takes statistics over the 2N,
        SyncBatchNorm 2N per rank; cls's Dropout2d draws for all 2N). With fp_weight > 0 only stream 1's layer4 features
        f_1 are perturbed: the context module and cls run on cat(f_1, f_2, f_1 * s) (3N images), one FP term
        main   = (main_1 + main_2) / 2 + fp_weight * FP,  main_k the main above of stream k's logits, y_k and teacher maps
                 (with mixing, of each pixel's source image), FP the term above on stream 1's logits, mask and target
        aux    = (aux_1 + aux_2) / 2;  pred = stream 1's argmax [N]

    With this, UniMatch's full loss (loss_x + 0.25 loss_s1 + 0.25 loss_s2 + 0.5 loss_fp) / 2 is ce_weight=0.5,
    pl_weight=0.25, fp_weight=0.25, the weights of the one-stream recipe. The accessors are stream-major: last_strong()
    holds 'image' [2N,3,H,W] and 'uniforms' [2N,12], MixPseudoLabelLoss.last_mix() 'mask' [2N,H,W], 'target'
    [2N,Ho,Wo] and 'uniforms' [2N, .]; last_fp() stays [N, 2048]. The student's activations are those of a 2N-image
    batch. streams=1 (the default) is the one-stream forward. Eval mode, validate(), the teacher's forward and the
    module form forward(logits, target, teacher_logits) are single-stream."""

    # two streams are two different views only through the strong view's draws (a mix criterion's boxes differ too)
    _streams_need_strong = True

    def __init__(self, teacher, threshold=0.95, pl_weight=1.0, ce_weight=1.0, ignore_index=255, strong=None,
                 fp_weight=0.0, fp_dropout=0.5, streams=1):
        super(PseudoLabelLoss, self).__init__(teacher, ignore_index, strong)
        if isinstance(threshold, bool) or not isinstance(threshold, (int, float)):
            raise TypeError("threshold must be a number, got %r" % (threshold,))
        if not math.isfinite(threshold):
            raise ValueError("threshold must be finite, got %r" % threshold)
        self.threshold = float(threshold)
        self.pl_weight = _non_negative("pl_weight", pl_weight)
        self.ce_weight = _non_negative("ce_weight", ce_weight)
        self.fp_weight = _non_negative("fp_weight", fp_weight)
        self.fp_dropout = _non_negative("fp_dropout", fp_dropout)
        if self.fp_dropout >= 1.0:
            raise ValueError("fp_dropout must lie in [0, 1), got %r" % fp_dropout)
        if isinstance(streams, bool):
            raise TypeError("streams must be the int 1 or 2, got %r" % (streams,))
        if not (isinstance(streams, int) and streams in (1, 2)):
            raise ValueError("streams must be the int 1 or 2, got %r" % (streams,))
        if streams == 2 and strong is None and self._streams_need_strong:
            raise ValueError("%s: streams=2 needs a strong view (strong=None would give two identical streams)" %
                             type(self).__name__)
        self.streams = streams
        self._fp_state = None

    def _fp_repr(self):
        return ", fp_weight=%g, fp_dropout=%g" % (self.fp_weight, self.fp_dropout) + \
            (", streams=2" if self.streams == 2 else "")

    def strong_streams(self, x, u):
        """The student's views of `x` from the strong uniforms `u` [streams * N, 12], stream-major: each stream's view
        from its own rows, concatenated along the batch; remembered for last_strong()."""
        if self.streams == 1:
            return self.strong_view(x, u)
        n = x.shape[0]
        xs = torch.cat([self.strong(x, u[k * n:(k + 1) * n]) for k in range(self.streams)])
        self._strong_state = {'image': xs, 'uniforms': u}
        return xs

    def extra_repr(self):
        return "teacher=%s, threshold=%g, pl_weight=%g, ce_weight=%g, ignore_index=%d" % (
            type(self.teacher).__name__, self.threshold, self.pl_weight, self.ce_weight,
            self.ignore_index) + self._fp_repr() + self._strong_repr()

    def last_fp(self):
        """{'uniforms', 'scale'} of the latest training forward's feature perturbation (None before the first one, or
        with fp_weight 0)."""
        return None if self._fp_state is None else dict(self._fp_state)

    def fp_draw(self, x, channels):
        """The per-(image, channel) factor s [N, channels] of the feature-perturbation stream from fresh uniforms of
        the default CUDA generator; remembered for last_fp()."""
        u = torch.rand((x.shape[0], channels), device=x.device)
        keep = 1.0 - self.fp_dropout
        s = (u < keep).float().div_(keep)
        self._fp_state = {'uniforms': u, 'scale': s}
        return s

    def fp_loss(self, logits, target, teacher_logits):
        """The feature-perturbation term alone, module form: fp_weight * the pseudo-label term of the perturbed stream's
        NCHW logits at the target size, with the teacher's logits of the same shape."""
        from . import functional as SF
        _check_native_logits(type(self).__name__, logits, target)
        t = self._teacher_logits_nhwc(logits, teacher_logits)
        loss, _ = SF.upsample_fp(logits.permute(0, 2, 3, 1).contiguous(), target, 1, self, t)
        return loss

    def forward(self, logits, target, teacher_logits=None):
        from . import functional as SF
        _check_native_logits("PseudoLabelLoss", logits, target)
        s = logits.permute(0, 2, 3, 1).contiguous()
        if teacher_logits is None:
            loss, _ = SF.upsample_ce(s, target, self.ignore_index, 1)
            return loss
        t = self._teacher_logits_nhwc(logits, teacher_logits)
        loss, _ = SF.upsample_ce(s, target, self.ignore_index, 1, criterion=self, teacher_logits=t)
        return loss


def _range_pair(name, v, upper):
    if not isinstance(v, (tuple, list)) or len(v) != 2 or \
            any(isinstance(a, bool) or not isinstance(a, (int, float)) for a in v):
        raise TypeError("%s must be a pair of numbers (lo, hi), got %r" % (name, v))
    lo, hi = float(v[0]), float(v[1])
    if not (math.isfinite(lo) and math.isfinite(hi) and 0.0 < lo <= hi <= upper):
        raise ValueError("%s must satisfy 0 < lo <= hi%s, got %r" % (name, " <= %g" % upper if upper < math.inf else "",
                                                                    v))
    return lo, hi


class MixPseudoLabelLoss(PseudoLabelLoss):
    """PseudoLabelLoss with mixed-sample perturbation: CutMix (French et al., BMVC 2020, the CutMix-Seg recipe; the box
    of UniMatch) or ClassMix (Olsson et al., WACV 2021; DACS). The teacher labels the clean batch, the student learns
    those labels, mixed the same way, on the mixed batch. Per training forward of a PSPNet / PSANet with this criterion,
    with input x [N,3,H,W] and target y [N,Ho,Wo]:

        u    = torch.rand(N, 5 [+ C for ClassMix]) on the device's default CUDA generator, before the teacher forward
               (graph-safe like Dropout2d: seeded runs reproduce, a graphed step equals the eager one); image n is mixed
               iff u[n, 0] < p, with its partner pi(n) = (n + 1) mod N (N = 1: itself, so mixing changes nothing)
        M    = the mask on the input grid, 1 where a pixel comes from the partner:
               'cutmix'  : one box per mixed image, area (area_lo + (area_hi - area_lo) u1) H W and aspect ratio
                           ratio_lo + (ratio_hi - ratio_lo) u2, placed by u3 (row) and u4 (column); computed in fp64
                           as include/semseg_b200.h semseg_mix_apply states (UniMatch's box without its retry loop)
               'classmix': A[m] = the teacher's argmax of image m after the x8 upsample to the input grid; the ceil(k/2)
                           of its k present classes with the smallest (u[m, 5 + c], c) are pasted: M(n) = 1 where
                           A[pi(n)] is one of them (at most 256 classes)
        x_m  = M ? x[pi(n)] : x[n]                        y_m = the same mix of y at the target pixels' input positions
        main = PseudoLabelLoss's main of (student(x_m), y_m), each pixel's pseudo-label and confidence from the teacher
               of its source image (the teacher runs on the unmixed x)
        aux  = plain CE of the aux head on y_m;  pred = the student's argmax on x_m

    `p` in [0, 1] (UniMatch: 0.5), `area` = (lo, hi) with 0 < lo <= hi <= 1, `ratio` = (lo, hi) with 0 < lo <= hi; the
    other arguments (fp_weight and fp_dropout included: the feature-perturbation stream runs on the mixed batch's
    features) and the teacher's rules are PseudoLabelLoss's. Labelled and unlabelled images share the batch: an
    unlabelled image has an all-ignore_index target, and the mixed target carries each pixel's own label or ignore.

    `last_mix()` returns {'mask': uint8 [N,H,W], 'target': y_m, 'uniforms': u} of the latest training forward, graphed
    or eager, as views that stay valid until the next forward. The trainer's logged training mIoU compares `pred` with
    the unmixed target; score against last_mix()['target'] instead. There is no gradient through the mixing: an input
    with requires_grad raises. Called as a module, forward(logits, target, teacher_logits=None) is PseudoLabelLoss's.

    With the network's fused tail the mixing, the mixed pseudo-label loss and the teacher forward run on native kernels
    (csrc/mix.cu and csrc/tail.cu), graphed at every zoom factor; where the fused tail does not apply (a target wider
    than its kernels stage), the mixing stays native and the teacher's upsampled maps are mixed with torch.where. Under
    DistributedDataParallel each rank mixes its own batch (multi-GPU runs have not been made).

    `streams=2` (PseudoLabelLoss's dual-stream perturbation) needs no strong view here: each stream mixes within itself
    from its own uniform rows, so the two streams differ by their boxes or class sets."""

    _streams_need_strong = False

    def __init__(self, teacher, mix='cutmix', p=0.5, area=(0.02, 0.4), ratio=(0.3, 1 / 0.3), threshold=0.95,
                 pl_weight=1.0, ce_weight=1.0, ignore_index=255, strong=None, fp_weight=0.0, fp_dropout=0.5,
                 streams=1):
        super(MixPseudoLabelLoss, self).__init__(teacher, threshold, pl_weight, ce_weight, ignore_index, strong,
                                                 fp_weight, fp_dropout, streams)
        if not isinstance(mix, str):
            raise TypeError("mix must be 'cutmix' or 'classmix', got %r" % (mix,))
        if mix not in ('cutmix', 'classmix'):
            raise ValueError("mix must be 'cutmix' or 'classmix', got %r" % (mix,))
        p = _non_negative("p", p)
        if p > 1.0:
            raise ValueError("p must lie in [0, 1], got %r" % p)
        self.mix = mix
        self.p = p
        self.area = _range_pair("area", area, 1.0)
        self.ratio = _range_pair("ratio", ratio, math.inf)
        self._mix_state = None

    def extra_repr(self):
        return "teacher=%s, mix=%r, p=%g, area=(%g, %g), ratio=(%g, %g), threshold=%g, pl_weight=%g, ce_weight=%g, " \
               "ignore_index=%d" % (type(self.teacher).__name__, self.mix, self.p, self.area[0], self.area[1],
                                    self.ratio[0], self.ratio[1], self.threshold, self.pl_weight, self.ce_weight,
                                    self.ignore_index) + self._fp_repr() + self._strong_repr()

    def last_mix(self):
        """{'mask', 'target', 'uniforms'} of the latest training forward (None before the first one)."""
        return None if self._mix_state is None else dict(self._mix_state)

    def draw(self, x, classes):
        """The forward's uniforms, drawn before the teacher runs: [streams * N, 5] (CutMix) or [streams * N,
        5 + classes] (ClassMix), stream-major."""
        name = type(self).__name__
        if x.requires_grad:
            raise RuntimeError("%s: there is no gradient through the mixing; the input must not require grad" % name)
        if not x.is_cuda or x.dtype != torch.float32 or x.dim() != 4:
            raise TypeError("%s: the input must be a CUDA fp32 [N, C, H, W] tensor, got %s %s on %s" %
                            (name, x.dtype, tuple(x.shape), x.device))
        if self.mix == 'classmix' and classes > 256:
            raise ValueError("%s: ClassMix needs at most 256 classes, got %d" % (name, classes))
        return torch.rand((self.streams * x.shape[0], 5 + (classes if self.mix == 'classmix' else 0)),
                          device=x.device)

    def mix_batch(self, x, y, u, t_logits, zoom):
        """(x_m, y_m, mask) from the input, target, `draw`'s uniforms and the teacher's NHWC logits of the unmixed
        input; remembered for last_mix(). With two streams `x` holds both streams' views ([2N], or the N images
        themselves for both without a strong view) and each stream is mixed within itself from its own uniform rows:
        x_m, y_m and the mask are [2N], stream-major."""
        from . import ops
        if y.dtype != torch.int64:
            raise TypeError("%s: int64 target expected, got %s" % (type(self).__name__, y.dtype))
        n = y.shape[0]
        x, y = x.contiguous(), y.contiguous()
        amap = present = None
        if self.mix == 'classmix':
            amap, present = ops.mix_argmax_x8(t_logits)
        outs = []
        for k in range(self.streams):
            rows = slice(k * n, (k + 1) * n)
            u_k = u[rows]
            sel = ops.mix_select(u_k, present, t_logits.shape[-1]) if amap is not None else None
            outs.append(ops.mix_apply(self.mix, x[rows] if x.shape[0] > n else x, y, u_k, self.p, self.area,
                                      self.ratio, zoom, amap, sel))
        mask, xm, ym = outs[0] if len(outs) == 1 else (torch.cat(t) for t in zip(*outs))
        self._mix_state = {'mask': mask, 'target': ym, 'uniforms': u}
        return xm, ym, mask


class LovaszSoftmaxLoss(nn.Module):
    """Lovász-Softmax loss (Berman, Triki, Blaschko, CVPR 2018), the standard surrogate for mIoU, optionally plus
    cross-entropy, for logits [N, C, H, W] and target [N, H, W]:

        valid    = target != ignore_index and 0 <= target < C     (other out-of-range targets are skipped)
        p        = softmax(logits) over C
        segment  = one class over every valid pixel of the call, or one (image, class) pair with per_image
        fg_i     = [target_i = c],  e_i = |fg_i - p_ic|,  G = sum fg_i                         per segment
        sort the valid pixels by e descending, ties by flat pixel index (torch.sort(stable=True) over Berman's order)
        J_k      = 1 - (G - A_k) / (G + B_k),  J_0 = 0   (A_k, B_k: fg / bg pixels among the first k)
        loss_seg = sum_k e_(k) (J_k - J_{k-1})
        loss     = mean of loss_seg over the considered segments + ce_weight * CE

    classes='present' considers the segments with G > 0; classes='all' every class (an absent class scores
    max_i p_ic). per_image=True averages each image's segments and then the N images; an image with no valid pixel adds 0
    and still counts in 1/N. CE is the mean cross-entropy over the valid pixels. With no valid pixel the loss is 0 and
    every gradient is 0. The counts are integers and J is float64, so the loss stays exact past 2^24 pixels per segment.
    Under DistributedDataParallel each rank computes its own loss. The gradient is autograd's with the sort order held
    fixed (torch's |x| backward: a pixel with e = 0 gets no Lovász gradient).

    With the network's fused tail (functional.upsample_ce) it runs inside the tail's kernels with an on-device segmented
    radix sort, graphed at every zoom factor; called as a module (validate()) it runs their zoom-1 form on an NHWC copy
    of the logits. CUDA fp32 logits with at most 256 classes only: there is no CPU or library fallback. The forward needs
    about 16 C bytes per output pixel of transient workspace and keeps 4 C bytes per output pixel for the backward."""

    def __init__(self, ignore_index=255, classes='present', per_image=False, ce_weight=0.0):
        super(LovaszSoftmaxLoss, self).__init__()
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        if not isinstance(classes, str):
            raise TypeError("classes must be 'present' or 'all', got %r" % (classes,))
        if classes not in ('present', 'all'):
            raise ValueError("classes must be 'present' or 'all', got %r" % (classes,))
        if not isinstance(per_image, bool):
            raise TypeError("per_image must be a bool, got %r" % (per_image,))
        self.ignore_index = ignore_index
        self.classes = classes
        self.per_image = per_image
        self.ce_weight = _non_negative("ce_weight", ce_weight)

    def extra_repr(self):
        return "ignore_index=%d, classes=%r, per_image=%s, ce_weight=%g" % (self.ignore_index, self.classes,
                                                                            self.per_image, self.ce_weight)

    def forward(self, logits, target):
        from . import functional as SF
        if logits.dim() != 4 or target.dim() != 3 or target.shape != logits.shape[:1] + logits.shape[2:]:
            raise ValueError("LovaszSoftmaxLoss: logits [N, C, H, W] and target [N, H, W] expected, got %s and %s" %
                             (tuple(logits.shape), tuple(target.shape)))
        if logits.shape[1] > 256:
            raise ValueError("LovaszSoftmaxLoss: at most 256 classes (got %d); no fallback" % logits.shape[1])
        if not (logits.is_cuda and target.is_cuda):
            raise RuntimeError("LovaszSoftmaxLoss runs on the native CUDA kernels only (no CPU fallback); got %s, %s"
                               % (logits.device, target.device))
        if logits.dtype != torch.float32 or target.dtype != torch.int64:
            raise TypeError("LovaszSoftmaxLoss: fp32 logits and int64 target expected, got %s and %s" %
                            (logits.dtype, target.dtype))
        loss, _ = SF.upsample_ce(logits.permute(0, 2, 3, 1).contiguous(), target, self.ignore_index, 1, criterion=self)
        return loss


class RMILoss(nn.Module):
    """Region Mutual Information loss (Zhao, Wang, Cai, "Region Mutual Information Loss for Semantic Segmentation",
    NeurIPS 2019) with its sigmoid BCE term, optionally plus cross-entropy, for logits z [N, C, H, W] and target
    t [N, H, W]:

        v      = t != ignore_index and 0 <= t < C          (other targets are not valid, as in DiceLoss)
        y_c    = [t = c] v,  s_c = sigmoid(z_c),  q_c = s_c v + 1e-6
        BCE    = sum over pixels and classes of v (softplus(z_c) - y_c z_c) / (n_valid + 1)
        Y, Q   = avg_pool(y, 4, stride 4), avg_pool(q, 4, stride 4)     (Hp = H // 4, Wp = W // 4, no padding)
        a_k, b_k = the 3x3 neighbourhoods of pooled cell k of Y and Q (9-vectors), K = (Hp - 2)(Wp - 2) of them
        S_aa, S_bb, S_ab = sums over k of the centred a a', b b', a b'   (float64, 9x9)
        r[n,c] = 1/2 log det(S_aa - S_ab (S_bb + pos_alpha I)^-1 S_ab' + pos_alpha I)
        RMI    = sum over c of (mean over n of r[n,c]) / 9
        loss   = bce_weight * BCE + (1 - bce_weight) * RMI + ce_weight * CE

    CE is the mean cross-entropy over the valid pixels. The sums run over the pixels of the call (per rank under
    DistributedDataParallel). Pixels in the last H mod 4 rows and W mod 4 columns reach BCE and CE but not RMI. With no
    valid pixel BCE is 0, r = 9/2 log(pos_alpha) and every gradient is 0. This is the authors' released code in its
    default configuration; its pooling (average, 4), radius (3), lambda_way (1) and clip (1e-6) are fixed, which lets
    the kernels specialise on them.

    With the network's fused tail (functional.upsample_ce) it runs inside the tail's kernels, graphed at every zoom
    factor, without the full-resolution logits; called as a module (validate()) it runs their zoom-1 form on an NHWC
    copy of the logits. H and W must be at least 12 (three pooled cells). CUDA fp32 logits with at most 256 classes
    only: there is no CPU or library fallback. The forward keeps 8 C bytes per pooled cell (the pooled Y and Q maps) for
    the backward."""

    def __init__(self, ignore_index=255, bce_weight=0.5, pos_alpha=5e-4, ce_weight=0.0):
        super(RMILoss, self).__init__()
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        bce_weight = _non_negative("bce_weight", bce_weight)
        if bce_weight > 1.0:
            raise ValueError("bce_weight must lie in [0, 1], got %r" % bce_weight)
        pos_alpha = _non_negative("pos_alpha", pos_alpha)
        if pos_alpha <= 0.0:
            raise ValueError("pos_alpha must be > 0, got %r" % pos_alpha)
        self.ignore_index = ignore_index
        self.bce_weight = bce_weight
        self.pos_alpha = pos_alpha
        self.ce_weight = _non_negative("ce_weight", ce_weight)

    def extra_repr(self):
        return "ignore_index=%d, bce_weight=%g, pos_alpha=%g, ce_weight=%g" % (self.ignore_index, self.bce_weight,
                                                                              self.pos_alpha, self.ce_weight)

    def forward(self, logits, target):
        from . import functional as SF
        if logits.dim() == 4 and (logits.shape[2] < 12 or logits.shape[3] < 12):
            raise ValueError("RMILoss: H and W must be at least 12 (three 4x4 pooled cells), got %dx%d" %
                             (logits.shape[2], logits.shape[3]))
        _check_native_logits("RMILoss", logits, target)
        loss, _ = SF.upsample_ce(logits.permute(0, 2, 3, 1).contiguous(), target, self.ignore_index, 1, criterion=self)
        return loss
