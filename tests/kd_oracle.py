"""float64 torch statement of the distillation contract (include/semseg_b200.h semseg_upsample_kd_*, semseg_b200/losses.py
DistillationLoss), the checker of the distillation tests.

`kd_loss` states the definition directly with F.interpolate (align_corners), log_softmax, the KL and the cross-entropy;
`kd_grad` is the closed-form gradient of the KL term that the kernels implement."""
import torch
import torch.nn.functional as F


def upsampled(logits_nhwc, zoom):
    """fp32 NHWC [N,h,w,C] -> float64 NCHW logits after the align-corners x`zoom` upsample (none at zoom 1)."""
    n, h, w, _ = logits_nhwc.shape
    x = logits_nhwc.double().permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    return x


def kl_term(s, t, temperature):
    """KL = (1/P) sum_pixels sum_c q_c (log q_c - log p_c), p = softmax(s/T), q = softmax(t/T) over dim 1 of NCHW maps
    (float64; P = N*H*W)."""
    lp = F.log_softmax(s.double() / temperature, dim=1)
    lq = F.log_softmax(t.double() / temperature, dim=1)
    n, _, h, w = s.shape
    return (lq.exp() * (lq - lp)).sum() / (n * h * w)


def ce_term(x, target, ignore_index=255):
    """Mean cross-entropy over the valid pixels (target != ignore_index, 0 <= target < C); 0 when none is valid."""
    c = x.shape[1]
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    if not bool(valid.any()):
        return x.sum() * 0.0
    t = torch.where(valid, target, torch.full_like(target, -100))
    return F.cross_entropy(x.double(), t, ignore_index=-100)


def kd_loss(s_nhwc, t_nhwc, target, zoom, temperature=1.0, kd_weight=1.0, ce_weight=1.0, ignore_index=255, at="output"):
    """main = ce_weight * CE(student xZ, target) + kd_weight * T^2 * KL, KL at the target's size (at='output') or on
    the raw maps (at='logits'). s_nhwc may require grad; the teacher is a constant. -> (main, KL)."""
    x = upsampled(s_nhwc, zoom)
    if at == "output":
        s_kd, t_kd = x, upsampled(t_nhwc.detach(), zoom)
    else:
        s_kd, t_kd = upsampled(s_nhwc, 1), upsampled(t_nhwc.detach(), 1)
    kl = kl_term(s_kd, t_kd, temperature)
    return ce_weight * ce_term(x, target, ignore_index) + kd_weight * temperature ** 2 * kl, kl


def kd_grad(s, t, temperature, kd_weight=1.0):
    """d(kd_weight T^2 KL)/ds = kd_weight T (p - q) / P for NCHW float64 maps at the KD resolution."""
    n, _, h, w = s.shape
    p = torch.softmax(s.double() / temperature, dim=1)
    q = torch.softmax(t.double() / temperature, dim=1)
    return kd_weight * temperature * (p - q) / (n * h * w)
