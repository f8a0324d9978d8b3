"""float64 torch statement of the class-incremental (MiB) contract (include/semseg_b200.h semseg_upsample_ce_unbiased_*
and semseg_upsample_unkd_*, semseg_b200/losses.py IncrementalLoss), the checker of the incremental tests.

`unce` and `unkd` state the definitions with logsumexp over class subsets; `unce_grad` and `unkd_grad` are the closed-form
gradients the kernels implement; `incremental_loss` is the whole main loss at either `at`."""
import torch

from tests.kd_oracle import upsampled


def _valid(target, c, ignore_index):
    return (target != ignore_index) & (target >= 0) & (target < c)


def unce(x, target, c_old, ignore_index=255):
    """Mean unbiased cross-entropy of NCHW logits x over the valid pixels; 0 when none is valid."""
    x = x.double()
    c = x.shape[1]
    valid = _valid(target, c, ignore_index)
    lse_all = torch.logsumexp(x, 1)
    lse_old = torch.logsumexp(x[:, :c_old], 1)
    tc = torch.where(valid, target, torch.zeros_like(target)).clamp(0, c - 1)
    s_t = x.gather(1, tc.unsqueeze(1)).squeeze(1)
    l = torch.where(tc < c_old, lse_all - lse_old, lse_all - s_t)
    n = int(valid.sum())
    if n == 0:
        return x.sum() * 0.0
    return torch.where(valid, l, torch.zeros_like(l)).sum() / n


def unce_grad(x, target, c_old, ignore_index=255):
    """d unce / d x for NCHW float64 logits."""
    x = x.double()
    c = x.shape[1]
    valid = _valid(target, c, ignore_index)
    n = int(valid.sum())
    if n == 0:
        return torch.zeros_like(x)
    p = torch.softmax(x, 1)
    old = torch.zeros_like(x)
    old[:, :c_old] = torch.softmax(x[:, :c_old], 1)
    tc = torch.where(valid, target, torch.zeros_like(target)).clamp(0, c - 1)
    is_old = (tc < c_old).unsqueeze(1).double()
    onehot = torch.nn.functional.one_hot(tc, c).permute(0, 3, 1, 2).double()
    g = p - is_old * old - (1 - is_old) * onehot
    return g * valid.unsqueeze(1).double() / n


def _subsets(s, c_old):
    c = s.shape[1]
    b = [0] + list(range(c_old, c))
    return torch.logsumexp(s, 1), torch.logsumexp(s[:, b], 1), b


def unkd(s, t, c_old, alpha=1.0):
    """Mean unbiased distillation over every pixel of NCHW student s [N, C] and teacher t [N, C_old] maps."""
    s, t = s.double(), t.double()
    lse_all, lse_b, _ = _subsets(s, c_old)
    q = torch.softmax(alpha * t, 1)
    k = q[:, 0] * (lse_b - lse_all) + (q[:, 1:] * (s[:, 1:c_old] - lse_all.unsqueeze(1))).sum(1)
    return -(k / c_old).mean()


def unkd_grad(s, t, c_old, alpha=1.0):
    """d unkd / d s for NCHW float64 maps."""
    s, t = s.double(), t.double()
    n, c, h, w = s.shape
    lse_all, lse_b, b = _subsets(s, c_old)
    q = torch.softmax(alpha * t, 1)
    g = torch.softmax(s, 1)
    g[:, 1:c_old] -= q[:, 1:]
    g[:, b] -= q[:, :1] * torch.exp(s[:, b] - lse_b.unsqueeze(1))
    return g / (c_old * n * h * w)


def incremental_loss(s_nhwc, t_nhwc, target, zoom, c_old, alpha=1.0, kd_weight=10.0, ce_weight=1.0, ignore_index=255,
                     at="output"):
    """main = ce_weight * unce(student xZ) + kd_weight * unkd at the target's size (at='output') or on the raw maps
    (at='logits'); s_nhwc may require grad, the teacher is a constant. -> (main, unce, unkd)."""
    x = upsampled(s_nhwc, zoom)
    if at == "output":
        s_kd, t_kd = x, upsampled(t_nhwc.detach(), zoom)
    else:
        s_kd, t_kd = upsampled(s_nhwc, 1), upsampled(t_nhwc.detach(), 1)
    ce = unce(x, target, c_old, ignore_index)
    kd = unkd(s_kd, t_kd, c_old, alpha)
    return ce_weight * ce + kd_weight * kd, ce, kd
