"""float64 torch statements of the Dice (+ cross-entropy) contract (include/semseg_b200.h, semseg_b200/losses.py
DiceLoss), the checker of the Dice tests.

`dice_ce` states the definition directly; `dice_ce_smp` states it again the way segmentation_models_pytorch's
multiclass DiceLoss structures it (one-hot target, masks, sums over dims (0, 2)); `dice_ce_grad` is the closed-form
gradient the kernels implement."""
import torch
import torch.nn.functional as F


def upsampled(logits_nhwc, zoom):
    """fp32 NHWC [N,h,w,C] -> float64 NCHW logits after the align-corners x`zoom` upsample (none at zoom 1)."""
    n, h, w, _ = logits_nhwc.shape
    x = logits_nhwc.double().permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    return x


def _valid(target, c, ignore_index):
    return (target != ignore_index) & (target >= 0) & (target < c)


def dice_ce(logits, target, ignore_index=255, smooth=0.0, eps=1e-7, ce_weight=0.0):
    """logits [N, C, H, W] (computed in float64; may require grad), target [N, H, W] int64 -> (loss, I, S, n), the
    last three per class:

        valid  = target != ignore_index and 0 <= target < C
        n_c    = #{valid, t = c},  I_c = sum_valid p_c [t = c],  S_c = sum_valid p_c + n_c
        loss   = (1/C) sum_{n_c > 0} (1 - (2 I_c + smooth) / max(S_c + smooth, eps)) + ce_weight * CE
        CE     = mean over the valid pixels of lse - v_t, 0 when none is valid"""
    x = logits.double()
    c = x.shape[1]
    valid = _valid(target, c, ignore_index)
    t = torch.where(valid, target, torch.zeros_like(target))
    p = torch.softmax(x, dim=1)
    vm = valid.unsqueeze(1).double()
    hot = (torch.arange(c, device=x.device).view(1, c, 1, 1) == t.unsqueeze(1)).double() * vm
    n = hot.sum((0, 2, 3))
    inter = (p * hot).sum((0, 2, 3))
    s = (p * vm).sum((0, 2, 3)) + n
    dice = (2 * inter + smooth) / torch.clamp(s + smooth, min=eps)
    loss = torch.where(n > 0, 1 - dice, torch.zeros_like(dice)).sum() / c
    nv = int(valid.sum())
    if ce_weight != 0.0 and nv > 0:
        nll = -torch.log_softmax(x, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
        loss = loss + ce_weight * (nll * valid).sum() / nv
    return loss, inter.detach(), s.detach(), n.detach()


def dice_ce_smp(logits, target, ignore_index=255, smooth=0.0, eps=1e-7, ce_weight=0.0):
    """The same loss written as segmentation_models_pytorch's DiceLoss(mode='multiclass', from_logits=True) writes it:
    [N, C, HW] probabilities and a one-hot [N, C, HW] target, both masked, soft Dice over dims (0, 2), absent classes
    masked out of the mean; plus ce_weight * F.cross_entropy(ignore_index) over the valid pixels."""
    x = logits.double()
    bs, c = x.shape[:2]
    y_true = target.reshape(bs, -1)
    y_pred = x.log_softmax(dim=1).exp().reshape(bs, c, -1)
    mask = _valid(y_true, c, ignore_index)
    y_pred = y_pred * mask.unsqueeze(1)
    y_true = F.one_hot((y_true * mask).long(), c).permute(0, 2, 1) * mask.unsqueeze(1)
    y_true = y_true.type_as(y_pred)
    intersection = torch.sum(y_pred * y_true, dim=(0, 2))
    cardinality = torch.sum(y_pred + y_true, dim=(0, 2))
    scores = (2.0 * intersection + smooth) / (cardinality + smooth).clamp_min(eps)
    loss = (1.0 - scores) * (y_true.sum((0, 2)) > 0).to(scores.dtype)
    loss = loss.mean()
    if ce_weight != 0.0 and bool(mask.any()):
        t = torch.where(mask, y_true.argmax(1), torch.full_like(y_true.argmax(1), -100)).view_as(target)
        loss = loss + ce_weight * F.cross_entropy(x, t, ignore_index=-100)
    return loss


def dice_ce_grad(logits, target, ignore_index=255, smooth=0.0, eps=1e-7, ce_weight=0.0):
    """Closed-form d loss / d logits (float64 [N, C, H, W]) of dice_ce:

        alpha_c = 2 m_c / (C D_c),  beta_c = m_c (2 I_c + smooth) / (C D_c^2)  (0 where S_c + smooth < eps)
        G_i     = sum_c p_ic beta_c - p_it alpha_t
        dL/dz   = p_ic (beta_c + lam - G_i) - [c = t_i] (p_ic alpha_c + lam),  lam = ce_weight / n_valid
    for valid pixels, 0 elsewhere (m_c = [n_c > 0], D_c = max(S_c + smooth, eps))."""
    x = logits.detach().double()
    c = x.shape[1]
    _, inter, s, n = dice_ce(x, target, ignore_index, smooth, eps, ce_weight)
    valid = _valid(target, c, ignore_index)
    t = torch.where(valid, target, torch.zeros_like(target))
    p = torch.softmax(x, dim=1)
    m = (n > 0).double()
    d = torch.clamp(s + smooth, min=eps)
    alpha = 2 * m / (c * d)
    beta = m * (2 * inter + smooth) / (c * d * d) * (s + smooth >= eps).double()
    nv = int(valid.sum())
    lam = ce_weight / nv if nv > 0 else 0.0
    hot = (torch.arange(c, device=x.device).view(1, c, 1, 1) == t.unsqueeze(1)).double()
    pt = p.gather(1, t.unsqueeze(1))
    g = (p * beta.view(1, c, 1, 1)).sum(1, keepdim=True) - pt * alpha[t].unsqueeze(1)
    grad = p * (beta.view(1, c, 1, 1) + lam - g) - hot * (p * alpha.view(1, c, 1, 1) + lam)
    return grad * valid.unsqueeze(1).double()
