"""float64 torch statement of the pseudo-label contract (include/semseg_b200.h semseg_upsample_pl_*, semseg_b200/losses.py
PseudoLabelLoss), the checker of the mean-teacher tests.

`pl_loss` states the definition directly with F.interpolate (align_corners), the teacher's argmax and confidence and the
two cross-entropy terms; `pl_grad` is the closed-form gradient the kernels implement, w_p (softmax(s) - onehot(y_p)) at
the target's size. Both take the pseudo-labels and the confidence mask from `effective`, or from a caller that holds
them fixed (the kernel's own, where the teacher's top-2 margin or conf - threshold lies within fp32 error)."""
import torch

from tests.kd_oracle import upsampled


def pl_definition(s_nhwc, t_nhwc, target, zoom, threshold, pl_weight=1.0, ce_weight=1.0, ignore_index=255):
    """main = ce_weight (1/|L|) sum_L (lse - s_target) + pl_weight (1/|U|) sum_{U, conf >= threshold} (lse - s_yhat),
    written out with log_softmax (a term whose set is empty is 0)."""
    x = upsampled(s_nhwc, zoom)
    t = upsampled(t_nhwc.detach(), zoom)
    c = x.shape[1]
    logp = torch.log_softmax(x, dim=1)
    lab = (target != ignore_index) & (target >= 0) & (target < c)
    unl = target == ignore_index
    yhat = t.argmax(1)                       # torch.argmax: the first maximum
    conf = torch.softmax(t, dim=1).gather(1, yhat.unsqueeze(1)).squeeze(1)
    nll_t = -logp.gather(1, target.clamp(0, c - 1).unsqueeze(1)).squeeze(1)
    nll_y = -logp.gather(1, yhat.unsqueeze(1)).squeeze(1)
    ce = nll_t[lab].sum() / int(lab.sum()) if bool(lab.any()) else x.sum() * 0.0
    keep = unl & (conf >= threshold)
    pl = nll_y[keep].sum() / int(unl.sum()) if bool(unl.any()) else x.sum() * 0.0
    return ce_weight * ce + pl_weight * pl


def effective(t_nhwc, target, zoom, threshold, pl_weight=1.0, ce_weight=1.0, ignore_index=255):
    """(effective target int64 [N,H,W], weight float64 [N,H,W], conf float64 [N,H,W]) of the definition: the target on
    the labelled pixels, the teacher's argmax (first maximum) on the unlabelled pixels with conf >= threshold, -1
    elsewhere; weights ce_weight / |L|, pl_weight / |U| and 0."""
    t = upsampled(t_nhwc.detach(), zoom)
    c = t.shape[1]
    lab = (target != ignore_index) & (target >= 0) & (target < c)
    unl = target == ignore_index
    yhat = t.argmax(1)
    conf = 1.0 / torch.exp(t - t.gather(1, yhat.unsqueeze(1))).sum(1)
    conf_u = unl & (conf >= threshold)
    eff = torch.full_like(target, -1)
    eff[lab] = target[lab]
    eff[conf_u] = yhat[conf_u]
    n_l, n_u = int(lab.sum()), int(unl.sum())
    wt = torch.zeros(target.shape, dtype=torch.float64)
    wt[lab] = ce_weight / n_l if n_l else 0.0
    wt[conf_u] = pl_weight / n_u if n_u else 0.0
    return eff, wt, conf


def pl_loss(s_nhwc, eff, wt, zoom):
    """sum_p w_p (lse(s)_p - s_p[eff_p]) over the pixels with eff >= 0: ce_weight * CE over L + pl_weight * the masked
    pseudo-label CE over U, for the weights of `effective`. s_nhwc may require grad."""
    x = upsampled(s_nhwc, zoom)
    sel = eff >= 0
    lse = torch.logsumexp(x, dim=1)
    picked = x.gather(1, eff.clamp(min=0).unsqueeze(1)).squeeze(1)
    return (wt.to(x.device)[sel] * (lse - picked)[sel]).sum()


def pl_grad(s_nhwc, eff, wt, zoom):
    """Closed form: d pl_loss / d s at the target's size, w_p (p_c - [c = eff_p]), taken back to the maps through the
    adjoint of the upsample."""
    sd = s_nhwc.detach().double().requires_grad_(True)
    x = upsampled(sd, zoom)
    p = torch.softmax(x.detach(), dim=1)
    onehot = torch.zeros_like(p)
    sel = eff >= 0
    onehot.scatter_(1, eff.clamp(min=0).unsqueeze(1), 1.0)
    g = wt.to(p.device).unsqueeze(1) * (p - onehot) * sel.unsqueeze(1)
    (gm,) = torch.autograd.grad(x, sd, g)
    return gm
