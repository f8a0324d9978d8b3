"""float64 torch statement of the entropy-loss contract (semseg_b200/losses.py EntropyLoss, include/semseg_b200.h), the
checker of the entropy and Tent tests.

    L = {target in [0, C), target != ignore_index},  U = {target == ignore_index}
    p = softmax(s),  lse = logsumexp(s),  H = lse - sum_c p_c s_c = -sum_c p_c log p_c
    loss = ce_weight (1/|L|) sum_L (lse - s_target) + ent_weight (1/|U|) sum_U H
    dloss/ds_c = ce_weight/|L| (p_c - [c = t]) on L,   -ent_weight/|U| p_c (log p_c + H) on U

`entropy_definition` is the definition written the plain way, for autograd; `entropy_loss` gives the gradient in closed
form; `entropy_tail` puts the align_corners upsample of the fused tail in front and returns the gradient at the
low-resolution maps."""
import torch
import torch.nn.functional as F


def _sets(target, c, ignore_index):
    lab = (target != ignore_index) & (target >= 0) & (target < c)
    unl = target == ignore_index
    return lab, unl, torch.where(lab, target, torch.zeros_like(target))


def entropy_definition(logits, target, ent_weight=1.0, ce_weight=1.0, ignore_index=255):
    """The contract as one would write it in PyTorch: logits [N, C, H, W] (float64, may require grad) -> loss."""
    x = logits.double()
    lab, unl, t = _sets(target, x.shape[1], ignore_index)
    logp = torch.log_softmax(x, dim=1)
    ce = -logp.gather(1, t.unsqueeze(1)).squeeze(1)
    ent = -(logp.exp() * logp).sum(1)
    nl, nu = int(lab.sum()), int(unl.sum())
    return ce_weight * (ce * lab).sum() / max(nl, 1) + ent_weight * (ent * unl).sum() / max(nu, 1)


def entropy_loss(logits, target, ent_weight=1.0, ce_weight=1.0, ignore_index=255):
    """logits [N, C, H, W], target [N, H, W] int64 -> (loss, |L|, |U|, H [N, H, W], dloss/dlogits [N, C, H, W]), all
    float64 (the counts as ints); the gradient is the closed form above."""
    x = logits.detach().double()
    c = x.shape[1]
    lab, unl, t = _sets(target, c, ignore_index)
    logp = torch.log_softmax(x, dim=1)
    p = logp.exp()
    ent = -(p * logp).sum(1)
    nl, nu = int(lab.sum()), int(unl.sum())
    ce = -logp.gather(1, t.unsqueeze(1)).squeeze(1)
    loss = ce_weight * (ce * lab).sum() / max(nl, 1) + ent_weight * (ent * unl).sum() / max(nu, 1)
    onehot = F.one_hot(t, c).permute(0, 3, 1, 2).double()
    g_l = (ce_weight / max(nl, 1)) * (p - onehot) * lab.unsqueeze(1)
    g_u = (-ent_weight / max(nu, 1)) * p * (logp + ent.unsqueeze(1)) * unl.unsqueeze(1)
    return loss, nl, nu, ent, g_l + g_u


def entropy_tail(logits_nhwc, target, zoom, ent_weight=1.0, ce_weight=1.0, ignore_index=255):
    """The fused tail's contract: fp32 / fp64 NHWC logits [N, h, w, C] -> F.interpolate(align_corners=True) to
    zoom*(h-1)+1 x zoom*(w-1)+1 in float64 -> entropy_loss. Returns (loss, |L|, |U|, H, dloss/dlogits_nhwc), the
    closed-form gradient carried back through the (linear) upsample."""
    lr = logits_nhwc.detach().double().clone().requires_grad_(True)
    n, h, w, _ = lr.shape
    x = lr.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    loss, nl, nu, ent, grad = entropy_loss(x, target, ent_weight, ce_weight, ignore_index)
    (dl,) = torch.autograd.grad(x, lr, grad)
    return loss, nl, nu, ent, dl
