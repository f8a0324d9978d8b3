"""float64 torch statement of the focal-loss contract (semseg_b200/losses.py FocalLoss, include/semseg_b200.h), the
checker of the focal tests.

    valid = target != ignore_index and 0 <= target < C
    p = softmax(v),  q = 1 - p_t,  nll = -log p_t,  l = w_t q^gamma nll,  loss = sum_valid l / n_valid
    dl/dv_c = w_t M (p_c - [c = t]),   M = q^gamma + gamma p_t q^(gamma-1) nll = q^(gamma-1) (q + gamma p_t nll)

`focal_definition` is the definition written the naive way, for autograd; `focal_loss` evaluates q as the softmax mass
off the target and nll as -log1p(-q), so both keep their relative accuracy as p_t -> 1, and gives the gradient in closed
form; `focal_tail` puts the align_corners upsample of the fused tail in front and returns the gradient at the
low-resolution maps."""
import torch
import torch.nn.functional as F


def _valid(target, c, ignore_index):
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    return valid, torch.where(valid, target, torch.zeros_like(target))


def _weights(weight, c, device):
    return torch.ones(c, dtype=torch.float64, device=device) if weight is None else weight.double().to(device)


def focal_definition(logits, target, gamma=2.0, weight=None, ignore_index=255):
    """The contract as one would write it in PyTorch: logits [N, C, H, W] (float64, may require grad) -> loss."""
    x = logits.double()
    c = x.shape[1]
    valid, t = _valid(target, c, ignore_index)
    logp_t = torch.log_softmax(x, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
    w = _weights(weight, c, x.device)
    pix = w[t] * torch.pow(1.0 - logp_t.exp(), gamma) * -logp_t
    n_valid = int(valid.sum())
    return (pix * valid).sum() / max(n_valid, 1)


def focal_loss(logits, target, gamma=2.0, weight=None, ignore_index=255):
    """logits [N, C, H, W], target [N, H, W] int64 -> (loss, n_valid, dloss/dlogits [N, C, H, W]), all float64; the
    gradient is the closed form above, with torch.pow's 0^0 = 1: at q = 0, l = 0 and M = [gamma = 0]."""
    x = logits.detach().double()
    c = x.shape[1]
    gamma = float(gamma)
    valid, t = _valid(target, c, ignore_index)
    logp = torch.log_softmax(x, dim=1)
    onehot = F.one_hot(t, c).permute(0, 3, 1, 2).bool()
    q = torch.logsumexp(logp.masked_fill(onehot, float("-inf")), dim=1).exp().clamp(max=1.0)
    logp_t = logp.gather(1, t.unsqueeze(1)).squeeze(1)
    nll = torch.where(q < 0.5, -torch.log1p(-q), -logp_t)
    p_t = logp_t.exp()
    w = _weights(weight, c, x.device)[t]
    pos = q > 0
    qs = torch.where(pos, q, torch.ones_like(q))
    qg = torch.where(pos, qs.pow(gamma), torch.full_like(q, 1.0 if gamma == 0.0 else 0.0))
    m = torch.where(pos, qs.pow(gamma - 1.0) * (qs + gamma * p_t * nll), qg)
    n_valid = int(valid.sum())
    loss = (w * qg * nll * valid).sum() / max(n_valid, 1)
    grad = (w * m * valid).unsqueeze(1) * (logp.exp() - onehot.double()) / max(n_valid, 1)
    return loss, n_valid, grad


def focal_tail(logits_nhwc, target, zoom, gamma=2.0, weight=None, ignore_index=255):
    """The fused tail's contract: fp32 / fp64 NHWC logits [N, h, w, C] -> F.interpolate(align_corners=True) to
    zoom*(h-1)+1 x zoom*(w-1)+1 in float64 -> focal_loss. Returns (loss, n_valid, dloss/dlogits_nhwc), the closed-form
    gradient carried back through the (linear) upsample."""
    lr = logits_nhwc.detach().double().clone().requires_grad_(True)
    n, h, w, _ = lr.shape
    x = lr.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    loss, n_valid, grad = focal_loss(x, target, gamma, weight, ignore_index)
    (dl,) = torch.autograd.grad(x, lr, grad)
    return loss, n_valid, dl
