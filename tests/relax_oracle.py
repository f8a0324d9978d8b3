"""float64 torch statement of the boundary label relaxation contract (semseg_b200/losses.py BoundaryRelaxationLoss,
include/semseg_b200.h), the checker of the relaxation tests.

    valid_j = target_j != ignore_index and 0 <= target_j < C
    S_i     = {target_j : valid_j, j in the (2 border + 1)^2 window of i, clipped to the image}     (valid i)
    p = softmax(v),  R_i = sum_{c not in S_i} p_c,  l_i = -log(1 - R_i),  omega_i = mean of w over S_i
    loss = sum_valid omega l / D,  D = sum_valid omega  (0 when D = 0)
    dl_i/dv_c = p_c - [c in S_i] p_c / (1 - R_i)

`relax_sets` builds S as a multi-hot map: the masked one-hot of the target through a border-radius max-pool (the pool's
padding adds no class). `relax_definition` writes the loss the naive way, for autograd; `relax_loss` takes l_i as
-log1p(-R_i) while R_i < 1/2 (log of the set's mass past it) and gives the gradient in closed form, the in-set term as
-p_c R / (1 - R); `relax_tail` puts the align_corners upsample of the fused tail in front and returns the gradient at
the low-resolution maps."""
import torch
import torch.nn.functional as F


def relax_sets(target, c, border, ignore_index=255):
    """target [N, H, W] int64 -> (valid [N, H, W] bool, S [N, C, H, W] bool, False at pixels that are not valid)."""
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    t = torch.where(valid, target, torch.zeros_like(target))
    onehot = F.one_hot(t, c).permute(0, 3, 1, 2).double() * valid.unsqueeze(1)
    if border > 0:
        onehot = F.max_pool2d(onehot, 2 * border + 1, stride=1, padding=border)
    return valid, (onehot > 0) & valid.unsqueeze(1)


def _omega(s, valid, weight):
    c = s.shape[1]
    w = torch.ones(c, dtype=torch.float64, device=s.device) if weight is None else weight.double().to(s.device)
    cnt = s.sum(1).clamp(min=1).double()
    return torch.where(valid, (s.double() * w.view(1, c, 1, 1)).sum(1) / cnt, torch.zeros_like(cnt))


def relax_definition(logits, target, border=1, weight=None, ignore_index=255):
    """The contract as one would write it in PyTorch: logits [N, C, H, W] (float64, may require grad) -> loss."""
    x = logits.double()
    valid, s = relax_sets(target, x.shape[1], border, ignore_index)
    lse_s = torch.logsumexp(x.masked_fill(~s, float("-inf")), dim=1)
    pix = torch.where(valid, torch.logsumexp(x, dim=1) - lse_s, torch.zeros_like(lse_s))
    om = _omega(s, valid, weight)
    d = om.sum()
    return (om * pix).sum() / d if d > 0 else (om * pix).sum() * 0.0


def relax_loss(logits, target, border=1, weight=None, ignore_index=255):
    """logits [N, C, H, W], target [N, H, W] int64 -> (loss, D, dloss/dlogits [N, C, H, W]), all float64."""
    x = logits.detach().double()
    valid, s = relax_sets(target, x.shape[1], border, ignore_index)
    logp = torch.log_softmax(x, dim=1)
    p = logp.exp()
    log_r = torch.logsumexp(logp.masked_fill(s, float("-inf")), dim=1)
    r = log_r.exp().clamp(max=1.0)
    log_ps = torch.logsumexp(logp.masked_fill(~s, float("-inf")), dim=1)
    nll = torch.where(r < 0.5, -torch.log1p(-r), -log_ps)
    nll = torch.where(valid, nll, torch.zeros_like(nll))
    om = _omega(s, valid, weight)
    d = float(om.sum())
    if d == 0.0:
        return torch.zeros((), dtype=torch.float64), 0.0, torch.zeros_like(x)
    log_q = torch.where(valid, log_r - log_ps, torch.zeros_like(log_r))   # log(R / (1 - R))
    g = torch.where(s, -(logp + log_q.unsqueeze(1)).exp(), p) * (om * valid).unsqueeze(1)
    return (om * nll).sum() / d, d, g / d


def relax_tail(logits_nhwc, target, zoom, border=1, weight=None, ignore_index=255):
    """The fused tail's contract: fp32 / fp64 NHWC logits [N, h, w, C] -> F.interpolate(align_corners=True) to
    zoom*(h-1)+1 x zoom*(w-1)+1 in float64 -> relax_loss. Returns (loss, D, dloss/dlogits_nhwc), the closed-form
    gradient carried back through the (linear) upsample."""
    lr = logits_nhwc.detach().double().clone().requires_grad_(True)
    n, h, w, _ = lr.shape
    x = lr.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    loss, d, grad = relax_loss(x, target, border, weight, ignore_index)
    (dl,) = torch.autograd.grad(x, lr, grad)
    return loss, d, dl
