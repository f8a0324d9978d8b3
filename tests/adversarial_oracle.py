"""Oracles of the adversarial attack (semseg_b200/adversarial.py, csrc/adversarial.cu, the SegPGD tail of csrc/tail.cu).

  * segpgd_tail: the SegPGD loss and its closed-form gradient in float64 from fp32 NHWC logits, the upsample written as
    ATen's align_corners bilinear interpolation and its adjoint;
  * box / step / start: the projected sign step and the random start as the same formula in torch fp32, from
    constants computed in float64 and rounded to fp32 once — the kernels must match these bit for bit;
  * lambdas: SegPGD's schedule."""
import numpy as np
import torch
import torch.nn.functional as F


def lambdas(steps):
    return [(t - 1) / (2.0 * steps) for t in range(1, steps + 1)]


def upsample(logits_nhwc, zoom):
    """fp NHWC [N,h,w,C] -> NCHW at zoom * (h-1) + 1 (no interpolation at zoom 1)."""
    n, h, w, _ = logits_nhwc.shape
    x = logits_nhwc.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    return x


def segpgd_weights(v, target, ignore_index, lam):
    """Per-pixel weights [N,Ho,Wo] of the upsampled logits `v` (NCHW): 1 - lam where the first-maximum argmax hits the
    target, lam elsewhere, 0 where the pixel is not valid; and the validity mask."""
    c = v.shape[1]
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    pred = v.argmax(1)                  # the first maximal index
    w = torch.where(pred == target, torch.full_like(v[:, 0], 1.0 - lam), torch.full_like(v[:, 0], lam))
    return torch.where(valid, w, torch.zeros_like(w)), valid


def segpgd_tail(logits, target, zoom, lam, ignore_index=255):
    """-> (loss, n_valid, dloss/dlogits NHWC), float64, from the fp32 NHWC `logits`; the gradient in closed form:
    w (p_c - [c = t]) / n_valid at each output pixel, folded back through the upsample's adjoint."""
    l64 = logits.detach().double().cpu().requires_grad_(True)
    t = target.detach().cpu()
    v = upsample(l64, zoom)
    w, valid = segpgd_weights(v.detach(), t, ignore_index, lam)
    n_valid = int(valid.sum())
    tc = torch.where(valid, t, torch.zeros_like(t))
    lsm = torch.log_softmax(v.detach(), 1)
    nll = -lsm.gather(1, tc.unsqueeze(1)).squeeze(1)
    if n_valid == 0:
        return torch.zeros((), dtype=torch.float64), 0, torch.zeros_like(l64.detach())
    loss = (w * nll).sum() / n_valid
    dv = lsm.exp() - F.one_hot(tc, v.shape[1]).permute(0, 3, 1, 2).double()
    dv = dv * (w / n_valid).unsqueeze(1)
    (dl,) = torch.autograd.grad(v, l64, dv)
    return loss, n_valid, dl


def box(eps, alpha, mean, std):
    """(step, eps, lo, hi) fp32 [3] each: computed in float64, rounded to fp32 once."""
    m, s = np.asarray(mean, np.float64), np.asarray(std, np.float64)
    vals = (alpha / s, eps / s, (0.0 - m) / s, (255.0 - m) / s)
    return tuple(torch.from_numpy(v.astype(np.float32)) for v in vals)


def _c(t, ref):
    return t.to(ref.device).view(1, 3, 1, 1)


def step(x, g, x0, consts):
    """One projected sign step in torch fp32: v = x + a sign(g); the eps-ball, then the pixel box."""
    a, e, lo, hi = (_c(t, x) for t in consts)
    v = x + a * torch.sign(g)
    v = torch.minimum(torch.maximum(v, x0 - e), x0 + e)
    return torch.minimum(torch.maximum(v, lo), hi)


def start(x0, u, consts):
    """The random start in torch fp32 from uniforms u."""
    _, e, lo, hi = (_c(t, x0) for t in consts)
    v = x0 + e * (2 * u - 1)
    v = torch.minimum(torch.maximum(v, x0 - e), x0 + e)
    return torch.minimum(torch.maximum(v, lo), hi)
