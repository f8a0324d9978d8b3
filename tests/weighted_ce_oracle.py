"""float64 torch statement of the class-weighted, label-smoothed cross-entropy contract and of weighted OHEM
(include/semseg_b200.h, semseg_b200/losses.py), the checker of the weighted cross-entropy tests."""
import torch

from tests.ohem_oracle import ohem_ce


def weighted_ce(logits, target, weight=None, ignore_index=255, label_smoothing=0.0):
    """logits [N, C, H, W] (computed in float64; may require grad), target [N, H, W] int64 -> (loss, D).

        valid     = target != ignore_index and 0 <= target < C
        loss_pix  = (1-eps) w_t (lse - v_t) + (eps/C) sum_c w_c (lse - v_c)       valid pixels only
        D         = sum over the valid pixels of w_t
        loss      = sum loss_pix / D, and 0 (with a zero gradient) when D = 0"""
    x = logits.double()
    c = x.shape[1]
    w = torch.ones(c, dtype=torch.float64, device=x.device) if weight is None else weight.double().to(x.device)
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    t = torch.where(valid, target, torch.zeros_like(target))
    nlogp = -torch.log_softmax(x, dim=1)                                     # lse - v_c
    wt = w[t] * valid
    nll_t = nlogp.gather(1, t.unsqueeze(1)).squeeze(1)
    smooth = (nlogp * w.view(1, c, 1, 1)).sum(1)
    eps = float(label_smoothing)
    loss_pix = ((1 - eps) * w[t] * nll_t + (eps / c) * smooth) * valid
    d = wt.sum()
    if float(d) == 0.0:
        return (loss_pix * 0.0).sum(), d
    return loss_pix.sum() / d, d


def weighted_ohem_ce(logits, target, weight=None, ignore_index=255, thresh=0.7, min_kept=100000, kept=None):
    """OHEM with class weights (HRNet's OhemCrossEntropy): the selection of tests/ohem_oracle.py, unweighted, and the
    loss the plain mean of w_t * nll over the kept pixels -> (loss, kept mask, thr, p_t). `kept` as in ohem_ce."""
    x = logits.double()
    c = x.shape[1]
    _, own, thr, pt = ohem_ce(x.detach(), target, ignore_index, thresh, min_kept)
    mask = own if kept is None else kept
    w = torch.ones(c, dtype=torch.float64, device=x.device) if weight is None else weight.double().to(x.device)
    t = torch.where(mask, target, torch.zeros_like(target))
    nll = -torch.log_softmax(x, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
    n_k = int(mask.sum())
    loss = (w[t] * nll * mask).sum() / max(n_k, 1)
    return loss, own, thr, pt
