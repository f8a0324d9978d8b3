"""float64 torch statement of the OHEM cross-entropy contract (semseg_b200/losses.py), the checker of the OHEM tests."""
import torch


def ohem_ce(logits, target, ignore_index=255, thresh=0.7, min_kept=100000, kept=None):
    """logits [N, C, H, W] (any float dtype, computed in float64; may require grad), target [N, H, W] int64 ->
    (loss, kept mask, thr, p_t). p_t is float64 and meaningful on the valid pixels only. `kept` given: the loss over that
    mask instead of the contract's own (to compare losses and gradients when a kernel's kept set differs from the
    oracle's only at pixels tied with the threshold)."""
    x = logits.double()
    c = x.shape[1]
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    t = torch.where(valid, target, torch.zeros_like(target))        # gather needs an index in [0, C) everywhere
    logp = torch.log_softmax(x, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
    pt = logp.detach().exp()
    n_v = int(valid.sum())
    if n_v == 0:
        thr = float(thresh)
    else:
        k = min(min_kept, n_v - 1)
        thr = max(float(thresh), float(pt[valid].sort().values[k]))
    own = valid & (pt < thr)
    mask = own if kept is None else kept
    n_k = int(mask.sum())
    loss = -(logp * mask).sum() / max(n_k, 1)                       # 0 (and a zero gradient) when nothing is kept
    return loss, own, thr, pt
