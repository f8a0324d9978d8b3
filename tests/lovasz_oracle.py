"""float64 statements of the Lovász-Softmax (+ cross-entropy) contract (include/semseg_b200.h, semseg_b200/losses.py
LovaszSoftmaxLoss), the checker of the Lovász tests.

`lovasz` is the numpy oracle: stable order, integer counts, float64 J, and the closed-form gradient the kernels
implement; it can take the sort order of each segment from outside (the kernel's own keys), so that near-ties that
fp32 and fp64 errors order differently do not count as errors. `lovasz_torch` states the loss the way Berman's
reference code does (torch.sort, cumsum, a dot product per class) in float64, for autograd."""
import numpy as np
import torch


def valid_mask(target, c, ignore_index):
    return (target != ignore_index) & (target >= 0) & (target < c)


def softmax64(logits):
    x = np.asarray(logits, dtype=np.float64)
    m = x.max(axis=1, keepdims=True)
    ex = np.exp(x - m)
    return ex / ex.sum(axis=1, keepdims=True)


def lovasz_weights(fg_sorted):
    """g_k = J_k - J_{k-1} of one segment from its fg flags in sorted order: integer counts, float64 J, J_0 = 0."""
    fg = np.asarray(fg_sorted, dtype=np.int64)
    g_all = int(fg.sum())
    a = np.cumsum(fg)
    k = np.arange(1, fg.size + 1, dtype=np.int64)
    b = k - a
    j = 1.0 - (g_all - a).astype(np.float64) / (g_all + b).astype(np.float64)
    return np.diff(np.concatenate([[0.0], j]))


def lovasz(logits, target, ignore_index=255, classes="present", per_image=False, ce_weight=0.0, orders=None):
    """logits [N, C, H, W] (float64-able), target [N, H, W] int -> (loss, dlogits [N, C, H, W], info) in float64.

    orders: None (np.argsort(-e, kind='stable') over the flat valid pixels), or a dict {(scope, c): flat pixel indices
    in sorted order} for every considered segment (scope = 0, or the image with per_image). info holds the per-segment
    weights and G, the valid count, gamma = w g_k sign(p - fg) [C, P] and `terms` [N, C, H, W], the sum of the
    magnitudes of the terms that make up each gradient element."""
    x = np.asarray(logits, dtype=np.float64)
    t = np.asarray(target).astype(np.int64)
    n, c, h, w = x.shape
    p = softmax64(x)
    hw = h * w
    pf = p.transpose(1, 0, 2, 3).reshape(c, -1)
    tf = t.reshape(-1)
    vf = valid_mask(tf, c, ignore_index)
    scopes = [np.arange(n * hw)] if not per_image else [np.arange(i * hw, (i + 1) * hw) for i in range(n)]
    gamma = np.zeros((c, n * hw))
    weight = np.zeros((c, n * hw))
    total = 0.0
    seg_info = {}
    for si, scope in enumerate(scopes):
        idx = scope[vf[scope]]
        if idx.size == 0:
            continue                                    # adds 0, still counts in 1/N
        segs = [k for k in range(c) if classes == "all" or bool((tf[idx] == k).any())]
        wgt = 1.0 / (len(segs) * len(scopes))
        for k in segs:
            if orders is None:
                e = np.abs((tf[idx] == k).astype(np.float64) - pf[k, idx])
                order = idx[np.argsort(-e, kind="stable")]
            else:
                order = np.asarray(orders[(si, k)], dtype=np.int64)
            fg = (tf[order] == k)
            e = np.abs(fg.astype(np.float64) - pf[k, order])
            g = lovasz_weights(fg)
            total += wgt * float(np.dot(e, g))
            gamma[k, order] = wgt * g * np.sign(pf[k, order] - fg)
            weight[k, order] = wgt * np.abs(g)
            seg_info[(si, k)] = (wgt, int(fg.sum()))
    nv = int(vf.sum())
    ce, lam = 0.0, 0.0
    if nv > 0:
        xf = x.transpose(1, 0, 2, 3).reshape(c, -1)
        m = xf.max(axis=0)
        lse = m + np.log(np.exp(xf - m).sum(axis=0))                   # log-softmax: finite where p_t underflows
        iv = np.nonzero(vf)[0]
        ce = float((lse[iv] - xf[tf[iv], iv]).mean())
        lam = ce_weight / nv
    loss = total + ce_weight * ce
    hot = np.zeros_like(pf)
    hot[tf[vf], np.nonzero(vf)[0]] = 1.0
    gsum = (pf * gamma).sum(axis=0, keepdims=True)
    grad = (pf * (gamma - gsum) + lam * (pf - hot)) * vf[None, :]
    grad = grad.reshape(c, n, h, w).transpose(1, 0, 2, 3)
    # the magnitude of the terms each dlogits element sums before they cancel, whatever the signs: a float32
    # implementation's error scales with it, not with |grad|
    terms = (pf * (weight + (pf * weight).sum(axis=0, keepdims=True)) + lam * (pf + hot)) * vf[None, :]
    terms = terms.reshape(c, n, h, w).transpose(1, 0, 2, 3)
    return loss, grad, {"segments": seg_info, "n_valid": nv, "gamma": gamma, "terms": terms}


def _lovasz_grad_torch(gt_sorted):
    gts = gt_sorted.sum()
    intersection = gts - gt_sorted.cumsum(0)
    union = gts + (1 - gt_sorted).cumsum(0)
    jaccard = 1.0 - intersection / union
    if gt_sorted.numel() > 1:
        jaccard[1:] = jaccard[1:] - jaccard[:-1]
    return jaccard


def _lovasz_flat_torch(probas, labels, classes):
    if probas.numel() == 0:
        return probas.sum() * 0.0
    losses = []
    for k in range(probas.shape[1]):
        fg = (labels == k).double()
        if classes == "present" and fg.sum() == 0:
            continue
        errors = (fg - probas[:, k]).abs()
        errors_sorted, perm = torch.sort(errors, dim=0, descending=True, stable=True)
        losses.append(torch.dot(errors_sorted, _lovasz_grad_torch(fg[perm])))
    return torch.stack(losses).mean()


def lovasz_torch(logits, target, ignore_index=255, classes="present", per_image=False, ce_weight=0.0):
    """Berman's lovasz_softmax(probas, labels, classes, per_image, ignore) on softmax(logits) in float64, with the
    tail's out-of-range rule, plus ce_weight * the mean CE over the valid pixels. Differentiable (sort order fixed)."""
    x = logits.double()
    c = x.shape[1]
    p = torch.softmax(x, dim=1)
    valid = valid_mask(target, c, ignore_index)

    def flat(pi, ti, vi):
        pr = pi.permute(0, 2, 3, 1).reshape(-1, c)
        return pr[vi.reshape(-1)], ti.reshape(-1)[vi.reshape(-1)]

    if per_image:
        loss = torch.stack([_lovasz_flat_torch(*flat(p[i:i + 1], target[i:i + 1], valid[i:i + 1]), classes)
                            for i in range(x.shape[0])]).mean()
    else:
        loss = _lovasz_flat_torch(*flat(p, target, valid), classes)
    nv = int(valid.sum())
    if ce_weight != 0.0 and nv > 0:
        t = torch.where(valid, target, torch.zeros_like(target))
        nll = -torch.log_softmax(x, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
        loss = loss + ce_weight * (nll * valid).sum() / nv
    return loss
