"""float64 restatement of the Active Boundary Loss (semseg_b200.losses.ActiveBoundaryLoss, csrc/boundary.cu) and of
Boundary IoU (semseg_b200.metrics.boundaryIoUGPU), in torch, numpy and scipy, straight from their contracts: the
distance map from scipy's exact EDT, the threshold level by counting, the selection with pooling, the KL logits with
autograd and the Boundary IoU bands with min / max filters. `mask_to_boundary` is the paper's per-class cv2 form."""
import numpy as np
import torch
import torch.nn.functional as F
from scipy import ndimage

LEVELS = 256
# n_0..n_7 as (drow, dcol); index 8 is the pixel itself
NEIGHBOURS = ((1, 0), (-1, 0), (0, -1), (0, 1), (-1, 1), (1, 1), (-1, -1), (1, -1))


def levels():
    """(float) t_j, t_0 = 1e-5, t_j+1 = 1.2 t_j in float64."""
    out, t = [], 1e-5
    for _ in range(LEVELS):
        out.append(t)
        t *= 1.2
    return np.array(out, dtype=np.float64).astype(np.float32)


def gt_boundary(target, ignore_index):
    t = np.asarray(target)
    b = t == ignore_index
    b[:, :-1, :] |= t[:, :-1, :] != t[:, 1:, :]
    b[:, :, :-1] |= t[:, :, :-1] != t[:, :, 1:]
    return b


def edt_sq(boundary):
    """Exact squared distance (int64) to each image's nearest boundary pixel; -1 on an image without one."""
    e = np.full(boundary.shape, -1, np.int64)
    for n in range(boundary.shape[0]):
        if not boundary[n].any():
            continue
        _, idx = ndimage.distance_transform_edt(~boundary[n], return_indices=True)
        yy, xx = np.indices(boundary[n].shape)
        e[n] = (idx[0] - yy) ** 2 + (idx[1] - xx) ** 2
    return e


def dist_map(target, ignore_index):
    """D = fp32(max(sqrt(e) - 1, 0)) computed in float64; +inf on an image without a GT boundary."""
    e = edt_sq(gt_boundary(target, ignore_index))
    D = np.maximum(np.sqrt(np.maximum(e, 0).astype(np.float64)) - 1.0, 0.0).astype(np.float32)
    D[e < 0] = np.inf
    return D


def kl_map(s):
    """k = KL(p | p_down) + KL(p | p_right) of float64 logits [N, C, H, W] -> [N, H, W]."""
    lp = torch.log_softmax(s.double(), 1)
    p = lp.exp()
    k = torch.zeros(s.shape[0], s.shape[2], s.shape[3], dtype=torch.float64)
    k[:, :-1, :] += (p[:, :, :-1, :] * (lp[:, :, :-1, :] - lp[:, :, 1:, :])).sum(1)
    k[:, :, :-1] += (p[:, :, :, :-1] * (lp[:, :, :, :-1] - lp[:, :, :, 1:])).sum(1)
    return k


def level(k, max_n):
    """j*: the smallest j < 256 with at most max_n pixels of k > (float) t_j (255 when none)."""
    thr = levels()
    k = np.asarray(k)
    for j in range(LEVELS):
        if (k > thr[j]).sum() <= max_n:
            return j
    return LEVELS - 1


def level_by_loop(k, max_n):
    """The published search: eps = 1e-5; while count(k > eps) > max_N: eps *= 1.2 (capped at 256 levels)."""
    k = np.asarray(k)
    eps, j = 1e-5, 0
    while (k > np.float32(eps)).sum() > max_n and j < LEVELS - 1:
        eps *= 1.2
        j += 1
    return j


def selection(k, D, jstar):
    """-> (B, dir, selected): dir 15 on an image without a GT boundary, as the kernel's code map."""
    thr = levels()[jstar]
    above = torch.from_numpy(np.asarray(k > thr)).double()
    B = (F.max_pool2d(above[:, None], 3, 1, 1)[:, 0] > 0).numpy()
    H, W = D.shape[1:]
    Dp = np.pad(D, ((0, 0), (1, 1), (1, 1)), constant_values=np.inf)
    stack = [Dp[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W] for dy, dx in NEIGHBOURS] + [D]
    direction = np.argmin(np.stack(stack), axis=0)
    has = np.isfinite(D)
    sel = B & (direction != 8) & has
    direction = np.where(has, direction, 15)
    return B, direction, sel


def term(s, D, direction, sel, label_smoothing, max_clip_dist):
    """ABL of float64 logits s [N, C, H, W] (differentiable) for a frozen selection -> (ABL, M). Each z_j's neighbour
    distribution is detached; out-of-image neighbours replicate the edge."""
    lp = torch.log_softmax(s, 1)
    pad = F.pad(lp.detach(), (1, 1, 1, 1), mode="replicate")
    H, W = s.shape[2:]
    z = torch.stack([(pad[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W].exp() *
                      (pad[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W] - lp)).sum(1) for dy, dx in NEIGHBOURS], 1)
    eps = label_smoothing
    d = torch.from_numpy(np.where(sel, direction, 0)).long()
    y = torch.full(z.shape, eps / 8, dtype=torch.float64).scatter(1, d[:, None], 1.0 - eps)
    loss = -(y * torch.log_softmax(z, 1)).sum(1)
    sel_t = torch.from_numpy(sel)
    w = torch.from_numpy(np.where(sel, np.minimum(D, max_clip_dist), 0.0).astype(np.float64)) / max_clip_dist
    M = int(sel.sum())
    return (w * loss)[sel_t].sum() / max(M, 1), M


def term_grad(s, D, direction, sel, label_smoothing, max_clip_dist):
    """Closed form of dABL/ds for a frozen selection: (w/M) sum_j g_j (p - p_nj), g = Y softmax(z) - y."""
    lp = torch.log_softmax(s.double(), 1)
    p = lp.exp()
    pad = F.pad(lp, (1, 1, 1, 1), mode="replicate")
    H, W = s.shape[2:]
    nbs = [pad[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W] for dy, dx in NEIGHBOURS]
    z = torch.stack([(n.exp() * (n - lp)).sum(1) for n in nbs], 1)
    eps = label_smoothing
    d = torch.from_numpy(np.where(sel, direction, 0)).long()
    y = torch.full(z.shape, eps / 8, dtype=torch.float64).scatter(1, d[:, None], 1.0 - eps)
    g = y.sum(1, keepdim=True) * torch.softmax(z, 1) - y
    M = max(int(sel.sum()), 1)
    w = torch.from_numpy(np.where(sel, np.minimum(D, max_clip_dist), 0.0).astype(np.float64)) / max_clip_dist
    g = g * (w / M)[:, None]
    return sum(g[:, j:j + 1] * (p - nbs[j].exp()) for j in range(8))


def contract(s, target, ignore_index, max_n_ratio, max_clip_dist, label_smoothing, k=None):
    """The whole ABL term on the grid of float64 logits s [N, C, H, W]; `k`, when given, is the boundary score the
    selection uses (the kernel's own map), else the oracle's. -> dict of the maps, ABL, M and dABL/ds."""
    D = dist_map(target, ignore_index)
    kk = kl_map(s).numpy() if k is None else np.asarray(k)
    H, W = D.shape[1:]
    jstar = level(kk, max_n_ratio * H * W)
    B, direction, sel = selection(kk, D, jstar)
    loss, M = term(s.double(), D, direction, sel, label_smoothing, max_clip_dist)
    grad = term_grad(s, D, direction, sel, label_smoothing, max_clip_dist)
    return {"D": D, "k": kk, "jstar": jstar, "B": B, "dir": direction, "sel": sel, "abl": float(loss), "M": M,
            "grad": grad}


# ------------------------------------------------------------------------------------------------ Boundary IoU
def band_width(H, W, dilation_ratio=0.02):
    return max(1, round(dilation_ratio * np.sqrt(H * H + W * W)))


def bands(x, d):
    """Pixels whose (2d+1)^2 window reaches outside the image or holds another label, per image of [N, H, W]."""
    size = (1, 2 * d + 1, 2 * d + 1)
    mixed = ndimage.maximum_filter(x, size=size, mode="nearest") != ndimage.minimum_filter(x, size=size, mode="nearest")
    edge = np.zeros(x.shape, bool)
    edge[:, :d], edge[:, -d:], edge[:, :, :d], edge[:, :, -d:] = True, True, True, True
    return mixed | edge


def biou_counts(output, target, K, ignore_index, d):
    """int64 [3, K]: (intersection, |output band|, |target band|) over the pixels whose target is not ignore_index."""
    o, t = np.asarray(output), np.asarray(target)
    bo, bt = bands(o, d), bands(t, d)
    valid = t != ignore_index
    out = np.zeros((3, K), np.int64)
    for c in range(K):
        out[0, c] = (valid & bt & bo & (t == c) & (o == c)).sum()
        out[1, c] = (valid & bo & (o == c)).sum()
        out[2, c] = (valid & bt & (t == c)).sum()
    return out


def mask_to_boundary(mask, d):
    """The paper's boundary of a binary mask: pad by 1, erode with a 3x3 kernel d times, subtract."""
    import cv2
    h, w = mask.shape
    m = cv2.copyMakeBorder(mask.astype(np.uint8), 1, 1, 1, 1, cv2.BORDER_CONSTANT, value=0)
    eroded = cv2.erode(m, np.ones((3, 3), np.uint8), iterations=d)[1:h + 1, 1:w + 1]
    return mask & ~eroded.astype(bool)


def biou_counts_cv2(output, target, K, ignore_index, d):
    o, t = np.asarray(output), np.asarray(target)
    out = np.zeros((3, K), np.int64)
    for n in range(o.shape[0]):
        valid = t[n] != ignore_index
        for c in range(K):
            bo, bt = mask_to_boundary(o[n] == c, d), mask_to_boundary(t[n] == c, d)
            out[0, c] += (valid & bt & bo).sum()
            out[1, c] += (valid & bo).sum()
            out[2, c] += (valid & bt).sum()
    return out
