"""Float64 statements of the Gated CRF loss of semseg_b200.losses.GatedCRFLoss (Obukhov et al., 2019).

`crf_contract` is the contract of the class docstring and include/semseg_b200.h with its closed-form gradient: the
window of a pixel holds only in-image neighbours. `crf_unfold` states the published formulation literally: the
features (positions in grid units and colours, each divided by its sigma) and the probabilities are unfolded with zero
padding, so an out-of-image neighbour has zero features (a non-zero gate) and zero probabilities. The two differ by
`crf_outside_constant`, a constant of the image alone. `crf_loop` is a brute-force loop over pixel pairs."""
import math

import torch
import torch.nn.functional as F

IMAGENET_MEAN = (0.485 * 255, 0.456 * 255, 0.406 * 255)
IMAGENET_STD = (0.229 * 255, 0.224 * 255, 0.225 * 255)


def grid_rgb(x, stride, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """The normalised NCHW image x point-sampled at `stride` and un-normalised to RGB in [0, 1], float64."""
    x = x.double()[:, :, ::stride, ::stride]
    m = torch.tensor(mean, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    s = torch.tensor(std, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    return (x * s + m) / 255.0


def _shift(t, dy, dx):
    """t[..., y + dy, x + dx] with zeros outside, and the in-image mask."""
    H, W = t.shape[-2:]
    out = torch.zeros_like(t)
    ok = torch.zeros(t.shape[-2:], dtype=torch.bool, device=t.device)
    if abs(dy) >= H or abs(dx) >= W:
        return out, ok
    ys, yd = slice(max(dy, 0), H + min(dy, 0)), slice(max(-dy, 0), H + min(-dy, 0))
    xs, xd = slice(max(dx, 0), W + min(dx, 0)), slice(max(-dx, 0), W + min(-dx, 0))
    out[..., yd, xd] = t[..., ys, xs]
    ok[yd, xd] = True
    return out, ok


def crf_contract(s, rgb, radius, sigma_xy, sigma_rgb):
    """s float64 logits [N, C, H, W] on the loss grid, rgb [N, 3, H, W] in [0, 1] -> (CRF, dCRF/ds, S)."""
    s, rgb = s.double(), rgb.double()
    N, C, H, W = s.shape
    P = N * H * W
    p = torch.softmax(s, 1)
    G = torch.zeros_like(p)
    K = torch.zeros((N, H, W), dtype=torch.float64, device=s.device)
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            if dy == 0 and dx == 0:
                continue
            pj, ok = _shift(p, dy, dx)
            cj, _ = _shift(rgb, dy, dx)
            k = torch.exp(-(dy * dy + dx * dx) / (2 * sigma_xy ** 2) - ((rgb - cj) ** 2).sum(1) / (2 * sigma_rgb ** 2))
            k = k * ok
            G += k.unsqueeze(1) * pj
            K += k
    S = (p * G).sum(1)
    loss = (K - S).sum() / P
    grad = -(2.0 / P) * p * (G - S.unsqueeze(1))
    return loss, grad, S


def crf_unfold(s, rgb, radius, sigma_xy, sigma_rgb, dtype=torch.float64):
    """The published formulation with zero-padded unfolds, differentiable by autograd -> CRF (in `dtype`)."""
    s, rgb = s.to(dtype), rgb.to(dtype)
    N, C, H, W = s.shape
    k = 2 * radius + 1
    yy, xx = torch.meshgrid(torch.arange(H, dtype=dtype, device=rgb.device),
                            torch.arange(W, dtype=dtype, device=rgb.device), indexing="ij")
    pos = torch.stack((yy, xx)).unsqueeze(0).expand(N, 2, H, W) / sigma_xy
    feat = torch.cat((pos, rgb / sigma_rgb), 1)                                        # [N, 5, H, W]
    fu = F.unfold(feat, k, padding=radius).view(N, 5, k * k, H, W)
    gate = torch.exp(-0.5 * ((fu - feat.unsqueeze(2)) ** 2).sum(1))                     # [N, k*k, H, W]
    gate[:, (k * k) // 2] = 0.0                                                         # not the pixel itself
    p = torch.softmax(s, 1)
    pu = F.unfold(p, k, padding=radius).view(N, C, k * k, H, W)
    compat = 1.0 - (p.unsqueeze(2) * pu).sum(1)                                         # Potts: 1 - p_i . p_j
    return (gate * compat).sum() / (N * H * W)


def crf_outside_constant(rgb, radius, sigma_xy, sigma_rgb):
    """What crf_unfold adds to crf_contract: the zero-feature gates of out-of-image neighbours, over P."""
    rgb = rgb.double()
    N, _, H, W = rgb.shape
    total = 0.0
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=rgb.device),
                            torch.arange(W, dtype=torch.float64, device=rgb.device), indexing="ij")
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            _, ok = _shift(rgb, dy, dx)
            out = ~ok
            k = torch.exp(-(yy ** 2 + xx ** 2) / (2 * sigma_xy ** 2) - (rgb ** 2).sum(1) / (2 * sigma_rgb ** 2))
            total += float((k * out).sum())
    return total / (N * H * W)


def crf_loop(s, rgb, radius, sigma_xy, sigma_rgb):
    """Brute force over every in-image pixel pair of every window -> CRF (tiny grids only)."""
    s, rgb = s.double(), rgb.double()
    N, C, H, W = s.shape
    p = torch.softmax(s, 1)
    total = 0.0
    for n in range(N):
        for y in range(H):
            for x in range(W):
                for v in range(max(0, y - radius), min(H, y + radius + 1)):
                    for u in range(max(0, x - radius), min(W, x + radius + 1)):
                        if v == y and u == x:
                            continue
                        d2 = float(((rgb[n, :, y, x] - rgb[n, :, v, u]) ** 2).sum())
                        k = math.exp(-((v - y) ** 2 + (u - x) ** 2) / (2 * sigma_xy ** 2) - d2 / (2 * sigma_rgb ** 2))
                        total += k * (1.0 - float((p[n, :, y, x] * p[n, :, v, u]).sum()))
    return total / (N * H * W)


def upsample(logits_nchw, zoom):
    """The network's bilinear xZ upsample (align_corners) in float64."""
    if zoom == 1:
        return logits_nchw.double()
    h, w = logits_nchw.shape[-2:]
    return F.interpolate(logits_nchw.double(), size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear",
                         align_corners=True)


def tail_loss(logits_nhwc, target, x, zoom, at, ignore_index, crf_weight, ce_weight, radius, sigma_xy, sigma_rgb,
              mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """The whole criterion on the fused tail in float64, differentiable by autograd: fp32 NHWC 1/8 logits [N,h,w,C],
    target [N,Ho,Wo], the normalised input x [N,3,8(h-1)+1,8(w-1)+1] -> main loss."""
    s8 = logits_nhwc.double().permute(0, 3, 1, 2)
    up = upsample(s8, zoom)
    C = up.shape[1]
    valid = (target != ignore_index) & (target >= 0) & (target < C)
    lsm = torch.log_softmax(up, 1)
    nll = -lsm.gather(1, target.clamp(0, C - 1).unsqueeze(1)).squeeze(1)
    ce = (nll * valid).sum() / max(int(valid.sum()), 1)
    grid, stride = (up, 8 // zoom) if at == "output" else (s8, 8)
    rgb = grid_rgb(x, stride, mean, std)
    crf = crf_unfold(grid, rgb, radius, sigma_xy, sigma_rgb) - crf_outside_constant(rgb, radius, sigma_xy, sigma_rgb)
    return ce_weight * ce + crf_weight * crf
