"""float64 torch statement of the strong view (include/semseg_b200.h semseg_strong_augment, semseg_b200/augment.py
StrongAugment), the checker of the strong-view tests.

`params` derives one image's flags, factors, order, sigma and radius from its uniforms exactly as the kernel does (the
fp64 arithmetic of Python floats, each result rounded once to fp32 where the header says so); `chain` applies them to
one de-normalised float64 image with torchvision.transforms.v2.functional's float formulas restated here; `strong`
is the whole batch, normalised in and out."""
import math

import numpy as np
import torch

GRAY = (0.2989, 0.587, 0.114)
OPS = ("brightness", "contrast", "saturation", "hue")


def f32(v):
    return float(np.float32(v))


def params(u, brightness, contrast, saturation, hue, p_jitter, p_gray, p_blur, sigma):
    """One image's operations from its uniforms u[0..11] (fp32 values, read exactly): {'ops': [(name, factor)] in
    order, 'gray': bool, 'sigma': float or None, 'r': int}."""
    u = [float(np.float32(v)) for v in u]
    strengths = (brightness, contrast, saturation, hue)
    ranges = [(max(0.0, 1.0 - brightness), 1.0 + brightness), (max(0.0, 1.0 - contrast), 1.0 + contrast),
              (max(0.0, 1.0 - saturation), 1.0 + saturation), (-hue, hue)]
    ops = []
    if u[0] < p_jitter:
        active = [k for k in range(4) if strengths[k] > 0.0]
        for k in sorted(active, key=lambda k: (u[5 + k], k)):
            lo, hi = ranges[k]
            ops.append((OPS[k], f32(lo + (hi - lo) * u[1 + k])))
    sig, r = None, 0
    if u[10] < p_blur:
        sig = f32(sigma[0] + (sigma[1] - sigma[0]) * u[11])
        r = min(math.ceil(3.0 * sig), math.ceil(3.0 * sigma[1]))
    return {'ops': ops, 'gray': u[9] < p_gray, 'sigma': sig, 'r': r}


def gray(v):
    return GRAY[0] * v[0] + GRAY[1] * v[1] + GRAY[2] * v[2]


def rgb_to_hsv(v):
    r, g, _ = v.unbind(0)
    minc, maxc = torch.aminmax(v, dim=0)
    eqc = maxc == minc
    cr = maxc - minc
    ones = torch.ones_like(maxc)
    s = cr / torch.where(eqc, ones, maxc)
    rc, gc, bc = ((maxc.unsqueeze(0) - v) / torch.where(eqc, ones, cr).unsqueeze(0)).unbind(0)
    h = torch.where(maxc == r, bc - gc, torch.where(maxc == g, 2.0 + rc - bc, 4.0 + gc - rc))
    h = torch.fmod(h / 6.0 + 1.0, 1.0)
    return h, s, maxc


def hsv_to_rgb(h, s, v):
    h6 = h * 6.0
    i = torch.floor(h6)
    f = h6 - i
    i = i.long().remainder(6)
    q = ((1.0 - s * f) * v).clamp(0.0, 1.0)
    t = ((s * f + 1.0 - s) * v).clamp(0.0, 1.0)
    p = ((1.0 - s) * v).clamp(0.0, 1.0)
    vpqt = torch.stack((v, p, q, t))
    select = torch.tensor([[0, 2, 1, 1, 3, 0], [3, 0, 0, 2, 1, 1], [1, 1, 3, 0, 0, 2]], device=v.device)[:, i]
    return vpqt.gather(0, select)


def apply_op(v, name, f):
    if name == "brightness":
        return (f * v).clamp(0.0, 1.0)
    if name == "contrast":
        return (f * v + (1.0 - f) * gray(v).mean()).clamp(0.0, 1.0)
    if name == "saturation":
        return (f * v + (1.0 - f) * gray(v)).clamp(0.0, 1.0)
    h, s, val = rgb_to_hsv(v)
    return hsv_to_rgb(torch.remainder(h + f, 1.0), s, val)


def taps(sig, r, device=None):
    k = torch.arange(-r, r + 1, dtype=torch.float64, device=device)
    w = torch.exp(-k * k / (2.0 * sig * sig))
    return w / w.sum()


def blur(v, sig, r):
    """Separable true Gaussian with reflect-101 borders: torchvision's gaussian_blur(v, [2r+1]*2, [sig]*2)."""
    w = taps(sig, r, v.device)
    p = torch.nn.functional.pad(v.unsqueeze(0), (r, r, r, r), mode="reflect")[0]
    k2 = (w.unsqueeze(1) * w.unsqueeze(0)).expand(3, 1, 2 * r + 1, 2 * r + 1)
    return torch.nn.functional.conv2d(p.unsqueeze(0), k2, groups=3)[0]


def chain(v, prm):
    """One de-normalised float64 image [3, H, W] (already clamped to [0, 1]) through the image's operations."""
    for name, f in prm['ops']:
        v = apply_op(v, name, f)
    if prm['gray']:
        v = gray(v).unsqueeze(0).expand(3, -1, -1).clone()
    if prm['r'] > 0:
        v = blur(v, prm['sigma'], prm['r'])
    return v


def strong(x, u, brightness=0.5, contrast=0.5, saturation=0.5, hue=0.25, p_jitter=0.8, p_gray=0.2, p_blur=0.5,
           sigma=(0.1, 2.0), mean=(0.485 * 255, 0.456 * 255, 0.406 * 255), std=(0.229 * 255, 0.224 * 255, 0.225 * 255)):
    """The strong view of a normalised batch x [N, 3, H, W] from uniforms u [N, 12], in float64 on x's device (x
    itself where no operation applies)."""
    x = x.detach().double()
    u = u.detach().cpu().float().numpy()
    m = torch.tensor(mean, dtype=torch.float64, device=x.device).view(3, 1, 1)
    s = torch.tensor(std, dtype=torch.float64, device=x.device).view(3, 1, 1)
    out = x.clone()
    for n in range(x.shape[0]):
        prm = params(u[n], brightness, contrast, saturation, hue, p_jitter, p_gray, p_blur, sigma)
        if not (prm['ops'] or prm['gray'] or prm['r']):
            continue
        v = ((x[n] * s + m) / 255.0).clamp(0.0, 1.0)
        out[n] = (255.0 * chain(v, prm) - m) / s
    return out
