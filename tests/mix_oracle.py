"""numpy / float64 statement of the CutMix / ClassMix contract (include/semseg_b200.h semseg_mix_*, semseg_b200/losses.py
MixPseudoLabelLoss), the checker of the mixing tests.

`cutmix_box` is the box in numpy float64, each operation correctly rounded (numpy's sqrt and arithmetic are IEEE), in
the order the header states; `classmix_selected` the ceil(k/2) present classes with the smallest (u, c); `mix_mask`,
`mixed_batch` the mask and the mixed input and target; `mixed_teacher` the teacher's upsampled maps mixed by the mask at
the target grid, from which tests/pl_oracle.py's `effective` / `pl_loss` / `pl_grad` state the mixed pseudo-label
loss."""
import numpy as np
import torch

from tests.kd_oracle import upsampled


def cutmix_box(u, H, W, area, ratio):
    """(x0, y0, bw, bh) of one image from its uniforms u[0..4] (fp32 values, read exactly as float64)."""
    u1, u2, u3, u4 = (np.float64(np.float32(v)) for v in u[1:5])
    lo, hi = np.float64(area[0]), np.float64(area[1])
    rlo, rhi = np.float64(ratio[0]), np.float64(ratio[1])
    a = (lo + (hi - lo) * u1) * np.float64(H) * np.float64(W)
    rho = rlo + (rhi - rlo) * u2
    bw = min(W, max(1, int(np.floor(np.sqrt(a / rho)))))
    bh = min(H, max(1, int(np.floor(np.sqrt(a * rho)))))
    x0 = min(W - bw, int(np.floor(u4 * np.float64(W - bw + 1))))
    y0 = min(H - bh, int(np.floor(u3 * np.float64(H - bh + 1))))
    return x0, y0, bw, bh


def mixed_flags(u, p):
    """Image n is mixed iff double(u[n, 0]) < p."""
    return np.asarray(u, dtype=np.float32)[:, 0].astype(np.float64) < np.float64(p)


def classmix_selected(prio, present):
    """The ceil(k/2) classes of `present` (k of them) with the smallest (prio[c], c), lexicographically."""
    present = sorted(int(c) for c in present)
    order = sorted(present, key=lambda c: (float(np.float32(prio[c])), c))
    return set(order[:(len(present) + 1) // 2])


def argmax_x8(t_nhwc):
    """The teacher's argmax (first maximum) after the x8 upsample to the input grid, in float64."""
    return upsampled(t_nhwc.detach().cpu(), 8).argmax(1)


def mix_mask(mode, u, H, W, p, area, ratio, amap=None):
    """uint8 [N, H, W]: 1 where input pixel (i, j) of image n comes from its partner (n + 1) mod N."""
    u = np.asarray(u, dtype=np.float32)
    n = u.shape[0]
    mixed = mixed_flags(u, p)
    m = np.zeros((n, H, W), dtype=np.uint8)
    for i in range(n):
        if not mixed[i]:
            continue
        if mode == "cutmix":
            x0, y0, bw, bh = cutmix_box(u[i], H, W, area, ratio)
            m[i, y0:y0 + bh, x0:x0 + bw] = 1
        else:
            pi = (i + 1) % n
            a = np.asarray(amap[pi])
            sel = classmix_selected(u[pi, 5:], np.unique(a))
            m[i] = np.isin(a, list(sel)).astype(np.uint8)
    return m


def mixed_batch(x, y, mask, zoom):
    """(x_m, y_m): x_m = M ? x[pi(n)] : x[n] per channel; y_m(n, i, j) = y[pi(n)] where M(n, i 8/zoom, j 8/zoom)."""
    m = torch.as_tensor(mask).bool().to(x.device)
    xm = torch.where(m.unsqueeze(1), x.roll(-1, 0), x)
    s = 8 // zoom
    mt = m[:, ::s, ::s]
    ym = torch.where(mt, y.roll(-1, 0), y)
    return xm, ym


def mixed_teacher(t_nhwc, mask, zoom):
    """float64 NHWC teacher maps at the target size, each pixel from its source image's map: the upsampled maps of
    image n, or of (n + 1) mod N where the mask (read at the target grid) is 1."""
    t = upsampled(t_nhwc.detach().cpu(), zoom)
    s = 8 // zoom
    mt = torch.as_tensor(mask).bool()[:, ::s, ::s].unsqueeze(1)
    return torch.where(mt, t.roll(-1, 0), t).permute(0, 2, 3, 1)
