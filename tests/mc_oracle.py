"""float64 restatement of Monte Carlo dropout scoring (csrc/window.cu's semseg_window_scores_mc and the finish of
semseg_b200/inference.py with mc_draws > 0), in torch so that it runs on the tensors' own device.

  * per draw t and image: the x8 bilinear align_corners upsample of the [h, w] node logits to 8(h-1)+1 x 8(w-1)+1, the
    softmax q over the classes and the sample entropy H = -sum_c q_c log q_c;
  * with flip, images G..2G-1 are the mirrors of 0..G-1: their maps are flipped back along the width and averaged with
    the originals, (a + a') / 2;
  * the draw mean of the scores and of H: out [G, C + 1, crop_h, crop_w];
  * from a scale-averaged total [C + 1, h, w] (p_bar, then E[H]): H[p_bar] = -sum p_bar log p_bar (0 log 0 = 0) and the
    mutual information H[p_bar] - E[H].
"""
import torch


def _axis(m, device):
    """Source nodes and weight of the x8 align_corners upsample along one axis of m nodes."""
    pos = torch.arange(8 * (m - 1) + 1, dtype=torch.float64, device=device) / 8.0
    i0 = pos.floor().long().clamp(max=m - 1)
    i1 = (i0 + 1).clamp(max=m - 1)
    return i0, i1, pos - i0


def upsample_x8(logits):
    """fp64 [n, C, 8(h-1)+1, 8(w-1)+1] of node logits [n, h, w, C] (NHWC, any float dtype)."""
    n, h, w, c = logits.shape
    v = logits.double().permute(0, 3, 1, 2)
    y0, y1, fy = _axis(h, v.device)
    x0, x1, fx = _axis(w, v.device)
    rows = v[:, :, y0] * (1.0 - fy)[:, None] + v[:, :, y1] * fy[:, None]
    return rows[..., x0] * (1.0 - fx) + rows[..., x1] * fx


def sample_maps(v):
    """fp64 [n, C + 1, H, W]: softmax over dim 1 of the logits v [n, C, H, W], then the sample entropy."""
    v = v.double()
    d = v - v.amax(1, keepdim=True)
    q = torch.softmax(d, 1)
    ent = torch.logsumexp(d, 1) - (q * d).sum(1)
    return torch.cat([q, ent[:, None]], 1)


def mc_scores(logits, flip, upsample=upsample_x8):
    """fp64 [G, C + 1, crop_h, crop_w] of T draws of node logits [T, G (+G mirrors when flip), h, w, C]. `upsample`
    maps one draw's [n, h, w, C] node logits to [n, C, crop_h, crop_w] (default: the fp64 upsample above)."""
    total = None
    for lt in logits:
        m = sample_maps(upsample(lt))
        if flip:
            g = m.shape[0] // 2
            m = (m[:g] + m[g:].flip(3)) / 2
        total = m if total is None else total + m
    return total / logits.shape[0]


def uncertainty(total, classes):
    """fp64 [2, h, w] (H[p_bar], mutual information) of a total [classes + 1, h, w] (p_bar, then E[H])."""
    total = total.double()
    pbar = total[:classes]
    hbar = -torch.where(pbar > 0, pbar * torch.log(torch.where(pbar > 0, pbar, 1.0)), 0.0).sum(0)
    return torch.stack([hbar, hbar - total[classes]])
