"""float64 numpy restatement of the anomaly-segmentation contract (semseg_b200/anomaly.py, csrc/anomaly.cu): the four
scores, the SML class statistics, boundary suppression and dilated smoothing, and AUROC / AP / FPR95 with ties
grouped. Vectorised; tests/test_anomaly_cpu.py checks it against per-pixel loops and sklearn."""
import numpy as np


def scores(kind, prob, ml, lse, pred=None, mean=None, std=None, **sml):
    """Anomaly map (higher = more anomalous) of prob [C, H, W], ml / lse [H, W]; sml options as AnomalyScorer's."""
    if kind == "msp":
        return 1.0 - prob.max(0)
    if kind == "maxlogit":
        return -ml
    if kind == "energy":
        return -lse
    return sml_map(ml, pred, mean, std, **sml)


def class_moments(pred, ml, classes):
    """[3, C]: per predicted class sum ML, sum ML^2, count."""
    pred, ml = pred.reshape(-1), ml.reshape(-1).astype(np.float64)
    return np.stack([np.bincount(pred, ml, classes), np.bincount(pred, ml * ml, classes),
                     np.bincount(pred, None, classes).astype(np.float64)])


def class_statistics(pred, ml, classes):
    """(mean, std) [C]: mean and population std of ML per predicted class; a class with fewer than 2 pixels or a zero
    std takes those of all pixels."""
    pred, ml = pred.reshape(-1), ml.reshape(-1).astype(np.float64)
    g_mean, g_std = ml.mean(), ml.std()
    mean, std = np.full(classes, g_mean), np.full(classes, g_std)
    for c in range(classes):
        v = ml[pred == c]
        if v.size >= 2 and v.std() > 0:
            mean[c], std[c] = v.mean(), v.std()
    return mean, std


def window_any_other(pred, r):
    """Boundary mask: the (2r+1)^2 window around each pixel, clipped to the image, holds another prediction."""
    H, W = pred.shape
    lo = np.full(pred.shape, np.iinfo(np.int64).max)
    hi = np.full(pred.shape, np.iinfo(np.int64).min)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            ys, ye = max(0, -dy), min(H, H - dy)
            xs, xe = max(0, -dx), min(W, W - dx)
            if ys >= ye or xs >= xe:
                continue
            src = pred[ys + dy:ye + dy, xs + dx:xe + dx]
            lo[ys:ye, xs:xe] = np.minimum(lo[ys:ye, xs:xe], src)
            hi[ys:ye, xs:xe] = np.maximum(hi[ys:ye, xs:xe], src)
    return lo != hi


def suppression_widths(width, iterations):
    return [width - i * (width // iterations) for i in range(iterations)]


def suppress(S, pred, width, iterations):
    """Jacobi boundary suppression: boundary pixels take the mean of the previous map over the non-boundary pixels of
    their clipped 3x3 neighbourhood (kept if there are none)."""
    S = S.astype(np.float64).copy()
    H, W = S.shape
    for r in suppression_widths(width, iterations) if iterations else []:
        edge = window_any_other(pred, r)
        keep = ~edge
        num, cnt = np.zeros_like(S), np.zeros(S.shape, dtype=np.int64)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                ys, ye = max(0, -dy), min(H, H - dy)
                xs, xe = max(0, -dx), min(W, W - dx)
                if ys >= ye or xs >= xe:
                    continue
                k = keep[ys + dy:ye + dy, xs + dx:xe + dx]
                num[ys:ye, xs:xe] += np.where(k, S[ys + dy:ye + dy, xs + dx:xe + dx], 0.0)
                cnt[ys:ye, xs:xe] += k
        upd = edge & (cnt > 0)
        S = np.where(upd, num / np.maximum(cnt, 1), S)
    return S


def smooth(S, kernel, sigma, dilation):
    """sum g(a,b) S(p + d (a,b)) / sum g(a,b) over the taps inside the image, g = exp(-(a^2 + b^2) / 2 sigma^2)."""
    H, W = S.shape
    half = kernel // 2
    num, den = np.zeros_like(S, dtype=np.float64), np.zeros_like(S, dtype=np.float64)
    for a in range(-half, half + 1):
        for b in range(-half, half + 1):
            dy, dx = dilation * a, dilation * b
            ys, ye = max(0, -dy), min(H, H - dy)
            xs, xe = max(0, -dx), min(W, W - dx)
            if ys >= ye or xs >= xe:
                continue
            g = np.exp(-(a * a + b * b) / (2.0 * sigma * sigma))
            num[ys:ye, xs:xe] += g * S[ys + dy:ye + dy, xs + dx:xe + dx]
            den[ys:ye, xs:xe] += g
    return num / den


def sml_map(ml, pred, mean, std, boundary_width=4, boundary_iterations=4, smooth_kernel=7, smooth_sigma=1.0,
            smooth_dilation=6):
    S = (ml.astype(np.float64) - mean[pred]) / std[pred]
    S = suppress(S, pred, boundary_width, boundary_iterations)
    return -smooth(S, smooth_kernel, smooth_sigma, smooth_dilation)


def metrics(score, label, ignore_index=255):
    """(auroc, ap, fpr95, positives, negatives) of the non-void pixels, sorted by score descending with equal scores
    (-0.0 = +0.0) one group: AUROC the Mann-Whitney statistic (ties 1/2), AP = sum_g p_g / P * TP_g / (TP_g + FP_g),
    FPR95 = FP_g / N at the first group with TP_g / P >= 0.95."""
    score, label = np.asarray(score).reshape(-1), np.asarray(label).reshape(-1)
    keep = label != ignore_index
    s = score[keep].astype(np.float64) + 0.0
    y = label[keep].astype(np.int64)
    order = np.argsort(-s, kind="stable")
    s, y = s[order], y[order]
    ends = np.r_[np.nonzero(s[1:] != s[:-1])[0], s.size - 1]
    tp = np.cumsum(y == 1)[ends].astype(np.float64)
    fp = np.cumsum(y == 0)[ends].astype(np.float64)
    P, N = tp[-1], fp[-1]
    tp0, fp0 = np.r_[0.0, tp[:-1]], np.r_[0.0, fp[:-1]]
    auroc = float(np.sum((fp - fp0) * (tp0 + tp)) / (2.0 * P * N))
    ap = float(np.sum((tp - tp0) * (tp / (tp + fp))) / P)
    first = int(np.argmax(tp / P >= 0.95))
    return auroc, ap, float(fp[first] / N), int(P), int(N)
