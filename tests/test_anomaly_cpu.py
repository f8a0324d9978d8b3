"""CPU tier for anomaly segmentation (semseg_b200/anomaly.py, csrc/anomaly.cu): the float64 contract
(tests/anomaly_oracle.py) against sklearn's ranking metrics and against per-pixel loops of suppression and smoothing,
the options' validation, the statistics finalisation, and the entry points' rejection of bad arguments before any
CUDA call."""
import ctypes

import numpy as np
import pytest
import torch
from sklearn.metrics import average_precision_score, roc_auc_score, roc_curve

from semseg_b200 import _lib
from semseg_b200.anomaly import AnomalyMeter, AnomalyScorer
from tests import anomaly_oracle as O

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


# ------------------------------------------------------------------------------------------------ metrics oracle
def _tied_scores(rng, n, levels):
    """Scores on `levels` distinct values (heavy ties, many exact duplicates), with +0.0 and -0.0 both present."""
    vals = np.round(rng.standard_normal(levels), 2)
    s = rng.choice(vals, n)
    s[rng.random(n) < 0.05] = 0.0
    s[rng.random(n) < 0.05] = -0.0
    return s.astype(np.float32)


@pytest.mark.parametrize("seed,n,levels,void", [(0, 5000, 7, False), (1, 5000, 7, True), (2, 20000, 300, True),
                                                (3, 3000, 2, False), (4, 10000, 10000, True)])
def test_oracle_matches_sklearn(seed, n, levels, void):
    rng = np.random.default_rng(seed)
    s = _tied_scores(rng, n, levels)
    y = (rng.random(n) < 0.5 * (s > 0) + 0.1).astype(np.int64)
    if void:
        y[rng.random(n) < 0.2] = 255
    auroc, ap, fpr95, pos, neg = O.metrics(s, y)
    keep = y != 255
    assert abs(auroc - roc_auc_score(y[keep], s[keep])) <= 1e-12
    assert abs(ap - average_precision_score(y[keep], s[keep])) <= 1e-12
    fpr, tpr, _ = roc_curve(y[keep], s[keep], drop_intermediate=False)
    assert fpr95 == fpr[np.argmax(tpr >= 0.95)]
    assert (pos, neg) == (int((y[keep] == 1).sum()), int((y[keep] == 0).sum()))


def test_oracle_folds_negative_zero():
    s = np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0], np.float32)
    y = np.array([1, 0, 0, 1, 1, 0])
    assert O.metrics(s, y)[0] == roc_auc_score(y, s)
    assert O.metrics(s, y) == O.metrics(np.where(s == 0, np.float32(0.0), s), y)
    assert O.metrics(s, y) != O.metrics(np.where(np.signbit(s), np.float32(-1e-30), s), y)


# ------------------------------------------------------------------------------------------------ SML oracle
def _brute_boundary(pred, y, x, r):
    H, W = pred.shape
    win = pred[max(0, y - r):min(H, y + r + 1), max(0, x - r):min(W, x + r + 1)]
    return bool((win != pred[y, x]).any())


def _brute_suppress(S, pred, width, iterations):
    S = S.copy()
    H, W = S.shape
    for r in O.suppression_widths(width, iterations) if iterations else []:
        edge = np.array([[_brute_boundary(pred, y, x, r) for x in range(W)] for y in range(H)])
        nxt = S.copy()
        for y in range(H):
            for x in range(W):
                if not edge[y, x]:
                    continue
                vals = [S[yy, xx] for yy in range(max(0, y - 1), min(H, y + 2))
                        for xx in range(max(0, x - 1), min(W, x + 2)) if not edge[yy, xx]]
                if vals:
                    nxt[y, x] = sum(vals) / len(vals)
        S = nxt
    return S


def _brute_smooth(S, k, sigma, d):
    H, W = S.shape
    out = np.empty_like(S)
    for y in range(H):
        for x in range(W):
            num = den = 0.0
            for a in range(-(k // 2), k // 2 + 1):
                for b in range(-(k // 2), k // 2 + 1):
                    yy, xx = y + d * a, x + d * b
                    if 0 <= yy < H and 0 <= xx < W:
                        g = np.exp(-(a * a + b * b) / (2 * sigma * sigma))
                        num += g * S[yy, xx]
                        den += g
            out[y, x] = num / den
    return out


def _pred_map(rng, H, W, classes):
    """Blocky predictions: regions of a few classes, so that boundaries and interiors both exist."""
    coarse = rng.integers(0, classes, (H // 5 + 1, W // 5 + 1))
    return np.kron(coarse, np.ones((5, 5), np.int64))[:H, :W]


@pytest.mark.parametrize("H,W,classes,width,iters", [(23, 31, 4, 4, 4), (17, 12, 3, 3, 2), (9, 40, 5, 1, 1),
                                                     (15, 15, 1, 4, 4), (7, 5, 3, 5, 3), (30, 20, 6, 2, 0)])
def test_oracle_suppression_matches_per_pixel_loop(H, W, classes, width, iters):
    rng = np.random.default_rng(H * W + width)
    pred = _pred_map(rng, H, W, classes)
    S = rng.standard_normal((H, W))
    got = O.suppress(S, pred, width, iters)
    ref = _brute_suppress(S, pred, width, iters)
    assert np.allclose(got, ref, rtol=0, atol=1e-13)
    if classes == 1:
        assert np.array_equal(got, S)                  # no boundary anywhere
    elif iters:
        assert not np.array_equal(got, S)


@pytest.mark.parametrize("H,W,k,sigma,d", [(23, 31, 7, 1.0, 6), (9, 11, 7, 1.0, 6), (5, 3, 5, 2.0, 3),
                                           (16, 16, 3, 0.5, 1), (12, 40, 1, 1.0, 6), (30, 7, 9, 3.0, 2)])
def test_oracle_smoothing_matches_per_pixel_loop(H, W, k, sigma, d):
    rng = np.random.default_rng(k * 100 + H)
    S = rng.standard_normal((H, W))
    got = O.smooth(S, k, sigma, d)
    assert np.allclose(got, _brute_smooth(S, k, sigma, d), rtol=0, atol=1e-13)
    if k == 1:
        assert np.array_equal(got, S)
    assert np.allclose(O.smooth(np.full((H, W), 2.5), k, sigma, d), 2.5, rtol=0, atol=1e-14)


def test_oracle_class_statistics_fall_back_for_rare_classes():
    rng = np.random.default_rng(5)
    pred = rng.integers(0, 3, 400)
    pred[7] = 3                                         # one pixel of class 3; class 4 never predicted
    ml = rng.standard_normal(400) * 3 + pred
    mean, std = O.class_statistics(pred, ml, 5)
    for c in range(3):
        assert mean[c] == pytest.approx(ml[pred == c].mean()) and std[c] == pytest.approx(ml[pred == c].std())
    assert mean[3] == mean[4] == pytest.approx(ml.mean()) and std[3] == std[4] == pytest.approx(ml.std())
    m, s = AnomalyScorer.statistics_from_moments(torch.from_numpy(O.class_moments(pred, ml, 5)))
    assert np.allclose(m.numpy(), mean, rtol=1e-12) and np.allclose(s.numpy(), std, rtol=1e-10)


def test_statistics_from_moments_rejects_degenerate_fits():
    with pytest.raises(ValueError):
        AnomalyScorer.statistics_from_moments(torch.tensor([[1.0, 0.0], [1.0, 0.0], [1.0, 0.0]], dtype=torch.float64))
    with pytest.raises(ValueError):          # every ML equal: no variance at all
        AnomalyScorer.statistics_from_moments(torch.tensor([[4.0, 2.0], [8.0, 4.0], [2.0, 1.0]], dtype=torch.float64))


# ------------------------------------------------------------------------------------------------ options
def test_defaults_and_repr():
    s = AnomalyScorer()
    assert (s.kind, s.statistics, s.boundary_width, s.boundary_iterations, s.smooth_kernel, s.smooth_sigma,
            s.smooth_dilation) == ("sml", None, 4, 4, 7, 1.0, 6)
    assert repr(s).startswith("AnomalyScorer(kind='sml'")
    AnomalyScorer(boundary_iterations=0, boundary_width=0)       # suppression off: the width is unused
    AnomalyScorer(smooth_kernel=1)


@pytest.mark.parametrize("kw,bad,exc", [
    ("kind", "entropy", ValueError), ("smooth_kernel", 4, ValueError), ("smooth_kernel", 0, ValueError),
    ("smooth_kernel", -3, ValueError), ("smooth_kernel", 65, ValueError), ("smooth_kernel", 7.0, TypeError),
    ("smooth_sigma", 0.0, ValueError), ("smooth_sigma", -1.0, ValueError), ("smooth_sigma", float("nan"), ValueError),
    ("smooth_sigma", float("inf"), ValueError), ("smooth_sigma", "1", TypeError), ("smooth_dilation", 0, ValueError),
    ("smooth_dilation", 2.5, TypeError), ("boundary_width", 0, ValueError), ("boundary_iterations", -1, ValueError),
    ("boundary_iterations", True, TypeError), ("statistics", 3, TypeError),
    ("statistics", ([0.0, 1.0], [1.0]), ValueError), ("statistics", ([0.0], [0.0]), ValueError),
    ("statistics", ([float("nan")], [1.0]), ValueError), ("statistics", ([0.0], [-1.0]), ValueError),
])
def test_option_validation(kw, bad, exc):
    with pytest.raises(exc):
        AnomalyScorer(**{kw: bad})


def test_statistics_are_kept_as_fp64_cpu_tensors():
    s = AnomalyScorer(statistics=([0.5, 1.5], np.array([1.0, 2.0], np.float32)))
    mean, std = s.statistics
    assert mean.dtype == std.dtype == torch.float64 and mean.device.type == "cpu"
    assert mean.tolist() == [0.5, 1.5] and std.tolist() == [1.0, 2.0]


def test_predictor_rejects_bad_combinations():
    from semseg_b200.densecrf import DenseCRF
    from semseg_b200.inference import SlidingWindowPredictor
    net = torch.nn.Conv2d(3, 2, 1)
    with pytest.raises(TypeError):
        SlidingWindowPredictor(net, 2, 9, 9, [0, 0, 0], anomaly="sml")
    with pytest.raises(ValueError):
        SlidingWindowPredictor(net, 2, 9, 9, [0, 0, 0], crf=DenseCRF(), anomaly=AnomalyScorer("maxlogit"))
    p = SlidingWindowPredictor(net, 2, 9, 9, [0, 0, 0], anomaly=AnomalyScorer("maxlogit"))
    with pytest.raises(ValueError):
        p(np.zeros((9, 9, 3), np.float32), 9, [1.0], exact=True)
    assert SlidingWindowPredictor(net, 2, 9, 9, [0, 0, 0]).anomaly is None


def test_meter_validates_on_the_host():
    m = AnomalyMeter()
    with pytest.raises(ValueError):
        m.compute()                                      # nothing stored
    with pytest.raises(ValueError):
        m.update(torch.zeros(4), torch.zeros(4, dtype=torch.int64))     # CPU tensors: no host metric
    with pytest.raises(TypeError):
        m.update(np.zeros(4), np.zeros(4))
    assert m.count == 0


# ------------------------------------------------------------------------------------------------ C-ABI validation
def test_window_scores_stats_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.semseg_window_scores_stats(None, 19, 1, 9, 9, 19, 1, P, 65, 65, None) == -1 and b"null" in _err()
    assert lib.semseg_window_scores_stats(P, 19, 1, 9, 9, 19, 1, None, 65, 65, None) == -1 and b"null" in _err()
    assert lib.semseg_window_scores_stats(P, 300, 1, 9, 9, 257, 1, P, 65, 65, None) == -1 and b"bad sizes" in _err()
    assert lib.semseg_window_scores_stats(P, 19, 1, 9, 9, 19, 2, P, 65, 65, None) == -1 and b"bad sizes" in _err()
    assert lib.semseg_window_scores_stats(P, 19, 1, 9, 9, 19, 1, P, 64, 65, None) == -1 and b"8(h-1)+1" in _err()
    assert b"window_scores_stats" in _err()


def test_class_moments_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.semseg_anomaly_class_moments_workspace_bytes(4096, 19) == 2 * 3 * 19 * 8
    assert lib.semseg_anomaly_class_moments_workspace_bytes(4097, 19) == 3 * 3 * 19 * 8
    assert lib.semseg_anomaly_class_moments_workspace_bytes(0, 19) == -1 and b"bad sizes" in _err()
    assert lib.semseg_anomaly_class_moments_workspace_bytes(10, 4097) == -1
    for i in range(4):
        args = [P, P, P, P]
        args[i] = None
        assert lib.semseg_anomaly_class_moments(args[0], args[1], 100, 19, args[2], args[3], None) == -1
        assert b"null" in _err()
    assert lib.semseg_anomaly_class_moments(P, P, 100, 0, P, P, None) == -1 and b"bad sizes" in _err()


def _sml(ml=P, pred=P, H=9, W=7, C=3, mean=P, std=P, width=4, iters=4, k=7, sigma=1.0, d=6, ws=P, out=P):
    return _lib.load().semseg_anomaly_sml(ml, pred, H, W, C, mean, std, width, iters, k, sigma, d, ws, out, None)


def test_sml_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.semseg_anomaly_sml_workspace_bytes(9, 7) == 40 * 63
    assert lib.semseg_anomaly_sml_workspace_bytes(0, 7) == -1 and b"empty image" in _err()
    for kw in ("ml", "pred", "mean", "std", "ws", "out"):
        assert _sml(**{kw: None}) == -1 and b"null" in _err(), kw
    assert _sml(H=0) == -1 and b"empty image" in _err()
    assert _sml(C=0) == -1 and b"class count" in _err()
    for kw, bad, msg in (("k", 4, b"odd"), ("k", 0, b"odd"), ("k", 65, b"odd"), ("sigma", 0.0, b"sigma"),
                         ("sigma", float("nan"), b"sigma"), ("sigma", float("inf"), b"sigma"), ("d", 0, b"dilation"),
                         ("iters", -1, b"suppression"), ("width", 0, b"suppression")):
        assert _sml(**{kw: bad}) == -1 and msg in _err(), (kw, bad)
    assert _sml(width=0, iters=0, out=None) == -1 and b"null" in _err()     # the options pass, the pointer does not


def test_metrics_rejects_bad_arguments():
    lib = _lib.load()
    nb = lib.semseg_anomaly_metrics_workspace_bytes(10 ** 6)
    assert 16 * 10 ** 6 <= nb <= 17 * 10 ** 6
    assert lib.semseg_anomaly_metrics_workspace_bytes(0) == -1 and b"pixel count" in _err()
    assert lib.semseg_anomaly_metrics_workspace_bytes(2 ** 31) == -1
    assert lib.semseg_anomaly_metrics_workspace_bytes(2 ** 31 - 1) > 0
    for i in range(5):
        args = [P, P, P, P, P]
        args[i] = None
        assert lib.semseg_anomaly_metrics(args[0], args[1], 8, 100, 255, args[2], args[3], args[4], None) == -1
        assert b"null" in _err()
    assert lib.semseg_anomaly_metrics(P, P, 4, 100, 255, P, P, P, None) == -1 and b"label_bytes" in _err()
    assert lib.semseg_anomaly_metrics(P, P, 8, 0, 255, P, P, P, None) == -1 and b"pixel count" in _err()
