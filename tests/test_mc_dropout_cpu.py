"""CPU tier for Monte Carlo dropout in the sliding-window predictor (semseg_b200/inference.py, mc_draws > 0): the
options' validation, the rejection of bad arguments by semseg_window_scores_mc before any CUDA call, the ATen path on a
tiny CPU network with a Dropout2d, and the float64 oracle (tests/mc_oracle.py) against a direct per-pixel loop."""
import ctypes
import math

import numpy as np
import pytest
import torch
from torch import nn

from semseg_b200 import _lib
from semseg_b200.inference import SlidingWindowPredictor, crop_origins, scaled_size
from tests import mc_oracle as O
from tests import util

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch
CLASSES = 5
MEAN, STD = util.SW_CFG["mean"], util.SW_CFG["std"]


def _err():
    return _lib.load().semseg_last_error()


class _TinyNet(nn.Module):
    """conv 3x3 -> ReLU -> Dropout2d -> 1x1 conv at half resolution (odd sizes: 2(h'-1)+1), so the predictor's ATen
    steps upsample the logits to the crop. `fail` makes the forward raise after the dropout."""

    def __init__(self, p=0.5, seed=0):
        super().__init__()
        torch.manual_seed(seed)
        self.body = nn.Conv2d(3, 16, 3, stride=2, padding=1)
        self.act = nn.ReLU()
        self.drop = nn.Dropout2d(p)
        self.aux_drop = nn.Dropout(0.2)          # a second dropout module: its own mode is restored too
        self.head = nn.Conv2d(16, CLASSES, 1)
        self.fail = False

    def forward(self, x):
        t = self.drop(self.act(self.body(x)))
        if self.fail:
            raise RuntimeError("forward failed")
        return self.head(t) * 3.0


def _predictor(net, crop=17, **kw):
    kw.setdefault("mc_draws", 4)
    kw.setdefault("max_batch", 4)
    return SlidingWindowPredictor(net, CLASSES, crop, crop, MEAN, STD, **kw)


# ------------------------------------------------------------------------------------------------ validation
def test_mc_draws_validation():
    net = _TinyNet().eval()
    for bad in (1.5, "3", True, None, torch.tensor(2)):
        with pytest.raises(TypeError):
            _predictor(net, mc_draws=bad)
    for bad in (-1, 129, 1000):
        with pytest.raises(ValueError):
            _predictor(net, mc_draws=bad)
    assert _predictor(net, mc_draws=0).mc_draws == 0
    assert _predictor(net, mc_draws=np.int64(128)).mc_draws == 128


def test_mc_draws_rejects_unsupported_combinations():
    from semseg_b200.anomaly import AnomalyScorer
    from semseg_b200.densecrf import DenseCRF
    from semseg_b200.fp8 import Fp8Eval
    net = _TinyNet().eval()
    with pytest.raises(ValueError):
        _predictor(net, crf=DenseCRF())
    with pytest.raises(ValueError):
        _predictor(net, anomaly=AnomalyScorer("msp"))
    fp8 = Fp8Eval.__new__(Fp8Eval)           # the type alone is refused; a real wrapper needs a CUDA network
    fp8.model = net
    with pytest.raises(ValueError):
        _predictor(fp8)
    with pytest.raises(ValueError):          # no dropout layer
        _predictor(nn.Sequential(nn.Conv2d(3, CLASSES, 1)).eval())
    zero = _TinyNet(p=0.0).eval()
    zero.aux_drop.p = 0.0
    with pytest.raises(ValueError):          # every dropout p == 0
        _predictor(zero)
    with pytest.raises(ValueError):
        _predictor(net)(util.sw_image(seed=1, h=20, w=24), 24, [1.0], exact=True)
    # the deterministic predictor keeps accepting what it accepted
    _predictor(zero, mc_draws=0, crf=DenseCRF())


# ------------------------------------------------------------------------------------------------ entry point
def test_window_scores_mc_rejects_bad_arguments():
    lib = _lib.load()
    f = lib.semseg_window_scores_mc
    assert f(None, 19, 2, 1, 9, 9, 19, 1, P, 65, 65, None) == -1 and b"null" in _err()
    assert f(P, 19, 2, 1, 9, 9, 19, 1, None, 65, 65, None) == -1 and b"null" in _err()
    assert f(P, 19, 0, 1, 9, 9, 19, 1, P, 65, 65, None) == -1 and b"draws" in _err()
    assert f(P, 19, 129, 1, 9, 9, 19, 1, P, 65, 65, None) == -1 and b"draws" in _err()
    assert f(P, 300, 2, 1, 9, 9, 257, 1, P, 65, 65, None) == -1 and b"bad sizes" in _err()
    assert f(P, 18, 2, 1, 9, 9, 19, 1, P, 65, 65, None) == -1 and b"bad sizes" in _err()
    assert f(P, 19, 2, 1, 9, 9, 19, 2, P, 65, 65, None) == -1 and b"bad sizes" in _err()
    assert f(P, 19, 2, 1, 9, 9, 19, 1, P, 64, 65, None) == -1 and b"8(h-1)+1" in _err()
    assert f(P, 19, 2, 1, 9, 9, 19, 1, P, 65, 73, None) == -1 and b"8(h-1)+1" in _err()
    assert b"window_scores_mc" in _err()


# ------------------------------------------------------------------------------------------------ ATen path
def _run(net, image, seed, base=24, scales=(1.0,), return_scores=True, **kw):
    p = _predictor(net, **kw)
    torch.manual_seed(seed)
    return p, p(image, base, list(scales), return_scores=return_scores)


def test_aten_path_same_seed_same_bits_and_different_seed_differs():
    net = _TinyNet().eval()
    image = util.sw_image(seed=2, h=20, w=24)
    _, (s1, a1, u1) = _run(net, image, 7, scales=(0.75, 1.0))
    _, (s2, a2, u2) = _run(net, image, 7, scales=(0.75, 1.0))
    _, (s3, _, u3) = _run(net, image, 8, scales=(0.75, 1.0))
    assert np.array_equal(s1, s2) and np.array_equal(a1, a2) and torch.equal(u1, u2)
    assert not np.array_equal(s1, s3) and not torch.equal(u1, u3)
    assert u1.dtype == torch.float32 and tuple(u1.shape) == (2, 20, 24) and s1.shape == (20, 24, CLASSES)
    none, a4, u4 = _run(net, image, 7, scales=(0.75, 1.0), return_scores=False)[1]
    assert none is None and np.array_equal(a4, a1) and torch.equal(u4, u1)
    assert np.array_equal(a1, np.argmax(s1, axis=2))


def test_aten_path_restores_dropout_modes():
    net = _TinyNet().eval()
    net.aux_drop.train()                     # mixed modes: each module gets its own back
    image = util.sw_image(seed=3, h=20, w=24)
    _run(net, image, 1)
    assert not net.drop.training and net.aux_drop.training and not net.training
    net.fail = True
    with pytest.raises(RuntimeError):
        _run(net, image, 1)
    assert not net.drop.training and net.aux_drop.training and not net.training


@pytest.mark.parametrize("flip", [True, False])
def test_aten_path_counts_forward_calls_and_keeps_its_invariants(flip):
    net = _TinyNet().eval()
    image = util.sw_image(seed=4, h=30, w=41)
    draws, base, scales, crop, max_batch = 3, 41, (0.5, 1.0, 1.25), 17, 4
    p, (scores, _, unc) = _run(net, image, 5, base=base, scales=scales, mc_draws=draws, flip=flip, crop=crop,
                               max_batch=max_batch)
    per_call = max_batch // 2 if flip else max_batch
    batches = 0
    for s in scales:
        nh, nw = scaled_size(30, 41, round(s * base))
        k = len(crop_origins(max(nh, crop), crop)) * len(crop_origins(max(nw, crop), crop))
        batches += math.ceil(k / per_call)
    assert p.forward_calls == draws * batches
    assert float(unc[1].min()) >= -1e-12
    assert float(unc[0].min()) >= 0.0 and float(unc[0].max()) <= math.log(CLASSES) + 1e-6
    # each sample's softmax is fp32: its class sum is 1 to a few fp32 ulps, and so is their mean
    assert np.abs(scores.sum(2) - 1.0).max() <= 4 * CLASSES * 2.0 ** -24


def test_single_sample_has_zero_mutual_information():
    """T = 1, no flip, one crop, one scale: p_bar is that crop's softmax, so H[p_bar] is its entropy and the mutual
    information vanishes. Both hold up to the fp32 rounding of the sample's softmax and entropy: the sample entropy
    enters the total in fp32, H[p_bar] is taken in fp64 from the fp32 softmax."""
    net = _TinyNet().eval()
    crop = 17
    image = util.sw_image(seed=6, h=crop, w=crop)
    p, (scores, _, unc) = _run(net, image, 9, base=crop, mc_draws=1, flip=False, crop=crop)
    assert p.forward_calls == 1
    torch.manual_seed(9)
    net.drop.train()
    with torch.no_grad():
        logits = net(p._normalised(image)[None])
    net.drop.eval()
    up = torch.nn.functional.interpolate(logits, (crop, crop), mode="bilinear", align_corners=True)
    q = torch.softmax(up.float(), 1)[0].double()
    assert np.array_equal(scores, q.permute(1, 2, 0).numpy())
    ent = -(q * q.log()).sum(0)
    assert float((unc[0].double() - ent).abs().max()) <= 1e-6
    assert float(unc[1].abs().max()) <= 1e-6


def test_mc_draws_zero_is_the_deterministic_predictor():
    net = _TinyNet().eval()
    image = util.sw_image(seed=7, h=20, w=24)
    ref = SlidingWindowPredictor(net, CLASSES, 17, 17, MEAN, STD, max_batch=4)(image, 24, [1.0, 1.5])
    got = _predictor(net, mc_draws=0)(image, 24, [1.0, 1.5])
    assert len(got) == 2 and np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


# ------------------------------------------------------------------------------------------------ oracle
def _loop_mc(logits, flip):
    """Direct per-pixel restatement of mc_oracle.mc_scores in Python floats."""
    T, n, h, w, c = logits.shape
    G = n // 2 if flip else n
    H, W = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    out = np.zeros((G, c + 1, H, W))

    def sample(t, im, y, x):
        i0, fy = min(y // 8, h - 1), (y % 8) / 8.0
        j0, fx = min(x // 8, w - 1), (x % 8) / 8.0
        i1, j1 = min(i0 + 1, h - 1), min(j0 + 1, w - 1)
        v = [(1 - fy) * ((1 - fx) * logits[t, im, i0, j0, k] + fx * logits[t, im, i0, j1, k]) +
             fy * ((1 - fx) * logits[t, im, i1, j0, k] + fx * logits[t, im, i1, j1, k]) for k in range(c)]
        m = max(v)
        e = [math.exp(a - m) for a in v]
        s = sum(e)
        q = [a / s for a in e]
        return q + [-sum(a * math.log(a) for a in q if a > 0)]

    for g in range(G):
        for y in range(H):
            for x in range(W):
                acc = np.zeros(c + 1)
                for t in range(T):
                    a = np.array(sample(t, g, y, x))
                    if flip:
                        a = (a + np.array(sample(t, G + g, y, W - 1 - x))) / 2
                    acc += a
                out[g, :, y, x] = acc / T
    return out


@pytest.mark.parametrize("flip", [True, False])
def test_oracle_matches_per_pixel_loop(flip):
    gen = torch.Generator().manual_seed(int(flip))
    T, G, h, w, c = 3, 2, 3, 4, 4
    logits = torch.randn((T, 2 * G if flip else G, h, w, c), generator=gen, dtype=torch.float64) * 3
    got = O.mc_scores(logits, flip).numpy()
    ref = _loop_mc(logits.numpy(), flip)
    assert np.allclose(got, ref, rtol=0, atol=1e-12)
    total = torch.from_numpy(ref[0])
    unc = O.uncertainty(total, c).numpy()
    pbar = ref[0, :c]
    hbar = -(pbar * np.log(pbar)).sum(0)
    assert np.allclose(unc[0], hbar, rtol=0, atol=1e-12)
    assert np.allclose(unc[1], hbar - ref[0, c], rtol=0, atol=1e-12)
    assert unc[1].min() >= -1e-12                    # the Jensen gap


def test_oracle_entropy_takes_zero_probabilities_as_zero():
    total = torch.zeros((3, 1, 2), dtype=torch.float64)
    total[0] = 1.0
    unc = O.uncertainty(total, 2)
    assert torch.equal(unc, torch.zeros((2, 1, 2), dtype=torch.float64))
