"""CPU tier: the strong view of mean-teacher training (augment.StrongAugment, csrc/strong.cu) — the float64 oracle
against torchvision.transforms.v2.functional (each operation, all 24 orders, hue at +-0.5, saturation 0, blur at sigma
0.1, 2 and 5), the per-image parameters at their edges, the argument checks of StrongAugment, of the three teacher
criteria and of the C entry point."""
import ctypes
import itertools
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200.augment import StrongAugment
from semseg_b200.losses import DistillationLoss, MixPseudoLabelLoss, PseudoLabelLoss
from tests import util
from tests.strong_oracle import OPS, apply_op, blur, chain, gray, params, strong

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch
U_MAX = 1.0 - 2.0 ** -24


def _err():
    return _lib.load().semseg_last_error()


def _image(seed, h=11, w=13):
    g = torch.Generator().manual_seed(seed)
    v = torch.rand((3, h, w), generator=g, dtype=torch.float64)
    v[:, 0, 0] = 0.5                                    # a gray pixel: max == min
    v[:, 0, 1] = torch.tensor([0.9, 0.9, 0.2])          # ties between the channels
    v[:, 0, 2] = torch.tensor([0.1, 0.7, 0.7])
    v[:, 1, 0] = 0.0
    v[:, 1, 1] = 1.0
    return v


# ------------------------------------------------------------------------------------------------ oracle vs torchvision
def _tv(v, name, f):
    TF = pytest.importorskip("torchvision.transforms.v2.functional")
    return {"brightness": TF.adjust_brightness, "contrast": TF.adjust_contrast, "saturation": TF.adjust_saturation,
            "hue": TF.adjust_hue}[name](v, f)


# torchvision's adjust_hue converts to fp32 internally; the other operations stay in float64
TOL = {"brightness": 1e-15, "contrast": 1e-15, "saturation": 1e-15, "hue": 1e-6}


@pytest.mark.parametrize("name,f", [("brightness", 0.5), ("brightness", 1.5), ("brightness", 0.0),
                                    ("contrast", 0.5), ("contrast", 1.5), ("contrast", 0.0),
                                    ("saturation", 0.5), ("saturation", 1.5), ("saturation", 0.0),
                                    ("hue", 0.25), ("hue", -0.25), ("hue", 0.5), ("hue", -0.5), ("hue", 0.0),
                                    ("hue", 0.01)])
def test_each_operation_matches_torchvision(name, f):
    for seed in range(3):
        v = _image(seed)
        got = apply_op(v, name, f)
        ref = _tv(v, name, f)
        assert float((got - ref.double()).abs().max()) <= TOL[name], (name, f)
        assert float(got.min()) >= 0.0 and float(got.max()) <= 1.0


@pytest.mark.parametrize("order", list(itertools.permutations(range(4))), ids=lambda o: "".join(OPS[k][0] for k in o))
def test_all_orders_match_torchvision(order):
    v = _image(7)
    u = np.zeros(12, np.float32)
    u[1:5] = [0.9, 0.1, 0.8, 0.3]
    for pos, k in enumerate(order):
        u[5 + k] = 0.1 + 0.2 * pos                      # operation k runs at position pos
    prm = params(u, 0.5, 0.5, 0.5, 0.25, 0.8, 0.2, 0.5, (0.1, 2.0))
    assert [name for name, _ in prm['ops']] == [OPS[k] for k in order]
    u[10] = 1.0 - 2.0 ** -24
    prm['r'], prm['gray'] = 0, False
    got = chain(v, prm)
    ref = v
    for name, f in prm['ops']:
        ref = _tv(ref.double(), name, f)
    assert float((got - ref.double()).abs().max()) <= 2e-6


def test_grayscale_matches_torchvision():
    TF = pytest.importorskip("torchvision.transforms.v2.functional")
    v = _image(3)
    got = chain(v, {'ops': [], 'gray': True, 'sigma': None, 'r': 0})
    assert float((got - TF.rgb_to_grayscale(v, num_output_channels=3)).abs().max()) <= 1e-15
    assert torch.equal(got[0], gray(v)) and torch.equal(got[1], got[0]) and torch.equal(got[2], got[0])


@pytest.mark.parametrize("sig", [0.1, 2.0, 5.0])
def test_blur_matches_torchvision(sig):
    TF = pytest.importorskip("torchvision.transforms.v2.functional")
    r = math.ceil(3.0 * sig)
    v = _image(5, 17, 23)
    got = blur(v, sig, r)
    ref = TF.gaussian_blur(v, [2 * r + 1, 2 * r + 1], [sig, sig])
    assert float((got - ref).abs().max()) <= 1e-12
    if sig == 0.1:                                      # one tap either side, weight ~2e-22: the image itself
        assert float((got - v).abs().max()) <= 1e-20


# ------------------------------------------------------------------------------------------------ parameters
def test_params_ranges_order_and_skips():
    u = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.5, 0.5, 0.5, 0.5, 0.0, 0.0, 0.0], np.float32)
    prm = params(u, 0.5, 1.5, 0.5, 0.25, 0.8, 0.2, 0.5, (0.1, 2.0))
    assert prm['ops'] == [("brightness", 0.5), ("contrast", 0.0), ("saturation", 0.5), ("hue", -0.25)]  # ties: index
    assert prm['gray'] and prm['sigma'] == np.float32(0.1) and prm['r'] == 1
    u[1:5] = U_MAX
    u[11] = U_MAX
    prm = params(u, 0.5, 1.5, 0.5, 0.25, 0.8, 0.2, 0.5, (0.1, 2.0))
    assert [f for _, f in prm['ops']] == [np.float32(0.5 + U_MAX), np.float32(2.5 * U_MAX),
                                          np.float32(0.5 + U_MAX), np.float32(-0.25 + 0.5 * U_MAX)]
    assert prm['r'] == 6
    # a strength of 0 skips its operation; probability 0 applies nothing, 1 everything
    assert [n for n, _ in params(u, 0.0, 0.5, 0.0, 0.0, 1.0, 0, 0, (1, 1))['ops']] == ["contrast"]
    assert params(u, 0.5, 0.5, 0.5, 0.5, 0.0, 0.0, 0.0, (1, 1)) == {'ops': [], 'gray': False, 'sigma': None, 'r': 0}
    u[[0, 9, 10]] = U_MAX
    prm = params(u, 0.5, 0.5, 0.5, 0.5, 1.0, 1.0, 1.0, (5.0, 5.0))
    assert len(prm['ops']) == 4 and prm['gray'] and prm['r'] == 15


def test_oracle_copies_untouched_images():
    g = torch.Generator().manual_seed(0)
    x = torch.randn((3, 3, 9, 9), generator=g) * 4
    u = torch.rand((3, 12), generator=g)
    u[0, [0, 9, 10]] = 0.99                             # no operation applies
    out = strong(x, u)
    assert torch.equal(out[0], x[0].double())
    ref = strong(x, u, p_jitter=0.0, p_gray=0.0, p_blur=0.0)
    assert torch.equal(ref, x.double())


# ------------------------------------------------------------------------------------------------ argument checks
def test_strong_augment_defaults_validation_and_repr():
    s = StrongAugment()
    assert (s.brightness, s.contrast, s.saturation, s.hue) == (0.5, 0.5, 0.5, 0.25)
    assert (s.p_jitter, s.p_gray, s.p_blur, s.sigma) == (0.8, 0.2, 0.5, (0.1, 2.0))
    assert s.mean == (0.485 * 255, 0.456 * 255, 0.406 * 255) and s.std == (0.229 * 255, 0.224 * 255, 0.225 * 255)
    r = repr(s)
    assert r.startswith("StrongAugment(") and "hue=0.25" in r and "sigma=(0.1, 2)" in r
    s = StrongAugment(brightness=0, hue=0.5, p_jitter=1, p_gray=0, sigma=[5, 5], mean=[0, 0, 0], std=[1, 2, 3])
    assert (s.brightness, s.hue, s.p_jitter, s.sigma, s.std) == (0.0, 0.5, 1.0, (5.0, 5.0), (1.0, 2.0, 3.0))
    for kw in ({"brightness": "0.5"}, {"hue": None}, {"p_gray": True}, {"sigma": 1.0}, {"sigma": (1.0, "2")},
               {"mean": (0, 0, "0")}):
        with pytest.raises(TypeError):
            StrongAugment(**kw)
    for kw in ({"brightness": -0.1}, {"contrast": float("inf")}, {"saturation": float("nan")}, {"hue": 0.51},
               {"p_jitter": -0.1}, {"p_gray": 1.01}, {"p_blur": float("nan")}, {"sigma": (0.0, 1.0)},
               {"sigma": (2.0, 1.0)}, {"sigma": (1.0, 5.01)}, {"std": (1, 0, 1)}, {"std": (1, -1, 1)},
               {"mean": (0, 0)}, {"std": (1, 1, 1, 1)}, {"mean": (0, float("nan"), 0)}):
        with pytest.raises(ValueError):
            StrongAugment(**kw)


def test_strong_augment_input_checks():
    s = StrongAugment(sigma=(0.1, 2.0))
    with pytest.raises(RuntimeError, match="no gradient through the strong view"):
        s(torch.zeros((1, 3, 9, 9)).requires_grad_(True))
    for bad in (torch.zeros((1, 3, 9, 9)), torch.zeros((1, 3, 9, 9), dtype=torch.float64), torch.zeros((3, 9, 9)),
                np.zeros((1, 3, 9, 9), np.float32)):
        with pytest.raises(TypeError):
            s.draw(bad)


@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


@pytest.mark.parametrize("cls", [DistillationLoss, PseudoLabelLoss, MixPseudoLabelLoss])
def test_teacher_losses_take_strong(cls, nets):
    teacher = nets[1]
    plain = cls(teacher)
    assert plain.strong is None and plain.last_strong() is None and "strong" not in repr(plain)
    s = StrongAugment(p_gray=0.3)
    d = cls(teacher, strong=s)
    assert d.strong is s and d.last_strong() is None
    assert "strong=StrongAugment(" in repr(d) and "p_gray=0.3" in repr(d)
    assert list(d.state_dict()) == [] and list(d.children()) == []
    for bad in (1, "strong", nn.Identity(), (0.5, 0.5)):
        with pytest.raises(TypeError, match="StrongAugment"):
            cls(teacher, strong=bad)


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _call(x=P, N=2, C=3, H=17, W=17, u=P, us=12, b=0.5, c=0.5, s=0.5, h=0.25, pj=0.8, pg=0.2, pb=0.5, slo=0.1,
          shi=2.0, mean=(1.0, 2.0, 3.0), std=(1.0, 1.0, 1.0), ws=P, out=ctypes.c_void_p(32)):
    m3 = (ctypes.c_float * 3)(*mean) if mean is not None else None
    s3 = (ctypes.c_float * 3)(*std) if std is not None else None
    return _lib.load().semseg_strong_augment(x, N, C, H, W, u, us, b, c, s, h, pj, pg, pb, slo, shi, m3, s3, ws, out,
                                             None)


def test_strong_entry_point_validates():
    for kw in ("x", "u", "ws", "out", "mean", "std"):
        assert _call(**{kw: None}) == -1 and b"null" in _err(), kw
    assert _call(out=P) == -1 and b"overwrite" in _err()
    for C in (1, 4):
        assert _call(C=C) == -1 and b"channels" in _err()
    assert _call(N=0) == -1 and b"batch" in _err()
    assert _call(us=11) == -1 and b"stride" in _err()
    for kw in ({"b": -0.1}, {"c": float("nan")}, {"s": float("inf")}, {"h": -0.1}):
        assert _call(**kw) == -1 and b"strength" in _err(), kw
    assert _call(h=0.6) == -1 and b"hue" in _err()
    for kw in ({"pj": -0.1}, {"pg": 1.1}, {"pb": float("nan")}):
        assert _call(**kw) == -1 and b"probability" in _err(), kw
    for slo, shi in ((0.0, 1.0), (2.0, 1.0), (1.0, 5.5), (float("nan"), 1.0)):
        assert _call(slo=slo, shi=shi) == -1 and b"sigma" in _err(), (slo, shi)
    assert _call(std=(1.0, 0.0, 1.0)) == -1 and b"std[1]" in _err()
    assert _call(mean=(1.0, float("inf"), 1.0)) == -1 and b"mean[1]" in _err()
    # H, W must exceed r = ceil(3 sigma_hi): 6 at sigma_hi = 2, 15 at 5
    assert _call(H=6) == -1 and b"ceil(3 sigma_hi) = 6" in _err()
    assert _call(W=6) == -1 and b"ceil(3 sigma_hi) = 6" in _err()
    assert _call(H=15, W=40, shi=5.0) == -1 and b"= 15" in _err()
