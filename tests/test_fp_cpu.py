"""CPU tier for the feature-perturbation stream of losses.PseudoLabelLoss / MixPseudoLabelLoss (fp_weight, fp_dropout):
option validation and repr, last_fp() before a forward, the fork / fold entry points' argument checks, and the oracle
of tests/fp_oracle.py against float64 autograd of its definition."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import _lib
from semseg_b200.losses import DistillationLoss, MixPseudoLabelLoss, PseudoLabelLoss
from tests import util
from tests.fp_oracle import fold, fork, fp_definition, fp_grad
from tests.pl_oracle import effective, pl_definition, pl_grad

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


# ------------------------------------------------------------------------------------------------ options
@pytest.mark.parametrize("cls", [PseudoLabelLoss, MixPseudoLabelLoss])
def test_fp_options_validation_and_repr(cls, nets):
    teacher = nets[1]
    d = cls(teacher)
    assert d.fp_weight == 0.0 and d.fp_dropout == 0.5
    assert "fp_weight=0, fp_dropout=0.5" in repr(d)
    c = cls(teacher, fp_weight=0.25, fp_dropout=0)
    assert c.fp_weight == 0.25 and c.fp_dropout == 0.0 and isinstance(c.fp_dropout, float)
    assert "fp_weight=0.25, fp_dropout=0" in repr(c)
    for kw in ({"fp_weight": True}, {"fp_weight": "0.5"}, {"fp_weight": None}, {"fp_dropout": False},
               {"fp_dropout": "0.5"}, {"fp_dropout": torch.tensor(0.5)}):
        with pytest.raises(TypeError):
            cls(teacher, **kw)
    for kw in ({"fp_weight": -0.1}, {"fp_weight": float("nan")}, {"fp_weight": float("inf")}, {"fp_dropout": 1},
               {"fp_dropout": 1.0}, {"fp_dropout": 1.5}, {"fp_dropout": -0.1}, {"fp_dropout": float("nan")}):
        with pytest.raises(ValueError):
            cls(teacher, **kw)
    assert cls(teacher, fp_weight=1.0, fp_dropout=0.999).fp_dropout == 0.999


@pytest.mark.parametrize("cls", [PseudoLabelLoss, MixPseudoLabelLoss])
def test_last_fp_is_none_before_a_forward(cls, nets):
    assert cls(nets[1]).last_fp() is None
    assert cls(nets[1], fp_weight=0.5).last_fp() is None


def test_distillation_loss_has_no_fp_options(nets):
    with pytest.raises(TypeError):
        DistillationLoss(nets[1], fp_weight=0.5)
    assert not hasattr(DistillationLoss(nets[1]), "fp_weight")


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _call(fn, x=P, x_lo=None, xp=16, s=P, out=ctypes.c_void_p(32), out_lo=None, op=16, N=2, HW=5, C=16):
    return getattr(_lib.load(), fn)(x, x_lo, xp, s, out, out_lo, op, N, HW, C, None)


@pytest.mark.parametrize("fn", ["semseg_fp_fork", "semseg_fp_fold"])
def test_fork_fold_entry_points_validate(fn):
    name = fn[len("semseg_"):].encode()
    for kw in ("x", "s", "out"):
        assert _call(fn, **{kw: None}) == -1 and b"null" in _err(), kw
    for kw in ({"N": 0}, {"HW": 0}, {"C": 0}, {"C": 12}):
        assert _call(fn, **kw) == -1 and name in _err(), kw
    for kw in ({"xp": 8}, {"op": 8}, {"xp": 20}, {"op": 20}):
        assert _call(fn, **kw) == -1 and b"pitch" in _err(), kw
    assert _call(fn, x_lo=ctypes.c_void_p(48)) == -1 and b"storage form" in _err()
    assert _call(fn, out_lo=ctypes.c_void_p(48)) == -1 and b"storage form" in _err()
    assert _call(fn, s=ctypes.c_void_p(20)) == -1 and b"scale" in _err()
    assert _call(fn, x=ctypes.c_void_p(24)) == -1 and b"aligned" in _err()


# ------------------------------------------------------------------------------------------------ oracle
def _stream(F2, w1, w2):
    """A small stand-in for the context module and cls on the 2N batch: 1x1 conv, batch-statistics BatchNorm over all
    2N images, ReLU, 1x1 conv -> NHWC logits."""
    t = F.conv2d(F2, w1)
    t = F.relu(F.batch_norm(t, None, None, training=True))
    return F.conv2d(t, w2).permute(0, 2, 3, 1)


@pytest.mark.parametrize("dropout", [0.0, 0.3, 0.5])
@pytest.mark.parametrize("threshold", [0.0, 0.5])
@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_fp_gradient_equals_autograd(zoom, threshold, dropout):
    """The closed form the kernels implement, the PL gradient on both streams' logits taken back through the stream
    and folded d[:N] + s d[N:], equals float64 autograd of the definition through the fork to 1e-12 of max |grad|."""
    g = torch.Generator().manual_seed(zoom * 10 + int(dropout * 10))
    n, cf, h, w, c = 3, 16, 5, 6, 7
    f = torch.randn((n, cf, h, w), generator=g, dtype=torch.float64)
    u = torch.rand((n, cf), generator=g)
    keep = 1.0 - dropout
    s = (u < keep).float().div_(keep)
    w1 = torch.randn((12, cf, 1, 1), generator=g, dtype=torch.float64) * 0.3
    w2 = torch.randn((c, 12, 1, 1), generator=g, dtype=torch.float64) * 0.5
    t = torch.randn((n, h, w, c), generator=g, dtype=torch.float64) * 3
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    y = torch.randint(0, c, (n, ho, wo), generator=g)
    y[0] = 255                                                  # an unlabelled image
    y[1][torch.rand((ho, wo), generator=g) < 0.5] = 255         # a partly labelled one
    pl_w, ce_w, fp_w = 0.7, 1.0, 0.4

    fd = f.clone().requires_grad_(True)
    logits = _stream(fork(fd, s), w1, w2)
    main = pl_definition(logits[:n], t, y, zoom, threshold, pl_w, ce_w) + \
        fp_definition(logits[n:], t, y, zoom, threshold, fp_w)
    (g_a,) = torch.autograd.grad(main, fd)

    lg = logits.detach()
    eff, wt, _ = effective(t, y, zoom, threshold, pl_w, ce_w)
    d_logits = torch.cat([pl_grad(lg[:n], eff, wt, zoom), fp_grad(lg[n:], t, y, zoom, threshold, fp_w)], 0)
    F2 = fork(f, s).requires_grad_(True)
    (d_f2,) = torch.autograd.grad(_stream(F2, w1, w2), F2, d_logits)
    g_c = fold(d_f2, s)
    scale = float(g_a.abs().max())
    assert scale > 0
    assert float((g_c - g_a).abs().max()) <= 1e-12 * scale


def test_oracle_fp_term_of_an_empty_set_is_zero():
    g = torch.Generator().manual_seed(3)
    s = torch.randn((2, 4, 5, 6), generator=g, dtype=torch.float64, requires_grad=True)
    t = torch.randn((2, 4, 5, 6), generator=g, dtype=torch.float64)
    y = torch.randint(0, 6, (2, 25, 33), generator=g)           # every pixel labelled: U is empty
    loss = fp_definition(s, t, y, 8, 0.0, 0.5)
    (gs,) = torch.autograd.grad(loss, s)
    assert loss.item() == 0.0 and float(gs.abs().max()) == 0.0
    assert float(fp_grad(s, t, y, 8, 0.0, 0.5).abs().max()) == 0.0
