"""CPU tier for the dual-stream perturbation of losses.PseudoLabelLoss / MixPseudoLabelLoss (streams=2): option
validation and repr, the prefix fork / fold entry points' argument checks, and the oracle of tests/dual_oracle.py
against float64 autograd of its definition."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import _lib
from semseg_b200.augment import StrongAugment
from semseg_b200.losses import DistillationLoss, MixPseudoLabelLoss, PseudoLabelLoss
from tests import util
from tests.dual_oracle import dual_definition, dual_grad, fold, fork

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


# ------------------------------------------------------------------------------------------------ options
@pytest.mark.parametrize("cls", [PseudoLabelLoss, MixPseudoLabelLoss])
def test_streams_validation_and_repr(cls, nets):
    teacher = nets[1]
    d = cls(teacher, strong=StrongAugment())
    assert d.streams == 1 and "streams" not in repr(d)
    c = cls(teacher, strong=StrongAugment(), streams=2)
    assert c.streams == 2 and type(c.streams) is int
    assert ", streams=2" in repr(c)
    for v in (True, False):
        with pytest.raises(TypeError):
            cls(teacher, strong=StrongAugment(), streams=v)
    for v in (0, 3, -1, 2.0, 1.5, "2", None, torch.tensor(2)):
        with pytest.raises(ValueError):
            cls(teacher, strong=StrongAugment(), streams=v)


def test_two_streams_of_the_plain_criterion_need_a_strong_view(nets):
    with pytest.raises(ValueError, match="strong"):
        PseudoLabelLoss(nets[1], streams=2)
    assert PseudoLabelLoss(nets[1], streams=1).streams == 1
    # the mix criterion's two streams differ by their boxes or class sets
    for mix in ("cutmix", "classmix"):
        assert MixPseudoLabelLoss(nets[1], mix=mix, streams=2).streams == 2


def test_distillation_loss_has_no_streams(nets):
    with pytest.raises(TypeError):
        DistillationLoss(nets[1], strong=StrongAugment(), streams=2)
    assert not hasattr(DistillationLoss(nets[1]), "streams")


def test_strong_draw_takes_views():
    """StrongAugment.draw's shape check runs before any draw; the row count is views * N."""
    s = StrongAugment()
    with pytest.raises(TypeError):
        s.draw(torch.zeros((2, 3, 17, 17)), 2)          # a CPU input: refused before torch.rand


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _call(fn, x=P, x_lo=None, xp=16, s=P, out=ctypes.c_void_p(32), out_lo=None, op=16, M=4, N=2, HW=5, C=16):
    return getattr(_lib.load(), fn)(x, x_lo, xp, s, out, out_lo, op, M, N, HW, C, None)


@pytest.mark.parametrize("fn", ["semseg_fp_fork_prefix", "semseg_fp_fold_prefix"])
def test_prefix_fork_fold_entry_points_validate(fn):
    name = fn[len("semseg_"):].encode()
    for kw in ("x", "s", "out"):
        assert _call(fn, **{kw: None}) == -1 and b"null" in _err(), kw
    for kw in ({"N": 0}, {"HW": 0}, {"C": 0}, {"C": 12}):
        assert _call(fn, **kw) == -1 and name in _err(), kw
    for kw in ({"M": 1}, {"M": 0}, {"M": -4}, {"M": 3, "N": 4}):
        assert _call(fn, **kw) == -1 and b"M >= N" in _err() and name in _err(), kw
    for kw in ({"xp": 8}, {"op": 8}, {"xp": 20}, {"op": 20}):
        assert _call(fn, **kw) == -1 and b"pitch" in _err(), kw
    assert _call(fn, x_lo=ctypes.c_void_p(48)) == -1 and b"storage form" in _err()
    assert _call(fn, out_lo=ctypes.c_void_p(48)) == -1 and b"storage form" in _err()
    assert _call(fn, s=ctypes.c_void_p(20)) == -1 and b"scale" in _err()
    assert _call(fn, x=ctypes.c_void_p(24)) == -1 and b"aligned" in _err()


# ------------------------------------------------------------------------------------------------ oracle
def test_oracle_fork_and_fold_are_adjoint():
    g = torch.Generator().manual_seed(1)
    for m, n in ((2, 1), (6, 3), (5, 2), (3, 3)):
        f = torch.randn((m, 4, 3, 2), generator=g, dtype=torch.float64)
        d = torch.randn((m + n, 4, 3, 2), generator=g, dtype=torch.float64)
        s = torch.rand((n, 4), generator=g, dtype=torch.float64)
        assert fork(f, s).shape[0] == m + n and fold(d, s).shape[0] == m
        assert abs(float((fork(f, s) * d).sum() - (f * fold(d, s)).sum())) <= 1e-12 * float(d.abs().sum())


def _body(x, w0):
    """A small stand-in for the backbone on the 2N views: 1x1 conv, batch-statistics BatchNorm over all 2N images."""
    return F.relu(F.batch_norm(F.conv2d(x, w0), None, None, training=True))


def _stream(F3, w1, w2):
    """A small stand-in for the context module and cls on [f_1, f_2, f_1 * s]: 1x1 conv, batch-statistics BatchNorm
    over all the images, ReLU, 1x1 conv -> NHWC logits."""
    t = F.conv2d(F3, w1)
    t = F.relu(F.batch_norm(t, None, None, training=True))
    return F.conv2d(t, w2).permute(0, 2, 3, 1)


@pytest.mark.parametrize("fp", [False, True], ids=["no_fp", "fp"])
@pytest.mark.parametrize("threshold", [0.0, 0.5])
@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_dual_gradient_equals_autograd(zoom, threshold, fp):
    """The closed form the kernels implement, each stream's PL gradient halved and the FP gradient of the perturbed
    rows, taken back through the head and folded d[:2N] + s d[2N:] into the first N images, then through the body on
    the 2N views, equals float64 autograd of the definition to 1e-12 of max |grad|."""
    g = torch.Generator().manual_seed(zoom * 10 + int(threshold * 10) + fp)
    n, cin, cf, h, w, c = 3, 5, 16, 5, 6, 7
    x2 = torch.randn((2 * n, cin, h, w), generator=g, dtype=torch.float64)
    w0 = torch.randn((cf, cin, 1, 1), generator=g, dtype=torch.float64) * 0.5
    u = torch.rand((n, cf), generator=g)
    s = (u < 0.5).float().div_(0.5) if fp else None
    w1 = torch.randn((12, cf, 1, 1), generator=g, dtype=torch.float64) * 0.3
    w2 = torch.randn((c, 12, 1, 1), generator=g, dtype=torch.float64) * 0.5
    t = torch.randn((n, h, w, c), generator=g, dtype=torch.float64) * 3
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    ys = []
    for k in range(2):
        y = torch.randint(0, c, (n, ho, wo), generator=g)
        y[k] = 255                                                  # an unlabelled image
        y[2][torch.rand((ho, wo), generator=g) < 0.5] = 255         # a partly labelled one
        ys.append(y)
    pl_w, ce_w, fp_w = 0.7, 1.0, 0.4

    xd = x2.clone().requires_grad_(True)
    f = _body(xd, w0)
    logits = _stream(fork(f, s) if fp else f, w1, w2)
    main = dual_definition(logits, t, ys, zoom, threshold, pl_w, ce_w, fp_w)
    (g_a,) = torch.autograd.grad(main, xd)

    d_logits = dual_grad(logits.detach(), t, ys, zoom, threshold, pl_w, ce_w, fp_w)
    xc = x2.clone().requires_grad_(True)
    fc = _body(xc, w0)
    F3 = (fork(fc, s) if fp else fc).detach().requires_grad_(True)
    (d_f3,) = torch.autograd.grad(_stream(F3, w1, w2), F3, d_logits)
    (g_c,) = torch.autograd.grad(fc, xc, fold(d_f3, s) if fp else d_f3)
    scale = float(g_a.abs().max())
    assert scale > 0
    assert float((g_c - g_a).abs().max()) <= 1e-12 * scale


def test_oracle_two_equal_streams_are_one_stream():
    """Two equal streams give the one-stream loss: the mean of two equal terms (the BatchNorm of a duplicated batch has
    the same statistics, so the logits of each copy are the one-stream ones)."""
    from tests.pl_oracle import pl_definition
    g = torch.Generator().manual_seed(5)
    n, h, w, c = 2, 4, 5, 6
    s1 = torch.randn((n, h, w, c), generator=g, dtype=torch.float64)
    t = torch.randn((n, h, w, c), generator=g, dtype=torch.float64)
    y = torch.randint(0, c, (n, 25, 33), generator=g)
    y[0] = 255
    one = pl_definition(s1, t, y, 8, 0.0, 0.7, 1.0)
    two = dual_definition(torch.cat([s1, s1]), t, [y, y], 8, 0.0, 0.7, 1.0, 0.0)
    assert abs(float(one - two)) <= 1e-14 * abs(float(one))
