"""CPU tier for entropy minimisation on the fused tail (csrc/tail.cu entropy kernels) and test-time adaptation
(semseg_b200/adapt.py): the float64 oracle of the GPU tests has the gradient of its own definition under autograd, with
mixed, all-unlabelled and all-labelled targets, out-of-range targets and at every zoom; EntropyLoss validates its options;
`fused_tail_supported` takes the native tail exactly where the kernels apply; the entry points reject bad arguments with
SEMSEG_E_INVALID and a message before any CUDA call; and Tent rejects a network it cannot adapt."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import EntropyLoss, FocalLoss
from tests.entropy_oracle import entropy_definition, entropy_loss, entropy_tail

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _case(kind, seed=7, n=2, c=5, h=6, w=7, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * scale
    y = torch.randint(0, c, (n, h, w), generator=g)
    if kind == "mixed":
        y[torch.rand((n, h, w), generator=g) < 0.4] = 255
        y[0, 0, 0], y[0, 0, 1] = c + 2, -3                  # out of range: in neither set
    elif kind == "all-U":
        y[:] = 255
    elif kind == "no-U":
        y[0, 1, 1] = c                                      # out of range
    return x, y


KINDS = ["mixed", "all-U", "no-U"]
WEIGHTS = [(1.0, 1.0), (1.0, 0.0), (0.0, 1.0), (0.3, 2.5)]


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("weights", WEIGHTS, ids=["1-1", "ent-only", "ce-only", "0.3-2.5"])
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_closed_form_equals_autograd_of_the_definition(kind, weights):
    ent_w, ce_w = weights
    x, y = _case(kind)
    xr = x.clone().requires_grad_(True)
    ref = entropy_definition(xr, y, ent_w, ce_w)
    (g_ref,) = torch.autograd.grad(ref, xr)
    loss, nl, nu, ent, grad = entropy_loss(x, y, ent_w, ce_w)
    assert nl == int(((y != 255) & (y >= 0) & (y < 5)).sum()) and nu == int((y == 255).sum())
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12, abs_tol=1e-15)
    assert float((grad - g_ref).abs().max()) <= 1e-12 * max(float(g_ref.abs().max()), 1e-300)
    assert bool((ent >= 0).all()) and bool((ent <= math.log(5) + 1e-12).all())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_oracle_tail_gradient_equals_autograd_through_the_upsample(zoom, kind):
    g = torch.Generator().manual_seed(3 + zoom)
    lr = torch.randn((2, 4, 5, 6), generator=g, dtype=torch.float64) * 3
    ho, wo = zoom * 3 + 1, zoom * 4 + 1
    y = torch.randint(0, 6, (2, ho, wo), generator=g)
    if kind == "mixed":
        y[torch.rand((2, ho, wo), generator=g) < 0.4] = 255
        y[1, 0, 0] = -1
    elif kind == "all-U":
        y[:] = 255
    loss, _, _, _, dl = entropy_tail(lr, y, zoom, 0.7, 1.3)
    lr_r = lr.clone().requires_grad_(True)
    x = lr_r.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(ho, wo), mode="bilinear", align_corners=True)
    ref = entropy_definition(x, y, 0.7, 1.3)
    (dl_r,) = torch.autograd.grad(ref, lr_r)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert float((dl - dl_r).abs().max()) <= 1e-12 * float(dl_r.abs().max())


def test_oracle_ce_term_is_cross_entropy_and_empty_sets_are_zero():
    x, y = _case("mixed")
    yc = y.clone()
    yc[(yc < 0) | (yc >= 5)] = 255
    xr = x.clone().requires_grad_(True)
    ref = F.cross_entropy(xr, yc, ignore_index=255)
    (g_ref,) = torch.autograd.grad(ref, xr)
    loss, _, _, _, grad = entropy_loss(x, y, 0.0, 1.0)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert torch.allclose(grad, g_ref, rtol=1e-10, atol=1e-14)
    # nothing in either set: loss 0, gradient exactly 0
    y0 = torch.full_like(y, 7)
    loss, nl, nu, _, grad = entropy_loss(x, y0, 1.0, 1.0)
    assert (nl, nu) == (0, 0) and loss.item() == 0.0 and float(grad.abs().max()) == 0.0
    # constant logits: H = log C, gradient 0
    loss, _, _, ent, grad = entropy_loss(torch.full_like(x, 0.25), torch.full_like(y, 255), 1.0, 0.0)
    assert torch.allclose(ent, torch.full_like(ent, math.log(5)), rtol=1e-14, atol=0)
    assert float(grad.abs().max()) <= 1e-16


# ------------------------------------------------------------------------------------------------ module
def test_entropy_constructor_validation():
    c = EntropyLoss()
    assert (c.ignore_index, c.ent_weight, c.ce_weight) == (255, 1.0, 1.0) and list(c.state_dict()) == []
    assert repr(c) == "EntropyLoss(ignore_index=255, ent_weight=1, ce_weight=1)"
    c = EntropyLoss(ignore_index=-1, ent_weight=0.5, ce_weight=0)
    assert repr(c) == "EntropyLoss(ignore_index=-1, ent_weight=0.5, ce_weight=0)" and c.ce_weight == 0.0
    assert isinstance(EntropyLoss(ent_weight=2).ent_weight, float)
    for kw in ("ent_weight", "ce_weight"):
        for bad in (True, "1", None, [1.0], torch.tensor(1.0)):
            with pytest.raises(TypeError):
                EntropyLoss(**{kw: bad})
        for bad in (-0.1, float("nan"), float("inf")):
            with pytest.raises(ValueError):
                EntropyLoss(**{kw: bad})
    for bad in (True, 255.0, "255", None):
        with pytest.raises(TypeError):
            EntropyLoss(ignore_index=bad)


def test_entropy_module_has_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        EntropyLoss()(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        EntropyLoss().aux_loss(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="at most 256 classes"):
        EntropyLoss()(torch.zeros((1, 257, 2, 2)), torch.zeros((1, 2, 2), dtype=torch.int64))
    with pytest.raises(ValueError, match="expected"):
        EntropyLoss()(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassEntropy(EntropyLoss):
    pass


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    y = torch.zeros((2, zoom * 8 + 1, zoom * 10 + 1), dtype=torch.int64)
    for crit in (EntropyLoss(), EntropyLoss(ce_weight=0.0), EntropyLoss(ignore_index=-1, ent_weight=0.0)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 256)), y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y[:, :-1], zoom)             # not the zoomed size
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, logits, y[0], zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    for crit in (_SubclassEntropy(), _SubclassEntropy(ce_weight=0.0)):             # a subclass keeps the ATen tail
        assert not SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert not SF.fused_tail_supported(crit, logits, y, zoom)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_width_limit_is_the_dice_one(zoom):
    # 12 bytes per pixel of the interval's `zoom` rows in 224 KB
    w_max = (224 * 1024 // (12 * zoom) - 1) // zoom + 1       # the widest logits whose target fits
    for w, ok in ((w_max, True), (w_max + 1, False)):
        wo = zoom * (w - 1) + 1
        y = torch.zeros((1, zoom * 2 + 1, wo), dtype=torch.int64)
        assert (12 * zoom * wo <= 224 * 1024) == ok
        assert SF.fused_tail_supported(EntropyLoss(), None, y, zoom, (1, 3, 17, 8 * (w - 1) + 1)) == ok
        assert SF.fused_tail_supported(FocalLoss(), None, y, zoom, (1, 3, 17, 8 * (w - 1) + 1)) == ok


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, ws=P, loss=P, amax=P, lse=P,
         mu=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_entropy_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, ws, loss,
                                                      amax, lse, mu, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, ent_weight=1.0, ce_weight=1.0,
         lse=P, mu=P, info=P, g=P, ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_entropy_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, ent_weight,
                                                      ce_weight, lse, mu, info, g, ws, dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_entropy_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(C=1, pitch=1) == -1 and b"bad sizes" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    assert call(h=1, Ho=1) == -1 and b"bad sizes" in _err()
    # the staged rows: 12 bytes per pixel of `zoom` rows in 224 KB -> Wo <= 2389 at zoom 8
    assert call(zoom=8, w=300) == -1 and b"too large" in _err() and b"2389" in _err()      # Wo = 2393
    assert call(zoom=1, w=19115) == -1 and b"too large" in _err()
    assert call(lse=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()
    assert call(mu=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()


def test_entropy_entry_points_validate_options_and_outputs():
    for kw in ("ent_weight", "ce_weight"):
        for bad in (-0.5, float("nan"), float("inf"), -float("inf")):
            assert _bwd(**{kw: bad}) == -1 and kw.encode() in _err(), (kw, bad)
    for kw in ("ws", "loss", "lse", "mu"):
        assert _fwd(**{kw: None}) == -1 and b"upsample_ce_entropy_fwd" in _err() and b"null" in _err(), kw
    for kw in ("lse", "mu", "info", "g", "ws", "dl"):
        assert _bwd(**{kw: None}) == -1 and b"upsample_ce_entropy_bwd" in _err() and b"null" in _err(), kw


def test_entropy_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        h, w, C = 60, 60, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        assert (lib.semseg_upsample_ce_entropy_workspace_floats(2, ho, wo, zoom) ==
                2 * lib.semseg_upsample_ce_zoom_workspace_floats(2, ho, wo, zoom) == 2 * 2 * 2 * h * -(-wo // 128))
        assert (lib.semseg_upsample_ce_entropy_bwd_workspace_floats(2, ho, w, C, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, ho, w, C, zoom) == 2 * 2 * h * w * C)
    assert lib.semseg_upsample_ce_entropy_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_entropy_workspace_floats(0, 33, 33, 8) == -1 and b"bad sizes" in _err()
    assert lib.semseg_upsample_ce_entropy_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()


# ------------------------------------------------------------------------------------------------ Tent
@pytest.fixture(scope="module")
def cpu_pspnet():
    from semseg_b200.pspnet import PSPNet
    torch.manual_seed(0)
    return PSPNet(layers=50, classes=5, zoom_factor=8, pretrained=False)


def test_tent_rejects_what_it_cannot_adapt(cpu_pspnet):
    import copy
    from semseg_b200.adapt import Tent
    net = cpu_pspnet
    with pytest.raises(TypeError, match="PSPNet or PSANet"):
        Tent(nn.Sequential(nn.Conv2d(3, 4, 1), nn.BatchNorm2d(4)), lr=1e-3)
    with pytest.raises(TypeError, match="DataParallel"):
        Tent(nn.DataParallel(net), lr=1e-3)
    ddp = nn.parallel.DistributedDataParallel.__new__(nn.parallel.DistributedDataParallel)
    with pytest.raises(TypeError, match="DistributedDataParallel"):
        Tent(ddp, lr=1e-3)
    no_aux = copy.deepcopy(net)
    del no_aux.aux
    with pytest.raises(ValueError, match="aux head"):
        Tent(no_aux, lr=1e-3)
    with pytest.raises(ValueError, match="CUDA"):
        Tent(net, lr=1e-3)
    # a rejected network is left as it was
    assert all(p.requires_grad for p in net.parameters())
    assert type(net.criterion) is nn.CrossEntropyLoss


def test_tent_checks_its_options_before_touching_the_model(cpu_pspnet):
    from semseg_b200.adapt import Tent
    net = cpu_pspnet
    for kw, bad, exc in (("lr", "1", TypeError), ("lr", True, TypeError), ("lr", -1.0, ValueError),
                         ("lr", float("nan"), ValueError), ("momentum", None, TypeError),
                         ("momentum", float("inf"), ValueError), ("steps", 1.0, TypeError), ("steps", True, TypeError),
                         ("steps", 0, ValueError)):
        args = dict(lr=1e-3)
        args[kw] = bad
        with pytest.raises(exc):
            Tent(net, **args)
    assert all(p.requires_grad for p in net.parameters())
