"""CPU tier for the Dice (+ cross-entropy) loss on the fused tail (csrc/tail.cu Dice kernels): the float64 oracle of
the GPU tests agrees with a second statement written the way segmentation_models_pytorch writes it, its closed-form
gradient agrees with autograd of the definition (the clamped denominator included), DiceLoss validates its options,
`fused_tail_supported` takes the native tail exactly for a DiceLoss of this type, and the new entry points reject bad
arguments with SEMSEG_E_INVALID and a message before any CUDA call."""
import ctypes
import math

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import DiceLoss, OhemCrossEntropyLoss
from tests.dice_oracle import dice_ce, dice_ce_grad, dice_ce_smp, upsampled

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _case(seed, n=2, c=6, h=5, w=7, zoom=2):
    """Upsampled float64 logits with ignored and out-of-range targets and one absent class (c - 1)."""
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn((n, h, w, c), generator=g, dtype=torch.float32) * 3
    x = upsampled(lg, zoom)
    ho, wo = x.shape[-2:]
    t = torch.randint(0, c - 1, (n, ho, wo), generator=g)
    t[torch.rand((n, ho, wo), generator=g) < 0.1] = 255
    t[torch.rand((n, ho, wo), generator=g) < 0.03] = c + 2
    t[torch.rand((n, ho, wo), generator=g) < 0.03] = -1
    return x, t


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("ce_weight", [0.0, 0.7])
@pytest.mark.parametrize("smooth", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("zoom", [1, 4])
def test_oracle_agrees_with_smp_statement(zoom, smooth, ce_weight):
    x, t = _case(zoom * 10 + int(2 * smooth), zoom=zoom)
    x.requires_grad_(True)
    loss, inter, s, n = dice_ce(x, t, 255, smooth, 1e-7, ce_weight)
    ref = dice_ce_smp(x, t, 255, smooth, 1e-7, ce_weight)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-13)
    assert n[-1] == 0 and bool((n[:-1] > 0).all())                  # one absent class
    (g_o,) = torch.autograd.grad(loss, x)
    (g_r,) = torch.autograd.grad(dice_ce_smp(x, t, 255, smooth, 1e-7, ce_weight), x)
    assert torch.allclose(g_o, g_r, rtol=1e-12, atol=1e-18)


def test_oracle_hand_computed():
    # two classes, three pixels: p(class 0) = 0.9, 0.2, 0.6; targets 0, 1, ignored
    p = torch.tensor([0.9, 0.2, 0.6], dtype=torch.float64)
    x = torch.stack([p.log(), (1 - p).log()]).view(1, 2, 1, 3)
    t = torch.tensor([[[0, 1, 255]]])
    loss, inter, s, n = dice_ce(x, t, 255, smooth=0.5)
    assert n.tolist() == [1.0, 1.0]
    assert torch.allclose(inter, torch.tensor([0.9, 0.8], dtype=torch.float64), rtol=1e-15)
    assert torch.allclose(s, torch.tensor([1.1 + 1, 0.9 + 1], dtype=torch.float64), rtol=1e-15)
    ref = ((1 - (1.8 + 0.5) / (2.1 + 0.5)) + (1 - (1.6 + 0.5) / (1.9 + 0.5))) / 2
    assert math.isclose(loss.item(), ref, rel_tol=1e-14)
    loss_ce, _, _, _ = dice_ce(x, t, 255, smooth=0.5, ce_weight=2.0)
    assert math.isclose(loss_ce.item(), ref - 2.0 * (math.log(0.9) + math.log(0.8)) / 2, rel_tol=1e-14)


def test_oracle_nothing_valid_is_zero():
    x, t = _case(3)
    x.requires_grad_(True)
    t = torch.full_like(t, 255)
    for ce_weight in (0.0, 1.0):
        loss, _, _, n = dice_ce(x, t, 255, 1.0, 1e-7, ce_weight)
        (g,) = torch.autograd.grad(loss, x)
        assert loss.item() == 0.0 and float(n.sum()) == 0.0 and float(g.abs().max()) == 0.0
        assert float(dice_ce_grad(x, t, 255, 1.0, 1e-7, ce_weight).abs().max()) == 0.0


def _clamp_eps(x, t, smooth):
    """An eps between the smallest and the largest S_c + smooth of the present classes: some clamp, some do not."""
    _, _, s, n = dice_ce(x, t, 255, smooth)
    v = (s + smooth)[n > 0].sort().values
    return float((v[0] + v[-1]) / 2)


@pytest.mark.parametrize("ce_weight", [0.0, 0.7])
@pytest.mark.parametrize("smooth", [0.0, 0.5])
@pytest.mark.parametrize("clamp", [False, True], ids=["no-clamp", "clamp"])
def test_closed_form_gradient_equals_autograd(clamp, smooth, ce_weight):
    x, t = _case(int(clamp) * 7 + int(smooth * 2) + 1, n=2, c=5, h=6, w=5, zoom=2)
    # unequal class sizes, so an eps between them clamps the small classes only
    t[:, :3] = torch.where((t[:, :3] >= 0) & (t[:, :3] < 5), torch.zeros_like(t[:, :3]), t[:, :3])
    eps = _clamp_eps(x, t, smooth) if clamp else 1e-7
    x.requires_grad_(True)
    loss, _, s, n = dice_ce(x, t, 255, smooth, eps, ce_weight)
    if clamp:
        present = n > 0
        assert bool((s + smooth < eps)[present].any()) and bool((s + smooth >= eps)[present].any())
    (g_a,) = torch.autograd.grad(loss, x)
    g_c = dice_ce_grad(x, t, 255, smooth, eps, ce_weight)
    scale = float(g_a.abs().max())
    assert scale > 1e-4
    assert float((g_c - g_a).abs().max()) <= 1e-13 * scale


# ------------------------------------------------------------------------------------------------ DiceLoss module
def test_dice_loss_validation():
    d = DiceLoss()
    assert (d.ignore_index, d.smooth, d.eps, d.ce_weight) == (255, 0.0, 1e-7, 0.0)
    d = DiceLoss(ignore_index=-1, smooth=1, eps=0, ce_weight=2)
    assert (d.ignore_index, d.smooth, d.eps, d.ce_weight) == (-1, 1.0, 0.0, 2.0)
    assert isinstance(d.smooth, float) and "ce_weight=2" in repr(d)
    assert list(d.state_dict()) == []
    for kw in ({"ignore_index": 255.0}, {"ignore_index": True}, {"smooth": "1"}, {"eps": None},
               {"ce_weight": True}, {"smooth": torch.tensor(1.0)}):
        with pytest.raises(TypeError):
            DiceLoss(**kw)
    for kw in ({"smooth": -0.1}, {"eps": -1e-7}, {"ce_weight": -1.0}, {"smooth": float("nan")},
               {"eps": float("inf")}, {"ce_weight": float("nan")}):
        with pytest.raises(ValueError):
            DiceLoss(**kw)


def test_dice_loss_has_no_cpu_fallback():
    crit = DiceLoss(ce_weight=1.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="256 classes"):
        crit(torch.zeros((1, 257, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="expected"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassDice(DiceLoss):
    pass


def _target(n, h, w):
    return torch.zeros((n, h, w), dtype=torch.int64)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    ho, wo = zoom * 8 + 1, zoom * 10 + 1
    y = _target(2, ho, wo)
    for crit in (DiceLoss(), DiceLoss(smooth=1.0, ce_weight=1.0)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 256)), y, zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
        for other in {1, 2, 4, 8} - {zoom}:
            yo = _target(2, other * 8 + 1, other * 10 + 1)
            assert not SF.fused_tail_supported(crit, None, yo, zoom, x_size)
            assert not SF.fused_tail_supported(crit, logits, yo, zoom)
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, logits, y[0], zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    # a subclass may change the loss: it keeps the ATen tail
    assert not SF.fused_tail_supported(_SubclassDice(), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(_SubclassDice(), logits, y, zoom)
    # the existing decisions are unchanged
    for crit in (nn.CrossEntropyLoss(ignore_index=255), OhemCrossEntropyLoss()):
        assert SF.fused_tail_supported(crit, logits, y, zoom)
    assert not SF.fused_tail_supported(nn.CrossEntropyLoss(reduction="sum"), logits, y, zoom)


def test_fused_tail_dice_width_limit():
    """The Dice rows kernels stage 12 bytes per pixel of Z rows in 224 KB: 2389 columns at zoom 8, 19114 at zoom 1."""
    for zoom, limit in ((8, 2389), (4, 4778), (2, 9557), (1, 19114)):
        for want, ok in ((limit, True), (limit + zoom, False)):
            w = (want - 1) // zoom + 1                      # the widest target of the zoom's form up to `want`
            wo = zoom * (w - 1) + 1
            assert (wo <= limit) == ok
            logits = torch.zeros((1, 3, w, 19))
            y = _target(1, 2 * zoom + 1, wo)
            assert SF.fused_tail_supported(DiceLoss(), logits, y, zoom) == ok, (zoom, wo)
            assert SF.fused_tail_supported(nn.CrossEntropyLoss(), logits, y, zoom)


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _dfwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, smooth=0.0, eps=1e-7,
          ce_weight=1.0, ws=P, loss=P, amax=P, lse=P, table=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_dice_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, smooth, eps,
                                                   ce_weight, ws, loss, amax, lse, table, None)


def _dbwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, lse=P, table=P, g=P, ws=P,
          dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_dice_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, lse, table, g,
                                                   ws, dl, None)


@pytest.mark.parametrize("call", [_dfwd, _dbwd], ids=["fwd", "bwd"])
def test_dice_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    # 12-byte staged words: at most 2389 output columns at zoom 8 (the plain form allows 2560)
    assert call(zoom=8, w=300) == -1 and b"too large" in _err() and b"at most 2389" in _err()
    assert call(zoom=1, w=19115) == -1 and b"too large" in _err()


def test_dice_entry_points_validate_options_and_outputs():
    for kw in ("smooth", "eps", "ce_weight"):
        for bad in (-0.01, float("nan"), float("inf")):
            assert _dfwd(**{kw: bad}) == -1 and kw.encode() in _err(), (kw, bad)
    for kw in ("ws", "loss", "lse", "table"):
        assert _dfwd(**{kw: None}) == -1 and b"upsample_ce_dice_fwd" in _err() and b"null" in _err(), kw
    assert _dfwd(ws=ctypes.c_void_p(20)) == -1 and b"aligned" in _err()
    for kw in ("lse", "table", "g", "ws", "dl"):
        assert _dbwd(**{kw: None}) == -1 and b"upsample_ce_dice_bwd" in _err() and b"null" in _err(), kw


def test_dice_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        n, h, w, c = 2, 60, 61, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        ctas = n * h * ((wo + 127) // 128)
        f = 2 * ctas + 3 * n * h * c
        assert lib.semseg_upsample_ce_dice_workspace_floats(n, ho, wo, c, zoom) == f + (f & 1) + 2 * c
        assert (lib.semseg_upsample_ce_dice_bwd_workspace_floats(n, ho, wo, w, c, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(n, ho, w, c, zoom) + n * ho * wo)
    assert lib.semseg_upsample_ce_dice_workspace_floats(2, 33, 33, 21, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_dice_bwd_workspace_floats(2, 33, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
