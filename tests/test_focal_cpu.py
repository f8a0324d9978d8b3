"""CPU tier for the focal loss on the fused tail (csrc/tail.cu focal kernels): the float64 oracle of the GPU tests has the
gradient of its own definition under autograd, is cross-entropy at gamma = 0 and follows torch.pow at q = 0;
FocalLoss validates its options and registers its weight like torch's losses; `fused_tail_supported` takes the native
tail exactly where the kernels apply; and the entry points reject bad arguments with SEMSEG_E_INVALID and a message
before any CUDA call."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import FocalLoss
from tests.focal_oracle import focal_definition, focal_loss, focal_tail

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _case(seed=7, n=2, c=5, h=6, w=7, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * scale
    y = torch.randint(0, c, (n, h, w), generator=g)
    y[torch.rand((n, h, w), generator=g) < 0.2] = 255
    y[0, 0, 0], y[0, 0, 1] = c + 2, -3                  # out of range: skipped
    wt = torch.rand(c, generator=g, dtype=torch.float64) + 0.2
    wt[1] = 0.0
    return x, y, wt


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("gamma", [0.0, 0.5, 1.0, 2.0, 5.0])
@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
def test_oracle_closed_form_equals_autograd_of_the_definition(weighted, gamma):
    x, y, wt = _case()
    wt = wt if weighted else None
    xr = x.clone().requires_grad_(True)
    ref = focal_definition(xr, y, gamma, wt)
    (g_ref,) = torch.autograd.grad(ref, xr)
    loss, n_valid, grad = focal_loss(x, y, gamma, wt)
    assert n_valid == int(((y != 255) & (y >= 0) & (y < 5)).sum())
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert float((grad - g_ref).abs().max()) <= 1e-12 * float(g_ref.abs().max())


@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_tail_gradient_equals_autograd_through_the_upsample(zoom):
    g = torch.Generator().manual_seed(3)
    lr = torch.randn((2, 4, 5, 6), generator=g, dtype=torch.float64) * 3
    ho, wo = zoom * 3 + 1, zoom * 4 + 1
    y = torch.randint(0, 6, (2, ho, wo), generator=g)
    y[torch.rand((2, ho, wo), generator=g) < 0.2] = 255
    wt = torch.rand(6, generator=g, dtype=torch.float64) + 0.2
    loss, _, dl = focal_tail(lr, y, zoom, 2.0, wt)
    lr_r = lr.clone().requires_grad_(True)
    x = lr_r.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(ho, wo), mode="bilinear", align_corners=True)
    ref = focal_definition(x, y, 2.0, wt)
    (dl_r,) = torch.autograd.grad(ref, lr_r)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert float((dl - dl_r).abs().max()) <= 1e-12 * float(dl_r.abs().max())


def test_oracle_gamma_zero_is_cross_entropy():
    x, y, wt = _case()
    yc = y.clone()
    yc[(yc < 0) | (yc >= 5)] = 255                      # F.cross_entropy rejects other out-of-range targets
    xr = x.clone().requires_grad_(True)
    ref = F.cross_entropy(xr, yc, ignore_index=255)
    (g_ref,) = torch.autograd.grad(ref, xr)
    loss, n_valid, grad = focal_loss(x, y, 0.0, None)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert torch.allclose(grad, g_ref, rtol=1e-10, atol=1e-14)
    # weighted: torch divides by sum w_t, the focal loss by n_valid
    ref = F.cross_entropy(xr, yc, weight=wt, ignore_index=255, reduction="sum") / n_valid
    (g_ref,) = torch.autograd.grad(ref, xr)
    loss, _, grad = focal_loss(x, y, 0.0, wt)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert torch.allclose(grad, g_ref, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("gamma", [0.0, 0.5, 2.0])
def test_oracle_q_zero_follows_torch_pow(gamma):
    # pixel 0: the other classes underflow in float64, q = 0 exactly; pixel 1: an ordinary pixel
    x = torch.tensor([[2000.0, 0.3], [0.0, 1.1], [-5.0, -0.4]], dtype=torch.float64).view(1, 3, 1, 2)
    y = torch.tensor([[[0, 2]]])
    loss, n_valid, grad = focal_loss(x, y, gamma, None)
    one, _, g_one = focal_loss(x[..., 1:], y[..., 1:], gamma, None)
    assert n_valid == 2 and torch.isfinite(grad).all()
    assert math.isclose(loss.item(), one.item() / 2, rel_tol=1e-12)         # l = 0^gamma * 0 = 0 at the q = 0 pixel
    assert float(grad[..., 0].abs().max()) == 0.0                          # M (p - onehot) = M * 0
    assert torch.allclose(grad[..., 1:], g_one / 2, rtol=1e-12, atol=0)
    # the naive definition agrees on the value (its autograd is nan for 0 < gamma < 1: inf * 0)
    assert math.isclose(focal_definition(x, y, gamma).item(), loss.item(), rel_tol=1e-12)


def test_oracle_keeps_relative_accuracy_near_p_t_one():
    # q = 2 e^-40 / (1 + 2 e^-40): 1 - p_t from a rounded p_t would be 0 in float64
    x = torch.tensor([40.0, 0.0, 0.0], dtype=torch.float64).view(1, 3, 1, 1)
    loss, _, _ = focal_loss(x, torch.zeros((1, 1, 1), dtype=torch.int64), 2.0, None)
    q = 2 * math.exp(-40.0)
    assert math.isclose(loss.item(), q ** 3, rel_tol=1e-9)


def test_oracle_nothing_valid_is_zero():
    x, y, _ = _case()
    loss, n_valid, grad = focal_loss(x, torch.full_like(y, 255), 2.0, None)
    assert n_valid == 0 and loss.item() == 0.0 and float(grad.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ module
def test_focal_constructor_validation():
    c = FocalLoss()
    assert c.gamma == 2.0 and c.ignore_index == 255 and c.weight is None and list(c.state_dict()) == []
    assert repr(c) == "FocalLoss(gamma=2, ignore_index=255)"
    assert FocalLoss(gamma=0).gamma == 0.0 and FocalLoss(gamma=0.5).gamma == 0.5 and FocalLoss(gamma=3).gamma == 3.0
    for bad in (True, "2", None, [2.0], torch.tensor(2.0)):
        with pytest.raises(TypeError):
            FocalLoss(gamma=bad)
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            FocalLoss(gamma=bad)
    for bad in (True, 255.0, "255", None):
        with pytest.raises(TypeError):
            FocalLoss(ignore_index=bad)
    for bad in ([1.0, 2.0], torch.ones(3, dtype=torch.int64), "w"):
        with pytest.raises(TypeError):
            FocalLoss(weight=bad)
    for bad in (torch.ones(2, 3), torch.ones(()), torch.ones(0)):
        with pytest.raises(ValueError):
            FocalLoss(weight=bad)


def test_focal_weight_is_a_buffer():
    w = torch.rand(19) + 0.5
    c = FocalLoss(gamma=1.5, weight=w, ignore_index=-1)
    assert torch.equal(c.weight, w) and dict(c.named_buffers())["weight"] is c.weight
    assert list(c.state_dict()) == ["weight"] and not c.weight.requires_grad
    assert repr(c) == "FocalLoss(gamma=1.5, ignore_index=-1, weight=[19])"
    c.double()
    assert c.weight.dtype == torch.float64
    net = torch.nn.Module()
    net.criterion = FocalLoss()
    assert list(net.state_dict()) == []


def test_focal_module_has_no_cpu_fallback():
    crit = FocalLoss(weight=torch.ones(3))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="at most 256 classes"):
        FocalLoss()(torch.zeros((1, 257, 2, 2)), torch.zeros((1, 2, 2), dtype=torch.int64))
    with pytest.raises(ValueError, match="expected"):
        FocalLoss()(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassFocal(FocalLoss):
    pass


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    y = torch.zeros((2, zoom * 8 + 1, zoom * 10 + 1), dtype=torch.int64)
    for crit in (FocalLoss(), FocalLoss(gamma=0.0), FocalLoss(gamma=0.5, ignore_index=-1)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y[:, :-1], zoom)             # not the zoomed size
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    rejected = [
        _SubclassFocal(),
        _SubclassFocal(gamma=0.0),
        FocalLoss(weight=torch.ones(21)),                                             # CPU weight
        FocalLoss(weight=torch.ones(21, dtype=torch.float64)),
    ]
    for crit in rejected:
        assert not SF.fused_tail_supported(crit, None, y, zoom, x_size), crit
        assert not SF.fused_tail_supported(crit, logits, y, zoom), crit


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_width_limit_is_the_dice_one(zoom):
    # 12 bytes per pixel of the interval's `zoom` rows in 224 KB
    w_max = (224 * 1024 // (12 * zoom) - 1) // zoom + 1       # the widest logits whose target fits
    for w, ok in ((w_max, True), (w_max + 1, False)):
        wo = zoom * (w - 1) + 1
        y = torch.zeros((1, zoom * 2 + 1, wo), dtype=torch.int64)
        assert (12 * zoom * wo <= 224 * 1024) == ok
        assert SF.fused_tail_supported(FocalLoss(), None, y, zoom, (1, 3, 17, 8 * (w - 1) + 1)) == ok


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, cw=P, gamma=2.0, ws=P, loss=P,
         amax=P, lse=P, mod=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_focal_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, cw, gamma, ws,
                                                    loss, amax, lse, mod, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, lse=P, mod=P, info=P, g=P, ws=P,
         dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_focal_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, lse, mod,
                                                    info, g, ws, dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_focal_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    # the staged rows: 12 bytes per pixel of `zoom` rows in 224 KB -> Wo <= 2389 at zoom 8
    assert call(zoom=8, w=300) == -1 and b"too large" in _err() and b"2389" in _err()      # Wo = 2393
    assert call(zoom=1, w=19115) == -1 and b"too large" in _err()
    assert call(mod=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()


def test_focal_entry_points_validate_options_and_outputs():
    for bad in (-0.5, float("nan"), float("inf"), -float("inf")):
        assert _fwd(gamma=bad) == -1 and b"gamma" in _err(), bad
    assert _fwd(cw=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()
    for kw in ("ws", "loss", "lse", "mod"):
        assert _fwd(**{kw: None}) == -1 and b"upsample_ce_focal_fwd" in _err() and b"null" in _err(), kw
    for kw in ("lse", "mod", "info", "g", "ws", "dl"):
        assert _bwd(**{kw: None}) == -1 and b"upsample_ce_focal_bwd" in _err() and b"null" in _err(), kw


def test_focal_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        h, w, C = 60, 60, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        assert (lib.semseg_upsample_ce_focal_workspace_floats(2, ho, wo, zoom) ==
                lib.semseg_upsample_ce_zoom_workspace_floats(2, ho, wo, zoom) == 2 * 2 * h * -(-wo // 128))
        assert (lib.semseg_upsample_ce_focal_bwd_workspace_floats(2, ho, w, C, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, ho, w, C, zoom) == 2 * 2 * h * w * C)
    assert lib.semseg_upsample_ce_focal_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_focal_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
