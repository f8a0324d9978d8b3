"""CPU tier for the Gated CRF loss (losses.GatedCRFLoss, csrc/crf.cu): the float64 contract of the GPU tests has the
published unfold formulation's gradient and differs from its loss by exactly the out-of-image constant, a brute-force
loop agrees, the closed-form gradient passes gradcheck; GatedCRFLoss validates its options; `fused_tail_supported` takes
the native tail exactly where the kernels apply; the entry points reject bad arguments with SEMSEG_E_INVALID and a
message before any CUDA call, and the workspace sizes are the stated ones."""
import ctypes
import math

import pytest
import torch

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import GatedCRFLoss
from tests.gatedcrf_oracle import crf_contract, crf_loop, crf_outside_constant, crf_unfold, grid_rgb

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _case(seed=3, n=2, c=5, h=7, w=9, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * scale
    x = torch.randn((n, 3, h, w), generator=g, dtype=torch.float64)
    return s, grid_rgb(x, 1)


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("radius,sigma_xy,sigma_rgb", [(1, 6.0, 0.1), (2, 1.5, 0.3), (5, 6.0, 0.1), (8, 3.0, 1.0)])
def test_contract_and_published_unfold_have_one_gradient(radius, sigma_xy, sigma_rgb):
    s, rgb = _case()
    loss, grad, _ = crf_contract(s, rgb, radius, sigma_xy, sigma_rgb)
    sv = s.clone().requires_grad_(True)
    pub = crf_unfold(sv, rgb, radius, sigma_xy, sigma_rgb)
    pub.backward()
    pub = pub.detach()
    assert torch.allclose(sv.grad, grad, rtol=1e-10, atol=1e-14)
    const = crf_outside_constant(rgb, radius, sigma_xy, sigma_rgb)
    assert abs(float(pub) - float(loss) - const) <= 1e-12 * max(1.0, abs(float(pub)))
    # the constant does not depend on the logits
    pub2 = crf_unfold(s * 3 + 1, rgb, radius, sigma_xy, sigma_rgb)
    loss2, _, _ = crf_contract(s * 3 + 1, rgb, radius, sigma_xy, sigma_rgb)
    assert abs(float(pub2) - float(loss2) - const) <= 1e-12 * max(1.0, abs(float(pub2)))


@pytest.mark.parametrize("shape,radius", [((1, 3, 4, 5), 1), ((2, 2, 3, 3), 2), ((1, 4, 2, 6), 5)])
def test_brute_force_loop_agrees_on_tiny_grids(shape, radius):
    n, c, h, w = shape
    s, rgb = _case(seed=11, n=n, c=c, h=h, w=w)
    loss, _, _ = crf_contract(s, rgb, radius, 2.0, 0.5)
    assert abs(float(loss) - crf_loop(s, rgb, radius, 2.0, 0.5)) <= 1e-12 * max(1.0, abs(float(loss)))


class _ClosedForm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s, rgb, radius):
        loss, grad, _ = crf_contract(s, rgb, radius, 2.0, 0.4)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return g * grad, None, None


@pytest.mark.parametrize("radius", [1, 3])
def test_closed_form_gradient_passes_gradcheck(radius):
    s, rgb = _case(seed=5, n=1, c=4, h=5, w=6)
    assert torch.autograd.gradcheck(lambda t: _ClosedForm.apply(t, rgb, radius), (s.requires_grad_(True),))


def test_constant_logits_have_zero_gradient_and_loss_of_the_gates():
    s, rgb = _case(n=1, c=4, h=5, w=6)
    s = torch.zeros_like(s)
    loss, grad, S = crf_contract(s, rgb, 2, 2.0, 0.5)
    assert float(grad.abs().max()) < 1e-15
    # p = 1/C everywhere: the term is (1 - 1/C) times the sum of the gates
    gates = crf_contract(torch.zeros((1, 1, 5, 6), dtype=torch.float64), rgb, 2, 2.0, 0.5)[2]    # one class: S = K
    assert abs(float(loss) - 0.75 * float(gates.sum()) / 30) < 1e-14
    _, _, S1 = crf_contract(torch.full_like(s, 3.0), rgb, 2, 2.0, 0.5)
    assert torch.allclose(S, S1)


# ------------------------------------------------------------------------------------------------ options
def test_constructor_defaults_and_repr():
    c = GatedCRFLoss()
    assert (c.ignore_index, c.crf_weight, c.ce_weight, c.radius, c.sigma_xy, c.sigma_rgb, c.at) == \
        (255, 0.1, 1.0, 5, 6.0, 0.1, 'output')
    assert c.mean == (0.485 * 255, 0.456 * 255, 0.406 * 255) and c.std == (0.229 * 255, 0.224 * 255, 0.225 * 255)
    assert "crf_weight=0.1" in repr(c) and "at='output'" in repr(c)
    c = GatedCRFLoss(ignore_index=-1, crf_weight=0, ce_weight=2, radius=8, sigma_xy=1, sigma_rgb=3, mean=[0, 1, 2],
                     std=(1, 2, 3), at='logits')
    assert c.mean == (0.0, 1.0, 2.0) and c.std == (1.0, 2.0, 3.0) and isinstance(c.sigma_xy, float)


@pytest.mark.parametrize("kw,bad,exc", [
    ("ignore_index", 255.0, TypeError), ("ignore_index", True, TypeError),
    ("crf_weight", -0.1, ValueError), ("crf_weight", float("nan"), ValueError), ("crf_weight", float("inf"), ValueError),
    ("crf_weight", "1", TypeError), ("ce_weight", -1.0, ValueError), ("ce_weight", float("nan"), ValueError),
    ("radius", 0, ValueError), ("radius", 9, ValueError), ("radius", 5.0, TypeError), ("radius", True, TypeError),
    ("sigma_xy", 0.0, ValueError), ("sigma_xy", -1.0, ValueError), ("sigma_xy", float("inf"), ValueError),
    ("sigma_rgb", 0.0, ValueError), ("sigma_rgb", float("nan"), ValueError), ("sigma_rgb", None, TypeError),
    ("at", "input", ValueError), ("at", None, ValueError),
    ("mean", (1.0, 2.0), TypeError), ("mean", (1.0, 2.0, float("nan")), ValueError), ("mean", 3.0, TypeError),
    ("mean", (1, 2, "3"), TypeError), ("std", (1.0, 0.0, 1.0), ValueError), ("std", (1.0, -2.0, 1.0), ValueError),
    ("std", (1.0, 1.0, float("inf")), ValueError), ("std", (1.0, 1.0, 1.0, 1.0), TypeError),
])
def test_constructor_validation(kw, bad, exc):
    with pytest.raises(exc):
        GatedCRFLoss(**{kw: bad})


def test_module_has_no_cpu_fallback():
    y = torch.zeros((1, 5, 5), dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        GatedCRFLoss()(torch.zeros((1, 3, 5, 5)), y, torch.zeros((1, 3, 5, 5)))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        GatedCRFLoss().aux_loss(torch.zeros((1, 3, 5, 5)), y)
    with pytest.raises(ValueError, match="at most 256 classes"):
        GatedCRFLoss()(torch.zeros((1, 257, 5, 5)), y)
    with pytest.raises(ValueError, match="expected"):
        GatedCRFLoss()(torch.zeros((1, 3, 5, 5)), y[:, :, :4])


def test_upsample_ce_without_image_raises_rather_than_dropping_the_term():
    with pytest.raises(ValueError, match="needs the image"):
        SF.upsample_ce(torch.zeros((1, 3, 3, 4)), torch.zeros((1, 17, 25), dtype=torch.int64), 255, 8,
                       criterion=GatedCRFLoss())


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassCRF(GatedCRFLoss):
    pass


@pytest.mark.parametrize("at", ["output", "logits"])
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom, at):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    y = torch.zeros((2, zoom * 8 + 1, zoom * 10 + 1), dtype=torch.int64)
    for crit in (GatedCRFLoss(at=at), GatedCRFLoss(crf_weight=0.0, at=at), GatedCRFLoss(radius=8, ce_weight=0, at=at),
                 GatedCRFLoss(radius=1, ignore_index=-1, at=at)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 256)), y, zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)   # classes > 256
        assert not SF.fused_tail_supported(crit, logits, y[:, :-1], zoom)                 # not the zoomed size
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, logits, y[0], zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    for crit in (_SubclassCRF(at=at), _SubclassCRF(crf_weight=0.0, at=at)):          # a subclass keeps the ATen tail
        assert not SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert not SF.fused_tail_supported(crit, logits, y, zoom)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_width_limit_is_the_plain_backward_one(zoom):
    # the plain backward stages 8 bytes per pixel of the interval's `zoom` rows in 160 KB: Wo <= 2560 at zoom 8
    w_max = (160 * 1024 // (8 * zoom) - 1) // zoom + 1
    for w, ok in ((w_max, True), (w_max + 1, False)):
        wo = zoom * (w - 1) + 1
        y = torch.zeros((1, zoom * 2 + 1, wo), dtype=torch.int64)
        assert SF.fused_tail_supported(GatedCRFLoss(), None, y, zoom, (1, 3, 17, 8 * (w - 1) + 1)) == ok


# ------------------------------------------------------------------------------------------------ C-ABI validation
_NORM = (123.675, 116.28, 103.53, 58.395, 57.12, 57.375)


def _geom(zoom, h, w, istride):
    hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    return istride * (hg - 1) + 1, istride * (wg - 1) + 1


def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, zoom=4, lse=P, compute_lse=0, image=P, H=None, W=None, istride=2,
         radius=5, sigma_xy=6.0, sigma_rgb=0.1, norm=_NORM, ws=P, s=P, loss=P):
    gh, gw = _geom(zoom, h, w, istride)
    H = gh if H is None else H
    W = gw if W is None else W
    return _lib.load().semseg_gated_crf_fwd(logits, pitch, N, h, w, C, zoom, lse, compute_lse, image, H, W, istride,
                                            radius, sigma_xy, sigma_rgb, *norm, ws, s, loss, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, zoom=4, lse=P, image=P, H=None, W=None, istride=2, radius=5,
         sigma_xy=6.0, sigma_rgb=0.1, norm=_NORM, s=P, crf_weight=0.1, g=P, ws=P, dl=P):
    gh, gw = _geom(zoom, h, w, istride)
    H = gh if H is None else H
    W = gw if W is None else W
    return _lib.load().semseg_gated_crf_bwd(logits, pitch, N, h, w, C, zoom, lse, image, H, W, istride, radius,
                                            sigma_xy, sigma_rgb, *norm, s, crf_weight, g, ws, dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_entry_points_validate_shapes_and_options(call):
    assert call(zoom=3) == -1 and b"zoom 3" in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(image=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(C=0, pitch=0) == -1 and b"bad sizes" in _err()
    assert call(pitch=20) == -1 and b"bad sizes" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    assert call(h=0) == -1 and b"bad sizes" in _err()
    for r in (0, 9, -1):
        assert call(radius=r) == -1 and b"radius" in _err()
    for kw in ("sigma_xy", "sigma_rgb"):
        for bad in (0.0, -1.0, float("nan"), float("inf")):
            assert call(**{kw: bad}) == -1 and b"sigmas" in _err(), (kw, bad)
    for i, bad in ((0, float("nan")), (1, float("inf")), (3, 0.0), (4, -1.0), (5, float("nan"))):
        norm = list(_NORM)
        norm[i] = bad
        assert call(norm=norm) == -1 and b"mean" in _err(), (i, bad)
    for zoom, istride in ((1, 8), (2, 4), (4, 2), (8, 1), (1, 1)):
        H, W = _geom(zoom, 9, 7, istride)
        assert call(zoom=zoom, istride=istride, H=H + 1) == -1 and b"stride" in _err()
        assert call(zoom=zoom, istride=istride, W=W - 1) == -1 and b"stride" in _err()
    assert call(istride=0, H=1, W=1) == -1 and b"stride" in _err()


def test_entry_points_validate_outputs_and_weights():
    for kw in ("lse", "ws", "s", "loss"):
        assert _fwd(**{kw: None}) == -1 and b"gated_crf_fwd" in _err() and b"null" in _err(), kw
    assert _fwd(compute_lse=1, zoom=4) == -1 and b"zoom 1" in _err()
    for kw in ("lse", "s", "g", "dl", "ws"):
        assert _bwd(**{kw: None}) == -1 and b"gated_crf_bwd" in _err() and b"null" in _err(), kw
    for bad in (-0.5, float("nan"), float("inf")):
        assert _bwd(crf_weight=bad) == -1 and b"crf_weight" in _err()


def test_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        for (n, h, w, C) in ((16, 60, 60, 21), (16, 60, 60, 150), (2, 3, 5, 2)):
            hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
            assert lib.semseg_gated_crf_workspace_floats(n, h, w, zoom) == 2 * n * -(-hg // 16) * -(-wg // 16)
            assert lib.semseg_gated_crf_bwd_workspace_floats(n, h, w, C, zoom) == (
                0 if zoom == 1 else n * C * wg * (hg + h))
    # the header's figures: 16 x 473^2 at zoom 8, 21 and 150 classes
    assert 0.33e9 < 4 * lib.semseg_gated_crf_bwd_workspace_floats(16, 60, 60, 21, 8) < 0.35e9
    assert 2.4e9 < 4 * lib.semseg_gated_crf_bwd_workspace_floats(16, 60, 60, 150, 8) < 2.5e9
    assert lib.semseg_gated_crf_workspace_floats(2, 9, 9, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_gated_crf_workspace_floats(0, 9, 9, 8) == -1
    assert lib.semseg_gated_crf_bwd_workspace_floats(2, 9, 9, 21, 5) == -1 and b"zoom 5" in _err()
    assert lib.semseg_gated_crf_bwd_workspace_floats(2, 9, 9, 0, 8) == -1
