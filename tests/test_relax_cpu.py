"""CPU tier for boundary label relaxation on the fused tail (csrc/tail.cu relaxation kernels): the float64 oracle of the
GPU tests matches a per-pixel loop and the gradient of its own definition under autograd, and is cross-entropy at
border 0; BoundaryRelaxationLoss validates its options and declares its graph options; `fused_tail_supported` takes
the native tail exactly where the kernels apply; and the entry points reject bad arguments with SEMSEG_E_INVALID and a
message before any CUDA call."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200 import losses
from semseg_b200.losses import BoundaryRelaxationLoss
from tests.relax_oracle import relax_definition, relax_loss, relax_sets, relax_tail

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


def _loop(x, y, border, wt, ignore_index=255):
    """The definition pixel by pixel in Python."""
    n, c, h, w = x.shape
    num = den = 0.0
    for b in range(n):
        for i in range(h):
            for j in range(w):
                t = int(y[b, i, j])
                if t == ignore_index or not 0 <= t < c:
                    continue
                s = set()
                for ii in range(max(i - border, 0), min(i + border, h - 1) + 1):
                    for jj in range(max(j - border, 0), min(j + border, w - 1) + 1):
                        u = int(y[b, ii, jj])
                        if u != ignore_index and 0 <= u < c:
                            s.add(u)
                p = torch.softmax(x[b, :, i, j], 0)
                om = sum(1.0 if wt is None else float(wt[k]) for k in s) / len(s)
                num += om * -math.log(sum(float(p[k]) for k in s))
                den += om
    return (num / den if den > 0 else 0.0), den


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("border", [0, 1, 2, 4])
@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
def test_oracle_matches_a_per_pixel_loop(weighted, border):
    x, y, wt = _case(c=6, h=7, w=9)
    wt = wt if weighted else None
    loss, d, _ = relax_loss(x, y, border, wt)
    ref, d_ref = _loop(x, y, border, wt)
    assert math.isclose(d, d_ref, rel_tol=1e-12)
    assert math.isclose(loss.item(), ref, rel_tol=1e-10)
    assert math.isclose(relax_definition(x, y, border, wt).item(), ref, rel_tol=1e-10)


def test_oracle_sets_are_clipped_and_skip_invalid_labels():
    y = torch.tensor([[[0, 255, 2],
                       [7, 1, -1],
                       [1, 1, 1]]])
    valid, s = relax_sets(y, 4, 1)
    assert valid.tolist() == [[[True, False, True], [False, True, False], [True, True, True]]]
    assert s[0, :, 0, 0].tolist() == [True, True, False, False]            # window clipped at the corner
    assert s[0, :, 1, 1].tolist() == [True, True, True, False]             # 255, 7 and -1 add no class
    assert not s[0, :, 0, 1].any() and not s[0, :, 1, 0].any()             # pixels that are not valid have no set
    assert s[0, :, 2, 2].tolist() == [False, True, False, False]


@pytest.mark.parametrize("border", [1, 3])
@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
def test_oracle_closed_form_equals_autograd_of_the_definition(weighted, border):
    x, y, wt = _case()
    wt = wt if weighted else None
    xr = x.clone().requires_grad_(True)
    (g_ref,) = torch.autograd.grad(relax_definition(xr, y, border, wt), xr)
    loss, _, grad = relax_loss(x, y, border, wt)
    assert float((grad - g_ref).abs().max()) <= 1e-12 * float(g_ref.abs().max())


@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_tail_gradient_equals_autograd_through_the_upsample(zoom):
    g = torch.Generator().manual_seed(3)
    lr = torch.randn((2, 4, 5, 6), generator=g, dtype=torch.float64) * 3
    ho, wo = zoom * 3 + 1, zoom * 4 + 1
    y = torch.randint(0, 6, (2, ho, wo), generator=g)
    y[torch.rand((2, ho, wo), generator=g) < 0.2] = 255
    wt = torch.rand(6, generator=g, dtype=torch.float64) + 0.2
    loss, _, dl = relax_tail(lr, y, zoom, 2, wt)
    lr_r = lr.clone().requires_grad_(True)
    x = lr_r.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(ho, wo), mode="bilinear", align_corners=True)
    ref = relax_definition(x, y, 2, wt)
    (dl_r,) = torch.autograd.grad(ref, lr_r)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    assert float((dl - dl_r).abs().max()) <= 1e-12 * float(dl_r.abs().max())


def test_oracle_border_zero_is_cross_entropy():
    x, y, wt = _case()
    yc = y.clone()
    yc[(yc < 0) | (yc >= 5)] = 255                      # F.cross_entropy rejects other out-of-range targets
    for w in (None, wt):
        xr = x.clone().requires_grad_(True)
        ref = F.cross_entropy(xr, yc, weight=w, ignore_index=255)
        (g_ref,) = torch.autograd.grad(ref, xr)
        loss, _, grad = relax_loss(x, y, 0, w)
        assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
        assert torch.allclose(grad, g_ref, rtol=1e-10, atol=1e-14)


def test_oracle_full_set_and_nothing_valid_are_zero():
    x, _, wt = _case(c=4)
    y = torch.zeros((2, 6, 7), dtype=torch.int64)
    y[:, ::2, ::2], y[:, 1::2, ::2], y[:, ::2, 1::2], y[:, 1::2, 1::2] = 0, 1, 2, 3
    y = y[:, :5, :5].contiguous()                      # every 3x3 window holds all four classes
    loss, d, grad = relax_loss(x[..., :5, :5], y, 1, wt)
    assert loss.item() == 0.0 and d > 0 and float(grad.abs().max()) == 0.0
    loss, d, grad = relax_loss(x, torch.full((2, 6, 7), 255), 2, wt)
    assert loss.item() == 0.0 and d == 0.0 and float(grad.abs().max()) == 0.0


def test_oracle_keeps_relative_accuracy_for_small_losses():
    # two classes share nearly all the mass and both lie in the set: l ~ 1e-12 from -log1p(-R), not from lse - lse_S
    x = torch.full((1, 4, 1, 2), -30.0, dtype=torch.float64)
    x[0, 0], x[0, 1] = 0.0, 0.0
    y = torch.tensor([[[0, 1]]])
    loss, _, _ = relax_loss(x, y, 1)
    ref = -math.log1p(-2 * math.exp(-30.0) / (2 + 2 * math.exp(-30.0)))
    assert math.isclose(loss.item(), ref, rel_tol=1e-12)


# ------------------------------------------------------------------------------------------------ module
def test_constructor_validation():
    assert BoundaryRelaxationLoss().border == 1 and BoundaryRelaxationLoss().ignore_index == 255
    for b in (0, 4):
        assert BoundaryRelaxationLoss(border=b).border == b
    for bad in (-1, 5, 100):
        with pytest.raises(ValueError, match="border"):
            BoundaryRelaxationLoss(border=bad)
    for bad in (1.0, True, "1", None):
        with pytest.raises(TypeError, match="border"):
            BoundaryRelaxationLoss(border=bad)
    with pytest.raises(TypeError, match="ignore_index"):
        BoundaryRelaxationLoss(ignore_index=2.5)
    with pytest.raises(TypeError, match="weight"):
        BoundaryRelaxationLoss(weight=[1.0, 2.0])
    with pytest.raises(TypeError, match="weight"):
        BoundaryRelaxationLoss(weight=torch.ones(3, dtype=torch.int64))
    with pytest.raises(ValueError, match="weight"):
        BoundaryRelaxationLoss(weight=torch.ones(3, 2))


def test_weight_is_a_buffer_and_graph_key():
    w = torch.ones(5)
    crit = BoundaryRelaxationLoss(border=2, weight=w)
    assert "weight" in dict(crit.named_buffers()) and "weight" in crit.state_dict()
    assert "weight" not in BoundaryRelaxationLoss().state_dict()
    assert "border=2" in repr(crit) and "weight=[5]" in repr(crit)
    assert BoundaryRelaxationLoss.graph_options == ("ignore_index", "border")
    k = losses.graph_key(crit)
    assert k == (BoundaryRelaxationLoss, 255, 2, w.data_ptr(), 5)
    crit.border = 1
    assert losses.graph_key(crit) != k                      # a new border captures anew
    crit.border = 2
    with torch.no_grad():
        crit.weight.mul_(2.0)
    assert losses.graph_key(crit) == k                      # an in-place edit does not
    assert losses.graph_key(BoundaryRelaxationLoss()) == (BoundaryRelaxationLoss, 255, 1, None)


def test_module_has_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="native CUDA"):
        BoundaryRelaxationLoss()(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="256 classes"):
        BoundaryRelaxationLoss()(torch.zeros((1, 257, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="expected"):
        BoundaryRelaxationLoss()(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassRelax(BoundaryRelaxationLoss):
    pass


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    y = torch.zeros((2, zoom * 8 + 1, zoom * 10 + 1), dtype=torch.int64)
    for crit in (BoundaryRelaxationLoss(), BoundaryRelaxationLoss(border=0), BoundaryRelaxationLoss(4, None, -1)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y[:, :-1], zoom)             # not the zoomed size
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    rejected = [
        _SubclassRelax(),
        _SubclassRelax(border=0),
        BoundaryRelaxationLoss(weight=torch.ones(21)),                                # CPU weight
        BoundaryRelaxationLoss(border=0, weight=torch.ones(21)),
        BoundaryRelaxationLoss(weight=torch.ones(21, dtype=torch.float64)),
    ]
    for crit in rejected:
        assert not SF.fused_tail_supported(crit, None, y, zoom, x_size), crit
        assert not SF.fused_tail_supported(crit, logits, y, zoom), crit


@pytest.mark.parametrize("border", [0, 1, 4])
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_width_limit_is_the_dice_one(zoom, border):
    # 12 bytes per pixel of the interval's `zoom` rows in 224 KB, at every border
    w_max = (224 * 1024 // (12 * zoom) - 1) // zoom + 1       # the widest logits whose target fits
    for w, ok in ((w_max, True), (w_max + 1, False)):
        wo = zoom * (w - 1) + 1
        y = torch.zeros((1, zoom * 2 + 1, wo), dtype=torch.int64)
        assert (12 * zoom * wo <= 224 * 1024) == ok
        crit = BoundaryRelaxationLoss(border=border)
        assert SF.fused_tail_supported(crit, None, y, zoom, (1, 3, 17, 8 * (w - 1) + 1)) == ok
    # the shipped crops fit at zoom 8
    for crop in (473, 713):
        y = torch.zeros((1, crop, crop), dtype=torch.int64)
        assert SF.fused_tail_supported(BoundaryRelaxationLoss(border=border), None, y, 8, (1, 3, crop, crop))


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, border=1, cw=P, ws=P, loss=P,
         amax=P, lse=P, sets=P, lq=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_relax_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, border, cw,
                                                    ws, loss, amax, lse, sets, lq, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, Ho=None, Wo=None, zoom=4, lse=P, sets=P, lq=P, info=P, g=P, ws=P,
         dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_relax_bwd(logits, pitch, N, h, w, C, Ho, Wo, zoom, lse, sets, lq, info, g, ws,
                                                    dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_relax_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    # the staged rows: 12 bytes per pixel of `zoom` rows in 224 KB -> Wo <= 2389 at zoom 8
    assert call(zoom=8, w=300) == -1 and b"too large" in _err() and b"2389" in _err()      # Wo = 2393
    assert call(zoom=1, w=19115) == -1 and b"too large" in _err()
    assert call(lq=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()
    assert call(sets=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()


def test_relax_entry_points_validate_options_and_outputs():
    for bad in (-1, 5, 1 << 20):
        assert _fwd(border=bad) == -1 and b"border" in _err(), bad
    assert _fwd(target=None) == -1 and b"null" in _err()
    assert _fwd(cw=ctypes.c_void_p(18)) == -1 and b"aligned" in _err()
    for kw in ("ws", "loss", "lse", "sets", "lq"):
        assert _fwd(**{kw: None}) == -1 and b"null" in _err(), kw
    for kw in ("lse", "sets", "lq", "info", "g", "ws", "dl"):
        assert _bwd(**{kw: None}) == -1 and b"null" in _err(), kw


def test_relax_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        h, w, C = 60, 60, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        assert (lib.semseg_upsample_ce_relax_workspace_floats(2, ho, wo, zoom) ==
                lib.semseg_upsample_ce_zoom_workspace_floats(2, ho, wo, zoom))
        assert (lib.semseg_upsample_ce_relax_bwd_workspace_floats(2, ho, w, C, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, ho, w, C, zoom))
    # tag and omega per pixel, then ceil(C / 32) mask words
    for c, words in ((2, 3), (19, 3), (32, 3), (33, 4), (150, 7), (256, 10)):
        assert lib.semseg_upsample_ce_relax_sets_words(2, 5, 7, c) == words * 70
    for bad in ((0, 5, 7, 19), (2, 5, 7, 1), (2, 5, 7, 257), (2, 0, 7, 19)):
        assert lib.semseg_upsample_ce_relax_sets_words(*bad) == -1 and b"bad sizes" in _err()
    assert lib.semseg_upsample_ce_relax_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_relax_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
