"""CPU tier for class-weighted and label-smoothed cross-entropy on the fused tail (csrc/tail.cu kWeighted kernels): the
float64 oracle of the GPU tests equals F.cross_entropy(weight, ignore_index, label_smoothing) and a weighted-OHEM case
worked by hand, `fused_tail_supported` takes the native tail exactly for the forms the kernels implement,
OhemCrossEntropyLoss(weight=...) validates and registers its weight like torch's losses, and the new entry points reject
bad arguments with SEMSEG_E_INVALID and a message before any CUDA call."""
import ctypes
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import OhemCrossEntropyLoss
from tests.weighted_ce_oracle import weighted_ce, weighted_ohem_ce

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
def test_oracle_equals_torch_cross_entropy(weighted, eps):
    g = torch.Generator().manual_seed(7)
    n, c, h, w = 2, 5, 6, 7
    x = (torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    y = torch.randint(0, c, (n, h, w), generator=g)
    y[torch.rand((n, h, w), generator=g) < 0.2] = 255
    wt = torch.rand(c, generator=g, dtype=torch.float64) + 0.2 if weighted else None
    ref = F.cross_entropy(x, y, weight=wt, ignore_index=255, label_smoothing=eps)
    loss, d = weighted_ce(x, y, wt, 255, eps)
    assert math.isclose(loss.item(), ref.item(), rel_tol=1e-12)
    valid = y != 255
    assert math.isclose(float(d), float(valid.sum()) if wt is None else float(wt[y[valid]].sum()), rel_tol=1e-12)
    (g_o,) = torch.autograd.grad(loss, x)
    (g_r,) = torch.autograd.grad(ref, x)
    assert torch.allclose(g_o, g_r, rtol=1e-10, atol=1e-14)


def test_oracle_d_zero_is_zero():
    x = torch.randn((1, 3, 2, 2), dtype=torch.float64, requires_grad=True)
    y = torch.tensor([[[0, 0], [255, 1]]])
    w = torch.tensor([0.0, 0.0, 2.0], dtype=torch.float64)
    loss, d = weighted_ce(x, y, w, 255, 0.1)          # every valid pixel in a zero-weight class
    (g,) = torch.autograd.grad(loss, x)
    assert float(d) == 0.0 and loss.item() == 0.0 and float(g.abs().max()) == 0.0
    loss, d = weighted_ce(x, torch.full_like(y, 255), None, 255, 0.1)   # nothing valid
    assert float(d) == 0.0 and loss.item() == 0.0


def _two_class_logits(p):
    """[1, 2, 1, len(p)] logits whose softmax gives class 0 the probability p[i] at pixel i."""
    p = torch.tensor(p, dtype=torch.float64)
    return torch.stack([p.log(), (1 - p).log()]).view(1, 2, 1, -1)


def test_weighted_ohem_oracle_hand_computed():
    # p_t of pixels 0..5; targets: class 0 at pixels 0, 1, 2 and 4, ignored at 3, class 1 at 5 (p_t = 1 - 0.3 = 0.7)
    x = _two_class_logits([0.9, 0.2, 0.6, 0.5, 0.4, 0.3])
    y = torch.tensor([[[0, 0, 0, 255, 0, 1]]])
    w = torch.tensor([2.0, 3.0], dtype=torch.float64)
    # valid p_t: 0.9 0.2 0.6 0.4 0.7; min_kept 1 -> k-th = 0.4 < thresh 0.65: thr 0.65, kept {0.2, 0.6, 0.4}
    loss, kept, thr, _ = weighted_ohem_ce(x, y, w, thresh=0.65, min_kept=1)
    assert thr == 0.65 and kept.view(-1).tolist() == [False, True, True, False, True, False]
    ref = -2.0 * (math.log(0.2) + math.log(0.6) + math.log(0.4)) / 3       # plain mean of w_t * nll, not / sum(w)
    assert math.isclose(loss.item(), ref, rel_tol=1e-12)
    # thresh 1 keeps every valid pixel, the class-1 pixel with weight 3
    loss, kept, _, _ = weighted_ohem_ce(x, y, w, thresh=1.0, min_kept=0)
    ref = -(2.0 * (math.log(0.9) + math.log(0.2) + math.log(0.6) + math.log(0.4)) + 3.0 * math.log(0.7)) / 5
    assert int(kept.sum()) == 5 and math.isclose(loss.item(), ref, rel_tol=1e-12)
    # weight None is the unweighted OHEM oracle
    from tests.ohem_oracle import ohem_ce
    assert math.isclose(weighted_ohem_ce(x, y, None, thresh=0.65, min_kept=1)[0].item(),
                        ohem_ce(x, y, thresh=0.65, min_kept=1)[0].item(), rel_tol=1e-15)


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassCE(nn.CrossEntropyLoss):
    pass


def _target(n, h, w):
    return torch.zeros((n, h, w), dtype=torch.int64)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    y = _target(2, zoom * 8 + 1, zoom * 10 + 1)
    # the ATen tail for everything the kernels do not implement, and for the weighted / smoothed forms on a CPU target
    # (tests/test_weighted_ce_gpu.py checks that they take the native tail on a CUDA one)
    rejected = [
        nn.CrossEntropyLoss(ignore_index=255, label_smoothing=0.1),
        nn.CrossEntropyLoss(ignore_index=255, label_smoothing=1.0),
        nn.CrossEntropyLoss(ignore_index=255, reduction="sum"),
        nn.CrossEntropyLoss(ignore_index=255, reduction="none"),
        nn.CrossEntropyLoss(ignore_index=255, label_smoothing=0.1, reduction="sum"),
        nn.CrossEntropyLoss(weight=torch.ones(21), ignore_index=255),                    # CPU weight
        nn.CrossEntropyLoss(weight=torch.ones(21, dtype=torch.float64), ignore_index=255),
        _SubclassCE(ignore_index=255),
        _SubclassCE(ignore_index=255, label_smoothing=0.1),
        OhemCrossEntropyLoss(weight=torch.ones(21)),                                     # CPU weight
        OhemCrossEntropyLoss(weight=torch.ones(21, dtype=torch.float64)),
    ]
    for crit in rejected:
        assert not SF.fused_tail_supported(crit, None, y, zoom, x_size), crit
        assert not SF.fused_tail_supported(crit, logits, y, zoom), crit
    # weight None with eps 0 is the default criterion, unweighted OHEM the OHEM form: both native, on any target
    for crit in (nn.CrossEntropyLoss(ignore_index=255, label_smoothing=0.0), OhemCrossEntropyLoss()):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)


# ------------------------------------------------------------------------------------------------ OHEM module weight
def test_ohem_weight_validation_and_buffer():
    w = torch.rand(19) + 0.5
    c = OhemCrossEntropyLoss(ignore_index=255, thresh=0.7, min_kept=100, weight=w)
    assert torch.equal(c.weight, w) and dict(c.named_buffers())["weight"] is c.weight
    assert list(c.state_dict()) == ["weight"]
    assert "weight=[19]" in repr(c)
    c.double()                                    # a buffer follows the module like nn.CrossEntropyLoss's
    assert c.weight.dtype == torch.float64
    plain = OhemCrossEntropyLoss()
    assert plain.weight is None and list(plain.state_dict()) == [] and "weight" not in repr(plain)
    # a network with an unweighted OHEM or default criterion keeps its state_dict keys
    net = nn.Module()
    net.criterion = OhemCrossEntropyLoss()
    assert list(net.state_dict()) == []
    net.criterion = nn.CrossEntropyLoss(ignore_index=255)
    assert list(net.state_dict()) == []
    for bad in ([1.0, 2.0], torch.ones(3, dtype=torch.int64), "w"):
        with pytest.raises(TypeError):
            OhemCrossEntropyLoss(weight=bad)
    for bad in (torch.ones(2, 3), torch.ones(()), torch.ones(0)):
        with pytest.raises(ValueError):
            OhemCrossEntropyLoss(weight=bad)


def test_ohem_weighted_module_has_no_cpu_fallback():
    crit = OhemCrossEntropyLoss(weight=torch.ones(3))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _wfwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, cw=P, eps=0.1, ws=P, loss=P,
          amax=P, lse=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_weighted_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, cw, eps,
                                                       ws, loss, amax, lse, None)


def _wbwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, cw=P, eps=0.1, lse=P, info=P,
          g=P, ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_weighted_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, cw, eps,
                                                       lse, info, g, ws, dl, None)


def _ofwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, thresh=0.7, min_kept=100,
          cw=P, ws=P, loss=P, amax=P, lse=P, pt=P, nll=P, thr=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_ohem_weighted_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255,
                                                            thresh, min_kept, cw, ws, loss, amax, lse, pt, nll, thr,
                                                            None)


def _obwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, cw=P, lse=P, pt=P, thr=P,
          info=P, g=P, ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_ohem_weighted_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, cw,
                                                            lse, pt, thr, info, g, ws, dl, None)


@pytest.mark.parametrize("call", [_wfwd, _wbwd, _ofwd, _obwd], ids=["fwd", "bwd", "ohem-fwd", "ohem-bwd"])
def test_weighted_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()


def test_weighted_entry_points_validate_options_and_outputs():
    for call in (_wfwd, _wbwd):
        for bad in (-0.01, 1.01, float("nan"), float("inf")):
            assert call(eps=bad) == -1 and b"label_smoothing" in _err(), (call, bad)
    for kw in ("ws", "loss", "lse"):
        assert _wfwd(**{kw: None}) == -1 and b"upsample_ce_weighted_fwd" in _err() and b"null" in _err(), kw
    for kw in ("lse", "info", "g", "ws", "dl"):
        assert _wbwd(**{kw: None}) == -1 and b"upsample_ce_weighted_bwd" in _err() and b"null" in _err(), kw
    for bad in (-0.01, 1.01, float("nan")):
        assert _ofwd(thresh=bad) == -1 and b"thresh" in _err(), bad
    assert _ofwd(min_kept=-1) == -1 and b"min_kept -1" in _err()
    for kw in ("ws", "loss", "lse", "pt", "nll", "thr"):
        assert _ofwd(**{kw: None}) == -1 and b"upsample_ce_ohem_weighted_fwd" in _err() and b"null" in _err(), kw
    for kw in ("lse", "pt", "thr", "info", "g", "ws", "dl"):
        assert _obwd(**{kw: None}) == -1 and b"upsample_ce_ohem_weighted_bwd" in _err() and b"null" in _err(), kw
    # the width limit of the staged rows is the plain backward's: 8 * Wo * 8 bytes <= 160 KB
    assert _wbwd(zoom=8, w=2600) == -1 and b"too large" in _err()
    assert _obwd(zoom=8, w=2600) == -1 and b"too large" in _err()


def test_weighted_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        h, w, C = 60, 60, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        assert (lib.semseg_upsample_ce_weighted_workspace_floats(2, ho, wo, zoom) ==
                lib.semseg_upsample_ce_zoom_workspace_floats(2, ho, wo, zoom))
        assert (lib.semseg_upsample_ce_weighted_bwd_workspace_floats(2, ho, w, C, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, ho, w, C, zoom))
    assert lib.semseg_upsample_ce_weighted_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_weighted_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
