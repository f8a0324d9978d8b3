"""CPU tier for the OHEM cross-entropy (semseg_b200/losses.py, csrc/tail.cu): the OHEM entry points reject bad arguments
with SEMSEG_E_INVALID and a message before any CUDA call, `fused_tail_supported` takes the native tail for
OhemCrossEntropyLoss exactly where it takes it for the default criterion, the module validates its options, and the
float64 oracle of the GPU tests agrees with a case computed by hand."""
import ctypes
import math

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import OhemCrossEntropyLoss
from tests.ohem_oracle import ohem_ce

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, thresh=0.7, min_kept=100,
         ws=P, loss=P, amax=P, lse=P, pt=P, nll=P, thr=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_ohem_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, thresh,
                                                   min_kept, ws, loss, amax, lse, pt, nll, thr, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, lse=P, pt=P, thr=P, info=P, g=P,
         ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_ohem_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, lse, pt, thr,
                                                   info, g, ws, dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_ohem_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()


def test_ohem_fwd_validates_options_and_outputs():
    for bad in (-0.01, 1.01, float("nan"), float("inf")):
        assert _fwd(thresh=bad) == -1 and b"upsample_ce_ohem" in _err() and b"thresh" in _err(), bad
    assert _fwd(min_kept=-1) == -1 and b"min_kept -1" in _err()
    for kw in ("ws", "loss", "lse", "pt", "nll", "thr"):
        assert _fwd(**{kw: None}) == -1 and b"upsample_ce_ohem_fwd" in _err() and b"null" in _err(), kw
    for kw in ("lse", "pt", "thr", "info", "g", "ws", "dl"):
        assert _bwd(**{kw: None}) == -1 and b"upsample_ce_ohem_bwd" in _err() and b"null" in _err(), kw
    assert _bwd(zoom=8, w=2600) == -1 and b"too large" in _err()


def test_ohem_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        h, w, C = 60, 60, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        # 4 + 4 x 256 selection words, then (loss, count) per 4096 pixels
        assert lib.semseg_upsample_ce_ohem_workspace_floats(2, ho, wo, zoom) == 1028 + 2 * -(-(2 * ho * wo) // 4096)
        assert (lib.semseg_upsample_ce_ohem_bwd_workspace_floats(2, ho, w, C, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, ho, w, C, zoom))
    assert lib.semseg_upsample_ce_ohem_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_ohem_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()


class _SubclassOhem(OhemCrossEntropyLoss):
    pass


def _target(n, h, w):
    return torch.zeros((n, h, w), dtype=torch.int64)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_supports_ohem_at_every_zoom(zoom):
    ohem = OhemCrossEntropyLoss(ignore_index=255, thresh=0.6, min_kept=1000)
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    ho, wo = zoom * 8 + 1, zoom * 10 + 1
    logits = torch.zeros((2, 9, 11, 21))
    y = _target(2, ho, wo)
    assert SF.fused_tail_supported(ohem, None, y, zoom, x_size)
    assert SF.fused_tail_supported(ohem, logits, y, zoom)
    assert SF.fused_tail_supported(ohem, torch.zeros((2, 9, 11, 256)), y, zoom)
    for other in {1, 2, 4, 8} - {zoom}:                     # the target at another zoom's size
        yo = _target(2, other * 8 + 1, other * 10 + 1)
        assert not SF.fused_tail_supported(ohem, None, yo, zoom, x_size)
        assert not SF.fused_tail_supported(ohem, logits, yo, zoom)
    assert not SF.fused_tail_supported(ohem, logits, _target(2, ho + 1, wo), zoom)
    assert not SF.fused_tail_supported(ohem, logits, y.int(), zoom)
    assert not SF.fused_tail_supported(ohem, torch.zeros((2, 9, 11, 257)), y, zoom)
    # a subclass may change the loss: it keeps the ATen tail
    assert not SF.fused_tail_supported(_SubclassOhem(), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(_SubclassOhem(), logits, y, zoom)


def test_ohem_constructor_validates():
    c = OhemCrossEntropyLoss()
    assert (c.ignore_index, c.thresh, c.min_kept) == (255, 0.7, 100000)
    c = OhemCrossEntropyLoss(ignore_index=-1, thresh=1, min_kept=0)
    assert (c.ignore_index, c.thresh, c.min_kept) == (-1, 1.0, 0) and isinstance(c.thresh, float)
    for kw in ({"thresh": -0.1}, {"thresh": 1.5}, {"thresh": float("nan")}, {"min_kept": -1}, {"min_kept": 2 ** 31}):
        with pytest.raises(ValueError):
            OhemCrossEntropyLoss(**kw)
    for kw in ({"min_kept": 1.5}, {"min_kept": True}, {"ignore_index": 255.0}):
        with pytest.raises(TypeError):
            OhemCrossEntropyLoss(**kw)
    assert "thresh=0.7" in repr(OhemCrossEntropyLoss())


def test_ohem_module_has_no_cpu_fallback():
    crit = OhemCrossEntropyLoss()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="256 classes"):
        crit(torch.zeros((1, 257, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match=r"\[N, H, W\]"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


def _two_class_logits(p):
    """[1, 2, 1, len(p)] logits whose softmax gives class 0 the probability p[i] at pixel i."""
    p = torch.tensor(p, dtype=torch.float64)
    return torch.stack([p.log(), (1 - p).log()]).view(1, 2, 1, -1)


def test_oracle_hand_computed():
    # p_t of the target class 0 at five pixels; the fourth is ignored, a sixth target is out of range
    x = _two_class_logits([0.9, 0.2, 0.6, 0.5, 0.4, 0.3])
    y = torch.tensor([[[0, 0, 0, 255, 0, 7]]])
    # valid p_t sorted: 0.2 0.4 0.6 0.9. min_kept 1 -> 0.4 < thresh 0.5: thr 0.5, kept {0.2, 0.4}
    loss, kept, thr, _ = ohem_ce(x, y, thresh=0.5, min_kept=1)
    assert thr == 0.5 and kept.view(-1).tolist() == [False, True, False, False, True, False]
    assert math.isclose(loss.item(), -(math.log(0.2) + math.log(0.4)) / 2, rel_tol=1e-12)
    # min_kept 3 -> k = 3 (the largest, 0.9) binds: thr 0.9, strict: 0.9 itself is not kept
    loss, kept, thr, _ = ohem_ce(x, y, thresh=0.5, min_kept=3)
    assert math.isclose(thr, 0.9, rel_tol=1e-12) and int(kept.sum()) == 3
    assert math.isclose(loss.item(), -(math.log(0.2) + math.log(0.4) + math.log(0.6)) / 3, rel_tol=1e-12)
    # min_kept above n_v is k = n_v - 1: the same
    assert math.isclose(ohem_ce(x, y, thresh=0.5, min_kept=10 ** 6)[0].item(), loss.item(), rel_tol=1e-15)
    # min_kept 0 with thresh 0: thr is the smallest p_t, nothing lies strictly below it: loss 0
    loss, kept, thr, _ = ohem_ce(x, y, thresh=0.0, min_kept=0)
    assert math.isclose(thr, 0.2, rel_tol=1e-12) and int(kept.sum()) == 0 and loss.item() == 0.0
    # no valid pixel: loss 0
    assert ohem_ce(x, torch.full_like(y, 255))[0].item() == 0.0
    # thresh 1 keeps every valid pixel: plain cross-entropy over the valid pixels
    ce = nn.CrossEntropyLoss(ignore_index=255)(x, torch.where(y == 7, torch.full_like(y, 255), y))
    assert math.isclose(ohem_ce(x, y, thresh=1.0, min_kept=0)[0].item(), ce.item(), rel_tol=1e-12)
