"""CPU tier for the fused tail at every zoom factor (csrc/tail.cu, semseg_b200/functional.py): the zoom entry points reject
bad arguments with SEMSEG_E_INVALID and a message before any CUDA call, and `fused_tail_supported` takes the native tail
exactly for the default criterion at zoom 1, 2, 4 and 8 with the target at the zoomed size."""
import ctypes

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, ws=P, loss=P, amax=P, lse=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_zoom_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, ws, loss, amax,
                                                   lse, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, lse=P, info=P, g=P, ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_zoom_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, lse, info, g,
                                                   ws, dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_zoom_entry_points_validate_arguments(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1
    assert b"upsample_ce" in _err() and b"zoom 3" in _err()
    assert call(zoom=16) == -1 and b"zoom 16" in _err()
    assert call(zoom=0, Ho=1, Wo=1) == -1 and b"zoom 0" in _err()
    for zoom in (1, 2, 4, 8):
        ho = zoom * 8 + 1
        assert call(zoom=zoom, Ho=ho + 1) == -1                        # Ho != zoom(h-1)+1
        assert b"upsample_ce" in _err() and (b"Ho=%d(h-1)+1" % zoom) in _err()
        assert call(zoom=zoom, Wo=zoom * 6 + 2) == -1
        assert (b"Wo=%d(w-1)+1" % zoom) in _err()
    assert call(zoom=2, Ho=33) == -1                                    # the x8 size at zoom 2
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()         # more than 256 classes
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()            # pitch < C
    assert call(C=1, pitch=1) == -1


def test_zoom_entry_points_validate_outputs():
    assert _fwd(ws=None) == -1 and b"upsample_ce_fwd" in _err() and b"null" in _err()
    assert _fwd(loss=None) == -1 and b"upsample_ce_fwd" in _err()
    assert _fwd(lse=None) == -1 and b"upsample_ce_fwd" in _err()
    for kw in ("lse", "info", "g", "ws", "dl"):
        assert _bwd(**{kw: None}) == -1 and b"upsample_ce_bwd" in _err() and b"null" in _err(), kw
    # the backward stages zoom * Wo (lse, target) words in shared memory: at most 160 KB
    assert _bwd(zoom=8, w=2600) == -1 and b"too large" in _err()
    assert _bwd(zoom=1, w=21000) == -1 and b"too large" in _err()


def test_zoom_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        h, w, C = 60, 60, 150
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        # (loss, count) per forward CTA: h interval rows x ceil(Wo / 128) column blocks per image
        assert lib.semseg_upsample_ce_zoom_workspace_floats(2, ho, wo, zoom) == 2 * 2 * h * -(-wo // 128)
        assert lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, ho, w, C, zoom) == 2 * 2 * h * w * C
    # zoom 8 is what the x8 entry points size
    assert (lib.semseg_upsample_ce_zoom_workspace_floats(3, 473, 473, 8) ==
            lib.semseg_upsample_ce_workspace_floats(3, 473, 473))
    assert (lib.semseg_upsample_ce_zoom_bwd_workspace_floats(3, 473, 60, 150, 8) ==
            lib.semseg_upsample_ce_bwd_workspace_floats(3, 473, 60, 150))
    assert lib.semseg_upsample_ce_zoom_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_zoom_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()


class _SubclassCE(nn.CrossEntropyLoss):
    pass


def _target(n, h, w):
    return torch.zeros((n, h, w), dtype=torch.int64)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_supported_at_every_zoom(zoom):
    ce = nn.CrossEntropyLoss(ignore_index=255)
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    ho, wo = zoom * 8 + 1, zoom * 10 + 1
    logits = torch.zeros((2, 9, 11, 21))
    y = _target(2, ho, wo)
    assert SF.fused_tail_supported(ce, None, y, zoom, x_size)
    assert SF.fused_tail_supported(ce, logits, y, zoom)
    # the target at another zoom's size, or transposed
    for other in {1, 2, 4, 8} - {zoom}:
        yo = _target(2, other * 8 + 1, other * 10 + 1)
        assert not SF.fused_tail_supported(ce, None, yo, zoom, x_size)
        assert not SF.fused_tail_supported(ce, logits, yo, zoom)
    assert not SF.fused_tail_supported(ce, logits, _target(2, wo, ho), zoom)
    assert not SF.fused_tail_supported(ce, logits, _target(2, ho + 1, wo), zoom)
    # target dtype / rank
    assert not SF.fused_tail_supported(ce, logits, y.int(), zoom)
    assert not SF.fused_tail_supported(ce, logits, y[0], zoom)
    assert not SF.fused_tail_supported(ce, logits, None, zoom)
    # more than 256 classes
    assert not SF.fused_tail_supported(ce, torch.zeros((2, 9, 11, 257)), y, zoom)
    assert SF.fused_tail_supported(ce, torch.zeros((2, 9, 11, 256)), y, zoom)
    # criteria the kernel does not implement: unchanged conditions
    for crit in (_SubclassCE(ignore_index=255), nn.CrossEntropyLoss(ignore_index=255, reduction="sum"),
                 nn.CrossEntropyLoss(ignore_index=255, weight=torch.ones(21)),
                 nn.CrossEntropyLoss(ignore_index=255, label_smoothing=0.1), nn.NLLLoss(ignore_index=255)):
        assert not SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert not SF.fused_tail_supported(crit, logits, y, zoom)


def test_fused_tail_rejects_other_zoom_factors():
    ce = nn.CrossEntropyLoss(ignore_index=255)
    logits = torch.zeros((1, 9, 9, 21))
    for zoom in (0, 3, 16):
        y = _target(1, zoom * 8 + 1, zoom * 8 + 1)
        assert not SF.fused_tail_supported(ce, logits, y, zoom)
        assert not SF.fused_tail_supported(ce, None, y, zoom, torch.Size((1, 3, 65, 65)))
