"""CPU tier for the Lovász-Softmax (+ cross-entropy) loss on the fused tail (csrc/tail.cu Lovász kernels and the
segmented sort of csrc/segsort.cu): the numpy float64 oracle of the GPU tests agrees with Berman's sort-based statement
in torch float64, and its closed-form gradient with autograd of that statement (sort order fixed), with and without
ties, with e = 0 elements, in 'all' mode with an absent class, for an image without a valid pixel and with nothing
valid; LovaszSoftmaxLoss validates its options; `fused_tail_supported` takes the native tail exactly for a
LovaszSoftmaxLoss of this type and within the width limit; the new entry points reject bad arguments with
SEMSEG_E_INVALID and a message before any CUDA call, and report their workspace sizes."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import DiceLoss, LovaszSoftmaxLoss, OhemCrossEntropyLoss
from tests.lovasz_oracle import lovasz, lovasz_torch, lovasz_weights

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch
MODES = [(cl, pi) for cl in ("present", "all") for pi in (False, True)]
MODE_IDS = ["present", "present-per-image", "all", "all-per-image"]


def _err():
    return _lib.load().semseg_last_error()


def _case(seed, n=2, c=5, h=6, w=7, ties=False, saturate=False):
    """float64 logits with ignored and out-of-range targets and one absent class (c - 1)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * 2
    if ties:
        x = torch.randint(0, 2, (n, c, h, w), generator=g).double()      # few distinct probabilities: many equal e
    t = torch.randint(0, c - 1, (n, h, w), generator=g)
    t[torch.rand((n, h, w), generator=g) < 0.1] = 255
    t[torch.rand((n, h, w), generator=g) < 0.03] = c + 2
    t[torch.rand((n, h, w), generator=g) < 0.03] = -1
    if saturate:
        # a third of the valid pixels are certain of their target: p = 1 there, p = 0 elsewhere, e = 0 in every class
        sat = (torch.rand((n, h, w), generator=g) < 0.3) & (t >= 0) & (t < c)
        hot = torch.nn.functional.one_hot(torch.where(sat, t, torch.zeros_like(t)), c).permute(0, 3, 1, 2).double()
        x = torch.where(sat.unsqueeze(1), 1000.0 * hot, x)
    return x, t


def _check(x, t, classes, per_image, ce_weight):
    x = x.clone().requires_grad_(True)
    ref = lovasz_torch(x, t, 255, classes, per_image, ce_weight)
    (g_a,) = torch.autograd.grad(ref, x)
    loss, grad, info = lovasz(x.detach().numpy(), t.numpy(), 255, classes, per_image, ce_weight)
    assert math.isclose(loss, ref.item(), rel_tol=1e-12, abs_tol=1e-15)
    scale = float(g_a.abs().max())
    assert float(np.abs(grad - g_a.numpy()).max()) <= 1e-12 * max(scale, 1e-300)
    return loss, grad, info


# ------------------------------------------------------------------------------------------------ oracle
def test_weights_hand_computed():
    # G = 2; fg flags in sorted order 1, 0, 1, 0
    g = lovasz_weights([1, 0, 1, 0])
    j = [1 - 1 / 2, 1 - 1 / 3, 1 - 0 / 3, 1 - 0 / 4]
    assert np.allclose(g, np.diff([0.0] + j), rtol=0, atol=1e-16)
    assert math.isclose(float(g.sum()), 1.0, rel_tol=1e-15)         # sum g_k = J_L = 1 whenever G > 0
    assert np.array_equal(lovasz_weights([0, 0, 0]), [1.0, 0.0, 0.0])  # G = 0: J_k = 1, the max error scores


def test_oracle_hand_computed():
    # two classes, three valid pixels: p(class 0) = 0.9, 0.2, 0.6; targets 0, 1, 0
    p = torch.tensor([0.9, 0.2, 0.6], dtype=torch.float64)
    x = torch.stack([p.log(), (1 - p).log()]).view(1, 2, 1, 3)
    t = torch.tensor([[[0, 1, 0]]])
    # class 0: e = 0.1, 0.2, 0.4 -> order 2, 1, 0; fg 1, 0, 1; G = 2: J = 1/2, 2/3, 1/3... computed by counts
    e0, fg0 = np.array([0.4, 0.2, 0.1]), [1, 0, 1]
    e1, fg1 = np.array([0.4, 0.2, 0.1]), [0, 1, 0]
    ref = (np.dot(e0, lovasz_weights(fg0)) + np.dot(e1, lovasz_weights(fg1))) / 2
    loss, _, _ = lovasz(x.numpy(), t.numpy())
    assert math.isclose(loss, ref, rel_tol=1e-14)
    assert math.isclose(lovasz_torch(x, t).item(), ref, rel_tol=1e-14)


@pytest.mark.parametrize("ce_weight", [0.0, 0.7])
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("kind", ["random", "ties", "saturated"])
def test_closed_form_gradient_equals_autograd(kind, mode, ce_weight):
    classes, per_image = mode
    x, t = _case({"random": 1, "ties": 2, "saturated": 3}[kind] + 10 * per_image, ties=kind == "ties",
                 saturate=kind == "saturated")
    _, _, info = _check(x, t, classes, per_image, ce_weight)
    if kind == "saturated":
        p = torch.softmax(x, 1)
        assert bool((p == 1.0).any())                                # e = 0 at the certain pixels
    if classes == "all":
        assert any(g == 0 for _, g in info["segments"].values())     # the absent class is scored
    else:
        assert all(g > 0 for _, g in info["segments"].values())


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_image_without_valid_pixel(mode):
    classes, per_image = mode
    x, t = _case(5, n=3)
    t[1] = 255
    loss, _, info = _check(x, t, classes, per_image, 0.5)
    assert all(si != 1 for si, _ in info["segments"]) if per_image else True
    if per_image:     # the empty image adds 0 but counts in 1/N
        w = {si: wv for (si, _), (wv, _) in info["segments"].items()}
        assert all(math.isclose(wv * 3 * sum(1 for (s, _) in info["segments"] if s == si), 1.0) for si, wv in w.items())


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_nothing_valid_is_zero(mode):
    classes, per_image = mode
    x, t = _case(6)
    t = torch.full_like(t, 255)
    t[0, 0, :2] = 7                                                  # out of range: not valid either
    for ce_weight in (0.0, 1.0):
        loss, grad, info = _check(x, t, classes, per_image, ce_weight)
        assert loss == 0.0 and float(np.abs(grad).max()) == 0.0 and info["n_valid"] == 0


def test_oracle_with_given_order_matches_its_own():
    x, t = _case(8, ties=True)
    loss, grad, info = lovasz(x.numpy(), t.numpy(), classes="all", per_image=True)
    # the orders the oracle would choose, handed back: the same result
    xv = x.numpy()
    p = np.exp(xv - xv.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    n, c, h, w = xv.shape
    pf, tf = p.transpose(1, 0, 2, 3).reshape(c, -1), t.numpy().reshape(-1)
    orders = {}
    for (si, k) in info["segments"]:
        idx = np.arange(si * h * w, (si + 1) * h * w)
        idx = idx[(tf[idx] != 255) & (tf[idx] >= 0) & (tf[idx] < c)]
        e = np.abs((tf[idx] == k) - pf[k, idx])
        orders[(si, k)] = idx[np.argsort(-e, kind="stable")]
    loss2, grad2, _ = lovasz(xv, t.numpy(), classes="all", per_image=True, orders=orders)
    assert loss2 == loss and np.array_equal(grad2, grad)


# ------------------------------------------------------------------------------------------------ module
def test_lovasz_loss_validation():
    d = LovaszSoftmaxLoss()
    assert (d.ignore_index, d.classes, d.per_image, d.ce_weight) == (255, "present", False, 0.0)
    d = LovaszSoftmaxLoss(ignore_index=-1, classes="all", per_image=True, ce_weight=2)
    assert (d.ignore_index, d.classes, d.per_image, d.ce_weight) == (-1, "all", True, 2.0)
    assert isinstance(d.ce_weight, float) and "per_image=True" in repr(d)
    assert list(d.state_dict()) == []
    for kw in ({"ignore_index": 255.0}, {"ignore_index": True}, {"classes": [0, 1]}, {"classes": None},
               {"classes": ("present",)}, {"per_image": 1}, {"per_image": None}, {"ce_weight": True},
               {"ce_weight": "1"}):
        with pytest.raises(TypeError):
            LovaszSoftmaxLoss(**kw)
    for kw in ({"classes": "Present"}, {"classes": "present "}, {"classes": ""}, {"ce_weight": -1.0},
               {"ce_weight": float("nan")}, {"ce_weight": float("inf")}):
        with pytest.raises(ValueError):
            LovaszSoftmaxLoss(**kw)


def test_lovasz_loss_has_no_cpu_fallback():
    crit = LovaszSoftmaxLoss(ce_weight=1.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="256 classes"):
        crit(torch.zeros((1, 257, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError, match="expected"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassLovasz(LovaszSoftmaxLoss):
    pass


def _target(n, h, w):
    return torch.zeros((n, h, w), dtype=torch.int64)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    ho, wo = zoom * 8 + 1, zoom * 10 + 1
    y = _target(2, ho, wo)
    for crit in (LovaszSoftmaxLoss(), LovaszSoftmaxLoss(classes="all", per_image=True, ce_weight=1.0)):
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
    assert not SF.fused_tail_supported(_SubclassLovasz(), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(_SubclassLovasz(), logits, y, zoom)
    # the existing decisions are unchanged
    for crit in (nn.CrossEntropyLoss(ignore_index=255), OhemCrossEntropyLoss(), DiceLoss()):
        assert SF.fused_tail_supported(crit, logits, y, zoom)
    assert not SF.fused_tail_supported(nn.CrossEntropyLoss(reduction="sum"), logits, y, zoom)


def test_fused_tail_lovasz_width_limit():
    """The Lovász rows kernel stages the Dice rows kernel's 12-byte words in 224 KB: 2389 columns at zoom 8, 19114 at
    zoom 1."""
    for zoom, limit in ((8, 2389), (4, 4778), (2, 9557), (1, 19114)):
        for want, ok in ((limit, True), (limit + zoom, False)):
            w = (want - 1) // zoom + 1
            wo = zoom * (w - 1) + 1
            assert (wo <= limit) == ok
            logits = torch.zeros((1, 3, w, 19))
            y = _target(1, 2 * zoom + 1, wo)
            assert SF.fused_tail_supported(LovaszSoftmaxLoss(), logits, y, zoom) == ok, (zoom, wo)
            assert SF.fused_tail_supported(nn.CrossEntropyLoss(), logits, y, zoom)


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _lfwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, classes_all=0, per_image=0,
          ce_weight=1.0, ws=P, loss=P, amax=P, lse=P, gamma=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_lovasz_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255,
                                                     classes_all, per_image, ce_weight, ws, loss, amax, lse, gamma,
                                                     None)


def _lbwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, target=P, Ho=None, Wo=None, zoom=4, lse=P, gamma=P, g=P, ws=P,
          dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_ce_lovasz_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, 255, lse, gamma,
                                                     g, ws, dl, None)


@pytest.mark.parametrize("call", [_lfwd, _lbwd], ids=["fwd", "bwd"])
def test_lovasz_entry_points_validate_shapes(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(target=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(pitch=20) == -1 and b"upsample_ce" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    assert call(zoom=8, w=300) == -1 and b"too large" in _err() and b"at most 2389" in _err()
    assert call(zoom=1, w=19115) == -1 and b"too large" in _err()
    # payloads hold a pixel index in 31 bits
    assert call(zoom=1, N=4000, h=800, w=700) == -1 and b"2^31" in _err()


def test_lovasz_entry_points_validate_options_and_outputs():
    for bad in (-0.01, float("nan"), float("inf")):
        assert _lfwd(ce_weight=bad) == -1 and b"ce_weight" in _err(), bad
    for kw in ("classes_all", "per_image"):
        for bad in (-1, 2):
            assert _lfwd(**{kw: bad}) == -1 and kw.encode() in _err(), (kw, bad)
    for kw in ("ws", "loss", "lse", "gamma"):
        assert _lfwd(**{kw: None}) == -1 and b"upsample_ce_lovasz_fwd" in _err() and b"null" in _err(), kw
    assert _lfwd(ws=ctypes.c_void_p(20)) == -1 and b"aligned" in _err()
    for kw in ("lse", "gamma", "g", "ws", "dl"):
        assert _lbwd(**{kw: None}) == -1 and b"upsample_ce_lovasz_bwd" in _err() and b"null" in _err(), kw


def test_segsort_validates_arguments():
    lib = _lib.load()
    for s, l in ((0, 5), (3, 0), (-1, 5), (2, 1 << 31)):
        assert lib.semseg_segsort_u32_pairs_workspace_bytes(s, l) == -1 and b"segsort" in _err(), (s, l)
        assert lib.semseg_segsort_u32_pairs(P, P, P, P, s, l, None, P, None) == -1 and b"segsort" in _err()
    for i in range(5):
        ptrs = [P] * 5
        ptrs[i] = None
        k, v, ka, va, ws = ptrs
        assert lib.semseg_segsort_u32_pairs(k, v, ka, va, 3, 100, None, ws, None) == -1 and b"null" in _err()


def test_workspace_sizes():
    lib = _lib.load()
    tile = 4096
    assert lib.semseg_segsort_u32_pairs_workspace_bytes(1, 1) == 1024
    assert lib.semseg_segsort_u32_pairs_workspace_bytes(150, 3579664) == 150 * 1024 * ((3579664 + tile - 1) // tile)
    for zoom in (1, 2, 4, 8):
        for per_image in (0, 1):
            n, h, w, c = 2, 20, 21, 150
            ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
            s, l = (n * c, ho * wo) if per_image else (c, n * ho * wo)
            nt = (l + tile - 1) // tile
            ev = lambda v: v + (v & 1)                       # noqa: E731
            f = ev(4 * s * l) + ev(s * 256 * nt) + n * (c + 1) + 2 * s
            f = ev(f) + 2 * s + s * nt
            f = ev(f) + 2 * s * nt + 2 * n * h * ((wo + 127) // 128)
            assert lib.semseg_upsample_ce_lovasz_workspace_floats(n, ho, wo, c, zoom, per_image) == f
            assert (lib.semseg_upsample_ce_lovasz_bwd_workspace_floats(n, ho, wo, w, c, zoom) ==
                    lib.semseg_upsample_ce_zoom_bwd_workspace_floats(n, ho, w, c, zoom) + n * ho * wo)
    assert lib.semseg_upsample_ce_lovasz_workspace_floats(2, 33, 33, 21, 3, 0) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_ce_lovasz_workspace_floats(2, 33, 33, 21, 4, 2) == -1 and b"per_image" in _err()
    assert lib.semseg_upsample_ce_lovasz_bwd_workspace_floats(2, 33, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
