"""CPU tier for the Active Boundary Loss (losses.ActiveBoundaryLoss, csrc/boundary.cu) and Boundary IoU
(metrics.boundaryIoUGPU): the float64 contract of the GPU tests has an exact distance map (brute force agrees, ignore
blobs and a boundary-free image included), finds the published threshold loop's level and has the closed-form
gradient autograd gives with the selection frozen; the Boundary IoU bands are the paper's per-class cv2 erosion; the
criterion validates its options and every option partitions the graph key; `fused_tail_supported` takes the native
tail where the kernels apply; the entry points reject bad arguments before any CUDA call and the workspace sizes are
the stated ones."""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import ActiveBoundaryLoss, graph_key
from tests import abl_oracle as O

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _labels(n, h, w, classes, seed, blobs=True):
    """Blocky label maps with a few ignored blobs, as scene labels look at the loss grid."""
    g = np.random.default_rng(seed)
    cells = g.integers(0, classes, (n, (h + 5) // 6, (w + 5) // 6))
    t = np.repeat(np.repeat(cells, 6, 1), 6, 2)[:, :h, :w].copy()
    if blobs:
        for k in range(n):
            y, x = g.integers(0, h), g.integers(0, w)
            t[k, y:y + 3, x:x + 4] = 255
    return t


# ------------------------------------------------------------------------------------------------ oracle
def _brute_e(b):
    e = np.full(b.shape, -1, np.int64)
    for n in range(b.shape[0]):
        ys, xs = np.nonzero(b[n])
        if len(ys) == 0:
            continue
        yy, xx = np.indices(b[n].shape)
        e[n] = ((yy[..., None] - ys) ** 2 + (xx[..., None] - xs) ** 2).min(-1)
    return e


@pytest.mark.parametrize("shape", [(2, 13, 17), (1, 1, 9), (3, 8, 1), (2, 23, 11)])
def test_distance_map_is_the_brute_force_one(shape):
    t = _labels(*shape, classes=3, seed=sum(shape))
    t[0] = 1                                                  # a uniform image: no GT boundary
    b = O.gt_boundary(t, 255)
    assert not b[0].any()
    e = O.edt_sq(b)
    assert np.array_equal(e, _brute_e(b))
    D = O.dist_map(t, 255)
    assert np.isinf(D[0]).all()
    ref = np.maximum(np.sqrt(e[1:].astype(np.float64)) - 1, 0).astype(np.float32)
    assert np.array_equal(D[1:], ref)


def test_gt_boundary_marks_ignore_and_label_changes():
    t = np.array([[[0, 0, 1], [0, 255, 1], [2, 2, 2]]])
    b = O.gt_boundary(t, 255)
    assert b.tolist() == [[[False, True, False], [True, True, True], [False, False, False]]]


@pytest.mark.parametrize("ratio", [0.0, 0.001, 0.01, 0.05, 0.5, 1.0])
def test_level_is_the_published_loop(ratio):
    g = torch.Generator().manual_seed(4)
    k = (torch.rand((2, 31, 29), generator=g, dtype=torch.float64) ** 6 * 3).float().numpy()
    k[0, :3] = 0.0
    max_n = ratio * 31 * 29
    assert O.level(k, max_n) == O.level_by_loop(k, max_n)


def test_levels_are_float64_products_rounded_once():
    t = O.levels()
    assert t.dtype == np.float32 and t[0] == np.float32(1e-5)
    assert t[1] == np.float32(1e-5 * 1.2) and t[255] == np.float32(np.prod([1e-5] + [1.2] * 255))
    assert (np.diff(t.astype(np.float64)) > 0).all()


@pytest.mark.parametrize("eps,clip", [(0.2, 20.0), (0.0, 1.5), (1.0, 3.0)])
def test_closed_form_gradient_is_autograd_with_the_selection_frozen(eps, clip):
    g = torch.Generator().manual_seed(7)
    t = _labels(2, 14, 12, 4, seed=3)
    s = torch.randn((2, 4, 14, 12), generator=g, dtype=torch.float64) * 2
    r = O.contract(s, t, 255, 0.2, clip, eps)
    assert r["M"] > 10
    sv = s.clone().requires_grad_(True)
    loss, M = O.term(sv, r["D"], r["dir"], r["sel"], eps, clip)
    loss.backward()
    assert M == r["M"] and abs(loss.item() - r["abl"]) < 1e-12
    assert torch.allclose(sv.grad, r["grad"], rtol=1e-9, atol=1e-13)


def test_no_selection_gives_zero_loss_and_gradient():
    s = torch.randn((1, 3, 9, 9), dtype=torch.float64)
    uniform = np.zeros((1, 9, 9), np.int64)                   # no GT boundary: nothing is selected
    r = O.contract(s, uniform, 255, 0.3, 20.0, 0.2)
    assert r["M"] == 0 and r["abl"] == 0.0 and float(r["grad"].abs().max()) == 0.0
    r = O.contract(s, _labels(1, 9, 9, 3, seed=1), 255, 0.0, 20.0, 0.2)   # max_N = 0: no pixel above t_j*
    assert r["M"] == 0 and not r["B"].any()


# ------------------------------------------------------------------------------------------------ Boundary IoU
@pytest.mark.parametrize("shape,d", [((2, 37, 53), 1), ((1, 40, 24), 3), ((3, 17, 17), 2), ((1, 9, 31), 5)])
def test_boundary_iou_bands_are_the_papers_cv2_erosion(shape, d):
    t = _labels(*shape, classes=5, seed=d)
    rng = np.random.default_rng(d)
    o = np.where(rng.random(shape) < 0.1, rng.integers(0, 5, shape), np.where(t == 255, 0, t))
    assert np.array_equal(O.biou_counts(o, t, 5, 255, d), O.biou_counts_cv2(o, t, 5, 255, d))


def test_band_width_rounds_like_python():
    assert O.band_width(473, 473) == round(0.02 * (2 * 473 * 473) ** 0.5) == 13
    assert O.band_width(5, 5) == 1


# ------------------------------------------------------------------------------------------------ criterion
def test_constructor_defaults_and_repr():
    c = ActiveBoundaryLoss()
    assert (c.ignore_index, c.abl_weight, c.ce_weight, c.label_smoothing, c.max_n_ratio, c.max_clip_dist) == (
        255, 1.0, 1.0, 0.2, 0.01, 20.0)
    assert "max_clip_dist=20" in repr(c)


@pytest.mark.parametrize("kw,bad,exc", [
    ("ignore_index", 2.5, TypeError), ("ignore_index", True, TypeError),
    ("abl_weight", -1.0, ValueError), ("abl_weight", float("nan"), ValueError), ("abl_weight", "1", TypeError),
    ("ce_weight", float("inf"), ValueError), ("ce_weight", None, TypeError),
    ("label_smoothing", 1.5, ValueError), ("label_smoothing", -0.1, ValueError),
    ("max_n_ratio", 1.01, ValueError), ("max_n_ratio", -0.01, ValueError), ("max_n_ratio", float("nan"), ValueError),
    ("max_clip_dist", 0.0, ValueError), ("max_clip_dist", -2.0, ValueError), ("max_clip_dist", float("inf"), ValueError),
    ("max_clip_dist", False, TypeError),
])
def test_constructor_validation(kw, bad, exc):
    with pytest.raises(exc):
        ActiveBoundaryLoss(**{kw: bad})


def test_module_has_no_cpu_fallback():
    c = ActiveBoundaryLoss()
    with pytest.raises(RuntimeError):
        c(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError):
        c(torch.zeros((1, 257, 5, 5)), torch.zeros((1, 5, 5), dtype=torch.int64))
    with pytest.raises(ValueError):
        c.aux_loss(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 6), dtype=torch.int64))


@pytest.mark.parametrize("attr,value", [("ignore_index", 0), ("abl_weight", 0.5), ("ce_weight", 0.0),
                                        ("label_smoothing", 0.1), ("max_n_ratio", 0.02), ("max_clip_dist", 10.0)])
def test_every_option_partitions_the_graph_key(attr, value):
    a, b = ActiveBoundaryLoss(), ActiveBoundaryLoss()
    assert graph_key(a) == graph_key(b)
    setattr(b, attr, value)
    assert graph_key(a) != graph_key(b)
    assert graph_key(ActiveBoundaryLoss(**{attr: value})) == graph_key(b)
    assert graph_key(a) != graph_key(nn.CrossEntropyLoss(ignore_index=255))


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom):
    h = w = 9
    x_size = (2, 3, 8 * (h - 1) + 1, 8 * (w - 1) + 1)
    y = torch.zeros((2, zoom * (h - 1) + 1, zoom * (w - 1) + 1), dtype=torch.int64)
    assert SF.fused_tail_supported(ActiveBoundaryLoss(), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(ActiveBoundaryLoss(), None, y[:, 1:], zoom, x_size)
    assert not SF.fused_tail_supported(ActiveBoundaryLoss(), None, y.int(), zoom, x_size)
    assert not SF.fused_tail_supported(type("Sub", (ActiveBoundaryLoss,), {})(), None, y, zoom, x_size)
    # the plain backward's width limit: 8 bytes per pixel of `zoom` rows in 160 KB
    w_max = (160 * 1024 // (8 * zoom) - 1) // zoom + 1
    for wl, ok in ((w_max, True), (w_max + 1, False)):
        yw = torch.zeros((1, zoom * 2 + 1, zoom * (wl - 1) + 1), dtype=torch.int64)
        assert SF.fused_tail_supported(ActiveBoundaryLoss(), None, yw, zoom, (1, 3, 17, 8 * (wl - 1) + 1)) == ok


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _fwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, zoom=4, lse=P, target=P, ignore=255, ratio=0.01, clip=20.0,
         eps=0.2, state=P, loss=P):
    return _lib.load().semseg_abl_fwd(logits, pitch, N, h, w, C, zoom, lse, target, ignore, ratio, clip, eps, state,
                                      loss, None)


def _bwd(logits=P, pitch=21, N=2, h=9, w=7, C=21, zoom=4, lse=P, state=P, info=P, weight=1.0, g=P, ws=P, dl=P):
    return _lib.load().semseg_abl_bwd(logits, pitch, N, h, w, C, zoom, lse, state, info, weight, g, ws, dl, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_entry_points_validate_shapes(call):
    assert call(zoom=3) == -1 and b"zoom 3" in _err()
    assert call(logits=None) == -1 and b"null" in _err()
    assert call(lse=None) == -1 and b"null" in _err()
    assert call(C=257, pitch=257) == -1 and b"C<=256" in _err()
    assert call(C=0, pitch=0) == -1 and b"bad sizes" in _err()
    assert call(pitch=20) == -1 and b"bad sizes" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    assert call(N=65536) == -1 and b"bad sizes" in _err()
    assert call(w=0) == -1 and b"bad sizes" in _err()


def test_entry_points_validate_outputs_and_options():
    for kw in ("target", "state", "loss"):
        assert _fwd(**{kw: None}) == -1 and b"abl_fwd" in _err() and b"null" in _err(), kw
    for bad in (-0.1, 1.5, float("nan"), float("inf")):
        assert _fwd(ratio=bad) == -1 and b"max_n_ratio" in _err()
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert _fwd(clip=bad) == -1 and b"max_clip_dist" in _err()
    for bad in (-0.1, 1.1, float("nan")):
        assert _fwd(eps=bad) == -1 and b"label_smoothing" in _err()
    for kw in ("state", "info", "g", "dl", "ws"):
        assert _bwd(**{kw: None}) == -1 and b"abl_bwd" in _err() and b"null" in _err(), kw
    assert _bwd(zoom=1, ws=None, dl=None) == -1 and b"null" in _err()
    for bad in (-0.5, float("nan"), float("inf")):
        assert _bwd(weight=bad) == -1 and b"abl_weight" in _err()


def test_boundary_iou_entry_point_validates():
    lib = _lib.load()

    def call(pred=P, target=P, N=2, H=9, W=7, K=21, ignore=255, d=1, ws=P, counts=P):
        return lib.semseg_boundary_iou_hist(pred, target, N, H, W, K, ignore, d, ws, counts, None)
    for kw in ("pred", "target", "ws", "counts"):
        assert call(**{kw: None}) == -1 and b"null" in _err(), kw
    for kw, bad in (("N", 0), ("H", 0), ("W", -1), ("K", 0), ("K", 4097)):
        assert call(**{kw: bad}) == -1 and b"bad sizes" in _err(), kw
    assert call(d=0) == -1 and b"band width" in _err()


def test_workspace_sizes():
    lib = _lib.load()
    for zoom in (1, 2, 4, 8):
        for (n, h, w, C) in ((16, 60, 60, 21), (16, 60, 60, 150), (2, 3, 5, 2)):
            hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
            p = n * hg * wg
            tiles = n * -(-hg // 16) * -(-wg // 16)
            assert lib.semseg_abl_workspace_floats(n, h, w, C, zoom, 0) == 10 * p + (p + 3) // 4 + 257 + 2 + 2 * tiles
            assert lib.semseg_abl_workspace_floats(n, h, w, C, zoom, 1) == (0 if zoom == 1 else n * C * wg * (hg + h))
    # the header's figures at 16 x 473^2, zoom 8
    assert 0.14e9 < 4 * lib.semseg_abl_workspace_floats(16, 60, 60, 21, 8, 0) < 0.16e9
    assert 0.33e9 < 4 * lib.semseg_abl_workspace_floats(16, 60, 60, 21, 8, 1) < 0.35e9
    assert 2.4e9 < 4 * lib.semseg_abl_workspace_floats(16, 60, 60, 150, 8, 1) < 2.5e9
    assert lib.semseg_abl_workspace_floats(2, 9, 9, 21, 3, 0) == -1 and b"zoom 3" in _err()
    assert lib.semseg_abl_workspace_floats(2, 9, 9, 21, 8, 2) == -1 and b"pass 2" in _err()
    assert lib.semseg_abl_workspace_floats(0, 9, 9, 21, 8, 0) == -1
