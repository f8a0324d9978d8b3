"""CPU tier: CutMix / ClassMix for mean-teacher training (losses.MixPseudoLabelLoss, csrc/mix.cu, the mixed form of
csrc/tail.cu upsample_pl_fwd) — the numpy oracle's box against a scalar statement at its edges, the ClassMix selection,
the oracle's closed-form gradient of the mixed pseudo-label loss against autograd, the criterion's validation, its place
outside the module tree, and the C entry points' argument checks."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import DiceLoss, MixPseudoLabelLoss, PseudoLabelLoss
from tests import util
from tests.mix_oracle import classmix_selected, cutmix_box, mix_mask, mixed_batch, mixed_teacher
from tests.pl_oracle import effective, pl_definition, pl_grad, pl_loss

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch
AREA, RATIO = (0.02, 0.4), (0.3, 1 / 0.3)
U_MAX = 1.0 - 2.0 ** -24     # the largest fp32 below 1: torch.rand's largest value


def _err():
    return _lib.load().semseg_last_error()


def _box_scalar(u, H, W, area, ratio):
    """The header's box in plain Python floats (IEEE doubles, math.sqrt correctly rounded)."""
    u1, u2, u3, u4 = (float(np.float32(v)) for v in u[1:5])
    a = (area[0] + (area[1] - area[0]) * u1) * H * W
    rho = ratio[0] + (ratio[1] - ratio[0]) * u2
    bw = min(W, max(1, math.floor(math.sqrt(a / rho))))
    bh = min(H, max(1, math.floor(math.sqrt(a * rho))))
    return (min(W - bw, math.floor(u4 * (W - bw + 1))), min(H - bh, math.floor(u3 * (H - bh + 1))), bw, bh)


# ------------------------------------------------------------------------------------------------ CutMix box
EDGE_U = [0.0, 2.0 ** -24, 0.5, U_MAX]


@pytest.mark.parametrize("hw", [(473, 473), (65, 129), (713, 97), (9, 9), (17, 2049)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("area", [AREA, (1.0, 1.0), (1e-6, 1e-6), (0.25, 0.25)], ids=["default", "area1", "tiny", "q"])
@pytest.mark.parametrize("ratio", [RATIO, (1.0, 1.0), (1e-3, 1e-3), (1e3, 1e3)], ids=["default", "1", "thin", "wide"])
def test_box_oracle_bit_exact_at_edges(hw, area, ratio):
    H, W = hw
    for u1 in EDGE_U:
        for u2 in EDGE_U:
            for u34 in ((0.0, 0.0), (U_MAX, U_MAX), (0.5, U_MAX), (U_MAX, 2.0 ** -24)):
                u = np.array([0.0, u1, u2, u34[0], u34[1]], dtype=np.float32)
                box = cutmix_box(u, H, W, area, ratio)
                assert box == _box_scalar(u, H, W, area, ratio)
                x0, y0, bw, bh = box
                assert 1 <= bw <= W and 1 <= bh <= H and 0 <= x0 <= W - bw and 0 <= y0 <= H - bh
    # u -> 0 puts the box at the origin, u = 1 - 2^-24 at the far edge
    x0, y0, bw, bh = cutmix_box(np.array([0, 0.5, 0.5, U_MAX, U_MAX], np.float32), H, W, area, ratio)
    assert (x0, y0) == (W - bw, H - bh)
    assert cutmix_box(np.array([0, 0.5, 0.5, 0, 0], np.float32), H, W, area, ratio)[:2] == (0, 0)


def test_box_edges_area_one_and_one_pixel():
    H, W = 65, 129
    # area 1 with ratio W/H... the box is clamped to the image
    x0, y0, bw, bh = cutmix_box(np.array([0, 0.0, 0.0, 0.3, 0.7], np.float32), H, W, (1.0, 1.0), (1.0, 1.0))
    assert (bw, bh) == (min(W, int(math.sqrt(H * W))), min(H, int(math.sqrt(H * W))))
    assert bh == H and x0 == min(W - bw, math.floor(np.float32(0.7) * (W - bw + 1)))
    # a tiny area: one pixel
    assert cutmix_box(np.array([0, 0.0, 0.0, 0.0, 0.0], np.float32), H, W, (1e-9, 1e-9), (1.0, 1.0))[2:] == (1, 1)
    # extreme ratios: one row or one column
    assert cutmix_box(np.array([0, 0.0, 0.0, 0.5, 0.5], np.float32), H, W, (0.01, 0.01), (1e4, 1e4))[2] == 1
    assert cutmix_box(np.array([0, 0.0, 0.0, 0.5, 0.5], np.float32), H, W, (0.01, 0.01), (1e-4, 1e-4))[3] == 1


def test_mask_and_mixed_batch_oracle():
    H, W, zoom = 17, 25, 2
    u = np.array([[0.1, 0.5, 0.5, 0.2, 0.9], [0.7, 0.5, 0.5, 0.2, 0.9], [0.49, 0.0, 0.0, 0.0, 0.0]], np.float32)
    m = mix_mask("cutmix", u, H, W, 0.5, AREA, RATIO)
    assert m[1].sum() == 0                                     # u0 = 0.7 >= p: not mixed
    x0, y0, bw, bh = cutmix_box(u[0], H, W, AREA, RATIO)
    assert m[0].sum() == bw * bh and m[0, y0:y0 + bh, x0:x0 + bw].all()
    assert mix_mask("cutmix", u, H, W, 0.0, AREA, RATIO).sum() == 0
    assert mix_mask("cutmix", u, H, W, 1.0, AREA, RATIO)[1].sum() > 0
    x = torch.randn((3, 3, H, W), dtype=torch.float64)
    y = torch.randint(0, 5, (3, (H - 1) // 8 * zoom + 1, (W - 1) // 8 * zoom + 1))
    xm, ym = mixed_batch(x, y, m, zoom)
    mb = torch.as_tensor(m).bool()
    assert torch.equal(xm[0][:, mb[0]], x[1][:, mb[0]]) and torch.equal(xm[0][:, ~mb[0]], x[0][:, ~mb[0]])
    assert torch.equal(xm[1], x[1]) and torch.equal(ym[1], y[1])
    s = 8 // zoom
    assert torch.equal(ym[0][mb[0, ::s, ::s]], y[1][mb[0, ::s, ::s]])


# ------------------------------------------------------------------------------------------------ ClassMix selection
def test_classmix_selection_ties_and_counts():
    prio = np.array([0.5, 0.5, 0.1, 0.5, 0.9, 0.2], np.float32)
    assert classmix_selected(prio, [3]) == {3}                             # k = 1: the class itself
    assert classmix_selected(prio, [0, 1]) == {0}                          # tie in u: the lower class
    assert classmix_selected(prio, [0, 1, 3]) == {0, 1}                    # k = 3: 2, ties by class
    assert classmix_selected(prio, [0, 2, 4, 5]) == {2, 5}                 # k = 4: 2
    assert classmix_selected(prio, [0, 1, 2, 3, 4]) == {2, 0, 1}           # k = 5: 3
    g = np.random.default_rng(0)
    prio = g.random(256).astype(np.float32)
    prio[10:20] = prio[10]                                                 # ties
    sel = classmix_selected(prio, range(256))                              # k = 256: 128
    order = sorted(range(256), key=lambda c: (prio[c], c))
    assert len(sel) == 128 and sel == set(order[:128])


def test_classmix_mask_pastes_partner_classes():
    amap = np.zeros((2, 9, 9), np.int64)
    amap[0, :4] = 3
    amap[1, :, :5] = 7
    amap[1, :, 5:] = 2
    u = np.zeros((2, 5 + 8), np.float32)
    u[:, 0] = 0.0                                                          # both mixed
    u[1, 5 + 7], u[1, 5 + 2] = 0.1, 0.9                                   # image 1 selects class 7
    u[0, 5 + 3], u[0, 5 + 0] = 0.8, 0.2                                   # image 0 selects class 0
    m = mix_mask("classmix", u, 9, 9, 0.5, AREA, RATIO, amap)
    assert (m[0] == (amap[1] == 7)).all() and (m[1] == (amap[0] == 0)).all()


# ------------------------------------------------------------------------------------------------ mixed loss oracle
@pytest.mark.parametrize("threshold", [0.0, 0.5, 1.5])
@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_mixed_oracle_gradient_equals_autograd(zoom, threshold):
    g = torch.Generator().manual_seed(zoom)
    n, h, w, c = 3, 4, 5, 6
    s = torch.randn((n, h, w, c), generator=g) * 3
    t = torch.randn((n, h, w, c), generator=g) * 3
    H, W = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    u = torch.rand((n, 5), generator=g).numpy()
    u[:, 0] = 0.0
    mask = mix_mask("cutmix", u, H, W, 0.5, (0.2, 0.6), RATIO)
    y = torch.randint(0, c, (n, zoom * (h - 1) + 1, zoom * (w - 1) + 1), generator=g)
    y[1] = 255
    _, ym = mixed_batch(torch.zeros((n, 1, H, W)), y, mask, zoom)
    tm = mixed_teacher(t, mask, zoom)                                      # float64 at the target size
    sd = s.double().requires_grad_(True)
    from tests.kd_oracle import upsampled
    ref = pl_definition(upsampled(sd, zoom).permute(0, 2, 3, 1), tm, ym, 1, threshold, 0.7, 1.0)
    (g_a,) = torch.autograd.grad(ref, sd)
    eff, wt, _ = effective(tm, ym, 1, threshold, 0.7, 1.0)
    assert abs(pl_loss(s.double(), eff, wt, zoom).item() - ref.item()) <= 1e-12 * max(abs(ref.item()), 1.0)
    g_c = pl_grad(s, eff, wt, zoom)
    assert float((g_c - g_a).abs().max()) <= 1e-12 * max(float(g_a.abs().max()), 1e-300)


def test_mixed_teacher_zero_and_full_mask():
    g = torch.Generator().manual_seed(1)
    t = torch.randn((3, 3, 4, 5), generator=g)
    H, W = 17, 25
    from tests.kd_oracle import upsampled
    zero = np.zeros((3, H, W), np.uint8)
    assert torch.equal(mixed_teacher(t, zero, 2), upsampled(t, 2).permute(0, 2, 3, 1))
    assert torch.equal(mixed_teacher(t, zero + 1, 2), upsampled(t.roll(-1, 0), 2).permute(0, 2, 3, 1))


# ------------------------------------------------------------------------------------------------ the criterion
@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


def test_mix_loss_validation_and_repr(nets):
    _, teacher = nets
    d = MixPseudoLabelLoss(teacher)
    assert (d.mix, d.p, d.area, d.ratio) == ('cutmix', 0.5, (0.02, 0.4), (0.3, 1 / 0.3))
    assert (d.threshold, d.pl_weight, d.ce_weight, d.ignore_index) == (0.95, 1.0, 1.0, 255)
    assert isinstance(d, PseudoLabelLoss) and d.last_mix() is None
    r = repr(d)
    assert "mix='cutmix'" in r and "p=0.5" in r and "area=(0.02, 0.4)" in r and "threshold=0.95" in r
    d = MixPseudoLabelLoss(teacher, mix='classmix', p=1, area=[0.1, 1], ratio=(1, 1), threshold=0, ignore_index=-1)
    assert (d.mix, d.p, d.area, d.ratio, d.threshold, d.ignore_index) == ('classmix', 1.0, (0.1, 1.0), (1.0, 1.0),
                                                                          0.0, -1)
    assert MixPseudoLabelLoss(teacher, p=0).p == 0.0
    for kw in ({"mix": 1}, {"mix": None}, {"p": "0.5"}, {"p": True}, {"area": 0.3}, {"area": (0.1,)},
               {"area": (0.1, "0.2")}, {"ratio": None}, {"ratio": (1, 2, 3)}, {"threshold": "0.9"},
               {"ignore_index": 255.0}):
        with pytest.raises(TypeError):
            MixPseudoLabelLoss(teacher, **kw)
    for kw in ({"mix": "mixup"}, {"p": -0.1}, {"p": 1.01}, {"p": float("nan")}, {"area": (0.0, 0.5)},
               {"area": (0.5, 0.2)}, {"area": (0.5, 1.5)}, {"area": (0.1, float("nan"))}, {"ratio": (0.0, 1.0)},
               {"ratio": (2.0, 1.0)}, {"ratio": (1.0, float("inf"))}, {"pl_weight": -1.0}):
        with pytest.raises(ValueError):
            MixPseudoLabelLoss(teacher, **kw)
    for bad in (nn.Conv2d(3, 3, 1), None, DiceLoss()):
        with pytest.raises(TypeError, match="PSPNet or PSANet"):
            MixPseudoLabelLoss(bad)


def test_mix_loss_teacher_held_outside_and_fixed(nets):
    student, teacher = nets
    d = MixPseudoLabelLoss(teacher, mix='classmix')
    assert list(d.state_dict()) == [] and list(d.children()) == []
    with pytest.raises(AttributeError, match="MixPseudoLabelLoss"):
        d.teacher = teacher
    with pytest.raises(AttributeError):
        d._teacher = student


def test_mix_loss_draw_checks(nets):
    d = MixPseudoLabelLoss(nets[1], mix='classmix')
    x = torch.zeros((2, 3, 17, 17))
    with pytest.raises(RuntimeError, match="no gradient through the mixing"):
        d.draw(x.requires_grad_(True), 21)
    with pytest.raises(TypeError, match="CUDA fp32"):
        d.draw(torch.zeros((2, 3, 17, 17)), 21)


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom, nets):
    teacher = nets[1]
    x_size = torch.Size((2, 3, 65, 81))
    logits = torch.zeros((2, 9, 11, 21))
    y = torch.zeros((2, zoom * 8 + 1, zoom * 10 + 1), dtype=torch.int64)
    for crit in (MixPseudoLabelLoss(teacher), MixPseudoLabelLoss(teacher, mix='classmix', p=1.0)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)

    class _Sub(MixPseudoLabelLoss):
        pass
    assert not SF.fused_tail_supported(_Sub(teacher), None, y, zoom, x_size)


def test_fused_tail_width_limit(nets):
    crit = MixPseudoLabelLoss(nets[1])
    for zoom, limit in ((8, 2389), (1, 19114)):
        w_ok = (limit - 1) // zoom + 1
        for w, expect in ((w_ok, True), (w_ok + 1, False)):
            y = torch.zeros((1, zoom + 1, zoom * (w - 1) + 1), dtype=torch.int64)
            assert SF.fused_tail_supported(crit, None, y, zoom, torch.Size((1, 3, 9, 8 * (w - 1) + 1))) == expect


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _apply(mode=0, x=P, N=2, Cin=3, H=65, W=81, y=P, Ho=None, Wo=None, zoom=8, u=P, us=5, p=0.5, alo=0.02, ahi=0.4,
           rlo=0.3, rhi=3.3, amap=P, sel=P, mask=P, xm=ctypes.c_void_p(32), ym=ctypes.c_void_p(48)):
    Ho = zoom * (H - 1) // 8 + 1 if Ho is None else Ho
    Wo = zoom * (W - 1) // 8 + 1 if Wo is None else Wo
    return _lib.load().semseg_mix_apply(mode, x, N, Cin, H, W, y, Ho, Wo, zoom, u, us, p, alo, ahi, rlo, rhi, amap,
                                        sel, mask, xm, ym, None)


def test_mix_apply_validates():
    assert _apply(mode=2) == -1 and b"mode 2" in _err()
    assert _apply(zoom=3) == -1 and b"zoom 3" in _err()
    for kw in ("x", "y", "u", "mask", "xm", "ym"):
        assert _apply(**{kw: None}) == -1 and b"null" in _err(), kw
    for kw in ("amap", "sel"):
        assert _apply(mode=1, **{kw: None}) == -1 and b"ClassMix needs" in _err(), kw
    assert _apply(H=64) == -1 and b"bad sizes" in _err()
    assert _apply(N=0) == -1 and b"bad sizes" in _err()
    assert _apply(Cin=0) == -1 and b"bad sizes" in _err()
    for zoom in (1, 2, 4, 8):
        assert _apply(zoom=zoom, Ho=zoom * 8 + 2) == -1 and b"needs Ho" in _err()
    assert _apply(us=4) == -1 and b"stride" in _err()
    for bad in (-0.1, 1.5, float("nan")):
        assert _apply(p=bad) == -1 and b"p " in _err(), bad
    for alo, ahi in ((0.0, 0.4), (0.5, 0.4), (0.1, 1.5), (0.1, float("nan"))):
        assert _apply(alo=alo, ahi=ahi) == -1 and b"area" in _err()
    for rlo, rhi in ((0.0, 1.0), (2.0, 1.0), (1.0, float("inf"))):
        assert _apply(rlo=rlo, rhi=rhi) == -1 and b"ratio" in _err()
    assert _apply(xm=P, x=P) == -1 and b"overwrite" in _err()


def test_mix_argmax_and_select_validate():
    lib = _lib.load()
    f = lib.semseg_mix_argmax_x8
    assert f(None, 21, 2, 9, 9, 21, P, P, None) == -1 and b"null" in _err()
    assert f(P, 21, 2, 9, 9, 21, None, P, None) == -1 and b"null" in _err()
    assert f(P, 257, 2, 9, 9, 257, P, P, None) == -1 and b"C<=256" in _err()
    assert f(P, 21, 0, 9, 9, 21, P, P, None) == -1 and b"bad sizes" in _err()
    assert f(P, 20, 2, 9, 9, 21, P, P, None) == -1 and b"pitch" in _err()
    g = lib.semseg_mix_select
    assert g(None, 26, P, 2, 21, P, None) == -1 and b"null" in _err()
    assert g(P, 25, P, 2, 21, P, None) == -1 and b"stride" in _err()
    assert g(P, 262, P, 2, 257, P, None) == -1 and b"C<=256" in _err()
    assert g(P, 26, P, 0, 21, P, None) == -1 and b"bad sizes" in _err()


def _pmix(mask=P, **kw):
    a = dict(s=P, ps=21, t=P, pt=24, N=2, h=9, w=7, C=21, tgt=P, zoom=4, ignore=255, thr=0.9, plw=1.0, cew=1.0, ws=P,
             info=P, amax=P, lse=P, eff=P, wt=P)
    a.update(kw)
    ho, wo = a["zoom"] * (a["h"] - 1) + 1, a["zoom"] * (a["w"] - 1) + 1
    return _lib.load().semseg_upsample_pl_mix_fwd(a["s"], a["ps"], a["t"], a["pt"], a["N"], a["h"], a["w"], a["C"],
                                                  a["tgt"], ho, wo, a["zoom"], a["ignore"], a["thr"], a["plw"],
                                                  a["cew"], mask, a["ws"], a["info"], a["amax"], a["lse"], a["eff"],
                                                  a["wt"], None)


def test_pl_mix_entry_point_validates():
    assert _pmix(mask=None) == -1 and b"null mix mask" in _err()
    assert _pmix(zoom=3) == -1 and b"zoom 3" in _err()
    assert _pmix(C=257, ps=257, pt=257) == -1 and b"C<=256" in _err()
    assert _pmix(thr=float("nan")) == -1 and b"threshold" in _err()
    assert _pmix(zoom=8, w=300) == -1 and b"at most 2389" in _err()
    for kw in ("ws", "lse", "eff", "wt", "info"):
        assert _pmix(**{kw: None}) == -1 and b"upsample_pl_mix_fwd" in _err() and b"null" in _err(), kw
    assert _pmix(ws=ctypes.c_void_p(20)) == -1 and b"8-byte aligned" in _err()
