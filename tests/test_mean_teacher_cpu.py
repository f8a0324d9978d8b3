"""CPU tier for mean-teacher training: the pseudo-label oracle (tests/pl_oracle.py) against float64 autograd of the
definition, optim.ModelEMA's construction and checkpoints, losses.PseudoLabelLoss's validation, `fused_tail_supported`
for it (the width limit included), and the new entry points' argument checks and workspace sizes, all before any CUDA
call."""
import ctypes

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import DiceLoss, DistillationLoss, PseudoLabelLoss
from semseg_b200.optim import ModelEMA
from tests import util
from tests.pl_oracle import effective, pl_definition, pl_grad, pl_loss

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _maps(seed, n=2, c=6, h=5, w=7):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, h, w, c), generator=g) * 3, torch.randn((n, h, w, c), generator=g) * 3


def _tgt(seed, n, ho, wo, c, p_ignore=0.4):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, c, (n, ho, wo), generator=g)
    t[torch.rand((n, ho, wo), generator=g) < p_ignore] = 255
    t[torch.rand((n, ho, wo), generator=g) < 0.03] = c + 2
    t[torch.rand((n, ho, wo), generator=g) < 0.02] = -3
    return t


# ------------------------------------------------------------------------------------------------ oracle
def _check_oracle(s, t, target, zoom, threshold, pl_weight, ce_weight):
    sd = s.double().requires_grad_(True)
    ref = pl_definition(sd, t, target, zoom, threshold, pl_weight, ce_weight)
    (g_a,) = torch.autograd.grad(ref, sd)
    eff, wt, _ = effective(t, target, zoom, threshold, pl_weight, ce_weight)
    assert abs(pl_loss(s.double(), eff, wt, zoom).item() - ref.item()) <= 1e-12 * max(abs(ref.item()), 1.0)
    g_c = pl_grad(s, eff, wt, zoom)
    scale = float(g_a.abs().max())
    assert float((g_c - g_a).abs().max()) <= 1e-12 * max(scale, 1e-300)
    return ref, g_a, eff


@pytest.mark.parametrize("weights", [(1.0, 1.0), (0.5, 2.0), (1.0, 0.0), (0.0, 1.0)], ids=["pl1-ce1", "pl0.5-ce2",
                                                                                        "pl1-ce0", "pl0-ce1"])
@pytest.mark.parametrize("threshold", [0.0, 0.3, 0.95, 1.5, -1.0])
@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_gradient_equals_autograd(zoom, threshold, weights):
    s, t = _maps(zoom * 7 + int(threshold * 10))
    n, h, w, c = s.shape
    target = _tgt(zoom, n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c)
    _check_oracle(s, t, target, zoom, threshold, *weights)


def test_oracle_ties_and_conf_at_threshold():
    """A teacher pixel with two equal top classes takes the first (torch.argmax); conf exactly equal to the threshold is
    confident (>=); both sides of the definition agree with the closed form there."""
    n, h, w, c = 1, 3, 4, 5
    s, _ = _maps(3, n, c, h, w)
    t = torch.full((n, h, w, c), -1e30)
    t[..., 1] = 0.0
    t[..., 3] = 0.0                     # classes 1 and 3 tie: yhat = 1, conf = 0.5 exactly
    t[0, 0, 0] = torch.tensor([0.0, 1.0, 2.0, 2.0, -1e30])      # tie between 2 and 3: yhat = 2
    target = torch.full((n, h, w), 255)
    eff0, _, _ = effective(t, target, 1, 0.0)
    assert int(eff0[0, 0, 0]) == 2 and bool((eff0.view(-1)[1:] == 1).all())
    eff, wt, conf = effective(t, target, 1, 0.5)
    assert int(eff[0, 0, 0]) == -1                             # conf < 0.5 there
    assert bool((eff.view(-1)[1:] == 1).all())
    assert bool((conf.view(-1)[1:] == 0.5).all())
    _check_oracle(s, t, target, 1, 0.5, 1.0, 1.0)
    eff2, _, _ = effective(t, target, 1, float(torch.nextafter(torch.tensor(0.5, dtype=torch.float64),
                                                               torch.tensor(1.0, dtype=torch.float64))))
    assert bool((eff2.view(-1)[1:] == -1).all())              # just above 0.5: not confident


@pytest.mark.parametrize("zoom", [1, 2])
def test_oracle_empty_sets(zoom):
    s, t = _maps(11)
    n, h, w, c = s.shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    # |L| = 0: every pixel unlabelled (an unlabelled batch), plus out-of-range targets that belong to neither set
    all_u = torch.full((n, ho, wo), 255)
    all_u[0, 0, :3] = c + 1
    ref, g, eff = _check_oracle(s, t, all_u, zoom, 0.0, 1.0, 1.0)
    assert bool((eff[0, 0, :3] == -1).all()) and ref.item() > 0
    # |U| = 0: a fully labelled batch is the plain mean CE times ce_weight
    all_l = torch.randint(0, c, (n, ho, wo), generator=torch.Generator().manual_seed(2))
    ref, g, _ = _check_oracle(s, t, all_l, zoom, 0.0, 1.0, 0.5)
    x = torch.nn.functional.interpolate(s.double().permute(0, 3, 1, 2), size=(ho, wo), mode="bilinear",
                                        align_corners=True) if zoom != 1 else s.double().permute(0, 3, 1, 2)
    assert abs(ref.item() - 0.5 * torch.nn.functional.cross_entropy(x, all_l).item()) <= 1e-12
    # neither: zero loss and an exactly zero gradient
    none = torch.full((n, ho, wo), c + 5)
    ref, g, _ = _check_oracle(s, t, none, zoom, 0.0, 1.0, 1.0)
    assert ref.item() == 0.0 and float(g.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ ModelEMA
@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


def test_model_ema_rejects_non_networks(nets):
    for bad in (nn.Conv2d(3, 3, 1), None, DiceLoss(), nn.Sequential(nn.Conv2d(3, 3, 1))):
        with pytest.raises(TypeError, match="PSPNet or PSANet"):
            ModelEMA(bad)
    for d in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="decay"):
            ModelEMA(nets[0], decay=d)
    for d in ("0.9", None, True):
        with pytest.raises(TypeError, match="decay"):
            ModelEMA(nets[0], decay=d)


def test_model_ema_shadow_is_a_separate_eval_copy(nets):
    student, teacher = nets
    student.criterion = DistillationLoss(teacher)
    try:
        ema = ModelEMA(student, decay=0.99)
        shadow = ema.module
        assert ema.decay == 0.99 and shadow is not student and not shadow.training
        assert getattr(shadow, "_sb_ema_shadow", False) and not getattr(student, "_sb_ema_shadow", False)
        assert all(not p.requires_grad for p in shadow.parameters())
        assert all(p.requires_grad for p in student.parameters())
        # no tensor, storage or module shared with the student (or with the student's teacher)
        ptrs = {t.untyped_storage().data_ptr() for t in list(student.parameters()) + list(student.buffers())}
        ptrs |= {t.untyped_storage().data_ptr() for t in list(teacher.parameters()) + list(teacher.buffers())}
        assert not any(t.untyped_storage().data_ptr() in ptrs for t in list(shadow.parameters()) + list(shadow.buffers()))
        assert not any(m is n for m in shadow.modules() for n in list(student.modules()) + list(teacher.modules()))
        # the criterion: a plain cross-entropy with the student's ignore_index, never the distillation loss
        assert type(shadow.criterion) is nn.CrossEntropyLoss and shadow.criterion.ignore_index == 255
        assert student.criterion.teacher is teacher
        # not a submodule of the student; the same state_dict keys and values
        assert all(m is not shadow for m in student.modules())
        sd_s, sd_e = student.state_dict(), shadow.state_dict()
        assert list(sd_s) == list(sd_e)
        assert all(torch.equal(sd_s[k], sd_e[k]) for k in sd_s)
        # a distillation loss on the shadow, then a second EMA of the student: the shadow is not copied into it
        student.criterion = DistillationLoss(shadow)
        ema2 = ModelEMA(student)
        assert type(ema2.module.criterion) is nn.CrossEntropyLoss
        assert not any(m is shadow for m in ema2.module.modules())
    finally:
        student.criterion = nn.CrossEntropyLoss(ignore_index=255)


def test_model_ema_unwraps_data_parallel(nets):
    student = nets[0]
    ema = ModelEMA(nn.DataParallel(student))
    assert type(ema.module) is type(student)
    assert list(ema.module.state_dict()) == list(student.state_dict())


def test_model_ema_state_dict_round_trip(nets):
    student = nets[0]
    ema = ModelEMA(student, decay=0.9)
    with torch.no_grad():
        for k, p in enumerate(ema.module.parameters()):
            p.add_(0.01 * (k + 1))
        ema.module.layer1[0].bn1.running_mean.add_(3.0)
        ema.module.layer1[0].bn1.num_batches_tracked.add_(7)
    sd = ema.state_dict()
    assert set(sd) == {"module", "decay"} and sd["decay"] == 0.9
    other = ModelEMA(student, decay=0.5)
    other.load_state_dict(sd)
    assert other.decay == 0.9
    a, b = ema.module.state_dict(), other.module.state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert not torch.equal(b["layer1.0.bn1.running_mean"], student.state_dict()["layer1.0.bn1.running_mean"])


def test_model_ema_update_has_no_cpu_fallback(nets):
    ema = ModelEMA(nets[0])
    with pytest.raises(_lib.SemsegError, match="no CPU fallback"):
        ema.update(nets[0])


def test_model_ema_update_checks_pairing(nets):
    student = nets[0]
    ema = ModelEMA(student)
    other = util.build_pspnet(50, 19)
    with pytest.raises(ValueError, match="cls.4.weight"):
        ema.update(other)
    ema.decay = 2.0
    with pytest.raises(ValueError, match="decay"):
        ema.update(student)


# ------------------------------------------------------------------------------------------------ PseudoLabelLoss
def test_pseudo_label_loss_validation(nets):
    _, teacher = nets
    d = PseudoLabelLoss(teacher)
    assert (d.threshold, d.pl_weight, d.ce_weight, d.ignore_index) == (0.95, 1.0, 1.0, 255)
    assert d.teacher is teacher and "threshold=0.95" in repr(d)
    d = PseudoLabelLoss(teacher, threshold=0, pl_weight=0, ce_weight=2, ignore_index=-1)
    assert (d.threshold, d.pl_weight, d.ce_weight, d.ignore_index) == (0.0, 0.0, 2.0, -1)
    assert PseudoLabelLoss(teacher, threshold=1.5).threshold == 1.5
    assert list(d.state_dict()) == [] and list(d.children()) == []
    with pytest.raises(AttributeError, match="PseudoLabelLoss"):
        d.teacher = teacher
    for kw in ({"ignore_index": 255.0}, {"threshold": "0.9"}, {"threshold": True}, {"pl_weight": None},
               {"ce_weight": False}):
        with pytest.raises(TypeError):
            PseudoLabelLoss(teacher, **kw)
    for kw in ({"threshold": float("nan")}, {"threshold": float("inf")}, {"pl_weight": -0.1},
               {"ce_weight": float("nan")}):
        with pytest.raises(ValueError):
            PseudoLabelLoss(teacher, **kw)
    for bad in (nn.Conv2d(3, 3, 1), None, DiceLoss()):
        with pytest.raises(TypeError, match="PSPNet or PSANet"):
            PseudoLabelLoss(bad)


def test_pseudo_label_run_teacher_checks(nets):
    _, teacher = nets
    x = torch.zeros((1, 3, 17, 17))
    teacher.train()
    try:
        with pytest.raises(RuntimeError, match="PseudoLabelLoss: the teacher must be in eval mode"):
            PseudoLabelLoss(teacher).run_teacher(x, 21)
    finally:
        teacher.eval()
    with pytest.raises(RuntimeError, match="move the teacher"):
        PseudoLabelLoss(teacher).run_teacher(x.to("meta"), 21)
    with pytest.raises(ValueError, match="21 classes, the student 19"):
        PseudoLabelLoss(teacher).run_teacher(x, 19)


def test_pseudo_label_module_has_no_cpu_fallback(nets):
    crit = PseudoLabelLoss(nets[1])
    y = torch.zeros((1, 5, 5), dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), y)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), y, torch.zeros((1, 3, 5, 5)))
    with pytest.raises(ValueError, match="256 classes"):
        crit(torch.zeros((1, 257, 5, 5)), y)


class _SubclassPL(PseudoLabelLoss):
    pass


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom, nets):
    teacher = nets[1]
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    ho, wo = zoom * 8 + 1, zoom * 10 + 1
    y = torch.zeros((2, ho, wo), dtype=torch.int64)
    for crit in (PseudoLabelLoss(teacher), PseudoLabelLoss(teacher, threshold=0.0, pl_weight=0.5, ce_weight=0.0)):
        assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
        assert SF.fused_tail_supported(crit, logits, y, zoom)
        assert SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 256)), y, zoom)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
        for other in {1, 2, 4, 8} - {zoom}:
            yo = torch.zeros((2, other * 8 + 1, other * 10 + 1), dtype=torch.int64)
            assert not SF.fused_tail_supported(crit, None, yo, zoom, x_size)
            assert not SF.fused_tail_supported(crit, logits, yo, zoom)
        assert not SF.fused_tail_supported(crit, logits, y.int(), zoom)
        assert not SF.fused_tail_supported(crit, logits, y[0], zoom)
        assert not SF.fused_tail_supported(crit, logits, y, 3)
    assert not SF.fused_tail_supported(_SubclassPL(teacher), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(_SubclassPL(teacher), logits, y, zoom)


def test_fused_tail_width_limit(nets):
    """The backward stages the focal rows kernel's 12-byte words: at most 224 KB / (12 Z) output columns."""
    crit = PseudoLabelLoss(nets[1])
    for zoom, limit in ((8, 2389), (4, 4778), (2, 9557), (1, 19114)):
        w_ok = (limit - 1) // zoom + 1                       # the widest logit map whose zoomed width fits
        for w, expect in ((w_ok, True), (w_ok + 1, False)):
            wo = zoom * (w - 1) + 1
            assert (wo <= limit) == expect
            y = torch.zeros((1, zoom + 1, wo), dtype=torch.int64)                   # 2 logit rows
            x_size = torch.Size((1, 3, 9, 8 * (w - 1) + 1))
            assert SF.fused_tail_supported(crit, None, y, zoom, x_size) == expect, (zoom, w)
            assert SF.fused_tail_supported(crit, torch.zeros((1, 2, w, 21)), y, zoom) == expect, (zoom, w)


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _pfwd(s=P, ps=21, t=P, pt=24, N=2, h=9, w=7, C=21, tgt=P, Ho=None, Wo=None, zoom=4, ignore=255, thr=0.9,
          plw=1.0, cew=1.0, ws=P, info=P, amax=P, lse=P, eff=P, wt=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_pl_fwd(s, ps, t, pt, N, h, w, C, tgt, Ho, Wo, zoom, ignore, thr, plw, cew, ws,
                                              info, amax, lse, eff, wt, None)


def test_pl_entry_point_validates():
    assert _pfwd(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert _pfwd(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    for kw in ("s", "t", "tgt"):
        assert _pfwd(**{kw: None}) == -1 and b"upsample_pl" in _err() and b"null" in _err(), kw
    assert _pfwd(C=257, ps=257, pt=257) == -1 and b"C<=256" in _err()
    assert _pfwd(N=0) == -1 and b"bad sizes" in _err()
    assert _pfwd(ps=20) == -1 and b"pitch" in _err()
    assert _pfwd(pt=20) == -1 and b"pitch" in _err()
    for bad in (float("nan"), float("inf"), -float("inf")):
        assert _pfwd(thr=bad) == -1 and b"threshold" in _err(), bad
    for kw in ("plw", "cew"):
        for bad in (-0.5, float("nan"), float("inf")):
            assert _pfwd(**{kw: bad}) == -1 and (b"pl_weight" if kw == "plw" else b"ce_weight") in _err()
    # the backward's 12-byte staged words: the Dice width limit
    assert _pfwd(zoom=8, w=300) == -1 and b"too large" in _err() and b"at most 2389" in _err()
    assert _pfwd(zoom=1, w=19115) == -1 and b"too large" in _err()
    for kw in ("ws", "info", "lse", "eff", "wt"):
        assert _pfwd(**{kw: None}) == -1 and b"upsample_pl_fwd" in _err() and b"null" in _err(), kw
    assert _pfwd(ws=ctypes.c_void_p(20)) == -1 and b"8-byte aligned" in _err()


def test_pl_workspace_sizes():
    lib = _lib.load()
    n, h, w = 2, 60, 61
    for zoom in (1, 2, 4, 8):
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        cols = 64 if zoom <= 2 else 128
        assert lib.semseg_upsample_pl_workspace_floats(n, ho, wo, zoom) == 4 + 4 * n * h * ((wo + cols - 1) // cols)
    assert lib.semseg_upsample_pl_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_pl_workspace_floats(0, 33, 33, 8) == -1 and b"bad sizes" in _err()


def test_ema_entry_point_validates():
    lib = _lib.load()
    assert lib.semseg_ema_multi(None, 1, 1, 0.9, None) == -1 and b"ema_multi" in _err() and b"null" in _err()
    assert lib.semseg_ema_multi(ctypes.c_void_p(20), 1, 1, 0.9, None) == -1 and b"aligned" in _err()
    for n_items, n_chunks in ((0, 1), (1, 0), (-1, 5)):
        assert lib.semseg_ema_multi(P, n_items, n_chunks, 0.9, None) == -1 and b"bad counts" in _err()
    for bad in (-1e-9, 1.0000001, float("nan"), float("inf")):
        assert lib.semseg_ema_multi(P, 1, 1, bad, None) == -1 and b"decay" in _err(), bad


def test_ema_item_layout_matches_header():
    import os
    import subprocess
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "semseg_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %d %d\n", sizeof(semseg_ema_item), offsetof(semseg_ema_item, source),
         offsetof(semseg_ema_item, n), offsetof(semseg_ema_item, kind), offsetof(semseg_ema_item, chunk0),
         SEMSEG_EMA_LERP_F32, SEMSEG_EMA_COPY_I64);
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), c, "-o", exe])
        v = list(map(int, subprocess.check_output([exe]).split()))
    E = _lib.EmaItem
    assert v == [ctypes.sizeof(E), E.source.offset, E.n.offset, E.kind.offset, E.chunk0.offset, _lib.EMA_LERP_F32,
                 _lib.EMA_COPY_I64]
