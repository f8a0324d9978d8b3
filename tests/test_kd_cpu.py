"""CPU tier for pixel-wise knowledge distillation on the fused tail (csrc/tail.cu distillation kernels,
losses.DistillationLoss): the float64 oracle's closed-form gradient equals autograd, KL >= 0 with 0 for s = t and the
T^2 scaling, DistillationLoss validates its options and holds its teacher outside the student's module tree,
`fused_tail_supported` takes the native tail exactly for a DistillationLoss of this type, and the new entry points
reject bad arguments with SEMSEG_E_INVALID and a message before any CUDA call."""
import ctypes
import json
import math
import os

import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.losses import DiceLoss, DistillationLoss
from tests import util
from tests.kd_oracle import kd_grad, kd_loss, kl_term, upsampled

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _maps(seed, n=2, c=6, h=5, w=7):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn((n, h, w, c), generator=g) * 3
    t = torch.randn((n, h, w, c), generator=g) * 3
    return s, t


def _tgt(seed, n, ho, wo, c):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, c, (n, ho, wo), generator=g)
    t[torch.rand((n, ho, wo), generator=g) < 0.1] = 255
    t[torch.rand((n, ho, wo), generator=g) < 0.03] = c + 2
    return t


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("at", ["output", "logits"])
@pytest.mark.parametrize("temperature", [0.5, 1.0, 4.0])
@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_gradient_equals_autograd(zoom, temperature, at):
    s, t = _maps(zoom * 10 + int(temperature * 2))
    n, h, w, c = s.shape
    target = _tgt(3, n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c)
    sd = s.double().requires_grad_(True)
    main, kl = kd_loss(sd, t, target, zoom, temperature, kd_weight=0.7, ce_weight=0.0, at=at)
    (g_a,) = torch.autograd.grad(main, sd)
    kz = zoom if at == "output" else 1
    g_c = kd_grad(upsampled(sd, kz).detach(), upsampled(t, kz), temperature, 0.7)
    # the adjoint of the upsample takes the closed form at the KD resolution back to the maps
    (g_c_maps,) = torch.autograd.grad(upsampled(sd, kz), sd, g_c)
    assert float((g_c_maps - g_a).abs().max()) <= 1e-12 * float(g_a.abs().max())


def test_oracle_kl_non_negative_zero_for_equal_and_t2_scaling():
    for seed in range(4):
        s, t = _maps(seed)
        x, y = upsampled(s, 2), upsampled(t, 2)
        for temperature in (0.5, 1.0, 4.0):
            assert kl_term(x, y, temperature).item() >= 0.0
            assert kl_term(x, x, temperature).item() == 0.0
    s, t = _maps(7)
    target = _tgt(1, 2, 9, 13, 6)
    for temperature in (0.5, 2.0, 4.0):
        main, kl = kd_loss(s, t, target, 2, temperature, kd_weight=1.0, ce_weight=0.0)
        assert math.isclose(main.item(), temperature ** 2 * kl.item(), rel_tol=1e-14)
        main2, _ = kd_loss(s, t, target, 2, temperature, kd_weight=0.25, ce_weight=1.5)
        ce = kd_loss(s, t, target, 2, temperature, kd_weight=0.0, ce_weight=1.0)[0]
        assert math.isclose(main2.item(), 1.5 * ce.item() + 0.25 * temperature ** 2 * kl.item(), rel_tol=1e-13)


def test_oracle_hand_computed():
    # one pixel, two classes: p = (0.25, 0.75), q = (0.5, 0.5) at T = 1
    s = torch.tensor([math.log(0.25), math.log(0.75)], dtype=torch.float64).view(1, 1, 1, 2)
    t = torch.zeros((1, 1, 1, 2), dtype=torch.float64)
    ref = 0.5 * math.log(0.5 / 0.25) + 0.5 * math.log(0.5 / 0.75)
    assert math.isclose(kl_term(upsampled(s, 1), upsampled(t, 1), 1.0).item(), ref, rel_tol=1e-14)


# ------------------------------------------------------------------------------------------------ DistillationLoss
@pytest.fixture(scope="module")
def nets():
    return util.build_pspnet(50, 21), util.build_pspnet(50, 21, seed=1).eval()


def test_distillation_loss_validation(nets):
    _, teacher = nets
    d = DistillationLoss(teacher)
    assert (d.temperature, d.kd_weight, d.ce_weight, d.ignore_index, d.at) == (1.0, 1.0, 1.0, 255, "output")
    assert d.teacher is teacher and "temperature=1" in repr(d)
    d = DistillationLoss(teacher, temperature=4, kd_weight=0, ce_weight=2, ignore_index=-1, at="logits")
    assert (d.temperature, d.kd_weight, d.ce_weight, d.ignore_index, d.at) == (4.0, 0.0, 2.0, -1, "logits")
    assert list(d.state_dict()) == [] and list(d.children()) == []
    with pytest.raises(AttributeError):
        d.teacher = teacher
    for kw in ({"ignore_index": 255.0}, {"temperature": "1"}, {"kd_weight": True}, {"ce_weight": None}, {"at": 1}):
        with pytest.raises(TypeError):
            DistillationLoss(teacher, **kw)
    for kw in ({"temperature": 0.0}, {"temperature": -1.0}, {"temperature": float("nan")},
               {"temperature": float("inf")}, {"kd_weight": -0.1}, {"ce_weight": float("nan")}, {"at": "features"}):
        with pytest.raises(ValueError):
            DistillationLoss(teacher, **kw)
    for bad in (nn.Conv2d(3, 3, 1), None, DiceLoss()):
        with pytest.raises(TypeError, match="PSPNet or PSANet"):
            DistillationLoss(bad)


def test_run_teacher_checks(nets):
    student, teacher = nets
    x = torch.zeros((1, 3, 17, 17))
    teacher.train()
    try:
        with pytest.raises(RuntimeError, match="eval mode"):
            DistillationLoss(teacher).run_teacher(x, 21)
        teacher.eval()
        teacher.cls[1].train()                     # one BatchNorm left in training mode
        with pytest.raises(RuntimeError, match="eval mode"):
            DistillationLoss(teacher).run_teacher(x, 21)
    finally:
        teacher.eval()
    with pytest.raises(RuntimeError, match="move the teacher"):
        DistillationLoss(teacher).run_teacher(x.to("meta"), 21)
    with pytest.raises(ValueError, match="21 classes, the student 19"):
        DistillationLoss(teacher).run_teacher(x, 19)


def test_distillation_module_has_no_cpu_fallback(nets):
    crit = DistillationLoss(nets[1])
    y = torch.zeros((1, 5, 5), dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), y)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 3, 5, 5)), y, torch.zeros((1, 3, 5, 5)))
    with pytest.raises(ValueError, match="256 classes"):
        crit(torch.zeros((1, 257, 5, 5)), y)
    with pytest.raises(ValueError, match="expected"):
        crit(torch.zeros((1, 3, 5, 5)), torch.zeros((1, 5, 4), dtype=torch.int64))


def test_teacher_outside_student_module_tree(nets):
    student, teacher = nets
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "meta.json")
    ref = json.load(open(golden))["pspnet50_keys"]
    plain_keys = list(student.state_dict().keys())
    student.criterion = DistillationLoss(teacher)
    try:
        assert list(student.state_dict().keys()) == list(ref.keys()) == plain_keys
        assert all(m is not teacher for m in student.modules())
        assert not any(n.startswith("criterion.") for n, _ in student.named_modules())
        assert not any(p is q for p in student.parameters() for q in teacher.parameters())
        sync = nn.SyncBatchNorm.convert_sync_batchnorm(student)
        assert sync.criterion.teacher is teacher
        assert not any(isinstance(m, nn.SyncBatchNorm) for m in teacher.modules())
        assert any(isinstance(m, nn.SyncBatchNorm) for m in sync.modules())
        assert type(teacher.layer1[0].bn1) is nn.BatchNorm2d
    finally:
        student.criterion = nn.CrossEntropyLoss(ignore_index=255)


# ------------------------------------------------------------------------------------------------ fused_tail_supported
class _SubclassKD(DistillationLoss):
    pass


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom, nets):
    teacher = nets[1]
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    logits = torch.zeros((2, 9, 11, 21))
    ho, wo = zoom * 8 + 1, zoom * 10 + 1
    y = torch.zeros((2, ho, wo), dtype=torch.int64)
    for crit in (DistillationLoss(teacher), DistillationLoss(teacher, temperature=4.0, at="logits")):
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
    # a subclass may change the loss: it keeps the eager route
    assert not SF.fused_tail_supported(_SubclassKD(teacher), None, y, zoom, x_size)
    assert not SF.fused_tail_supported(_SubclassKD(teacher), logits, y, zoom)
    assert SF.fused_tail_supported(nn.CrossEntropyLoss(ignore_index=255), logits, y, zoom)


# ------------------------------------------------------------------------------------------------ C-ABI validation
def _kfwd(s=P, ps=21, t=P, pt=24, N=2, h=9, w=7, C=21, Ho=None, Wo=None, zoom=4, T=1.0, ws=P, kl=P, lse=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_kd_fwd(s, ps, t, pt, N, h, w, C, Ho, Wo, zoom, T, ws, kl, lse, None)


def _kbwd(s=P, ps=21, t=P, pt=24, N=2, h=9, w=7, C=21, Ho=None, Wo=None, zoom=4, T=1.0, kd_weight=1.0, lse=P, g=P,
          ws=P, dl=P):
    Ho = zoom * (h - 1) + 1 if Ho is None else Ho
    Wo = zoom * (w - 1) + 1 if Wo is None else Wo
    return _lib.load().semseg_upsample_kd_bwd(s, ps, t, pt, N, h, w, C, Ho, Wo, zoom, T, kd_weight, lse, g, ws, dl,
                                              None)


@pytest.mark.parametrize("call", [_kfwd, _kbwd], ids=["fwd", "bwd"])
def test_kd_entry_points_validate(call):
    assert call(zoom=3, Ho=25, Wo=19) == -1 and b"zoom 3" in _err()
    for zoom in (1, 2, 4, 8):
        assert call(zoom=zoom, Ho=zoom * 8 + 2) == -1 and (b"Ho=%d(h-1)+1" % zoom) in _err()
    assert call(s=None) == -1 and b"null" in _err()
    assert call(t=None) == -1 and b"null" in _err()
    assert call(C=257, ps=257, pt=257) == -1 and b"C<=256" in _err()
    assert call(N=0) == -1 and b"bad sizes" in _err()
    assert call(ps=20) == -1 and b"pitch" in _err()
    assert call(pt=20) == -1 and b"pitch" in _err()
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert call(T=bad) == -1 and b"temperature" in _err(), bad
    # 8-byte staged words: at most 2560 output columns at zoom 8, as the plain backward
    assert call(zoom=8, w=321) == -1 and b"too large" in _err() and b"at most 2560" in _err()
    assert call(zoom=1, w=20481) == -1 and b"too large" in _err()


def test_kd_entry_points_validate_outputs():
    for kw in ("ws", "kl", "lse"):
        assert _kfwd(**{kw: None}) == -1 and b"upsample_kd_fwd" in _err() and b"null" in _err(), kw
    for kw in ("lse", "g", "ws", "dl"):
        assert _kbwd(**{kw: None}) == -1 and b"upsample_kd_bwd" in _err() and b"null" in _err(), kw
    for bad in (-0.5, float("nan"), float("inf")):
        assert _kbwd(kd_weight=bad) == -1 and b"kd_weight" in _err(), bad


def test_kd_workspace_sizes():
    lib = _lib.load()
    n, h, w, c = 2, 60, 61, 150
    for zoom in (1, 2, 4, 8):
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        cols = 64 if zoom <= 2 else 128
        assert lib.semseg_upsample_kd_workspace_floats(n, ho, wo, zoom) == 2 * n * h * ((wo + cols - 1) // cols)
        assert (lib.semseg_upsample_kd_bwd_workspace_floats(n, ho, w, c, zoom) ==
                lib.semseg_upsample_ce_zoom_bwd_workspace_floats(n, ho, w, c, zoom) == 2 * n * h * w * c)
    assert lib.semseg_upsample_kd_workspace_floats(2, 33, 33, 3) == -1 and b"zoom 3" in _err()
    assert lib.semseg_upsample_kd_bwd_workspace_floats(2, 33, 9, 21, 5) == -1 and b"zoom 5" in _err()
    assert lib.semseg_upsample_kd_workspace_floats(0, 33, 33, 8) == -1 and b"bad sizes" in _err()
