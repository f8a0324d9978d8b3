"""CPU tier for class-incremental training (MiB's unbiased cross-entropy and distillation on the fused tail,
losses.IncrementalLoss, incremental.expand_classifier):

  * the float64 oracle agrees with a per-pixel loop on hand-sized cases (old labels count as background, ignored and
    out-of-range targets, an all-ignored batch gives 0) and its closed-form gradients equal autograd;
  * IncrementalLoss validates its options and its teacher, and its graph key changes with each option;
  * the new entry points reject bad arguments and sizes before any CUDA call, and fused_tail_supported takes the native
    tail exactly for an IncrementalLoss within the staged width;
  * expand_classifier gives a fresh network's state_dict keys and shapes, keeps the old rows, imprints the background,
    composes over two steps, and keeps the old network's old-class probabilities and background mass."""
import copy
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from semseg_b200 import _lib
from semseg_b200 import functional as SF
from semseg_b200.incremental import expand_classifier
from semseg_b200.losses import DistillationLoss, IncrementalLoss, graph_key
from tests import util
from tests.incremental_oracle import incremental_loss, unce, unce_grad, unkd, unkd_grad
from tests.kd_oracle import upsampled

P = ctypes.c_void_p(16)      # never dereferenced: validation fails before any launch


def _err():
    return _lib.load().semseg_last_error()


def _lse(v):
    m = max(v)
    return m + math.log(sum(math.exp(a - m) for a in v))


# ------------------------------------------------------------------------------------------------ oracle
def _loop_unce(x, target, c_old, ignore_index=255):
    x = x.double().numpy()
    n, c, h, w = x.shape
    tot, cnt = 0.0, 0
    for i in range(n):
        for y in range(h):
            for z in range(w):
                t = int(target[i, y, z])
                if t == ignore_index or t < 0 or t >= c:
                    continue
                v = list(x[i, :, y, z])
                tot += _lse(v) - (_lse(v[:c_old]) if t < c_old else v[t])
                cnt += 1
    return tot / cnt if cnt else 0.0


def _loop_unkd(s, t, c_old, alpha):
    s, t = s.double().numpy(), t.double().numpy()
    n, c, h, w = s.shape
    tot = 0.0
    for i in range(n):
        for y in range(h):
            for z in range(w):
                v = list(s[i, :, y, z])
                u = [alpha * a for a in t[i, :, y, z]]
                lt = _lse(u)
                q = [math.exp(a - lt) for a in u]
                la = _lse(v)
                lb = _lse([v[0]] + v[c_old:])
                k = q[0] * (lb - la) + sum(q[j] * (v[j] - la) for j in range(1, c_old))
                tot += -k / c_old
    return tot / (n * h * w)


def _case(seed, n=2, c=5, c_old=3, h=3, w=4):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn((n, c, h, w), generator=g, dtype=torch.float64) * 3
    t = torch.randn((n, c_old, h, w), generator=g, dtype=torch.float64) * 3
    y = torch.randint(0, c, (n, h, w), generator=g)
    y[0, 0, 0], y[0, 0, 1], y[1, 2, 3] = 255, c + 1, -3       # ignored and out-of-range targets
    y[0, 1, 0], y[1, 0, 0] = 0, c_old - 1                      # an old label of each end
    return s, t, y


@pytest.mark.parametrize("seed", range(3))
def test_oracle_matches_per_pixel_loop(seed):
    s, t, y = _case(seed)
    assert math.isclose(unce(s, y, 3).item(), _loop_unce(s, y, 3), rel_tol=1e-12)
    for alpha in (1.0, 0.5):
        assert math.isclose(unkd(s, t, 3, alpha).item(), _loop_unkd(s, t, 3, alpha), rel_tol=1e-12)


def test_oracle_old_labels_count_as_background():
    s, _, y = _case(5)
    old = y.clone()
    old[(old >= 0) & (old < 3)] = 1                  # any old label: the same loss
    assert math.isclose(unce(s, y, 3).item(), unce(s, old, 3).item(), rel_tol=1e-13)
    # C_old = C - 1 with every label new except the background: a confident new-class pixel labelled background stays
    # finite
    x = torch.tensor([[-1e4, -1e4, 50.0]], dtype=torch.float64).view(1, 3, 1, 1)
    v = unce(x, torch.zeros((1, 1, 1), dtype=torch.int64), 2).item()
    assert math.isfinite(v) and v > 0


def test_oracle_all_ignored_gives_zero():
    s, _, y = _case(1)
    y.fill_(255)
    assert unce(s, y, 3).item() == 0.0
    assert float(unce_grad(s, y, 3).abs().max()) == 0.0


@pytest.mark.parametrize("at", ["output", "logits"])
@pytest.mark.parametrize("alpha", [1.0, 0.5])
@pytest.mark.parametrize("zoom", [1, 2, 8])
def test_oracle_gradients_equal_autograd(zoom, alpha, at):
    g = torch.Generator().manual_seed(zoom)
    n, h, w, c, c_old = 2, 4, 5, 7, 4
    s = torch.randn((n, h, w, c), generator=g) * 3
    t = torch.randn((n, h, w, c_old), generator=g) * 3
    y = torch.randint(0, c, (n, zoom * (h - 1) + 1, zoom * (w - 1) + 1), generator=g)
    y[:, ::3, ::2] = 255
    sd = s.double().requires_grad_(True)
    main, _, _ = incremental_loss(sd, t, y, zoom, c_old, alpha, kd_weight=0.7, ce_weight=1.3, at=at)
    (g_a,) = torch.autograd.grad(main, sd)
    kz = zoom if at == "output" else 1
    x = upsampled(sd, zoom)
    (g_ce,) = torch.autograd.grad(x, sd, unce_grad(x.detach(), y, c_old) * 1.3)
    xk = upsampled(sd, kz)
    (g_kd,) = torch.autograd.grad(xk, sd, unkd_grad(xk.detach(), upsampled(t, kz), c_old, alpha) * 0.7)
    assert float((g_ce + g_kd - g_a).abs().max()) <= 1e-12 * float(g_a.abs().max())


# ------------------------------------------------------------------------------------------------ IncrementalLoss
@pytest.fixture(scope="module")
def nets():
    teacher = util.build_pspnet(50, 5, seed=1).eval()
    student = expand_classifier(copy.deepcopy(teacher).train(), 3)
    return student, teacher


def test_incremental_loss_validation(nets):
    _, teacher = nets
    d = IncrementalLoss(teacher)
    assert (d.kd_weight, d.alpha, d.ce_weight, d.ignore_index, d.at, d.c_old) == (10.0, 1.0, 1.0, 255, "output", 5)
    assert d.teacher is teacher and "kd_weight=10" in repr(d)
    d = IncrementalLoss(teacher, kd_weight=0, alpha=0.5, ce_weight=2, ignore_index=-1, at="logits")
    assert (d.kd_weight, d.alpha, d.ce_weight, d.ignore_index, d.at) == (0.0, 0.5, 2.0, -1, "logits")
    assert list(d.state_dict()) == [] and list(d.children()) == []
    with pytest.raises(AttributeError):
        d.teacher = teacher
    for kw in ({"ignore_index": 255.0}, {"alpha": "1"}, {"kd_weight": True}, {"ce_weight": None}, {"at": 1}):
        with pytest.raises(TypeError):
            IncrementalLoss(teacher, **kw)
    for kw in ({"alpha": 0.0}, {"alpha": -1.0}, {"alpha": float("nan")}, {"alpha": float("inf")},
               {"kd_weight": -0.1}, {"ce_weight": float("nan")}, {"at": "features"}):
        with pytest.raises(ValueError):
            IncrementalLoss(teacher, **kw)
    for bad in (nn.Conv2d(3, 3, 1), None):
        with pytest.raises(TypeError, match="PSPNet or PSANet"):
            IncrementalLoss(bad)


def test_run_teacher_checks(nets):
    student, teacher = nets
    x = torch.zeros((1, 3, 17, 17))
    crit = IncrementalLoss(teacher)
    for classes in (5, 4):                           # the teacher must have fewer classes than the student
        with pytest.raises(ValueError, match="the teacher has 5 classes, the student %d" % classes):
            crit.run_teacher(x, classes)
    # the other teacher criteria keep their exact check
    with pytest.raises(ValueError, match="the teacher has 5 classes, the student 8$"):
        DistillationLoss(teacher).run_teacher(x, 8)
    teacher.train()
    try:
        with pytest.raises(RuntimeError, match="eval mode"):
            crit.run_teacher(x, 8)
    finally:
        teacher.eval()


def test_module_forward_checks(nets):
    _, teacher = nets
    crit = IncrementalLoss(teacher)
    y = torch.zeros((1, 9, 9), dtype=torch.int64)
    with pytest.raises(ValueError, match="the student must have more"):
        crit(torch.zeros((1, 5, 9, 9)), y)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        crit(torch.zeros((1, 8, 9, 9)), y)


def test_graph_key_changes_with_each_option(nets):
    _, teacher = nets
    base = IncrementalLoss(teacher)
    k0 = graph_key(base)
    assert graph_key(IncrementalLoss(teacher)) == k0
    for kw in ({"kd_weight": 1.0}, {"alpha": 0.5}, {"ce_weight": 0.5}, {"ignore_index": 0}, {"at": "logits"}):
        assert graph_key(IncrementalLoss(teacher, **kw)) != k0, kw
    other = util.build_pspnet(50, 5, seed=2).eval()
    assert graph_key(IncrementalLoss(other)) != k0


# ------------------------------------------------------------------------------------------------ entry points
def test_entry_points_reject_bad_arguments():
    lib = _lib.load()
    # semseg_upsample_ce_unbiased_fwd(logits, pitch, N, h, w, C, C_old, target, Ho, Wo, zoom, ignore_index, ws, loss,
    #                                 argmax, lse, lse_old, stream)
    fwd = lambda c=8, c_old=5, zoom=8, wo=9, lse_old=P: lib.semseg_upsample_ce_unbiased_fwd(  # noqa: E731
        P, c, 1, 2, 2, c, c_old, P, 9, wo, zoom, 255, P, P, P, P, lse_old, None)
    assert fwd(zoom=3) == -1 and b"zoom 3" in _err()
    assert fwd(c_old=8) == -1 and b"C_old = 8" in _err()
    assert fwd(c_old=1) == -1 and b"C_old = 1" in _err()
    assert fwd(c=257, c_old=5) == -1 and b"bad sizes" in _err()
    assert fwd(wo=10) == -1 and b"Ho=8(h-1)+1" in _err()
    assert fwd(lse_old=None) == -1 and b"null output" in _err()
    bwd = lambda c_old=5, lse_old=P: lib.semseg_upsample_ce_unbiased_bwd(  # noqa: E731
        P, 8, 1, 2, 2, 8, c_old, P, 9, 9, 8, 255, P, lse_old, P, P, P, P, None)
    assert bwd(c_old=9) == -1 and b"C_old = 9" in _err()
    assert bwd(lse_old=None) == -1 and b"null pointer" in _err()
    # the 12-byte staged rows: Wo <= 229376 / (12 zoom)
    w = 300                                          # Wo = 2393
    assert lib.semseg_upsample_ce_unbiased_bwd(P, 8, 1, 2, w, 8, 5, P, 9, 8 * (w - 1) + 1, 8, 255, P, P, P, P, P, P,
                                               None) == -1
    assert b"too large for the staged rows (at most 2389 at zoom 8)" in _err()
    # semseg_upsample_unkd_fwd(s, pitch_s, t, pitch_t, N, h, w, C, C_old, Ho, Wo, zoom, alpha, ws, loss, lse, stream)
    kd = lambda pt=5, c_old=5, alpha=1.0, zoom=8, lse=P: lib.semseg_upsample_unkd_fwd(  # noqa: E731
        P, 8, P, pt, 1, 2, 2, 8, c_old, 9, 9, zoom, alpha, P, P, lse, None)
    assert kd(pt=4) == -1 and b"pitch 8 / 4 below" in _err()
    assert kd(c_old=8, pt=8) == -1 and b"C_old = 8" in _err()
    assert kd(alpha=0.0) == -1 and b"alpha 0" in _err()
    assert kd(alpha=float("nan")) == -1 and b"alpha" in _err()
    assert kd(zoom=5) == -1 and b"zoom 5" in _err()
    assert kd(lse=None) == -1 and b"null output" in _err()
    assert lib.semseg_upsample_unkd_bwd(P, 8, P, 5, 1, 2, 2, 8, 5, 9, 9, 8, 1.0, -1.0, P, P, P, P, None) == -1
    assert b"kd_weight -1" in _err()
    assert lib.semseg_upsample_unkd_bwd(P, 8, P, 5, 1, 2, 2, 8, 5, 9, 9, 8, 1.0, 1.0, P, None, P, P, None) == -1
    assert b"null pointer" in _err()
    # workspace sizes: the zoom forward's / backward's, -1 for a bad zoom or size
    assert lib.semseg_upsample_ce_unbiased_workspace_floats(2, 65, 65, 8) == \
        lib.semseg_upsample_ce_zoom_workspace_floats(2, 65, 65, 8)
    assert lib.semseg_upsample_ce_unbiased_bwd_workspace_floats(2, 65, 9, 21, 8) == 2 * 2 * 9 * 9 * 21
    assert lib.semseg_upsample_unkd_workspace_floats(2, 65, 65, 8) == lib.semseg_upsample_kd_workspace_floats(2, 65, 65, 8)
    assert lib.semseg_upsample_unkd_bwd_workspace_floats(2, 65, 9, 21, 8) == 2 * 2 * 9 * 9 * 21
    for fn in (lib.semseg_upsample_ce_unbiased_workspace_floats, lib.semseg_upsample_unkd_workspace_floats):
        assert fn(2, 65, 65, 3) == -1
    assert lib.semseg_upsample_unkd_workspace_floats(0, 65, 65, 8) == -1
    assert lib.semseg_upsample_unkd_bwd_workspace_floats(2, 65, 9, 0, 8) == -1


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_fused_tail_decisions(zoom, nets):
    _, teacher = nets
    crit = IncrementalLoss(teacher)
    x_size = torch.Size((2, 3, 65, 81))                     # -> 9 x 11 logits
    y = torch.zeros((2, zoom * 8 + 1, zoom * 10 + 1), dtype=torch.int64)
    assert SF.fused_tail_supported(crit, None, y, zoom, x_size)
    assert SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 8)), y, zoom)
    assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257)), y, zoom)
    assert not SF.fused_tail_supported(crit, None, y.transpose(1, 2).contiguous(), zoom, x_size)

    class Sub(IncrementalLoss):
        pass
    assert not SF.fused_tail_supported(Sub(teacher), None, y, zoom, x_size)
    # the width limit of the 12-byte staged rows (Dice's): 2389 columns at zoom 8
    w = 229376 // (12 * zoom)
    x_ok = torch.Size((1, 3, 9, 8 * ((w - 1) // zoom) + 1))
    y_ok = torch.zeros((1, zoom + 1, zoom * ((w - 1) // zoom) + 1), dtype=torch.int64)
    assert SF.fused_tail_supported(crit, None, y_ok, zoom, x_ok)
    n_over = (w - 1) // zoom + 1
    x_big = torch.Size((1, 3, 9, 8 * n_over + 1))
    y_big = torch.zeros((1, zoom + 1, zoom * n_over + 1), dtype=torch.int64)
    assert not SF.fused_tail_supported(crit, None, y_big, zoom, x_big)


# ------------------------------------------------------------------------------------------------ expand_classifier
def test_expand_state_dict_matches_fresh_network():
    for arch in ("psp", "psa"):
        build = util.build_pspnet if arch == "psp" else util.build_psanet
        old = build(50, 5, seed=3)
        net = expand_classifier(copy.deepcopy(old), 4)
        fresh = build(50, 9, seed=4)
        sd, ref = net.state_dict(), fresh.state_dict()
        assert list(sd) == list(ref)
        assert all(sd[k].shape == ref[k].shape for k in ref)
        for head in ("cls", "aux"):
            a, b = getattr(old, head)[4], getattr(net, head)[4]
            assert b.out_channels == 9 and b.weight.requires_grad and b.bias.requires_grad
            assert torch.equal(b.weight[:5], a.weight)                  # old rows bit for bit
            assert torch.equal(b.bias[1:5], a.bias[1:])
            for j in range(5, 9):
                assert torch.equal(b.weight[j], a.weight[0])            # the background row, imprinted
            b0 = a.bias[0] - math.log(5)
            assert torch.allclose(b.bias[0], b0, rtol=0, atol=0) and torch.equal(b.bias[5:], b.bias[0].expand(4))


def test_expand_rejects():
    net = util.build_pspnet(50, 250, seed=0)
    with pytest.raises(TypeError, match="before wrapping"):
        expand_classifier(nn.DataParallel(net), 2)
    with pytest.raises(TypeError, match="PSPNet or PSANet"):
        expand_classifier(nn.Conv2d(3, 3, 1), 2)
    for bad in (0, -1):
        with pytest.raises(ValueError, match="new_classes"):
            expand_classifier(net, bad)
    for bad in (1.0, True, "2"):
        with pytest.raises(TypeError, match="new_classes"):
            expand_classifier(net, bad)
    with pytest.raises(ValueError, match="257 classes"):
        expand_classifier(net, 7)
    assert expand_classifier(net, 6).cls[4].out_channels == 256


def test_two_expansions_compose():
    old = util.build_pspnet(50, 4, seed=6)
    once = expand_classifier(copy.deepcopy(old), 2)
    twice = expand_classifier(copy.deepcopy(once), 3)
    w, b = twice.cls[4].weight, twice.cls[4].bias
    assert w.shape[0] == 9
    assert torch.equal(w[:6], once.cls[4].weight) and torch.equal(b[1:6], once.cls[4].bias[1:])
    assert all(torch.equal(w[j], old.cls[4].weight[0]) for j in range(4, 9))
    assert math.isclose(b[0].item(), old.cls[4].bias[0].item() - math.log(3) - math.log(4), rel_tol=0, abs_tol=1e-6)


def test_expanded_network_keeps_old_probabilities():
    """Through the fp32 oracle: the grown network's old-class probabilities (classes 1..C_old-1) equal the old
    network's, and its background + new mass equals the old background probability, to fp32 rounding."""
    torch.manual_seed(0)
    old = util.build_pspnet(50, 6, seed=7).eval()
    with torch.no_grad():             # a larger background bias spread than the default init, so that it matters
        old.cls[4].bias.copy_(torch.randn(6) * 2)
    new = expand_classifier(copy.deepcopy(old), 3)
    x = torch.randn((1, 3, 33, 33), generator=torch.Generator().manual_seed(1))
    po, _ = util.oracle_from(old, "psp", layers=50, classes=6)
    pn, _ = util.oracle_from(new, "psp", layers=50, classes=9)
    po.eval()
    pn.eval()
    with torch.no_grad():
        qo = torch.softmax(po.forward(x).double(), 1)
        qn = torch.softmax(pn.forward(x).double(), 1)
    assert float((qn[:, 1:6] - qo[:, 1:]).abs().max()) <= 1e-6
    mass = qn[:, 0] + qn[:, 6:].sum(1)
    assert float((mass - qo[:, 0]).abs().max()) <= 1e-6
    assert float((qn[:, 6:] - qn[:, :1]).abs().max()) <= 1e-6      # split evenly
    assert np.isfinite(qn.numpy()).all()
