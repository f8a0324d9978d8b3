"""GPU tier: class-incremental training on the fused tail (csrc/tail.cu unbiased cross-entropy and unbiased
distillation kernels through semseg_b200/functional.py, losses.IncrementalLoss and incremental.expand_classifier).

  * kernel vs the float64 oracle of tests/incremental_oracle.py at zoom 1, 2, 4, 8 with (C_old, C) = (2, 3),
    (100, 150), (255, 256), padded and unequal pitches, both `at`, alpha 1 / 0.5, kd_weight 0 / > 0, ignored and
    out-of-range targets: the loss, dlogits and the argmax;
  * reruns are bit-identical, the argmax is the plain tail's;
  * graphed PSPNet and PSANet steps equal eager ones (losses, pred, parameters and gradients) at every zoom, and the
    teacher is left untouched without a gradient;
  * after expand_classifier the UNKD gradient into cls[4] vanishes at alpha = 1;
  * the network's loss is the oracle's on its own logits, and the module path.

Tolerances: the loss within 1e-5 of the oracle (relative, or absolute below 1) and dlogits within 2e-5 of the larger of
the largest oracle entry and one valid pixel's unit gradient (grad * ce_weight / n_valid). The second scale is there
because a pixel labelled with an old class has the gradient p_c - exp(s_c - lse_old) on the old classes: two fp32 terms
that cancel when the new classes hold little of its mass, which is what a batch of almost only old labels (C_old = 255
of 256) makes the largest entry. The kernels' fp32 sums and ex2.approx / lg2 rounding stay well inside both."""
import copy

import pytest
import torch

from tests.incremental_oracle import incremental_loss, unce, unkd
from tests.kd_oracle import upsampled
from tests.test_weighted_ce_gpu import _n_graphs
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
# (n, h, w, C_old, C, student pitch, teacher pitch)
SHAPES = [(2, 9, 13, 2, 3, 3, 4), (1, 7, 70, 100, 150, 152, 100), (1, 6, 11, 255, 256, 256, 264)]
SHAPE_IDS = ["2-3", "100-150-p152", "255-256-p264"]
# (at, alpha, kd_weight, ce_weight)
OPTIONS = [("output", 1.0, 10.0, 1.0), ("output", 0.5, 1.0, 0.5), ("logits", 1.0, 2.0, 1.0), ("logits", 0.5, 0.0, 1.0),
           ("output", 1.0, 0.0, 1.0)]


def _incremental_target(n, ho, wo, c, seed):
    t = _target(n, ho, wo, c, seed)                  # ~5 % ignored, a few out of range
    g = torch.Generator(device="cuda").manual_seed(seed + 3)
    t[torch.rand((n, ho, wo), device="cuda", generator=g) < 0.3] = 0     # plenty of background labels
    return t


def _run(s, t, target, zoom, c_old, at, alpha, kd_weight, ce_weight, grad=0.7):
    from semseg_b200 import functional as SF
    sg = s.detach().requires_grad_(True)
    kd_zoom = zoom if at == "output" else 1
    out = SF._UpsampleCEIncremental.apply(sg, t, target, 255, zoom, kd_zoom, c_old, alpha, kd_weight, ce_weight)
    (dl,) = torch.autograd.grad(out[0] * grad, sg)
    return out[0].detach(), out[1], dl


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1.0)


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_incremental_kernels_vs_oracle(zoom, shape):
    from semseg_b200 import ops
    n, h, w, c_old, c, ps, pt = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    s = _logits(n, h, w, c, ps, seed=zoom + 30)
    t = _logits(n, h, w, c_old, pt, seed=zoom + 40)
    target = _incremental_target(n, ho, wo, c, seed=zoom)
    for at, alpha, kd_weight, ce_weight in OPTIONS:
        loss, amax, dl = _run(s, t, target, zoom, c_old, at, alpha, kd_weight, ce_weight)
        sr = s.detach().clone().requires_grad_(True)
        main, _, _ = incremental_loss(sr, t, target, zoom, c_old, alpha, kd_weight, ce_weight, at=at)
        (dl_o,) = torch.autograd.grad(main * 0.7, sr)
        e_loss = _rel(loss.item(), main.item())
        n_valid = int(((target != 255) & (target >= 0) & (target < c)).sum())
        scale = max(float(dl_o.abs().max()), 0.7 * ce_weight / max(n_valid, 1))
        e_dl = float((dl.double() - dl_o).abs().max()) / scale
        print("incr-err zoom=%d C=%d/%d at=%s alpha=%g kd=%g ce=%g loss=%.3g dl=%.3g" % (
            zoom, c_old, c, at, alpha, kd_weight, ce_weight, e_loss, e_dl))
        assert e_loss <= 1e-5
        assert e_dl <= 2e-5
        x = upsampled(s, zoom)
        clear = _clear_of_ties(x.float())
        assert torch.equal(amax[clear], x.argmax(1)[clear])
    # the argmax over all C classes is the plain tail's
    _, amax_plain, _ = ops.upsample_ce_fwd(s, target, 255, zoom=zoom)
    assert torch.equal(amax, amax_plain)


@pytest.mark.parametrize("zoom", [1, 8])
def test_incremental_all_ignored_and_confident_new_class(zoom):
    n, h, w, c_old, c = 1, 5, 9, 10, 15
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    s = _logits(n, h, w, c, c, seed=7)
    t = _logits(n, h, w, c_old, c_old, seed=8)
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    loss, _, dl = _run(s, t, target, zoom, c_old, "output", 1.0, 0.0, 1.0)
    assert loss.item() == 0.0 and float(dl.abs().max()) == 0.0
    # a confidently new-class pixel labelled background: a large finite loss, as the oracle's
    s2 = s.detach().clone()
    s2[..., :c_old] = -60.0
    s2[..., c_old] = 60.0
    target.fill_(0)
    loss, _, dl = _run(s2, t, target, zoom, c_old, "output", 1.0, 1.0, 1.0)
    ref = unce(upsampled(s2, zoom), target, c_old) + unkd(upsampled(s2, zoom), upsampled(t, zoom), c_old)
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(dl).all()) and loss.item() > 100.0
    assert _rel(loss.item(), ref.item()) <= 1e-5


@pytest.mark.parametrize("zoom", [1, 8])
def test_incremental_deterministic(zoom):
    n, h, w, c_old, c = 2, 17, 23, 100, 150
    s = _logits(n, h, w, c, 152, seed=zoom)
    t = _logits(n, h, w, c_old, 100, seed=zoom + 1)
    target = _incremental_target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom)
    a = _run(s, t, target, zoom, c_old, "output", 0.5, 10.0, 1.0)
    b = _run(s, t, target, zoom, c_old, "output", 0.5, 10.0, 1.0)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_unkd_gradient_vanishes_after_expansion():
    """The expanded classifier on the teacher's own features: at alpha = 1 the UNKD gradient into cls[4]'s weight and
    bias is zero to fp32 rounding (and at alpha = 0.5 it is not)."""
    from semseg_b200 import functional as SF
    from semseg_b200.incremental import expand_classifier
    teacher = _build("psp", 8, classes=21, seed=3).cuda().eval()
    with torch.no_grad():
        teacher.cls[4].bias.copy_(torch.randn(21, device="cuda"))
    student = expand_classifier(copy.deepcopy(teacher).train(), 9)
    g = torch.Generator(device="cuda").manual_seed(2)
    f = torch.relu(torch.randn((2, 9, 13, 512), device="cuda", generator=g))
    target = _incremental_target(2, 65, 97, 30, seed=2)
    t = torch.nn.functional.linear(f, teacher.cls[4].weight.view(21, 512), teacher.cls[4].bias).contiguous()
    norms = {}
    for alpha in (1.0, 0.5):
        wt = student.cls[4].weight.detach().clone().requires_grad_(True)
        bs = student.cls[4].bias.detach().clone().requires_grad_(True)
        s = torch.nn.functional.linear(f, wt.view(30, 512), bs).contiguous()
        loss, _ = SF._UpsampleCEIncremental.apply(s, t, target, 255, 8, 8, 21, alpha, 1.0, 0.0)
        gw, gb = torch.autograd.grad(loss, (wt, bs))
        norms[alpha] = (float(gw.abs().max()), float(gb.abs().max()))
    print("unkd grad after expansion: alpha=1 %s, alpha=0.5 %s" % (norms[1.0], norms[0.5]))
    assert max(norms[1.0]) <= 1e-5 * max(norms[0.5])
    assert max(norms[0.5]) > 1e-4


# ------------------------------------------------------------------------------------------------ networks
def _teacher(arch, zoom):
    return _build(arch, zoom, classes=21, seed=5).cuda().eval()


def _student(teacher, new=4, **kw):
    from semseg_b200.incremental import expand_classifier
    from semseg_b200.losses import IncrementalLoss
    m = expand_classifier(copy.deepcopy(teacher).train(), new)
    m.criterion = IncrementalLoss(teacher, **kw)
    return m


def _state(m):
    return [v.detach().clone() for v in list(m.parameters()) + list(m.buffers())], m.training


@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_graphed_incremental_steps_equal_eager(arch, zoom, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import graphs
    teacher = _teacher(arch, zoom)
    before, flag = _state(teacher)
    base = _student(teacher, kd_weight=10.0, alpha=0.5, at="output" if zoom != 2 else "logits")
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    for m in (eager, graphed):
        m.criterion = base.criterion
    batches = [_batch(zoom, classes=25, seed=s) for s in (1, 2, 3)]
    assert SF.fused_tail_supported(base.criterion, None, batches[0][1], zoom, batches[0][0].size())
    n_steps = graphs.WARMUP_CALLS + 3
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, n_steps)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, n_steps)
    assert le == lg, (le, lg)
    assert _n_graphs(graphed) == 1
    x, y = batches[0]
    outs = []
    for m in (eager, graphed):
        for p in m.parameters():
            p.grad = None
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "0" if m is eager else "1")
        pred, main, aux = m(x, y)
        (main + 0.4 * aux).backward()
        outs.append((pred, main.item(), aux.item()))
    assert torch.equal(outs[0][0], outs[1][0]) and outs[0][1:] == outs[1][1:]
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.equal(pe, pg), k
        assert (pe.grad is None) == (pg.grad is None) and (pe.grad is None or torch.equal(pe.grad, pg.grad)), k
    for (k, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), k
    after, flag_after = _state(teacher)
    assert flag_after is False and flag is False
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    assert all(p.grad is None for p in teacher.parameters())


@pytest.mark.parametrize("at", ["output", "logits"])
@pytest.mark.parametrize("zoom", [2, 8])
def test_network_loss_matches_oracle_statement(zoom, at, monkeypatch):
    """The native step's main and aux losses are the oracle's on the network's own student, aux and teacher logits."""
    from semseg_b200 import precision
    from semseg_b200.pspnet import head_forward_nhwc
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    teacher = _teacher("psp", zoom)
    model = _student(teacher, kd_weight=2.0, alpha=0.5, ce_weight=0.5, at=at)
    x, y = _batch(zoom, classes=25)
    seen = {}
    orig = model._logits_nhwc

    def spy(inp):
        out = orig(inp)
        seen["s"] = out[0].detach().clone()
        seen["aux"] = head_forward_nhwc(model.aux, out[1]).detach().clone()
        return out
    model._logits_nhwc = spy
    with precision.mode("bf16x3"):
        _, main, aux = model(x, y)
        t = model.criterion.run_teacher(x, 25)
    ref, _, _ = incremental_loss(seen["s"], t, y, zoom, 21, 0.5, 2.0, 0.5, at=at)
    assert _rel(main.item(), ref.item()) <= 1e-5
    aux_ref = unce(upsampled(seen["aux"], zoom), y, 21)
    assert _rel(aux.item(), aux_ref.item()) <= 1e-4


def test_module_path_matches_oracle():
    from semseg_b200.losses import IncrementalLoss
    teacher = _teacher("psa", 8)
    model = _student(teacher).eval()
    x, y = _batch(8, classes=25)
    with torch.no_grad():
        out = model(x)
        t_out = teacher(x)
    crit = IncrementalLoss(teacher, kd_weight=3.0, alpha=0.5, ce_weight=1.5)
    loss = crit(out, y)
    assert _rel(loss.item(), unce(out, y, 21).item()) <= 1e-6
    loss = crit(out, y, t_out)
    ref = 1.5 * unce(out, y, 21) + 3.0 * unkd(out, t_out, 21, 0.5)
    assert _rel(loss.item(), ref.item()) <= 1e-5
    with pytest.raises(ValueError, match="teacher_logits must be fp32"):
        crit(out, y, out)
