"""GPU tier: mean-teacher training — optim.ModelEMA's one-launch update (csrc/sgd.cu ema_multi_kernel), an EMA teacher
in the graphed training step, and the confidence-masked pseudo-label loss on the fused tail (csrc/tail.cu
upsample_pl_*, losses.PseudoLabelLoss).

  * the EMA kernel: bit-equal to torch._foreach_lerp_ over a PSPNet50's tensors, integer buffers copied, odd lengths and
    misaligned tails, decay 0 / 1 exact, reruns bit-identical, and an updated shadow evaluates like a fresh network
    loaded with its state_dict (no stale operand slab);
  * a PSPNet50 student with DistillationLoss / PseudoLabelLoss on ema.module, 10 FusedSGD steps + ema.update: captured
    once, then replayed, with the losses, parameters and shadow bits of the same steps run eagerly; a frozen teacher is
    still captured anew after a weight edit;
  * the pseudo-label kernels against the float64 oracle of tests/pl_oracle.py (zoom 1-8, 19-256 classes, padded and
    unequal pitches, thresholds 0 / 0.5 / 0.95 / > 1, weights 0 / 1, labelled / unlabelled / mixed batches, out-of-range
    targets, teacher = student), reruns bit-identical, lse / pred the plain tail's bits;
  * PSPNet50 / PSANet50 students with an EMA teacher against the same loss in PyTorch on the eager ATen route, no ATen
    tail kernel in a graphed step, the teacher without gradient, and the module path."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.kd_oracle import upsampled
from tests.pl_oracle import effective, pl_grad, pl_loss
from tests.test_zoom_gpu import _batch, _build, _logits, _target

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ EMA kernel
def _tensors(m):
    return list(m.parameters()) + list(m.buffers())


def _perturbed(model, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for t in _tensors(model):
            if t.dtype == torch.float32:
                t.add_(torch.randn(t.shape, device="cuda", generator=g) * 0.05)
            else:
                t.add_(seed)
    return model


@pytest.mark.parametrize("decay", [0.999, 0.9, 0.3, 0.0, 1.0])
def test_ema_update_bit_equal_to_foreach_lerp(decay):
    from semseg_b200.optim import ModelEMA
    student = _build("psp", 8).cuda().train()
    ema = ModelEMA(student, decay=decay)
    _perturbed(student, 3)
    shadow = ema.module
    ref_f = [t.detach().clone() for t in _tensors(shadow) if t.dtype == torch.float32]
    src_f = [t.detach() for t in _tensors(student) if t.dtype == torch.float32]
    torch._foreach_lerp_(ref_f, src_f, 1 - decay)
    ema.update(student)
    got_f = [t for t in _tensors(shadow) if t.dtype == torch.float32]
    assert all(torch.equal(a, b) for a, b in zip(got_f, ref_f))
    if decay == 0.0:
        assert all(torch.equal(a, b) for a, b in zip(got_f, src_f))
    ints = [(a, b) for a, b in zip(_tensors(shadow), _tensors(student)) if a.dtype == torch.int64]
    assert ints and all(torch.equal(a, b) for a, b in ints)


def test_ema_decay_one_is_a_no_op_and_reruns_are_bit_identical():
    from semseg_b200.optim import ModelEMA
    student = _build("psp", 8).cuda().train()
    a, b = ModelEMA(student, decay=0.99), ModelEMA(student, decay=0.99)
    _perturbed(student, 5)
    before = [t.clone() for t in _tensors(a.module)]
    a.decay = 1.0
    a.update(student)
    for x, y, w in zip(_tensors(a.module), before, _tensors(student)):
        assert torch.equal(x, y if x.dtype == torch.float32 else w)      # integer buffers are copied at any decay
    a.decay = 0.99
    a.update(student)
    b.update(student)
    assert all(torch.equal(x, y) for x, y in zip(_tensors(a.module), _tensors(b.module)))


@pytest.mark.parametrize("decay", [0.0, 0.25, 0.5, 0.75, 0.999])
@pytest.mark.parametrize("offset", [0, 1, 3])
def test_ema_kernel_odd_lengths_and_misaligned_tails(offset, decay):
    """Raw item tables: lengths 1 .. 2 chunks + 5 at element offsets that break the 16-byte alignment (scalar path) or
    keep it, int64 items between them. Both branches of torch.lerp's form: weight 1 - decay below 0.5 (decay 0.75,
    0.999) and from 0.5 up (decay 0.5, 0.25, and 0: the first two updates of a min(decay, 1 - 1/(t+1)) ramp)."""
    from semseg_b200 import ops
    from semseg_b200.optim import ema_table
    g = torch.Generator(device="cuda").manual_seed(offset)
    lengths = [1, 3, 4, 5, 4095, 4096, 4097, 8197, 13]
    pairs, refs = [], []
    for k, n in enumerate(lengths):
        if k % 3 == 2:
            e = torch.randint(0, 1000, (n + offset,), device="cuda", generator=g)[offset:]
            w = torch.randint(0, 1000, (n + offset,), device="cuda", generator=g)[offset:]
            refs.append(w.clone())
        else:
            e = torch.randn((n + offset,), device="cuda", generator=g)[offset:]
            w = torch.randn((n + offset,), device="cuda", generator=g)[offset:]
            r = e.clone()
            torch._foreach_lerp_([r], [w], 1 - decay)
            refs.append(r)
        pairs.append((e, w))
    items, n_items, chunks = ema_table(pairs)
    ops.ema_multi(items, n_items, chunks, decay)
    for (e, _), r in zip(pairs, refs):
        assert torch.equal(e, r)


def test_ema_updated_shadow_has_no_stale_slabs():
    """After update, an eval forward of ema.module equals a fresh network loaded with the shadow's state_dict, bit for
    bit: the update's version bump re-packs the operand slabs the previous forward cached."""
    from semseg_b200.optim import ModelEMA
    student = _build("psp", 8).cuda().train()
    ema = ModelEMA(student, decay=0.5)
    x, _ = _batch(8)
    with torch.no_grad():
        ema.module(x)                               # caches the shadow's slabs
        _perturbed(student, 7)
        ema.update(student)
        out = ema.module(x)
        fresh = _build("psp", 8, seed=9).cuda().eval()
        fresh.load_state_dict(ema.module.state_dict())
        ref = fresh(x)
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------ graphed EMA teacher
def _ema_run(base, kind, n_steps, batches, graph, monkeypatch):
    from semseg_b200.losses import DistillationLoss, PseudoLabelLoss
    from semseg_b200.optim import FusedSGD, ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    model = copy.deepcopy(base)
    ema = ModelEMA(model, decay=0.9)
    if kind == "kd":
        model.criterion = DistillationLoss(ema.module, temperature=2.0, kd_weight=0.5)
    else:
        model.criterion = PseudoLabelLoss(ema.module, threshold=0.06, pl_weight=1.0, ce_weight=1.0)
    opt = FusedSGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    losses = []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
        ema.update(model)                 # after the optimizer, on the same stream
        losses.append((ml.item(), al.item()))
    return model, ema, losses


@pytest.mark.parametrize("kind", ["kd", "pl"])
def test_graphed_ema_teacher_captured_once_and_bit_identical_to_eager(kind, monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    batches = []
    for s in (1, 2, 3):
        x, y = _batch(8, seed=s)
        y[0] = 255                        # image 0 unlabelled: the pseudo-label term trains on it
        batches.append((x, y))
    me, ee, le = _ema_run(base, kind, 10, batches, False, monkeypatch)
    mg, eg, lg = _ema_run(base, kind, 10, batches, True, monkeypatch)
    assert le == lg, (le, lg)
    assert len(mg.__dict__["_sb_graph_steps"]) == 1
    assert graphs.launches_per_step(mg) > 100
    assert graphs.launches_per_step(me) == 0
    for a, b in zip(_tensors(me), _tensors(mg)):
        assert torch.equal(a, b)
    for a, b in zip(_tensors(ee.module), _tensors(eg.module)):
        assert torch.equal(a, b)
    assert len(set(le)) > 5               # the shadow and the losses move from step to step


def test_frozen_teacher_still_recaptured_after_weight_edit(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import PseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    teacher = _build("psp", 8, seed=4).cuda().eval()
    model = _build("psp", 8).cuda().train()
    model.criterion = PseudoLabelLoss(teacher, threshold=0.0)
    x, y = _batch(8)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for _ in range(graphs.WARMUP_CALLS + 2):
        _, ml, al = model(x, y)
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
    assert sum(1 for s in model._sb_graph_steps.values() if s.fwd is not None) == 1
    with torch.no_grad():
        teacher.cls[4].weight.mul_(1.5)
    for _ in range(graphs.WARMUP_CALLS + 2):
        _, ml, al = model(x, y)
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
    assert sum(1 for s in model._sb_graph_steps.values() if s.fwd is not None) == 2


# ------------------------------------------------------------------------------------------------ kernel vs oracle
ZOOMS = [1, 2, 4, 8]
# (n, h, w, C, student pitch, teacher pitch)
SHAPES = [(2, 9, 13, 150, 152, 160), (1, 17, 11, 19, 19, 24), (1, 6, 140, 21, 24, 21), (1, 7, 10, 256, 256, 264)]
SHAPE_IDS = ["9x13-150-p152-p160", "17x11-19-p24", "6x140-21-p24", "7x10-256-p264"]
# (threshold, pl_weight, ce_weight)
OPTIONS = [(0.0, 1.0, 1.0), (0.5, 1.0, 1.0), (0.95, 1.0, 0.0), (1.5, 1.0, 1.0), (0.5, 0.0, 1.0), (0.05, 1.0, 1.0)]
OPTION_IDS = ["thr0", "thr0.5", "thr0.95-ce0", "thr1.5", "thr0.5-pl0", "thr0.05"]


def _run(s, t, target, zoom, threshold, pl_weight, ce_weight, grad=0.7):
    from semseg_b200 import functional as SF
    sg = s.detach().requires_grad_(True)
    out = SF._UpsampleCEPL.apply(sg, t, target, 255, zoom, threshold, pl_weight, ce_weight)
    saved = out[0].grad_fn.saved_tensors              # (logits, effective target, lse, weight, loss_info)
    eff, lse, wt = saved[1], saved[2], saved[3]
    (dl,) = torch.autograd.grad(out[0] * grad, sg)
    return out[0].detach(), out[1], dl, eff, wt, lse


def _ambiguous(t, zoom, threshold):
    """Pixels whose teacher top-2 margin or conf - threshold lies within fp32 interpolation error (float64 oracle)."""
    x = upsampled(t, zoom)
    top2 = x.topk(2, dim=1).values
    scale = float(x.abs().max())
    near_tie = (top2[:, 0] - top2[:, 1]) <= 1e-5 * scale
    conf = 1.0 / torch.exp(x - top2[:, :1]).sum(1)
    return near_tie | ((conf - threshold).abs() <= 1e-5), top2


def _check(s, t, target, zoom, threshold, pl_weight, ce_weight, label=""):
    loss, amax, dl, eff, wt, _ = _run(s, t, target, zoom, threshold, pl_weight, ce_weight)
    eff_o, wt_o, _ = effective(t.cpu(), target.cpu(), zoom, threshold, pl_weight, ce_weight)
    eff_o, wt_o = eff_o.cuda(), wt_o.cuda()
    amb, _ = _ambiguous(t, zoom, threshold)
    unl = target == 255
    amb = amb & unl
    # away from fp32 ties the kernel's pseudo-labels and mask are the definition's; at the ambiguous pixels the oracle
    # takes the kernel's, which must still be a near-top class or "not confident"
    assert torch.equal(eff[~amb], eff_o[~amb]), label
    if bool(amb.any()):
        x = upsampled(t, zoom)
        k = eff[amb]
        top = x.permute(0, 2, 3, 1)[amb]
        picked = top.gather(1, k.clamp(min=0).unsqueeze(1)).squeeze(1)
        assert bool(((k < 0) | (picked >= top.max(1).values - 1e-5 * float(x.abs().max()))).all()), label
    eff_use = torch.where(amb, eff, eff_o)
    wt_use = torch.where(amb, wt.double(), wt_o)
    assert float((wt.double() - wt_use).abs().max()) <= 1e-7 * max(float(wt_use.abs().max()), 1e-30), label
    sr = s.detach().double()
    ref = pl_loss(sr, eff_use, wt_use, zoom)
    g_ref = pl_grad(s, eff_use, wt_use, zoom) * 0.7
    e_loss = abs(loss.item() - ref.item()) / max(abs(ref.item()), 1e-30)
    scale = float(g_ref.abs().max())
    e_dl = float((dl.double() - g_ref).abs().max()) / scale if scale > 0 else float(dl.abs().max())
    print("pl-err %s zoom=%d C=%d thr=%g pl=%g ce=%g amb=%d loss=%.3g dl=%.3g" % (
        label, zoom, s.shape[-1], threshold, pl_weight, ce_weight, int(amb.sum()), e_loss, e_dl))
    if ref.item() == 0.0:
        assert loss.item() == 0.0 and float(dl.abs().max()) == 0.0
    else:
        assert e_loss <= 1e-6, label            # measured on an H100: <= 8.9e-8
        assert e_dl <= 5e-6, label              # measured: <= 1.2e-6 of max |dlogits|
    return loss, amax, dl


@pytest.mark.parametrize("opts", OPTIONS, ids=OPTION_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_pl_kernel_vs_oracle(zoom, shape, opts):
    n, h, w, c, ps, pt = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    s = _logits(n, h, w, c, ps, seed=zoom + 40)
    t = _logits(n, h, w, c, pt, seed=zoom + 50) * 2.0
    base = _target(n, ho, wo, c, seed=zoom + 40)         # ~5 % ignored, a few out-of-range classes
    mixed = base.clone()
    mixed[0, : ho // 2] = 255                             # half of image 0 unlabelled
    unlabelled = torch.full_like(base, 255)
    unlabelled[..., 0] = c + 3                            # out of range: in neither set
    labelled = base.clone()
    labelled[labelled == 255] = 0
    for name, target in (("mixed", mixed), ("unlabelled", unlabelled), ("labelled", labelled)):
        _check(s, t, target, zoom, *opts, label=name)


@pytest.mark.parametrize("zoom", ZOOMS)
def test_pl_teacher_equal_to_student(zoom):
    n, h, w, c = 2, 9, 13, 21
    s = _logits(n, h, w, c, 24, seed=zoom)
    t = s.detach().clone().contiguous()
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom)
    target[1] = 255
    loss, amax, dl = _check(s, t, target, zoom, 0.0, 1.0, 1.0, label="t=s")
    _, _, _, eff, _, _ = _run(s, t, target, zoom, 0.0, 1.0, 1.0)
    unl = target == 255
    assert torch.equal(eff[unl], amax[unl])               # the pseudo-label is the student's own argmax


@pytest.mark.parametrize("zoom", [1, 8])
def test_pl_deterministic_and_lse_pred_are_plain(zoom):
    from semseg_b200 import ops
    n, h, w, c = 2, 17, 23, 150
    s = _logits(n, h, w, c, 152, seed=zoom)
    t = _logits(n, h, w, c, 150, seed=zoom + 1) * 3
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom)
    target[0, :20] = 255
    a = _run(s, t, target, zoom, 0.5, 1.0, 1.0)
    b = _run(s, t, target, zoom, 0.5, 1.0, 1.0)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    _, amax, lse = ops.upsample_ce_fwd(s, target, 255, zoom=zoom)
    assert torch.equal(a[1], amax)
    assert torch.equal(a[5], lse)


# ------------------------------------------------------------------------------------------------ networks
def _torch_pl_class():
    from semseg_b200.losses import PseudoLabelLoss

    class _TorchPL(PseudoLabelLoss):
        """PseudoLabelLoss written in fp32 PyTorch under another type: the network keeps the eager route (interpolate
        both maps -> criterion)."""

        def forward(self, logits, target, teacher_logits=None):
            c = logits.shape[1]
            lab = (target != self.ignore_index) & (target >= 0) & (target < c)
            ce = F.cross_entropy(logits, torch.where(lab, target, torch.full_like(target, -100)), ignore_index=-100) \
                if bool(lab.any()) else logits.sum() * 0
            if teacher_logits is None:
                return ce
            unl = target == self.ignore_index
            q = torch.softmax(teacher_logits, dim=1)
            conf, yhat = q.max(1)
            keep = unl & (conf >= self.threshold)
            nll = F.cross_entropy(logits, torch.where(keep, yhat, torch.full_like(yhat, -100)), ignore_index=-100,
                                  reduction="sum")
            pl = nll / int(unl.sum()) if bool(unl.any()) else logits.sum() * 0
            return self.ce_weight * ce + self.pl_weight * pl

    return _TorchPL


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_pl_matches_aten(arch, zoom, mode, monkeypatch):
    """One step of a PSPNet50 / PSANet50 student with an EMA teacher on the native pseudo-label tail against the same
    loss in PyTorch on the eager ATen route (the teacher's logits a detached constant in both), x.grad included; the
    shadow gets no gradient and is not modified by the step."""
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import PseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    ema = ModelEMA(native, decay=0.5)
    _perturbed(native, 2)
    ema.update(native)                           # a shadow that differs from the student
    aten = copy.deepcopy(native)
    native.criterion = PseudoLabelLoss(ema.module, threshold=0.0, pl_weight=0.7, ce_weight=1.0)
    aten.criterion = _torch_pl_class()(ema.module, threshold=0.0, pl_weight=0.7, ce_weight=1.0)
    x, y = _batch(zoom)
    y[1] = 255                                   # an unlabelled image in the batch
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    before = [t.clone() for t in _tensors(ema.module)]
    with precision.mode(mode):
        xn = x.clone().requires_grad_(True)
        pred, main, aux = native(xn, y)
        (main + 0.4 * aux).backward()
        xa = x.clone().requires_grad_(True)
        pred_r, main_r, aux_r = aten(xa, y)
        (main_r + 0.4 * aux_r).backward()
    print("pl-net %s zoom=%d %s main=%.3g aux=%.3g" % (arch, zoom, mode, abs(main.item() - main_r.item()) /
                                                       abs(main_r.item()), abs(aux.item() - aux_r.item()) /
                                                       abs(aux_r.item())))
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01
    if mode == "bf16x3":
        bad = []
        for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
            assert (pn.grad is None) == (pa.grad is None), k
            if pn.grad is not None:
                err = util.rel_l2(pn.grad, pa.grad)
                if err > 3e-4:
                    bad.append((k, err))
        assert not bad, bad
        assert util.rel_l2(xn.grad, xa.grad) <= 1e-4
    assert all(p.grad is None for p in ema.module.parameters())
    assert all(torch.equal(a, b) for a, b in zip(_tensors(ema.module), before))


def test_graphed_pl_step_launches_no_aten_tail(monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import PseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    model = _build("psp", 8).cuda().train()
    ema = ModelEMA(model)
    model.criterion = PseudoLabelLoss(ema.module, threshold=0.0)
    x, y = _batch(8)
    y[0] = 255
    for _ in range(graphs.WARMUP_CALLS + 2):
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        ema.update(model)
    torch.cuda.synchronize()
    assert graphs.launches_per_step(model) > 100
    for p in model.parameters():
        p.grad = None
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        ema.update(model)
        torch.cuda.synchronize()
    bad = sorted({e.name for e in prof.events() if any(k in e.name for k in ("upsample_bilinear2d", "_softmax",
                                                                             "nll_loss", "lerp"))})
    assert not bad, bad


def test_pl_module_path_matches_oracle():
    """validate()'s call: NCHW logits at the target size; without teacher logits the mean CE over the labelled pixels,
    with them the pseudo-label loss at that size."""
    from semseg_b200.losses import PseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    model = _build("psp", 8).cuda().eval()
    ema = ModelEMA(model)
    x, y = _batch(8)
    y[0, :30] = 255
    with torch.no_grad():
        out = model(x)
        t_out = ema.module(x)
    crit = PseudoLabelLoss(ema.module, threshold=0.0, pl_weight=0.5, ce_weight=1.0)
    ref_ce = F.cross_entropy(out.double(), y, ignore_index=255)
    assert abs(crit(out, y).item() - ref_ce.item()) <= 1e-6 * abs(ref_ce.item())
    t_nhwc = t_out.permute(0, 2, 3, 1).contiguous()
    eff, wt, _ = effective(t_nhwc.cpu(), y.cpu(), 1, 0.0, 0.5, 1.0)
    ref = pl_loss(out.permute(0, 2, 3, 1).double(), eff.cuda(), wt.cuda(), 1)
    assert abs(crit(out, y, t_out).item() - ref.item()) <= 1e-6 * abs(ref.item())
