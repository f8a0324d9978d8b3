"""GPU tier: pixel-wise knowledge distillation on the fused tail (csrc/tail.cu distillation kernels through
semseg_b200/functional.py and losses.DistillationLoss).

  * kernel vs the float64 oracle of tests/kd_oracle.py at zoom 1, 2, 4, 8 with odd h != w, widths off and across the
    forward CTA, 19 / 21 / 150 / 256 classes, padded and unequal pitches, T = 0.5 / 1 / 4, kd_weight / ce_weight 0 / 1
    and ignored / out-of-range targets: the loss and dlogits;
  * s = t gives KL and gradient 0; saturated logits at T = 0.5 stay finite; reruns are bit-identical; lse / pred are
    the plain tail's bits;
  * the kernels that need the > 48 KB shared-memory opt-in run on every device;
  * PSPNet50 students with PSPNet101 / PSANet50 teachers against the same loss on the ATen tail, the teacher untouched;
  * graphed KD steps are bit-identical to eager ones and re-captured for a new option, teacher or teacher weight;
  * the module path."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.kd_oracle import ce_term, kd_loss, kl_term, upsampled
from tests.test_weighted_ce_gpu import _n_graphs
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
# (n, h, w, C, student pitch, teacher pitch)
SHAPES = [(2, 9, 13, 150, 152, 160), (1, 17, 11, 19, 19, 24), (1, 6, 140, 21, 24, 21), (1, 7, 10, 256, 256, 264)]
SHAPE_IDS = ["9x13-150-p152-p160", "17x11-19-p24", "6x140-21-p24", "7x10-256-p264"]
OPTIONS = [(1.0, 1.0, 1.0), (0.5, 1.0, 0.0), (4.0, 0.0, 1.0), (1.0, 1.0, 0.0), (4.0, 1.0, 1.0)]
OPTION_IDS = ["T1-kd1-ce1", "T0.5-kd1-ce0", "T4-kd0-ce1", "T1-kd1-ce0", "T4-kd1-ce1"]


def _run(s, t, target, zoom, kd_zoom, temperature, kd_weight, ce_weight, grad=0.7):
    from semseg_b200 import functional as SF
    sg = s.detach().requires_grad_(True)
    out = SF._UpsampleCEKD.apply(sg, t, target, 255, zoom, kd_zoom, temperature, kd_weight, ce_weight)
    (dl,) = torch.autograd.grad(out[0] * grad, sg)
    return out[0].detach(), out[1], dl


def _check(s, t, target, zoom, at, temperature, kd_weight, ce_weight):
    kd_zoom = zoom if at == "output" else 1
    loss, amax, dl = _run(s, t, target, zoom, kd_zoom, temperature, kd_weight, ce_weight)
    sr = s.detach().clone().requires_grad_(True)
    main, _ = kd_loss(sr, t, target, zoom, temperature, kd_weight, ce_weight, at=at)
    (dl_o,) = torch.autograd.grad(main * 0.7, sr)
    e_loss = abs(loss.item() - main.item()) / abs(main.item())
    e_dl = float((dl.double() - dl_o).abs().max()) / float(dl_o.abs().max())
    print("kd-err zoom=%d at=%s C=%d T=%g kd=%g ce=%g loss=%.3g dl=%.3g" % (zoom, at, s.shape[-1], temperature,
                                                                           kd_weight, ce_weight, e_loss, e_dl))
    assert e_loss <= 1e-6
    assert e_dl <= 1e-5
    x = upsampled(s, zoom)
    clear = _clear_of_ties(x.float())
    assert torch.equal(amax[clear], x.argmax(1)[clear])


@pytest.mark.parametrize("opts", OPTIONS, ids=OPTION_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_kd_kernel_vs_oracle(zoom, shape, opts):
    n, h, w, c, ps, pt = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    s = _logits(n, h, w, c, ps, seed=zoom + 80)
    t = _logits(n, h, w, c, pt, seed=zoom + 90)
    target = _target(n, ho, wo, c, seed=zoom + 80)
    for at in ("output", "logits"):
        _check(s, t, target, zoom, at, *opts)


@pytest.mark.parametrize("zoom", ZOOMS)
def test_kd_equal_maps_give_zero(zoom):
    from semseg_b200 import ops
    n, h, w, c = 2, 9, 13, 150
    s = _logits(n, h, w, c, 152, seed=zoom)
    t = s.detach().clone().contiguous()          # same values, another pitch
    for temperature in (0.5, 1.0, 4.0):
        kl, lse = ops.upsample_kd_fwd(s, t, temperature, zoom=zoom)
        bound = 1e-6 * float(s.abs().mean()) / temperature
        assert abs(kl[0].item()) <= bound
        dl = torch.zeros((n, h, w, c), device="cuda")
        ops.upsample_kd_bwd(s, t, temperature, 1.0, lse, torch.ones((), device="cuda"), dl, zoom=zoom)
        assert float(dl.abs().max()) <= bound
        assert torch.equal(lse[..., 0], lse[..., 1])


@pytest.mark.parametrize("zoom", [1, 8])
def test_kd_saturated_logits_finite(zoom):
    n, h, w, c = 1, 9, 11, 21
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=4)
    s = _logits(n, h, w, c, c, seed=5) * 300.0
    t = _logits(n, h, w, c, c, seed=6) * 300.0
    loss, _, dl = _run(s, t, target, zoom, zoom, 0.5, 1.0, 1.0)
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(dl).all())
    sr = s.detach().clone().requires_grad_(True)
    main, _ = kd_loss(sr, t, target, zoom, 0.5, 1.0, 1.0)
    assert abs(loss.item() - main.item()) <= 1e-5 * abs(main.item())


@pytest.mark.parametrize("zoom", [1, 8])
def test_kd_deterministic_and_pred_is_plain(zoom):
    from semseg_b200 import ops
    n, h, w, c = 2, 17, 23, 150
    s = _logits(n, h, w, c, 152, seed=zoom)
    t = _logits(n, h, w, c, 150, seed=zoom + 1)
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom)
    a = _run(s, t, target, zoom, zoom, 2.0, 1.0, 1.0)
    b = _run(s, t, target, zoom, zoom, 2.0, 1.0, 1.0)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    info, amax, lse = ops.upsample_ce_fwd(s, target, 255, zoom=zoom)
    assert torch.equal(a[1], amax)
    from semseg_b200 import functional as SF
    sg = s.detach().requires_grad_(True)
    out = SF._UpsampleCEKD.apply(sg, t, target, 255, zoom, zoom, 2.0, 1.0, 1.0)
    assert torch.equal(out[0].grad_fn.saved_tensors[3], lse)


# ------------------------------------------------------------------------------------------------ every device
def test_kd_kernels_on_every_device():
    """Shapes whose distillation kernels need more than 48 KB of dynamic shared memory: the forward with 150 / 256
    classes at every zoom, the rows kernel at zoom 8 with Wo = 793; every device computes the bits of device 0."""
    import threading
    from semseg_b200 import ops
    cases = [(1, (1, 9, 140, 256, 256)), (2, (1, 9, 70, 256, 256)), (4, (1, 5, 40, 150, 152)), (8, (1, 5, 100, 21, 24))]
    inputs = [(zoom, _logits(n, h, w, c, p, seed=zoom).cpu(), _logits(n, h, w, c, p, seed=zoom + 5).cpu())
              for zoom, (n, h, w, c, p) in cases]
    results, errors = {}, []

    def run(dev):
        try:
            with torch.cuda.device(dev):
                out = []
                for zoom, s, t in inputs:
                    s, t = s.to(dev), t.to(dev)
                    kl, lse = ops.upsample_kd_fwd(s, t, 2.0, zoom=zoom)
                    dl = torch.zeros(s.shape, device=dev)
                    ops.upsample_kd_bwd(s, t, 2.0, 1.0, lse, torch.ones((), device=dev), dl, zoom=zoom)
                    out.append(tuple(v.cpu() for v in (kl, lse, dl)))
                results[dev] = out
        except Exception as e:      # noqa: BLE001 - reported below
            errors.append((dev, e))

    threads = [threading.Thread(target=run, args=(d,)) for d in range(torch.cuda.device_count())]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for dev, out in results.items():
        for got, ref in zip(out, results[0]):
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), dev


# ------------------------------------------------------------------------------------------------ networks
def _torch_kd_class():
    from semseg_b200.losses import DistillationLoss

    class _TorchKD(DistillationLoss):
        """DistillationLoss written in fp32 PyTorch under another type: the network keeps the eager route (interpolate
        both maps -> criterion). Its KD term is at the size it is given: the 'output' form."""

        def forward(self, logits, target, teacher_logits=None):
            valid = (target != self.ignore_index) & (target >= 0) & (target < logits.shape[1])
            ce = F.cross_entropy(logits, torch.where(valid, target, torch.full_like(target, -100)), ignore_index=-100)
            if teacher_logits is None:
                return ce
            T = self.temperature
            lp = F.log_softmax(logits / T, dim=1)
            lq = F.log_softmax(teacher_logits / T, dim=1)
            kl = (lq.exp() * (lq - lp)).sum(1).mean()
            return self.ce_weight * ce + self.kd_weight * T * T * kl

    return _TorchKD


def _teacher(kind, zoom):
    torch.manual_seed(5)
    if kind == "psp101":
        from semseg_b200.pspnet import PSPNet
        t = PSPNet(layers=101, classes=21, zoom_factor=zoom, dropout=0.0, pretrained=False)
    else:
        t = _build("psa", zoom, seed=5)
    return t.cuda().eval()


def _state(m):
    return [v.detach().clone() for v in list(m.parameters()) + list(m.buffers())], m.training


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("teacher_kind", ["psp101", "psa50"])
def test_network_native_kd_matches_aten(teacher_kind, zoom, mode, monkeypatch):
    """One step of a PSPNet50 student on the native KD tail against the same loss in PyTorch on the ATen tail (the
    teacher's logits a detached constant in both), x.grad included; then two more native steps leave the teacher's
    parameters, buffers and training flag bit-identical and give it no gradient."""
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import DistillationLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    teacher = _teacher(teacher_kind, zoom)
    before, flag = _state(teacher)
    native = _build("psp", zoom).cuda().train()
    aten = copy.deepcopy(native)
    native.criterion = DistillationLoss(teacher, temperature=2.0, kd_weight=0.5, ce_weight=1.0)
    aten.criterion = _torch_kd_class()(teacher, temperature=2.0, kd_weight=0.5, ce_weight=1.0)
    x, y = _batch(zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    with precision.mode(mode):
        xn = x.clone().requires_grad_(True)
        pred, main, aux = native(xn, y)
        (main + 0.4 * aux).backward()
        xa = x.clone().requires_grad_(True)
        pred_r, main_r, aux_r = aten(xa, y)
        (main_r + 0.4 * aux_r).backward()
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01
    if mode == "bf16x3":    # as tests/test_zoom_gpu.py: in bf16 the tails' ~1e-6 dlogits differences flip bf16 roundings
        loose = {"layer0.7.bias": 3e-4}
        bad = []
        for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
            assert (pn.grad is None) == (pa.grad is None), k
            if pn.grad is not None:
                err = util.rel_l2(pn.grad, pa.grad)
                if err > loose.get(k, 1e-4):
                    bad.append((k, err))
        assert not bad, bad
        assert util.rel_l2(xn.grad, xa.grad) <= 1e-4
    with precision.mode(mode):
        for _ in range(2):
            _, main, aux = native(x, y)
            (main + 0.4 * aux).backward()
    after, flag_after = _state(teacher)
    assert flag_after is False and flag is False
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    assert all(p.grad is None for p in teacher.parameters())


@pytest.mark.parametrize("zoom", [2, 8])
def test_network_at_logits_matches_oracle_statement(zoom, monkeypatch):
    """at='logits': the main loss is CE at the target size plus the KL of the raw maps, stated with the network's own
    student and teacher logits."""
    from semseg_b200 import precision
    from semseg_b200.losses import DistillationLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    teacher = _teacher("psa50", zoom)
    model = _build("psp", zoom).cuda().train()
    model.criterion = DistillationLoss(teacher, temperature=4.0, kd_weight=1.0, ce_weight=0.5, at="logits")
    x, y = _batch(zoom)
    seen = {}
    orig = model._logits_nhwc

    def spy(inp):
        out = orig(inp)
        seen["s"] = out[0].detach().clone()
        return out
    model._logits_nhwc = spy
    with precision.mode("bf16x3"):
        _, main, _ = model(x, y)
        t = model.criterion.run_teacher(x, 21)
    ref, _ = kd_loss(seen["s"], t, y, zoom, 4.0, 1.0, 0.5, at="logits")
    assert abs(main.item() - ref.item()) <= 1e-5 * abs(ref.item())


# ------------------------------------------------------------------------------------------------ graphs
def _kd_model(teacher, **kw):
    from semseg_b200.losses import DistillationLoss
    m = _build("psp", 8).cuda().train()
    m.criterion = DistillationLoss(teacher, **kw)
    return m


def _graphed_and_eager(teacher, monkeypatch, **kw):
    from semseg_b200.losses import DistillationLoss
    base = _kd_model(teacher, **kw)
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    for m in (eager, graphed):
        m.criterion = DistillationLoss(teacher, **kw)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]

    def both(expect_graphs):
        from semseg_b200 import graphs
        n_steps = graphs.WARMUP_CALLS + 3
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
        le = _sgd_steps(eager, batches, n_steps)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
        lg = _sgd_steps(graphed, batches, n_steps)
        assert le == lg, (le, lg)
        assert _n_graphs(graphed) == expect_graphs
        return lg
    return eager, graphed, both


def test_graphed_kd_steps_bit_identical_to_eager_and_recaptured_for_options(monkeypatch):
    from semseg_b200 import graphs
    teacher = _teacher("psp101", 8)
    eager, graphed, both = _graphed_and_eager(teacher, monkeypatch, temperature=2.0, kd_weight=0.5)
    both(1)
    assert graphs.launches_per_step(graphed) > 100
    print("kd launches per step", graphs.launches_per_step(graphed))
    # a new temperature, kd_weight or `at` is a new launch argument: captured anew
    for k, (attr, val) in enumerate((("temperature", 1.0), ("kd_weight", 1.0), ("at", "logits"))):
        for m in (eager, graphed):
            setattr(m.criterion, attr, val)
        both(2 + k)


def test_graphed_kd_recaptured_for_teacher_edit_and_new_teacher(monkeypatch):
    from semseg_b200.losses import DistillationLoss
    teacher = _teacher("psp101", 8)
    eager, graphed, both = _graphed_and_eager(teacher, monkeypatch, temperature=2.0)
    first = both(1)
    # an in-place edit of a teacher weight: captured anew, and the replayed losses are the eager ones with the edit
    with torch.no_grad():
        teacher.cls[4].weight.mul_(1.5)
    edited = both(2)
    assert edited != first
    other = _teacher("psa50", 8)
    for m in (eager, graphed):
        m.criterion = DistillationLoss(other, temperature=2.0)
    both(3)


def test_graphed_kd_step_launches_no_aten_tail():
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    teacher = _teacher("psp101", 8)
    model = _kd_model(teacher, temperature=2.0)
    x, y = _batch(8)
    for _ in range(graphs.WARMUP_CALLS + 2):
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
    torch.cuda.synchronize()
    assert graphs.launches_per_step(model) > 100
    for p in model.parameters():
        p.grad = None            # no gradient accumulation (an add_ per parameter) in the profiled step
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    n_logits = 2 * 21 * 9 * 9
    bad = []
    for e in prof.events():
        if any(k in e.name for k in ("upsample_bilinear2d", "_softmax", "_log_softmax", "kl_div")):
            bad.append(e.name)
        elif e.name in ("aten::add", "aten::add_") and any(
                s and int(torch.tensor(s).prod()) >= n_logits for s in (e.input_shapes or []) if isinstance(s, list)):
            bad.append(e.name)
    assert not bad, sorted(set(bad))


# ------------------------------------------------------------------------------------------------ module path
def test_kd_module_path_matches_oracle():
    from semseg_b200.losses import DistillationLoss
    teacher = _teacher("psa50", 8)
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
        t_out = teacher(x)
    crit = DistillationLoss(teacher, temperature=2.0, kd_weight=0.5, ce_weight=1.0)
    loss = crit(out, y)
    ref = ce_term(out, y)
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    loss = crit(out, y, t_out)
    ref = ce_term(out, y) + 0.5 * 4.0 * kl_term(out, t_out, 2.0)
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    lg = out.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(crit(lg, y, t_out), lg)
    lr = out.detach().double().requires_grad_(True)
    (g_ref,) = torch.autograd.grad(ce_term(lr, y) + 2.0 * kl_term(lr, t_out, 2.0), lr)
    assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
