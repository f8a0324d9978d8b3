"""GPU tier: the focal loss on the fused tail (csrc/tail.cu focal kernels through semseg_b200/functional.py).

  * kernel vs the float64 oracle of tests/focal_oracle.py at zoom 1, 2, 4, 8, with odd h != w, widths off and across the
    128-column CTA, 19 / 21 / 150 / 256 classes, a padded pitch, gamma 0 / 0.5 / 1 / 2 / 5, weight None / random with a
    zero class, ignored and out-of-range targets;
  * gamma = 0 is the plain tail (lse and argmax bit-equal), all-ones weights change no bit;
  * saturated logits (every valid pixel at p_t >= 1 - 1e-5, some at p_t = 1 in fp32), constant logits, nothing valid and
    an all-zero-weight batch; the kernels are deterministic and run on every device;
  * PSPNet50 / PSANet50 on the native focal tail against the same loss written in PyTorch on the ATen tail;
  * graphed focal steps are bit-identical to eager ones, re-captured for a new gamma or weight tensor, see in-place
    weight edits, and launch no ATen tail kernel;
  * the module path FocalLoss(...)(eval_logits, y) against the oracle."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.focal_oracle import focal_loss, focal_tail
from tests.test_ohem_gpu import _upsampled
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
GAMMAS = [0.0, 0.5, 1.0, 2.0, 5.0]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24), (1, 7, 10, 256, 256)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24", "7x10-256"]


def _weights(c, seed, zero_class=True):
    """Seeded positive class weights in [0.25, 2.25), one class weighted 0."""
    g = torch.Generator(device="cuda").manual_seed(seed + 100)
    w = torch.rand(c, device="cuda", generator=g) * 2 + 0.25
    if zero_class:
        w[seed % c] = 0.0
    return w


def _run(logits, target, zoom, weight, gamma, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse, mod = ops.upsample_ce_focal_fwd(logits, target, 255, weight, gamma, zoom=zoom)
    dl = ops.upsample_ce_focal_bwd(logits, target, 255, lse, mod, info, torch.tensor([grad], device="cuda"), zoom=zoom)
    return info, amax, lse, mod, dl


@pytest.mark.parametrize("gamma", GAMMAS)
@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_focal_kernel_vs_oracle(zoom, shape, weighted, gamma):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 20)
    target = _target(n, ho, wo, c, seed=zoom + 20)
    weight = _weights(c, zoom) if weighted else None
    info, amax, _, mod, dl = _run(logits, target, zoom, weight, gamma)
    loss_o, n_valid, dl_o = focal_tail(logits, target, zoom, gamma, weight)
    valid = (target != 255) & (target >= 0) & (target < c)
    assert n_valid == int(valid.sum()) > 0 and info[1].item() == n_valid
    # measured on an H100 over this grid: loss 2.8e-7 relative, dlogits 1.1e-6 of max |dlogits|
    assert abs(info[0].item() - loss_o.item()) <= 2e-6 * abs(loss_o.item())
    assert float((dl.double() - 0.7 * dl_o).abs().max()) <= 5e-6 * float(0.7 * dl_o.abs().max())
    assert float(mod[~valid].abs().max()) == 0.0 and bool((mod >= 0).all())
    x = _upsampled(logits, zoom)
    clear = _clear_of_ties(x)
    assert torch.equal(amax[clear], x.argmax(1)[clear])


@pytest.mark.parametrize("zoom", ZOOMS)
def test_focal_gamma_zero_is_the_plain_tail(zoom):
    from semseg_b200 import ops
    n, h, w, c, pitch = 2, 9, 13, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 40)
    target = _target(n, ho, wo, c, seed=zoom + 40)
    g = torch.tensor([0.7], device="cuda")
    info_p, amax_p, lse_p = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    dl_p = ops.upsample_ce_bwd(logits, target, 255, lse_p, info_p, g, zoom=zoom)
    info, amax, lse, mod, dl = _run(logits, target, zoom, None, 0.0)
    assert torch.equal(lse, lse_p) and torch.equal(amax, amax_p) and info[1].item() == info_p[1].item()
    assert abs(info[0].item() - info_p[0].item()) <= 1e-6 * abs(info_p[0].item())
    valid = (target != 255) & (target >= 0) & (target < c)
    assert bool((mod[valid] == 1.0).all())                       # M = 1 at gamma = 0
    assert float((dl - dl_p).abs().max()) <= 1e-6 * float(dl_p.abs().max())
    # all-ones weights change no bit, at any gamma
    ones = torch.ones(c, device="cuda")
    for gamma in (0.0, 2.0):
        for u, v in zip(_run(logits, target, zoom, ones, gamma), _run(logits, target, zoom, None, gamma)):
            assert torch.equal(u, v)
    # every gamma keeps the plain forward's lse and argmax
    _, amax2, lse2, _, _ = _run(logits, target, zoom, _weights(c, 3), 2.0)
    assert torch.equal(lse2, lse_p) and torch.equal(amax2, amax_p)


@pytest.mark.parametrize("gamma", [0.5, 2.0])
@pytest.mark.parametrize("zoom", ZOOMS)
def test_focal_saturated_logits(zoom, gamma):
    """Every valid pixel has p_t >= 1 - 1e-5 and some have p_t = 1 in fp32 (down to q = 0 exactly in fp32): q from a
    rounded p_t, or nll from a rounded lse - v_t, would have no correct digit here."""
    n, h, w, c, k = 2, 9, 13, 21, 3
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    g = torch.Generator(device="cuda").manual_seed(zoom + 60)
    logits = torch.randn((n, h, w, c), device="cuda", generator=g).clamp_(-3, 3)
    levels = torch.tensor([20.0, 25.0, 40.0, 120.0], device="cuda")
    logits[..., k] = levels[torch.randint(0, 4, (n, h, w), device="cuda", generator=g)]
    target = torch.full((n, ho, wo), k, dtype=torch.int64, device="cuda")
    target[torch.rand((n, ho, wo), device="cuda", generator=g) < 0.05] = 255
    valid = target != 255
    x = _upsampled(logits, zoom).double()
    logp = torch.log_softmax(x, 1)
    q_o = torch.logsumexp(torch.cat([logp[:, :k], logp[:, k + 1:]], 1), 1).exp()
    assert float(q_o.max()) <= 1e-5 and bool(((1.0 - q_o).float() == 1.0)[valid].any())
    for weight in (None, _weights(c, 1, zero_class=False)):
        info, _, lse, mod, dl = _run(logits, target, zoom, weight, gamma)
        loss_o, n_valid, dl_o = focal_tail(logits, target, zoom, gamma, weight)
        for t in (info, lse, mod, dl):
            assert bool(torch.isfinite(t).all())
        assert info[1].item() == n_valid and loss_o.item() > 0
        assert abs(info[0].item() - loss_o.item()) <= 1e-4 * loss_o.item()
        # the other classes' gradient w_t M p_c keeps its relative accuracy; the target's is minus their sum up to the
        # fp32 rounding of p_t - 1, so only its finiteness is held
        others = [i for i in range(c) if i != k]
        err = (dl.double() - 0.7 * dl_o)[..., others].abs().max()
        assert float(err) <= 1e-3 * float(0.7 * dl_o[..., others].abs().max())
        assert bool((mod[valid & (q_o.float() == 0)] == 0).all())          # 0^gamma = 0 for gamma > 0


@pytest.mark.parametrize("zoom", [1, 8])
def test_focal_constant_logits(zoom):
    n, h, w, c = 1, 5, 9, 19
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = torch.full((n, h, w, c), 1.25, device="cuda")
    target = _target(n, ho, wo, c, seed=5)
    for gamma in (0.0, 2.0):
        info, _, lse, mod, dl = _run(logits, target, zoom, None, gamma)
        loss_o, n_valid, dl_o = focal_tail(logits, target, zoom, gamma, None)
        assert info[1].item() == n_valid
        assert abs(info[0].item() - loss_o.item()) <= 2e-6 * loss_o.item()          # (1 - 1/C)^gamma log C
        assert float((dl.double() - 0.7 * dl_o).abs().max()) <= 1e-5 * float(0.7 * dl_o.abs().max())


@pytest.mark.parametrize("zoom", ZOOMS)
def test_focal_nothing_to_train_gives_zero(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    # every pixel ignored or out of range
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    target[:, ::3] = c
    target[:, 1::3] = -1
    for weight in (None, _weights(c, 1)):
        for gamma in (0.0, 0.5, 2.0):
            info, _, _, mod, dl = _run(logits, target, zoom, weight, gamma)
            assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0 and float(mod.abs().max()) == 0.0
    # every valid pixel in a zero-weight class: the count stays, loss and gradient are 0
    target = _target(n, ho, wo, c, seed=3)
    weight = torch.ones(c, device="cuda")
    weight[target[(target >= 0) & (target < c)].unique()] = 0.0
    weight[0] = 1.0
    target[target == 0] = 255                      # class 0 keeps a weight but no pixel
    n_valid = int(((target >= 0) & (target < c)).sum())
    for gamma in (0.0, 0.5, 2.0):
        info, _, _, _, dl = _run(logits, target, zoom, weight, gamma)
        assert info.tolist() == [0.0, float(n_valid)] and float(dl.abs().max()) == 0.0, gamma


@pytest.mark.parametrize("zoom", [1, 8])
def test_focal_deterministic(zoom):
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    weight = _weights(c, zoom)
    for u, v in zip(_run(logits, target, zoom, weight, 2.0), _run(logits, target, zoom, weight, 2.0)):
        assert torch.equal(u, v)


def test_focal_kernels_on_every_device():
    """Shapes whose kernels need more than 48 KB of dynamic shared memory: the forward at zoom 1 and 2 with 150 classes,
    the rows kernel at zoom 8 with Wo = 793, from one thread per device; every device computes the bits of device 0."""
    import threading
    cases = [(1, (2, 9, 140, 150, 152)), (2, (2, 9, 70, 150, 150)), (8, (1, 5, 100, 21, 24))]
    inputs = []
    for zoom, (n, h, w, c, pitch) in cases:
        inputs.append((zoom, _logits(n, h, w, c, pitch, seed=zoom).cpu(),
                       _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom).cpu(), _weights(c, zoom).cpu()))
    results, errors = {}, []

    def run(dev):
        try:
            with torch.cuda.device(dev):
                from semseg_b200 import ops
                out = []
                for zoom, logits, target, weight in inputs:
                    lg, t, wt = logits.to(dev), target.to(dev), weight.to(dev)
                    info, amax, lse, mod = ops.upsample_ce_focal_fwd(lg, t, 255, wt, 2.0, zoom=zoom)
                    dl = ops.upsample_ce_focal_bwd(lg, t, 255, lse, mod, info, torch.tensor([1.0], device=dev),
                                                   zoom=zoom)
                    out.append(tuple(v.cpu() for v in (info, amax, lse, mod, dl)))
                results[dev] = out
        except Exception as e:      # noqa: BLE001 - reported below
            errors.append((dev, e))

    threads = [threading.Thread(target=run, args=(d,)) for d in range(torch.cuda.device_count())]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert sorted(results) == list(range(torch.cuda.device_count()))
    for dev, out in results.items():
        for (zoom, _, _, _), got, ref in zip(inputs, out, results[0]):
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), (dev, zoom)


def test_fused_tail_accepts_focal_with_cuda_weights():
    from semseg_b200 import functional as SF
    from semseg_b200.losses import FocalLoss
    x_size = torch.Size((2, 3, 65, 81))
    logits = torch.zeros((2, 9, 11, 21), device="cuda")
    y = torch.zeros((2, 65, 81), dtype=torch.int64, device="cuda")
    w = _weights(21, 0)
    crit = FocalLoss(weight=w)
    assert SF.fused_tail_supported(crit, None, y, 8, x_size) and SF.fused_tail_supported(crit, logits, y, 8)
    assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 19), device="cuda"), y, 8)      # length != C
    assert not SF.fused_tail_supported(crit, logits, y.cpu(), 8)
    assert FocalLoss(weight=w.cpu()).cuda().weight.is_cuda                                          # a buffer
    for bad in (torch.ones((21, 2), device="cuda")[:, 0], w.double()):
        assert not SF.fused_tail_supported(FocalLoss(weight=bad), logits, y, 8)
    assert not SF.fused_tail_supported(_torch_focal_class()(weight=w), logits, y, 8)


# ------------------------------------------------------------------------------------------------ networks
def _torch_focal(logits, target, gamma, weight, ignore_index):
    valid = target != ignore_index
    t = torch.where(valid, target, torch.zeros_like(target))
    logp_t = F.log_softmax(logits, dim=1).gather(1, t.unsqueeze(1)).squeeze(1)
    pix = torch.pow(1.0 - logp_t.exp(), gamma) * -logp_t
    if weight is not None:
        pix = pix * weight[t]
    return (pix * valid).sum() / valid.sum().clamp(min=1)


def _torch_focal_class():
    from semseg_b200.losses import FocalLoss

    class _TorchFocal(FocalLoss):
        """FocalLoss written in PyTorch under another type: the network keeps the ATen tail (interpolate -> criterion)."""

        def forward(self, logits, target):
            return _torch_focal(logits, target, self.gamma, self.weight, self.ignore_index)

    return _TorchFocal


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_focal_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import FocalLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    weight = _weights(21, 4, zero_class=False)
    native.criterion = FocalLoss(gamma=2.0, weight=weight, ignore_index=255)
    aten = copy.deepcopy(native)
    aten.criterion = _torch_focal_class()(gamma=2.0, weight=weight.clone(), ignore_index=255)
    x, y = _batch(zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    with precision.mode(mode):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert pred.shape == pred_r.shape == y.shape
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01          # argmax: equal but at top-1 / top-2 ties
    assert native.criterion.weight.grad is None
    if mode != "bf16x3":
        return      # as tests/test_zoom_gpu.py: in bf16 the tails' ~1e-6 dlogits differences flip bf16 roundings
    loose = {"layer0.7.bias": 3e-4}                               # as tests/test_zoom_gpu.py: a cancelling sum
    bad = []
    for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
        assert (pn.grad is None) == (pa.grad is None), k
        if pn.grad is not None:
            err = util.rel_l2(pn.grad, pa.grad)
            if err > loose.get(k, 1e-4):
                bad.append((k, err))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ graphs
def _n_graphs(model):
    return sum(1 for s in model._sb_graph_steps.values() if s.fwd is not None)


def _both(eager, graphed, batches, n_steps, monkeypatch):
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, n_steps)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, n_steps)
    assert le == lg, (le, lg)
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.equal(pe, pg), k
        assert (pe.grad is None) == (pg.grad is None) and (pe.grad is None or torch.equal(pe.grad, pg.grad)), k


def test_graphed_focal_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import FocalLoss
    base = _build("psp", 8).cuda().train()
    base.criterion = FocalLoss(gamma=2.0, weight=_weights(21, 2), ignore_index=255)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    _both(eager, graphed, batches, n_steps, monkeypatch)
    assert graphs.launches_per_step(graphed) > 100 and _n_graphs(graphed) == 1
    # an in-place edit of the weights needs no capture: the next replay reads the new values
    for m in (eager, graphed):
        with torch.no_grad():
            m.criterion.weight.mul_(torch.linspace(0.5, 1.5, 21, device="cuda"))
    _both(eager, graphed, batches, 2, monkeypatch)
    assert _n_graphs(graphed) == 1
    # a new gamma and a replaced weight tensor each capture anew, never replay the old graph
    for change in (lambda m: setattr(m.criterion, "gamma", 0.5),
                   lambda m: setattr(m.criterion, "weight", _weights(21, 9))):
        for m in (eager, graphed):
            change(m)
        _both(eager, graphed, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 3


def test_graphed_focal_step_kernel_count_and_no_aten_tail():
    """A graphed focal step launches as many kernels as the default criterion's (each plain tail kernel is replaced one
    for one) and none of ATen's upsample / log-softmax / nll / pow kernels."""
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import FocalLoss
    x, y = _batch(8)
    counts = {}
    for name in ("ce", "focal"):
        model = _build("psp", 8).cuda().train()
        if name == "focal":
            model.criterion = FocalLoss(gamma=2.0, weight=_weights(21, 1))
        for _ in range(graphs.WARMUP_CALLS + 2):
            _, ml, al = model(x, y)
            (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
        counts[name] = graphs.launches_per_step(model)
    assert counts["focal"] == counts["ce"] > 100, counts
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    bad = [n for n in names if any(k in n for k in ("upsample_bilinear2d", "_log_softmax", "log_softmax", "LogSoftMax",
                                                    "nll_loss", "pow"))]
    assert not bad, sorted(set(bad))


# ------------------------------------------------------------------------------------------------ module path
def test_focal_module_path_matches_oracle():
    """FocalLoss(...)(eval_model(x), y) as validate() calls it, and its gradient."""
    from semseg_b200.losses import FocalLoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    w = _weights(21, 2)
    for crit in (FocalLoss(), FocalLoss(gamma=0.5, weight=w), FocalLoss(gamma=0.0)):
        loss = crit(out, y)
        ref, _, g_ref = focal_loss(out, y, crit.gamma, crit.weight, crit.ignore_index)
        assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
        lg = out.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(crit(lg, y), lg)
        assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
    with pytest.raises(ValueError, match="weight"):
        FocalLoss(weight=torch.ones(19, device="cuda"))(out, y)
