"""GPU tier: class-weighted and label-smoothed cross-entropy, and weighted OHEM, on the fused tail (csrc/tail.cu kWeighted
kernels through semseg_b200/functional.py).

  * kernel vs the float64 oracle of tests/weighted_ce_oracle.py at zoom 1, 2, 4, 8, with odd h != w, widths off the
    128-column CTA, 19 / 21 / 150 / 256 classes, a padded pitch, weight None / random with a zero class, eps 0 / 0.1 / 1,
    ignored and out-of-range targets; and vs torch's own F.cross_entropy on ATen-upsampled logits;
  * D = 0 gives loss 0 and an exactly zero gradient; the kernels are deterministic; weight None with eps 0 still runs
    the plain kernels, and all-ones weights reproduce the unweighted kernels bit for bit;
  * weighted OHEM vs the oracle in the four regimes of tests/test_ohem_gpu.py;
  * PSPNet50 / PSANet50 on the native weighted tail against the same network on the ATen tail;
  * the kernels that need the > 48 KB shared-memory opt-in run on every device;
  * graphed weighted steps are bit-identical to eager ones, re-captured for a new label_smoothing or weight tensor, see
    in-place weight edits, and launch no ATen tail kernel;
  * the module path OhemCrossEntropyLoss(weight=w)(eval_logits, y) against the oracle."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import util
from tests.test_ohem_gpu import REGIMES, _upsampled
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target
from tests.weighted_ce_oracle import weighted_ce, weighted_ohem_ce

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24), (1, 7, 10, 256, 256)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24", "7x10-256"]


def _weights(c, seed, zero_class=True):
    """Seeded positive class weights in [0.25, 2.25), one class weighted 0."""
    g = torch.Generator(device="cuda").manual_seed(seed + 100)
    w = torch.rand(c, device="cuda", generator=g) * 2 + 0.25
    if zero_class:
        w[seed % c] = 0.0
    return w


def _run(logits, target, zoom, weight, eps, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse = ops.upsample_ce_weighted_fwd(logits, target, 255, weight, eps, zoom=zoom)
    dl = ops.upsample_ce_weighted_bwd(logits, target, 255, weight, eps, lse, info, torch.tensor([grad], device="cuda"),
                                      zoom=zoom)
    return info, amax, lse, dl


@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_weighted_kernel_vs_oracle(zoom, shape, weighted, eps):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 20)
    target = _target(n, ho, wo, c, seed=zoom + 20)
    weight = _weights(c, zoom) if weighted else None
    info, amax, _, dl = _run(logits, target, zoom, weight, eps)

    lr = logits.detach().clone().requires_grad_(True)
    x = _upsampled(lr, zoom)
    loss_o, d_o = weighted_ce(x, target, weight, 255, eps)
    (dl_o,) = torch.autograd.grad(loss_o * 0.7, lr)
    assert float(d_o) > 0
    assert abs(info[1].item() - float(d_o)) <= 1e-6 * float(d_o)
    assert abs(info[0].item() - loss_o.item()) <= 2e-5 * abs(loss_o.item())
    assert float((dl.double() - dl_o).abs().max()) <= 1e-5 * float(dl_o.abs().max())
    clear = _clear_of_ties(x.detach())
    assert torch.equal(amax[clear], x.detach().argmax(1)[clear])


@pytest.mark.parametrize("zoom", [2, 8])
def test_weighted_kernel_vs_torch_cross_entropy(zoom):
    """Against torch's own CUDA F.cross_entropy(weight, ignore_index, label_smoothing) on ATen-upsampled fp32 logits.
    In-range targets only: torch's CUDA loss device-asserts on any other."""
    from semseg_b200 import functional as SF
    n, h, w, c, pitch = 2, 9, 13, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=31)
    target = _target(n, ho, wo, c, seed=31)
    target[(target != 255) & ((target < 0) | (target >= c))] = 255
    weight = _weights(c, 3)
    for eps in (0.0, 0.1):
        crit = nn.CrossEntropyLoss(weight=weight, ignore_index=255, label_smoothing=eps)
        lg = logits.detach().clone().requires_grad_(True)
        loss, _ = SF.upsample_ce(lg, target, 255, zoom=zoom, criterion=crit)
        (dl,) = torch.autograd.grad(loss, lg)
        lr = logits.detach().clone().requires_grad_(True)
        ref = F.cross_entropy(_upsampled(lr, zoom), target, weight=weight, ignore_index=255, label_smoothing=eps)
        (dl_r,) = torch.autograd.grad(ref, lr)
        assert abs(loss.item() - ref.item()) <= 2e-5 * abs(ref.item()), eps
        assert float((dl - dl_r).abs().max()) <= 1e-5 * float(dl_r.abs().max()), eps


@pytest.mark.parametrize("zoom", ZOOMS)
def test_weighted_d_zero_gives_zero(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    # every pixel ignored
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    for weight in (None, _weights(c, 1)):
        info, _, _, dl = _run(logits, target, zoom, weight, 0.1)
        assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0
    # every valid pixel in a zero-weight class: the smoothing term is non-zero, D is 0
    target = _target(n, ho, wo, c, seed=3)
    weight = torch.ones(c, device="cuda")
    weight[target[(target >= 0) & (target < c)].unique()] = 0.0
    weight[0] = 1.0
    target[target == 0] = 255                      # class 0 keeps a weight but no pixel
    for eps in (0.0, 0.1, 1.0):
        info, _, _, dl = _run(logits, target, zoom, weight, eps)
        assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0, eps


@pytest.mark.parametrize("zoom", [1, 8])
def test_weighted_deterministic(zoom):
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    weight = _weights(c, zoom)
    a = _run(logits, target, zoom, weight, 0.1)
    b = _run(logits, target, zoom, weight, 0.1)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    a = _ohem_run(logits, target, zoom, 0.2, n * ho * wo // 4, weight)
    b = _ohem_run(logits, target, zoom, 0.2, n * ho * wo // 4, weight)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.parametrize("zoom", ZOOMS)
def test_unweighted_forms_unchanged(zoom, monkeypatch):
    """nn.CrossEntropyLoss() (weight None, eps 0) runs the plain kernels and OhemCrossEntropyLoss() the OHEM ones,
    bit-equal to ops.upsample_ce_* / ops.upsample_ce_ohem_*; with all-ones weights the weighted kernels compute the
    same bits as the unweighted ones."""
    from semseg_b200 import functional as SF
    from semseg_b200 import ops
    from semseg_b200.losses import OhemCrossEntropyLoss
    n, h, w, c, pitch = 2, 9, 13, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 40)
    target = _target(n, ho, wo, c, seed=zoom + 40)
    g = torch.tensor([0.7], device="cuda")
    info, amax, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    dl = ops.upsample_ce_bwd(logits, target, 255, lse, info, g, zoom=zoom)
    called = []
    real = ops.upsample_ce_weighted_fwd
    monkeypatch.setattr(ops, "upsample_ce_weighted_fwd", lambda *a, **k: called.append(1) or real(*a, **k))
    lg = logits.detach().clone().requires_grad_(True)
    loss, pred = SF.upsample_ce(lg, target, 255, zoom=zoom, criterion=nn.CrossEntropyLoss(ignore_index=255))
    (dl_s,) = torch.autograd.grad(loss * 0.7, lg)
    assert not called
    assert torch.equal(loss, info[0]) and torch.equal(pred, amax) and torch.equal(dl_s, dl)
    ones = torch.ones(c, device="cuda")
    info_w, amax_w, lse_w, dl_w = _run(logits, target, zoom, ones, 0.0)
    assert torch.equal(info_w, info) and torch.equal(amax_w, amax) and torch.equal(lse_w, lse)
    assert torch.equal(dl_w, dl)

    thresh, min_kept = 0.3, n * ho * wo // 3
    ref = _ohem_run(logits, target, zoom, thresh, min_kept, None)
    for u, v in zip(_ohem_run(logits, target, zoom, thresh, min_kept, ones), ref):
        assert torch.equal(u, v)
    lg = logits.detach().clone().requires_grad_(True)
    loss, pred = SF.upsample_ce(lg, target, 255, zoom=zoom, criterion=OhemCrossEntropyLoss(255, thresh, min_kept))
    (dl_s,) = torch.autograd.grad(loss * 0.7, lg)
    assert torch.equal(loss, ref[0][0]) and torch.equal(pred, ref[1]) and torch.equal(dl_s, ref[-1])


# ------------------------------------------------------------------------------------------------ weighted OHEM
def _ohem_run(logits, target, zoom, thresh, min_kept, weight, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse, pt, nll, thr = ops.upsample_ce_ohem_fwd(logits, target, 255, thresh, min_kept, zoom=zoom,
                                                             weight=weight)
    dl = ops.upsample_ce_ohem_bwd(logits, target, 255, lse, pt, thr, info, torch.tensor([grad], device="cuda"),
                                  zoom=zoom, weight=weight)
    return info, amax, pt, nll, thr, dl


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("shape", SHAPES[:3], ids=SHAPE_IDS[:3])
@pytest.mark.parametrize("zoom", ZOOMS)
def test_weighted_ohem_kernel_vs_oracle(zoom, shape, regime):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    thresh, frac, _ = REGIMES[regime]
    min_kept = int(frac * n * ho * wo)
    logits = _logits(n, h, w, c, pitch, seed=zoom + 10)
    target = _target(n, ho, wo, c, seed=zoom + 10)
    weight = _weights(c, zoom + 5)
    info, amax, pt, nll, thr, dl = _ohem_run(logits, target, zoom, thresh, min_kept, weight)
    # the selection is the unweighted one, bit for bit
    _, _, pt_u, nll_u, thr_u, _ = _ohem_run(logits, target, zoom, thresh, min_kept, None)
    assert torch.equal(pt, pt_u) and torch.equal(thr, thr_u)
    valid = pt >= 0
    t = torch.where(valid, target, torch.zeros_like(target))
    assert torch.equal(nll[valid], (weight[t] * nll_u)[valid])

    lr = logits.detach().clone().requires_grad_(True)
    x = _upsampled(lr, zoom)
    _, kept_o, thr_o, pt_o = weighted_ohem_ce(x.detach(), target, weight, 255, thresh, min_kept)
    kept_k = valid & (pt < thr)
    differ = kept_k != kept_o
    assert bool(((pt_o[differ] - thr_o).abs() < 1e-5).all()), "kept sets differ away from the threshold"
    assert int(info[1]) == int(kept_k.sum()) > 0
    loss_o, _, _, _ = weighted_ohem_ce(x, target, weight, 255, thresh, min_kept, kept=kept_k)
    (dl_o,) = torch.autograd.grad(loss_o * 0.7, lr)
    assert abs(info[0].item() - loss_o.item()) <= 2e-5 * abs(loss_o.item())
    assert float((dl.double() - dl_o).abs().max()) <= 1e-5 * float(dl_o.abs().max())
    clear = _clear_of_ties(x.detach())
    assert torch.equal(amax[clear], x.detach().argmax(1)[clear])


def test_fused_tail_accepts_cuda_weights():
    from semseg_b200 import functional as SF
    from semseg_b200.losses import OhemCrossEntropyLoss
    x_size = torch.Size((2, 3, 65, 81))
    logits = torch.zeros((2, 9, 11, 21), device="cuda")
    y = torch.zeros((2, 65, 81), dtype=torch.int64, device="cuda")
    w = _weights(21, 0)
    for eps in (0.0, 0.1, 1.0):
        crit = nn.CrossEntropyLoss(ignore_index=255, label_smoothing=eps)
        assert SF.fused_tail_supported(crit, None, y, 8, x_size)
        assert SF.fused_tail_supported(crit, logits, y, 8)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 257), device="cuda"), y, 8)
    for crit in (nn.CrossEntropyLoss(weight=w, ignore_index=255), nn.CrossEntropyLoss(weight=w, label_smoothing=0.1),
                 OhemCrossEntropyLoss(weight=w)):
        assert SF.fused_tail_supported(crit, None, y, 8, x_size)
        assert SF.fused_tail_supported(crit, logits, y, 8)
        assert not SF.fused_tail_supported(crit, torch.zeros((2, 9, 11, 19), device="cuda"), y, 8)   # length != C
        assert not SF.fused_tail_supported(crit, logits, y.cpu(), 8)
    for crit in (nn.CrossEntropyLoss(weight=w, reduction="sum"), nn.CrossEntropyLoss(label_smoothing=0.1,
                                                                                      reduction="none"),
                 _ATenCE(weight=w), _ATenCE(label_smoothing=0.1)):
        assert not SF.fused_tail_supported(crit, None, y, 8, x_size)
        assert not SF.fused_tail_supported(crit, logits, y, 8)
    for bad in (torch.ones((21, 2), device="cuda")[:, 0], w.double(), torch.ones((1, 21), device="cuda")):
        for crit in (nn.CrossEntropyLoss(weight=bad, ignore_index=255), ):
            assert not SF.fused_tail_supported(crit, None, y, 8, x_size)
            assert not SF.fused_tail_supported(crit, logits, y, 8)


# ------------------------------------------------------------------------------------------------ every device
def test_weighted_kernels_on_every_device():
    """Shapes whose weighted kernels need more than 48 KB of dynamic shared memory: the forward at zoom 1 and 2 with 150
    classes, the backward at zoom 8 with Wo = 793, weighted CE and weighted OHEM, from one thread per device; every
    device computes the bits of device 0."""
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
                out = []
                for zoom, logits, target, weight in inputs:
                    lg, t, wt = logits.to(dev), target.to(dev), weight.to(dev)
                    from semseg_b200 import ops
                    info, amax, lse = ops.upsample_ce_weighted_fwd(lg, t, 255, wt, 0.1, zoom=zoom)
                    dl = ops.upsample_ce_weighted_bwd(lg, t, 255, wt, 0.1, lse, info,
                                                      torch.tensor([1.0], device=dev), zoom=zoom)
                    o = ops.upsample_ce_ohem_fwd(lg, t, 255, 0.5, 1000, zoom=zoom, weight=wt)
                    dlo = ops.upsample_ce_ohem_bwd(lg, t, 255, o[2], o[3], o[5], o[0], torch.tensor([1.0], device=dev),
                                                   zoom=zoom, weight=wt)
                    out.append(tuple(v.cpu() for v in (info, amax, lse, dl, o[0], o[4], dlo)))
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


# ------------------------------------------------------------------------------------------------ networks
class _ATenCE(nn.CrossEntropyLoss):
    """nn.CrossEntropyLoss under another type: the network keeps the ATen tail (interpolate -> criterion -> max)."""


@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_weighted_tail_matches_aten_tail(arch, zoom, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    weight = _weights(21, 4, zero_class=False)
    native.criterion = nn.CrossEntropyLoss(weight=weight, ignore_index=255, label_smoothing=0.1)
    aten = copy.deepcopy(native)
    aten.criterion = _ATenCE(weight=weight.clone(), ignore_index=255, label_smoothing=0.1)
    x, y = _batch(zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    with precision.mode("bf16x3"):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert pred.shape == pred_r.shape == y.shape
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01          # argmax: equal but at top-1 / top-2 ties
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
def _graphed_vs_eager(base, batches, n_steps, monkeypatch):
    from semseg_b200 import graphs
    eager = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, n_steps)
    graphed = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, n_steps)
    assert graphs.launches_per_step(graphed) > 100
    assert le == lg, (le, lg)
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert torch.equal(pe, pg), k
        assert (pe.grad is None) == (pg.grad is None) and (pe.grad is None or torch.equal(pe.grad, pg.grad)), k
    return eager, graphed


def _n_graphs(model):
    return sum(1 for s in model._sb_graph_steps.values() if s.fwd is not None)


def test_graphed_weighted_ce_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    base.criterion = nn.CrossEntropyLoss(weight=_weights(21, 2), ignore_index=255, label_smoothing=0.1)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = _graphed_vs_eager(base, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 1
    # an in-place edit of the weights needs no capture: the next replay reads the new values
    for m in (eager, graphed):
        with torch.no_grad():
            m.criterion.weight.mul_(torch.linspace(0.5, 1.5, 21, device="cuda"))
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, 2)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, 2)
    assert le == lg, (le, lg)
    assert _n_graphs(graphed) == 1
    # a new label_smoothing and a replaced weight tensor each capture anew, never replay the old graph
    for change in (lambda m: setattr(m.criterion, "label_smoothing", 0.2),
                   lambda m: setattr(m.criterion, "weight", _weights(21, 9))):
        for m in (eager, graphed):
            change(m)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
        le = _sgd_steps(eager, batches, n_steps)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
        lg = _sgd_steps(graphed, batches, n_steps)
        assert le == lg, (le, lg)
    assert _n_graphs(graphed) == 3


def test_graphed_weighted_ohem_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import OhemCrossEntropyLoss
    base = _build("psp", 8).cuda().train()
    base.criterion = OhemCrossEntropyLoss(ignore_index=255, thresh=0.05, min_kept=100, weight=_weights(21, 6))
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    _graphed_vs_eager(base, batches, graphs.WARMUP_CALLS + 4, monkeypatch)


@pytest.mark.parametrize("crit", ["ce", "ohem"])
def test_graphed_weighted_step_launches_no_aten_tail(crit):
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import OhemCrossEntropyLoss
    model = _build("psp", 8).cuda().train()
    w = _weights(21, 1)
    model.criterion = (nn.CrossEntropyLoss(weight=w, ignore_index=255, label_smoothing=0.1) if crit == "ce" else
                       OhemCrossEntropyLoss(thresh=0.05, min_kept=3000, weight=w))
    x, y = _batch(8)
    for _ in range(graphs.WARMUP_CALLS + 2):
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
    torch.cuda.synchronize()
    assert graphs.launches_per_step(model) > 100
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    bad = [n for n in names if any(k in n for k in ("upsample_bilinear2d", "_log_softmax", "log_softmax", "LogSoftMax",
                                                    "nll_loss", "aten::sort"))]
    assert not bad, sorted(set(bad))


# ------------------------------------------------------------------------------------------------ module path
def test_weighted_ohem_module_path_matches_oracle():
    """OhemCrossEntropyLoss(weight=w)(eval_model(x), y) as validate() calls it, and its gradient."""
    from semseg_b200.losses import OhemCrossEntropyLoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    w = _weights(21, 2)
    for crit in (OhemCrossEntropyLoss(weight=w), OhemCrossEntropyLoss(thresh=0.5, min_kept=2000, weight=w)):
        loss = crit(out, y)
        ref, _, _, _ = weighted_ohem_ce(out, y, w, crit.ignore_index, crit.thresh, crit.min_kept)
        assert abs(loss.item() - ref.item()) <= 2e-5 * abs(ref.item())
    lg = out.detach().clone().requires_grad_(True)
    crit = OhemCrossEntropyLoss(thresh=0.6, min_kept=3000, weight=w)
    (g,) = torch.autograd.grad(crit(lg, y), lg)
    lr = out.detach().clone().requires_grad_(True)
    _, kept, _, _ = weighted_ohem_ce(lr.detach(), y, w, 255, crit.thresh, crit.min_kept)
    (g_ref,) = torch.autograd.grad(weighted_ohem_ce(lr, y, w, 255, crit.thresh, crit.min_kept, kept=kept)[0], lr)
    assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
    with pytest.raises(ValueError, match="weight"):
        OhemCrossEntropyLoss(weight=torch.ones(19, device="cuda"))(out, y)
