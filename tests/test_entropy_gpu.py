"""GPU tier: entropy minimisation plus cross-entropy on the fused tail (csrc/tail.cu entropy kernels through
semseg_b200/functional.py).

  * kernel vs the float64 oracle of tests/entropy_oracle.py at zoom 1, 2, 4, 8, with odd h != w, widths off and across
    the 128-column CTA, 19 / 21 / 150 / 256 classes, a padded pitch, mixed / all-unlabelled / all-labelled targets with
    out-of-range ones, and several (ent_weight, ce_weight);
  * ent_weight = 0 is the plain tail; constant logits give H = log C and a gradient of exactly 0; saturated logits stay
    finite with H >= 0; nothing to train gives 0; the kernels are deterministic;
  * PSPNet50 / PSANet50 at every zoom on the native entropy tail against the same loss written in PyTorch on the ATen
    tail;
  * graphed entropy steps are bit-identical to eager ones and re-captured for a new ent_weight or a toggled head dropout;
  * the module path EntropyLoss(...)(eval_logits, y) against the oracle."""
import copy
import math

import pytest
import torch

from tests import util
from tests.entropy_oracle import entropy_loss, entropy_tail
from tests.test_ohem_gpu import _upsampled
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24), (1, 7, 10, 256, 256)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24", "7x10-256"]
WEIGHTS = [(1.0, 1.0), (1.0, 0.0), (0.4, 2.5)]
WEIGHT_IDS = ["1-1", "ent-only", "0.4-2.5"]


def _target_kind(n, ho, wo, c, seed, kind):
    t = _target(n, ho, wo, c, seed)            # ~5 % ignored, a few out of range
    if kind == "mixed":
        g = torch.Generator(device="cuda").manual_seed(seed + 7)
        t[torch.rand((n, ho, wo), device="cuda", generator=g) < 0.4] = 255
    elif kind == "all-U":
        t.fill_(255)
    else:                                       # no unlabelled pixel; out-of-range ones stay
        t[t == 255] = c + 1
    return t


def _run(logits, target, zoom, ent_weight, ce_weight, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse, mu = ops.upsample_ce_entropy_fwd(logits, target, 255, zoom=zoom)
    dl = ops.upsample_ce_entropy_bwd(logits, target, 255, ent_weight, ce_weight, lse, mu, info,
                                     torch.tensor([grad], device="cuda"), zoom=zoom)
    loss = ce_weight * info[0].item() + ent_weight * info[2].item()
    return loss, info, amax, lse, mu, dl


@pytest.mark.parametrize("weights", WEIGHTS, ids=WEIGHT_IDS)
@pytest.mark.parametrize("kind", ["mixed", "all-U", "no-U"])
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_entropy_kernel_vs_oracle(zoom, shape, kind, weights):
    ent_w, ce_w = weights
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 20)
    target = _target_kind(n, ho, wo, c, zoom + 20, kind)
    loss, info, amax, _, mu, dl = _run(logits, target, zoom, ent_w, ce_w)
    loss_o, nl, nu, _, dl_o = entropy_tail(logits, target, zoom, ent_w, ce_w)
    assert (info[1].item(), info[3].item()) == (nl, nu) and info[4].item() == 0.0 and info[5].item() == 1.0
    if loss_o.item() == 0.0:                    # the only weighted term's set is empty
        assert loss == 0.0 and float(dl.abs().max()) == 0.0
        return
    # the focal tests' bars: loss 2e-6 relative, dlogits 5e-6 of max |dlogits|
    assert abs(loss - loss_o.item()) <= 2e-6 * abs(loss_o.item())
    assert float((dl.double() - 0.7 * dl_o).abs().max()) <= 5e-6 * float(0.7 * dl_o.abs().max())
    x = _upsampled(logits, zoom).double()
    mu_o = (torch.softmax(x, 1) * x).sum(1)
    assert float((mu.double() - mu_o).abs().max()) <= 2e-6 * max(1.0, float(x.abs().max()))
    clear = _clear_of_ties(x.float())
    assert torch.equal(amax[clear], x.argmax(1)[clear])


@pytest.mark.parametrize("zoom", ZOOMS)
def test_entropy_weight_zero_is_the_plain_tail(zoom):
    from semseg_b200 import ops
    n, h, w, c, pitch = 2, 9, 13, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 40)
    target = _target_kind(n, ho, wo, c, zoom + 40, "mixed")
    g = torch.tensor([0.7], device="cuda")
    info_p, amax_p, lse_p = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    dl_p = ops.upsample_ce_bwd(logits, target, 255, lse_p, info_p, g, zoom=zoom)
    loss, info, amax, lse, _, dl = _run(logits, target, zoom, 0.0, 1.0)
    assert torch.equal(lse, lse_p) and torch.equal(amax, amax_p) and info[1].item() == info_p[1].item()
    assert abs(loss - info_p[0].item()) <= 1e-6 * abs(info_p[0].item())
    assert float((dl - dl_p).abs().max()) <= 1e-6 * float(dl_p.abs().max())


@pytest.mark.parametrize("zoom", ZOOMS)
def test_entropy_constant_logits(zoom):
    n, h, w, c = 1, 5, 9, 19
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = torch.full((n, h, w, c), 1.25, device="cuda")
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    loss, info, _, _, mu, dl = _run(logits, target, zoom, 1.0, 1.0)
    assert abs(info[2].item() - math.log(c)) <= 2e-6 * math.log(c)
    assert bool((mu == 1.25).all()) and float(dl.abs().max()) == 0.0


@pytest.mark.parametrize("zoom", ZOOMS)
def test_entropy_saturated_logits(zoom):
    """Every pixel's top class is 20 to 1000 above the others: p of the others underflows in fp32."""
    n, h, w, c, k = 2, 9, 13, 21, 3
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    g = torch.Generator(device="cuda").manual_seed(zoom + 60)
    logits = torch.randn((n, h, w, c), device="cuda", generator=g).clamp_(-3, 3)
    levels = torch.tensor([20.0, 40.0, 120.0, 1000.0], device="cuda")
    logits[..., k] = levels[torch.randint(0, 4, (n, h, w), device="cuda", generator=g)]
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    loss, info, _, lse, mu, dl = _run(logits, target, zoom, 1.0, 0.0)
    for t in (info, lse, mu, dl):
        assert bool(torch.isfinite(t).all())
    loss_o, _, _, ent_o, dl_o = entropy_tail(logits, target, zoom, 1.0, 0.0)
    assert loss >= 0.0 and abs(loss - loss_o.item()) <= 1e-3 * loss_o.item() + 1e-7
    # one unlabelled pixel: the loss is that pixel's H, never negative, at every saturation level
    for level in (20.0, 120.0, 1000.0):
        one = torch.full((1, h, w, c), -2.0, device="cuda")
        one[..., k] = level
        t1 = torch.zeros((1, ho, wo), dtype=torch.int64, device="cuda")
        t1[0, 0, 0] = 255
        loss1, info1, _, _, _, dl1 = _run(one, t1, zoom, 1.0, 0.0)
        assert info1[2].item() >= 0.0 and math.isfinite(info1[2].item()) and bool(torch.isfinite(dl1).all())


@pytest.mark.parametrize("zoom", ZOOMS)
def test_entropy_nothing_to_train_gives_zero(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    target = torch.full((n, ho, wo), c, dtype=torch.int64, device="cuda")    # every pixel out of range
    target[:, 1::3] = -1
    loss, info, _, _, _, dl = _run(logits, target, zoom, 1.0, 1.0)
    assert info.tolist() == [0.0, 0.0, 0.0, 0.0, 0.0, 1.0] and loss == 0.0 and float(dl.abs().max()) == 0.0
    # both weights 0 on an ordinary target: loss 0, gradient exactly 0
    target = _target_kind(n, ho, wo, c, 3, "mixed")
    loss, _, _, _, _, dl = _run(logits, target, zoom, 0.0, 0.0)
    assert loss == 0.0 and float(dl.abs().max()) == 0.0


@pytest.mark.parametrize("zoom", [1, 8])
def test_entropy_deterministic(zoom):
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target_kind(n, ho, wo, c, zoom, "mixed")
    a, b = _run(logits, target, zoom, 0.7, 1.3), _run(logits, target, zoom, 0.7, 1.3)
    assert a[0] == b[0] and all(torch.equal(u, v) for u, v in zip(a[1:], b[1:]))


# ------------------------------------------------------------------------------------------------ networks
def _torch_entropy(logits, target, ent_weight, ce_weight, ignore_index):
    c = logits.shape[1]
    lab = (target != ignore_index) & (target >= 0) & (target < c)
    unl = target == ignore_index
    t = torch.where(lab, target, torch.zeros_like(target))
    logp = torch.log_softmax(logits, dim=1)
    ce = -logp.gather(1, t.unsqueeze(1)).squeeze(1)
    ent = -(logp.exp() * logp).sum(1)
    return (ce_weight * (ce * lab).sum() / lab.sum().clamp(min=1) +
            ent_weight * (ent * unl).sum() / unl.sum().clamp(min=1))


def _torch_entropy_class():
    from semseg_b200.losses import EntropyLoss

    class _TorchEntropy(EntropyLoss):
        """EntropyLoss written in PyTorch under another type: the network keeps the ATen tail (interpolate ->
        criterion)."""

        def forward(self, logits, target):
            return _torch_entropy(logits, target, self.ent_weight, self.ce_weight, self.ignore_index)

    return _TorchEntropy


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_entropy_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import EntropyLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    native.criterion = EntropyLoss(ignore_index=255, ent_weight=0.6, ce_weight=1.0)
    aten = copy.deepcopy(native)
    aten.criterion = _torch_entropy_class()(ignore_index=255, ent_weight=0.6, ce_weight=1.0)
    x, y = _batch(zoom)
    g = torch.Generator(device="cuda").manual_seed(zoom)
    y[torch.rand(y.shape, device="cuda", generator=g) < 0.5] = 255          # half the pixels unlabelled
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
    for (k, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), k


def test_graphed_entropy_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import EntropyLoss
    base = _build("psp", 8).cuda().train()          # dropout 0: eager and graphed steps draw no mask
    base.criterion = EntropyLoss(ignore_index=255, ent_weight=1.0, ce_weight=0.5)
    batches = []
    for s in (1, 2, 3):
        x, y = _batch(8, seed=s)
        y[:, : y.shape[1] // 2] = 255                   # the top half of every image unlabelled
        batches.append((x, y))
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    _both(eager, graphed, batches, n_steps, monkeypatch)
    assert graphs.launches_per_step(graphed) > 100 and _n_graphs(graphed) == 1
    # a new ent_weight captures anew, never replays the old graph
    for m in (eager, graphed):
        m.criterion.ent_weight = 0.25
    _both(eager, graphed, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 2
    # so does a head's Dropout2d switched to eval mode after a capture
    for m in (eager, graphed):
        m.cls[3].eval()
        m.aux[3].eval()
    _both(eager, graphed, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 3


def test_graphed_dropout_toggle_captures_anew_with_default_criterion(monkeypatch):
    """The capture key holds the Dropout2d modes: toggling a head's dropout after a capture never replays the stale
    graph (which would still draw the dropout mask)."""
    from semseg_b200 import graphs
    from semseg_b200.pspnet import PSPNet
    torch.manual_seed(0)
    base = PSPNet(layers=50, classes=21, zoom_factor=8, dropout=0.3, pretrained=False).cuda().train()
    batches = [_batch(8, seed=s) for s in (1, 2)]
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    for m in (eager, graphed):
        m.cls[3].eval()
        m.aux[3].eval()
    _both(eager, graphed, batches, graphs.WARMUP_CALLS + 2, monkeypatch)
    assert _n_graphs(graphed) == 1
    for m in (eager, graphed):
        m.cls[3].train()
    torch.manual_seed(5)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    x, y = batches[0]
    _sgd_steps(graphed, [(x, y)], graphs.WARMUP_CALLS + 1)
    assert _n_graphs(graphed) == 2


# ------------------------------------------------------------------------------------------------ module path
def test_entropy_module_path_matches_oracle():
    """EntropyLoss(...)(eval_model(x), y) as validate() calls it, and its gradient; aux_loss is the plain CE."""
    import torch.nn.functional as F
    from semseg_b200.losses import EntropyLoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    y[0, :20] = 255
    with torch.no_grad():
        out = model(x)
    for crit in (EntropyLoss(), EntropyLoss(ent_weight=0.3, ce_weight=0.0), EntropyLoss(ent_weight=0.0)):
        loss = crit(out, y)
        ref, _, _, _, g_ref = entropy_loss(out, y, crit.ent_weight, crit.ce_weight, crit.ignore_index)
        assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
        lg = out.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(crit(lg, y), lg)
        assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
    ce = F.cross_entropy(out, y, ignore_index=255)
    assert abs(EntropyLoss().aux_loss(out, y).item() - ce.item()) <= 1e-5 * ce.item()
