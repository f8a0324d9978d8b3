"""GPU tier: boundary label relaxation on the fused tail (csrc/tail.cu relaxation kernels through
semseg_b200/functional.py).

  * kernel vs the float64 oracle of tests/relax_oracle.py at zoom 1, 2, 4, 8, with odd h != w, widths off and across
    the 128-column CTA, 19 / 21 / 150 / 256 classes, a padded pitch, border 1 - 4, weight None / random with a zero
    class, ignored and out-of-range targets, on blocky targets (interior and boundary pixels) and on a checkerboard
    (every pixel on a boundary, |S| at its maximum);
  * lse and argmax are the plain forward's bits, repeated runs give the same bits;
  * a single-label target is cross-entropy, an all-ignored batch is 0, a window that covers every class gives a loss
    and a gradient of exactly 0;
  * the widest supported target and one column past it; border 0 steps are the cross-entropy steps bit for bit;
  * PSPNet50 / PSANet50 on the native tail against the same loss written in PyTorch on the ATen tail;
  * graphed steps are bit-identical to eager ones, re-captured for a new border, and launch no ATen tail kernel;
  * the module path BoundaryRelaxationLoss(...)(eval_logits, y) against the oracle."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.relax_oracle import relax_loss, relax_sets, relax_tail
from tests.test_ohem_gpu import _upsampled
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
BORDERS = [1, 2, 3, 4]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24), (1, 7, 10, 256, 256)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24", "7x10-256"]


def _weights(c, seed, zero_class=True):
    """Seeded positive class weights in [0.25, 2.25), one class weighted 0."""
    g = torch.Generator(device="cuda").manual_seed(seed + 100)
    w = torch.rand(c, device="cuda", generator=g) * 2 + 0.25
    if zero_class:
        w[seed % c] = 0.0
    return w


def _blocky_target(n, ho, wo, c, seed, block=6):
    """Labels constant on block x block tiles (interior pixels and boundaries between tiles), ~5 % ignored pixels in
    small clumps and a few out-of-range labels."""
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    hb, wb = -(-ho // block), -(-wo // block)
    t = torch.randint(0, c, (n, hb, wb), device="cuda", generator=g)
    t = t.repeat_interleave(block, 1).repeat_interleave(block, 2)[:, :ho, :wo].contiguous()
    ign = torch.rand((n, hb * 3, wb * 3), device="cuda", generator=g) < 0.05
    ign = ign.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :ho, :wo]
    t[ign] = 255
    odd = torch.rand((n, ho, wo), device="cuda", generator=g) < 0.003
    t[odd] = torch.where(torch.rand((n, ho, wo), device="cuda", generator=g)[odd] < 0.5, c + 3, -2)
    return t


def _checkerboard(n, ho, wo, c, border):
    """Every pixel on a boundary: each window of the given border holds (2 border + 1)^2 distinct labels (C allowing)."""
    k = 2 * border + 1
    yy = torch.arange(ho, device="cuda").view(1, ho, 1)
    xx = torch.arange(wo, device="cuda").view(1, 1, wo)
    return (((yy % k) * k + (xx % k)) % c).expand(n, ho, wo).contiguous()


def _run(logits, target, zoom, border, weight=None, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse, sets, lq = ops.upsample_ce_relax_fwd(logits, target, 255, weight, border, zoom=zoom)
    dl = ops.upsample_ce_relax_bwd(logits, lse, sets, lq, info, torch.tensor([grad], device="cuda"), zoom=zoom)
    return info, amax, lse, lq, dl


def _check(logits, target, zoom, border, weight, loss_tol=2e-6, grad_tol=5e-6):
    info, amax, lse, lq, dl = _run(logits, target, zoom, border, weight)
    loss_o, d, dl_o = relax_tail(logits, target, zoom, border, weight)
    assert abs(info[1].item() - d) <= 1e-5 * max(d, 1.0)
    assert abs(info[0].item() - loss_o.item()) <= loss_tol * abs(loss_o.item())
    scale = float(0.7 * dl_o.abs().max())
    assert float((dl.double() - 0.7 * dl_o).abs().max()) <= grad_tol * scale
    return info, amax, lse, dl


@pytest.mark.parametrize("weighted", [False, True], ids=["no-weight", "weight"])
@pytest.mark.parametrize("border", BORDERS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_relax_kernel_vs_oracle(zoom, shape, border, weighted):
    from semseg_b200 import ops
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 20)
    weight = _weights(c, zoom + border) if weighted else None
    # measured on an H100 over this grid (both targets): loss 1.6e-7 relative, D 2.6e-7 relative, dlogits 1.7e-6 of
    # max |dlogits|
    for target in (_blocky_target(n, ho, wo, c, seed=zoom + border), _checkerboard(n, ho, wo, c, border)):
        _, amax, lse, _ = _check(logits, target, zoom, border, weight)
        # lse and argmax are the plain forward's bits
        _, amax_p, lse_p = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
        assert torch.equal(lse, lse_p) and torch.equal(amax, amax_p)
    x = _upsampled(logits, zoom)
    clear = _clear_of_ties(x)
    assert torch.equal(amax[clear], x.argmax(1)[clear])


@pytest.mark.parametrize("zoom", ZOOMS)
def test_relax_checkerboard_reaches_the_largest_set(zoom):
    n, h, w, c = 1, 9, 13, 150
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    for border in BORDERS:
        t = _checkerboard(n, ho, wo, c, border)
        _, s = relax_sets(t, c, border)
        interior = s[:, :, border:ho - border, border:wo - border].sum(1)
        assert int(interior.min()) == int(interior.max()) == min(c, (2 * border + 1) ** 2)


@pytest.mark.parametrize("zoom", ZOOMS)
def test_relax_single_label_is_cross_entropy(zoom):
    from semseg_b200 import ops
    n, h, w, c, pitch = 2, 9, 13, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 40)
    target = torch.full((n, ho, wo), 7, dtype=torch.int64, device="cuda")
    target[:, ::5, ::3] = 255
    g = torch.tensor([0.7], device="cuda")
    for weight in (None, _weights(c, 2, zero_class=False)):
        if weight is None:
            info_p, amax_p, lse_p = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
            dl_p = ops.upsample_ce_bwd(logits, target, 255, lse_p, info_p, g, zoom=zoom)
        else:
            info_p, amax_p, lse_p = ops.upsample_ce_weighted_fwd(logits, target, 255, weight, 0.0, zoom=zoom)
            dl_p = ops.upsample_ce_weighted_bwd(logits, target, 255, weight, 0.0, lse_p, info_p, g, zoom=zoom)
        for border in (1, 4):
            info, amax, lse, _, dl = _run(logits, target, zoom, border, weight)
            assert torch.equal(lse, lse_p) and torch.equal(amax, amax_p)
            assert abs(info[1].item() - info_p[1].item()) <= 1e-6 * info_p[1].item()
            assert abs(info[0].item() - info_p[0].item()) <= 1e-6 * abs(info_p[0].item())
            # measured on an H100: 1.6e-6 of max |dlogits| (zoom 1, weighted). The plain kernel rounds p_t - 1 near
            # p_t = 1, this one forms -p_t R / (1 - R)
            assert float((dl - dl_p).abs().max()) <= 5e-6 * float(dl_p.abs().max())


@pytest.mark.parametrize("zoom", ZOOMS)
def test_relax_nothing_to_train_gives_zero(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    target[:, ::3] = c
    target[:, 1::3] = -1
    for weight in (None, _weights(c, 1)):
        for border in BORDERS:
            info, _, _, _, dl = _run(logits, target, zoom, border, weight)
            assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0


@pytest.mark.parametrize("zoom", ZOOMS)
def test_relax_window_covering_every_class_is_exactly_zero(zoom):
    n, h, w, c = 1, 6, 9, 4
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=zoom)
    yy = torch.arange(ho, device="cuda").view(1, ho, 1)
    xx = torch.arange(wo, device="cuda").view(1, 1, wo)
    target = ((yy % 2) * 2 + (xx % 2)).expand(n, ho, wo).contiguous()       # every 3x3 window holds all 4 classes
    for weight in (None, _weights(c, 1, zero_class=False)):
        info, _, _, lq, dl = _run(logits, target, zoom, 1, weight)
        assert info[0].item() == 0.0 and info[1].item() > 0
        assert float(dl.abs().max()) == 0.0 and bool(torch.isinf(lq).all())


def test_relax_saturated_sets_keep_relative_accuracy():
    """Two classes hold nearly all the mass and every set holds both: the losses are ~1e-9 and keep their digits."""
    n, h, w, c, zoom = 1, 9, 13, 21, 8
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    g = torch.Generator(device="cuda").manual_seed(5)
    logits = torch.randn((n, h, w, c), device="cuda", generator=g).clamp_(-3, 3)
    logits[..., 0] = 20.0 + torch.rand((n, h, w), device="cuda", generator=g)
    logits[..., 1] = 20.0 + torch.rand((n, h, w), device="cuda", generator=g)
    xx = torch.arange(wo, device="cuda").view(1, 1, wo)
    target = (xx % 2).expand(n, ho, wo).contiguous()
    info, _, _, _, dl = _run(logits, target, zoom, 1)
    loss_o, _, dl_o = relax_tail(logits, target, zoom, 1)
    assert 0 < loss_o.item() < 1e-6
    assert abs(info[0].item() - loss_o.item()) <= 1e-4 * loss_o.item()
    assert float((dl.double() - 0.7 * dl_o).abs().max()) <= 1e-4 * float(0.7 * dl_o.abs().max())


@pytest.mark.parametrize("zoom", [1, 8])
def test_relax_deterministic(zoom):
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _blocky_target(n, ho, wo, c, seed=zoom)
    weight = _weights(c, zoom)
    for u, v in zip(_run(logits, target, zoom, 2, weight), _run(logits, target, zoom, 2, weight)):
        assert torch.equal(u, v)


def test_relax_widest_target_and_one_past_it():
    """Wo = 2389 at zoom 8 is the widest target the rows kernel stages; one logit column more (Wo = 2397) flips
    fused_tail_supported and the module path, on the NCHW logits, still runs (the zoom-1 kernels' limit is wider)."""
    from semseg_b200 import functional as SF
    from semseg_b200.losses import BoundaryRelaxationLoss
    c, zoom = 19, 8
    w_max = (224 * 1024 // (12 * zoom) - 1) // zoom + 1
    crit = BoundaryRelaxationLoss(border=2)
    for w, ok in ((w_max, True), (w_max + 1, False)):
        h = 3
        ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
        logits = _logits(1, h, w, c, c, seed=w)
        target = _blocky_target(1, ho, wo, c, seed=w)
        assert SF.fused_tail_supported(crit, logits, target, zoom) == ok
        if ok:
            _check(logits, target, zoom, 2, None)
        x = _upsampled(logits, zoom).contiguous()
        loss = crit(x, target)
        ref, _, _ = relax_loss(x, target, 2)
        assert abs(loss.item() - ref.item()) <= 2e-6 * abs(ref.item())


# ------------------------------------------------------------------------------------------------ networks
def _torch_relax(logits, target, border, weight, ignore_index):
    """The loss in PyTorch with a multi-hot [N, C, H, W] target, the way one writes it without the fused tail."""
    c = logits.shape[1]
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    t = torch.where(valid, target, torch.zeros_like(target))
    onehot = F.one_hot(t, c).permute(0, 3, 1, 2).float() * valid.unsqueeze(1)
    s = F.max_pool2d(onehot, 2 * border + 1, stride=1, padding=border) > 0
    pix = torch.logsumexp(logits, 1) - torch.logsumexp(logits.masked_fill(~s, float("-inf")), 1)
    w = torch.ones(c, device=logits.device) if weight is None else weight
    om = (s.float() * w.view(1, c, 1, 1)).sum(1) / s.sum(1).clamp(min=1)
    om = om * valid
    pix = torch.where(valid, pix, torch.zeros_like(pix))
    return (om * pix).sum() / om.sum().clamp(min=1e-30)


def _torch_relax_class():
    from semseg_b200.losses import BoundaryRelaxationLoss

    class _TorchRelax(BoundaryRelaxationLoss):
        """BoundaryRelaxationLoss in PyTorch under another type: the network keeps the ATen tail."""

        def forward(self, logits, target):
            return _torch_relax(logits, target, self.border, self.weight, self.ignore_index)

    return _TorchRelax


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_relax_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import BoundaryRelaxationLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    weight = _weights(21, 4, zero_class=False)
    native.criterion = BoundaryRelaxationLoss(border=2, weight=weight, ignore_index=255)
    aten = copy.deepcopy(native)
    aten.criterion = _torch_relax_class()(border=2, weight=weight.clone(), ignore_index=255)
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
    assert (pred != pred_r).float().mean().item() < 0.01
    assert native.criterion.weight.grad is None
    if mode != "bf16x3":
        return      # as tests/test_zoom_gpu.py: in bf16 the tails' ~1e-6 dlogits differences flip bf16 roundings
    loose = {"layer0.7.bias": 3e-4}
    bad = []
    for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
        assert (pn.grad is None) == (pa.grad is None), k
        if pn.grad is not None:
            err = util.rel_l2(pn.grad, pa.grad)
            if err > loose.get(k, 1e-4):
                bad.append((k, err))
    assert not bad, bad


def test_border_zero_steps_are_cross_entropy_steps(monkeypatch):
    from torch import nn
    from semseg_b200.losses import BoundaryRelaxationLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    batches = [_batch(8, seed=s) for s in (1, 2)]
    w = _weights(21, 3)
    for ce, relax in ((nn.CrossEntropyLoss(ignore_index=255), BoundaryRelaxationLoss(border=0)),
                      (nn.CrossEntropyLoss(weight=w, ignore_index=255), BoundaryRelaxationLoss(0, w.clone()))):
        a, b = _build("psp", 8).cuda().train(), _build("psp", 8).cuda().train()
        a.criterion, b.criterion = ce, relax
        assert _sgd_steps(a, batches, 3) == _sgd_steps(b, batches, 3)
        for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
            assert torch.equal(pa, pb), k


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


def test_graphed_relax_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import BoundaryRelaxationLoss
    base = _build("psp", 8).cuda().train()
    base.criterion = BoundaryRelaxationLoss(border=2, weight=_weights(21, 2), ignore_index=255)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    _both(eager, graphed, batches, n_steps, monkeypatch)
    assert graphs.launches_per_step(graphed) > 100 and _n_graphs(graphed) == 1
    for m in (eager, graphed):
        with torch.no_grad():
            m.criterion.weight.mul_(torch.linspace(0.5, 1.5, 21, device="cuda"))
    _both(eager, graphed, batches, 2, monkeypatch)
    assert _n_graphs(graphed) == 1
    # the published schedule lowers the border after some epochs: a new border captures anew
    for m in (eager, graphed):
        m.criterion.border = 1
    _both(eager, graphed, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 2


def test_graphed_relax_step_kernel_count_and_no_aten_tail():
    """A graphed relaxation step launches the default criterion's kernels plus one label-set pass per head, and none of
    ATen's upsample / log-softmax / nll / max-pool / logsumexp kernels."""
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import BoundaryRelaxationLoss
    x, y = _batch(8)
    counts = {}
    for name in ("ce", "relax"):
        model = _build("psp", 8).cuda().train()
        if name == "relax":
            model.criterion = BoundaryRelaxationLoss(border=1, weight=_weights(21, 1))
        for _ in range(graphs.WARMUP_CALLS + 2):
            _, ml, al = model(x, y)
            (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
        counts[name] = graphs.launches_per_step(model)
    assert counts["relax"] == counts["ce"] + 2 and counts["ce"] > 100, counts
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    bad = [n for n in names if any(k in n for k in ("upsample_bilinear2d", "_log_softmax", "log_softmax", "LogSoftMax",
                                                    "nll_loss", "max_pool", "logsumexp"))]
    assert not bad, sorted(set(bad))


# ------------------------------------------------------------------------------------------------ module path
def test_relax_module_path_matches_oracle():
    """BoundaryRelaxationLoss(...)(eval_model(x), y) as validate() calls it, and its gradient."""
    from semseg_b200.losses import BoundaryRelaxationLoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    w = _weights(21, 2)
    for crit in (BoundaryRelaxationLoss(), BoundaryRelaxationLoss(border=3, weight=w), BoundaryRelaxationLoss(0, w)):
        loss = crit(out, y)
        ref, _, g_ref = relax_loss(out, y, crit.border, crit.weight, crit.ignore_index)
        assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
        lg = out.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(crit(lg, y), lg)
        assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
    with pytest.raises(ValueError, match="weight"):
        BoundaryRelaxationLoss(weight=torch.ones(19, device="cuda"))(out, y)
