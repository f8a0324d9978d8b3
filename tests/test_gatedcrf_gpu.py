"""GPU tier: the Gated CRF loss (losses.GatedCRFLoss) on the fused tail: the plain cross-entropy kernels plus the
csrc/crf.cu stencil, graphed.

  * kernel vs the float64 contract of tests/gatedcrf_oracle.py at zoom 1, 2, 4, 8 and both `at`, radius 1 / 5 / 8,
    2 / 19 / 21 / 150 / 256 classes, grids that end mid-tile and grids narrower than the window, a padded pitch; the
    worst errors are printed next to their gates;
  * reruns are bit-identical, the argmax and the CE term are the plain tail's bits, and both passes capture into a CUDA
    graph (no host synchronisation) whose replay gives the eager bits;
  * PSPNet50 / PSANet50 with batch-statistics and frozen BatchNorm at every zoom: the native tail against the ATen
    tail on a scribble-like target; graphed steps are bit-identical to eager ones and a changed option captures anew;
    crf_weight = 0 is the nn.CrossEntropyLoss step bit for bit; x.grad holds the network path only;
  * the module path against the oracle."""
import copy

import pytest
import torch

from tests import util
from tests.gatedcrf_oracle import crf_contract, grid_rgb, upsample
from tests.test_zoom_gpu import _batch, _build, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
LOSS_GATE, GRAD_GATE = 1e-5, 1e-4      # relative loss, dlogits over max |dlogits|
_worst = {"loss": 0.0, "grad": 0.0}


def _image(n, h, w, seed, stride):
    """A normalised input batch [n, 3, 8(h-1)+1, 8(w-1)+1] with smooth regions and edges, as the networks see it."""
    g = torch.Generator(device="cuda").manual_seed(seed + 5)
    H, W = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    base = torch.randn((n, 3, 4, 4), device="cuda", generator=g)
    x = torch.nn.functional.interpolate(base, size=(H, W), mode="nearest")
    return (x + 0.05 * torch.randn((n, 3, H, W), device="cuda", generator=g)).contiguous()


def _oracle(logits, target, x, zoom, at, crit, stride=None):
    """float64: (loss, dloss/dlogits NHWC) of ce_weight CE + crf_weight CRF on the tail."""
    s8 = logits.detach().double().permute(0, 3, 1, 2).requires_grad_(True)
    up = upsample(s8, zoom)
    C = up.shape[1]
    valid = (target != crit.ignore_index) & (target >= 0) & (target < C)
    nll = -torch.log_softmax(up, 1).gather(1, target.clamp(0, C - 1).unsqueeze(1)).squeeze(1)
    ce = (nll * valid).sum() / max(int(valid.sum()), 1)
    grid, default_stride = (up, 8 // zoom) if at == "output" else (s8, 8)
    rgb = grid_rgb(x, default_stride if stride is None else stride, crit.mean, crit.std)
    crf, g, _ = crf_contract(grid.detach(), rgb, crit.radius, crit.sigma_xy, crit.sigma_rgb)
    surrogate = crit.ce_weight * ce + crit.crf_weight * (grid * g).sum()
    (dl,) = torch.autograd.grad(surrogate, s8)
    return float(crit.ce_weight * ce + crit.crf_weight * crf), dl.permute(0, 2, 3, 1)


def _native(logits, target, x, zoom, crit, grad=0.7):
    from semseg_b200 import functional as SF
    lv = logits.detach().requires_grad_(True)
    loss, amax = SF.upsample_ce(lv, target, crit.ignore_index, zoom, criterion=crit, image=x)
    loss.backward(torch.tensor(grad, device="cuda"))
    return loss.detach(), lv.grad, amax


def _check(logits, target, x, zoom, crit, label):
    loss, dl, _ = _native(logits, target, x, zoom, crit)
    ref, rdl = _oracle(logits, target, x, zoom, crit.at, crit)
    el = abs(loss.item() - ref) / abs(ref)
    eg = float((dl.double() - 0.7 * rdl).abs().max() / (0.7 * rdl).abs().max())
    _worst["loss"], _worst["grad"] = max(_worst["loss"], el), max(_worst["grad"], eg)
    print("%s: loss rel %.2e (gate %.0e, worst %.2e), dlogits %.2e of max (gate %.0e, worst %.2e)" %
          (label, el, LOSS_GATE, _worst["loss"], eg, GRAD_GATE, _worst["grad"]))
    assert el <= LOSS_GATE and eg <= GRAD_GATE, (label, el, eg)


def _crit(**kw):
    from semseg_b200.losses import GatedCRFLoss
    return GatedCRFLoss(**kw)


@pytest.mark.parametrize("at", ["output", "logits"])
@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("classes", [2, 21, 150])
@pytest.mark.parametrize("radius", [1, 5, 8])
def test_kernel_vs_oracle(radius, classes, zoom, at):
    n, h, w = 2, 5, 7                           # grids of 5x7 .. 33x49: every one ends mid-tile
    logits = _logits(n, h, w, classes, classes + (classes & 1), seed=radius + zoom)     # padded pitch when odd
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, classes, seed=3)
    x = _image(n, h, w, seed=zoom, stride=1)
    crit = _crit(radius=radius, crf_weight=0.5, ce_weight=1.0, sigma_xy=3.0 if radius < 5 else 6.0, at=at)
    _check(logits, target, x, zoom, crit, "r%d C%d Z%d %s" % (radius, classes, zoom, at))


@pytest.mark.parametrize("case", [(1, 19, 2, 3, 1, "output"), (2, 256, 9, 11, 2, "output"), (1, 256, 6, 5, 8, "logits"),
                                  (1, 19, 3, 2, 8, "output"), (2, 21, 2, 2, 1, "logits"), (1, 150, 21, 19, 4, "output")],
                         ids=["19-narrow", "256-z2", "256-logits", "19-z8-tiny", "21-2x2", "150-z4-two-tiles"])
def test_kernel_vs_oracle_edges(case):
    n, c, h, w, zoom, at = case
    logits = _logits(n, h, w, c, c, seed=c)
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=4)
    x = _image(n, h, w, seed=c, stride=1)
    for crit in (_crit(at=at), _crit(at=at, crf_weight=2.0, ce_weight=0.0, radius=3, sigma_rgb=0.3)):
        _check(logits, target, x, zoom, crit, "edge %s w%g" % (case, crit.crf_weight))


@pytest.mark.parametrize("zoom", ZOOMS)
def test_deterministic_plain_bits_and_graph_capture(zoom):
    from semseg_b200 import ops
    n, h, w, c = 2, 9, 13, 21
    logits = _logits(n, h, w, c, c, seed=1).contiguous()
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=2)
    x = _image(n, h, w, seed=3, stride=1)
    for at in ("output", "logits"):
        crit = _crit(at=at, crf_weight=0.3)
        l1, g1, a1 = _native(logits, target, x, zoom, crit)
        l2, g2, a2 = _native(logits, target, x, zoom, crit)
        assert torch.equal(l1, l2) and torch.equal(g1, g2) and torch.equal(a1, a2)
        info, amax, _ = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
        assert torch.equal(a1, amax)                                   # pred: the plain tail's argmax
        ce_only = _native(logits, target, x, zoom, _crit(at=at, crf_weight=0.0))[0]
        assert torch.equal(ce_only, info[0])                           # the CE term: the plain tail's bits
        # both passes in one CUDA graph: a host synchronisation inside either would fail the capture
        from semseg_b200 import functional as SF
        lv = logits.detach().clone().requires_grad_(True)
        gout = torch.tensor(0.7, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                lv.grad = None
                loss, _ = SF.upsample_ce(lv, target, 255, zoom, criterion=crit, image=x)
                loss.backward(gout)
        torch.cuda.current_stream().wait_stream(s)
        lv.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss, _ = SF.upsample_ce(lv, target, 255, zoom, criterion=crit, image=x)
            loss.backward(gout)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(loss, l1) and torch.equal(lv.grad, g1)


def test_constant_logits_zero_crf_gradient():
    n, h, w, c = 1, 6, 7, 21
    logits = torch.zeros((n, h, w, c), device="cuda")
    target = torch.full((n, 8 * (h - 1) + 1, 8 * (w - 1) + 1), 255, dtype=torch.int64, device="cuda")
    x = _image(n, h, w, seed=1, stride=1)
    loss, dl, _ = _native(logits, target, x, 8, _crit(crf_weight=1.0))
    # p = 1/C everywhere: G_c = K / C = S, so the gradient is 0 up to the fp32 rounding of p (1e-5 of its scale 2 g / P)
    P = target.numel()
    assert float(dl.abs().max()) < 1e-5 * 2 * 0.7 / P
    ref, _ = _oracle(logits, target, x, 8, "output", _crit(crf_weight=1.0))
    assert abs(loss.item() - ref) <= LOSS_GATE * ref


# ------------------------------------------------------------------------------------------------ networks
def _scribbles(y, seed):
    """~2 % of the pixels labelled, in short horizontal strokes, the rest ignore_label."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    keep = torch.rand((y.shape[0], y.shape[1], (y.shape[2] + 7) // 8), device="cuda", generator=g) < 0.02
    keep = keep.repeat_interleave(8, dim=2)[:, :, : y.shape[2]]
    out = torch.full_like(y, 255)
    out[keep] = y[keep]
    return out


class _SubclassCRF:
    """A GatedCRFLoss subclass: the fused gate refuses it, so the network runs its ATen tail."""

    @staticmethod
    def make(**kw):
        from semseg_b200.losses import GatedCRFLoss

        class _Aten(GatedCRFLoss):
            pass
        return _Aten(**kw)


def _freeze_bn(model):
    for m in model.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.eval()


@pytest.mark.parametrize("at", ["output", "logits"])
@pytest.mark.parametrize("bn", ["batch", "frozen"])
@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_tail_matches_aten_tail(arch, zoom, bn, at, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    if bn == "frozen":
        _freeze_bn(native)
    native.criterion = _crit(crf_weight=0.5, at=at)
    aten = copy.deepcopy(native)
    aten.criterion = _SubclassCRF.make(crf_weight=0.5, at=at)
    x, y = _batch(zoom)
    y = _scribbles(y, zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    with precision.mode("bf16x3"):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item()), (main.item(), main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01
    loose = {"layer0.7.bias": 3e-4}                               # as tests/test_zoom_gpu.py: a cancelling sum
    bad = []
    for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
        assert (pn.grad is None) == (pa.grad is None), k
        if pn.grad is not None:
            err = util.rel_l2(pn.grad, pa.grad)
            if err > loose.get(k, 1e-4):
                bad.append((k, err))
    assert not bad, bad


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
    for (k, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), k


def test_graphed_steps_bit_identical_to_eager_and_options_recapture(monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    base.criterion = _crit(crf_weight=0.5)
    batches = []
    for s in (1, 2):
        x, y = _batch(8, seed=s)
        batches.append((x, _scribbles(y, s)))
    n_steps = graphs.WARMUP_CALLS + 2
    # a fresh pair per option: a model keeps at most graphs.MAX_GRAPHS captured steps
    for attr, value in (("crf_weight", 0.2), ("radius", 3), ("sigma_xy", 2.0), ("sigma_rgb", 0.3), ("at", "logits"),
                        ("mean", (120.0, 110.0, 100.0)), ("std", (50.0, 60.0, 70.0))):
        eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
        _both(eager, graphed, batches, n_steps, monkeypatch)
        assert _n_graphs(graphed) == 1
        for m in (eager, graphed):
            setattr(m.criterion, attr, value)
        _both(eager, graphed, batches, n_steps, monkeypatch)
        assert _n_graphs(graphed) == 2, attr


@pytest.mark.parametrize("zoom", [2, 8])
def test_crf_weight_zero_is_the_cross_entropy_step(zoom, monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", zoom).cuda().train()
    batches = [_batch(zoom, seed=s) for s in (1, 2)]
    ce, crf = copy.deepcopy(base), copy.deepcopy(base)
    ce.criterion = torch.nn.CrossEntropyLoss(ignore_index=255)
    crf.criterion = _crit(crf_weight=0.0)
    for graph in ("0", "1"):
        monkeypatch.setenv("SEMSEG_B200_GRAPH", graph)
        lc = _sgd_steps(ce, batches, graphs.WARMUP_CALLS + 2)
        lr = _sgd_steps(crf, batches, graphs.WARMUP_CALLS + 2)
        assert lc == lr
        for (k, a), (_, b) in zip(ce.named_parameters(), crf.named_parameters()):
            assert torch.equal(a, b), k


def test_input_gradient_is_the_network_path_only(monkeypatch):
    """x.grad of CE + w CRF is x.grad of the CE step plus x.grad of the w CRF step (the image gate is a constant)."""
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    base = _build("psp", 8).cuda().train()
    x0, y = _batch(8)
    y = _scribbles(y, 3)
    grads = []
    for ce_w, crf_w in ((1.0, 0.5), (1.0, 0.0), (0.0, 0.5)):
        m = copy.deepcopy(base)
        m.criterion = _crit(ce_weight=ce_w, crf_weight=crf_w)
        x = x0.clone().requires_grad_(True)
        with precision.mode("bf16x3"):
            _, main, _ = m(x, y)
            main.backward()
        grads.append(x.grad.double())
    both, ce_only, crf_only = grads
    assert util.rel_l2(both, ce_only + crf_only) < 1e-4
    assert util.rel_l2(both, ce_only) > 1e-3                       # the CRF term does reach x through the network


def test_module_path_matches_oracle():
    """GatedCRFLoss(...)(logits, y, image) on the target grid, and without the image the plain mean CE."""
    import torch.nn.functional as F
    n, c, H, W = 2, 21, 41, 57
    g = torch.Generator(device="cuda").manual_seed(9)
    logits = (torch.randn((n, c, H, W), device="cuda", generator=g) * 2).requires_grad_(True)
    y = _scribbles(torch.randint(0, c, (n, H, W), device="cuda", generator=g), 1)
    img = torch.randn((n, 3, H, W), device="cuda", generator=g)
    for crit in (_crit(), _crit(crf_weight=1.0, ce_weight=0.0, radius=2, at="logits")):
        logits.grad = None
        loss = crit(logits, y, img)
        loss.backward()
        ref, rdl = _oracle(logits.detach().permute(0, 2, 3, 1), y, img, 1, crit.at,
                           type("C", (), {k: getattr(crit, k) for k in ("ignore_index", "ce_weight", "crf_weight",
                                                                         "radius", "sigma_xy", "sigma_rgb", "mean",
                                                                         "std")})(), stride=1)
        assert abs(loss.item() - ref) <= LOSS_GATE * abs(ref)
        rdl = rdl.permute(0, 3, 1, 2)
        assert float((logits.grad.double() - rdl).abs().max() / rdl.abs().max()) <= GRAD_GATE
    plain = _crit()(logits.detach(), y)
    ref = F.cross_entropy(logits.detach(), y, ignore_index=255)
    assert abs(plain.item() - ref.item()) <= 1e-5 * ref.item()
