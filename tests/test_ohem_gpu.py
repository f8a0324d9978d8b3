"""GPU tier: OHEM cross-entropy on the fused tail (csrc/tail.cu kOhem kernels, semseg_b200/losses.py).

  * kernel vs the float64 oracle of tests/ohem_oracle.py at zoom 1, 2, 4, 8, in four regimes (thresh binding, min_kept
    binding, min_kept >= n_v, min_kept = 0), with odd h != w, widths off the 128-column CTA, 19 / 21 / 150 classes, a
    padded pitch, ignored and out-of-range targets;
  * the device threshold is bit-equal to sorting the kernel's own p_t map; edge cases; determinism;
  * PSPNet50 / PSANet50 with the native OHEM tail against the same network on the ATen tail;
  * graphed OHEM steps are bit-identical to eager ones, re-captured when thresh changes, and launch no ATen kernel;
  * the module path OhemCrossEntropyLoss()(eval_model(x), y) (validate(), tool/train.py:362) against the oracle."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.ohem_oracle import ohem_ce
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24"]
# (thresh, min_kept as a fraction of the pixels, which bound gives thr)
REGIMES = {"thresh": (0.7, 0.001, "thresh"), "min_kept": (0.0, 0.5, "kth"), "min_kept_ge_nv": (0.3, 10.0, "kth"),
           "min_kept_0": (0.3, 0.0, "thresh")}


def _upsampled(logits, zoom):
    """fp32 NHWC [N,h,w,C] -> the fp32 NCHW logits the fused tail scores (ATen's align_corners upsample)."""
    n, h, w, _ = logits.shape
    x = logits.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    return x


def _run(logits, target, zoom, thresh, min_kept, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse, pt, nll, thr = ops.upsample_ce_ohem_fwd(logits, target, 255, thresh, min_kept, zoom=zoom)
    dl = ops.upsample_ce_ohem_bwd(logits, target, 255, lse, pt, thr, info, torch.tensor([grad], device="cuda"),
                                  zoom=zoom)
    return info, amax, pt, nll, thr, dl


@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_ohem_kernel_vs_oracle(zoom, shape, regime):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    thresh, frac, bound = REGIMES[regime]
    min_kept = int(frac * n * ho * wo)
    logits = _logits(n, h, w, c, pitch, seed=zoom + 10)
    target = _target(n, ho, wo, c, seed=zoom + 10)
    info, amax, pt, nll, thr, dl = _run(logits, target, zoom, thresh, min_kept)

    lr = logits.detach().clone().requires_grad_(True)
    x = _upsampled(lr, zoom)
    _, kept_o, thr_o, pt_o = ohem_ce(x.detach(), target, 255, thresh, min_kept)
    valid = (target != 255) & (target >= 0) & (target < c)
    assert torch.equal(pt >= 0, valid)                                  # sentinel exactly on the non-valid pixels
    assert float((pt[valid].double() - pt_o[valid]).abs().max()) <= 3e-6
    thr_k = float(thr)
    thresh32 = torch.tensor(thresh, dtype=torch.float32).item()
    assert (thr_k == thresh32) == (bound == "thresh"), (thr_k, thresh)  # the regime is the one named
    assert abs(thr_k - thr_o) <= 3e-6
    kept_k = valid & (pt < thr)
    differ = kept_k != kept_o
    assert bool(((pt_o[differ] - thr_o).abs() < 1e-5).all()), "kept sets differ away from the threshold"
    assert int(info[1]) == int(kept_k.sum()) > 0
    # loss and gradient against the oracle on the kernel's kept set (equal to the oracle's but at threshold ties)
    loss_o, _, _, _ = ohem_ce(x, target, 255, thresh, min_kept, kept=kept_k)
    (dl_o,) = torch.autograd.grad(loss_o * 0.7, lr)
    assert abs(info[0].item() - loss_o.item()) <= 1e-5 * abs(loss_o.item())
    assert float((dl.double() - dl_o).abs().max()) <= 1e-5 * float(dl_o.abs().max())
    clear = _clear_of_ties(x.detach())
    assert torch.equal(amax[clear], x.detach().argmax(1)[clear])        # argmax covers every pixel


@pytest.mark.parametrize("zoom", ZOOMS)
def test_ohem_threshold_is_the_exact_kth(zoom):
    """thr == max(thresh, sort(kernel p_t over the valid pixels)[min(min_kept, n_v - 1)]), bit for bit."""
    n, h, w, c, pitch = 2, 9, 13, 21, 24
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    for thresh, min_kept in ((0.0, 0), (0.0, 1), (0.0, 37), (0.0, n * ho * wo // 3), (0.0, 10 ** 9), (0.5, 5),
                             (1.0, 5)):
        info, _, pt, nll, thr, _ = _run(logits, target, zoom, thresh, min_kept)
        vals = pt[pt >= 0].sort().values
        kth = vals[min(min_kept, vals.numel() - 1)]
        assert torch.equal(thr, torch.maximum(kth, torch.tensor(thresh, device="cuda")).view(1)), (thresh, min_kept)
        kept = (pt >= 0) & (pt < thr)
        assert info[1].item() == float(kept.sum())
        ref = nll[kept].double().sum() / max(int(kept.sum()), 1)
        assert abs(info[0].item() - ref.item()) <= 1e-6 * max(abs(ref.item()), 1e-30)


@pytest.mark.parametrize("zoom", ZOOMS)
def test_ohem_nothing_valid_or_kept(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    # every pixel ignored
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    info, _, pt, _, thr, dl = _run(logits, target, zoom, 0.7, 1000)
    assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0 and bool((pt == -1).all())
    assert thr.item() == pytest.approx(0.7)
    # thresh 0 and min_kept 0: thr is the smallest p_t, nothing lies strictly below it
    target = _target(n, ho, wo, c, seed=3)
    info, _, pt, _, thr, dl = _run(logits, target, zoom, 0.0, 0)
    assert thr.item() == pt[pt >= 0].min().item()
    assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0


@pytest.mark.parametrize("zoom", ZOOMS)
def test_ohem_exact_ties_follow_strict_less(zoom):
    """Constant logits: every valid p_t is the same value (~1/C). A min_kept bound at that value keeps nothing; thresh 1
    keeps every valid pixel and the loss is log(C)."""
    n, h, w, c = 1, 9, 7, 19
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = torch.zeros((n, h, w, c), device="cuda")
    target = _target(n, ho, wo, c, seed=5)
    info, _, pt, _, thr, dl = _run(logits, target, zoom, 0.0, 10)
    p = pt[pt >= 0]
    assert bool((p == p[0]).all()) and abs(p[0].item() - 1 / c) < 1e-6 and thr.item() == p[0].item()
    assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0
    info, _, pt, _, thr, dl = _run(logits, target, zoom, 1.0, 10)
    assert thr.item() == 1.0 and info[1].item() == float((pt >= 0).sum())
    assert abs(info[0].item() - torch.log(torch.tensor(float(c))).item()) < 1e-5


@pytest.mark.parametrize("zoom", [1, 8])
def test_ohem_deterministic(zoom):
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    a = _run(logits, target, zoom, 0.2, n * ho * wo // 4)
    b = _run(logits, target, zoom, 0.2, n * ho * wo // 4)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------------ networks
def _ohem(**kw):
    from semseg_b200.losses import OhemCrossEntropyLoss
    # p_t is near 1/21 in a fresh 21-class network: thresh 0.05 splits the pixels
    return OhemCrossEntropyLoss(**dict(dict(ignore_index=255, thresh=0.05, min_kept=3000), **kw))


def _aten_ohem(**kw):
    from semseg_b200.losses import OhemCrossEntropyLoss

    class ATenOhem(OhemCrossEntropyLoss):
        """OhemCrossEntropyLoss under another type: the network keeps the ATen tail (interpolate -> criterion -> max)."""
    c = _ohem(**kw)
    return ATenOhem(c.ignore_index, c.thresh, c.min_kept)


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_ohem_matches_aten_tail(arch, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, 8).cuda().train()
    native.criterion = _ohem()
    aten = copy.deepcopy(native)
    aten.criterion = _aten_ohem()
    x, y = _batch(8)
    assert SF.fused_tail_supported(native.criterion, None, y, 8, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, 8, x.size())
    with precision.mode(mode):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01          # argmax: equal but at top-1 / top-2 ties
    if mode == "bf16x3":
        loose = {"layer0.7.bias": 3e-4}                           # as tests/test_zoom_gpu.py: a cancelling sum
        bad = []
        for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
            assert (pn.grad is None) == (pa.grad is None), k
            if pn.grad is not None:
                err = util.rel_l2(pn.grad, pa.grad)
                if err > loose.get(k, 1e-4):
                    bad.append((k, err))
        assert not bad, bad


def test_graphed_ohem_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    base.criterion = _ohem(thresh=0.05, min_kept=100)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
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
    # a new thresh must never replay the graph captured with the old one
    for m in (eager, graphed):
        m.criterion.thresh = 0.04
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le2 = _sgd_steps(eager, batches, n_steps)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg2 = _sgd_steps(graphed, batches, n_steps)
    assert le2 == lg2, (le2, lg2)
    assert sum(1 for s in graphed._sb_graph_steps.values() if s.fwd is not None) == 2


def test_graphed_ohem_step_launches_no_aten_tail():
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    model = _build("psp", 8).cuda().train()
    model.criterion = _ohem()
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
    bad = [n for n in names if any(k in n for k in ("aten::sort", "aten::topk", "aten::kthvalue", "_softmax",
                                                    "upsample_bilinear2d", "nll_loss"))]
    assert not bad, sorted(set(bad))


def test_module_path_matches_oracle():
    """OhemCrossEntropyLoss()(eval_model(x), y) as validate() calls it (tool/train.py:362), and its gradient."""
    from semseg_b200.losses import OhemCrossEntropyLoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    for crit in (OhemCrossEntropyLoss(), OhemCrossEntropyLoss(thresh=0.5, min_kept=2000)):
        loss = crit(out, y)
        ref, _, _, _ = ohem_ce(out, y, crit.ignore_index, crit.thresh, crit.min_kept)
        assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    lg = out.detach().clone().requires_grad_(True)
    crit = OhemCrossEntropyLoss(thresh=0.6, min_kept=3000)
    (g,) = torch.autograd.grad(crit(lg, y), lg)
    lr = out.detach().clone().requires_grad_(True)
    _, kept, _, pt = ohem_ce(lr.detach(), y, 255, crit.thresh, crit.min_kept)
    (g_ref,) = torch.autograd.grad(ohem_ce(lr, y, 255, crit.thresh, crit.min_kept, kept=kept)[0], lr)
    assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
