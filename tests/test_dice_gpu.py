"""GPU tier: the Dice (+ cross-entropy) loss on the fused tail (csrc/tail.cu Dice kernels through
semseg_b200/functional.py).

  * kernel vs the float64 oracle of tests/dice_oracle.py at zoom 1, 2, 4, 8, with odd h != w, widths off and across the
    128-column CTA, 19 / 21 / 150 / 256 classes, a padded pitch, ignored and out-of-range targets, an absent class,
    smooth 0 / 1 and ce_weight 0 / 1: the loss, the per-class (I_c, S_c, n_c) and dlogits;
  * a clamped denominator (an absent class with p = 0 everywhere and smooth 0, so S_c = 0);
  * no valid pixel gives loss 0 and a zero gradient; two runs are bit-identical; lse and pred are the plain tail's bits;
  * PSPNet50 / PSANet50 on the native Dice tail against a PyTorch Dice subclass on the ATen tail;
  * graphed Dice steps are bit-identical to eager ones, re-captured for a new smooth, and launch no ATen tail kernel;
  * the module path DiceLoss()(eval_logits, y) against the oracle;
  * the kernels that need the > 48 KB shared-memory opt-in run on every device."""
import copy

import pytest
import torch

from tests import util
from tests.dice_oracle import dice_ce, upsampled
from tests.test_weighted_ce_gpu import _graphed_vs_eager, _n_graphs
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24), (1, 7, 10, 256, 256)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24", "7x10-256"]
OPTIONS = [(0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (1.0, 1.0)]
OPTION_IDS = ["smooth0-ce0", "smooth1-ce0", "smooth0-ce1", "smooth1-ce1"]


def _run(logits, target, zoom, smooth, eps, ce_weight, grad=0.7):
    from semseg_b200 import ops
    info, amax, lse, table = ops.upsample_ce_dice_fwd(logits, target, 255, smooth, eps, ce_weight, zoom=zoom)
    dl = ops.upsample_ce_dice_bwd(logits, target, 255, lse, table, torch.tensor([grad], device="cuda"), zoom=zoom)
    return info, amax, lse, table, dl


def _absent(target, c):
    """Class c - 1 gets no pixel (its pixels become ignored)."""
    t = target.clone()
    t[t == c - 1] = 255
    return t


def _check_vs_oracle(logits, target, zoom, smooth, eps, ce_weight):
    """-> (loss rel. error, max I/S rel. error, dlogits error / max |dlogits|), asserting the gates."""
    c = logits.shape[-1]
    info, amax, _, table, dl = _run(logits, target, zoom, smooth, eps, ce_weight)
    lr = logits.detach().clone().requires_grad_(True)
    x = upsampled(lr, zoom)
    loss_o, inter_o, s_o, n_o = dice_ce(x, target, 255, smooth, eps, ce_weight)
    (dl_o,) = torch.autograd.grad(loss_o * 0.7, lr)
    tab = table.double()
    inter, s, n = tab[2 * c:3 * c], tab[3 * c:4 * c], tab[4 * c:5 * c]
    assert torch.equal(n, n_o)
    assert int(info[1]) == int(n_o.sum())
    e_loss = abs(info[0].item() - loss_o.item()) / abs(loss_o.item())
    e_is = max(float(((inter - inter_o).abs() / inter_o.clamp_min(1e-30))[n_o > 0].max()),
               float(((s - s_o).abs() / s_o.clamp_min(1e-30)).max()))
    e_dl = float((dl.double() - dl_o).abs().max()) / float(dl_o.abs().max())
    print("dice-err zoom=%d C=%d smooth=%g ce=%g loss=%.3g IS=%.3g dl=%.3g" % (zoom, c, smooth, ce_weight, e_loss, e_is,
                                                                              e_dl))
    assert e_loss <= 1e-6
    assert e_is <= 1e-5
    assert e_dl <= 1e-5
    clear = _clear_of_ties(x.detach().float())
    assert torch.equal(amax[clear], x.detach().argmax(1)[clear])
    return info, table


@pytest.mark.parametrize("opts", OPTIONS, ids=OPTION_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_dice_kernel_vs_oracle(zoom, shape, opts):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    smooth, ce_weight = opts
    logits = _logits(n, h, w, c, pitch, seed=zoom + 50)
    target = _absent(_target(n, ho, wo, c, seed=zoom + 50), c)
    _, table = _check_vs_oracle(logits, target, zoom, smooth, 1e-7, ce_weight)
    assert float(table[4 * c - 1]) > 0 and float(table[5 * c - 1]) == 0.0        # the absent class: S > 0, n = 0
    assert float(table[c - 1]) == 0.0 and float(table[2 * c - 1]) == 0.0         # ... and no gradient coefficient


@pytest.mark.parametrize("zoom", ZOOMS)
def test_dice_clamped_denominator(zoom):
    """smooth 0 and an absent class whose probability underflows to 0 everywhere: S_c + smooth = 0 < eps."""
    n, h, w, c, pitch = 2, 9, 13, 21, 24
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 60)
    logits[..., c - 1] = -1e4
    target = _absent(_target(n, ho, wo, c, seed=zoom + 60), c)
    for ce_weight in (0.0, 1.0):
        _, table = _check_vs_oracle(logits, target, zoom, 0.0, 1e-7, ce_weight)
        assert float(table[4 * c - 1]) == 0.0 and float(table[5 * c - 1]) == 0.0


@pytest.mark.parametrize("zoom", ZOOMS)
def test_dice_nothing_valid_gives_zero(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    target[0, 0, :3] = c + 1                             # out of range: not valid either
    for smooth, ce_weight in OPTIONS:
        info, _, _, table, dl = _run(logits, target, zoom, smooth, 1e-7, ce_weight)
        assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0
        assert float(table[:2 * c].abs().max()) == 0.0


@pytest.mark.parametrize("zoom", [1, 8])
def test_dice_deterministic_and_pred_is_plain(zoom):
    from semseg_b200 import ops
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    a = _run(logits, target, zoom, 1.0, 1e-7, 1.0)
    b = _run(logits, target, zoom, 1.0, 1e-7, 1.0)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    info, amax, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    assert torch.equal(a[1], amax) and torch.equal(a[2], lse)
    assert a[0][1].item() == info[1].item()


def test_dice_functional_and_module_dispatch():
    """SF.upsample_ce with a DiceLoss criterion runs the Dice kernels (same bits as ops.upsample_ce_dice_*)."""
    from semseg_b200 import functional as SF
    from semseg_b200.losses import DiceLoss
    zoom, (n, h, w, c, pitch) = 8, SHAPES[0]
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=70)
    target = _target(n, ho, wo, c, seed=70)
    crit = DiceLoss(ignore_index=255, smooth=0.5, ce_weight=0.3)
    info, amax, _, _, dl = _run(logits, target, zoom, 0.5, 1e-7, 0.3)
    lg = logits.detach().clone().requires_grad_(True)
    loss, pred = SF.upsample_ce(lg, target, 255, zoom=zoom, criterion=crit)
    (dl_s,) = torch.autograd.grad(loss * 0.7, lg)
    assert torch.equal(loss, info[0]) and torch.equal(pred, amax) and torch.equal(dl_s, dl)


# ------------------------------------------------------------------------------------------------ every device
def test_dice_kernels_on_every_device():
    """Shapes whose Dice kernels need more than 48 KB of dynamic shared memory: the G pass at zoom 1 and 2 with 150
    classes, the rows kernels at zoom 8 with Wo = 793; from one thread per device, every device computes the bits of
    device 0."""
    import threading
    from semseg_b200 import ops
    cases = [(1, (2, 9, 140, 150, 152)), (2, (2, 9, 70, 150, 150)), (8, (1, 5, 100, 21, 24))]
    inputs = [(zoom, _logits(n, h, w, c, pitch, seed=zoom).cpu(),
               _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom).cpu())
              for zoom, (n, h, w, c, pitch) in cases]
    results, errors = {}, []

    def run(dev):
        try:
            with torch.cuda.device(dev):
                out = []
                for zoom, logits, target in inputs:
                    lg, t = logits.to(dev), target.to(dev)
                    info, amax, lse, table = ops.upsample_ce_dice_fwd(lg, t, 255, 1.0, 1e-7, 1.0, zoom=zoom)
                    dl = ops.upsample_ce_dice_bwd(lg, t, 255, lse, table, torch.tensor([1.0], device=dev), zoom=zoom)
                    out.append(tuple(v.cpu() for v in (info, amax, lse, table, dl)))
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
        for (zoom, _, _), got, ref in zip(inputs, out, results[0]):
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), (dev, zoom)


# ------------------------------------------------------------------------------------------------ networks
def _torch_dice(logits, target, ignore_index, smooth, eps, ce_weight):
    """The Dice (+ CE) loss in fp32 PyTorch on NCHW logits."""
    import torch.nn.functional as F
    c = logits.shape[1]
    valid = (target != ignore_index) & (target >= 0) & (target < c)
    t = torch.where(valid, target, torch.zeros_like(target))
    p = torch.softmax(logits, dim=1) * valid.unsqueeze(1)
    hot = F.one_hot(t, c).permute(0, 3, 1, 2).float() * valid.unsqueeze(1)
    inter = (p * hot).sum((0, 2, 3))
    n = hot.sum((0, 2, 3))
    s = p.sum((0, 2, 3)) + n
    dice = (2 * inter + smooth) / (s + smooth).clamp_min(eps)
    loss = ((1 - dice) * (n > 0)).sum() / c
    if ce_weight:
        loss = loss + ce_weight * F.cross_entropy(logits, torch.where(valid, target, torch.full_like(target, -100)),
                                                  ignore_index=-100)
    return loss


def _torch_dice_class():
    from semseg_b200.losses import DiceLoss

    class _TorchDice(DiceLoss):
        """DiceLoss written in PyTorch under another type: the network keeps the ATen tail (interpolate -> criterion)."""

        def forward(self, logits, target):
            return _torch_dice(logits, target, self.ignore_index, self.smooth, self.eps, self.ce_weight)

    return _TorchDice


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_dice_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import DiceLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    native.criterion = DiceLoss(ignore_index=255, smooth=1.0, ce_weight=1.0)
    aten = copy.deepcopy(native)
    aten.criterion = _torch_dice_class()(ignore_index=255, smooth=1.0, ce_weight=1.0)
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
def test_graphed_dice_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import DiceLoss
    base = _build("psp", 8).cuda().train()
    base.criterion = DiceLoss(ignore_index=255, smooth=1.0, ce_weight=1.0)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = _graphed_vs_eager(base, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 1
    # a new smooth is a new launch argument: it captures anew, never replays the old graph
    for m in (eager, graphed):
        m.criterion.smooth = 0.5
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, n_steps)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, n_steps)
    assert le == lg, (le, lg)
    assert _n_graphs(graphed) == 2


def test_graphed_dice_step_launches_no_aten_tail():
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import DiceLoss
    model = _build("psp", 8).cuda().train()
    model.criterion = DiceLoss(ignore_index=255, ce_weight=1.0)
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
    bad = [n for n in names if any(k in n for k in ("upsample_bilinear2d", "_softmax", "softmax", "SoftMax",
                                                    "one_hot", "nll_loss"))]
    assert not bad, sorted(set(bad))


# ------------------------------------------------------------------------------------------------ module path
def test_dice_module_path_matches_oracle():
    """DiceLoss()(eval_model(x), y) as validate() calls it, and its gradient."""
    from semseg_b200.losses import DiceLoss
    from tests.dice_oracle import dice_ce_grad
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    for crit in (DiceLoss(), DiceLoss(smooth=1.0, ce_weight=1.0)):
        loss = crit(out, y)
        ref = dice_ce(out, y, 255, crit.smooth, crit.eps, crit.ce_weight)[0]
        assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
        lg = out.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(crit(lg, y), lg)
        g_ref = dice_ce_grad(out, y, 255, crit.smooth, crit.eps, crit.ce_weight)
        assert float((g.double() - g_ref).abs().max()) <= 1e-5 * float(g_ref.abs().max())
