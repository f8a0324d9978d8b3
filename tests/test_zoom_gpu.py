"""GPU tier: the fused tail at zoom factors 1, 2 and 4 (csrc/tail.cu through semseg_b200/functional.py).

  * kernel vs ATen: F.interpolate(align_corners=True) (none at zoom 1) -> F.cross_entropy(ignore_index=255) -> max(1) in
    fp32, at odd h != w, widths off the 128-column CTA, 19 / 21 / 150 classes and a padded logits pitch;
  * zoom 8 through the zoom entry points is the x8 entry point, bit for bit;
  * a PSPNet50 / PSANet50 at zoom 1, 2, 4 with the native tail agrees with the same network on the ATen tail;
  * graphed training steps at zoom 4 are bit-identical to eager ones, and an eager step launches no ATen tail kernel;
  * sliding-window scores of a zoom-4 PSPNet: the native x8 finish agrees with the ATen xZ-then-x(8/Z) finish."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4]


class _ATenCE(torch.nn.CrossEntropyLoss):
    """nn.CrossEntropyLoss under another type: the network keeps today's ATen tail (interpolate -> criterion -> max)."""


def _logits(n, h, w, c, pitch, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn((n, h, w, pitch), device="cuda", generator=g) * 3
    return base[..., :c]                          # stride(2) == pitch: a padded NHWC row as the classifier writes it


def _target(n, ho, wo, c, seed):
    """~5 % ignored pixels (255) and a few out-of-range classes (which contribute nothing)."""
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    t = torch.randint(0, c, (n, ho, wo), device="cuda", generator=g)
    t[torch.rand((n, ho, wo), device="cuda", generator=g) < 0.05] = 255
    odd = torch.rand((n, ho, wo), device="cuda", generator=g) < 0.003
    t[odd] = torch.where(torch.rand((n, ho, wo), device="cuda", generator=g)[odd] < 0.5, c + 3, -2)
    return t


def _aten_tail(logits, target, zoom):
    """The reference's tail in fp32 -> (loss, dlogits NHWC, upsampled NCHW logits). ATen's nll_loss asserts on a target
    outside [0, C) that is not ignore_index, so those pixels are handed to it as ignored: the fused kernel skips them."""
    c = logits.shape[-1]
    n, h, w = logits.shape[:3]
    t = target.clone()
    t[(t != 255) & ((t < 0) | (t >= c))] = 255
    lr = logits.detach().clone().requires_grad_(True)
    x = lr.permute(0, 3, 1, 2)
    if zoom != 1:
        x = F.interpolate(x, size=(zoom * (h - 1) + 1, zoom * (w - 1) + 1), mode="bilinear", align_corners=True)
    loss = F.cross_entropy(x, t, ignore_index=255)
    (dl,) = torch.autograd.grad(loss, lr)
    return loss.detach(), dl, x.detach()


def _clear_of_ties(x, gap=1e-5):
    """Pixels whose top-1 / top-2 fp32 logit gap is at least `gap` (argmax is well defined there)."""
    top2 = x.topk(2, dim=1).values
    return (top2[:, 0] - top2[:, 1]) >= gap


@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("shape", [(2, 9, 13, 150, 150), (1, 45, 37, 19, 19), (3, 17, 9, 21, 24), (2, 33, 40, 150, 152),
                                   (1, 20, 140, 150, 152)],
                         ids=["9x13-150", "45x37-19", "17x9-21-pitch24", "33x40-150-pitch152", "20x140-150-pitch152"])
def test_upsample_ce_zoom_vs_aten(zoom, shape):
    from semseg_b200 import functional as SF
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    runs = []
    for _ in range(2):
        lg = logits.detach().requires_grad_(True)
        loss, pred = SF.upsample_ce(lg, target, 255, zoom=zoom)
        (dl,) = torch.autograd.grad(loss, lg)
        runs.append((loss.detach(), pred, dl))
    (loss, pred, dl), (loss2, pred2, dl2) = runs
    assert torch.equal(loss, loss2) and torch.equal(pred, pred2) and torch.equal(dl, dl2)     # deterministic
    assert pred.shape == (n, ho, wo) and dl.shape == (n, h, w, c)
    loss_ref, dl_ref, x = _aten_tail(logits, target, zoom)
    assert abs(loss.item() - loss_ref.item()) <= 1e-5 * abs(loss_ref.item())
    clear = _clear_of_ties(x)
    assert clear.float().mean().item() > 0.99
    assert torch.equal(pred[clear], x.argmax(1)[clear])
    assert float((dl - dl_ref).abs().max()) <= 1e-5 * float(dl_ref.abs().max())


@pytest.mark.parametrize("zoom", ZOOMS)
def test_upsample_ce_zoom_all_ignored(zoom):
    from semseg_b200 import functional as SF
    logits = _logits(2, 9, 11, 21, 21, seed=3).requires_grad_(True)
    target = torch.full((2, zoom * 8 + 1, zoom * 10 + 1), 255, dtype=torch.int64, device="cuda")
    loss, _ = SF.upsample_ce(logits, target, 255, zoom=zoom)
    (dl,) = torch.autograd.grad(loss, logits)
    assert loss.item() == 0.0 and float(dl.abs().max()) == 0.0


def test_zoom8_is_the_x8_entry_point():
    """ops.upsample_ce_fwd / _bwd (the zoom entry points at zoom 8) == semseg_upsample_ce_fwd / _bwd, bit for bit."""
    from semseg_b200 import _lib, ops
    lib = _lib.load()
    n, h, w, c = 2, 17, 23, 150
    ho, wo = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    logits = _logits(n, h, w, c, 152, seed=8)
    target = _target(n, ho, wo, c, seed=8)
    info, amax, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=8)
    grad = torch.tensor([0.4], device="cuda")
    dl = ops.upsample_ce_bwd(logits, target, 255, lse, info, grad, zoom=8)

    p = lambda t: ctypes.c_void_p(t.data_ptr())                 # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ws = torch.empty((lib.semseg_upsample_ce_workspace_floats(n, ho, wo),), device="cuda")
    info_o = torch.empty(2, device="cuda")
    amax_o = torch.empty((n, ho, wo), dtype=torch.int64, device="cuda")
    lse_o = torch.empty((n, ho, wo), device="cuda")
    _lib.check(lib.semseg_upsample_ce_fwd(p(logits), 152, n, h, w, c, p(target), ho, wo, 255, p(ws), p(info_o),
                                          p(amax_o), p(lse_o), stream), "semseg_upsample_ce_fwd")
    wsb = torch.empty((lib.semseg_upsample_ce_bwd_workspace_floats(n, ho, w, c),), device="cuda")
    dl_o = torch.empty((n, h, w, c), device="cuda")
    _lib.check(lib.semseg_upsample_ce_bwd(p(logits), 152, n, h, w, c, p(target), ho, wo, 255, p(lse_o), p(info_o),
                                          p(grad), p(wsb), p(dl_o), stream), "semseg_upsample_ce_bwd")
    torch.cuda.synchronize()
    assert torch.equal(info, info_o) and torch.equal(amax, amax_o) and torch.equal(lse, lse_o)
    assert torch.equal(dl, dl_o)


def test_zoom8_matches_the_x8_kernel_golden():
    """The zoom-8 instance of the templated kernels reproduces, bit for bit, what the x8-only kernels they replaced
    computed (tests/golden/tail_x8.npz, written by tests/golden/make_tail_x8_golden.py with that library): loss and
    count, argmax, lse and dlogits, at a padded pitch, with ignored and out-of-range targets, over two column CTAs."""
    import os
    from semseg_b200 import ops
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tail_x8.npz"))
    for key in ("c21", "c150"):
        logits_p = torch.from_numpy(g[key + "_logits"]).cuda()
        c = g[key + "_dlogits"].shape[-1]
        logits = logits_p[..., :c]
        target = torch.from_numpy(g[key + "_target"].astype(np.int64)).cuda()
        info, amax, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=8)
        dl = ops.upsample_ce_bwd(logits, target, 255, lse, info, torch.tensor([0.4], device="cuda"), zoom=8)
        assert np.array_equal(info.cpu().numpy(), g[key + "_info"]), key
        assert np.array_equal(amax.cpu().numpy(), g[key + "_argmax"].astype(np.int64)), key
        assert np.array_equal(lse.cpu().numpy(), g[key + "_lse"]), key
        assert np.array_equal(dl.cpu().numpy(), g[key + "_dlogits"]), key


def test_upsample_ce_on_every_device():
    """Shapes whose kernels need more than 48 KB of dynamic shared memory: the forward at zoom 1 and 2 with 150 classes,
    the backward at zoom 8 with Wo = 793. The opt-in is per device, so every device runs them, from one thread per device
    as nn.DataParallel replicas do, and must compute the same bits as device 0."""
    import threading
    from semseg_b200 import ops
    cases = [(1, (2, 9, 140, 150, 152)), (2, (2, 9, 70, 150, 150)), (8, (1, 5, 100, 21, 24))]
    inputs = []
    for zoom, (n, h, w, c, pitch) in cases:
        inputs.append((zoom, _logits(n, h, w, c, pitch, seed=zoom).cpu(),
                       _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom).cpu()))
    results, errors = {}, []

    def run(dev):
        try:
            with torch.cuda.device(dev):
                out = []
                for zoom, logits, target in inputs:
                    lg, t = logits.to(dev), target.to(dev)
                    info, amax, lse = ops.upsample_ce_fwd(lg, t, 255, zoom=zoom)
                    dl = ops.upsample_ce_bwd(lg, t, 255, lse, info, torch.tensor([1.0], device=dev), zoom=zoom)
                    out.append(tuple(v.cpu() for v in (info, amax, lse, dl)))
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
def _build(arch, zoom, classes=21, seed=0):
    """A seeded PSPNet50 / PSANet50 at zoom factor `zoom` (tests/util's builders pin zoom 8)."""
    from semseg_b200.psanet import PSANet
    from semseg_b200.pspnet import PSPNet
    torch.manual_seed(seed)
    if arch == "psp":
        return PSPNet(layers=50, classes=classes, zoom_factor=zoom, dropout=0.0, pretrained=False)
    return PSANet(layers=50, classes=classes, zoom_factor=zoom, dropout=0.0, psa_type=2, compact=False, shrink_factor=2,
                  mask_h=9, mask_w=9, pretrained=False)


def _zoom_target(y, zoom, seed):
    """The training target at zoom `zoom` as tool/train.py:262-266 builds it (bilinear, align_corners, truncation), from
    a full-resolution label map without ignored pixels — interpolating 255 into class ids would yield labels >= classes,
    on which ATen's nll_loss asserts; the ignored pixels are marked afterwards."""
    if zoom != 8:
        h = int((y.size()[1] - 1) / 8 * zoom + 1)
        w = int((y.size()[2] - 1) / 8 * zoom + 1)
        y = F.interpolate(y.unsqueeze(1).float(), size=(h, w), mode='bilinear', align_corners=True).squeeze(1).long()
    g = torch.Generator(device=y.device).manual_seed(seed)
    y = y.clone()
    y[torch.rand(y.shape, device=y.device, generator=g) < 0.05] = 255
    return y


def _batch(zoom, classes=21, seed=1, n=2, size=65):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, 3, size, size), generator=g).cuda()
    y = torch.randint(0, classes, (n, size, size), generator=g).cuda()
    return x, _zoom_target(y, zoom, seed)


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", ZOOMS)
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200 import pspnet as pspnet_mod
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    aten = copy.deepcopy(native)
    aten.criterion = _ATenCE(ignore_index=255)
    x, y = _batch(zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    seen = []

    def upsample_logits(logits_nhwc, size, zoom_factor):
        out = real(logits_nhwc, size, zoom_factor)
        seen.append(out.detach())
        return out

    real = pspnet_mod.upsample_logits
    with precision.mode(mode):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        with monkeypatch.context() as mp:
            mp.setattr(pspnet_mod, "upsample_logits", upsample_logits)
            pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert len(seen) == 2, "the ATen copy must run the ATen tail"
    assert pred.shape == pred_r.shape == y.shape
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    clear = _clear_of_ties(seen[0])
    assert clear.float().mean().item() > 0.99
    assert torch.equal(pred[clear], pred_r[clear])
    if mode == "bf16x3":
        # in bf16 the tails' ~1e-6 differences in dlogits flip bf16 roundings further down the backward. In bf16x3 they
        # still flip hi/lo roundings; every gradient agrees to 1e-4 except that of the stem's last BatchNorm bias, the
        # far end of the backward and a cancelling sum over every pixel, which differs by up to ~1.3e-4
        loose = {"layer0.7.bias": 3e-4}
        bad = []
        for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
            assert (pn.grad is None) == (pa.grad is None), k
            if pn.grad is not None:
                err = util.rel_l2(pn.grad, pa.grad)
                if err > loose.get(k, 1e-4):
                    bad.append((k, err))
        assert not bad, bad


def _sgd_steps(model, batches, n_steps):
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    losses = []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        loss = ml + 0.4 * al
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append((ml.item(), al.item()))
    return losses


def test_graphed_steps_at_zoom4_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", 4).cuda().train()
    batches = [_batch(4, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4                    # eager warm-up calls, capture, then replays
    eager = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, n_steps)
    assert graphs.launches_per_step(eager) == 0
    graphed = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, n_steps)
    assert graphs.launches_per_step(graphed) > 100       # the zoom-4 step really was captured and replayed
    assert le == lg, (le, lg)
    se, sg = eager.state_dict(), graphed.state_dict()
    for k in se:
        assert torch.equal(se[k], sg[k]), k              # weights, running statistics, num_batches_tracked
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert (pe.grad is None) == (pg.grad is None), k
        if pe.grad is not None:
            assert torch.equal(pe.grad, pg.grad), k


@pytest.mark.parametrize("zoom", ZOOMS)
def test_training_step_launches_no_aten_tail(zoom, monkeypatch):
    """One eager training step at zoom 1, 2, 4 runs no ATen upsample / log_softmax / nll_loss kernel."""
    from torch.profiler import ProfilerActivity, profile
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _build("psp", zoom).cuda().train()
    x, y = _batch(zoom)
    _, ml, al = model(x, y)                              # warm-up (weight packs, workspaces)
    (ml + 0.4 * al).backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("upsample_ce" in n for n in names), "the fused tail kernels must run"
    bad = [n for n in names if any(k in n for k in ("upsample_bilinear2d", "log_softmax", "LogSoftMax", "nll_loss"))]
    assert not bad, sorted(set(bad))


def test_sliding_window_native_finish_at_zoom4(monkeypatch):
    from semseg_b200 import inference
    c = util.SW_CFG
    classes, crop = 7, 65
    model = _build("psp", 4, classes=classes).cuda().eval()
    assert inference._native_net(model, classes, crop, crop, torch.device("cuda")) is model
    image = util.sw_image(seed=11, h=100, w=150)
    scales, base = [0.4, 1.0, 1.25], 150
    with monkeypatch.context() as mp:                    # the ATen finish: xZ (the module output), then x(8/Z)
        mp.setattr(inference, "_native_net", lambda *a, **k: None)
        aten = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8)
        ref_scores, ref_amax = aten(image, base, scales)
    native = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8)
    scores, amax = native(image, base, scales)
    assert native.forward_calls == aten.forward_calls
    assert scores.shape == ref_scores.shape == (100, 150, classes)
    assert np.abs(scores - ref_scores).max() <= 1e-6
    top2 = np.sort(ref_scores, axis=2)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 2e-6
    assert clear.mean() > 0.9 and np.array_equal(amax[clear], ref_amax[clear])
