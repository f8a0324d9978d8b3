"""GPU tier: CutMix / ClassMix for mean-teacher training (csrc/mix.cu, the mixed form of csrc/tail.cu upsample_pl_fwd,
losses.MixPseudoLabelLoss).

  * the mixing kernels against tests/mix_oracle.py, bit for bit: mask, mixed input and mixed target for both modes,
    zoom 1-8, N = 1, 2, 3, 16, square and non-square inputs, p = 0, 0.5, 1;
  * the ClassMix argmax: equal to the pseudo-label forward's yhat at zoom 8, against the float64 argmax away from fp32
    ties, presence and selection exact;
  * the mixed pseudo-label forward and backward against the float64 oracle (19-256 classes, thresholds 0-1.5, weights
    0 / 1, padded pitches, labelled / unlabelled / mixed batches); all-zero and all-one masks against the plain kernel;
    reruns bit-identical;
  * PSPNet50 / PSANet50 students with an EMA teacher against the ATen route, p = 0 against PseudoLabelLoss bit for bit,
    an input that requires grad rejected;
  * ten graphed FusedSGD steps with ema.update: one capture, losses, parameters, shadow and last_mix bit-identical to
    the eager steps, no ATen tail kernel; with two alternating shapes last_mix follows the replayed step."""
import copy

import numpy as np
import pytest
import torch

from tests.kd_oracle import upsampled
from tests.mix_oracle import argmax_x8, classmix_selected, mix_mask, mixed_batch, mixed_teacher
from tests.pl_oracle import effective, pl_grad, pl_loss
from tests.test_mean_teacher_gpu import _perturbed, _tensors
from tests.test_zoom_gpu import _batch, _build, _logits, _target

pytestmark = pytest.mark.gpu
AREA, RATIO = (0.02, 0.4), (0.3, 1 / 0.3)


def _bits_to_set(words):
    w = [int(v) & 0xFFFFFFFF for v in words]
    return {32 * k + b for k in range(8) for b in range(32) if (w[k] >> b) & 1}


def _set_to_bits(classes, n):
    out = torch.zeros((n, 8), dtype=torch.int64)
    for i, cs in enumerate(classes):
        for c in cs:
            out[i, c >> 5] |= 1 << (c & 31)
    return torch.where(out >= 2 ** 31, out - 2 ** 32, out).int()


# ------------------------------------------------------------------------------------------------ mixing kernels
@pytest.mark.parametrize("hw", [(65, 65), (41, 97)], ids=["65x65", "41x97"])
@pytest.mark.parametrize("n", [1, 2, 3, 16])
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", ["cutmix", "classmix"])
def test_mix_apply_bit_exact(mode, zoom, n, hw):
    from semseg_b200 import ops
    H, W = hw
    C = 21
    g = torch.Generator(device="cuda").manual_seed(zoom * 100 + n)
    x = torch.randn((n, 3, H, W), device="cuda", generator=g)
    y = torch.randint(0, C, (n, (H - 1) // 8 * zoom + 1, (W - 1) // 8 * zoom + 1), device="cuda", generator=g)
    y[0, 0, :3] = 255
    u = torch.rand((n, 5 + C), device="cuda", generator=g)
    u[0, 1:5] = torch.tensor([0.9, 0.1, 0.0, 1.0 - 2.0 ** -24])         # a thin box at the far column edge
    amap = sel = None
    amap_np = None
    if mode == "classmix":
        amap = torch.randint(0, C, (n, H, W), device="cuda", generator=g).to(torch.uint8)
        amap[-1] = 4                                                    # an image with one class: k = 1
        amap_np = amap.cpu().numpy()
        present = _set_to_bits([set(np.unique(a).tolist()) for a in amap_np], n).cuda()
        sel = ops.mix_select(u, present, C)
        ref_sel = [classmix_selected(u[i, 5:].cpu().numpy(), np.unique(amap_np[i])) for i in range(n)]
        assert [_bits_to_set(s) for s in sel.cpu().tolist()] == ref_sel
    for p in (0.0, 0.5, 1.0):
        mask, xm, ym = ops.mix_apply(mode, x, y, u, p, AREA, RATIO, zoom, amap, sel)
        ref_m = mix_mask(mode, u.cpu().numpy(), H, W, p, AREA, RATIO, amap_np)
        assert np.array_equal(mask.cpu().numpy(), ref_m), p
        rx, ry = mixed_batch(x, y, ref_m, zoom)
        assert torch.equal(xm, rx) and torch.equal(ym, ry), p
        if p == 0.0:
            assert int(mask.sum()) == 0 and torch.equal(xm, x)


def test_mix_apply_misaligned_planes_and_unit_batch():
    """Odd plane sizes (the float4 path only where a plane's 4 pixels are aligned) and N = 1 (the partner is the image
    itself: the batch is unchanged, the mask is still written)."""
    from semseg_b200 import ops
    H, W = 17, 9
    x = torch.randn((1, 5, H, W), device="cuda")
    y = torch.randint(0, 3, (1, 5, 3), device="cuda")
    u = torch.tensor([[0.0, 1.0 - 2.0 ** -24, 0.5, 0.5, 0.5]], device="cuda")
    mask, xm, ym = ops.mix_apply("cutmix", x, y, u, 1.0, (0.5, 1.0), RATIO, 2)
    assert int(mask.sum()) > 0 and torch.equal(xm, x) and torch.equal(ym, y)


# ------------------------------------------------------------------------------------------------ ClassMix argmax
@pytest.mark.parametrize("shape", [(2, 9, 13, 21, 24), (3, 7, 19, 150, 152), (1, 5, 6, 256, 264), (2, 17, 11, 19, 19)],
                         ids=["21-p24", "150-p152", "256-p264", "19"])
def test_mix_argmax_x8_equals_pl_yhat_and_oracle(shape):
    from semseg_b200 import ops
    n, h, w, c, pitch = shape
    t = _logits(n, h, w, c, pitch, seed=c) * 2.0
    amap, present = ops.mix_argmax_x8(t)
    H, W = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    # the pseudo-label forward's yhat at zoom 8: an all-ignore target at threshold 0 makes the effective target yhat
    target = torch.full((n, H, W), 255, dtype=torch.int64, device="cuda")
    _, _, _, eff, _ = ops.upsample_pl_fwd(t, t, target, 255, 0.0, 1.0, 1.0, zoom=8)
    assert torch.equal(amap.long(), eff)
    assert [_bits_to_set(r) for r in present.cpu().tolist()] == [set(np.unique(a).tolist())
                                                                  for a in amap.cpu().numpy()]
    ref = argmax_x8(t).cuda()
    x = upsampled(t, 8)
    top2 = x.topk(2, dim=1).values
    amb = (top2[:, 0] - top2[:, 1]) <= 1e-5 * float(x.abs().max())
    assert torch.equal(amap.long()[~amb], ref[~amb])
    if bool(amb.any()):
        picked = x.permute(0, 2, 3, 1)[amb].gather(1, amap.long()[amb].unsqueeze(1)).squeeze(1)
        assert bool((picked >= top2[:, 0][amb] - 1e-5 * float(x.abs().max())).all())
    u = torch.rand((n, 5 + c), device="cuda")
    u[:, 5:15] = 0.25                                                  # ties in the priorities
    sel = ops.mix_select(u, present, c)
    for i in range(n):
        assert _bits_to_set(sel[i].tolist()) == classmix_selected(u[i, 5:].cpu().numpy(),
                                                                  np.unique(amap[i].cpu().numpy()))


# ------------------------------------------------------------------------------------------------ mixed PL kernel
SHAPES = [(3, 9, 13, 150, 152, 160), (2, 17, 11, 19, 19, 24), (2, 6, 40, 21, 24, 21), (2, 7, 10, 256, 256, 264)]
SHAPE_IDS = ["150-p152-p160", "19-p24", "21-p24", "256-p264"]
OPTIONS = [(0.0, 1.0, 1.0), (0.5, 1.0, 1.0), (0.95, 1.0, 0.0), (1.5, 1.0, 1.0), (0.5, 0.0, 1.0)]
OPTION_IDS = ["thr0", "thr0.5", "thr0.95-ce0", "thr1.5", "thr0.5-pl0"]


def _run_mix(s, t, target, zoom, mask, threshold, pl_weight, ce_weight, grad=0.7):
    from semseg_b200 import functional as SF
    sg = s.detach().requires_grad_(True)
    if mask is None:
        out = SF._UpsampleCEPL.apply(sg, t, target, 255, zoom, threshold, pl_weight, ce_weight)
    else:
        out = SF._UpsampleCEPLMix.apply(sg, t, target, 255, zoom, threshold, pl_weight, ce_weight, mask)
    saved = out[0].grad_fn.saved_tensors
    (dl,) = torch.autograd.grad(out[0] * grad, sg)
    return out[0].detach(), out[1], dl, saved[1], saved[3], saved[2]


def _box_mask(n, h, w, seed):
    H, W = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    g = np.random.default_rng(seed)
    u = g.random((n, 5)).astype(np.float32)
    u[:, 0] = 0.0
    u[-1, 0] = 0.9                                                      # the last image is not mixed
    return torch.from_numpy(mix_mask("cutmix", u, H, W, 0.5, (0.2, 0.6), RATIO)).cuda()


@pytest.mark.parametrize("opts", OPTIONS, ids=OPTION_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_mixed_pl_kernel_vs_oracle(zoom, shape, opts):
    n, h, w, c, ps, pt = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    s = _logits(n, h, w, c, ps, seed=zoom + 60)
    t = _logits(n, h, w, c, pt, seed=zoom + 70) * 2.0
    mask = _box_mask(n, h, w, zoom + c)
    base = _target(n, ho, wo, c, seed=zoom + 60)
    mixed = base.clone()
    mixed[0] = 255                                                     # an unlabelled image
    unlabelled = torch.full_like(base, 255)
    labelled = base.clone()
    labelled[labelled == 255] = 0
    threshold, plw, cew = opts
    for name, target in (("mixed", mixed), ("unlabelled", unlabelled), ("labelled", labelled)):
        loss, _, dl, eff, wt, _ = _run_mix(s, t, target, zoom, mask, *opts)
        tm = mixed_teacher(t, mask.cpu(), zoom)
        eff_o, wt_o, conf = effective(tm, target.cpu(), 1, threshold, plw, cew)
        eff_o, wt_o = eff_o.cuda(), wt_o.cuda()
        top2 = tm.topk(2, dim=-1).values.cuda()
        scale = float(tm.abs().max())
        amb = ((top2[..., 0] - top2[..., 1]) <= 1e-5 * scale) | ((conf.cuda() - threshold).abs() <= 1e-5)
        amb = amb & (target == 255)
        assert torch.equal(eff[~amb], eff_o[~amb]), name
        eff_use = torch.where(amb, eff, eff_o)
        wt_use = torch.where(amb, wt.double(), wt_o)
        ref = pl_loss(s.detach().double(), eff_use, wt_use, zoom)
        g_ref = pl_grad(s, eff_use, wt_use, zoom) * 0.7
        if ref.item() == 0.0:
            assert loss.item() == 0.0 and float(dl.abs().max()) == 0.0
            continue
        e_loss = abs(loss.item() - ref.item()) / abs(ref.item())
        e_dl = float((dl.double() - g_ref).abs().max()) / float(g_ref.abs().max())
        print("mixpl-err %s zoom=%d C=%d thr=%g loss=%.3g dl=%.3g" % (name, zoom, c, threshold, e_loss, e_dl))
        assert e_loss <= 1e-6, name
        assert e_dl <= 5e-6, name


@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_mixed_pl_zero_and_full_masks_against_plain(zoom):
    n, h, w, c = 3, 9, 13, 150
    s = _logits(n, h, w, c, 152, seed=zoom)
    t = _logits(n, h, w, c, 150, seed=zoom + 1) * 3
    target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom)
    target[1] = 255
    target[0, :5] = 255
    H, W = 8 * (h - 1) + 1, 8 * (w - 1) + 1
    zero = torch.zeros((n, H, W), dtype=torch.uint8, device="cuda")
    a = _run_mix(s, t, target, zoom, zero, 0.3, 1.0, 1.0)
    b = _run_mix(s, t, target, zoom, None, 0.3, 1.0, 1.0)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    one = torch.ones_like(zero)
    a = _run_mix(s, t, target, zoom, one, 0.3, 1.0, 1.0)
    b = _run_mix(s, t.roll(-1, 0).contiguous(), target, zoom, None, 0.3, 1.0, 1.0)
    for k in (1, 2, 3, 4, 5):                                          # pred, dlogits, eff, weight, lse
        assert torch.equal(a[k], b[k]), k
    assert abs(a[0].item() - b[0].item()) <= 1e-6 * abs(b[0].item())
    c1 = _run_mix(s, t, target, zoom, _box_mask(n, h, w, 3), 0.3, 1.0, 1.0)
    c2 = _run_mix(s, t, target, zoom, _box_mask(n, h, w, 3), 0.3, 1.0, 1.0)
    for u, v in zip(c1, c2):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------------ networks
def _net_pair(arch, zoom, mix, p=0.5):
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    native = _build(arch, zoom).cuda().train()
    ema = ModelEMA(native, decay=0.5)
    _perturbed(native, 2)
    ema.update(native)
    other = copy.deepcopy(native)
    kw = dict(mix=mix, p=p, area=(0.2, 0.5), threshold=0.0, pl_weight=0.7, ce_weight=1.0)
    native.criterion = MixPseudoLabelLoss(ema.module, **kw)
    other.criterion = MixPseudoLabelLoss(ema.module, **kw)
    return native, other, ema


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("mix", ["cutmix", "classmix"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_mix_matches_aten_route(arch, mix, zoom, mode, monkeypatch):
    """One step on the fused mixed tail against the ATen route of the same forward (the teacher's upsampled maps mixed
    with torch.where, the module form of the loss), from the same seed."""
    from semseg_b200 import functional as SF
    from semseg_b200 import pspnet as pspnet_mod
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, aten, ema = _net_pair(arch, zoom, mix)
    x, y = _batch(zoom, n=3)
    y[1] = 255
    before = [t.clone() for t in _tensors(ema.module)]
    real = SF.fused_tail_supported
    with precision.mode(mode):
        torch.manual_seed(7)
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        lm = native.criterion.last_mix()
        assert int(lm['mask'].sum()) > 0
        monkeypatch.setattr(pspnet_mod.SF, "fused_tail_supported", lambda crit, logits, *a, **k:
                            False if logits is not None else real(crit, logits, *a, **k))
        torch.manual_seed(7)
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    lr = aten.criterion.last_mix()
    for k in ("mask", "target", "uniforms"):
        assert torch.equal(lm[k], lr[k]), k
    e_main = abs(main.item() - main_r.item()) / abs(main_r.item())
    e_aux = abs(aux.item() - aux_r.item()) / abs(aux_r.item())
    print("mix-net %s %s zoom=%d %s main=%.3g aux=%.3g" % (arch, mix, zoom, mode, e_main, e_aux))
    assert e_main <= 1e-7 and e_aux <= 1e-7
    assert (pred != pred_r).float().mean().item() < 0.01
    assert all(p.grad is None for p in ema.module.parameters())
    assert all(torch.equal(a, b) for a, b in zip(_tensors(ema.module), before))


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("mix", ["cutmix", "classmix"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_p0_equals_pseudo_label_loss(arch, mix, zoom, mode, monkeypatch):
    from semseg_b200 import precision
    from semseg_b200.losses import PseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, plain, ema = _net_pair(arch, zoom, mix, p=0.0)
    plain.criterion = PseudoLabelLoss(ema.module, threshold=0.0, pl_weight=0.7, ce_weight=1.0)
    x, y = _batch(zoom, n=3)
    y[1] = 255
    with precision.mode(mode):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = plain(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert torch.equal(main, main_r) and torch.equal(aux, aux_r) and torch.equal(pred, pred_r)
    for pa, pb in zip(native.parameters(), plain.parameters()):
        assert (pa.grad is None) == (pb.grad is None)
        if pa.grad is not None:
            assert torch.equal(pa.grad, pb.grad)
    assert int(native.criterion.last_mix()['mask'].sum()) == 0


def test_network_input_requiring_grad_raises(monkeypatch):
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, _, _ = _net_pair("psp", 8, "cutmix")
    x, y = _batch(8)
    with pytest.raises(RuntimeError, match="no gradient through the mixing"):
        native(x.requires_grad_(True), y)


# ------------------------------------------------------------------------------------------------ graphs
def _mix_run(base, mix, n_steps, batches, graph, monkeypatch, seed=11):
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import FusedSGD, ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    model = copy.deepcopy(base)
    ema = ModelEMA(model, decay=0.9)
    model.criterion = MixPseudoLabelLoss(ema.module, mix=mix, p=0.5, area=(0.1, 0.5), threshold=0.06)
    opt = FusedSGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    torch.manual_seed(seed)
    losses, mixes = [], []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        lm = model.criterion.last_mix()
        mixes.append({key: v.clone() for key, v in lm.items()})
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
        ema.update(model)
        losses.append((ml.item(), al.item()))
    return model, ema, losses, mixes


@pytest.mark.parametrize("mix", ["cutmix", "classmix"])
def test_graphed_mix_step_bit_identical_to_eager(mix, monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    batches = []
    for s in (1, 2, 3):
        x, y = _batch(8, seed=s, n=3)
        y[0] = 255
        batches.append((x, y))
    me, ee, le, xe = _mix_run(base, mix, 10, batches, False, monkeypatch)
    mg, eg, lg, xg = _mix_run(base, mix, 10, batches, True, monkeypatch)
    assert le == lg, (le, lg)
    assert len(mg.__dict__["_sb_graph_steps"]) == 1
    assert graphs.launches_per_step(mg) > 100
    for a, b in zip(_tensors(me), _tensors(mg)):
        assert torch.equal(a, b)
    for a, b in zip(_tensors(ee.module), _tensors(eg.module)):
        assert torch.equal(a, b)
    for a, b in zip(xe, xg):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert len({float(m['uniforms'][0, 0]) for m in xg}) > 5          # fresh draws at every replayed step
    assert all(p.grad is None for p in eg.module.parameters())


def test_graphed_mix_step_launches_no_aten_tail(monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    model = _build("psp", 8).cuda().train()
    ema = ModelEMA(model)
    model.criterion = MixPseudoLabelLoss(ema.module, mix='classmix', threshold=0.0)
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


def test_graphed_last_mix_follows_the_replayed_shape(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    model = _build("psp", 8).cuda().train()
    ema = ModelEMA(model)
    model.criterion = MixPseudoLabelLoss(ema.module, p=1.0)
    a = _batch(8, seed=1, n=2, size=65)
    b = _batch(8, seed=2, n=2, size=81)
    for _ in range(graphs.WARMUP_CALLS + 2):
        for x, y in (a, b):
            _, ml, al = model(x, y)
            (ml + 0.4 * al).backward()
            assert tuple(model.criterion.last_mix()['mask'].shape) == (2, x.shape[2], x.shape[3])
            assert tuple(model.criterion.last_mix()['target'].shape) == tuple(y.shape)
    assert sum(1 for s in model._sb_graph_steps.values() if s.fwd is not None) == 2
    for x, y in (a, b, a):
        _, ml, al = model(x, y)
        lm = model.criterion.last_mix()
        assert lm['mask'].shape[1] == x.shape[2]
        from tests.mix_oracle import mixed_batch as mb
        _, ym = mb(x, y, lm['mask'].cpu().numpy(), 8)
        assert torch.equal(lm['target'], ym)
