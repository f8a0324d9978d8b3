"""GPU tier: the feature-perturbation stream of mean-teacher training (UniMatch's FP; csrc/bn.cu fp_fork / fp_fold,
functional._FPFork, losses.PseudoLabelLoss(fp_weight, fp_dropout)).

  * the fork and fold kernels bit for bit against a torch statement of the same fp32 arithmetic, plain and split, N = 1,
    2, 3, 16, C = 2048 and 72, an odd pixel count, padded pitches, fp_dropout 0 / 0.3 / 0.5; the fork's second half
    equal to scale_nc, and at fp_dropout 0.5 the fold equal to add_act(d[:N], scale_nc(d[N:], s));
  * PSPNet50 / PSANet50 students with an EMA teacher against the ATen route of the same forward (PseudoLabelLoss,
    CutMix and ClassMix with a strong view; zoom 2 and 8; bf16 and bf16x3), with the bars of the pseudo-label test;
  * fp_dropout 0 (equal logit halves, the loss of pl_weight + fp_weight) and fp_weight 0 (today's step bit for bit,
    the same graphed launches, no draw);
  * bf16x3 parity of the step against tests/fp_oracle.py; ten graphed FusedSGD + ema.update steps bit-identical to eager
    ones, without an ATen tail kernel; a frozen-BatchNorm head and input gradients against the ATen route."""
import copy

import pytest
import torch

from tests import fp_oracle, util
from tests.test_mean_teacher_gpu import _perturbed, _tensors
from tests.test_zoom_gpu import _batch, _build

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ kernels
def _act(n, h, w, c, pitch, split, seed):
    """An activation [N, h, w, c] (plain) or [2, N, h, w, c] (split) whose rows are `pitch` channels apart."""
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn((n, h, w, pitch), device="cuda", generator=g) * 3
    a = ops.f32_to_act(v, True) if split else v.to(torch.bfloat16)
    return a[..., :c]


def _val(a):
    return a[0].float() + a[1].float() if a.dim() == 5 else a.float()


def _store(v, split):
    """The activation store of csrc/act.cuh: hi = bf16(v), lo = bf16(v - hi)."""
    hi = v.to(torch.bfloat16)
    return torch.stack([hi, (v - hi.float()).to(torch.bfloat16)]) if split else hi


def _scale(n, c, dropout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    keep = 1.0 - dropout
    return (torch.rand((n, c), device="cuda", generator=g) < keep).float().div_(keep)


@pytest.mark.parametrize("dropout", [0.0, 0.3, 0.5])
@pytest.mark.parametrize("pad", [0, 8], ids=["dense", "padded"])
@pytest.mark.parametrize("c", [2048, 72])
@pytest.mark.parametrize("n", [1, 2, 3, 16])
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "bf16x3"])
def test_fork_and_fold_bit_exact(split, n, c, pad, dropout):
    from semseg_b200 import ops
    h, w = 7, 9                                                    # 63 pixels
    s = _scale(n, c, dropout, n * 7 + c)
    bd = -4                                                        # the batch dimension in either form
    x = _act(n, h, w, c, c + pad, split, 1)
    out = ops.fp_fork(x, s)
    v = _val(x)
    ref = torch.cat([_store(v, split), _store(v * s[:, None, None, :], split)], bd)
    assert out.shape == ref.shape and torch.equal(out, ref)
    assert torch.equal(ops.act_batch_slice(out, n, 2 * n), ops.scale_nc(x, s))

    d = _act(2 * n, h, w, c, c + pad, split, 2)
    got = ops.fp_fold(d, s)
    dv = _val(d)
    ref = _store(dv[:n] + s[:, None, None, :] * dv[n:], split)
    assert got.shape == ref.shape and torch.equal(got, ref)
    if dropout == 0.5:                                             # s in {0, 2}: every product exact
        alt = ops.add_act(ops.act_batch_slice(d, 0, n), ops.scale_nc(ops.act_batch_slice(d, n, 2 * n), s))
        assert torch.equal(got, alt)


def test_fork_backward_is_the_fold():
    from semseg_b200 import functional as SF
    from semseg_b200 import ops
    x = _act(3, 5, 7, 64, 64, True, 3).contiguous().requires_grad_(True)
    s = _scale(3, 64, 0.3, 5)
    y = SF.fp_fork(x, s)
    d = _act(6, 5, 7, 64, 64, True, 4).contiguous()
    (g,) = torch.autograd.grad(y, x, d)
    assert torch.equal(g, ops.fp_fold(d, s))


# ------------------------------------------------------------------------------------------------ networks
def _student(arch, zoom, crit_cls, **kw):
    """(student, copy, ema): two equal students with the criterion on one EMA shadow that differs from them."""
    from semseg_b200.optim import ModelEMA
    native = _build(arch, zoom).cuda().train()
    ema = ModelEMA(native, decay=0.5)
    _perturbed(native, 2)
    ema.update(native)
    other = copy.deepcopy(native)
    native.criterion = crit_cls(ema.module, **kw)
    other.criterion = crit_cls(ema.module, **kw)
    return native, other, ema


def _aten_route(monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import pspnet as pspnet_mod
    real = SF.fused_tail_supported
    monkeypatch.setattr(pspnet_mod.SF, "fused_tail_supported", lambda crit, logits, *a, **k:
                        False if logits is not None else real(crit, logits, *a, **k))


def _against_aten(native, aten, ema, x, y, mode, monkeypatch, input_grad=False, label=""):
    from semseg_b200 import precision
    before = [t.clone() for t in _tensors(ema.module)]
    with precision.mode(mode):
        torch.manual_seed(7)
        xn = x.clone().requires_grad_(True) if input_grad else x
        pred, main, aux = native(xn, y)
        (main + 0.4 * aux).backward()
        fn = native.criterion.last_fp()
        _aten_route(monkeypatch)
        torch.manual_seed(7)
        xa = x.clone().requires_grad_(True) if input_grad else x
        pred_r, main_r, aux_r = aten(xa, y)
        (main_r + 0.4 * aux_r).backward()
    fa = aten.criterion.last_fp()
    assert torch.equal(fn['uniforms'], fa['uniforms']) and torch.equal(fn['scale'], fa['scale'])
    assert 0.0 < float(fn['scale'].eq(0).float().mean()) < 1.0
    e_main = abs(main.item() - main_r.item()) / abs(main_r.item())
    e_aux = abs(aux.item() - aux_r.item()) / abs(aux_r.item())
    print("fp-net %s %s main=%.3g aux=%.3g" % (label, mode, e_main, e_aux))
    assert e_main <= 1e-5 and e_aux <= 1e-5
    assert (pred != pred_r).float().mean().item() < 0.01
    if mode == "bf16x3":
        bad = []
        for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
            assert (pn.grad is None) == (pa.grad is None), k
            if pn.grad is not None:
                err = util.rel_l2(pn.grad, pa.grad)
                if err > 3e-4:
                    bad.append((k, err))
        assert not bad, bad
        if input_grad:
            assert util.rel_l2(xn.grad, xa.grad) <= 1e-4
    assert all(p.grad is None for p in ema.module.parameters())
    assert all(torch.equal(a, b) for a, b in zip(_tensors(ema.module), before))


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("loss", ["pl", "cutmix", "classmix"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_fp_matches_aten_route(arch, loss, zoom, mode, monkeypatch):
    """One step with the FP stream on the fused tail against the ATen route of the same forward (the module form of
    the loss on the upsampled perturbed logits), from the same seed."""
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import MixPseudoLabelLoss, PseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    kw = dict(threshold=0.0, pl_weight=0.7, ce_weight=1.0, fp_weight=0.5)
    if loss == "pl":
        native, aten, ema = _student(arch, zoom, PseudoLabelLoss, **kw)
    else:
        native, aten, ema = _student(arch, zoom, MixPseudoLabelLoss, mix=loss, area=(0.2, 0.5), strong=StrongAugment(),
                                     **kw)
    x, y = _batch(zoom, n=3)
    y[1] = 255
    _against_aten(native, aten, ema, x, y, mode, monkeypatch, label="%s %s zoom=%d" % (arch, loss, zoom))


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("case", ["frozen_head_bn", "input_grad"])
def test_frozen_bn_head_and_input_grad_against_aten(case, mode, monkeypatch):
    from semseg_b200.losses import PseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, aten, ema = _student("psp", 8, PseudoLabelLoss, threshold=0.0, pl_weight=0.7, fp_weight=0.5,
                                 fp_dropout=0.3)
    if case == "frozen_head_bn":
        native.cls[1].eval()
        aten.cls[1].eval()
    x, y = _batch(8, n=2)
    y[0] = 255
    _against_aten(native, aten, ema, x, y, mode, monkeypatch, input_grad=case == "input_grad", label=case)


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_fp_dropout_zero_is_the_loss_of_the_summed_weight(arch, monkeypatch):
    """s = 1: the two logit halves are bit-equal and main is the no-FP loss with pl_weight + fp_weight (not bit-equal:
    the head's statistics are sums over 2N images instead of N)."""
    from semseg_b200.losses import PseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, plain, ema = _student(arch, 8, PseudoLabelLoss, threshold=0.0, pl_weight=0.7, fp_weight=0.3, fp_dropout=0)
    plain.criterion = PseudoLabelLoss(ema.module, threshold=0.0, pl_weight=1.0)
    x, y = _batch(8, n=3)
    y[2] = 255
    _, main, aux = native(x, y)
    assert bool(native.criterion.last_fp()['scale'].eq(1).all())
    _, main_r, aux_r = plain(x, y)
    print("fp_dropout 0 %s: main %.3g" % (arch, abs(main.item() - main_r.item()) / abs(main_r.item())))
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert torch.equal(aux, aux_r)
    with torch.no_grad():
        logits, _ = native._logits_nhwc(x, torch.ones((3, 2048), device="cuda"))
    assert logits.shape[0] == 6 and torch.equal(logits[:3], logits[3:])


def test_fp_weight_zero_is_todays_step(monkeypatch):
    """fp_weight 0: no draw (the generator is where it was), N images in the head, the step bit for bit that of the
    criterion without the options, last_fp() None, and a graphed step with as many launches."""
    from semseg_b200 import graphs
    from semseg_b200.losses import MixPseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    a, b, ema = _student("psp", 8, MixPseudoLabelLoss, threshold=0.0)
    a.criterion = MixPseudoLabelLoss(ema.module, threshold=0.0, fp_weight=0.0, fp_dropout=0.3)
    x, y = _batch(8, n=3)
    y[0] = 255
    outs, states = [], []
    for m in (a, b):
        torch.manual_seed(5)
        pred, main, aux = m(x, y)
        (main + 0.4 * aux).backward()
        outs.append((pred, main, aux))
        states.append(torch.cuda.get_rng_state())
    assert a.criterion.last_fp() is None
    assert torch.equal(states[0], states[1])
    for u, v in zip(*outs):
        assert torch.equal(u, v)
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.equal(pa.grad, pb.grad)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    launches = []
    for m in (a, b):
        for _ in range(graphs.WARMUP_CALLS + 2):
            _, main, aux = m(x, y)
            (main + 0.4 * aux).backward()
        launches.append(graphs.launches_per_step(m))
    assert launches[0] == launches[1] > 100
    assert a.criterion.last_fp() is None


# ------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_parity_x3_against_fp_oracle(arch, monkeypatch):
    """bf16x3 step at 65x65 against the fp32 oracle composed on cat(f, f * s), s from last_fp(): main and aux within 1e-4
    (the train-step bar of tests/test_parity_x3_gpu.py), cls[4]'s weight gradient within 1e-3 rel-L2."""
    from semseg_b200 import precision
    from semseg_b200.losses import PseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        model = (util.build_pspnet(50, 21) if arch == "psp" else util.build_psanet(50, 21)).cuda().train()
        ema = ModelEMA(model, decay=0.5)
        _perturbed(model, 2)
        ema.update(model)
        okw = {} if arch == "psp" else dict(psa_type=2, compact=False, shrink_factor=2, mask_h=9, mask_w=9)
        orc, sd = util.oracle_from(model, arch, layers=50, classes=21, **okw)
        crit = PseudoLabelLoss(ema.module, threshold=0.0, pl_weight=0.7, ce_weight=1.0, fp_weight=0.5)
        model.criterion = crit
        x, y = util.synth(2, 65, 65, 21, device="cuda")
        y[1] = 255
        with precision.mode("bf16x3"):
            t_nhwc = crit.run_teacher(x, 21)
            _, ml, al = model(x, y)
            (ml + 0.4 * al).backward()
        s = crit.last_fp()['scale']
        orc.train()
        mlo, alo = fp_oracle.forward(orc, x, s, y, t_nhwc, 8, 0.0, 0.7, 1.0, 0.5)
        (mlo + 0.4 * alo).backward()
        e_main = abs(ml.item() - mlo.item()) / abs(mlo.item())
        e_aux = abs(al.item() - alo.item()) / abs(alo.item())
        e_w = util.rel_l2(model.cls[4].weight.grad, sd["cls.4.weight"].grad)
        print("fp parity %s: main %.3g aux %.3g cls.4.weight grad %.3g" % (arch, e_main, e_aux, e_w))
        assert e_main < 1e-4 and e_aux < 1e-4
        assert e_w < 1e-3
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


# ------------------------------------------------------------------------------------------------ graphs
def _fp_run(base, n_steps, batches, graph, monkeypatch, seed=11):
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import FusedSGD, ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    model = copy.deepcopy(base)
    ema = ModelEMA(model, decay=0.9)
    model.criterion = MixPseudoLabelLoss(ema.module, mix='cutmix', p=0.5, area=(0.1, 0.5), threshold=0.06,
                                         strong=StrongAugment(), fp_weight=0.5)
    opt = FusedSGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    torch.manual_seed(seed)
    losses, fps = [], []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        fps.append({key: v.clone() for key, v in model.criterion.last_fp().items()})
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
        ema.update(model)
        losses.append((ml.item(), al.item()))
    return model, ema, losses, fps, batches[0]


def test_graphed_fp_step_bit_identical_to_eager_without_aten_tail(monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    batches = []
    for s in (1, 2, 3):
        x, y = _batch(8, seed=s, n=3)
        y[0] = 255
        batches.append((x, y))
    me, ee, le, fe, _ = _fp_run(base, 10, batches, False, monkeypatch)
    mg, eg, lg, fg, (x, y) = _fp_run(base, 10, batches, True, monkeypatch)
    assert le == lg, (le, lg)
    assert len(mg.__dict__["_sb_graph_steps"]) == 1
    assert graphs.launches_per_step(mg) > 100
    for a, b in zip(_tensors(me), _tensors(mg)):
        assert torch.equal(a, b)
    for a, b in zip(_tensors(ee.module), _tensors(eg.module)):
        assert torch.equal(a, b)
    for a, b in zip(fe, fg):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert len({float(f['uniforms'][0, 0]) for f in fg}) > 5          # fresh draws at every replayed step
    assert all(p.grad is None for p in eg.module.parameters())
    for p in mg.parameters():
        p.grad = None
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = mg(x, y)
        (ml + 0.4 * al).backward()
        eg.update(mg)
        torch.cuda.synchronize()
    assert len(mg.__dict__["_sb_graph_steps"]) == 1
    bad = sorted({e.name for e in prof.events() if any(k in e.name for k in ("upsample_bilinear2d", "_softmax",
                                                                             "nll_loss", "lerp"))})
    assert not bad, bad
