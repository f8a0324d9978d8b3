"""GPU tier: the dual-stream perturbation of mean-teacher training (UniMatch's two strong views; csrc/bn.cu's prefix
fp_fork / fp_fold, losses.PseudoLabelLoss / MixPseudoLabelLoss(streams=2)).

  * the prefix fork and fold kernels bit for bit against a torch statement of the same fp32 arithmetic, plain and
    split, (M, N) = (2, 1), (6, 3), (32, 16), C = 2048 and 72, padded pitches; at M = N equal to the plain symbols;
  * the streams are independent: each stream's view and mix rebuilt from its own uniform rows with ops.strong_augment /
    ops.mix_apply equal the accessors' tensors bit for bit (CutMix and ClassMix), and the two streams differ;
  * two identical streams (no mix, an identity strong view, dropout 0) give the one-stream step in bf16x3: main, aux,
    parameter gradients, the EMA update and pred within the bars stated there;
  * PSPNet50 / PSANet50 students with an EMA teacher against the ATen route of the same dual-stream forward (CutMix and
    ClassMix with a strong view, with and without fp_weight; zoom 2 and 8; bf16 and bf16x3), with the bars of the FP
    test;
  * bf16x3 parity of the step against tests/dual_oracle.py; ten graphed FusedSGD + ema.update steps bit-identical to
    eager ones, captured once, without an ATen tail kernel, and streams=1 with the launches of the default criterion."""
import copy

import pytest
import torch

from tests import dual_oracle, util
from tests.test_fp_gpu import _act, _aten_route, _scale, _store, _student, _val
from tests.test_mean_teacher_gpu import _tensors
from tests.test_zoom_gpu import _batch, _build

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("pad", [0, 8], ids=["dense", "padded"])
@pytest.mark.parametrize("c", [2048, 72])
@pytest.mark.parametrize("mn", [(2, 1), (6, 3), (32, 16), (3, 3)], ids=["2-1", "6-3", "32-16", "3-3"])
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "bf16x3"])
def test_prefix_fork_and_fold_bit_exact(split, mn, c, pad):
    from semseg_b200 import ops
    m, n = mn
    h, w = 7, 9                                                    # 63 pixels
    s = _scale(n, c, 0.3, m * 7 + c)
    bd = -4                                                        # the batch dimension in either form
    x = _act(m, h, w, c, c + pad, split, 1)
    out = ops.fp_fork_prefix(x, s)
    v = _val(x)
    ref = torch.cat([_store(v, split), _store(v[:n] * s[:, None, None, :], split)], bd)
    assert out.shape == ref.shape and torch.equal(out, ref)

    d = _act(m + n, h, w, c, c + pad, split, 2)
    got = ops.fp_fold_prefix(d, s)
    dv = _val(d)
    ref = _store(torch.cat([dv[:n] + s[:, None, None, :] * dv[m:], dv[n:m]]), split)
    assert got.shape == ref.shape and torch.equal(got, ref)
    if m == n:                                                     # the plain symbols' launch, bit for bit
        assert torch.equal(out, ops.fp_fork(x, s))
        assert torch.equal(got, ops.fp_fold(d, s))


def test_prefix_fork_backward_is_the_prefix_fold():
    from semseg_b200 import functional as SF
    from semseg_b200 import ops
    x = _act(6, 5, 7, 64, 64, True, 3).contiguous().requires_grad_(True)
    s = _scale(3, 64, 0.3, 5)
    y = SF.fp_fork(x, s)
    assert y.shape[-4] == 9
    d = _act(9, 5, 7, 64, 64, True, 4).contiguous()
    (g,) = torch.autograd.grad(y, x, d)
    assert torch.equal(g, ops.fp_fold_prefix(d, s))


# ------------------------------------------------------------------------------------------------ streams
@pytest.mark.parametrize("mix", ["cutmix", "classmix"])
def test_streams_are_independent(mix, monkeypatch):
    """Each stream's strong view and mix, rebuilt from its own rows of last_strong() / last_mix() uniforms with the
    native ops, equal the accessors' tensors bit for bit; the teacher runs once on the unmixed batch."""
    from semseg_b200 import ops
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import MixPseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model, _, ema = _student("psp", 8, MixPseudoLabelLoss, mix=mix, p=1.0, area=(0.2, 0.5), threshold=0.0,
                             strong=StrongAugment(), streams=2)
    crit = model.criterion
    n = 3
    x, y = _batch(8, n=n)
    y[1] = 255
    torch.manual_seed(3)
    pred, main, aux = model(x, y)
    assert pred.shape[0] == n
    st, mx = crit.last_strong(), crit.last_mix()
    assert st['image'].shape == (2 * n,) + tuple(x.shape[1:]) and st['uniforms'].shape == (2 * n, 12)
    assert mx['mask'].shape == (2 * n,) + tuple(x.shape[2:]) and mx['target'].shape == (2 * n,) + tuple(y.shape[1:])
    assert mx['uniforms'].shape == (2 * n, 5 + (21 if mix == 'classmix' else 0))
    t = crit.run_teacher(x, 21)
    amap = present = None
    if mix == 'classmix':
        amap, present = ops.mix_argmax_x8(t)
    for k in range(2):
        rows = slice(k * n, (k + 1) * n)
        view = crit.strong(x, st['uniforms'][rows])
        assert torch.equal(view, st['image'][rows]), k
        u = mx['uniforms'][rows]
        sel = ops.mix_select(u, present, 21) if mix == 'classmix' else None
        mask, _, ym = ops.mix_apply(mix, view, y, u, crit.p, crit.area, crit.ratio, 8, amap, sel)
        assert torch.equal(mask, mx['mask'][rows]) and torch.equal(ym, mx['target'][rows]), k
    assert not torch.equal(st['image'][:n], st['image'][n:])
    assert not torch.equal(mx['mask'][:n], mx['mask'][n:])


def test_two_identical_streams_are_one_stream(monkeypatch):
    """p = 0 and an identity strong view make both views bit copies of x: the dual step equals the one-stream step in
    exact arithmetic (the BatchNorm of a duplicated batch has the same statistics and gradient), and in bf16x3 up to the
    rounding of the BatchNorm sums over 2N instead of N images. That rounding is amplified the way the project's parity
    tests see it: losses within 1e-5, the classifiers' weight gradients within 1e-3, every parameter gradient within
    0.2 rel-L2 and every EMA tensor within 0.1 (worst measured on an H100: 0.099, a layer1 BatchNorm bias, and 0.046),
    and at most 0.5 % of pred's pixels flipped at near-ties of the untrained network (measured 0.18 %). The EMA's running
    variances are left out: their unbiased correction n / (n - 1) counts the 2N-image batch's samples. Four 97 x 97
    images: at N = 2 the PPM's bin-1 BatchNorm input gradient is zero in exact arithmetic, so rounding noise would be
    all that reaches layer4 through it."""
    from semseg_b200 import precision
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import FusedSGD, ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    ident = StrongAugment(p_jitter=0.0, p_gray=0.0, p_blur=0.0)
    kw = dict(p=0.0, threshold=0.0, pl_weight=0.7, strong=ident, fp_weight=0.0)
    one, two, ema = _student("psp", 8, MixPseudoLabelLoss, **kw)
    ema2 = ModelEMA(two, decay=0.5)                       # a second shadow, equal to the first
    ema2.module.load_state_dict(ema.module.state_dict())
    two.criterion = MixPseudoLabelLoss(ema2.module, streams=2, **kw)
    x, y = _batch(8, n=4, size=97)
    y[1] = 255
    outs = []
    with precision.mode("bf16x3"):
        for m, e in ((one, ema), (two, ema2)):
            opt = FusedSGD(m.parameters(), lr=0.01, momentum=0.9)
            torch.manual_seed(9)
            pred, main, aux = m(x, y)
            (main + 0.4 * aux).backward()
            opt.step()
            e.update(m)
            outs.append((pred, main.item(), aux.item()))
    assert torch.equal(two.criterion.last_strong()['image'], torch.cat([x, x]))
    (p1, m1, a1), (p2, m2, a2) = outs
    e_main, e_aux = abs(m1 - m2) / abs(m1), abs(a1 - a2) / abs(a1)
    errs = sorted(((util.rel_l2(pa.grad, pb.grad), k) for (k, pa), (_, pb) in zip(one.named_parameters(),
                                                                                   two.named_parameters())), reverse=True)
    worst = errs[0][0]
    emas = sorted(((util.rel_l2(a, b), k) for (k, a), (_, b) in zip(ema.module.state_dict().items(),
                                                                    ema2.module.state_dict().items())
                   if a.is_floating_point() and not k.endswith("running_var")), reverse=True)
    e_ema = emas[0][0]
    print("two equal streams: main %.3g aux %.3g grad %s ema %s pred %d" % (e_main, e_aux, errs[:3], emas[:3],
                                                                           int((p1 != p2).sum())))
    assert (p1 != p2).float().mean().item() <= 0.005
    assert e_main <= 1e-5 and e_aux <= 1e-5
    for head in ("cls.4.weight", "aux.4.weight"):
        assert util.rel_l2(dict(one.named_parameters())[head].grad, dict(two.named_parameters())[head].grad) <= 1e-3
    assert worst <= 0.2
    assert e_ema <= 0.1


def _against_aten(native, aten, ema, x, y, mode, monkeypatch, label=""):
    from semseg_b200 import precision
    before = [t.clone() for t in _tensors(ema.module)]
    with precision.mode(mode):
        torch.manual_seed(7)
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        _aten_route(monkeypatch)
        torch.manual_seed(7)
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    for get in ("last_strong", "last_mix", "last_fp"):
        if not hasattr(native.criterion, get):
            continue
        a, b = getattr(native.criterion, get)(), getattr(aten.criterion, get)()
        assert (a is None) == (b is None), get
        for k in (a or {}):
            assert torch.equal(a[k], b[k]), (get, k)
    assert pred.shape == pred_r.shape == y.shape
    e_main = abs(main.item() - main_r.item()) / abs(main_r.item())
    e_aux = abs(aux.item() - aux_r.item()) / abs(aux_r.item())
    print("dual-net %s %s main=%.3g aux=%.3g" % (label, mode, e_main, e_aux))
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
    assert all(p.grad is None for p in ema.module.parameters())
    assert all(torch.equal(a, b) for a, b in zip(_tensors(ema.module), before))


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("fp", [0.0, 0.5], ids=["no_fp", "fp"])
@pytest.mark.parametrize("mix", ["cutmix", "classmix"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_dual_matches_aten_route(arch, mix, fp, zoom, mode, monkeypatch):
    """One dual-stream step on the fused tail (one call of the tail kernels per stream) against the ATen route of the
    same forward (the per-stream module form, each stream's teacher map mixed by its own mask), from the same seed."""
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import MixPseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, aten, ema = _student(arch, zoom, MixPseudoLabelLoss, mix=mix, area=(0.2, 0.5), strong=StrongAugment(),
                                 threshold=0.0, pl_weight=0.7, ce_weight=1.0, fp_weight=fp, streams=2)
    x, y = _batch(zoom, n=3)
    y[1] = 255
    _against_aten(native, aten, ema, x, y, mode, monkeypatch, label="%s %s fp=%g zoom=%d" % (arch, mix, fp, zoom))


def test_plain_criterion_dual_matches_aten_route(monkeypatch):
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import PseudoLabelLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native, aten, ema = _student("psp", 8, PseudoLabelLoss, strong=StrongAugment(), threshold=0.0, pl_weight=0.7,
                                 fp_weight=0.5, streams=2)
    x, y = _batch(8, n=3)
    y[0] = 255
    _against_aten(native, aten, ema, x, y, "bf16x3", monkeypatch, label="psp pl")


# ------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("fp", [0.0, 0.5], ids=["no_fp", "fp"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_parity_x3_against_dual_oracle(arch, fp, monkeypatch):
    """bf16x3 step at 65x65 against the fp32 oracle on the 2N views of last_strong(), s from last_fp(): main and aux
    within 1e-4 (the train-step bar of tests/test_parity_x3_gpu.py), cls[4]'s and aux[4]'s weight gradients within 1e-3
    rel-L2 (the bar of tests/test_fp_gpu.py)."""
    from semseg_b200 import precision
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import PseudoLabelLoss
    from semseg_b200.optim import ModelEMA
    from tests.test_mean_teacher_gpu import _perturbed
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
        crit = PseudoLabelLoss(ema.module, threshold=0.0, pl_weight=0.7, ce_weight=1.0, fp_weight=fp,
                               strong=StrongAugment(), streams=2)
        model.criterion = crit
        x, y = util.synth(4, 65, 65, 21, device="cuda")
        y[1] = 255
        with precision.mode("bf16x3"):
            t_nhwc = crit.run_teacher(x, 21)
            _, ml, al = model(x, y)
            (ml + 0.4 * al).backward()
        x2 = crit.last_strong()['image']
        s = crit.last_fp()['scale'] if fp > 0 else None
        orc.train()
        mlo, alo = dual_oracle.forward(orc, x2, s, [y, y], t_nhwc, 8, 0.0, 0.7, 1.0, fp)
        (mlo + 0.4 * alo).backward()
        e_main = abs(ml.item() - mlo.item()) / abs(mlo.item())
        e_aux = abs(al.item() - alo.item()) / abs(alo.item())
        e_w = util.rel_l2(model.cls[4].weight.grad, sd["cls.4.weight"].grad)
        e_a = util.rel_l2(model.aux[4].weight.grad, sd["aux.4.weight"].grad)
        # deeper gradients are printed, not asserted: at this size the small-count BatchNorms amplify rounding (the
        # one-stream step against itself on a duplicated batch differs by 0.1 there, see above)
        e_l4 = util.rel_l2(model.layer4[0].conv1.weight.grad, sd["layer4.0.conv1.weight"].grad)
        print("dual parity %s fp=%g: main %.3g aux %.3g cls.4.weight grad %.3g aux.4.weight grad %.3g "
              "layer4.0.conv1.weight grad %.3g" % (arch, fp, e_main, e_aux, e_w, e_a, e_l4))
        assert e_main < 1e-4 and e_aux < 1e-4
        assert e_w < 1e-3 and e_a < 1e-3
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


# ------------------------------------------------------------------------------------------------ graphs
def _dual_run(base, n_steps, batches, graph, monkeypatch, streams=2, seed=11):
    from semseg_b200.augment import StrongAugment
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import FusedSGD, ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    model = copy.deepcopy(base)
    ema = ModelEMA(model, decay=0.9)
    kw = dict(mix='cutmix', p=0.5, area=(0.1, 0.5), threshold=0.06, strong=StrongAugment(), fp_weight=0.5)
    if streams is not None:
        kw['streams'] = streams
    model.criterion = MixPseudoLabelLoss(ema.module, **kw)
    opt = FusedSGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    torch.manual_seed(seed)
    losses, states = [], []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        crit = model.criterion
        states.append({get + "." + key: v.clone() for get in ("last_strong", "last_mix", "last_fp")
                       for key, v in getattr(crit, get)().items()})
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
        ema.update(model)
        losses.append((ml.item(), al.item()))
    return model, ema, losses, states, batches[0]


def test_graphed_dual_step_bit_identical_to_eager_without_aten_tail(monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    base = _build("psp", 8).cuda().train()
    batches = []
    for s in (1, 2, 3):
        x, y = _batch(8, seed=s, n=3)
        y[0] = 255
        batches.append((x, y))
    me, ee, le, se, _ = _dual_run(base, 10, batches, False, monkeypatch)
    mg, eg, lg, sg, (x, y) = _dual_run(base, 10, batches, True, monkeypatch)
    assert le == lg, (le, lg)
    assert len(mg.__dict__["_sb_graph_steps"]) == 1
    for a, b in zip(_tensors(me), _tensors(mg)):
        assert torch.equal(a, b)
    for a, b in zip(_tensors(ee.module), _tensors(eg.module)):
        assert torch.equal(a, b)
    for a, b in zip(se, sg):
        assert a.keys() == b.keys()
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert sg[0]['last_strong.image'].shape[0] == 6 and sg[0]['last_mix.mask'].shape[0] == 6
    assert sg[0]['last_fp.scale'].shape[0] == 3
    assert len({float(s['last_mix.uniforms'][3, 0]) for s in sg}) > 5       # fresh stream-2 draws at every replay
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
    dual = graphs.launches_per_step(mg)
    # streams=1 against the criterion built without the option (the FP test's step): the same graphed launches
    counts = []
    for streams in (1, None):
        m1, _, _, _, _ = _dual_run(base, graphs.WARMUP_CALLS + 2, batches, True, monkeypatch, streams=streams)
        counts.append(graphs.launches_per_step(m1))
    print("native launches per graphed step: streams=2 %d, streams=1 %d, default %d" % (dual, counts[0], counts[1]))
    assert counts[0] == counts[1] > 100
    assert dual > counts[0]
