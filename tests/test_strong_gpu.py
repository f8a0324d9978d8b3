"""GPU tier: the strong view of mean-teacher training (csrc/strong.cu, augment.StrongAugment, the `strong` argument of
the teacher criteria).

  * the kernel against the float64 oracle (tests/strong_oracle.py), per element, within 1e-5 in normalised-input units:
    N = 1, 2, 3, 16, 24; 9x9 to 713x713; each operation alone at both ends of its range; all 24 orders with every
    operation on (contrast after each other one among them); grayscale; blur radius 1, 6, 15; non-default mean / std;
    inputs whose de-normalised values fall outside [0, 1];
  * every probability 0 copies the batch bit for bit; two calls are bit-identical;
  * PSPNet50 / PSANet50 students with an EMA teacher: with every probability 0, losses, gradients and pred equal the
    criterion without a view, bit for bit; with the view on, main and aux match the composed route (teacher on x,
    student on last_strong()['image'], the module form with teacher_logits); under MixPseudoLabelLoss the student's
    input is ops.mix_apply of the view, bit for bit; an input that requires grad raises;
  * ten graphed FusedSGD steps with ema.update: one capture, losses, parameters, shadow, last_strong and last_mix
    bit-identical to the eager steps, two more launches per step than without the view."""
import copy
import itertools

import pytest
import torch

from tests.strong_oracle import strong as oracle
from tests.test_mean_teacher_gpu import _perturbed, _tensors
from tests.test_zoom_gpu import _batch, _build

pytestmark = pytest.mark.gpu
U_MAX = 1.0 - 2.0 ** -24
TOL = 1e-5
DEFAULTS = dict(brightness=0.5, contrast=0.5, saturation=0.5, hue=0.25, p_jitter=0.8, p_gray=0.2, p_blur=0.5,
                sigma=(0.1, 2.0), mean=(0.485 * 255, 0.456 * 255, 0.406 * 255),
                std=(0.229 * 255, 0.224 * 255, 0.225 * 255))


def _x(n, h, w, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((n, 3, h, w), device="cuda", generator=g) * scale


def _u(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand((n, 12), device="cuda", generator=g)


def _check(x, u, **kw):
    from semseg_b200.augment import StrongAugment
    opts = dict(DEFAULTS, **kw)
    got = StrongAugment(**opts)(x, u)
    ref = oracle(x, u, **opts)
    err = float((got.double() - ref).abs().max())
    print("strong-err N=%d %dx%d %s: %.3g" % (x.shape[0], x.shape[2], x.shape[3], kw, err))
    assert err <= TOL, err
    return got


# ------------------------------------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("n,h,w", [(1, 9, 9), (2, 9, 9), (3, 17, 33), (16, 17, 33), (2, 97, 129), (16, 97, 129),
                                   (3, 465, 465), (16, 473, 473), (2, 713, 713)], ids=lambda v: str(v))
def test_kernel_matches_oracle_default_pipeline(n, h, w):
    x = _x(n, h, w, seed=h + n)
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + w)
    u = torch.rand((n, 12), device="cuda", generator=g)
    u[0, [0, 9, 10]] = 0.0                              # image 0: every operation, blurred
    if n > 1:
        u[1, [0, 9, 10]] = 0.9                          # image 1: nothing applies, a bit copy
    got = _check(x, u)
    if n > 1:
        assert torch.equal(got[1], x[1])


@pytest.mark.parametrize("op,strength", [("brightness", 0.9), ("contrast", 1.0), ("saturation", 1.0), ("hue", 0.5)])
def test_each_operation_alone_at_both_ends(op, strength):
    n = 4
    x = _x(n, 33, 47, seed=3)
    u = _u(n, 3)
    u[:, 1:5] = torch.tensor([[0.0] * 4, [U_MAX] * 4, [0.5] * 4, [2.0 ** -24] * 4], device="cuda")
    kw = dict(brightness=0.0, contrast=0.0, saturation=0.0, hue=0.0, p_jitter=1.0, p_gray=0.0, p_blur=0.0)
    kw[op] = strength
    _check(x, u, **kw)


def test_all_orders_with_every_operation():
    """One image per order of the four operations: contrast after none, one, two and all three of the others."""
    orders = list(itertools.permutations(range(4)))
    n = len(orders)
    x = _x(n, 33, 47, seed=5)
    u = _u(n, 5)
    for i, order in enumerate(orders):
        for pos, k in enumerate(order):
            u[i, 5 + k] = 0.1 + 0.2 * pos
    _check(x, u, p_jitter=1.0, p_gray=0.0, p_blur=0.0, brightness=0.8, contrast=0.8, saturation=0.8, hue=0.5)
    _check(x, u, p_jitter=1.0, p_gray=1.0, p_blur=1.0)


def test_grayscale_alone():
    x = _x(3, 17, 33, seed=6)
    u = _u(3, 6)
    got = _check(x, u, p_jitter=0.0, p_gray=1.0, p_blur=0.0)
    v = got * torch.tensor(DEFAULTS["std"], device="cuda").view(1, 3, 1, 1) + \
        torch.tensor(DEFAULTS["mean"], device="cuda").view(1, 3, 1, 1)
    assert float((v - v[:, :1]).abs().max()) <= 1e-3      # every channel the same gray (in 0..255 units)


@pytest.mark.parametrize("sig,r", [(0.3, 1), (2.0, 6), (5.0, 15)])
@pytest.mark.parametrize("hw", [(17, 33), (97, 129)], ids=lambda s: "%dx%d" % s)
def test_blur_radius(sig, r, hw):
    x = _x(3, hw[0], hw[1], seed=r)
    u = _u(3, r)
    _check(x, u, p_jitter=0.0, p_gray=0.0, p_blur=1.0, sigma=(sig, sig))
    _check(x, u, p_blur=1.0, sigma=(0.1, sig))


def test_non_default_mean_std_and_out_of_range_inputs():
    x = _x(16, 41, 57, seed=9, scale=4.0)                # de-normalised values far outside [0, 1]
    u = _u(16, 9)
    _check(x, u)
    _check(x, u, p_jitter=1.0, p_gray=0.5, p_blur=1.0)
    _check(x * 0.05, u, mean=(10.0, 200.0, 128.0), std=(40.0, 90.0, 64.0), p_jitter=1.0, p_blur=0.5)


def test_probability_zero_is_a_bit_copy_and_reruns_are_identical():
    from semseg_b200.augment import StrongAugment
    x = _x(3, 97, 129, seed=11, scale=3.0)
    u = _u(3, 11)
    off = StrongAugment(p_jitter=0.0, p_gray=0.0, p_blur=0.0)
    assert torch.equal(off(x, u), x) and torch.equal(off(x), x)
    on = StrongAugment(p_jitter=1.0, p_gray=0.5, p_blur=1.0)
    a, b = on(x, u), on(x, u)
    assert torch.equal(a, b) and not torch.equal(a, x)
    v = on(x.clone())
    assert v.shape == x.shape and v.dtype == torch.float32


def test_draw_is_one_rand_on_the_default_generator():
    from semseg_b200.augment import StrongAugment
    x = _x(5, 9, 9, seed=1)
    torch.manual_seed(3)
    u = StrongAugment().draw(x)
    torch.manual_seed(3)
    assert torch.equal(u, torch.rand((5, 12), device="cuda"))


# ------------------------------------------------------------------------------------------------ networks
def _pair(arch, cls, strong, **kw):
    from semseg_b200.optim import ModelEMA
    native = _build(arch, 8).cuda().train()
    ema = ModelEMA(native, decay=0.5)
    _perturbed(native, 2)
    ema.update(native)
    other = copy.deepcopy(native)
    native.criterion = cls(ema.module, strong=strong, **kw)
    return native, other, ema


def _crit(name):
    from semseg_b200.losses import DistillationLoss, MixPseudoLabelLoss, PseudoLabelLoss
    return {"kd": (DistillationLoss, dict(temperature=2.0, kd_weight=0.5)),
            "pl": (PseudoLabelLoss, dict(threshold=0.0, pl_weight=0.7)),
            "mix": (MixPseudoLabelLoss, dict(p=0.5, area=(0.2, 0.5), threshold=0.0, pl_weight=0.7))}[name]


@pytest.mark.parametrize("crit", ["kd", "pl", "mix"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_probability_zero_equals_no_view(arch, crit, monkeypatch):
    from semseg_b200.augment import StrongAugment
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    cls, kw = _crit(crit)
    native, plain, ema = _pair(arch, cls, StrongAugment(p_jitter=0.0, p_gray=0.0, p_blur=0.0), **kw)
    plain.criterion = cls(ema.module, **kw)
    x, y = _batch(8, n=3)
    y[1] = 255
    torch.manual_seed(4)
    pred, main, aux = native(x, y)
    (main + 0.4 * aux).backward()
    torch.manual_seed(4)
    pred_r, main_r, aux_r = plain(x, y)
    (main_r + 0.4 * aux_r).backward()
    assert torch.equal(main, main_r) and torch.equal(aux, aux_r) and torch.equal(pred, pred_r)
    for pa, pb in zip(native.parameters(), plain.parameters()):
        assert (pa.grad is None) == (pb.grad is None)
        if pa.grad is not None:
            assert torch.equal(pa.grad, pb.grad)
    ls = native.criterion.last_strong()
    assert torch.equal(ls['image'], x) and tuple(ls['uniforms'].shape) == (3, 12)
    assert plain.criterion.last_strong() is None


@pytest.mark.parametrize("crit", ["kd", "pl"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_view_matches_composed_route(arch, crit, monkeypatch):
    """Teacher on x, student on last_strong()['image'], then the module form with teacher_logits (the ATen route)."""
    from semseg_b200 import functional as SF
    from semseg_b200 import pspnet as pspnet_mod
    from semseg_b200.augment import StrongAugment
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    cls, kw = _crit(crit)
    native, composed, ema = _pair(arch, cls, StrongAugment(p_jitter=1.0, p_gray=0.3, p_blur=0.7), **kw)
    composed.criterion = cls(ema.module, **kw)
    x, y = _batch(8, n=3)
    y[1] = 255
    torch.manual_seed(7)
    pred, main, aux = native(x, y)
    (main + 0.4 * aux).backward()
    xs = native.criterion.last_strong()['image']
    assert not torch.equal(xs, x)
    t_x = composed.criterion.run_teacher(x, 21)
    composed.criterion.run_teacher = lambda _x, classes: t_x
    real = SF.fused_tail_supported
    monkeypatch.setattr(pspnet_mod.SF, "fused_tail_supported", lambda c, logits, *a, **k:
                        False if logits is not None else real(c, logits, *a, **k))
    pred_r, main_r, aux_r = composed(xs, y)
    (main_r + 0.4 * aux_r).backward()
    e_main = abs(main.item() - main_r.item()) / abs(main_r.item())
    e_aux = abs(aux.item() - aux_r.item()) / abs(aux_r.item())
    print("strong-net %s %s main=%.3g aux=%.3g" % (arch, crit, e_main, e_aux))
    assert e_main <= 1e-6 and e_aux <= 1e-6
    assert (pred != pred_r).float().mean().item() < 0.01
    assert all(p.grad is None for p in ema.module.parameters())


@pytest.mark.parametrize("mix", ["cutmix", "classmix"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_mix_takes_the_view(arch, mix, monkeypatch):
    """The student's input is ops.mix_apply of the view with last_mix()'s uniforms, bit for bit; the fused tail matches
    the ATen route of the same forward."""
    from semseg_b200 import functional as SF
    from semseg_b200 import ops
    from semseg_b200 import pspnet as pspnet_mod
    from semseg_b200.augment import StrongAugment
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    cls, kw = _crit("mix")
    kw = dict(kw, mix=mix)
    strong = StrongAugment(p_jitter=1.0, p_gray=0.3, p_blur=0.7)
    native, aten, ema = _pair(arch, cls, strong, **kw)
    aten.criterion = cls(ema.module, strong=strong, **kw)
    seen = []
    stem = native.layer0.forward_nchw
    native.layer0.forward_nchw = lambda t: (seen.append(t.detach().clone()), stem(t))[1]
    x, y = _batch(8, n=3)
    y[1] = 255
    torch.manual_seed(9)
    pred, main, aux = native(x, y)
    (main + 0.4 * aux).backward()
    ls, lm = native.criterion.last_strong(), native.criterion.last_mix()
    assert int(lm['mask'].sum()) > 0 and not torch.equal(ls['image'], x)
    amap = sel = None
    if mix == 'classmix':
        t = native.criterion.run_teacher(x, 21)
        amap, present = ops.mix_argmax_x8(t)
        sel = ops.mix_select(lm['uniforms'], present, 21)
    mask, xm, ym = ops.mix_apply(mix, ls['image'], y, lm['uniforms'], 0.5, (0.2, 0.5), (0.3, 1 / 0.3), 8, amap, sel)
    assert torch.equal(mask, lm['mask']) and torch.equal(ym, lm['target'])
    assert torch.equal(seen[-1], xm)
    real = SF.fused_tail_supported
    monkeypatch.setattr(pspnet_mod.SF, "fused_tail_supported", lambda c, logits, *a, **k:
                        False if logits is not None else real(c, logits, *a, **k))
    torch.manual_seed(9)
    pred_r, main_r, aux_r = aten(x, y)
    (main_r + 0.4 * aux_r).backward()
    for k in ("image", "uniforms"):
        assert torch.equal(ls[k], aten.criterion.last_strong()[k]), k
    e_main = abs(main.item() - main_r.item()) / abs(main_r.item())
    e_aux = abs(aux.item() - aux_r.item()) / abs(aux_r.item())
    print("strong-mix-net %s %s main=%.3g aux=%.3g" % (arch, mix, e_main, e_aux))
    assert e_main <= 1e-6 and e_aux <= 1e-6


def test_network_input_requiring_grad_raises(monkeypatch):
    from semseg_b200.augment import StrongAugment
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    cls, kw = _crit("pl")
    native, _, _ = _pair("psp", cls, StrongAugment(), **kw)
    x, y = _batch(8)
    with pytest.raises(RuntimeError, match="no gradient through the strong view"):
        native(x.requires_grad_(True), y)


# ------------------------------------------------------------------------------------------------ graphs
def _run(base, strong, n_steps, batches, graph, monkeypatch, seed=11):
    from semseg_b200.losses import MixPseudoLabelLoss
    from semseg_b200.optim import FusedSGD, ModelEMA
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    model = copy.deepcopy(base)
    ema = ModelEMA(model, decay=0.9)
    model.criterion = MixPseudoLabelLoss(ema.module, mix='cutmix', p=0.5, area=(0.1, 0.5), threshold=0.06,
                                         strong=strong)
    opt = FusedSGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    torch.manual_seed(seed)
    losses, views = [], []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        lm, ls = model.criterion.last_mix(), model.criterion.last_strong()
        views.append({key: v.clone() for key, v in list(lm.items()) +
                      ([("s_" + a, b) for a, b in ls.items()] if ls is not None else [])})
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        opt.step()
        ema.update(model)
        losses.append((ml.item(), al.item()))
    return model, ema, losses, views


def test_graphed_strong_step_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.augment import StrongAugment
    base = _build("psp", 8).cuda().train()
    batches = []
    for s in (1, 2, 3):
        x, y = _batch(8, seed=s, n=3)
        y[0] = 255
        batches.append((x, y))
    strong = StrongAugment(p_jitter=0.9, p_gray=0.3, p_blur=0.6)
    me, ee, le, ve = _run(base, strong, 10, batches, False, monkeypatch)
    mg, eg, lg, vg = _run(base, strong, 10, batches, True, monkeypatch)
    assert le == lg, (le, lg)
    assert len(mg.__dict__["_sb_graph_steps"]) == 1
    for a, b in zip(_tensors(me), _tensors(mg)):
        assert torch.equal(a, b)
    for a, b in zip(_tensors(ee.module), _tensors(eg.module)):
        assert torch.equal(a, b)
    for a, b in zip(ve, vg):
        assert set(a) == set(b) and "s_image" in a
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert len({float(v['s_uniforms'][0, 0]) for v in vg}) > 5          # fresh draws at every replayed step
    mp, _, _, _ = _run(base, None, 5, batches, True, monkeypatch)
    assert graphs.launches_per_step(mg) == graphs.launches_per_step(mp) + 2
