"""GPU tier (-m gpu): training with frozen BatchNorm — BN layers in eval mode inside a network in training mode
(`model.train()`, then `.eval()` on the BN layers). They normalise with their running statistics, never update them, and
still pass gradients to the convolutions, to gamma / beta and to the input.

  * the one-pass backward kernel (ops.bn_bwd_frozen) against torch fp32 autograd of F.batch_norm(training=False),
    in bf16 and bf16x3, deterministic;
  * a Bottleneck (d = 2, 4) with every BN frozen against the oracle with the same layers frozen (bf16x3);
  * PSPNet50 / PSANet50 training steps with two freeze patterns against the frozen oracle: every parameter that
    requires a gradient gets one, frozen running statistics stay put;
  * the CUDA-graph step: bit-identical to eager with frozen BN, and freezing after a capture captures anew.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.frozen_oracle import frozen_oracle_from

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _strict_fp32():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _act(x_nhwc_f32, split, pitch=None):
    """fp32 NHWC -> activation (optionally a channel slice of a wider buffer: padded pitch)."""
    from semseg_b200 import ops
    a = ops.f32_to_act(x_nhwc_f32.contiguous(), split)
    if pitch is None:
        return a
    c = a.shape[-1]
    buf = torch.zeros(a.shape[:-1] + (pitch,), dtype=a.dtype, device=a.device)
    buf[..., :c] = a
    return buf[..., :c]


def _f32(a):
    from semseg_b200 import ops
    return ops.act_to_f32(a)


def _bn_params(c, g):
    gamma = torch.rand((c,), device="cuda", generator=g) + 0.5
    beta = torch.randn((c,), device="cuda", generator=g) * 0.3
    rm = torch.randn((c,), device="cuda", generator=g) * 0.5
    rv = torch.rand((c,), device="cuda", generator=g) * 2 + 0.25
    return gamma, beta, rm, rv


def _kernel_cases():
    cases = []
    for c in (64, 72, 2048):
        for res in (False, True):
            for relu in (False, True):
                for src in (("y", "raw") if relu and not res else ("y",) if relu else ("none",)):
                    cases.append((c, res, relu, src, True, None))
    cases += [(64, False, True, "raw", False, None), (72, True, True, "y", False, None),
              (64, True, True, "y", True, 128), (72, False, True, "raw", True, 136)]
    return cases


@pytest.mark.parametrize("split", [False, True], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("case", _kernel_cases())
def test_bn_bwd_frozen_kernel_vs_torch_autograd(case, split):
    from semseg_b200 import ops
    c, res, relu, src, sums_on, pitch = case
    g = torch.Generator(device="cuda").manual_seed(c + 2 * res + 4 * relu)
    n, h, w = (2, 9, 11) if c == 2048 else (2, 30, 31)
    eps = 1e-5
    gamma, beta, rm, rv = _bn_params(c, g)
    raw = _act(torch.randn((n, h, w, c), device="cuda", generator=g) * 1.5 + 0.2, split, pitch)
    dy = _act(torch.randn((n, h, w, c), device="cuda", generator=g), split, pitch)
    r = _act(torch.randn((n, h, w, c), device="cuda", generator=g), split, pitch) if res else None
    # the forward as the product runs it: folded scale / shift, bn_apply (mask source of the backward)
    ss = ops.bn_fold_eval(gamma, beta, rm, rv, eps)
    y = ops.bn_apply(raw, ss, residual=r, relu=relu)

    def run():
        return ops.bn_bwd_frozen(dy, y if src == "y" else None, raw if (src == "raw" or sums_on) else None, gamma,
                                 beta, rm, rv, eps, relu, want_dres=res, want_sums=sums_on)

    d_raw, dres, sums = run()
    again = run()
    for a, b in zip((d_raw, dres, sums), again):        # deterministic: no atomics, fixed reduction order
        assert (a is None and b is None) or torch.equal(a, b)

    # torch fp32 autograd on the same inputs, with the kernel's own ReLU mask (the sign of fma(raw, s, t) vs torch's
    # (raw - mean) * invstd * gamma + beta may differ at exact near-ties; those are checked separately below)
    rawt = _f32(raw).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    z = F.batch_norm(rawt, rm, rv, gt, bt, False, 0.1, eps)
    rt = None
    if res:
        rt = _f32(r).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
        z = z + rt
    if relu:
        mask = (_f32(y) > 0).permute(0, 3, 1, 2)
        ties = mask != (z.detach() > 0)
        assert bool((z.detach()[ties].abs() <= 1e-5 * (1 + z.detach().abs().max())).all())
        z = z * mask
    z.backward(_f32(dy).permute(0, 3, 1, 2))
    ref_draw = rawt.grad.permute(0, 2, 3, 1)
    got = _f32(d_raw)
    if split:
        assert bool(((got - ref_draw).abs() <= 1e-5 * ref_draw.abs() + 1e-30).all())
    else:   # one bf16 rounding of the fp32 product: within one bf16 ulp of the fp32 gradient
        ulp = torch.exp2(torch.floor(torch.log2(ref_draw.abs().clamp_min(1e-30))) - 7)
        assert bool(((got - ref_draw).abs() <= ulp).all())
    if res:
        assert torch.equal(_f32(dres), rt.grad.permute(0, 2, 3, 1))        # dres = dz exactly
    else:
        assert dres is None
    if sums_on:
        assert util.rel_l2(sums[0], bt.grad) <= 1e-5
        assert util.rel_l2(sums[1], gt.grad) <= 1e-5
    else:
        assert sums is None


def test_bn_bwd_frozen_without_raw_sums_dz_only():
    """gamma frozen, beta trained: raw is not kept, only sum dz is formed (the dz*xhat row is zero)."""
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    c = 128
    gamma, beta, rm, rv = _bn_params(c, g)
    raw = _act(torch.randn((2, 17, 19, c), device="cuda", generator=g), False)
    dy = _act(torch.randn((2, 17, 19, c), device="cuda", generator=g), False)
    y = ops.bn_apply(raw, ops.bn_fold_eval(gamma, beta, rm, rv, 1e-5), relu=True)
    _, _, sums = ops.bn_bwd_frozen(dy, y, None, gamma, beta, rm, rv, 1e-5, True)
    dz = _f32(dy) * (_f32(y) > 0)
    assert util.rel_l2(sums[0], dz.reshape(-1, c).sum(0)) <= 1e-5
    assert bool((sums[1] == 0).all())


# ---------------------------------------------------------------------------------------------------------- Bottleneck
def _frozen_block(dil, planes):
    from semseg_b200.resnet import Bottleneck
    torch.manual_seed(0)
    blk = Bottleneck(planes * 4, planes).cuda()
    blk.conv2.dilation, blk.conv2.padding = (dil, dil), (dil, dil)
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            torch.nn.init.uniform_(m.weight, 0.5, 1.5)
            torch.nn.init.normal_(m.bias, 0, 0.2)
            torch.nn.init.normal_(m.running_mean, 0, 0.2)
            torch.nn.init.uniform_(m.running_var, 0.5, 2.0)
    blk.train()
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()
    return blk


def _bn_eval(x, blk, name, w):
    bn = getattr(blk, name)
    return F.batch_norm(x, bn.running_mean, bn.running_var, w[name + ".weight"], w[name + ".bias"], False, 0.1, 1e-5)


@pytest.mark.parametrize("affine_grad", [True, False], ids=["gamma_beta_trained", "gamma_beta_frozen"])
@pytest.mark.parametrize("dil,planes", [(2, 256), (4, 512)])
def test_bottleneck_frozen_bn_x3_vs_oracle(dil, planes, affine_grad):
    """Forward <= 1e-4 against the oracle with every BN frozen; gradients <= 1e-3 against the fp32 reference evaluated
    with the same ReLU masks (method and reasons as tests/test_parity_x3_gpu.py::test_bottleneck_block_x3_vs_oracle),
    <= 1e-2 against the plain oracle. With gamma / beta frozen their gradients stay None and the forward is the eval
    kernel, bit for bit."""
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from tests.frozen_oracle import FrozenBNOracle
    blk = _frozen_block(dil, planes)
    if not affine_grad:
        for m in blk.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.requires_grad_(False)
                m.bias.requires_grad_(False)
    bn_names = ("bn1", "bn2", "bn3")
    running = {k: v.clone() for k, v in blk.state_dict().items() if "running" in k or "num_batches" in k}
    with precision.mode("bf16x3"):
        x = torch.randn((2, planes * 4, 30, 30), device="cuda")
        sd = {"layer1.0." + k: v.detach().clone() for k, v in blk.state_dict().items()}
        trained = {"layer1.0." + k for k, p in blk.named_parameters() if p.requires_grad}
        for k, v in sd.items():
            if k in trained:
                v.requires_grad_(True)
        orc = FrozenBNOracle(sd, frozen={"layer1.0." + b for b in bn_names})
        xi = SF.to_nhwc_bf16(x).requires_grad_(True)
        xo = _f32(xi.detach()).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
        yo = orc.bottleneck(xo, "layer1.0", 1, dil, False)
        with SF.network_mode(True):
            yi = blk.forward_nhwc(xi)
        assert util.rel_l2(_f32(yi).permute(0, 3, 1, 2), yo) < 1e-4
        go = _act(torch.randn((2, 30, 30, planes * 4), device="cuda"), True)
        gof = _f32(go).permute(0, 3, 1, 2)
        yo.backward(gof)
        yi.backward(go)
        for k, v in blk.state_dict().items():
            if k in running:
                assert torch.equal(v, running[k]), k           # running statistics and counters untouched
        assert util.rel_l2(_f32(xi.grad).permute(0, 3, 1, 2), xo.grad) < 1e-2
        for k, p in blk.named_parameters():
            if p.requires_grad:
                assert util.rel_l2(p.grad, sd["layer1.0." + k].grad) < 1e-2, k
            else:
                assert p.grad is None, k
        # stage outputs of the same kernels give the masks (stage by stage == fused, bit for bit)
        with SF.network_mode(True):
            y1 = SF.conv_bn_act(xi.detach(), blk.conv1, blk.bn1, relu=True)
            y2 = SF.conv_bn_act(y1, blk.conv2, blk.bn2, relu=True)
        if not affine_grad:
            with torch.no_grad():        # eval mode: the folded single kernels
                blk.eval()
                ye = blk.forward_nhwc(xi.detach())
                blk.train()
                for b in bn_names:
                    getattr(blk, b).eval()
            assert torch.equal(ye, yi.detach())
    m1 = (_f32(y1.detach()) > 0).permute(0, 3, 1, 2).float()
    m2 = (_f32(y2.detach()) > 0).permute(0, 3, 1, 2).float()
    m3 = (_f32(yi.detach()) > 0).permute(0, 3, 1, 2).float()
    w = {k: v.detach().clone().requires_grad_(True) for k, v in blk.named_parameters()}
    xm = xo.detach().clone().requires_grad_(True)
    a1 = _bn_eval(F.conv2d(xm, w["conv1.weight"]), blk, "bn1", w) * m1
    a2 = _bn_eval(F.conv2d(a1, w["conv2.weight"], padding=dil, dilation=dil), blk, "bn2", w) * m2
    a3 = (_bn_eval(F.conv2d(a2, w["conv3.weight"]), blk, "bn3", w) + xm) * m3
    a3.backward(gof)
    e_dx = util.rel_l2(_f32(xi.grad).permute(0, 3, 1, 2), xm.grad)
    e_p = {k: util.rel_l2(p.grad, w[k].grad) for k, p in blk.named_parameters() if p.requires_grad}
    print("frozen bottleneck d%d bf16x3 mask-matched: dx %.2e, worst param %.2e" % (dil, e_dx, max(e_p.values())))
    assert e_dx < 1e-3, e_dx
    assert all(v < 1e-3 for v in e_p.values()), e_p


# ---------------------------------------------------------------------------------------------------------- networks
HEADS = ("ppm.", "psa.", "cls.", "aux.")


def _warm_running_stats(model, x, y):
    """Running statistics of one batch (momentum 1), so that frozen layers normalise with realistic statistics."""
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    moms = [m.momentum for m in bns]
    for m in bns:
        m.momentum = 1.0
    model.train()
    with torch.no_grad():
        model(x, y)
    for m, mom in zip(bns, moms):
        m.momentum = mom


@pytest.mark.parametrize("pattern", ["all", "backbone"])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_step_with_frozen_bn_vs_oracle(arch, pattern, monkeypatch):
    """A training step of PSPNet50 / PSANet50 (bf16x3) with every BN frozen, or only the backbone's (heads keep batch
    statistics), against the fp32 oracle with the same layers frozen."""
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    build = util.build_pspnet if arch == "psp" else util.build_psanet
    model = build(50, 21).cuda()
    x, y = util.synth(2, 65, 65, 21, seed=4, device="cuda")
    _warm_running_stats(model, x, y)
    model.train()
    frozen = set()
    for name, m in model.named_modules():
        if isinstance(m, torch.nn.BatchNorm2d) and (pattern == "all" or not name.startswith(HEADS)):
            m.eval()
            frozen.add(name)
    assert frozen and (pattern == "all" or len(frozen) < sum(isinstance(m, torch.nn.BatchNorm2d)
                                                            for m in model.modules()))
    okw = {} if arch == "psp" else dict(mask_h=9, mask_w=9)
    orc, sd = frozen_oracle_from(model, arch, frozen=frozen, layers=50, classes=21, **okw)
    before = {k: v.clone() for k, v in model.state_dict().items() if "running" in k or "num_batches" in k}
    with precision.mode("bf16x3"):
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
    orc.train()
    _, mlo, alo = orc.forward(x, y)
    (mlo + 0.4 * alo).backward()
    print("%s frozen=%s bf16x3: main %.6f (oracle %.6f) aux %.6f (oracle %.6f)" % (arch, pattern, ml.item(), mlo.item(),
                                                                                  al.item(), alo.item()))
    assert abs(ml.item() - mlo.item()) < 1e-4 * abs(mlo.item())
    assert abs(al.item() - alo.item()) < 1e-4 * abs(alo.item())
    # Per-parameter gradients of a whole network are not comparable element by element: ReLU near-ties flip with any
    # rounding, and depth amplifies the flips. The fp32 oracle against itself with a 1e-6 relative perturbation of the
    # input already differs by 3-4 % per parameter at this shape, and the batch-statistics path (BN in training mode)
    # against the oracle by up to 16 %, like the frozen one. Element-wise accuracy is asserted by the kernel and
    # Bottleneck tests above; here every parameter must receive a finite gradient of the right direction and size.
    errs, ratios = {}, {}
    for k, p in model.named_parameters():
        assert p.grad is not None, k                              # no stage is detached
        assert bool(torch.isfinite(p.grad).all()), k
        if k.startswith("ppm.features.0.") and "ppm.features.0.2" not in frozen:
            continue     # bin 1 with batch statistics: BN over 2 single-pixel samples, analytically ~zero gradients
        errs[k] = util.rel_l2(p.grad, sd[k].grad)
        ratios[k] = float(p.grad.double().norm() / sd[k].grad.double().norm().clamp_min(1e-30))
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    print("worst gradient rel-L2:", ", ".join("%s %.2e" % kv for kv in worst))
    assert all(v <= 0.35 for v in errs.values()), worst
    assert all(0.8 < v < 1.25 for v in ratios.values()), {k: v for k, v in ratios.items() if not 0.8 < v < 1.25}
    for k in ("cls.4.weight", "cls.4.bias", "aux.4.weight", "aux.4.bias"):     # upstream of nothing chaotic
        assert errs[k] < 2e-2, (k, errs[k])
    state = model.state_dict()
    for k, v in before.items():
        layer = k.rsplit(".", 1)[0]
        if layer in frozen:
            assert torch.equal(state[k], v), k                    # frozen: statistics and counter untouched
        elif k.endswith("num_batches_tracked"):
            assert int(state[k]) == int(v) + 1, k
        elif k.endswith("running_var"):
            assert not torch.equal(state[k], v), k                # batch statistics: still updated


# ---------------------------------------------------------------------------------------------------------- graphs
def _run(model, opt, batches, n_steps, graph, monkeypatch):
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    losses = []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        _, ml, al = model(x, y)
        loss = ml + 0.4 * al
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append((ml.item(), al.item()))
    assert all(torch.isfinite(torch.tensor(v)).all() for v in losses), losses
    return losses


def _opt(model):
    # small steps: without batch statistics the stem's gradient norm is in the hundreds at this toy shape, and lr 0.01
    # diverges within two steps (the comparison is bit for bit, so only finite values are useful)
    return torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-4, momentum=0.9,
                           weight_decay=1e-4)


def _freeze(model):
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()


def _assert_same(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(pa.grad, pb.grad), k


def test_graphed_frozen_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    base = util.build_pspnet(50, 21).cuda()
    batches = [util.synth(2, 65, 65, 21, seed=s, device="cuda") for s in (1, 2, 3)]
    _warm_running_stats(base, *batches[0])
    base.train()
    _freeze(base)
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    n_steps = graphs.WARMUP_CALLS + 3                      # 3 eager warm-up calls, then three steps from the graphs
    le = _run(eager, _opt(eager), batches, n_steps, False, monkeypatch)
    lg = _run(graphed, _opt(graphed), batches, n_steps, True, monkeypatch)
    assert graphs.launches_per_step(graphed) > 100
    assert le == lg, (le, lg)
    _assert_same(eager, graphed)
    for k, v in base.state_dict().items():
        if "running" in k or "num_batches" in k:
            assert torch.equal(graphed.state_dict()[k], v), k


def test_freezing_after_capture_does_not_replay_stale_graph(monkeypatch):
    from semseg_b200 import graphs
    base = util.build_pspnet(50, 21).cuda().train()
    batches = [util.synth(2, 65, 65, 21, seed=s, device="cuda") for s in (1, 2)]
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    oe, og = _opt(eager), _opt(graphed)
    n = graphs.WARMUP_CALLS + 2                            # batch statistics: captured, then replayed
    assert _run(eager, oe, batches, n, False, monkeypatch) == _run(graphed, og, batches, n, True, monkeypatch)
    assert graphs.launches_per_step(graphed) > 100
    _freeze(eager)
    _freeze(graphed)
    stats = {k: v.clone() for k, v in graphed.state_dict().items() if "running" in k or "num_batches" in k}
    n = graphs.WARMUP_CALLS + 2                            # frozen: eager warm-up again, then a capture of its own
    le = _run(eager, oe, batches, n, False, monkeypatch)
    lg = _run(graphed, og, batches, n, True, monkeypatch)
    assert le == lg, (le, lg)
    _assert_same(eager, graphed)
    for k, v in stats.items():
        assert torch.equal(graphed.state_dict()[k], v), k
    assert len([s for s in graphed.__dict__["_sb_graph_steps"].values() if s.fwd is not None]) == 2
