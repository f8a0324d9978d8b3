"""GPU tier (-m gpu): input gradients through PSPNet / PSANet in training and eval mode.

  * the stem dgrad kernel (ops.stem_dgrad3x3s2) element by element against float64 on its exact operands, deterministic;
  * the first stem stage with an fp32 NCHW input that needs a gradient, with batch statistics, frozen and in an eval
    network, against the fp32 oracle under the kernel's ReLU mask;
  * Bottleneck, PPM, PSA and Stem called on their own on an NCHW input;
  * eval networks (the attack set-up): the forward bit-identical to the no_grad forward, x.grad against the oracle;
  * training: x.grad with frozen BN against the oracle, graphed steps bit-identical to eager ones, x.requires_grad
    toggled between steps, and a step whose input needs no gradient still on the patch-form stem.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.frozen_oracle import frozen_oracle_from
from tests.input_grad_floor import INPUT_GRAD_TOL, frozen_eval_oracle, oracle_input_grad

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _strict_fp32():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _act(x_nhwc_f32, split, pitch=None):
    """fp32 NHWC -> activation, optionally a channel slice of a wider buffer (padded pitch)."""
    from semseg_b200 import ops
    a = ops.f32_to_act(x_nhwc_f32.contiguous(), split)
    if pitch is None:
        return a
    buf = torch.zeros(a.shape[:-1] + (pitch,), dtype=a.dtype, device=a.device)
    buf[..., :a.shape[-1]] = a
    return buf[..., :a.shape[-1]]


def _planes(a):
    """(hi, lo) fp64 NCHW planes of an activation (lo zero for plain bf16)."""
    hi = (a[0] if a.dim() == 5 else a).double().permute(0, 3, 1, 2)
    lo = a[1].double().permute(0, 3, 1, 2) if a.dim() == 5 else torch.zeros_like(hi)
    return hi, lo


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("split", [False, True], ids=["bf16", "bf16x3"])
@pytest.mark.parametrize("n, h, w, cin, pitch", [
    (1, 65, 65, 3, None), (3, 64, 64, 3, None), (1, 473, 473, 3, None), (3, 33, 81, 3, 72), (1, 3, 5, 3, None),
    (3, 65, 64, 1, None), (1, 33, 81, 2, 72), (3, 1, 1, 3, None),
])
def test_stem_dgrad_kernel_vs_float64(n, h, w, cin, pitch, split):
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(h * 7 + w + cin)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    wt = torch.randn((64, cin, 3, 3), device="cuda", generator=g) * 0.2
    wp = ops.WeightPackPlan([wt], split, dgrad=False, patches=[True])
    wp.refresh()
    slab = wp.packs[0].wp
    dy = _act(torch.randn((n, ho, wo, 64), device="cuda", generator=g), split, pitch)
    dx = ops.stem_dgrad3x3s2(dy, slab, cin, h, w)
    assert dx.shape == (n, cin, h, w) and dx.dtype == torch.float32
    assert torch.equal(dx, ops.stem_dgrad3x3s2(dy, slab, cin, h, w))             # deterministic
    # the weights the kernel multiplies by: unpacked from the patch slab (column (r*3+s)*cin + c)
    sl = slab if split else slab.unsqueeze(0)
    wh, wl = [sl[k, 0, :, :9 * cin].double().reshape(64, 3, 3, cin).permute(0, 3, 1, 2) for k in range(sl.shape[0])] \
        + [None] * (2 - sl.shape[0])
    dh, dl = _planes(dy)
    op = (h - (2 * ho - 1), w - (2 * wo - 1))

    def ct(a, b):
        return F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=op)
    ref, s = ct(dh, wh), ct(dh.abs(), wh.abs())
    if split:      # the conv kernels' three products: hi*hi + lo*hi + hi*lo
        ref = ref + ct(dl, wh) + ct(dh, wl)
        s = s + ct(dl.abs(), wh.abs()) + ct(dh.abs(), wl.abs())
    chain = 4 * 64 * (3 if split else 1)             # the longest fp32 chain: 4 taps x 64 channels x products
    bound = (chain + 2) * 2.0 ** -24 * s
    err = (dx.double() - ref).abs()
    assert bool((err <= bound).all()), float((err - bound).max())
    assert float(ref.abs().max()) > 0


# ------------------------------------------------------------------------------------------------ stem stage
@pytest.mark.parametrize("mode", ["batch", "frozen", "eval-net"])
def test_stem_stage_input_grad_vs_oracle(mode):
    from semseg_b200 import functional as SF
    from semseg_b200 import ops, precision
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(3, 64, 3, stride=2, padding=1, bias=False).cuda()
    bn = torch.nn.BatchNorm2d(64).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5), bn.bias.normal_(0, 0.2)
        bn.running_mean.normal_(0, 0.3), bn.running_var.uniform_(0.5, 2.0)
    bn.train(mode == "batch")
    x = torch.randn((2, 3, 65, 65), device="cuda", generator=g).requires_grad_(True)
    with precision.mode("bf16x3"), SF.network_mode(mode != "eval-net"):
        y = SF.stem_conv_bn_act(x, conv, bn, relu=True)
        gy = _act(torch.randn(tuple(y.shape[-4:]), device="cuda", generator=g), True)
        y.backward(gy)
    assert x.grad is not None and x.grad.shape == x.shape and x.grad.dtype == torch.float32
    xr = x.detach().clone().requires_grad_(True)
    z = F.batch_norm(F.conv2d(xr, conv.weight.detach(), None, 2, 1), bn.running_mean.clone(), bn.running_var.clone(),
                     bn.weight.detach(), bn.bias.detach(), mode == "batch", 0.1, 1e-5)
    mask = (ops.act_to_f32(y.detach()) > 0).permute(0, 3, 1, 2)          # the kernel's ReLU mask
    (z * mask).backward(ops.act_to_f32(gy).permute(0, 3, 1, 2))
    assert util.rel_l2(x.grad, xr.grad) <= 1e-3, util.rel_l2(x.grad, xr.grad)


# ------------------------------------------------------------------------------------------------ standalone modules
def _module_oracle(mod, prefix, **kw):
    from oracle.torch_oracle import Oracle
    sd = {prefix + k: v.detach().clone() for k, v in mod.state_dict().items()}
    return Oracle(sd, **kw).train()


@pytest.mark.parametrize("which", ["bottleneck-d2", "bottleneck-d4", "ppm", "psa", "stem"])
def test_standalone_module_input_grad(which):
    """A module called on its own on an fp32 NCHW input that needs a gradient (training mode, bf16x3): x.grad exists and
    agrees with the fp32 oracle."""
    from semseg_b200 import precision
    from semseg_b200.pspnet import PPM
    from semseg_b200.psanet import PSA
    from semseg_b200.resnet import Bottleneck, resnet50
    torch.manual_seed(0)
    g = torch.Generator(device="cuda").manual_seed(5)
    if which.startswith("bottleneck"):
        d = int(which[-1])
        mod = Bottleneck(256, 64).cuda().train()
        mod.conv2.dilation, mod.conv2.padding = (d, d), (d, d)
        x = torch.relu(torch.randn((2, 256, 17, 17), device="cuda", generator=g))
        orc = _module_oracle(mod, "b.")
        ref = lambda t: orc.bottleneck(t, "b", 1, d, False)                    # noqa: E731
    elif which == "ppm":
        mod = PPM(2048, 512, (1, 2, 3, 6)).cuda().train()
        x = torch.relu(torch.randn((2, 2048, 9, 9), device="cuda", generator=g))
        orc = _module_oracle(mod, "ppm.")
        ref = orc.ppm
    elif which == "psa":
        mod = PSA(2048, 512, 2, False, 2, 9, 9).cuda().train()
        x = torch.relu(torch.randn((2, 2048, 9, 9), device="cuda", generator=g))
        orc = _module_oracle(mod, "psa.", arch="psa", psa_type=2, mask_h=9, mask_w=9)
        ref = orc.psa
    else:
        mod = resnet50().stem().cuda().train()
        x = torch.randn((2, 3, 65, 65), device="cuda", generator=g)
        orc = _module_oracle(mod, "layer0.")

        def ref(t):
            t = orc.cbr(t, "layer0.0", "layer0.1", stride=2, padding=1)
            t = orc.cbr(t, "layer0.3", "layer0.4", padding=1)
            t = orc.cbr(t, "layer0.6", "layer0.7", padding=1)
            return F.max_pool2d(t, 3, 2, 1)
    xg = x.clone().requires_grad_(True)
    with precision.mode("bf16x3"):
        out = mod(xg)
    gy = torch.randn(out.shape, device="cuda", generator=g)
    out.backward(gy)
    xr = x.clone().requires_grad_(True)
    out_r = ref(xr)
    out_r.backward(gy)
    assert xg.grad is not None and xg.grad.shape == x.shape
    assert bool(torch.isfinite(xg.grad).all())
    assert util.rel_l2(out, out_r) < 1e-3, util.rel_l2(out, out_r)
    err = util.rel_l2(xg.grad, xr.grad)
    print("%s: x.grad rel-L2 %.3e" % (which, err))
    assert err < INPUT_GRAD_TOL, err


# ------------------------------------------------------------------------------------------------ eval networks
def _build(arch):
    from semseg_b200.psanet import PSANet
    if arch == "psp":
        return util.build_pspnet(50, 21), {}
    if arch == "psa-window":
        return util.build_psanet(50, 21), dict(mask_h=9, mask_w=9)
    torch.manual_seed(0)           # compact: 65 -> 9x9 features -> 5x5 after the 2x shrink, a dense 5x5 mask
    return (PSANet(layers=50, classes=21, zoom_factor=8, dropout=0.0, psa_type=2, compact=True, shrink_factor=2,
                   mask_h=5, mask_w=5, pretrained=False), dict(compact=True, mask_h=5, mask_w=5))


@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
@pytest.mark.parametrize("arch", ["psp", "psa-window", "psa-compact"])
def test_eval_network_input_grad(arch, prec):
    from semseg_b200 import precision
    model, okw = _build(arch)
    model = model.cuda().eval()
    for p in model.parameters():
        p.requires_grad_(False)
    orc = frozen_eval_oracle(model, "psp" if arch == "psp" else "psa", layers=50, classes=21, **okw)
    x, y = util.synth(2, 65, 65, 21, seed=4, device="cuda")
    with precision.mode(prec):
        with torch.no_grad():
            ref_out = model(x)
        xg = x.clone().requires_grad_(True)
        out = model(xg)
        assert out.requires_grad
        assert torch.equal(out.detach(), ref_out)            # the attack's forward is the eval forward, bit for bit
        F.cross_entropy(out, y, ignore_index=255).backward()
    assert xg.grad is not None and xg.grad.shape == x.shape and xg.grad.dtype == torch.float32
    assert all(p.grad is None for p in model.parameters())
    go = oracle_input_grad(orc, x, y)
    err = util.rel_l2(xg.grad, go)
    big = go.abs() > 0.1 * go.abs().max()
    sign = float((torch.sign(xg.grad[big]) == torch.sign(go[big])).double().mean())
    print("%s %s eval x.grad: rel-L2 %.3e, sign agreement %.4f on %d elements" % (arch, prec, err, sign, int(big.sum())))
    if prec == "bf16x3":
        assert err < INPUT_GRAD_TOL, err
    else:          # bf16 operands (8 mantissa bits) flip far more ReLU masks than the oracle's own floor
        assert err < 0.5, err
        assert sign > 0.9, sign


@pytest.mark.parametrize("arch", ["psp", "psa-window", "psa-compact"])
def test_eval_network_parameter_grads(arch):
    """Eval network, parameters and input need gradients: parameter gradients through the frozen-BN backward, against
    the oracle at the frozen-BN network tests' tolerances."""
    from semseg_b200 import precision
    model, okw = _build(arch)
    model = model.cuda().eval()
    orc, sd = frozen_oracle_from(model, "psp" if arch == "psp" else "psa", layers=50, classes=21, **okw)
    orc.eval()
    x, y = util.synth(2, 65, 65, 21, seed=4, device="cuda")
    xg = x.clone().requires_grad_(True)
    with precision.mode("bf16x3"):
        F.cross_entropy(model(xg), y, ignore_index=255).backward()
    xr = x.clone().requires_grad_(True)
    F.cross_entropy(orc.forward(xr), y, ignore_index=255).backward()
    assert util.rel_l2(xg.grad, xr.grad) < INPUT_GRAD_TOL
    errs, ratios = {}, {}
    for k, p in model.named_parameters():
        if k.startswith("aux."):
            assert p.grad is None, k                 # not part of the eval forward
            continue
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
        errs[k] = util.rel_l2(p.grad, sd[k].grad)
        ratios[k] = float(p.grad.double().norm() / sd[k].grad.double().norm().clamp_min(1e-30))
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    print("%s worst gradient rel-L2: %s" % (arch, ", ".join("%s %.2e" % kv for kv in worst)))
    assert all(v <= 0.35 for v in errs.values()), worst
    assert all(0.8 < v < 1.25 for v in ratios.values()), {k: v for k, v in ratios.items() if not 0.8 < v < 1.25}
    assert errs["cls.4.weight"] < 2e-2 and errs["cls.4.bias"] < 2e-2


# ------------------------------------------------------------------------------------------------ training
def test_training_frozen_bn_input_grad_vs_oracle(monkeypatch):
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = util.build_pspnet(50, 21).cuda().train()
    frozen = set()
    for name, m in model.named_modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()
            frozen.add(name)
    orc, _ = frozen_oracle_from(model, "psp", frozen=frozen, layers=50, classes=21)
    x, y = util.synth(2, 65, 65, 21, seed=4, device="cuda")
    xg = x.clone().requires_grad_(True)
    with precision.mode("bf16x3"):
        _, ml, al = model(xg, y)
        (ml + 0.4 * al).backward()
    xr = x.clone().requires_grad_(True)
    _, mlo, alo = orc.train().forward(xr, y)
    (mlo + 0.4 * alo).backward()
    err = util.rel_l2(xg.grad, xr.grad)
    print("train, frozen BN: x.grad rel-L2 %.3e" % err)
    assert err < INPUT_GRAD_TOL, err
    # batch statistics: x.grad exists, finite and non-zero
    model2 = util.build_pspnet(50, 21).cuda().train()
    xg2 = x.clone().requires_grad_(True)
    _, ml2, al2 = model2(xg2, y)
    (ml2 + 0.4 * al2).backward()
    assert xg2.grad is not None and bool(torch.isfinite(xg2.grad).all()) and float(xg2.grad.abs().max()) > 0


def _steps(model, batches, pattern):
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    out = []
    for k, want_dx in enumerate(pattern):
        x, y = batches[k % len(batches)]
        x = x.clone().requires_grad_(want_dx)
        _, ml, al = model(x, y)
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        grads = [None if p.grad is None else p.grad.clone() for p in model.parameters()]
        opt.step()
        out.append((ml.item(), al.item(), None if x.grad is None else x.grad.clone(), grads))
    return out


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_graphed_input_grad_steps_bit_identical_to_eager(arch, monkeypatch):
    """Adversarial-training steps: graphed and eager agree bit for bit on the losses, x.grad and every parameter
    gradient, also when x.requires_grad is toggled between steps (each setting has its own capture)."""
    from semseg_b200 import graphs
    build = util.build_pspnet if arch == "psp" else util.build_psanet
    base = build(50, 21).cuda().train()
    batches = [util.synth(2, 65, 65, 21, seed=s, device="cuda") for s in (1, 2, 3)]
    w = graphs.WARMUP_CALLS
    pattern = [True] * (w + 3) + [False] * (w + 2) + [True, False, True]
    eager = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    re_ = _steps(eager, batches, pattern)
    graphed = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    rg = _steps(graphed, batches, pattern)
    steps = [s for s in graphed.__dict__["_sb_graph_steps"].values() if s.fwd is not None]
    assert sorted(s.dx_slot for s in steps) == [False, True]              # one capture per setting
    for k, ((me, ae, xe, ge), (mg, ag, xg, gg)) in enumerate(zip(re_, rg)):
        assert (me, ae) == (mg, ag), k
        assert (xe is None) == (not pattern[k]) and (xg is None) == (not pattern[k]), k
        if xe is not None:
            assert torch.equal(xe, xg), k
        for a, b in zip(ge, gg):
            assert (a is None and b is None) or torch.equal(a, b), k


def test_input_without_grad_keeps_patch_stem(monkeypatch):
    """A training step whose input needs no gradient runs the patch-form stem and launches as many kernels as before a
    step with an input gradient ever ran; one whose input needs a gradient runs the phase form and the stem dgrad."""
    from semseg_b200 import _lib, ops
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = util.build_pspnet(50, 21).cuda().train()
    x, y = util.synth(2, 65, 65, 21, seed=1, device="cuda")
    calls = {"im2col": 0, "dgrad": 0}
    im2col, dgrad = ops.im2col3x3s2, ops.stem_dgrad3x3s2
    monkeypatch.setattr(ops, "im2col3x3s2", lambda *a: calls.__setitem__("im2col", calls["im2col"] + 1) or im2col(*a))
    monkeypatch.setattr(ops, "stem_dgrad3x3s2",
                        lambda *a: calls.__setitem__("dgrad", calls["dgrad"] + 1) or dgrad(*a))

    def step(want_dx):
        for k in calls:
            calls[k] = 0
        xi = x.clone().requires_grad_(want_dx)
        l0 = _lib.launch_count()
        _, ml, al = model(xi, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
        return _lib.launch_count() - l0, dict(calls)

    step(False)                                     # first call packs and allocates
    n0, c0 = step(False)
    n1, c1 = step(True)
    n2, c2 = step(False)
    assert c0 == {"im2col": 1, "dgrad": 0} and c2 == c0
    assert c1 == {"im2col": 0, "dgrad": 1}
    assert n2 == n0, (n0, n2)
    assert n1 > n0
