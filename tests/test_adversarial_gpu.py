"""GPU tier (-m gpu): PGD / SegPGD attacks and PGD adversarial training (semseg_b200/adversarial.py,
losses.AdversarialLoss, csrc/adversarial.cu, the SegPGD tail of csrc/tail.cu). Small shapes: 65x65, 21 classes.

  1. the step and start kernels bit-identical to the torch fp32 formula, zero gradients and ball / box clamps included;
  2. the SegPGD forward and backward against the float64 oracle at zoom 1, 2, 4, 8;
  3. kind='pgd' in bf16x3: one iteration's dx against this package's eval-differentiable forward plus ATen's
     F.cross_entropy on the upsampled logits;
  4. the graphed attack bit-identical to the eager one (both kinds, random start on / off, PSPNet / PSANet, zoom 8 and 4),
     also after an in-place weight edit between replays;
  5. invariants: ball and box exactly, parameters / buffers / .grad / modes unchanged, no wgrad kernel, eps = 0;
  6. adversarial training graphed vs eager over several steps: losses, gradients, running statistics, last_adv();
  7. one AdversarialLoss step == the standalone attack then a plain-CE step, over several optimizer steps;
  8. the adversarial step's launches = the plain step's + K iterations + the start;
  9. a training model with BatchNorm layers individually in eval keeps them so."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests import adversarial_oracle as O
from tests import util
from tests.test_zoom_gpu import _batch, _build, _logits, _target

pytestmark = pytest.mark.gpu

MEAN, STD = (0.485 * 255, 0.456 * 255, 0.406 * 255), (0.229 * 255, 0.224 * 255, 0.225 * 255)


@pytest.fixture(autouse=True)
def _strict_fp32():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _image_batch(zoom=8, seed=1, n=2):
    """A normalised batch of valid images (pixels in [0, 255]) and its target at zoom `zoom`."""
    x, y = _batch(zoom, seed=seed, n=n)
    g = torch.Generator(device="cuda").manual_seed(seed)
    pix = torch.rand(x.shape, device="cuda", generator=g) * 255
    m = torch.tensor(MEAN, device="cuda").view(1, 3, 1, 1)
    s = torch.tensor(STD, device="cuda").view(1, 3, 1, 1)
    return ((pix - m) / s).contiguous(), y


def _consts():
    return tuple(t.cuda() for t in O.box(8.0, 2.0, MEAN, STD))


# ------------------------------------------------------------------------------------------------ 1. step / start
def test_step_and_start_kernels_bit_identical_to_torch():
    from semseg_b200 import ops
    consts = _consts()
    box = ops.adv_box(8.0, 2.0, MEAN, STD)
    g = torch.Generator(device="cuda").manual_seed(0)
    for shape in ((2, 3, 65, 65), (1, 3, 7, 5), (3, 3, 129, 33)):
        x0, _ = _image_batch() if shape == (2, 3, 65, 65) else (None, None)
        if x0 is None:
            x0 = torch.rand(shape, device="cuda", generator=g) * 4 - 2
        x0 = x0.clone()
        x0.view(-1)[:7] = torch.tensor([-2.2, 2.3, -2.04, 2.64, 0.0, 1.0, -1.0], device="cuda")   # at / beyond the box
        x = (x0 + (torch.rand(x0.shape, device="cuda", generator=g) - 0.5) * 0.2).contiguous()
        grad = torch.randn(x0.shape, device="cuda", generator=g)
        grad[torch.rand(x0.shape, device="cuda", generator=g) < 0.2] = 0.0                   # sign(0) = 0
        grad.view(-1)[:3] = torch.tensor([0.0, -0.0, 1e-40], device="cuda")
        ref = O.step(x, grad, x0, consts)
        assert torch.equal(ops.adv_step(x, grad, x0, box), ref), shape
        xi = x.clone()
        ops.adv_step(xi, grad, x0, box, out=xi)                                             # in place
        assert torch.equal(xi, ref)
        # many steps: the ball clamps bind
        for _ in range(8):
            xi = ops.adv_step(xi, torch.ones_like(grad), x0, box)
            ref = O.step(ref, torch.ones_like(grad), x0, consts)
        assert torch.equal(xi, ref)
        e, hi = consts[1].view(1, 3, 1, 1), consts[3].view(1, 3, 1, 1)
        assert bool(((xi == x0 + e) | (xi == hi)).float().mean() > 0.9)
        u = torch.rand(x0.shape, device="cuda", generator=g)
        u.view(-1)[:2] = torch.tensor([0.0, 0.9999999], device="cuda")
        assert torch.equal(ops.adv_start(x0, u, box), O.start(x0, u, consts)), shape


# ------------------------------------------------------------------------------------------------ 2. SegPGD tail
@pytest.mark.parametrize("lam", [0.0, 0.25, 0.45])
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_segpgd_tail_vs_oracle(zoom, lam):
    from semseg_b200 import ops
    for (n, h, w, c, pitch) in ((2, 9, 13, 21, 24), (1, 6, 140, 150, 152)):
        logits = _logits(n, h, w, c, pitch, seed=zoom + 3)
        target = _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom + 3)
        info, amax, lse, mod = ops.upsample_segpgd_fwd(logits, target, 255, lam, zoom=zoom)
        dl = ops.upsample_ce_focal_bwd(logits, target, 255, lse, mod, info, torch.tensor([0.7], device="cuda"),
                                       zoom=zoom)
        loss_o, n_valid, dl_o = O.segpgd_tail(logits, target, zoom, lam)
        assert info[1].item() == n_valid > 0
        # the same tolerances as the focal tail (tests/test_focal_gpu.py)
        assert abs(info[0].item() - loss_o.item()) <= 2e-6 * abs(loss_o.item())
        assert float((dl.double().cpu() - 0.7 * dl_o).abs().max()) <= 5e-6 * float(0.7 * dl_o.abs().max())
        # the plain forward's lse and argmax bits
        info_p, amax_p, lse_p = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
        assert torch.equal(lse, lse_p) and torch.equal(amax, amax_p)
        valid = (target != 255) & (target >= 0) & (target < c)
        hit = amax == target
        assert bool((mod[valid & hit] == 1 - lam).all()) and bool((mod[valid & ~hit] == lam).all())
        assert float(mod[~valid].abs().max()) == 0.0
    t0 = torch.full_like(target, 255)
    info, _, lse, mod = ops.upsample_segpgd_fwd(logits, t0, 255, lam, zoom=zoom)
    dl = ops.upsample_ce_focal_bwd(logits, t0, 255, lse, mod, info, torch.tensor([1.0], device="cuda"), zoom=zoom)
    assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ 3. dx vs ATen tail
# rel-L2 bound of one PGD iteration's dx (bf16x3, fused tail) against the same network's eval-differentiable forward with
# ATen's upsample + F.cross_entropy: the network bits are the same, only the tail's arithmetic differs (MUFU exp / log,
# summation order). Measured on an H100: 1.6e-5 (PSPNet50) and 1.7e-5 (PSANet50), between tests/input_grad_floor.py's
# floors at a 1e-6 relative input perturbation (~1e-6) and at bf16x3's operand rounding (9.5e-3): the tail's last-bit
# differences flip a few ReLU masks. The bound is 6x the measured value
DX_TAIL_TOL = 1e-4


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_pgd_iteration_dx_matches_aten_tail(arch, monkeypatch):
    from semseg_b200 import adversarial, precision
    from semseg_b200 import functional as SF
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _build(arch, 8).cuda().eval()
    x, y = _image_batch()
    with precision.mode("bf16x3"):
        SF.prepack(model)
        with adversarial.constant_parameters(model), SF.network_mode(False, input_grad=True):
            xf = x.clone().requires_grad_(True)
            loss, _ = SF._UpsampleCE.apply(model._logits_nhwc(xf)[0], y, 255, 8)
            (g_fused,) = torch.autograd.grad(loss, xf)
            xa = x.clone().requires_grad_(True)
            up = model._logits_nhwc(xa)[0].permute(0, 3, 1, 2)
            up = F.interpolate(up, size=y.shape[1:], mode="bilinear", align_corners=True)
            (g_aten,) = torch.autograd.grad(F.cross_entropy(up, y, ignore_index=255), xa)
        err = util.rel_l2(g_fused, g_aten)
        print("dx rel-L2 fused vs ATen tail (%s): %.3e" % (arch, err))
        assert err <= DX_TAIL_TOL, err
        # and one iteration through PGDAttack is the sign step of that gradient
        atk = adversarial.PGDAttack(8, 2, 1, random_start=False)
        x_adv = atk(model, x, y)
        ref = O.step(x, g_fused, x, _consts())
        assert float((x_adv != ref).float().mean()) < 1e-3           # signs of near-zero gradients may differ


# ------------------------------------------------------------------------------------------------ 4. graphed vs eager
def _attack_runs(model, atk, x, y, n, graph, monkeypatch, seed=7):
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
    out = []
    for k in range(n):
        torch.manual_seed(seed + k)
        out.append((atk(model, x, y), atk.losses))
    return out


@pytest.mark.parametrize("arch, zoom", [("psp", 8), ("psa", 8), ("psp", 4)])
@pytest.mark.parametrize("kind", ["pgd", "segpgd"])
@pytest.mark.parametrize("random_start", [True, False], ids=["rs", "no-rs"])
def test_graphed_attack_bit_identical_to_eager(arch, zoom, kind, random_start, monkeypatch):
    from semseg_b200 import adversarial, graphs
    model = _build(arch, zoom).cuda().eval()
    x, y = _image_batch(zoom)
    atk = adversarial.PGDAttack(8, 2, 3, kind=kind, random_start=random_start)
    n = graphs.WARMUP_CALLS + 3
    eager = _attack_runs(model, atk, x, y, n, False, monkeypatch)
    graphed = _attack_runs(model, atk, x, y, n, True, monkeypatch)
    assert sum(1 for s in model._sb_adv_graphs.values() if s.graph is not None) == 1
    for (xe, le), (xg, lg) in zip(eager, graphed):
        assert torch.equal(xe, xg) and torch.equal(le, lg)
    assert not torch.equal(eager[0][0], x)
    if random_start:
        assert not torch.equal(graphed[-1][0], graphed[-2][0])          # fresh draws every replay
    # an in-place weight edit between replays is seen
    with torch.no_grad():
        model.cls[4].weight.mul_(1.5)
        model.layer1[0].conv1.weight.mul_(0.9)
    e2 = _attack_runs(model, atk, x, y, 2, False, monkeypatch, seed=50)
    g2 = _attack_runs(model, atk, x, y, 2, True, monkeypatch, seed=50)
    for (xe, le), (xg, lg) in zip(e2, g2):
        assert torch.equal(xe, xg) and torch.equal(le, lg)
    assert sum(1 for s in model._sb_adv_graphs.values() if s.graph is not None) == 1
    assert not torch.equal(e2[0][1], eager[0][1])


# ------------------------------------------------------------------------------------------------ 5. invariants
def test_attack_invariants(monkeypatch):
    from semseg_b200 import adversarial, graphs, ops
    model = _build("psp", 8).cuda().eval()
    for p in model.parameters():
        p.grad = torch.full_like(p, 0.25)
    model.layer2[0].conv1.weight.requires_grad_(False)
    before = copy.deepcopy(model.state_dict())
    modes = [m.training for m in model.modules()]
    grads = [p.grad.clone() for p in model.parameters()]
    x, y = _image_batch()
    calls = {"wgrad": 0}
    real = ops.conv_wgrad

    def counting(*a, **k):
        calls["wgrad"] += 1
        return real(*a, **k)
    monkeypatch.setattr(ops, "conv_wgrad", counting)
    consts = _consts()
    for graph in (False, True):
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "1" if graph else "0")
        for kind in ("pgd", "segpgd"):
            atk = adversarial.PGDAttack(8, 2, 4, kind=kind)
            for _ in range(graphs.WARMUP_CALLS + 2 if graph else 1):
                xa = atk(model, x, y)
            e, lo, hi = (c.view(1, 3, 1, 1) for c in consts[1:])
            assert bool((xa >= x - e).all()) and bool((xa <= x + e).all())
            assert bool((xa >= lo).all()) and bool((xa <= hi).all())
            assert xa.dtype == torch.float32 and not xa.requires_grad and atk.losses.shape == (4,)
            assert atk.losses.device.type == "cuda"
    assert calls["wgrad"] == 0
    after = model.state_dict()
    for k, v in before.items():
        assert torch.equal(v, after[k]), k
    assert [m.training for m in model.modules()] == modes
    assert all(torch.equal(p.grad, g) for p, g in zip(model.parameters(), grads))
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    zero = adversarial.PGDAttack(0, 2, 3)
    assert torch.equal(zero(model, x, y), x)
    # a non-contiguous input (channels-last strides, as a permuted image batch has) attacks like its contiguous copy
    torch.manual_seed(3)
    ref = adversarial.PGDAttack(8, 2, 2)(model, x, y)
    torch.manual_seed(3)
    assert torch.equal(adversarial.PGDAttack(8, 2, 2)(model, x.to(memory_format=torch.channels_last), y), ref)


def test_attack_rejects_bad_models_and_inputs():
    from semseg_b200 import adversarial
    from semseg_b200.fp8 import Fp8Eval
    model = _build("psp", 8).cuda()
    x, y = _image_batch()
    atk = adversarial.PGDAttack(8, 2, 1)
    with pytest.raises(RuntimeError, match="eval mode"):
        atk(model.train(), x, y)
    model.eval()
    model.layer1[0].bn1.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        atk(model, x, y)
    model.eval()
    with pytest.raises(TypeError, match="bare network"):
        atk(torch.nn.DataParallel(model), x, y)
    with pytest.raises(TypeError, match="Fp8Eval"):
        atk(Fp8Eval(model), x, y)
    with pytest.raises(ValueError, match="8k\\+1"):
        atk(model, x[:, :, :64], y)
    with pytest.raises(ValueError, match="target"):
        atk(model, x, y[:, :64])


# ------------------------------------------------------------------------------------------------ 6-9. training
def _adv_model(arch="psp", zoom=8, kind="pgd", steps=2):
    from semseg_b200.adversarial import PGDAttack
    from semseg_b200.losses import AdversarialLoss
    model = _build(arch, zoom).cuda().train()
    model.criterion = AdversarialLoss(PGDAttack(8, 2, steps, kind=kind))
    return model


def _train(model, batches, n_steps, seed=11):
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    out = []
    for k in range(n_steps):
        x, y = batches[k % len(batches)]
        torch.manual_seed(seed + k)
        _, ml, al = model(x, y)
        opt.zero_grad()
        (ml + 0.4 * al).backward()
        grads = [None if p.grad is None else p.grad.clone() for p in model.parameters()]
        opt.step()
        rec = model.criterion.last_adv() if hasattr(model.criterion, "last_adv") else None
        out.append((ml.item(), al.item(), grads, None if rec is None else (rec["image"].clone(), rec["losses"].clone())))
    return out


@pytest.mark.parametrize("kind", ["pgd", "segpgd"])
def test_adversarial_training_graphed_bit_identical_to_eager(kind, monkeypatch):
    from semseg_b200 import graphs
    base = _adv_model(kind=kind)
    batches = [_image_batch(seed=s) for s in (1, 2)]
    n = graphs.WARMUP_CALLS + 3
    eager, graphed = copy.deepcopy(base), copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    re_ = _train(eager, batches, n)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    rg = _train(graphed, batches, n)
    assert graphs.launches_per_step(graphed) > 100
    for k, (a, b) in enumerate(zip(re_, rg)):
        assert a[0] == b[0] and a[1] == b[1], k
        assert all((ga is None) == (gb is None) and (ga is None or torch.equal(ga, gb)) for ga, gb in zip(a[2], b[2])), k
        assert torch.equal(a[3][0], b[3][0]) and torch.equal(a[3][1], b[3][1]), k
    for (name, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), name


def test_adversarial_step_is_attack_then_plain_step(monkeypatch):
    """Seed, one AdversarialLoss step on (x, y) == reseed, the standalone attack on the eval model, then a plain-CE
    step on (x_adv, y): over several optimizer steps, so the attack inside the step sees the re-packed weights."""
    from semseg_b200 import adversarial
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    adv = _adv_model(steps=2)
    atk = adv.criterion.attack
    plain = copy.deepcopy(adv)
    plain.criterion = torch.nn.CrossEntropyLoss(ignore_index=255)
    oa = torch.optim.SGD(adv.parameters(), lr=0.05, momentum=0.9)
    op = torch.optim.SGD(plain.parameters(), lr=0.05, momentum=0.9)
    for k in range(3):
        x, y = _image_batch(seed=k + 1)
        torch.manual_seed(100 + k)
        _, ma, aa = adv(x, y)
        oa.zero_grad()
        (ma + 0.4 * aa).backward()
        torch.manual_seed(100 + k)
        plain.eval()
        x_adv = adversarial.PGDAttack(atk.eps, atk.alpha, atk.steps)(plain, x, y)
        plain.train()
        _, mp, ap = plain(x_adv, y)
        op.zero_grad()
        (mp + 0.4 * ap).backward()
        assert torch.equal(adv.criterion.last_adv()["image"], x_adv), k
        assert ma.item() == mp.item() and aa.item() == ap.item(), k
        for (n_, pa), (_, pp) in zip(adv.named_parameters(), plain.named_parameters()):
            assert torch.equal(pa.grad, pp.grad), (k, n_)
        oa.step()
        op.step()


def test_adversarial_step_launch_count(monkeypatch):
    from semseg_b200 import _lib, adversarial, graphs
    from semseg_b200 import functional as SF
    x, y = _image_batch()
    counts = {}
    for name, steps in (("plain", 0), ("k1", 1), ("k3", 3)):
        model = _build("psp", 8).cuda().train() if steps == 0 else _adv_model(steps=steps)
        for _ in range(graphs.WARMUP_CALLS + 2):
            _, ml, al = model(x, y)
            (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
        counts[name] = graphs.launches_per_step(model)
    # one eager iteration of the attack alone (the packs are current: no re-pack launch)
    model = _build("psp", 8).cuda().eval()
    SF.prepack(model)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    l0 = _lib.launch_count()
    adversarial.run(model, adversarial.PGDAttack(8, 2, 1, random_start=False), x, y)
    per_iter = _lib.launch_count() - l0
    assert per_iter > 50
    assert counts["k1"] == counts["plain"] + per_iter + 1, (counts, per_iter)
    assert counts["k3"] == counts["plain"] + 3 * per_iter + 1, (counts, per_iter)


def test_adversarial_step_keeps_frozen_batchnorm_modes(monkeypatch):
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _adv_model(steps=1)
    frozen = [model.layer0[1], model.layer1[0].bn2, model.layer3[1].bn1]
    for m in frozen:
        m.eval()
    modes = [m.training for m in model.modules()]
    x, y = _image_batch()
    _, ml, al = model(x, y)
    (ml + 0.4 * al).backward()
    assert [m.training for m in model.modules()] == modes
    assert model.training and not any(m.training for m in frozen)
    with pytest.raises(RuntimeError, match="requires grad|require grad"):
        model(x.clone().requires_grad_(True), y)
