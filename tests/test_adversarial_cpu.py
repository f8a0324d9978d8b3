"""CPU tier: the adversarial attack's oracles, options and C-ABI argument checks (no GPU).

  * the float64 SegPGD oracle (tests/adversarial_oracle.py) against torch autograd with detached weights at zoom 1, 2,
    4, 8, with ignored and out-of-range pixels, argmax ties, lambda 0 / 0.25 / 0.5 and no valid pixel;
  * the step and start formulas: sign(0) = 0, the ball before the box, constants rounded to fp32 once;
  * SegPGD's lambda schedule;
  * PGDAttack / AdversarialLoss argument validation and the graph key of every option;
  * semseg_adv_step, semseg_adv_start and semseg_upsample_segpgd_fwd reject bad arguments before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import adversarial_oracle as O


def _case(n, h, w, c, zoom, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn((n, h, w, c), generator=g) * 2
    if ties:                      # whole rows of equal logits: every class ties, the argmax is class 0
        logits[:, ::2] = 0.5
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    t = torch.randint(0, c, (n, ho, wo), generator=g)
    t[torch.rand((n, ho, wo), generator=g) < 0.1] = 255
    t[torch.rand((n, ho, wo), generator=g) < 0.01] = c + 2
    return logits, t


@pytest.mark.parametrize("lam", [0.0, 0.25, 0.5])
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
@pytest.mark.parametrize("ties", [False, True], ids=["distinct", "ties"])
def test_segpgd_oracle_matches_autograd(zoom, lam, ties):
    logits, t = _case(2, 5, 7, 6, zoom, seed=zoom * 10 + int(lam * 4), ties=ties)
    loss, n_valid, dl = O.segpgd_tail(logits, t, zoom, lam)
    l64 = logits.double().requires_grad_(True)
    v = O.upsample(l64, zoom)
    w, valid = O.segpgd_weights(v.detach(), t, 255, lam)          # detached: no gradient through the argmax
    tc = torch.where(valid, t, torch.zeros_like(t))
    nll = F.cross_entropy(v, tc, reduction="none")
    ref = (w * nll).sum() / valid.sum()
    ref.backward()
    assert n_valid == int(valid.sum()) > 0
    assert abs(float(loss) - float(ref.detach())) <= 1e-12 * abs(float(ref.detach()))
    assert float((dl - l64.grad).abs().max()) <= 1e-12 * float(l64.grad.abs().max())
    if ties:
        assert bool((v.detach().argmax(1)[:, ::zoom * 2] == 0).all())
    if lam == 0.0:    # only the correctly classified pixels count
        assert bool(((w > 0) == (valid & (v.detach().argmax(1) == t))).all())


def test_segpgd_lambda_half_is_half_the_cross_entropy():
    logits, t = _case(1, 6, 5, 4, 4, seed=3)
    loss, _, dl = O.segpgd_tail(logits, t, 4, 0.5)
    v = O.upsample(logits.double().requires_grad_(True), 4)
    valid = (t != 255) & (t < 4)
    ce = F.cross_entropy(v, torch.where(valid, t, torch.full_like(t, 255)), ignore_index=255).detach()
    assert abs(float(loss) - 0.5 * float(ce)) <= 1e-12


def test_segpgd_no_valid_pixel_is_zero():
    logits, t = _case(1, 4, 4, 3, 2, seed=5)
    t[:] = 255
    loss, n_valid, dl = O.segpgd_tail(logits, t, 2, 0.25)
    assert n_valid == 0 and float(loss) == 0.0 and float(dl.abs().max()) == 0.0


def test_lambda_schedule():
    from semseg_b200.adversarial import segpgd_lambdas
    assert segpgd_lambdas(1) == [0.0] == O.lambdas(1)
    assert segpgd_lambdas(4) == [0.0, 0.125, 0.25, 0.375] == O.lambdas(4)
    assert segpgd_lambdas(10)[-1] == 0.45


# ------------------------------------------------------------------------------------------------ step and start
MEAN, STD = (0.485 * 255, 0.456 * 255, 0.406 * 255), (0.229 * 255, 0.224 * 255, 0.225 * 255)


def test_box_constants_rounded_once_from_float64():
    from semseg_b200 import ops
    for eps, alpha in ((8.0, 2.0), (4.0, 1.0), (2.0, 0.5), (0.0, 1.0)):
        b = ops.adv_box(eps, alpha, MEAN, STD)
        ref = O.box(eps, alpha, MEAN, STD)
        for name, r in zip(("step", "eps", "lo", "hi"), ref):
            got = np.array(list(getattr(b, name)), dtype=np.float32)
            assert np.array_equal(got, r.numpy()), (name, got, r)
        # one rounding of the fp64 quotient, not a quotient of fp32-rounded operands
        s64 = np.float64(eps) / np.float64(STD[0])
        assert np.float32(b.eps[0]) == np.float32(s64)


def test_step_sign_of_zero_is_zero_and_ball_before_box():
    consts = O.box(8.0, 2.0, MEAN, STD)
    a, e, lo, hi = (float(v[0]) for v in consts)
    x0 = torch.tensor([0.0, 0.0, hi - a / 2, lo + a / 4], dtype=torch.float32)
    x0 = x0.view(1, 1, 2, 2).expand(1, 3, 2, 2).contiguous()
    g = torch.tensor([0.0, -0.0, 1.0, -3.0]).view(1, 1, 2, 2).expand(1, 3, 2, 2).contiguous()
    out = O.step(x0, g, x0, consts)
    assert torch.equal(out[0, 0].flatten()[:2], x0[0, 0].flatten()[:2])          # sign(+-0) = 0: x stays
    # a step past hi (or lo) inside the ball: the box holds
    assert float(out[0, 0, 1, 0]) == hi and float(out[0, 0, 1, 1]) == lo
    # the ball is applied before the box: a clean pixel outside the box (not a valid image) still ends inside it,
    # where box-then-ball would leave it at x0 - e > hi
    xo = torch.full((1, 3, 1, 1), hi + 3 * e)
    got = O.step(xo, torch.ones_like(xo), xo, consts)
    assert float(got[0, 0]) == hi
    box_first = torch.minimum(torch.maximum(torch.clamp(xo + a, lo, hi), xo - e), xo + e)
    assert float(box_first[0, 0]) > hi


def test_start_stays_in_ball_and_box():
    consts = O.box(8.0, 2.0, MEAN, STD)
    g = torch.Generator().manual_seed(0)
    x0 = (torch.randn((2, 3, 9, 9), generator=g) * 2).clamp(-1.9, 2.0)     # a valid image: inside the box
    u = torch.rand((2, 3, 9, 9), generator=g)
    x = O.start(x0, u, consts)
    _, e, lo, hi = (O._c(t, x0) for t in consts)
    assert bool(((x >= x0 - e) | (x == lo)).all()) and bool(((x <= x0 + e) | (x == hi)).all())
    assert bool(((x >= lo) & (x <= hi)).all())


# ------------------------------------------------------------------------------------------------ options
def test_pgd_attack_validation():
    from semseg_b200.adversarial import PGDAttack
    PGDAttack(8, 2, 10)
    PGDAttack(0, 1.0, 1, random_start=False)
    for kw, exc in ((dict(eps=-1.0), ValueError), (dict(eps="8"), TypeError), (dict(eps=float("nan")), ValueError),
                    (dict(eps=True), TypeError), (dict(alpha=0.0), ValueError), (dict(alpha=-1), ValueError),
                    (dict(alpha=float("inf")), ValueError), (dict(steps=0), ValueError), (dict(steps=2.0), TypeError),
                    (dict(steps=True), TypeError), (dict(kind="fgsm"), ValueError), (dict(kind=1), TypeError),
                    (dict(random_start=1), TypeError), (dict(mean=(1.0, 2.0)), TypeError),
                    (dict(mean="abc"), TypeError), (dict(mean=(1.0, float("nan"), 2.0)), ValueError),
                    (dict(std=(1.0, 0.0, 1.0)), ValueError), (dict(std=(1.0, -1.0, 1.0)), ValueError),
                    (dict(std=(1.0, 1.0, float("inf"))), ValueError), (dict(ignore_index=1.5), TypeError),
                    (dict(ignore_index=True), TypeError)):
        args = dict(eps=8.0, alpha=2.0, steps=3)
        args.update(kw)
        with pytest.raises(exc):
            PGDAttack(**args)


def test_adversarial_loss_validation():
    from semseg_b200.adversarial import PGDAttack
    from semseg_b200.losses import AdversarialLoss
    a = PGDAttack(8, 2, 3)
    assert AdversarialLoss(a).attack is a and AdversarialLoss(a).last_adv() is None
    with pytest.raises(TypeError):
        AdversarialLoss(None)
    with pytest.raises(TypeError):
        AdversarialLoss(a, ignore_index="255")
    with pytest.raises(TypeError):
        AdversarialLoss(a, ignore_index=False)


def test_graph_key_changes_with_every_option():
    from semseg_b200.adversarial import PGDAttack
    from semseg_b200.losses import AdversarialLoss, graph_key
    base = dict(eps=8.0, alpha=2.0, steps=3, kind="pgd", random_start=True, mean=MEAN, std=STD, ignore_index=255)
    changes = dict(eps=4.0, alpha=1.0, steps=2, kind="segpgd", random_start=False, mean=(1.0, 2.0, 3.0),
                   std=(50.0, 60.0, 70.0), ignore_index=0)
    k0 = graph_key(AdversarialLoss(PGDAttack(**base)))
    assert k0 == graph_key(AdversarialLoss(PGDAttack(**base)))
    keys = {k0}
    for name, v in changes.items():
        kw = dict(base)
        kw[name] = v
        k = graph_key(AdversarialLoss(PGDAttack(**kw)))
        assert k != k0, name
        keys.add(k)
        assert PGDAttack(**kw).key() != PGDAttack(**base).key(), name
    assert graph_key(AdversarialLoss(PGDAttack(**base), ignore_index=0)) != k0
    assert len(keys) == len(changes) + 1


def test_fused_tail_takes_adversarial_loss():
    from semseg_b200 import functional as SF
    from semseg_b200.adversarial import PGDAttack
    from semseg_b200.losses import AdversarialLoss
    crit = AdversarialLoss(PGDAttack(8, 2, 1))
    y = torch.zeros((2, 65, 65), dtype=torch.int64)
    assert SF.fused_tail_supported(crit, None, y, 8, (2, 3, 65, 65))
    assert not SF.fused_tail_supported(crit, None, y[:, :64], 8, (2, 3, 65, 65))


# ------------------------------------------------------------------------------------------------ C-ABI
def test_new_entry_points_validate_before_any_cuda_call():
    from semseg_b200 import _lib, ops
    lib = _lib.load()
    err = lambda: lib.semseg_last_error()      # noqa: E731
    P, Q = ctypes.c_void_p(16), ctypes.c_void_p(18)
    good = ops.adv_box(8.0, 2.0, MEAN, STD)
    b = ctypes.byref(good)
    assert lib.semseg_adv_step(P, P, P, P, 1, 5, 5, None, None) == -1 and b"null constants" in err()
    assert lib.semseg_adv_step(None, P, P, P, 1, 5, 5, b, None) == -1 and b"adv_step: null pointer" in err()
    assert lib.semseg_adv_step(P, P, Q, P, 1, 5, 5, b, None) == -1 and b"4-byte aligned" in err()
    assert lib.semseg_adv_step(P, P, P, P, 0, 5, 5, b, None) == -1 and b"bad shape" in err()
    assert lib.semseg_adv_step(P, P, P, P, 21846, 5, 5, b, None) == -1 and b"bad shape" in err()
    for field, k, v in (("eps", 1, -1.0), ("step", 2, float("nan")), ("lo", 0, float("inf")), ("hi", 0, -1e9)):
        bad = ops.adv_box(8.0, 2.0, MEAN, STD)
        getattr(bad, field)[k] = v
        assert lib.semseg_adv_step(P, P, P, P, 1, 5, 5, ctypes.byref(bad), None) == -1, field
        assert b"adv_step" in err()
    assert lib.semseg_adv_start(P, None, P, 1, 5, 5, b, None) == -1 and b"adv_start: null pointer" in err()
    assert lib.semseg_adv_start(P, P, P, 1, -5, 5, b, None) == -1 and b"bad shape" in err()
    # semseg_upsample_segpgd_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, zoom, ignore, lambda, ws, loss, amax, lse,
    #                            mod, stream)
    args = lambda **kw: [kw.get(k, d) for k, d in (                      # noqa: E731
        ("logits", P), ("pitch", 21), ("N", 1), ("h", 9), ("w", 9), ("C", 21), ("t", P), ("Ho", 65), ("Wo", 65),
        ("zoom", 8), ("ign", 255), ("lam", 0.25), ("ws", P), ("loss", P), ("amax", None), ("lse", P), ("mod", P),
        ("stream", None))]
    assert lib.semseg_upsample_segpgd_fwd(*args(zoom=3)) == -1 and b"zoom" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(Ho=64)) == -1 and b"Ho=8(h-1)+1" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(lam=1.5)) == -1 and b"lambda" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(lam=float("nan"))) == -1 and b"lambda" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(mod=None)) == -1 and b"null output" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(mod=Q)) == -1 and b"aligned" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(logits=None)) == -1 and b"null pointer" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(C=300, pitch=300)) == -1 and b"bad sizes" in err()
    assert lib.semseg_upsample_segpgd_fwd(*args(w=400, Wo=3193)) == -1 and b"too large" in err()
