"""GPU tier: the CUDA-graph replay of a training step (semseg_b200/graphs.py) is the same computation as the eager path.

The kernels are deterministic, so three optimiser steps taken through the captured graphs must leave the model in
bit-identical state to three eager steps: losses, parameter gradients, updated weights, BatchNorm running statistics and
num_batches_tracked. Also: a changed input shape falls back to eager warm-up and captures a second graph; eval mode and
SEMSEG_B200_GRAPH=0 never capture. FusedSGD against torch.optim.SGD."""
import copy

import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


def _steps(model, batches, n_steps, lr=0.01):
    opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)
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


@pytest.mark.parametrize("arch, frozen_stem", [("psp", False), ("psa", False), ("psp", True)],
                         ids=["psp", "psa", "psp-frozen-stem"])
def test_graphed_steps_bit_identical_to_eager(arch, frozen_stem, monkeypatch):
    from semseg_b200 import graphs
    build = util.build_pspnet if arch == "psp" else util.build_psanet
    base = build(50, 21).cuda().train()
    if frozen_stem:
        # fine-tuning with a frozen stem conv whose BatchNorm keeps batch statistics: its weight never changes, so its
        # operand slabs (the patch slab included) are packed once, and the captured step must still own them
        base.layer0[0].weight.requires_grad_(False)
    batches = [util.synth(2, 65, 65, 21, seed=s, device="cuda") for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4                    # 3 eager warm-up calls, capture, then replays
    eager = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _steps(eager, batches, n_steps)
    assert graphs.launches_per_step(eager) == 0
    graphed = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _steps(graphed, batches, n_steps)
    assert graphs.launches_per_step(graphed) > 100       # the step really was captured and replayed
    assert le == lg, (le, lg)
    se, sg = eager.state_dict(), graphed.state_dict()
    for k in se:
        assert torch.equal(se[k], sg[k]), k              # weights, running statistics, num_batches_tracked
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert (pe.grad is None) == (pg.grad is None), k
        if pe.grad is not None:
            assert torch.equal(pe.grad, pg.grad), k
    # eval on the trained weights still goes through the eager single-kernel path and agrees
    eager.eval(), graphed.eval()
    with torch.no_grad():
        assert torch.equal(eager(batches[0][0]), graphed(batches[0][0]))
    # another input shape: eager warm-up again, then a second captured step; training continues to work
    graphed.train()
    other = [util.synth(2, 81, 81, 21, seed=9, device="cuda")]     # 81 -> 11x11 maps (PSA's 2x shrink needs an odd size)
    l2 = _steps(graphed, other, graphs.WARMUP_CALLS + 2)
    assert all(torch.isfinite(torch.tensor(v)).all() for v in l2)
    assert len([s for s in graphed.__dict__["_sb_graph_steps"].values() if s.fwd is not None]) == 2


def test_fused_sgd_matches_torch_sgd():
    """SURVEY §8 f4: FusedSGD (one launch) == torch.optim.SGD as configured at tool/train.py:140 (momentum 0.9, weight
    decay 1e-4, 8 groups whose learning rates change every iteration), bit for bit over several steps, and its state_dict
    loads into torch.optim.SGD."""
    from semseg_b200.optim import FusedSGD
    torch.manual_seed(0)
    shapes = [(64, 3, 3, 3), (64,), (256, 64, 1, 1), (150, 512, 1, 1), (150,), (512, 4096, 3, 3), (7,), (1000003,)]
    pa = [torch.nn.Parameter(torch.randn(s, device="cuda")) for s in shapes]
    pb = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    groups = lambda ps: [dict(params=ps[:3], lr=0.01), dict(params=ps[3:], lr=0.1)]      # noqa: E731
    oa = torch.optim.SGD(groups(pa), lr=0.01, momentum=0.9, weight_decay=1e-4)
    ob = FusedSGD(groups(pb), lr=0.01, momentum=0.9, weight_decay=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    for it in range(4):
        for a, b in zip(pa, pb):
            gr = torch.randn(a.shape, device="cuda", generator=g)
            a.grad, b.grad = gr.clone(), gr.clone()
        if it == 2:
            pa[1].grad = pb[1].grad = None           # a parameter without gradient is skipped
        v0 = pb[0]._version
        oa.step()
        ob.step()
        assert pb[0]._version > v0                   # the conv operand caches see the update
        for o in (oa, ob):                           # the trainer's poly schedule (tool/train.py:299-304)
            o.param_groups[0]["lr"] *= 0.9
            o.param_groups[1]["lr"] *= 0.9
        for a, b in zip(pa, pb):
            assert util.rel_l2(b, a) < 1e-6, it          # fused multiply-adds vs torch's separate roundings
    for a, b in zip(pa, pb):
        assert util.rel_l2(b, a) < 1e-6
        assert util.rel_l2(ob.state[b]["momentum_buffer"], oa.state[a]["momentum_buffer"]) < 1e-6
    oc = torch.optim.SGD(groups(pb), lr=0.01, momentum=0.9, weight_decay=1e-4)
    oc.load_state_dict(ob.state_dict())
    assert torch.equal(oc.state[pb[0]]["momentum_buffer"], ob.state[pb[0]]["momentum_buffer"])
