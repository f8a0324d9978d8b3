"""GPU tier: test-time adaptation (semseg_b200/adapt.py Tent) on PSPNet50 / PSANet50.

  * the constructor leaves exactly the listed BatchNorm gamma / beta trainable, the head dropouts in eval mode and the
    EntropyLoss installed;
  * a step changes only those parameters, launches no weight-gradient convolution, and equals one SGD step from the
    gradient of the entropy written in PyTorch on the ATen tail;
  * the prediction is the argmax of a same-mode forward before the update; reset() restores every parameter and buffer
    bit for bit; episodic calls repeat their predictions; the entropy falls; one input shape replays one graph."""
import copy

import pytest
import torch
from torch import nn

from tests import util
from tests.test_entropy_gpu import _torch_entropy_class
from tests.test_zoom_gpu import _batch, _build

pytestmark = pytest.mark.gpu

ADAPTED = ("layer0", "layer1", "layer2", "layer3", "layer4", "ppm", "psa", "cls")


def _bn_affine_names(model):
    names = set()
    for prefix in ADAPTED:
        mod = getattr(model, prefix, None)
        if mod is None:
            continue
        for mn, m in mod.named_modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                names.update("%s.%s%s" % (prefix, mn + "." if mn else "", k) for k in ("weight", "bias"))
    return names


def _x(seed=1, n=2, size=65):
    return _batch(8, seed=seed, n=n, size=size)[0]


def _n_graphs(model):
    return sum(1 for s in model.__dict__.get("_sb_graph_steps", {}).values() if s.fwd is not None)


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_tent_constructor_configures_the_model(arch):
    from semseg_b200.adapt import Tent
    from semseg_b200.losses import EntropyLoss
    from semseg_b200.optim import FusedSGD
    model = _build(arch, 8).cuda()
    model.eval()
    model.criterion = nn.CrossEntropyLoss(ignore_index=7)
    tent = Tent(model, lr=1e-3)
    trainable = {k for k, p in model.named_parameters() if p.requires_grad}
    expected = _bn_affine_names(model)
    assert trainable == expected and len(expected) > 100
    assert not any(k.startswith("aux.") for k in trainable) and "cls.4.bias" not in trainable
    assert model.training and all(m.training for m in model.modules()
                                  if isinstance(m, nn.modules.batchnorm._BatchNorm))
    assert not model.cls[3].training and not model.aux[3].training
    c = model.criterion
    assert type(c) is EntropyLoss and (c.ignore_index, c.ent_weight, c.ce_weight) == (7, 1.0, 0.0)
    assert isinstance(tent.optimizer, FusedSGD) and tent.optimizer.param_groups[0]["weight_decay"] == 0.0
    assert {id(p) for p in tent.optimizer.param_groups[0]["params"]} == {id(p) for p in model.parameters()
                                                                        if p.requires_grad}


def test_tent_step_changes_only_the_bn_affine_and_runs_no_wgrad(monkeypatch):
    from semseg_b200 import ops
    from semseg_b200.adapt import Tent
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _build("psp", 8).cuda()
    tent = Tent(model, lr=1e-2)
    before = {k: p.detach().clone() for k, p in model.named_parameters()}
    calls = []
    real = ops.conv_wgrad

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(ops, "conv_wgrad", counting)
    tent(_x())
    torch.cuda.synchronize()
    assert calls == []
    adapted = _bn_affine_names(model)
    changed = {k for k, p in model.named_parameters() if not torch.equal(p, before[k])}
    assert changed <= adapted and len(changed) > 0.9 * len(adapted)
    for k, p in model.named_parameters():
        if k not in adapted:
            assert torch.equal(p, before[k]), k                   # conv weights, cls bias, all of aux


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_tent_update_is_one_sgd_step_of_the_aten_entropy(arch, monkeypatch):
    from semseg_b200 import precision
    from semseg_b200.adapt import Tent
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _build(arch, 8).cuda()
    lr = 1.0                                    # the step is large against the parameters' fp32 rounding
    tent = Tent(model, lr=lr, momentum=0.9)
    ref = copy.deepcopy(model)
    ref.criterion = _torch_entropy_class()(ignore_index=255, ent_weight=1.0, ce_weight=0.0)
    x = _x(seed=3)
    y = torch.full((2, 65, 65), 255, dtype=torch.int64, device="cuda")
    p0 = {k: p.detach().clone() for k, p in model.named_parameters() if p.requires_grad}
    with precision.mode("bf16x3"):
        _, main_r, aux_r = ref(x, y)
        (main_r + aux_r).backward()
        tent(x)
    assert abs(tent.loss.item() - main_r.item()) <= 1e-5 * main_r.item()
    got = torch.cat([(p.detach() - p0[k]).flatten() for k, p in model.named_parameters() if p.requires_grad])
    want = torch.cat([(-lr * p.grad).flatten() for k, p in ref.named_parameters() if p.requires_grad])
    assert util.rel_l2(got, want) <= 1e-3, util.rel_l2(got, want)


def test_tent_prediction_is_the_forward_before_the_update(monkeypatch):
    from semseg_b200.adapt import Tent
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _build("psp", 8).cuda()
    tent = Tent(model, lr=1e-2)
    ref = copy.deepcopy(model)
    x = _x(seed=4)
    y = torch.full((2, 65, 65), 255, dtype=torch.int64, device="cuda")
    pred_ref, main_ref, _ = ref(x, y)
    pred = tent(x)
    assert pred.dtype == torch.int64 and pred.shape == (2, 65, 65)
    assert torch.equal(pred, pred_ref) and torch.equal(tent.loss, main_ref.detach())
    # the next call's prediction comes from the updated weights
    pred2 = tent(x)
    assert tent.loss.item() != main_ref.item() and pred2.shape == pred.shape


def test_tent_reset_restores_every_parameter_and_buffer():
    from semseg_b200 import graphs
    from semseg_b200.adapt import Tent
    model = _build("psa", 8).cuda()
    tent = Tent(model, lr=1e-2, steps=2)
    state = {k: v.detach().clone() for k, v in list(model.named_parameters()) + list(model.named_buffers())}
    x = _x(seed=5)
    for _ in range(graphs.WARMUP_CALLS + 2):                # eager calls, the capture, replays
        tent(x)
    assert any(not torch.equal(v, state[k]) for k, v in model.named_buffers())       # running statistics moved
    assert len(tent.optimizer.state) > 0
    tent.reset()
    for k, v in list(model.named_parameters()) + list(model.named_buffers()):
        assert torch.equal(v, state[k]), k
    assert len(tent.optimizer.state) == 0
    # after a reset the adaptation starts over: the same predictions as the first call
    fresh = Tent(_build("psa", 8).cuda(), lr=1e-2, steps=2)
    assert torch.equal(tent(x), fresh(x))


def test_tent_episodic_repeats_its_predictions():
    from semseg_b200 import graphs
    from semseg_b200.adapt import Tent
    model = _build("psp", 8).cuda()
    tent = Tent(model, lr=5e-2, episodic=True)
    x = _x(seed=6)
    preds = [tent(x) for _ in range(graphs.WARMUP_CALLS + 3)]
    losses = [tent.loss.item()]
    assert all(torch.equal(p, preds[0]) for p in preds[1:])
    assert _n_graphs(model) == 1
    tent.episodic = False
    tent(x)
    tent(x)
    losses.append(tent.loss.item())
    assert losses[1] != losses[0]


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_tent_entropy_falls_and_one_shape_replays_one_graph(arch):
    from semseg_b200 import graphs, precision
    from semseg_b200.adapt import Tent
    model = _build(arch, 8).cuda()
    tent = Tent(model, lr=1e-3, momentum=0.0)
    x = _x(seed=7, n=4)
    losses = []
    # bf16x3: in bf16 a small step also flips activation roundings, a loss jitter of the size of the step's decrease
    with precision.mode("bf16x3"), torch.no_grad():        # Tent enables autograd itself
        for _ in range(graphs.WARMUP_CALLS + 5):
            tent(x)
            losses.append(tent.loss.item())
    assert losses[-1] < losses[0], losses
    assert _n_graphs(model) == 1 and graphs.launches_per_step(model) > 100


def test_tent_rejects_bad_inputs():
    from semseg_b200.adapt import Tent
    tent = Tent(_build("psp", 8).cuda(), lr=1e-3)
    for bad in (torch.zeros((1, 3, 64, 65), device="cuda"), torch.zeros((1, 1, 65, 65), device="cuda"),
                torch.zeros((1, 3, 65, 65), device="cuda", dtype=torch.float16), torch.zeros((1, 3, 65, 65))):
        with pytest.raises(ValueError):
            tent(bad)
