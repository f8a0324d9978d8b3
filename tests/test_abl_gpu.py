"""GPU tier: the Active Boundary Loss (losses.ActiveBoundaryLoss) on the fused tail: the plain cross-entropy kernels
plus csrc/boundary.cu, graphed.

  * the distance map is bit-equal to the float64 contract of tests/abl_oracle.py (scipy's exact EDT) at 473^2, 713^2
    and odd non-square grids, ignore blobs and a boundary-free image included;
  * the boundary score k is the contract's within 1e-5 relative or 1e-7 absolute at zoom 1, where the kernel reads
    the oracle's logits; at zoom > 1 the kernel's grid logits are the tail's fp32 interpolation, whose rounding
    (measured up to 1.7 times the zoom-1 gate) the gate triples; given the kernel's own k, the level j*, the
    dilation B, the directions and the selected set are the contract's exactly;
  * loss within 1e-5 relative and dlogits within 1e-4 of max |grad| at zoom 1 / 2 / 4 / 8 and 2 / 19 / 150 / 256
    classes, a padded pitch, M = 0 and a batch without any GT boundary;
  * PSPNet50 / PSANet50 steps: graphed equal to eager, two runs bit-identical, abl_weight = 0 bit-identical to the
    nn.CrossEntropyLoss step; the module form against the contract."""
import copy

import numpy as np
import pytest
import torch

from tests import abl_oracle as O
from tests.gatedcrf_oracle import upsample
from tests.test_abl_cpu import _labels
from tests.test_zoom_gpu import _batch, _build, _sgd_steps

pytestmark = pytest.mark.gpu

LOSS_GATE, GRAD_GATE = 1e-5, 1e-4      # relative loss, dlogits over max |dlogits|
K_REL, K_ABS = 1e-5, 1e-7             # k at zoom 1; x3 at zoom > 1 (the fp32 interpolated grid logits)
_worst = {"loss": 0.0, "grad": 0.0, "k": 0.0}


def _logits(n, h, w, c, seed, pitch=None, scale=2.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn((n, h, w, pitch or c), device="cuda", generator=g) * scale
    return base[..., :c]


def _target(n, hg, wg, c, seed, uniform_first=False):
    t = torch.from_numpy(_labels(n, hg, wg, c, seed)).cuda()
    if uniform_first:
        t[0] = 0
    return t.contiguous()


def _forward(logits, target, zoom, ratio=0.05, clip=20.0, eps=0.2):
    from semseg_b200 import ops
    n, h, w, _ = logits.shape
    hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    _, _, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    info, state = ops.abl_fwd(logits, lse, target, 255, zoom, ratio, clip, eps)
    maps = {k: v.clone() for k, v in ops.abl_maps(state, n, hg, wg).items()}
    return info, maps


def _grid(logits, zoom):
    return upsample(logits.detach().permute(0, 3, 1, 2).cpu(), zoom)


@pytest.mark.parametrize("case", [(2, 60, 60, 8), (1, 90, 90, 8), (3, 97, 61, 1), (2, 13, 40, 4), (1, 2, 7, 2)],
                         ids=["473", "713", "97x61", "49x157", "3x13"])
def test_distance_map_bit_equal(case):
    n, h, w, zoom = case
    hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    t = _target(n, hg, wg, 5, seed=h + w, uniform_first=n > 1)
    _, maps = _forward(_logits(n, h, w, 3, seed=1), t, zoom)
    ref = O.dist_map(t.cpu().numpy(), 255)
    got = maps["D"].cpu().numpy()
    assert np.array_equal(got, ref), np.argwhere(got != ref)[:5]
    if n > 1:
        assert np.isinf(got[0]).all() and (maps["code"][0] & 15 == 15).all()


@pytest.mark.parametrize("zoom,classes", [(1, 19), (2, 150), (4, 21), (8, 19), (8, 150)])
def test_score_map_and_selection(zoom, classes):
    n, h, w = 2, (37 if zoom == 1 else 80 // zoom + 1), (29 if zoom == 1 else 64 // zoom + 1)
    hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, classes, seed=zoom + classes)
    t = _target(n, hg, wg, 6, seed=3)
    ratio = 0.03
    _, maps = _forward(logits, t, zoom, ratio=ratio)
    k = maps["k"].cpu()
    ref = O.kl_map(_grid(logits, zoom))
    err = (k.double() - ref).abs()
    widen = 1.0 if zoom == 1 else 3.0
    tol = torch.clamp(widen * K_REL * ref.abs(), min=widen * K_ABS)
    _worst["k"] = max(_worst["k"], float((err / tol).max()))
    print("k: worst error %.2f of its gate" % _worst["k"])
    assert bool((err <= tol).all()), float((err / tol).max())
    kn = k.numpy()
    jstar = O.level(kn, ratio * hg * wg)
    assert int(maps["jstar"].item()) == jstar
    B, direction, sel = O.selection(kn, maps["D"].cpu().numpy(), jstar)
    code = maps["code"].cpu().numpy()
    assert np.array_equal((code >> 4) & 1, B.astype(np.uint8))
    assert np.array_equal(code & 15, direction.astype(np.uint8))
    assert np.array_equal((code >> 5) & 1, sel.astype(np.uint8))
    assert sel.sum() > 0


def _native(logits, target, zoom, crit, grad=0.7):
    from semseg_b200 import functional as SF
    lv = logits.detach().requires_grad_(True)
    loss, amax = SF.upsample_ce(lv, target, crit.ignore_index, zoom, criterion=crit)
    loss.backward(torch.tensor(grad, device="cuda"))
    return loss.detach(), lv.grad


def _oracle(logits, target, zoom, crit, k):
    """float64: (loss, dloss/dlogits NHWC) of ce_weight CE + abl_weight ABL with the selection from score map k."""
    s8 = logits.detach().double().permute(0, 3, 1, 2).cpu().requires_grad_(True)
    up = upsample(s8, zoom)
    C = up.shape[1]
    t = target.cpu()
    valid = (t != crit.ignore_index) & (t >= 0) & (t < C)
    nll = -torch.log_softmax(up, 1).gather(1, t.clamp(0, C - 1).unsqueeze(1)).squeeze(1)
    ce = (nll * valid).sum() / max(int(valid.sum()), 1)
    r = O.contract(up.detach(), t.numpy(), crit.ignore_index, crit.max_n_ratio, crit.max_clip_dist,
                   crit.label_smoothing, k=k)
    surrogate = crit.ce_weight * ce + crit.abl_weight * (up * r["grad"]).sum()
    (dl,) = torch.autograd.grad(surrogate, s8)
    return crit.ce_weight * ce.item() + crit.abl_weight * r["abl"], dl.permute(0, 2, 3, 1), r["M"]


def _check(logits, target, zoom, crit, label):
    info, maps = _forward(logits, target, zoom, crit.max_n_ratio, crit.max_clip_dist, crit.label_smoothing)
    loss, dl = _native(logits, target, zoom, crit)
    ref, rdl, M = _oracle(logits, target, zoom, crit, maps["k"].cpu().numpy())
    assert int(info[1].item()) == M
    el = abs(loss.item() - ref) / abs(ref)
    scale = (0.7 * rdl).abs().max()
    eg = float((dl.double().cpu() - 0.7 * rdl).abs().max() / scale)
    _worst["loss"], _worst["grad"] = max(_worst["loss"], el), max(_worst["grad"], eg)
    print("%s: M %d, loss rel %.2e (gate %.0e, worst %.2e), dlogits %.2e of max (gate %.0e, worst %.2e)" %
          (label, M, el, LOSS_GATE, _worst["loss"], eg, GRAD_GATE, _worst["grad"]))
    assert el <= LOSS_GATE and eg <= GRAD_GATE, (label, el, eg)
    return M


def _crit(**kw):
    from semseg_b200.losses import ActiveBoundaryLoss
    return ActiveBoundaryLoss(**kw)


_SIZES = {1: (37, 29), 2: (19, 15), 4: (10, 8), 8: (6, 5)}


@pytest.mark.parametrize("classes", [2, 19, 150, 256])
@pytest.mark.parametrize("zoom", [1, 2, 4, 8])
def test_loss_and_gradient_vs_oracle(zoom, classes):
    h, w = _SIZES[zoom]
    hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(2, h, w, classes, seed=zoom * 7 + classes, pitch=classes + (3 if classes == 19 else 0))
    t = _target(2, hg, wg, min(classes, 6), seed=zoom)
    M = _check(logits, t, zoom, _crit(max_n_ratio=0.05, abl_weight=2.0), "zoom %d, %d classes" % (zoom, classes))
    assert M > 0
    _check(logits, t, zoom, _crit(ce_weight=0.5, label_smoothing=0.0, max_clip_dist=3.0), "defaults-ish")


@pytest.mark.parametrize("zoom", [1, 8])
def test_no_selection_cases(zoom):
    h, w = _SIZES[zoom]
    hg, wg = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(2, h, w, 19, seed=5)
    t = _target(2, hg, wg, 6, seed=1)
    assert _check(logits, t, zoom, _crit(max_n_ratio=0.0), "max_n_ratio 0") == 0
    uniform = torch.full_like(t, 3)
    assert _check(logits, uniform, zoom, _crit(), "no GT boundary") == 0
    _, dl = _native(logits, uniform, zoom, _crit())
    _, dce = _native(logits, uniform, zoom, torch.nn.CrossEntropyLoss(ignore_index=255))
    assert torch.equal(dl, dce)


def test_reruns_are_bit_identical_and_capture_into_a_graph():
    from semseg_b200 import functional as SF
    logits = _logits(2, 12, 10, 21, seed=2).contiguous()
    t = _target(2, 89, 73, 6, seed=2)
    crit = _crit()
    runs = []
    for _ in range(2):
        runs.append(_native(logits, t, 8, crit))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    lv = logits.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):                       # warm up on the side stream, as torch.cuda.graphs asks
            lv.grad = None
            SF.upsample_ce(lv, t, 255, 8, criterion=crit)[0].backward()
    torch.cuda.current_stream().wait_stream(s)
    lv.grad = None
    gout = torch.tensor(0.7, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, _ = SF.upsample_ce(lv, t, 255, 8, criterion=crit)
        loss.backward(gout)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, runs[0][0]) and torch.equal(lv.grad, runs[0][1])


def _blocky_batches(zoom, seeds):
    out = []
    for s in seeds:
        x, y = _batch(zoom, seed=s)
        out.append((x, torch.from_numpy(_labels(*y.shape, classes=21, seed=s)).cuda()))
    return out


@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_graphed_steps_equal_eager_and_reruns(arch, monkeypatch):
    from semseg_b200 import graphs
    base = _build(arch, 8).cuda().train()
    base.criterion = _crit()
    batches = _blocky_batches(8, (1, 2))
    n_steps = graphs.WARMUP_CALLS + 2
    runs = []
    for graph in ("0", "1", "1"):
        monkeypatch.setenv("SEMSEG_B200_GRAPH", graph)
        m = copy.deepcopy(base)
        runs.append((m, _sgd_steps(m, batches, n_steps)))
    (eager, le), (g1, l1), (g2, l2) = runs
    assert le == l1 == l2, (le, l1, l2)
    for (k, pe), (_, p1), (_, p2) in zip(eager.named_parameters(), g1.named_parameters(), g2.named_parameters()):
        assert torch.equal(pe, p1) and torch.equal(p1, p2), k
    assert sum(1 for s in g1._sb_graph_steps.values() if s.fwd is not None) == 1


@pytest.mark.parametrize("zoom", [2, 8])
def test_abl_weight_zero_is_the_cross_entropy_step(zoom, monkeypatch):
    from semseg_b200 import graphs
    base = _build("psp", zoom).cuda().train()
    batches = _blocky_batches(zoom, (1, 2))
    ce, abl = copy.deepcopy(base), copy.deepcopy(base)
    ce.criterion = torch.nn.CrossEntropyLoss(ignore_index=255)
    abl.criterion = _crit(abl_weight=0.0)
    for graph in ("0", "1"):
        monkeypatch.setenv("SEMSEG_B200_GRAPH", graph)
        lc = _sgd_steps(ce, batches, graphs.WARMUP_CALLS + 2)
        la = _sgd_steps(abl, batches, graphs.WARMUP_CALLS + 2)
        assert lc == la
        for (k, a), (_, b) in zip(ce.named_parameters(), abl.named_parameters()):
            assert torch.equal(a, b), k


def test_module_path_matches_oracle():
    """ActiveBoundaryLoss(...)(logits, y) on the target grid, and its aux form the plain mean CE."""
    import torch.nn.functional as F
    n, c, H, W = 2, 21, 41, 57
    g = torch.Generator(device="cuda").manual_seed(9)
    logits = (torch.randn((n, c, H, W), device="cuda", generator=g) * 2).requires_grad_(True)
    y = _target(n, H, W, 6, seed=4)
    crit = _crit(max_n_ratio=0.05)
    loss = crit(logits, y)
    loss.backward()
    nhwc = logits.detach().permute(0, 2, 3, 1).contiguous()
    _, maps = _forward(nhwc, y, 1, 0.05)
    ref, rdl, _ = _oracle(nhwc, y, 1, crit, maps["k"].cpu().numpy())
    assert abs(loss.item() - ref) <= LOSS_GATE * abs(ref)
    rdl = rdl.permute(0, 3, 1, 2)
    assert float((logits.grad.double().cpu() - rdl).abs().max() / rdl.abs().max()) <= GRAD_GATE
    plain = crit.aux_loss(logits.detach(), y)
    assert abs(plain.item() - F.cross_entropy(logits.detach(), y, ignore_index=255).item()) <= 1e-5 * plain.item()
