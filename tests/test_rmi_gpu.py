"""GPU tier: the RMI (+ BCE + cross-entropy) loss on the fused tail (csrc/tail.cu RMI kernels through
semseg_b200/functional.py).

  * kernel vs the float64 contract of tests/rmi_oracle.py at zoom 1, 2, 4, 8, with odd h != w, widths off and across
    the CTA columns, 19 / 21 / 150 / 256 classes, a padded pitch, ignored and out-of-range targets, an absent class,
    bce_weight 0 / 0.5 / 1 and ce_weight 0 / 1: the pooled Y (exact) and Q maps against float64; the raw moment sums,
    r and the gradient table against the oracle's algebra fed the kernel's own pooled maps (so the conditioning of P
    does not hide kernel error); dlogits against the oracle's gradient from those maps; and end to end, the loss and
    dlogits against the oracle from the logits;
  * no valid pixel gives r = 9/2 log alpha and a zero gradient; two runs are bit-identical; lse and pred are the plain
    tail's bits; neither pass synchronises;
  * PSPNet50 / PSANet50 on the native RMI tail against the paper's statement in PyTorch on the ATen tail;
  * graphed RMI steps are bit-identical to eager ones, and a new bce_weight or pos_alpha captures anew;
  * the module path RMILoss()(eval_logits, y) against the oracle.

Gates: the worst errors measured on an H100 over these cases, printed by every case ("rmi-err"), are recorded next to
each gate below."""
import copy

import pytest
import torch

from tests import util
from tests.dice_oracle import upsampled
from tests.rmi_oracle import rmi_algebra, rmi_contract, rmi_grad, rmi_grad_logits, rmi_literal
from tests.test_weighted_ce_gpu import _graphed_vs_eager, _n_graphs
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
SHAPES = [(2, 13, 17, 150, 152), (1, 17, 13, 19, 19), (1, 14, 140, 21, 24), (1, 13, 16, 256, 256)]
SHAPE_IDS = ["13x17-150-pitch152", "17x13-19", "14x140-21-pitch24", "13x16-256"]
OPTIONS = [(0.0, 0.0), (0.5, 0.0), (1.0, 0.0), (0.0, 1.0), (0.5, 1.0), (1.0, 1.0)]
OPTION_IDS = ["bce0-ce0", "bce.5-ce0", "bce1-ce0", "bce0-ce1", "bce.5-ce1", "bce1-ce1"]
ALPHA = 5e-4
A32 = float(torch.tensor(ALPHA, dtype=torch.float32))     # pos_alpha crosses the C-ABI as fp32: the kernels' alpha

# gates, with the worst error measured on an H100 80GB HBM3 over the cases of this file
G_Q = 5e-7          # pooled Q map and the table's means, absolute                    (measured 1.2e-7)
G_MOM = 1e-13       # raw fp64 moment sums, relative to the largest of their group     (3.9e-15)
G_R = 1e-9          # fp64 r from the kernel's pooled maps, absolute                  (1.4e-12)
G_R32 = 2e-7        # the table's fp32 r, relative                                     (6.3e-8)
G_T = 5e-7          # gradient table from the kernel's pooled maps, relative to max |T| (7.0e-8)
G_DL_OWN = 5e-5     # dlogits against the oracle fed the kernel's pooled maps, / max |dl| (2.2e-5)
G_BCE = 5e-7        # BCE and CE, relative                                             (8.8e-8)
G_LOSS = 1e-6       # loss end to end, relative                                        (2.6e-7)
G_DL = 5e-5         # dlogits end to end, relative to max |dl|                         (2.2e-5)


def _run(logits, target, zoom, bw, cw, alpha=ALPHA, grad=0.7):
    from semseg_b200 import _lib, ops
    n, h, w, c = logits.shape
    _, ho, wo = target.shape
    nws = int(_lib.load().semseg_upsample_ce_rmi_workspace_floats(n, ho, wo, c, zoom))
    ws = torch.empty((nws,), dtype=torch.float32, device="cuda")
    info, amax, lse, pooled, table = ops.upsample_ce_rmi_fwd(logits, target, 255, bw, alpha, cw, zoom=zoom,
                                                             workspace=ws)
    dl = ops.upsample_ce_rmi_bwd(logits, target, 255, lse, pooled, table, torch.tensor([grad], device="cuda"),
                                 zoom=zoom)
    return info, amax, lse, pooled, table, dl, ws


def _absent(target, c):
    t = target.clone()
    t[t == c - 1] = 255
    return t


def _blocky_target(n, ho, wo, c, seed, block=5):
    """Piecewise-constant labels (so the pooled one-hot maps vary between cells), a few ignored and out-of-range."""
    g = torch.Generator(device="cuda").manual_seed(seed + 7)
    t = torch.randint(0, c, (n, (ho + block - 1) // block, (wo + block - 1) // block), device="cuda", generator=g)
    t = t.repeat_interleave(block, 1).repeat_interleave(block, 2)[:, :ho, :wo].contiguous()
    t[torch.rand((n, ho, wo), device="cuda", generator=g) < 0.05] = 255
    t[torch.rand((n, ho, wo), device="cuda", generator=g) < 0.003] = c + 3
    return t


def _table(table, n, c):
    rec = table[:n * c * 184].view(n, c, 184).double()
    return rec[..., :162].reshape(n, c, 9, 18), rec[..., 162:171], rec[..., 171:180], rec[..., 180]


def _check(logits, target, zoom, bw, cw):
    n, h, w, c = logits.shape
    info, amax, lse, pooled, table, dl, ws = _run(logits, target, zoom, bw, cw)
    x = upsampled(logits, zoom)
    res = rmi_contract(x, target, 255, bw, ALPHA, cw)
    Yk, Qk = pooled[0].double(), pooled[1].double()
    # pooled maps against float64
    assert torch.equal(Yk, res["Y"])
    e_q = float((Qk - res["Q"]).abs().max())
    # the algebra fed the kernel's own pooled maps
    own = rmi_algebra(Yk, Qk, A32)
    mom = ws[:2 * n * c * 189].view(torch.float64).view(n, c, 189)
    e_mom = 0.0
    for lo, hi in ((0, 18), (18, 63), (63, 108), (108, 189)):
        ref = own["mom"][..., lo:hi]
        e_mom = max(e_mom, float((mom[..., lo:hi] - ref).abs().max()) / max(float(ref.abs().max()), 1e-300))
    T, ma, mb, r = _table(table, n, c)
    r64 = ws[2 * n * c * 189:2 * n * c * 190].view(torch.float64).view(n, c)
    e_r = float((r64 - own["r"]).abs().max())
    e_r32 = float(((r - own["r"]).abs() / own["r"].abs()).max())
    e_t = float((T - own["T"]).abs().max()) / max(float(own["T"].abs().max()), 1e-30)
    e_m = max(float((ma - own["ma"]).abs().max()), float((mb - own["mb"]).abs().max()))
    # dlogits: the oracle's gradient from the kernel's pooled maps, and end to end
    own_res = dict(nv=res["nv"], dQ=own["dQ"])
    dl_own = rmi_grad_logits(logits, zoom, 0.7 * rmi_grad(x, target, 255, bw, ALPHA, cw, res=own_res))
    dl_ref = rmi_grad_logits(logits, zoom, 0.7 * rmi_grad(x, target, 255, bw, ALPHA, cw, res=res))
    scale = max(float(dl_ref.abs().max()), 1e-30)
    e_dl_own = float((dl.double() - dl_own).abs().max()) / scale
    e_dl = float((dl.double() - dl_ref).abs().max()) / scale
    e_bce = abs(info[2].item() - res["bce"].item()) / max(abs(res["bce"].item()), 1e-30)
    e_ce = abs(info[4].item() - res["ce"].item()) / max(abs(res["ce"].item()), 1e-30)
    e_loss = abs(info[0].item() - res["loss"].item()) / max(abs(res["loss"].item()), 1e-30)
    print("rmi-err zoom=%d C=%d bw=%g cw=%g Q=%.3g mom=%.3g r=%.3g r32=%.3g T=%.3g mean=%.3g dl_own=%.3g bce=%.3g "
          "ce=%.3g loss=%.3g dl=%.3g" % (zoom, c, bw, cw, e_q, e_mom, e_r, e_r32, e_t, e_m, e_dl_own, e_bce, e_ce,
                                        e_loss, e_dl))
    assert int(info[1]) == res["nv"]
    assert e_q <= G_Q and e_m <= G_Q
    assert e_mom <= G_MOM
    assert e_r <= G_R and e_r32 <= G_R32 and e_t <= G_T
    assert e_dl_own <= G_DL_OWN
    assert e_bce <= G_BCE and (cw == 0.0 or e_ce <= G_BCE)
    assert e_loss <= G_LOSS and e_dl <= G_DL
    clear = _clear_of_ties(x.float())
    assert torch.equal(amax[clear], x.argmax(1)[clear])
    return info, table, T, r


@pytest.mark.parametrize("opts", OPTIONS, ids=OPTION_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_rmi_kernel_vs_oracle(zoom, shape, opts):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom + 80)
    target = _absent(_blocky_target(n, ho, wo, c, seed=zoom + 80), c)
    _, _, T, r = _check(logits, target, zoom, *opts)
    # the absent class: S_ab = 0, so no gradient coefficient
    assert float(T[:, c - 1].abs().max()) == 0.0


@pytest.mark.parametrize("zoom", ZOOMS)
def test_rmi_nothing_valid(zoom):
    import math
    n, h, w, c = 2, 13, 15, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    target[0, 0, :3] = c + 1
    for bw, cw in OPTIONS:
        info, _, _, _, table, dl, ws = _run(logits, target, zoom, bw, cw)
        T, _, _, _ = _table(table, n, c)
        r64 = ws[2 * n * c * 189:2 * n * c * 190].view(torch.float64)
        assert info[1].item() == 0.0 and info[2].item() == 0.0 and info[4].item() == 0.0
        assert float((r64 - 4.5 * math.log(A32)).abs().max()) <= 1e-12
        assert float(T.abs().max()) == 0.0 and float(dl.abs().max()) == 0.0


@pytest.mark.parametrize("zoom", [1, 8])
def test_rmi_deterministic_and_pred_is_plain(zoom):
    from semseg_b200 import ops
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _blocky_target(n, ho, wo, c, seed=zoom)
    a = _run(logits, target, zoom, 0.5, 1.0)
    b = _run(logits, target, zoom, 0.5, 1.0)
    for u, v in zip(a[:6], b[:6]):
        assert torch.equal(u, v)
    nc = n * c
    assert torch.equal(a[6][:2 * nc * 190].view(torch.int32), b[6][:2 * nc * 190].view(torch.int32))  # fp64 moments, r
    info, amax, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    assert torch.equal(a[1], amax) and torch.equal(a[2], lse)
    assert a[0][1].item() == info[1].item()
    assert abs(a[0][4].item() - info[0].item()) <= 1e-6 * abs(info[0].item())


def test_rmi_passes_do_not_synchronise():
    """Forward and backward capture into a CUDA graph (a host read or synchronisation would fail the capture) and the
    replay gives the eager bits."""
    from semseg_b200 import ops
    n, h, w, c, pitch, zoom = 2, 13, 17, 21, 24, 8
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=5)
    target = _blocky_target(n, ho, wo, c, seed=5)
    eager = _run(logits, target, zoom, 0.5, 1.0)
    g_out = torch.tensor([0.7], device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                       # warm-up: module load and the shared-memory opt-in
        out = ops.upsample_ce_rmi_fwd(logits, target, 255, 0.5, ALPHA, 1.0, zoom=zoom)
        ops.upsample_ce_rmi_bwd(logits, target, 255, out[2], out[3], out[4], g_out, zoom=zoom)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        info, amax, lse, pooled, table = ops.upsample_ce_rmi_fwd(logits, target, 255, 0.5, ALPHA, 1.0, zoom=zoom)
        dl = ops.upsample_ce_rmi_bwd(logits, target, 255, lse, pooled, table, g_out, zoom=zoom)
    graph.replay()
    torch.cuda.synchronize()
    for u, v in zip((info, amax, lse, pooled, table, dl), eager[:6]):
        assert torch.equal(u, v)


def test_rmi_functional_and_module_dispatch():
    from semseg_b200 import functional as SF
    from semseg_b200.losses import RMILoss
    zoom, (n, h, w, c, pitch) = 8, SHAPES[0]
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=70)
    target = _blocky_target(n, ho, wo, c, seed=70)
    crit = RMILoss(ignore_index=255, bce_weight=0.3, pos_alpha=1e-3, ce_weight=0.2)
    info, amax, _, _, _, dl, _ = _run(logits, target, zoom, 0.3, 0.2, alpha=1e-3)
    lg = logits.detach().clone().requires_grad_(True)
    loss, pred = SF.upsample_ce(lg, target, 255, zoom=zoom, criterion=crit)
    (dl_s,) = torch.autograd.grad(loss * 0.7, lg)
    assert torch.equal(loss, info[0]) and torch.equal(pred, amax) and torch.equal(dl_s, dl)


# ------------------------------------------------------------------------------------------------ networks
def _torch_rmi_class():
    from semseg_b200.losses import RMILoss

    class _TorchRMI(RMILoss):
        """RMILoss as the paper's code writes it in PyTorch, under another type: the network keeps the ATen tail."""

        def forward(self, logits, target):
            return rmi_literal(logits, target, self.ignore_index, self.bce_weight, self.pos_alpha,
                               self.ce_weight).to(logits.dtype)

    return _TorchRMI


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_rmi_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import RMILoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    native.criterion = RMILoss(ignore_index=255, ce_weight=1.0)
    aten = copy.deepcopy(native)
    aten.criterion = _torch_rmi_class()(ignore_index=255, ce_weight=1.0)
    x, y = _batch(zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    with precision.mode(mode):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    print("rmi-net %s zoom=%d %s main=%.3g aux=%.3g" % (arch, zoom, mode, abs(main.item() - main_r.item()) /
                                                        abs(main_r.item()), abs(aux.item() - aux_r.item()) /
                                                        abs(aux_r.item())))          # measured <= 7.3e-8
    assert pred.shape == pred_r.shape == y.shape
    assert abs(main.item() - main_r.item()) <= G_LOSS * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= G_LOSS * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01
    if mode != "bf16x3":
        return
    bad, worst = [], 0.0
    for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
        assert (pn.grad is None) == (pa.grad is None), k
        if pn.grad is not None:
            err = util.rel_l2(pn.grad, pa.grad)
            worst = max(worst, err)
            if err > 1e-3:                                        # measured <= 1.1e-4
                bad.append((k, err))
    print("rmi-net %s zoom=%d worst parameter-gradient rel. L2 %.3g" % (arch, zoom, worst))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ graphs
def test_graphed_rmi_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import RMILoss
    base = _build("psp", 8).cuda().train()
    base.criterion = RMILoss(ignore_index=255, ce_weight=1.0)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = _graphed_vs_eager(base, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 1
    # a new bce_weight or pos_alpha is a new launch argument: each captures anew, never replays the old graph
    for k, (attr, val) in enumerate((("bce_weight", 0.25), ("pos_alpha", 1e-3))):
        for m in (eager, graphed):
            setattr(m.criterion, attr, val)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
        le = _sgd_steps(eager, batches, n_steps)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
        lg = _sgd_steps(graphed, batches, n_steps)
        assert le == lg, (attr, le, lg)
        assert _n_graphs(graphed) == 2 + k


# ------------------------------------------------------------------------------------------------ module path
def test_rmi_module_path_matches_oracle():
    """RMILoss()(eval_logits, y) as validate() calls it, and its gradient."""
    from semseg_b200.losses import RMILoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    for crit in (RMILoss(), RMILoss(bce_weight=0.0, ce_weight=1.0)):
        loss = crit(out, y)
        res = rmi_contract(out, y, 255, crit.bce_weight, crit.pos_alpha, crit.ce_weight)
        print("rmi-module bw=%g loss=%.3g" % (crit.bce_weight, abs(loss.item() - res["loss"].item()) /
                                             abs(res["loss"].item())))
        assert abs(loss.item() - res["loss"].item()) <= G_LOSS * abs(res["loss"].item())     # measured 3.9e-8
        lg = out.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(crit(lg, y), lg)
        g_ref = rmi_grad(out, y, 255, crit.bce_weight, crit.pos_alpha, crit.ce_weight, res=res)
        assert float((g.double() - g_ref).abs().max()) <= G_DL * float(g_ref.abs().max())
