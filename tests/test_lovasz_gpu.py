"""GPU tier: the Lovász-Softmax (+ cross-entropy) loss on the fused tail (csrc/tail.cu Lovász kernels, csrc/segsort.cu
through semseg_b200/functional.py).

  * the segmented sort against np.argsort(kind='stable'): random keys, heavy ties, all keys equal, a length off the
    tile, L = 1, skipped segments left untouched, S = 256; bit-equal, and two runs bit-equal;
  * the kernels against the float64 oracle of tests/lovasz_oracle.py at zoom 1, 2, 4, 8 with 19 / 21 / 150 / 256
    classes, odd h != w, widths off and across the 128-column CTA, a padded pitch, ignored and out-of-range targets,
    'present' / 'all', per_image on and off, ce_weight 0 / 1. The oracle takes each segment's order from the kernel's
    sorted payloads, read from the documented workspace, after checking that the payloads are a permutation of the
    segment's pixels, the keys non-decreasing, tied keys in increasing pixel order and the fg bits right. Measured
    worst errors on an H100 are printed ("lovasz-err") and gated below;
  * saturated logits (p = 1, e = 0), constant logits (every error tied), no valid pixel, a whole-call segment longer
    than 2^24 pixels;
  * lse and argmax are the plain tail's bits; two runs are bit-identical; forward and backward never synchronise;
  * PSPNet50 / PSANet50 on the native tail against Berman's statement on the ATen tail (a subclass);
  * graphed steps are bit-identical to eager ones, re-captured for a new per_image / classes, and launch no sort,
    softmax or upsample; the module path; every device."""
import copy

import numpy as np
import pytest
import torch

from tests import util
from tests.dice_oracle import upsampled
from tests.lovasz_oracle import lovasz, lovasz_torch, valid_mask
from tests.test_weighted_ce_gpu import _graphed_vs_eager, _n_graphs
from tests.test_zoom_gpu import _batch, _build, _clear_of_ties, _logits, _sgd_steps, _target

pytestmark = pytest.mark.gpu

ZOOMS = [1, 2, 4, 8]
SHAPES = [(2, 9, 13, 150, 152), (1, 17, 11, 19, 19), (1, 6, 140, 21, 24), (1, 7, 10, 256, 256)]
SHAPE_IDS = ["9x13-150-pitch152", "17x11-19", "6x140-21-pitch24", "7x10-256"]
MODES = [("present", False, 0.0), ("present", True, 1.0), ("all", False, 1.0), ("all", True, 0.0)]
MODE_IDS = ["present-ce0", "present-per-image-ce1", "all-ce1", "all-per-image-ce0"]
# Measured worst values on an H100 (80GB HBM3, 700 W) over this file's cases are printed as "lovasz-err": loss 7.3e-7
# relative; dlogits 8.5e-6 of the term scale below, on the +-1e4 saturated logits, where the plain tail's fp32
# lse * log2(e) (ulp 1e-3 at 1.4e4) moves p by up to 3e-4 from 1; 2.7e-6 on the random logits.
LOSS_TOL = 3e-6
DL_TOL = 2e-5
INVALID = 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ the sort
def _sort(keys, skip=None):
    from semseg_b200 import ops
    k = torch.from_numpy(keys.view(np.int32).copy()).cuda()
    v = torch.arange(keys.size, dtype=torch.int32, device="cuda").view(keys.shape).contiguous()
    sk = None if skip is None else torch.from_numpy(np.asarray(skip, dtype=np.int32)).cuda()
    ops.segsort_u32_pairs(k, v, sk)
    return k.cpu().numpy().view(np.uint32), v.cpu().numpy()


@pytest.mark.parametrize("kind", ["random", "ties", "equal", "top-bits"])
@pytest.mark.parametrize("sl", [(3, 5000), (2, 4096), (4, 1), (256, 300), (1, 70001)],
                         ids=["off-tile", "one-tile", "L1", "S256", "many-tiles"])
def test_segsort_vs_numpy_stable(sl, kind):
    s, l = sl
    rng = np.random.default_rng(s * 7 + l)
    keys = {"random": rng.integers(0, 2 ** 32, (s, l), dtype=np.uint64),
            "ties": rng.integers(0, 4, (s, l), dtype=np.uint64),
            "equal": np.full((s, l), 0xDEADBEEF, dtype=np.uint64),
            "top-bits": rng.integers(0, 4, (s, l), dtype=np.uint64) << 30}[kind].astype(np.uint32)
    ks, vs = _sort(keys)
    base = np.arange(s, dtype=np.int64)[:, None] * l
    for i in range(s):
        o = np.argsort(keys[i], kind="stable")
        assert np.array_equal(ks[i], keys[i][o])
        assert np.array_equal(vs[i] - base[i], o)
    ks2, vs2 = _sort(keys)
    assert np.array_equal(ks, ks2) and np.array_equal(vs, vs2)


def test_segsort_skipped_segments_untouched():
    s, l = 5, 9000
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 1000, (s, l), dtype=np.uint64).astype(np.uint32)
    skip = [0, 1, 0, 1, 1]
    ks, vs = _sort(keys, skip)
    for i in range(s):
        if skip[i]:
            assert np.array_equal(ks[i], keys[i]) and np.array_equal(vs[i], np.arange(i * l, (i + 1) * l))
        else:
            o = np.argsort(keys[i], kind="stable")
            assert np.array_equal(ks[i], keys[i][o]) and np.array_equal(vs[i] - i * l, o)


# ------------------------------------------------------------------------------------------------ kernels vs oracle
def _run(logits, target, zoom, classes, per_image, ce_weight, grad=0.7):
    from semseg_b200 import ops
    g = grad if torch.is_tensor(grad) else torch.tensor([grad], device="cuda")
    info, amax, lse, gamma, ws = ops.upsample_ce_lovasz_fwd(logits, target, 255, classes == "all", per_image,
                                                            ce_weight, zoom=zoom, return_workspace=True)
    dl = ops.upsample_ce_lovasz_bwd(logits, target, 255, lse, gamma, g, zoom=zoom)
    return info, amax, lse, gamma, dl, ws


def _kernel_orders(ws, target, c, classes, per_image):
    """The sorted segments from the workspace, checked -> {(scope, class): valid pixel indices in sorted order}."""
    n, ho, wo = target.shape
    hw = ho * wo
    s, l = (n * c, hw) if per_image else (c, n * hw)
    words = ws[:2 * s * l].cpu().numpy().view(np.uint32)
    keys, vals = words[:s * l].reshape(s, l), words[s * l:].reshape(s, l)
    tf = target.reshape(-1).cpu().numpy()
    vf = valid_mask(tf, c, 255)
    orders = {}
    for si in range(n if per_image else 1):
        scope = np.arange(si * hw, (si + 1) * hw) if per_image else np.arange(n * hw)
        if not vf[scope].any():
            continue
        for k in range(c):
            if classes == "present" and not (tf[scope][vf[scope]] == k).any():
                continue
            seg = si * c + k if per_image else k
            key, val = keys[seg], vals[seg]
            pix = (val >> 1).astype(np.int64)
            assert np.array_equal(np.sort(pix), scope), (si, k)                     # a permutation of the scope
            assert bool((np.diff(key.astype(np.int64)) >= 0).all())                 # keys non-decreasing
            tied = np.diff(key.astype(np.int64)) == 0
            assert bool((np.diff(pix)[tied] > 0).all())                              # stable: ties by pixel index
            assert np.array_equal(val & 1, (vf[pix] & (tf[pix] == k)).astype(np.uint32))
            valid = key != INVALID
            assert int(valid.sum()) == int(vf[scope].sum())
            assert bool(valid[:int(valid.sum())].all())                              # invalid pixels sort last
            orders[(si, k)] = pix[valid]
    return orders


def _check_vs_oracle(logits, target, zoom, classes, per_image, ce_weight):
    """-> (loss_info, dlogits), asserting the gates."""
    c = logits.shape[-1]
    info, amax, _, _, dl, ws = _run(logits, target, zoom, classes, per_image, ce_weight)
    orders = _kernel_orders(ws, target, c, classes, per_image)
    lr = logits.detach().clone().requires_grad_(True)
    x = upsampled(lr, zoom)
    loss_o, grad_o, meta = lovasz(x.detach().cpu().numpy(), target.cpu().numpy(), 255, classes, per_image, ce_weight,
                                  orders=orders)
    (dl_o,) = torch.autograd.grad(x, lr, torch.from_numpy(grad_o).cuda() * 0.7)
    assert int(info[1]) == meta["n_valid"]
    e_loss = abs(info[0].item() - loss_o) / max(abs(loss_o), 1e-30)
    # dL/dv = p (gamma - Gamma) + lam (p - fg) cancels where p is near 1, and the upsample adjoint sums terms of both
    # signs (constant logits): the fp32 error follows the size of the terms that cancel, so the gate is relative to the
    # adjoint of their magnitudes. Relative to max |dlogits| itself the worst case measured was 6.5e-4 (saturated
    # logits without CE, where every gradient is a cancellation); that figure is printed as dl_max.
    (dl_abs,) = torch.autograd.grad(x, lr, torch.from_numpy(meta["terms"]).cuda() * 0.7)
    err = float((dl.double() - dl_o).abs().max())
    e_dl = err / max(float(dl_abs.max()), 1e-30)
    e_dl_max = err / max(float(dl_o.abs().max()), 1e-30)
    print("lovasz-err zoom=%d C=%d %s per_image=%d ce=%g loss=%.3g dl_max=%.3g dl=%.3g" % (
        zoom, c, classes, per_image, ce_weight, e_loss, e_dl_max, e_dl))
    assert e_loss <= LOSS_TOL
    assert e_dl <= DL_TOL
    clear = _clear_of_ties(x.detach().float())
    assert torch.equal(amax[clear], x.detach().argmax(1)[clear])
    return info, dl


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_lovasz_kernel_vs_oracle(zoom, shape, mode):
    n, h, w, c, pitch = shape
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    classes, per_image, ce_weight = mode
    logits = _logits(n, h, w, c, pitch, seed=zoom + 80)
    target = _target(n, ho, wo, c, seed=zoom + 80)
    target[target == c - 1] = 255                                   # an absent class
    _check_vs_oracle(logits, target, zoom, classes, per_image, ce_weight)


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("zoom", ZOOMS)
def test_lovasz_saturated_and_constant_logits(zoom, mode):
    classes, per_image, ce_weight = mode
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    target = _target(n, ho, wo, c, seed=zoom + 90)
    # constant logits: p = 1/C everywhere, every error of a class tied
    _check_vs_oracle(torch.zeros((n, h, w, c), device="cuda"), target, zoom, classes, per_image, ce_weight)
    # saturated: one class certain at every node (p = 1 and e = 0 wherever the target agrees)
    lg = torch.full((n, h, w, c), -1e4, device="cuda")
    lg[..., 3] = 1e4
    target[:, ::2] = 3
    _check_vs_oracle(lg, target, zoom, classes, per_image, ce_weight)


@pytest.mark.parametrize("zoom", ZOOMS)
def test_lovasz_nothing_valid_gives_zero(zoom):
    n, h, w, c = 2, 9, 11, 21
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, c, seed=3)
    target = torch.full((n, ho, wo), 255, dtype=torch.int64, device="cuda")
    target[0, 0, :3] = c + 1                             # out of range: not valid either
    for classes, per_image, ce_weight in MODES:
        info, _, _, gamma, dl, _ = _run(logits, target, zoom, classes, per_image, ce_weight)
        assert info.tolist() == [0.0, 0.0] and float(dl.abs().max()) == 0.0
        assert float(gamma[:-2].abs().max()) == 0.0


def test_lovasz_segment_longer_than_2_pow_24():
    """2 classes over one image of 4097 x 4097 pixels (zoom 2): every count stays exact, the sort spans 4099 tiles."""
    n, h, w, c = 1, 2049, 2049, 2
    zoom = 2
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    assert n * ho * wo > 2 ** 24
    logits = _logits(n, h, w, c, c, seed=5)
    target = _target(n, ho, wo, c, seed=5)
    _check_vs_oracle(logits, target, zoom, "present", False, 1.0)


@pytest.mark.parametrize("zoom", [1, 8])
def test_lovasz_deterministic_pred_is_plain_and_never_syncs(zoom):
    from semseg_b200 import ops
    n, h, w, c, pitch = 2, 17, 23, 150, 152
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=zoom)
    target = _target(n, ho, wo, c, seed=zoom)
    g = torch.tensor([0.7], device="cuda")
    _run(logits, target, zoom, "present", True, 1.0, g)              # loads the library, allocates
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = _run(logits, target, zoom, "present", True, 1.0, g)
        b = _run(logits, target, zoom, "present", True, 1.0, g)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for u, v in zip(a[:5], b[:5]):       # (loss_info, argmax, lse, gamma, dlogits): not the scratch workspace
        assert torch.equal(u, v)
    info, amax, lse = ops.upsample_ce_fwd(logits, target, 255, zoom=zoom)
    assert torch.equal(a[1], amax) and torch.equal(a[2], lse)
    assert a[0][1].item() == info[1].item()


def test_lovasz_functional_dispatch():
    """SF.upsample_ce with a LovaszSoftmaxLoss criterion runs the Lovász kernels (same bits as ops)."""
    from semseg_b200 import functional as SF
    from semseg_b200.losses import LovaszSoftmaxLoss
    zoom, (n, h, w, c, pitch) = 8, SHAPES[0]
    ho, wo = zoom * (h - 1) + 1, zoom * (w - 1) + 1
    logits = _logits(n, h, w, c, pitch, seed=70)
    target = _target(n, ho, wo, c, seed=70)
    crit = LovaszSoftmaxLoss(classes="all", per_image=True, ce_weight=0.3)
    info, amax, _, _, dl, _ = _run(logits, target, zoom, "all", True, 0.3)
    lg = logits.detach().clone().requires_grad_(True)
    loss, pred = SF.upsample_ce(lg, target, 255, zoom=zoom, criterion=crit)
    (dl_s,) = torch.autograd.grad(loss * 0.7, lg)
    assert torch.equal(loss, info[0]) and torch.equal(pred, amax) and torch.equal(dl_s, dl)


# ------------------------------------------------------------------------------------------------ every device
def test_lovasz_kernels_on_every_device():
    """Shapes whose Lovász kernels need more than 48 KB of dynamic shared memory (the key pass at zoom 1 and 2 with 150
    classes, the rows kernel at zoom 8 with Wo = 793); from one thread per device, every device computes the bits of
    device 0."""
    import threading
    from semseg_b200 import ops
    cases = [(1, (2, 9, 140, 150, 152)), (2, (2, 9, 70, 150, 150)), (8, (1, 5, 100, 21, 24))]
    inputs = [(zoom, _logits(n, h, w, c, pitch, seed=zoom).cpu(),
               _target(n, zoom * (h - 1) + 1, zoom * (w - 1) + 1, c, seed=zoom).cpu())
              for zoom, (n, h, w, c, pitch) in cases]
    results, errors = {}, []

    def run(dev):
        try:
            with torch.cuda.device(dev):
                out = []
                for zoom, logits, target in inputs:
                    lg, t = logits.to(dev), target.to(dev)
                    info, amax, lse, gamma = ops.upsample_ce_lovasz_fwd(lg, t, 255, False, True, 1.0, zoom=zoom)
                    dl = ops.upsample_ce_lovasz_bwd(lg, t, 255, lse, gamma, torch.tensor([1.0], device=dev),
                                                    zoom=zoom)
                    out.append(tuple(v.cpu() for v in (info, amax, lse, gamma, dl)))
                results[dev] = out
        except Exception as e:      # noqa: BLE001 - reported below
            errors.append((dev, e))

    threads = [threading.Thread(target=run, args=(d,)) for d in range(torch.cuda.device_count())]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert sorted(results) == list(range(torch.cuda.device_count()))
    for dev, out in results.items():
        for (zoom, _, _), got, ref in zip(inputs, out, results[0]):
            assert all(torch.equal(a, b) for a, b in zip(got, ref)), (dev, zoom)


# ------------------------------------------------------------------------------------------------ networks
def _torch_lovasz_class():
    from semseg_b200.losses import LovaszSoftmaxLoss

    class _TorchLovasz(LovaszSoftmaxLoss):
        """Berman's Lovász-Softmax in PyTorch under another type: the network keeps the ATen tail."""

        def forward(self, logits, target):
            return lovasz_torch(logits, target, self.ignore_index, self.classes, self.per_image,
                                self.ce_weight).float()

    return _TorchLovasz


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("zoom", [2, 8])
@pytest.mark.parametrize("arch", ["psp", "psa"])
def test_network_native_lovasz_tail_matches_aten_tail(arch, zoom, mode, monkeypatch):
    from semseg_b200 import functional as SF
    from semseg_b200 import precision
    from semseg_b200.losses import LovaszSoftmaxLoss
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    native = _build(arch, zoom).cuda().train()
    native.criterion = LovaszSoftmaxLoss(ignore_index=255, ce_weight=1.0)
    aten = copy.deepcopy(native)
    aten.criterion = _torch_lovasz_class()(ignore_index=255, ce_weight=1.0)
    x, y = _batch(zoom)
    assert SF.fused_tail_supported(native.criterion, None, y, zoom, x.size())
    assert not SF.fused_tail_supported(aten.criterion, None, y, zoom, x.size())
    with precision.mode(mode):
        pred, main, aux = native(x, y)
        (main + 0.4 * aux).backward()
        pred_r, main_r, aux_r = aten(x, y)
        (main_r + 0.4 * aux_r).backward()
    assert pred.shape == pred_r.shape == y.shape
    assert abs(main.item() - main_r.item()) <= 1e-5 * abs(main_r.item())
    assert abs(aux.item() - aux_r.item()) <= 1e-5 * abs(aux_r.item())
    assert (pred != pred_r).float().mean().item() < 0.01
    if mode != "bf16x3":
        return      # as tests/test_zoom_gpu.py: in bf16 the tails' ~1e-6 dlogits differences flip bf16 roundings
    # errors that fp32 and fp64 order differently swap neighbouring g_k: a few pixels' gradients move (measured worst
    # rel-L2 1.0e-4 against the Dice tail's 1e-4 gate), hence 3e-4
    worst, bad = 0.0, []
    for (k, pn), (_, pa) in zip(native.named_parameters(), aten.named_parameters()):
        assert (pn.grad is None) == (pa.grad is None), k
        if pn.grad is not None:
            err = util.rel_l2(pn.grad, pa.grad)
            worst = max(worst, err)
            if err > 3e-4:
                bad.append((k, err))
    print("lovasz-net-err %s zoom=%d worst param-grad rel_l2=%.3g" % (arch, zoom, worst))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ graphs
def test_graphed_lovasz_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    from semseg_b200.losses import LovaszSoftmaxLoss
    base = _build("psp", 8).cuda().train()
    base.criterion = LovaszSoftmaxLoss(ignore_index=255, ce_weight=1.0)
    batches = [_batch(8, seed=s) for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4
    eager, graphed = _graphed_vs_eager(base, batches, n_steps, monkeypatch)
    assert _n_graphs(graphed) == 1
    # per_image and classes change the launches: each captures anew, never replays the old graph
    for k, (attr, value) in enumerate((("per_image", True), ("classes", "all"))):
        for m in (eager, graphed):
            setattr(m.criterion, attr, value)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
        le = _sgd_steps(eager, batches, n_steps)
        monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
        lg = _sgd_steps(graphed, batches, n_steps)
        assert le == lg, (attr, le, lg)
        assert _n_graphs(graphed) == 2 + k


def test_graphed_lovasz_step_launches_no_aten_tail():
    from torch.profiler import ProfilerActivity, profile
    from semseg_b200 import graphs
    from semseg_b200.losses import LovaszSoftmaxLoss
    model = _build("psp", 8).cuda().train()
    model.criterion = LovaszSoftmaxLoss(ignore_index=255, per_image=True, ce_weight=1.0)
    x, y = _batch(8)
    for _ in range(graphs.WARMUP_CALLS + 2):
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
    torch.cuda.synchronize()
    assert graphs.launches_per_step(model) > 100
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    bad = [n for n in names if any(k in n for k in ("aten::sort", "upsample_bilinear2d", "_softmax", "softmax",
                                                    "SoftMax", "cumsum", "nll_loss"))]
    assert not bad, sorted(set(bad))


# ------------------------------------------------------------------------------------------------ module path
def test_lovasz_module_path():
    """LovaszSoftmaxLoss()(eval_logits, y) as validate() calls it: the zoom-1 kernels on an NHWC copy (the same bits as
    the ops call), checked against the oracle with the kernel's order."""
    from semseg_b200 import ops
    from semseg_b200.losses import LovaszSoftmaxLoss
    model = _build("psp", 8).cuda().eval()
    x, y = _batch(8)
    with torch.no_grad():
        out = model(x)
    nhwc = out.permute(0, 2, 3, 1).contiguous()
    for crit in (LovaszSoftmaxLoss(), LovaszSoftmaxLoss(classes="all", per_image=True, ce_weight=1.0)):
        loss = crit(out, y)
        info, _, lse, gamma = ops.upsample_ce_lovasz_fwd(nhwc, y, 255, crit.classes == "all", crit.per_image,
                                                         crit.ce_weight, zoom=1)
        dl = ops.upsample_ce_lovasz_bwd(nhwc, y, 255, lse, gamma, torch.ones(1, device="cuda"), zoom=1)
        assert torch.equal(loss, info[0])
        lg = out.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(crit(lg, y), lg)
        assert torch.equal(g, dl.permute(0, 3, 1, 2))
        _check_vs_oracle(nhwc, y, 1, crit.classes, crit.per_image, crit.ce_weight)
