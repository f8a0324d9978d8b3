"""GPU tier of PSANet's compact (dense mask) and softmax-free attention on the fused kernels (csrc/psa_fused.cu):
  * the kernels in every form (window / dense x softmax on / off x collect / distribute x bf16 / bf16x3) against the fp32
    torch composition of model/psanet.py:63-70 on the same rounded operands;
  * the default form (window + softmax) reproduces, bit for bit, the digests the kernels of the parent commit wrote
    (tests/golden/psa_attend_default.json), through the original entry points and the `_ex` ones;
  * PSANet50 in all 12 (psa_type, compact, psa_softmax) combinations against the fp32 oracle, a compact PSANet50 at the
    config-3 shape against the north_star gate, and the fused path against the ATen composition (SEMSEG_B200_PSA_FUSED=0);
  * an eager step runs no ATen attention kernel, graphed steps are bit-identical to eager ones, and sliding-window
    evaluation of a compact PSANet takes the native finish."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle.torch_oracle import psa_mask_torch
from tests import psa_attend_cases as pc
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _strict_fp32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _composition(attn, feat32, psa_type, mh, mw, scale, compact, softmax):
    """model/psanet.py:63-70 in fp32 on NHWC operands: attn [n,h,w,>=mh*mw], feat32 [n,h,w,c] -> [n,h,w,c]."""
    n, h, w, c = feat32.shape
    q = h * w
    y = attn[..., :mh * mw].permute(0, 3, 1, 2).contiguous()          # NCHW, the layout the reference works on
    if compact:
        if psa_type == 1:
            y = y.view(n, q, q).transpose(1, 2).reshape(n, q, h, w)
    else:
        y = psa_mask_torch(y, psa_type, mh, mw)
    if softmax:
        y = torch.softmax(y, dim=1)
    out = torch.bmm(feat32.reshape(n, q, c).transpose(1, 2), y.reshape(n, q, q)) * scale      # [n, c, q]
    return out.transpose(1, 2).reshape(n, h, w, c)


# (n, h, w, mask_h, mask_w, extra logit columns). Dense: the 65^2 compact map, a non-square map, partial last tiles, the
# 465^2 / 473^2 compact map (Q = 900), and a logit pitch wider than h*w. Window: a full and two smaller masks.
DENSE_GEOMS = [(2, 5, 5, 5, 5, 0), (1, 7, 11, 7, 11, 0), (2, 13, 9, 13, 9, 0), (1, 30, 30, 30, 30, 0),
               (2, 6, 7, 6, 7, 6)]
WINDOW_GEOMS = [(2, 13, 13, 25, 25, 0), (1, 9, 12, 9, 7, 0), (1, 5, 40, 9, 79, 0)]


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("psa_type", [0, 1])
@pytest.mark.parametrize("softmax", [True, False], ids=["softmax", "nosoftmax"])
@pytest.mark.parametrize("form", ["dense", "window"])
def test_psa_attend_forms_vs_torch_composition(form, softmax, psa_type, mode):
    from semseg_b200 import functional as SF, ops
    compact, split = form == "dense", mode == "bf16x3"
    c, scale = 512, 1.0 / 3.0
    for n, h, w, mh, mw, pad in (DENSE_GEOMS if compact else WINDOW_GEOMS):
        g = torch.Generator(device="cuda").manual_seed(h * 100 + w + psa_type)
        attn = (torch.randn((n, h, w, mh * mw + pad), device="cuda", generator=g) * 2).requires_grad_(True)
        f32 = torch.relu(torch.randn((n, h, w, c), device="cuda", generator=g))
        feat = (ops.f32_to_act(f32, True) if split else f32.to(torch.bfloat16)).requires_grad_(True)
        go32 = torch.randn((n, h, w, c), device="cuda", generator=g)
        go = ops.f32_to_act(go32, True) if split else go32.to(torch.bfloat16)
        assert SF.psa_attend_supported(feat, mh, mw, compact)
        out = SF.psa_attend(attn, feat, psa_type, mh, mw, scale, compact, softmax)
        out.backward(go)
        ar = attn.detach().clone().requires_grad_(True)
        fr = ops.act_to_f32(feat.detach()).requires_grad_(True)
        ref = _composition(ar, fr, psa_type, mh, mw, scale, compact, softmax)
        ref.backward(ops.act_to_f32(go))
        tol_f, tol_g = (3e-5, 1e-4) if split else (4e-3, 1e-2)
        geom = (n, h, w, mh, mw, pad)
        assert util.rel_l2(ops.act_to_f32(out), ref) < tol_f, geom
        assert util.rel_l2(ops.act_to_f32(feat.grad), fr.grad) < tol_g, geom
        assert util.rel_l2(attn.grad, ar.grad) < tol_g, geom
        # logit entries that no (target, source) pair reads (outside every window, the padding columns) are exactly zero
        unread = ar.grad == 0
        assert bool((attn.grad[unread] == 0).all()), geom
        if pad:
            assert bool((attn.grad[..., mh * mw:] == 0).all()) and bool(unread[..., mh * mw:].all())


def test_psa_attend_without_softmax_keeps_no_statistics():
    from semseg_b200 import ops
    attn = torch.randn((1, 5, 5, 25), device="cuda")
    feat = torch.relu(torch.randn((1, 5, 5, 512), device="cuda")).to(torch.bfloat16)
    for compact in (False, True):
        out, stats = ops.psa_attend(attn, feat, 0, 5, 5, 1.0, compact=compact, softmax=False)
        assert stats is None
        dattn = ops.psa_attend_bwd_attn(attn, None, feat, None, feat, 1, 5, 5, 1.0, compact=compact, softmax=False)
        assert bool(torch.isfinite(dattn).all())


# ------------------------------------------------------------------------------------------------ default form, bit for bit
def test_default_form_matches_the_parent_kernels_bit_for_bit(golden_dir):
    """Window + softmax through semseg_psa_attend / semseg_psa_attend_bwd_attn (ctypes, the original argument lists) and
    through ops (the `_ex` entry points with form 0) write the bits the kernels of the parent commit wrote: forward, stats,
    feature gradient and logit gradient, bf16 and bf16x3, collect and distribute, 8- to 128-row tiles, partial last tiles
    and masks smaller than 2H-1 x 2W-1."""
    from semseg_b200 import _lib, ops
    lib = _lib.load()
    ref = json.load(open(os.path.join(golden_dir, "psa_attend_default.json")))["digests"]
    p = lambda t: ctypes.c_void_p(t.data_ptr())      # noqa: E731
    c, scale = pc.C, pc.SCALE
    checked = 0
    for k, (key, geom) in enumerate(pc.CASES.items()):
        n, h, w, mh, mw = geom
        for split_form in (False, True):
            attn, feat, dout = (t.cuda() for t in pc.operands(geom, 100 + k, split_form))
            for psa_type in (0, 1):
                want = ref["%s/t%d/%s" % (key, psa_type, "bf16x3" if split_form else "bf16")]
                # the original entry points
                stats = torch.empty((n, h * w, 2), device="cuda")
                y, dfeat, dattn = torch.empty_like(feat), torch.empty_like(feat), torch.empty_like(attn)
                _lib.check(lib.semseg_psa_attend(0, psa_type, p(attn), mh * mw, p(feat), ops._lo(feat), c, p(stats), p(y),
                                                 ops._lo(y), c, n, h, w, mh, mw, c, scale, None), "psa_attend")
                _lib.check(lib.semseg_psa_attend(1, psa_type, p(attn), mh * mw, p(dout), ops._lo(dout), c, p(stats),
                                                 p(dfeat), ops._lo(dfeat), c, n, h, w, mh, mw, c, scale, None), "psa_attend")
                _lib.check(lib.semseg_psa_attend_bwd_attn(psa_type, p(attn), mh * mw, p(stats), p(feat), ops._lo(feat), c,
                                                          p(y), ops._lo(y), c, p(dout), ops._lo(dout), c, p(dattn), n, h,
                                                          w, mh, mw, c, scale, None), "psa_attend_bwd_attn")
                torch.cuda.synchronize()
                got = {"out": pc.digest(y), "stats": pc.digest(stats), "dfeat": pc.digest(dfeat),
                       "dattn": pc.digest(dattn)}
                assert got == want, (key, psa_type, split_form)
                # the _ex entry points through ops, on torch's current stream
                y2, stats2 = ops.psa_attend(attn, feat, psa_type, mh, mw, scale)
                dfeat2, _ = ops.psa_attend(attn, dout, psa_type, mh, mw, scale, stats=stats2, mode=1)
                dattn2 = ops.psa_attend_bwd_attn(attn, stats2, feat, y2, dout, psa_type, mh, mw, scale)
                got2 = {"out": pc.digest(y2), "stats": pc.digest(stats2), "dfeat": pc.digest(dfeat2),
                        "dattn": pc.digest(dattn2)}
                assert got2 == want, (key, psa_type, split_form)
                checked += 1
    assert checked == 16


# ------------------------------------------------------------------------------------------------ networks
def _build(psa_type, compact, softmax, size=65, classes=150, seed=0, zoom=8):
    """PSANet50 with the mask sized as tool/train.py:63-70 sizes it for a square crop of `size`."""
    from semseg_b200.psanet import PSANet
    h = (size - 1) // 16 + 1
    mask = h if compact else 2 * h - 1
    torch.manual_seed(seed)
    return PSANet(layers=50, classes=classes, zoom_factor=zoom, dropout=0.0, psa_type=psa_type, compact=compact,
                  shrink_factor=2, mask_h=mask, mask_w=mask, psa_softmax=softmax, pretrained=False), mask


COMBOS = [(t, c, s) for t in (0, 1, 2) for c in (False, True) for s in (True, False)]


def _combo_id(v):
    t, c, s = v
    return "t%d-%s-%s" % (t, "compact" if c else "window", "softmax" if s else "nosoftmax")


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("combo", COMBOS, ids=[_combo_id(v) for v in COMBOS])
def test_psanet50_variant_vs_oracle(combo, mode, monkeypatch):
    from semseg_b200 import functional as SF, precision
    psa_type, compact, softmax = combo
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model, mask = _build(psa_type, compact, softmax)
    model = model.cuda()
    calls = []
    real = SF.psa_attend
    monkeypatch.setattr(SF, "psa_attend", lambda *a: calls.append(a[6:]) or real(*a))
    orc, sd = util.oracle_from(model, "psa", layers=50, classes=150, psa_type=psa_type, compact=compact, mask_h=mask,
                               mask_w=mask, psa_softmax=softmax)
    x, y = util.synth(2, 65, 65, 150, seed=321, device="cuda")
    model.eval()
    orc.eval()
    with torch.no_grad(), precision.mode(mode):
        lm = model(x)
    with torch.no_grad():
        lo = orc.forward(x)
    assert calls and all(cl == (compact, softmax) for cl in calls), calls      # the fused kernels ran, in this form
    model.train()
    orc.train()
    with precision.mode(mode):
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
    _, mlo, alo = orc.forward(x, y)
    (mlo + 0.4 * alo).backward()
    e = util.rel_l2(lm, lo)
    if mode == "bf16":                                 # test_psanet50_small_vs_oracle's bounds
        assert e < 2e-2, e
        loss_tol = 2e-3
    else:
        assert e < 1e-3, e
        loss_tol = 1e-4
    assert abs(ml.item() - mlo.item()) < loss_tol * abs(mlo.item()), (ml.item(), mlo.item())
    assert abs(al.item() - alo.item()) < loss_tol * abs(alo.item()), (al.item(), alo.item())
    for k, prm in model.named_parameters():             # test_parity_gpu._grad_sanity
        assert prm.grad is not None and bool(torch.isfinite(prm.grad).all()), k
        a, b = float(prm.grad.double().norm()), float(sd[k].grad.double().norm())
        if b > 1e-6:
            assert 0.2 < a / b < 5.0, (k, a, b)


def test_compact_psanet50_465_north_star_gate():
    """DESIGN §4's network gate at the config-3 shape for the compact model: PSANet50 @ 465x465 (59x59 maps, 30x30
    attention over a dense 30x30 mask, Q = 900), 150 classes, fresh model, eval, bf16x3."""
    from semseg_b200 import precision
    model, mask = _build(2, True, True, size=465)
    model = model.cuda().eval()
    orc, _ = util.oracle_from(model, "psa", layers=50, classes=150, psa_type=2, compact=True, mask_h=mask, mask_w=mask)
    orc.eval()
    x, _ = util.synth(2, 465, 465, 150, device="cuda")
    with torch.no_grad():
        lo = orc.forward(x)
        with precision.mode("bf16x3"):
            lm = model(x)
    e = util.rel_l2(lm, lo)
    am, ao = lm.argmax(1), lo.argmax(1)
    flips = int((am != ao).sum().item())
    top2 = lo.topk(2, dim=1).values
    max_err = float((lm - lo).abs().max())
    hard = int(((am != ao) & (top2[:, 0] - top2[:, 1] > 2 * max_err)).sum().item())
    print("compact PSANet50@465 bf16x3: rel_l2 %.3e, max abs err %.3e, argmax flips %d / %d (margin-aware %d)"
          % (e, max_err, flips, am.numel(), hard))
    assert mask == 30 and e < 1e-3, (mask, e)
    assert hard == 0
    assert flips <= 64, flips


@pytest.mark.parametrize("combo", [(2, True, True), (2, False, False), (1, True, False)], ids=_combo_id)
def test_fused_matches_aten_composition(combo, monkeypatch):
    """Same seeded model, one training step in bf16x3: the fused kernels against SEMSEG_B200_PSA_FUSED=0 (psa_mask /
    dense view -> softmax -> bmm in ATen)."""
    from semseg_b200 import precision
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    fused = _build(*combo)[0].cuda().train()
    aten = copy.deepcopy(fused)
    x, y = util.synth(2, 65, 65, 150, seed=321, device="cuda")
    with precision.mode("bf16x3"):
        _, ml, al = fused(x, y)
        (ml + 0.4 * al).backward()
        monkeypatch.setenv("SEMSEG_B200_PSA_FUSED", "0")
        _, ml_r, al_r = aten(x, y)
        (ml_r + 0.4 * al_r).backward()
    assert abs(ml.item() - ml_r.item()) <= 1e-5 * abs(ml_r.item())
    assert abs(al.item() - al_r.item()) <= 1e-5 * abs(al_r.item())
    # every gradient to 1e-4 except, as in test_zoom_gpu's native / ATen tail comparison, the stem's last BatchNorm bias:
    # the far end of the backward and a cancelling sum over every pixel, where flipped hi/lo roundings leave ~1e-4
    loose = {"layer0.7.bias": 3e-4}
    bad = []
    for (k, pf), (_, pa) in zip(fused.named_parameters(), aten.named_parameters()):
        assert (pf.grad is None) == (pa.grad is None), k
        if pf.grad is not None and util.rel_l2(pf.grad, pa.grad) > loose.get(k, 1e-4):
            bad.append((k, util.rel_l2(pf.grad, pa.grad)))
    assert not bad, bad


@pytest.mark.parametrize("combo", [(2, True, True), (2, False, False)], ids=_combo_id)
def test_training_step_launches_no_aten_attention(combo, monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    model = _build(*combo)[0].cuda().train()
    x, y = util.synth(2, 65, 65, 150, seed=321, device="cuda")
    _, ml, al = model(x, y)                              # warm-up (weight packs, workspaces)
    (ml + 0.4 * al).backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _, ml, al = model(x, y)
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert any("psa_attend_kernel" in n for n in names) and any("psa_attn_grad_kernel" in n for n in names)
    bad = [n for n in names if any(k in n for k in ("aten::bmm", "aten::_softmax", "psamask"))]
    assert not bad, sorted(set(bad))


def _sgd_steps(model, batches, n_steps):
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
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


def test_graphed_compact_softmax_free_steps_bit_identical_to_eager(monkeypatch):
    from semseg_b200 import graphs
    base = _build(2, True, False, classes=21)[0].cuda().train()
    batches = [util.synth(2, 65, 65, 21, seed=s, device="cuda") for s in (1, 2, 3)]
    n_steps = graphs.WARMUP_CALLS + 4                    # eager warm-up calls, capture, then replays
    eager = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "0")
    le = _sgd_steps(eager, batches, n_steps)
    assert graphs.launches_per_step(eager) == 0
    graphed = copy.deepcopy(base)
    monkeypatch.setenv("SEMSEG_B200_GRAPH", "1")
    lg = _sgd_steps(graphed, batches, n_steps)
    assert graphs.launches_per_step(graphed) > 100       # the step really was captured and replayed
    assert le == lg, (le, lg)
    se, sg = eager.state_dict(), graphed.state_dict()
    for k in se:
        assert torch.equal(se[k], sg[k]), k              # weights, running statistics, num_batches_tracked
    for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
        assert (pe.grad is None) == (pg.grad is None), k
        if pe.grad is not None:
            assert torch.equal(pe.grad, pg.grad), k


def test_sliding_window_native_finish_compact_psanet(monkeypatch):
    from semseg_b200 import inference
    c = util.SW_CFG
    classes, crop = 7, 65
    model = _build(2, True, True, size=crop, classes=classes)[0].cuda().eval()
    assert inference._native_net(model, classes, crop, crop, torch.device("cuda")) is model
    image = util.sw_image(seed=11, h=100, w=150)
    scales, base = [0.4, 1.0, 1.25], 150
    with monkeypatch.context() as mp:                    # the ATen finish
        mp.setattr(inference, "_native_net", lambda *a, **k: None)
        aten = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8)
        ref_scores, ref_amax = aten(image, base, scales)
    native = inference.SlidingWindowPredictor(model, classes, crop, crop, c["mean"], c["std"], max_batch=8)
    scores, amax = native(image, base, scales)
    assert native.forward_calls == aten.forward_calls
    assert scores.shape == ref_scores.shape == (100, 150, classes)
    assert np.abs(scores - ref_scores).max() <= 1e-6
    top2 = np.sort(ref_scores, axis=2)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 2e-6
    assert clear.mean() > 0.9 and np.array_equal(amax[clear], ref_amax[clear])
