"""GPU tier: the step-glue kernels at their branch, group and chunk edges.

  * csrc/sgd.cu sgd_multi_kernel, raw and through FusedSGD, one step at a time against the float64 reference of
    tests/step_glue_cases.py from the kernel's own state before the step (no error carried across steps): 16 groups with
    their own lr (one 0), momentum 0 / 0.5 / 0.9, dampening, weight decay and Nesterov, interleaved items of every chunk
    edge length (an empty one between two others), parameters, gradients and buffers at element offsets 0-3, five steps
    with late, skipped and non-contiguous gradients;
  * FusedSGD beside torch.optim.SGD over whole runs: a late first gradient, a momentum switched off and on, Nesterov
    per group, state_dict round trips both ways mid-run, a frozen parameter (untouched, and no table rebuild per step);
  * csrc/metrics.cu iou_hist_kernel against oracle/metrics.py: ignore_index at 0, K-1 and -1, out-of-range labels
    (2^32 + 3 included), K 1 / 2 / 19 / 4096 (a 48 KB shared histogram), empty to multi-pass grids, every pixel
    ignored, 2^24 + 3 pixels of one class, write_back 0 / 1, a counts buffer full of garbage before the call.

tests/test_step_glue_cpu.py shows on the same inputs that the SGD bound rejects plausible wrong kernels."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from semseg_b200 import _lib
from tests import step_glue_cases as C

pytestmark = pytest.mark.gpu


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ SGD, step by step
def _view(values, off, n, fill=0.0):
    """A length-n fp32 CUDA view at element `off` of a fresh (16-byte aligned) allocation."""
    s = torch.full((n + 4,), fill, device="cuda")
    v = s[off:off + n]
    if values is not None:
        v.copy_(torch.from_numpy(values))
    assert n == 0 or v.data_ptr() == s.data_ptr() + 4 * off
    return v


def _grad(k, s):
    if not C.has_grad(k, s):
        return None
    _, n, _, g_off, _ = C.ITEMS[k]
    if (k, s) in C.NONCONTIGUOUS:
        g = torch.empty((n, 2), device="cuda")[:, 1]
        g.copy_(torch.from_numpy(C.grad(k, s)))
        assert not g.is_contiguous()
        return g
    return _view(C.grad(k, s), g_off, n)


def _check(where, s, k, w0, g, b0, w, b):
    """w0, b0: the kernel's fp32 state before step s (b0 None: no momentum buffer), w, b: after; g: the gradient."""
    gi, n = C.ITEMS[k][:2]
    hp = C.hyper(gi, s)
    msg = "%s: step %d, item %d (n %d, group %d %s)" % (where, s, k, n, gi, hp)
    if g is None:                                   # skipped: nothing moves
        assert _same_bits(w, w0) and (b is None) == (b0 is None) and (b is None or _same_bits(b, b0)), msg
        return
    w1, b1, tol_w, tol_b = C.reference(w0.double(), g.double(), None if b0 is None else b0.double(), hp)
    assert C.outside(w.double(), w1, tol_w) == 0, msg
    if hp.lr == 0:
        assert _same_bits(w, w0), msg
    if tol_b is None:                               # no momentum: no buffer, or the old one untouched
        assert (b is None) == (b0 is None) and (b is None or _same_bits(b, b0)), msg
    else:
        assert b is not None and C.outside(b.double(), b1, tol_b) == 0, msg


def _raw_history():
    """semseg_sgd_multi on a table in C.ITEMS order (neighbours in different groups), with the test's own buffers at
    offsets: `first` where torch would start a buffer; a buffer not started yet holds NaN (recycled memory) and must
    stay NaN until it is."""
    lib = _lib.load()
    chunk = lib.semseg_sgd_chunk_elems()
    ws = [_view(C.weights(k), w_off, n) for k, (_, n, w_off, _, _) in enumerate(C.ITEMS)]
    bs = [_view(None, b_off, n, float("nan")) for (_, n, _, _, b_off) in C.ITEMS]
    started = [False] * len(C.ITEMS)
    for s in range(C.STEPS):
        gs = [_grad(k, s) for k in range(len(C.ITEMS))]
        gs = [g if g is None or g.is_contiguous() else g.contiguous() for g in gs]     # the kernel reads dense rows
        items = (_lib.SgdItem * len(C.ITEMS))()
        c0 = 0
        for k, (gi, n, *_) in enumerate(C.ITEMS):
            it = items[k]
            it.w, it.buf, it.n, it.group, it.chunk0, it.first = ws[k].data_ptr(), bs[k].data_ptr(), n, gi, c0, \
                int(not started[k])
            c0 += (n + chunk - 1) // chunk
        h = _lib.SgdHyper()
        for gi in range(len(C.GROUPS)):
            hp = C.hyper(gi, s)
            h.lr[gi], h.momentum[gi], h.dampening[gi], h.weight_decay[gi] = hp[:4]
            h.nesterov |= int(hp.nesterov) << gi
        dev = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
        ptrs = torch.tensor([g.data_ptr() if g is not None else 0 for g in gs], dtype=torch.int64, device="cuda")
        w0 = [w.clone() for w in ws]
        b0 = [b.clone() for b in bs]
        _lib.check(lib.semseg_sgd_multi(ctypes.c_void_p(dev.data_ptr()), ctypes.c_void_p(ptrs.data_ptr()),
                                        len(C.ITEMS), c0, ctypes.byref(h), _stream()), "semseg_sgd_multi")
        torch.cuda.synchronize()
        for k, (gi, *_) in enumerate(C.ITEMS):
            now = started[k] or (gs[k] is not None and C.GROUPS[gi][1] != 0)
            if not now:
                assert _same_bits(bs[k], b0[k]), (s, k)
            _check("raw", s, k, w0[k], gs[k], b0[k] if started[k] else None, ws[k], bs[k] if now else None)
            started[k] = now


def _fused_history():
    """FusedSGD over Parameters that are views at offsets, 16 groups whose learning rates are rewritten every step."""
    from semseg_b200.optim import FusedSGD
    ps = [torch.nn.Parameter(_view(C.weights(k), w_off, n)) for k, (_, n, w_off, _, _) in enumerate(C.ITEMS)]
    groups = [dict(params=[p for p, it in zip(ps, C.ITEMS) if it[0] == gi], lr=C.lr(gi, 0), momentum=mom,
                   dampening=damp, weight_decay=wd, nesterov=nesterov)
              for gi, (_, mom, damp, wd, nesterov) in enumerate(C.GROUPS)]
    opt = FusedSGD(groups)

    def buf(p):
        return opt.state.get(p, {}).get("momentum_buffer")

    for s in range(C.STEPS):
        for gi, g in enumerate(opt.param_groups):
            g["lr"] = C.lr(gi, s)
        for k, p in enumerate(ps):
            p.grad = _grad(k, s)
        w0 = [p.detach().clone() for p in ps]
        b0 = [None if buf(p) is None else buf(p).clone() for p in ps]
        g0 = [None if p.grad is None else p.grad.clone() for p in ps]
        opt.step()
        torch.cuda.synchronize()
        for k, p in enumerate(ps):
            if (k, s) in C.NONCONTIGUOUS:           # converted in place, as torch.optim.SGD would read it
                assert p.grad.is_contiguous() and torch.equal(p.grad, g0[k])
            _check("FusedSGD", s, k, w0[k], g0[k], b0[k], p.detach(), buf(p))


@pytest.mark.parametrize("driver", ["raw", "fused"])
def test_sgd_step_by_step_against_float64(driver):
    (_raw_history if driver == "raw" else _fused_history)()


# ------------------------------------------------------------------------------------------------ FusedSGD vs torch
def _pair(groups, seed=0):
    """Identical parameters under torch.optim.SGD and FusedSGD; `groups`: [(shapes, hyper-parameter dict)]."""
    from semseg_b200.optim import FusedSGD
    g = torch.Generator(device="cuda").manual_seed(seed)
    pa = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g)) for shapes, _ in groups for s in shapes]
    pb = [torch.nn.Parameter(p.detach().clone()) for p in pa]

    def param_groups(ps):
        out, k = [], 0
        for shapes, hyper in groups:
            out.append(dict(params=ps[k:k + len(shapes)], **hyper))
            k += len(shapes)
        return out

    return pa, pb, torch.optim.SGD(param_groups(pa), lr=0.1), FusedSGD(param_groups(pb), lr=0.1), param_groups


def _give_grads(pa, pb, step, missing=()):
    g = torch.Generator(device="cuda").manual_seed(77 + step)
    for k, (a, b) in enumerate(zip(pa, pb)):
        gr = torch.randn(a.shape, device="cuda", generator=g)
        a.grad, b.grad = (None, None) if k in missing else (gr, gr.clone())


def _buffer(opt, p):
    return opt.state.get(p, {}).get("momentum_buffer")


def _assert_same_run(ta, pa, fb, pb, what):
    """Weights and momentum buffers of the two optimisers agree element by element, and have buffers for the same
    parameters."""
    for k, (a, b) in enumerate(zip(pa, pb)):
        torch.testing.assert_close(b.detach(), a.detach(), rtol=1e-5, atol=1e-6, msg="%s: weight %d" % (what, k))
    for k, (a, b) in enumerate(zip(pa, pb)):
        ba, bb = _buffer(ta, a), _buffer(fb, b)
        assert (ba is None) == (bb is None), (what, k)
        if ba is not None:
            torch.testing.assert_close(bb, ba, rtol=1e-5, atol=1e-6, msg="%s: buffer %d" % (what, k))


def test_late_first_gradient_starts_a_fresh_buffer():
    """Parameter 1 has no gradient on steps 0-1 (a head whose loss starts later, a backbone unfrozen after warm-up):
    torch starts its buffer from its first gradient at step 2. Storage FusedSGD might keep for it meanwhile is filled
    with NaN, which must never be read."""
    pa, pb, ta, fb, _ = _pair([([(300,), (4097,), (5,)], dict(momentum=0.9, weight_decay=1e-4, dampening=0.1))])
    for s in range(6):
        _give_grads(pa, pb, s, missing=(1,) if s < 2 else ())
        w1 = pb[1].detach().clone()
        ta.step()
        fb.step()
        if s < 2:
            assert _buffer(ta, pa[1]) is None and torch.equal(pb[1], w1)
            kept = fb.state.get(pb[1], {}).get("momentum_buffer")
            if kept is not None:
                kept.fill_(float("nan"))
        else:
            _assert_same_run(ta, pa, fb, pb, "step %d" % s)


def test_momentum_switched_off_and_on_follows_torch():
    """Group 0's momentum goes 0 -> 0.9 (a fresh buffer from that step's gradient), -> 0 (the buffer is left as it is)
    and -> 0.9 again (that buffer continues), beside a group that keeps its momentum."""
    pa, pb, ta, fb, _ = _pair([([(257,), (4099,)], dict(momentum=0.0, dampening=0.3, weight_decay=5e-2)),
                               ([(1000,)], dict(momentum=0.9, weight_decay=1e-4))])
    for s, mom in enumerate([0.0, 0.0, 0.9, 0.9, 0.0, 0.9, 0.9]):
        for o in (ta, fb):
            o.param_groups[0]["momentum"] = mom
        _give_grads(pa, pb, s)
        ta.step()
        fb.step()
        _assert_same_run(ta, pa, fb, pb, "step %d, momentum %g" % (s, mom))


@pytest.mark.parametrize("first_nesterov", [False, True])
def test_nesterov_per_group(first_nesterov):
    on, off = dict(momentum=0.9, nesterov=True), dict(momentum=0.9, nesterov=False)
    a, b = (on, off) if first_nesterov else (off, on)
    pa, pb, ta, fb, _ = _pair([([(4096,), (3,)], a), ([(515,)], b),
                               ([(64, 3, 3, 3)], dict(momentum=0.5, weight_decay=5e-2, nesterov=not first_nesterov))])
    for s in range(5):
        _give_grads(pa, pb, s)
        for o in (ta, fb):
            for g in o.param_groups:
                g["lr"] = 0.1 * 0.9 ** s
        ta.step()
        fb.step()
        _assert_same_run(ta, pa, fb, pb, "step %d" % s)


def test_state_dict_round_trips_mid_run():
    """After three steps (a group without momentum, a parameter still without a gradient), FusedSGD's state_dict goes
    into a torch.optim.SGD and torch's into a FusedSGD, as checkpoints do; three more steps on each side agree."""
    from semseg_b200.optim import FusedSGD
    groups = [([(300,), (17,), (4097,)], dict(momentum=0.9, weight_decay=1e-4)), ([(129,)], dict(momentum=0.0))]
    pa, pb, ta, fb, param_groups = _pair(groups)
    for s in range(3):
        _give_grads(pa, pb, s, missing=(2,))
        ta.step()
        fb.step()
    _assert_same_run(ta, pa, fb, pb, "before the round trip")
    assert sorted(fb.state_dict()["state"]) == sorted(ta.state_dict()["state"]) == [0, 1]
    pc = [torch.nn.Parameter(p.detach().clone()) for p in pb]
    tc = torch.optim.SGD(param_groups(pc), lr=0.1)
    tc.load_state_dict(copy.deepcopy(fb.state_dict()))
    pd = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    fd = FusedSGD(param_groups(pd), lr=0.1)
    fd.load_state_dict(copy.deepcopy(ta.state_dict()))
    for s in range(3, 6):
        grads = torch.Generator(device="cuda").manual_seed(s)
        for ps in zip(pa, pb, pc, pd):
            gr = torch.randn(ps[0].shape, device="cuda", generator=grads)
            for p in ps:
                p.grad = gr.clone()
        for o in (ta, fb, tc, fd):
            o.step()
        _assert_same_run(ta, pa, fb, pb, "step %d" % s)
        _assert_same_run(ta, pa, tc, pc, "step %d, torch from FusedSGD's state" % s)
        _assert_same_run(ta, pa, fd, pd, "step %d, FusedSGD from torch's state" % s)


def test_frozen_parameter_untouched_without_table_rebuilds(monkeypatch):
    """A parameter that never gets a gradient keeps its bits and no momentum buffer, and FusedSGD builds its item
    table at most twice in six steps (with and then without first-step flags), not at every step."""
    from semseg_b200.optim import FusedSGD
    builds = []
    real = FusedSGD._build
    monkeypatch.setattr(FusedSGD, "_build", lambda self, *a: builds.append(1) or real(self, *a))
    pa, pb, ta, fb, _ = _pair([([(300,), (4097,), (64, 3, 3, 3)], dict(momentum=0.9, weight_decay=1e-4))])
    pb[1].requires_grad_(False)
    frozen = pb[1].detach().clone()
    for s in range(6):
        _give_grads(pa, pb, s, missing=(1,))
        ta.step()
        fb.step()
        assert _same_bits(pb[1].detach(), frozen) and _buffer(fb, pb[1]) is None
        _assert_same_run(ta, pa, fb, pb, "step %d" % s)
    assert len(builds) <= 2, len(builds)


# ------------------------------------------------------------------------------------------------ IoU histogram
OUT_OF_RANGE = [-5, 2 ** 32 + 3]      # with K and K + 1: the low 32 bits of 2^32 + 3 are a class below K = 4096


def _labels(rng, n, K, ignore):
    """Labels in [0, K) with ignore_index and out-of-range values mixed in."""
    v = rng.integers(0, K, size=n).astype(np.int64)
    odd = np.array(OUT_OF_RANGE + [K, K + 1, ignore], dtype=np.int64)
    pick = rng.random(n) < 0.3
    v[pick] = odd[rng.integers(0, len(odd), size=int(pick.sum()))]
    return v


def _iou_raw(pred, target, K, ignore, write_back):
    """semseg_iou_hist's int32 [3][K] counts, the counts buffer full of garbage before the call."""
    lib = _lib.load()
    counts = torch.randint(-2 ** 31, 2 ** 31 - 1, (3, K), dtype=torch.int32, device="cuda")
    _lib.check(lib.semseg_iou_hist(ctypes.c_void_p(pred.data_ptr()), ctypes.c_void_p(target.data_ptr()), pred.numel(),
                                   K, ignore, write_back, ctypes.c_void_p(counts.data_ptr()), _stream()),
               "semseg_iou_hist")
    return counts.cpu().numpy().astype(np.int64)


def _check_iou(pred_np, target_np, K, ignore, write_back):
    from oracle import metrics as om
    pred, target = torch.from_numpy(pred_np).cuda(), torch.from_numpy(target_np).cuda()
    got = _iou_raw(pred, target, K, ignore, write_back)
    inter, union, area_t, masked = om.intersection_and_union(pred_np, target_np, K, ignore)
    what = "K %d, ignore %d, n %d, write_back %d" % (K, ignore, pred_np.size, write_back)
    assert np.array_equal(got[0], inter), what
    assert np.array_equal(got[1], union - area_t + inter), what
    assert np.array_equal(got[2], area_t), what
    assert np.array_equal(pred.cpu().numpy(), masked if write_back else pred_np), what


@pytest.mark.parametrize("K", [1, 2, 19, 4096])
@pytest.mark.parametrize("ignore", ["0", "K-1", "-1", "255"])
def test_iou_hist_edges(K, ignore):
    ign = {"0": 0, "K-1": K - 1, "-1": -1, "255": 255}[ignore]
    rng = np.random.default_rng(K * 7 + len(ignore))
    for k, n in enumerate([0, 1, 255, 257, 4099]):
        _check_iou(_labels(rng, n, K, ign), _labels(rng, n, K, ign), K, ign, k % 2)


@pytest.mark.parametrize("K, ignore", [(150, 255), (4096, 0)])
def test_iou_hist_past_the_grid_cap(K, ignore):
    """More pixels than 1184 blocks x 2048 take in one pass: three grid-stride passes and a remainder."""
    rng = np.random.default_rng(K)
    n = 3 * 1184 * 2048 + 1001
    _check_iou(_labels(rng, n, K, ignore), _labels(rng, n, K, ignore), K, ignore, 1)


@pytest.mark.parametrize("K, ignore", [(19, 255), (19, 3), (4096, -1)])
def test_iou_hist_every_pixel_ignored(K, ignore):
    rng = np.random.default_rng(5)
    n = 70001
    _check_iou(_labels(rng, n, K, ignore), np.full(n, ignore, dtype=np.int64), K, ignore, 1)


def test_iou_hist_one_class_counts_stay_exact():
    """2^24 + 3 pixels of class 1: the int32 counts are exact (a float32 count would round to 2^24 + 4)."""
    n = 2 ** 24 + 3
    pred = torch.ones(n, dtype=torch.int64, device="cuda")
    target = torch.ones(n, dtype=torch.int64, device="cuda")
    got = _iou_raw(pred, target, 2, 255, 1)
    assert np.array_equal(got, [[0, n], [0, n], [0, n]])


def test_iou_on_an_empty_batch_is_zero():
    """Like the reference's histc, an empty batch counts nothing (its tensors have no storage)."""
    from semseg_b200.metrics import intersectionAndUnionGPU
    e = torch.zeros((0, 5), dtype=torch.int64, device="cuda")
    for t in intersectionAndUnionGPU(e, e.clone(), 19, 255):
        assert t.shape == (19,) and not t.any()
