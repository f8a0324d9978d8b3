"""CPU tier for the step-glue kernels (csrc/sgd.cu, csrc/metrics.cu).

  * the float64 bound that tests/test_step_glue_gpu.py holds FusedSGD to, on that test's own inputs, hyper-parameters
    and five-step history (tests/step_glue_cases.py): an fp32 kernel that rounds every operation separately stays
    inside it, and each plausible wrong kernel leaves it;
  * the case table covers the edges it is there for;
  * semseg_iou_hist rejects a class count over 4096 (its shared-memory histogram) and a negative pixel count before
    anything is launched."""
import ctypes

import numpy as np
import pytest

from semseg_b200 import _lib
from tests import step_glue_cases as C

F32 = np.float32

WRONG = [
    "dampening on the first step",
    "dampening ignored",
    "weight decay on the update",
    "nesterov ignored",
    "nesterov from group 0",
    "group index off by one",
    "stale buffer on a first step",
]


def _hyper(gi, step, wrong):
    if wrong == "group index off by one":
        return C.hyper((gi + 1) % len(C.GROUPS), step)
    hp = C.hyper(gi, step)
    if wrong == "nesterov ignored":
        hp = hp._replace(nesterov=False)
    if wrong == "nesterov from group 0":
        hp = hp._replace(nesterov=C.GROUPS[0][4])
    return hp


def _step32(w, g, buf, hp, wrong, stale):
    """One step of an fp32 kernel, every operation rounded on its own; `wrong` names the mistake it makes."""
    lr, mom, damp, wd = (F32(v) for v in hp[:4])
    gd = g if wrong == "weight decay on the update" else g + wd * w
    if mom == 0:
        d, b = gd, buf
    else:
        if buf is None and wrong == "stale buffer on a first step":
            buf = stale
        if buf is None:
            b = (F32(1) - damp) * gd if wrong == "dampening on the first step" else gd
        else:
            b = mom * buf + (gd if wrong == "dampening ignored" else (F32(1) - damp) * gd)
        d = gd + mom * b if hp.nesterov else b
    if wrong == "weight decay on the update":
        d = d + wd * w
    return w - lr * d, b


def _outside_over_history(wrong=None):
    """Elements outside the bound over the five steps, each step judged from the state the kernel left, as the GPU test
    does (a buffer that appears, disappears or changes where torch's would not counts as one)."""
    ws = [C.weights(k) for k in range(len(C.ITEMS))]
    bufs = [None] * len(C.ITEMS)
    bad = 0
    for s in range(C.STEPS):
        for k, (gi, n, *_) in enumerate(C.ITEMS):
            if not C.has_grad(k, s):
                continue
            g, before = C.grad(k, s), bufs[k]
            w1, b1, tol_w, tol_b = C.reference(ws[k].astype(np.float64), g.astype(np.float64),
                                               None if before is None else before.astype(np.float64), C.hyper(gi, s))
            stale = np.random.default_rng(k).standard_normal(n).astype(F32)      # what recycled memory may hold
            ws[k], bufs[k] = _step32(ws[k], g, before, _hyper(gi, s, wrong), wrong, stale)
            bad += C.outside(ws[k], w1, tol_w)
            if tol_b is not None:
                bad += C.outside(bufs[k], b1, tol_b) if bufs[k] is not None else 1
            else:                                   # no momentum: no buffer, or the old one untouched
                bad += not (bufs[k] is before or (bufs[k] is not None and before is not None
                                                  and np.array_equal(bufs[k], before)))
    return bad


def test_fp32_kernel_stays_inside_the_bound():
    assert _outside_over_history() == 0


@pytest.mark.parametrize("wrong", WRONG)
def test_bound_rejects_wrong_kernel(wrong):
    assert _outside_over_history(wrong) > 0


def test_cases_cover_the_kernel_edges():
    groups = [it[0] for it in C.ITEMS]
    assert sorted(set(groups)) == list(range(16)) and all(a != b for a, b in zip(groups, groups[1:]))
    lengths = [it[1] for it in C.ITEMS]
    assert {0, 1, 3, 4, 5, 4095, 4096, 4097, 8191, 8193, 1000003} <= set(lengths)
    assert all(0 < k < len(lengths) - 1 and lengths[k - 1] and lengths[k + 1] for k, n in enumerate(lengths) if n == 0)
    # offsets are in fp32 elements: the 16-byte vector path runs only where all three are multiples of 4
    mis = [(w % 4 != 0, g % 4 != 0, b % 4 != 0) for _, _, w, g, b in C.ITEMS]
    for kind in ((True, False, False), (False, True, False), (True, True, False), (False, False, True)):
        assert kind in mis, kind
    assert any(m == (False, False, False) and n % 4 and n > 4096 for m, n in zip(mis, lengths))   # float4 tail
    col = list(zip(*C.GROUPS))
    assert 0.0 in col[0] and set(col[1]) == {0.0, 0.5, 0.9} and set(col[2]) == {0.0, 0.3}
    assert set(col[3]) == {0.0, 1e-4, 5e-2} and set(col[4]) == {False, True} and col[4][0] is False
    assert any(C.GROUPS[gi][1] and C.GROUPS[gi][0] and C.GROUPS[gi][4] for gi in range(16))
    moving = [k for k, (gi, n, *_) in enumerate(C.ITEMS) if n and C.GROUPS[gi][1]]
    assert any(not C.has_grad(k, 0) and C.has_grad(k, C.STEPS - 1) for k in moving)             # a late first gradient
    assert any(C.has_grad(k, 0) and not all(C.has_grad(k, s) for s in range(C.STEPS)) for k in moving)
    assert all(C.has_grad(k, s) and C.ITEMS[k][1] > 1 for k, s in C.NONCONTIGUOUS)


def test_iou_hist_rejects_bad_sizes_before_launch():
    lib = _lib.load()
    P = ctypes.c_void_p(16)               # never dereferenced: every call here fails validation
    before = lib.semseg_launch_count()
    assert lib.semseg_iou_hist(P, P, 10, 4097, 255, 1, P, None) == -1
    assert b"iou_hist" in lib.semseg_last_error() and b"4097" in lib.semseg_last_error()
    assert lib.semseg_iou_hist(P, P, -1, 19, 255, 1, P, None) == -1
    assert b"iou_hist" in lib.semseg_last_error()
    assert lib.semseg_launch_count() == before
