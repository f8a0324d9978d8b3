"""How sensitive are train-mode gradients of a random-init PSPNet50 to a tiny input perturbation?

Control experiment behind the parity tolerances (DESIGN.md §4): the same probe is run on the fp32 oracle (pure
PyTorch, TF32 off) and on the native path. If the *oracle's own* gradients decorrelate under a 1e-3 input
perturbation, element-wise end-to-end gradient parity between any two implementations that differ by rounding is not
a meaningful test, and parity has to be asserted per kernel / per block instead.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests import util  # noqa: E402


def grads_oracle(model, x, y, classes):
    orc, sd = util.oracle_from(model, "psp", layers=50, classes=classes)
    orc.train()
    _, ml, al = orc.forward(x, y)
    (ml + 0.4 * al).backward()
    return ml.item(), {k: v.grad for k, v in sd.items() if v.grad is not None}


def grads_b200(model, x, y):
    import copy
    m = copy.deepcopy(model).train()
    _, ml, al = m(x, y)
    (ml + 0.4 * al).backward()
    return ml.item(), {k: p.grad for k, p in m.named_parameters()}


def compare(ga, gb):
    errs = sorted(util.rel_l2(ga[k], gb[k]) for k in ga)
    return errs[len(errs) // 2], errs[-1]


def main():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    classes, size = 21, 129
    model = util.build_pspnet(50, classes).cuda()
    x, y = util.synth(4, size, size, classes, device="cuda")
    for eps in (1e-3, 1e-5):
        xp = x + eps * torch.randn_like(x)
        l0, g0 = grads_oracle(model, x, y, classes)
        l1, g1 = grads_oracle(model, xp, y, classes)
        med, worst = compare(g0, g1)
        print("fp32 oracle : input eps %.0e -> loss %.6f vs %.6f, grad rel-L2 median %.2e worst %.2e" %
              (eps, l0, l1, med, worst), flush=True)
        l0, g0 = grads_b200(model, x, y)
        l1, g1 = grads_b200(model, xp, y)
        med, worst = compare(g0, g1)
        print("b200 (bf16) : input eps %.0e -> loss %.6f vs %.6f, grad rel-L2 median %.2e worst %.2e" %
              (eps, l0, l1, med, worst), flush=True)
    # determinism of the b200 path: identical input twice -> identical bits
    l0, g0 = grads_b200(model, x, y)
    l1, g1 = grads_b200(model, x, y)
    same = all(torch.equal(g0[k], g1[k]) for k in g0)
    print("b200 run-to-run bit-identical gradients:", same)


if __name__ == "__main__":
    main()
