"""The FusedSGD cases of tests/test_step_glue_gpu.py, and the float64 reference of one step with its error bound, shared
with tests/test_step_glue_cpu.py, which shows on these same inputs that the bound rejects plausible wrong kernels.

Sixteen parameter groups, items of every chunk-edge length (an empty one between non-empty ones) interleaved over the
groups at element offsets 0-3 of their storage, and a five-step history with rescaled learning rates, late and skipped
gradients and non-contiguous gradients."""
import collections

import numpy as np

Hyper = collections.namedtuple("Hyper", "lr momentum dampening weight_decay nesterov")

# (lr, momentum, dampening, weight decay, nesterov) of groups 0-15
GROUPS = [
    (0.1, 0.9, 0.0, 1e-4, False),
    (0.05, 0.9, 0.0, 5e-2, True),
    (0.2, 0.5, 0.3, 0.0, False),
    (0.0, 0.9, 0.3, 1e-4, False),        # lr 0: the weights stay, the buffer still moves
    (0.3, 0.0, 0.0, 5e-2, False),
    (0.07, 0.5, 0.0, 1e-4, True),
    (0.15, 0.9, 0.3, 5e-2, False),
    (0.01, 0.0, 0.3, 0.0, True),         # Nesterov without momentum is a plain step, as in torch
    (0.5, 0.5, 0.3, 5e-2, True),
    (0.02, 0.9, 0.0, 0.0, False),
    (0.25, 0.0, 0.0, 1e-4, False),
    (0.08, 0.5, 0.3, 1e-4, False),
    (0.12, 0.9, 0.3, 0.0, True),
    (0.4, 0.5, 0.0, 5e-2, False),
    (0.03, 0.0, 0.3, 5e-2, False),
    (0.06, 0.9, 0.0, 1e-4, True),
]
LENGTHS = [5, 0, 4097, 1, 4095, 3, 8193, 4, 4096, 1000003, 8191,
           4097, 8191, 1, 0, 3, 4096, 5, 4095, 4, 8193, 13]
# element offsets (parameter, gradient, buffer) into storage that starts 16-byte aligned; the buffer offset is used
# where the test owns the buffer (FusedSGD allocates its own)
OFFSETS = [(0, 0, 0), (1, 0, 0), (0, 0, 0), (0, 2, 0), (3, 3, 0), (0, 0, 0), (0, 0, 1), (2, 1, 3)]
# (group, length, parameter offset, gradient offset, buffer offset); neighbours are in different groups
ITEMS = [(k % 16, n) + OFFSETS[k % len(OFFSETS)] for k, n in enumerate(LENGTHS)]
STEPS = 5
NONCONTIGUOUS = {(2, 1), (7, 3)}        # (item, step): the gradient is a stride-2 view


def lr(gi, step):
    """Group gi's learning rate at `step`: a decaying schedule, rewritten before every step as the trainer does."""
    return GROUPS[gi][0] * 0.8 ** step


def hyper(gi, step):
    """Group gi's hyper-parameters at `step` as the kernel receives them: fp32 values."""
    _, mom, damp, wd, nesterov = GROUPS[gi]
    f = lambda v: float(np.float32(v))      # noqa: E731
    return Hyper(f(lr(gi, step)), f(mom), f(damp), f(wd), nesterov)


def has_grad(k, step):
    """Items 1, 6, 11, ... get their first gradient at step 2; items 3, 8, 13, ... have none at step 2."""
    return not ((k % 5 == 1 and step < 2) or (k % 5 == 3 and step == 2))


def weights(k):
    return np.random.default_rng(1000 + k).standard_normal(ITEMS[k][1]).astype(np.float32)


def grad(k, step):
    return np.random.default_rng(100 * k + step + 7).standard_normal(ITEMS[k][1]).astype(np.float32)


def reference(w, g, buf, hp):
    """One torch.optim.SGD step of a parameter with a gradient, in the precision of the inputs (float64 numpy arrays or
    torch tensors): (w', buf', bound on |w - w'|, bound on |buf - buf'|). buf None: no momentum buffer yet; buf' is
    None while there is none, and is `buf` itself (to be left bit for bit) in a group without momentum.

    The bounds cover an fp32 kernel with or without fused multiply-adds: a few roundings of 2^-24 relative error each on
    g' = g + wd w, buf' = mom buf + (1 - damp) g' (1 - damp rounded too), the Nesterov sum and w - lr d, so 2^-24 of the
    result plus 2^-21 (8 roundings) of every term that entered it."""
    lr_, mom, damp, wd, nesterov = hp
    gd = g + wd * w
    size_g = abs(g) + abs(wd * w)
    if mom == 0:
        w1 = w - lr_ * gd
        return w1, buf, 2.0 ** -24 * abs(w1) + 2.0 ** -21 * abs(lr_) * size_g, None
    b1 = gd if buf is None else mom * buf + (1 - damp) * gd
    d = gd + mom * b1 if nesterov else b1
    w1 = w - lr_ * d
    size_b = abs(b1) if buf is None else abs(buf) + abs(b1)
    tol_w = 2.0 ** -24 * abs(w1) + 2.0 ** -21 * abs(lr_) * (size_g + mom * size_b)
    tol_b = 2.0 ** -24 * abs(b1) + 2.0 ** -21 * (size_g if buf is None else size_g + mom * abs(buf))
    return w1, b1, tol_w, tol_b


def outside(got, want, tol):
    """Number of elements with |got - want| > tol; NaN counts as outside."""
    return int((~(abs(got - want) <= tol)).sum())
