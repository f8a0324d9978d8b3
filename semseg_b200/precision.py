"""Operand precision of the hot path — one backend, two operand policies (SURVEY.md §7 hard part 1):

  "bf16"    single-pass bf16 conv operands, bf16 activation storage: the speed configuration.
  "bf16x3"  error-compensated operands: activations and packed weights are stored as (hi, lo) bf16 pairs
            (16 mantissa bits) and every convolution accumulates x_hi*w_hi + x_lo*w_hi + x_hi*w_lo in fp32 on the
            same wgmma kernel (three K segments per block). This is the mode that meets north_star's parity bar
            (eval logits within 1e-3 of the fp32 reference, identical argmax) — the reference itself computes in
            fp32 (CPU) / TF32 (cuDNN default), model/resnet.py:63-92.

The mode is read when a model call converts its NCHW fp32 input (functional.to_nhwc_bf16); every kernel downstream
follows the storage form of its input tensor, so the two modes never mix inside one call.
Select with the environment variable SEMSEG_B200_PRECISION or `semseg_b200.precision.set_mode(...)` /
`with semseg_b200.precision.mode("bf16x3"): ...`.
"""
import contextlib
import os

MODES = ("bf16", "bf16x3")
_mode = os.environ.get("SEMSEG_B200_PRECISION", "bf16").lower()
if _mode not in MODES:
    raise ValueError("SEMSEG_B200_PRECISION must be one of %s (got %r)" % (MODES, _mode))


def get_mode():
    return _mode


def set_mode(m):
    global _mode
    if m not in MODES:
        raise ValueError("precision mode must be one of %s (got %r)" % (MODES, m))
    _mode = m


def split_enabled():
    """True when activations / weights are stored as (hi, lo) bf16 pairs."""
    return _mode == "bf16x3"


@contextlib.contextmanager
def mode(m):
    prev = _mode
    set_mode(m)
    try:
        yield
    finally:
        set_mode(prev)
