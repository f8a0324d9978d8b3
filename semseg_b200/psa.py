"""psa_mask (collect / distribute) autograd op: drop-in for lib.psa.functional.psa_mask
(lib/psa/functional.py:4-5, lib/psa/functions/psamask.py:6-39) on the sm_90a kernel."""
import torch
from torch.autograd import Function

from . import ops


class PSAMask(Function):
    @staticmethod
    def forward(ctx, input, psa_type=0, mask_H_=None, mask_W_=None):
        assert psa_type in [0, 1]  # 0-col, 1-dis
        assert (mask_H_ is None and mask_W_ is None) or (mask_H_ is not None and mask_W_ is not None)
        num_, channels_, feature_H_, feature_W_ = input.size()
        if mask_H_ is None and mask_W_ is None:
            mask_H_, mask_W_ = 2 * feature_H_ - 1, 2 * feature_W_ - 1
        assert (mask_H_ % 2 == 1) and (mask_W_ % 2 == 1)
        assert channels_ == mask_H_ * mask_W_
        if input.dtype != torch.float32:
            raise RuntimeError("expected scalar type Float but found %s" % input.dtype)
        ctx.psa_type, ctx.mask_H_, ctx.mask_W_ = psa_type, mask_H_, mask_W_
        return ops.psamask_fwd(input.contiguous(), psa_type, mask_H_, mask_W_)

    @staticmethod
    def backward(ctx, grad_output):
        grad_input = ops.psamask_bwd(grad_output.contiguous(), ctx.psa_type, ctx.mask_H_, ctx.mask_W_)
        return grad_input, None, None, None


def psa_mask(input, psa_type=0, mask_H_=None, mask_W_=None):
    return PSAMask.apply(input, psa_type, mask_H_, mask_W_)
