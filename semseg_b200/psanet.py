"""PSANet, drop-in for the reference's model/psanet.py (same constructor / forward signatures, child module
names, state_dict keys and return values — model/psanet.py:9-179), executed on NHWC bf16 activations.

The point-wise spatial attention block keeps the reference's arithmetic order: reduce (1x1+BN+ReLU) ->
bilinear shrink -> attention (1x1+BN+ReLU, 1x1) -> psa_mask collect/distribute -> softmax over the
H*W source positions -> aggregation bmm -> proj -> bilinear upsample -> concat.
"""
import os

import torch
from torch import nn
import torch.nn.functional as F

from . import functional as SF
from . import ops
from .psa import psa_mask
from .pspnet import _SegNet


def _interp_nhwc(x, size):
    """bilinear (align_corners=True) resize of an NHWC activation (model/psanet.py:61,97) on the native kernel."""
    return SF.resize_bilinear(x, size)


class PSA(nn.Module):
    def __init__(self, in_channels=2048, mid_channels=512, psa_type=2, compact=False, shrink_factor=2, mask_h=59,
                 mask_w=59, normalization_factor=1.0, psa_softmax=True):
        super(PSA, self).__init__()
        assert psa_type in [0, 1, 2]
        self.psa_type = psa_type
        self.compact = compact
        self.shrink_factor = shrink_factor
        self.mask_h = mask_h
        self.mask_w = mask_w
        self.psa_softmax = psa_softmax
        if normalization_factor is None:
            normalization_factor = mask_h * mask_w
        self.normalization_factor = normalization_factor

        self.reduce = nn.Sequential(
            nn.Conv2d(in_channels, mid_channels, kernel_size=1, bias=False),
            nn.BatchNorm2d(mid_channels),
            nn.ReLU(inplace=True)
        )
        self.attention = nn.Sequential(
            nn.Conv2d(mid_channels, mid_channels, kernel_size=1, bias=False),
            nn.BatchNorm2d(mid_channels),
            nn.ReLU(inplace=True),
            nn.Conv2d(mid_channels, mask_h * mask_w, kernel_size=1, bias=False),
        )
        if psa_type == 2:
            self.reduce_p = nn.Sequential(
                nn.Conv2d(in_channels, mid_channels, kernel_size=1, bias=False),
                nn.BatchNorm2d(mid_channels),
                nn.ReLU(inplace=True)
            )
            self.attention_p = nn.Sequential(
                nn.Conv2d(mid_channels, mid_channels, kernel_size=1, bias=False),
                nn.BatchNorm2d(mid_channels),
                nn.ReLU(inplace=True),
                nn.Conv2d(mid_channels, mask_h * mask_w, kernel_size=1, bias=False),
            )
        self.proj = nn.Sequential(
            nn.Conv2d(mid_channels * (2 if psa_type == 2 else 1), in_channels, kernel_size=1, bias=False),
            nn.BatchNorm2d(in_channels),
            nn.ReLU(inplace=True)
        )

    # ---- one attention branch -------------------------------------------------------------------------
    def _branch(self, x, reduce, attention, mask_type):
        """x NHWC bf16 [n,H,W,C] -> aggregated features NHWC bf16 [n,h,w,mid] at the shrunk resolution."""
        t = SF.conv_bn_act(x, reduce[0], reduce[1], relu=True)
        split = ops.is_split(t)
        n, h, w, c = t.shape[-4:]
        if self.shrink_factor != 1:
            h = (h - 1) // self.shrink_factor + 1
            w = (w - 1) // self.shrink_factor + 1
            t = _interp_nhwc(t, (h, w))
        t, t_agg = SF.fork(t, 2)                              # t feeds the attention convs and the aggregation
        a = SF.conv_bn_act(t, attention[0], attention[1], relu=True)
        y = SF.conv_bias_f32(a, attention[3])                 # fp32 NHWC [n,h,w,mask_h*mask_w]
        if (SF.psa_attend_supported(t_agg, self.mask_h, self.mask_w, self.compact)
                and os.environ.get("SEMSEG_B200_PSA_FUSED", "1") != "0"):
            # one kernel: mask gather (compact: the dense view) -> softmax over the h*w source positions (unless
            # psa_softmax is off) -> aggregation -> 1/normalization_factor (model/psanet.py:76-91); the [n, hw, hw]
            # attention map is never written to HBM. A compact mask that does not match the feature map falls through to
            # the composition below, which rejects it as the reference does.
            return SF.psa_attend(y, t_agg, mask_type, self.mask_h, self.mask_w, 1.0 / self.normalization_factor,
                                 self.compact, self.psa_softmax), (h, w)
        y = y.permute(0, 3, 1, 2).contiguous()                # NCHW fp32, the layout psa_mask is defined on
        if self.compact:
            if mask_type == 1:
                y = y.view(n, h * w, h * w).transpose(1, 2).reshape(n, h * w, h, w)
        else:
            y = psa_mask(y, mask_type, self.mask_h, self.mask_w)
        if self.psa_softmax:
            y = F.softmax(y, dim=1)
        # reference: bmm(x[n,c,hw], y[n,hw,hw]) -> [n,c,hw]; in NHWC that is y^T @ x[n,hw,c]
        tf = SF.act_to_f32(t_agg) if split else t_agg.float()
        agg = torch.bmm(y.view(n, h * w, h * w).transpose(1, 2), tf.reshape(n, h * w, c))
        agg = (agg * (1.0 / self.normalization_factor)).view(n, h, w, c)
        return (SF.f32_to_act(agg, True) if split else agg.to(torch.bfloat16)), (h, w)

    def forward_nhwc(self, x):
        if self.psa_type in [0, 1]:
            out, x1 = SF.fork(x, 2)
            t, (h, w) = self._branch(x1, self.reduce, self.attention, self.psa_type)
        else:
            out, x1, x2 = SF.fork(x, 3)
            t_col, (h, w) = self._branch(x1, self.reduce, self.attention, 0)
            t_dis, _ = self._branch(x2, self.reduce_p, self.attention_p, 1)
            t = torch.cat([t_col, t_dis], -1)
        t = SF.conv_bn_act(t, self.proj[0], self.proj[1], relu=True)
        if self.shrink_factor != 1:
            h = (h - 1) * self.shrink_factor + 1
            w = (w - 1) * self.shrink_factor + 1
            t = _interp_nhwc(t, (h, w))
        return torch.cat((out, t), -1)

    @SF.network_forward
    def forward(self, x):
        return SF.to_nchw_f32(self.forward_nhwc(SF.to_nhwc_bf16(x)))


class PSANet(_SegNet):
    def __init__(self, layers=50, dropout=0.1, classes=2, zoom_factor=8, use_psa=True, psa_type=2, compact=False,
                 shrink_factor=2, mask_h=59, mask_w=59, normalization_factor=1.0, psa_softmax=True,
                 criterion=nn.CrossEntropyLoss(ignore_index=255), pretrained=True):
        assert psa_type in [0, 1, 2]
        context = ("psa", lambda dim: PSA(dim, 512, psa_type, compact, shrink_factor, mask_h, mask_w,
                                          normalization_factor, psa_softmax))
        super(PSANet, self).__init__(layers, dropout, classes, zoom_factor, criterion, pretrained,
                                     context if use_psa else None)
        self.use_psa = use_psa

    def _context_nhwc(self, t):
        return self.psa.forward_nhwc(t) if self.use_psa else t
