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
from . import graphs
from . import ops
from . import p2p
from . import resnet as models
from .psa import psa_mask
from .pspnet import head_forward_nhwc, upsample_logits


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
        if (self.psa_softmax and not self.compact and SF.psa_attend_supported(t_agg, self.mask_h, self.mask_w)
                and os.environ.get("SEMSEG_B200_PSA_FUSED", "1") != "0"):
            # one kernel: mask gather -> softmax over the h*w source positions -> aggregation -> 1/normalization_factor
            # (model/psanet.py:81-91); the [n, hw, hw] attention map is never written to HBM
            return SF.psa_attend(y, t_agg, mask_type, self.mask_h, self.mask_w, 1.0 / self.normalization_factor), (h, w)
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


class PSANet(nn.Module):
    def __init__(self, layers=50, dropout=0.1, classes=2, zoom_factor=8, use_psa=True, psa_type=2, compact=False,
                 shrink_factor=2, mask_h=59, mask_w=59, normalization_factor=1.0, psa_softmax=True,
                 criterion=nn.CrossEntropyLoss(ignore_index=255), pretrained=True):
        super(PSANet, self).__init__()
        assert layers in [50, 101, 152]
        assert classes > 1
        assert zoom_factor in [1, 2, 4, 8]
        assert psa_type in [0, 1, 2]
        self.zoom_factor = zoom_factor
        self.use_psa = use_psa
        self.criterion = criterion

        if layers == 50:
            resnet = models.resnet50(pretrained=pretrained)
        elif layers == 101:
            resnet = models.resnet101(pretrained=pretrained)
        else:
            resnet = models.resnet152(pretrained=pretrained)
        self.layer0 = resnet.stem()
        self.layer1, self.layer2, self.layer3, self.layer4 = resnet.layer1, resnet.layer2, resnet.layer3, resnet.layer4

        for n, m in self.layer3.named_modules():
            if 'conv2' in n:
                m.dilation, m.padding, m.stride = (2, 2), (2, 2), (1, 1)
            elif 'downsample.0' in n:
                m.stride = (1, 1)
        for n, m in self.layer4.named_modules():
            if 'conv2' in n:
                m.dilation, m.padding, m.stride = (4, 4), (4, 4), (1, 1)
            elif 'downsample.0' in n:
                m.stride = (1, 1)

        fea_dim = 2048
        if use_psa:
            self.psa = PSA(fea_dim, 512, psa_type, compact, shrink_factor, mask_h, mask_w, normalization_factor,
                           psa_softmax)
            fea_dim *= 2
        self.cls = nn.Sequential(
            nn.Conv2d(fea_dim, 512, kernel_size=3, padding=1, bias=False),
            nn.BatchNorm2d(512),
            nn.ReLU(inplace=True),
            nn.Dropout2d(p=dropout),
            nn.Conv2d(512, classes, kernel_size=1)
        )
        if self.training:
            self.aux = nn.Sequential(
                nn.Conv2d(1024, 256, kernel_size=3, padding=1, bias=False),
                nn.BatchNorm2d(256),
                nn.ReLU(inplace=True),
                nn.Dropout2d(p=dropout),
                nn.Conv2d(256, classes, kernel_size=1)
            )

    _sb_head_modules = ("layer0", "layer1", "layer2")     # modules whose parameters lie before graphs.note_boundary

    def forward(self, x, y=None):
        x_size = x.size()
        assert (x_size[2] - 1) % 8 == 0 and (x_size[3] - 1) % 8 == 0
        if (self.training and torch.is_grad_enabled() and y is not None and
                SF.fused_tail_supported(self.criterion, None, y, self.zoom_factor, x_size)):
            # whole training step (forward and, later, backward) as two replayed CUDA graphs behind one autograd node
            out = graphs.train_step(self, self._forward_impl, x, y)
            if out is not None:
                return out
        return self._forward_impl(x, y)

    @SF.network_forward
    def _forward_impl(self, x, y=None):
        x_size = x.size()
        h = int((x_size[2] - 1) / 8 * self.zoom_factor + 1)
        w = int((x_size[3] - 1) / 8 * self.zoom_factor + 1)

        if self.training and torch.is_grad_enabled():
            SF.prepack(self, force=graphs.capturing())   # all conv operand slabs refreshed in one launch
            p2p.begin_step(force=graphs.capturing())     # new SyncBN exchange epoch (device-resident step counter)
        logits, t_aux = self._logits_nhwc(x)

        if self.training:
            aux_logits = head_forward_nhwc(self.aux, t_aux)
            if SF.fused_tail_supported(self.criterion, logits, y, self.zoom_factor):
                # upsample + cross-entropy + argmax fused: [N, classes, H, W] never exists (model/pspnet.py:94-103)
                main_loss, pred = SF.upsample_ce(logits, y, self.criterion.ignore_index)
                aux_loss, _ = SF.upsample_ce(aux_logits, y, self.criterion.ignore_index)
                return pred, main_loss, aux_loss
            x = upsample_logits(logits, (h, w), self.zoom_factor)
            aux = upsample_logits(aux_logits, (h, w), self.zoom_factor)
            main_loss = self.criterion(x, y)
            aux_loss = self.criterion(aux, y)
            return x.max(1)[1], main_loss, aux_loss
        else:
            x = ops.nhwc_f32_to_nchw(logits) if not logits.requires_grad else logits.permute(0, 3, 1, 2).contiguous()
            if self.zoom_factor != 1:
                x = F.interpolate(x, size=(h, w), mode='bilinear', align_corners=True)
            return x

    def _logits_nhwc(self, x):
        """fp32 NHWC classifier logits [N, h', w', classes] before the final upsample, and in training mode layer3's
        output for the aux head (None in eval mode)."""
        t = SF.to_nhwc_bf16(x)
        t = self.layer0.forward_nhwc(t)
        t = self.layer1.forward_nhwc(t)
        t = graphs.note_boundary(self.layer2.forward_nhwc(t))     # where a captured backward is cut in two
        t_tmp = self.layer3.forward_nhwc(t)
        t_aux = None
        if self.training:       # layer3's output feeds layer4 and the aux head: explicit fan-out (native gradient add)
            t_tmp, t_aux = SF.fork(t_tmp, 2)
        t = self.layer4.forward_nhwc(t_tmp)
        if self.use_psa:
            t = self.psa.forward_nhwc(t)
        return head_forward_nhwc(self.cls, t), t_aux

    def _eval_logits_nhwc(self, x):
        """The eval forward up to the classifier: fp32 NHWC logits [N, h', w', classes]. The sliding-window engine
        (inference.py) upsamples, scores and flip-averages them in one native kernel."""
        assert not self.training, "_eval_logits_nhwc is the eval-mode forward"
        return self._logits_nhwc(x)[0]
