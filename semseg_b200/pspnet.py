"""PSPNet, drop-in for the reference's model/pspnet.py (same constructor / forward signatures, same child
module names and state_dict keys, same return values — model/pspnet.py:29-105), executed on NHWC bf16
activations by the sm_90a kernels behind semseg_b200/functional.py.
"""
import torch
from torch import nn
import torch.nn.functional as F

from . import functional as SF
from . import graphs
from . import losses
from . import ops
from . import p2p
from . import resnet as models


class PPM(nn.Module):
    """Pyramid pooling module (model/pspnet.py:8-26): per bin AdaptiveAvgPool2d -> 1x1 conv -> BN -> ReLU ->
    bilinear upsample (align_corners=True) -> concat with the input."""

    def __init__(self, in_dim, reduction_dim, bins):
        super(PPM, self).__init__()
        self.features = []
        for bin in bins:
            self.features.append(nn.Sequential(
                nn.AdaptiveAvgPool2d(bin),
                nn.Conv2d(in_dim, reduction_dim, kernel_size=1, bias=False),
                nn.BatchNorm2d(reduction_dim),
                nn.ReLU(inplace=True)
            ))
        self.features = nn.ModuleList(self.features)

    def forward_nhwc(self, x):
        bins = []
        for f in self.features:
            b = f[0].output_size
            bins.append(b if isinstance(b, int) else b[0])
        link = SF.ppm_link()                                     # the two gradients of x are summed in the pool-bwd kernel
        pooled = SF.ppm_pool(x, bins, link)                      # one launch: every bin's AdaptiveAvgPool2d
        feats = [SF.conv_bn_act(p, f[1], f[2], relu=True) for p, f in zip(pooled, self.features)]
        return SF.ppm_upsample_concat(x, feats, bins, link)      # one launch: upsample x4 + concat, written in place

    @SF.network_forward
    def forward(self, x):
        return SF.to_nchw_f32(self.forward_nhwc(SF.to_nhwc_bf16(x)))


def head_forward_nhwc(head, t):
    """cls / aux head: 3x3 conv + BN + ReLU + Dropout2d + 1x1 conv with bias -> fp32 NHWC logits."""
    t = SF.conv_bn_act(t, head[0], head[1], relu=True)
    t = SF.dropout2d_nhwc(t, head[3].p, head[3].training)
    return SF.conv_bias_f32(t, head[4])


def upsample_logits(logits_nhwc, size, zoom_factor):
    """fp32 NHWC logits -> NCHW (view) bilinearly upsampled to `size` (model/pspnet.py:94-95)."""
    x = logits_nhwc.permute(0, 3, 1, 2)
    if zoom_factor != 1:
        x = F.interpolate(x, size=size, mode='bilinear', align_corners=True)
    return x


def _chunks(t, k):
    """`t` split into k equal chunks along the batch (k = 1: the tensor itself, no view)."""
    return t.chunk(k) if k > 1 else (t,)


def _stream_mean(terms):
    """The mean of the per-stream losses (one stream: its loss itself, no extra kernel)."""
    return terms[0] if len(terms) == 1 else sum(terms[1:], terms[0]) / len(terms)


class _SegNet(nn.Module):
    """The network body PSPNet and PSANet share (model/pspnet.py:29-105, model/psanet.py:101-179): the dilated ResNet,
    a context module between layer4 and `cls`, the `cls` / `aux` heads and the forward. `context` is None or
    (attribute name, factory called with the feature width); the subclass applies the module in `_context_nhwc`."""

    def __init__(self, layers, dropout, classes, zoom_factor, criterion, pretrained, context):
        super(_SegNet, self).__init__()
        assert layers in [50, 101, 152]
        assert classes > 1
        assert zoom_factor in [1, 2, 4, 8]
        self.zoom_factor = zoom_factor
        self.criterion = criterion

        if layers == 50:
            resnet = models.resnet50(pretrained=pretrained)
        elif layers == 101:
            resnet = models.resnet101(pretrained=pretrained)
        else:
            resnet = models.resnet152(pretrained=pretrained)
        self.layer0 = resnet.stem()
        self.layer1, self.layer2, self.layer3, self.layer4 = resnet.layer1, resnet.layer2, resnet.layer3, resnet.layer4

        # output stride 8: dilate layer3 / layer4 instead of striding (model/pspnet.py:49-58)
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
        if context is not None:
            name, make = context
            setattr(self, name, make(fea_dim))       # built here: construction order decides the initial weights
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
        t_logits = mix_mask = fp_scale = None
        streams = 1
        if self.training and y is not None and isinstance(self.criterion, losses._TeacherLoss):
            classes = self.cls[4].out_channels
            mixing = isinstance(self.criterion, losses.MixPseudoLabelLoss)
            streams = getattr(self.criterion, "streams", 1)
            u = self.criterion.draw(x, classes) if mixing else None      # the draws come before the teacher forward
            strong = self.criterion.strong
            u_s = None if strong is None else strong.draw(x) if streams == 1 else strong.draw(x, streams)
            if getattr(self.criterion, "fp_weight", 0.0) > 0.0:
                fp_scale = self.criterion.fp_draw(x, self.layer4[-1].conv3.out_channels)
            # the teacher first (distillation, pseudo-labels): its activations are transient before the student's saved
            # ones exist. It sees the batch; the student and both heads' losses see its strong view, mixed
            t_logits = self.criterion.run_teacher(x, classes)
            if strong is not None:
                x = self.criterion.strong_streams(x, u_s) if streams > 1 else self.criterion.strong_view(x, u_s)
            if mixing:
                x, y, mix_mask = self.criterion.mix_batch(x, y, u, t_logits, self.zoom_factor)
        # the student's batch: `streams` views of the N images, stream-major, and with the FP stream stream 1's
        # perturbed copy after them. Each stream's logits, aux logits, target and mix mask are a contiguous N-image chunk
        # without the FP stream the call is the one-argument form it always was (subclasses and wrappers override it)
        out, t_aux = self._logits_nhwc(x) if fp_scale is None else self._logits_nhwc(x, fp_scale)
        logits = _chunks(out, streams + (fp_scale is not None))
        fp_logits = logits[streams] if fp_scale is not None else None

        if self.training:
            aux_logits = _chunks(head_forward_nhwc(self.aux, t_aux), streams)
            ys = _chunks(y, streams) if mix_mask is not None else (y,) * streams      # the mixed target is [2N]
            masks = _chunks(mix_mask, streams) if mix_mask is not None else (None,) * streams
            if SF.fused_tail_supported(self.criterion, logits[0], y, self.zoom_factor):
                # upsample + cross-entropy + argmax fused: [N, classes, H, W] never exists (model/pspnet.py:94-103);
                # one call per stream: each has its own target, mask and normalisers, and the one teacher map
                mains, preds = zip(*(SF.upsample_ce(logits[k], ys[k], self.criterion.ignore_index, self.zoom_factor,
                                                    criterion=self.criterion, teacher_logits=t_logits,
                                                    mix_mask=masks[k]) for k in range(streams)))
                main_loss = _stream_mean(mains)
                if fp_logits is not None:
                    main_loss = main_loss + SF.upsample_fp(fp_logits, ys[0], self.zoom_factor, self.criterion,
                                                           t_logits, masks[0])[0]
                aux_loss = _stream_mean([SF.upsample_ce(a, y_k, self.criterion.ignore_index, self.zoom_factor,
                                                        criterion=self.criterion)[0] for a, y_k in zip(aux_logits, ys)])
                return preds[0], main_loss, aux_loss
            ups = [upsample_logits(v, (h, w), self.zoom_factor) for v in logits[:streams]]
            aux_ups = [upsample_logits(v, (h, w), self.zoom_factor) for v in aux_logits]
            if t_logits is not None:
                t_up = upsample_logits(t_logits, (h, w), self.zoom_factor)
                t_ups = [t_up] * streams
                if mix_mask is not None:
                    # each target pixel's teacher map is its source image's: the mask read at the target grid
                    s = 8 // self.zoom_factor
                    t_ups = [torch.where(m[:, ::s, ::s].unsqueeze(1).bool(), t_up.roll(-1, 0), t_up) for m in masks]
                main_loss = _stream_mean([self.criterion(v, y_k, teacher_logits=t_k)
                                          for v, y_k, t_k in zip(ups, ys, t_ups)])
                if fp_logits is not None:
                    main_loss = main_loss + self.criterion.fp_loss(upsample_logits(fp_logits, (h, w), self.zoom_factor),
                                                                   ys[0], t_ups[0])
            else:
                main_loss = self.criterion(ups[0], y)
            aux_loss = _stream_mean([self.criterion(a, y_k) for a, y_k in zip(aux_ups, ys)])
            return ups[0].max(1)[1], main_loss, aux_loss
        else:
            x = logits[0]
            x = ops.nhwc_f32_to_nchw(x) if not x.requires_grad else x.permute(0, 3, 1, 2).contiguous()
            if self.zoom_factor != 1:
                x = F.interpolate(x, size=(h, w), mode='bilinear', align_corners=True)
            return x

    def _logits_nhwc(self, x, fp_scale=None):
        """fp32 NHWC classifier logits [M, h', w', classes] of an M-image batch before the final upsample, and in
        training mode layer3's output for the aux head (None in eval mode). With `fp_scale` (fp32 [N, 2048], N <= M, the
        feature-perturbation factor of losses.PseudoLabelLoss) the context module and cls run on cat(f, f[:N] *
        fp_scale) of layer4's output f: logits [M + N, h', w', classes], the unperturbed images first."""
        t = self.layer0.forward_nchw(x)          # x.grad, when asked for, straight from the stem dgrad kernel
        t = self.layer1.forward_nhwc(t)
        t = graphs.note_boundary(self.layer2.forward_nhwc(t))     # where a captured backward is cut in two
        t_tmp = self.layer3.forward_nhwc(t)
        t_aux = None
        if self.training:       # layer3's output feeds layer4 and the aux head: explicit fan-out (native gradient add)
            t_tmp, t_aux = SF.fork(t_tmp, 2)
        t = self.layer4.forward_nhwc(t_tmp)
        if fp_scale is not None:
            t = SF.fp_fork(t, fp_scale)
        return head_forward_nhwc(self.cls, self._context_nhwc(t)), t_aux

    def _eval_logits_nhwc(self, x):
        """The eval forward up to the classifier: fp32 NHWC logits [N, h', w', classes]. The sliding-window engine
        (inference.py) upsamples, scores and flip-averages them in one native kernel."""
        assert not self.training, "_eval_logits_nhwc is the eval-mode forward"
        return self._logits_nhwc(x)[0]


class PSPNet(_SegNet):
    def __init__(self, layers=50, bins=(1, 2, 3, 6), dropout=0.1, classes=2, zoom_factor=8, use_ppm=True,
                 criterion=nn.CrossEntropyLoss(ignore_index=255), pretrained=True):
        assert 2048 % len(bins) == 0
        super(PSPNet, self).__init__(layers, dropout, classes, zoom_factor, criterion, pretrained,
                                     ("ppm", lambda dim: PPM(dim, int(dim / len(bins)), bins)) if use_ppm else None)
        self.use_ppm = use_ppm

    def _context_nhwc(self, t):
        return self.ppm.forward_nhwc(t) if self.use_ppm else t
