"""torch statement of the feature-perturbation contract of losses.PseudoLabelLoss (fp_weight > 0; UniMatch's FP stream),
the checker of tests/test_fp_cpu.py and tests/test_fp_gpu.py.

`fork` / `fold` state the batch fork cat(f, f * s) and its adjoint d[:N] + s * d[N:]; `fp_definition` the FP term
(the pseudo-label term of tests/pl_oracle.py on the perturbed logits, weight fp_weight, no labelled term) and `fp_grad`
its closed-form gradient; `forward` composes oracle/torch_oracle.Oracle's backbone, context module and heads on the
forked batch into the training step's (main, aux) losses."""
import torch
import torch.nn.functional as F

from tests.pl_oracle import effective, pl_definition, pl_grad


def fork(f, s):
    """NCHW f [N, C, h, w], scale s [N, C] -> cat(f, f * s) [2N, C, h, w]."""
    return torch.cat([f, f * s[:, :, None, None].to(f.dtype)], 0)


def fold(d, s):
    """The fork's adjoint: d [2N, C, h, w] -> d[:N] + s * d[N:]."""
    n = d.shape[0] // 2
    return d[:n] + s[:, :, None, None].to(d.dtype) * d[n:]


def fp_definition(s_fp_nhwc, t_nhwc, target, zoom, threshold, fp_weight, ignore_index=255):
    """fp_weight (1/|U|) sum_{U, conf >= threshold} (lse(s_fp) - s_fp[yhat]) at the target's size (0 for an empty U)."""
    return pl_definition(s_fp_nhwc, t_nhwc, target, zoom, threshold, fp_weight, 0.0, ignore_index)


def fp_grad(s_fp_nhwc, t_nhwc, target, zoom, threshold, fp_weight, ignore_index=255):
    """Closed form of d fp_definition / d s_fp: (fp_weight / |U|) (softmax(s_fp) - onehot(yhat)) on the confident
    unlabelled pixels, taken back through the upsample's adjoint."""
    eff, wt, _ = effective(t_nhwc, target, zoom, threshold, fp_weight, 0.0, ignore_index)
    return pl_grad(s_fp_nhwc, eff, wt, zoom)


def logits(orc, x, s):
    """(main, fp, aux) 1/8-resolution NCHW logits of an Oracle in training mode: the backbone on x, the context module
    (PPM or PSA) and cls once on the forked layer4 output (BatchNorm statistics over the 2N images), aux on layer3."""
    f3, f4 = orc.backbone(x)
    t = fork(f4, s)
    ctx = orc.ppm(t) if orc.arch == 'psp' else orc.psa(t)
    both = orc.head(ctx, 'cls')
    n = x.shape[0]
    return both[:n], both[n:], orc.head(f3, 'aux')


def forward(orc, x, s, y, t_nhwc, zoom, threshold, pl_weight, ce_weight, fp_weight, ignore_index=255):
    """(main, aux) of the step: PseudoLabelLoss's main of the clean stream plus the FP term of the perturbed one, and
    the plain cross-entropy of the aux head on the labelled pixels."""
    main, fp, aux = logits(orc, x, s)
    nhwc = lambda v: v.permute(0, 2, 3, 1)          # noqa: E731
    loss = pl_definition(nhwc(main), t_nhwc, y, zoom, threshold, pl_weight, ce_weight, ignore_index) + \
        fp_definition(nhwc(fp), t_nhwc, y, zoom, threshold, fp_weight, ignore_index)
    if zoom != 1:
        aux = F.interpolate(aux, size=y.shape[1:], mode='bilinear', align_corners=True)
    return loss, F.cross_entropy(aux, y, ignore_index=ignore_index)
