"""torch statement of the dual-stream contract of losses.PseudoLabelLoss (streams=2; UniMatch's two strong views of
every image), the checker of tests/test_dual_cpu.py and tests/test_dual_gpu.py.

`fork` / `fold` state the prefix fork cat(f, f[:N] * s) of an M-image batch and its adjoint, d[:M] with s * d[M:] added
to its first N images; `dual_definition` the step's main loss on the per-stream logits, (main_1 + main_2) / 2 plus the
FP term of stream 1 (tests/pl_oracle.py's terms, tests/fp_oracle.py's FP term) and `dual_grad` its closed-form gradient;
`forward` composes oracle/torch_oracle.Oracle's backbone on the 2N views, its context module and cls once on
[f_1, f_2, f_1 * s] and its aux head on the 2N into the training step's (main, aux) losses. Both streams share the one
teacher map: the unmixed criterion's rule (a mix criterion's per-pixel source teacher is checked against the ATen
route instead)."""
import torch
import torch.nn.functional as F

from tests.fp_oracle import fp_definition, fp_grad
from tests.pl_oracle import effective, pl_definition, pl_grad


def fork(f, s):
    """NCHW f [M, C, h, w], scale s [N, C] (N <= M) -> cat(f, f[:N] * s) [M + N, C, h, w]."""
    n = s.shape[0]
    return torch.cat([f, f[:n] * s[:, :, None, None].to(f.dtype)], 0)


def fold(d, s):
    """The fork's adjoint: d [M + N, C, h, w] -> d[:M] with s * d[M:] added to its first N images."""
    n = s.shape[0]
    m = d.shape[0] - n
    return torch.cat([d[:n] + s[:, :, None, None].to(d.dtype) * d[m:], d[n:m]], 0)


def dual_definition(logits_nhwc, t_nhwc, ys, zoom, threshold, pl_weight, ce_weight, fp_weight, ignore_index=255):
    """main of the step from the student's NHWC logits [2N (+ N)]: the mean of PseudoLabelLoss's main on stream k's
    logits and target ys[k], plus the FP term of the perturbed logits (rows [2N, 3N)) on stream 1's target."""
    n = ys[0].shape[0]
    main = (pl_definition(logits_nhwc[:n], t_nhwc, ys[0], zoom, threshold, pl_weight, ce_weight, ignore_index) +
            pl_definition(logits_nhwc[n:2 * n], t_nhwc, ys[1], zoom, threshold, pl_weight, ce_weight,
                          ignore_index)) / 2
    if logits_nhwc.shape[0] > 2 * n:
        main = main + fp_definition(logits_nhwc[2 * n:], t_nhwc, ys[0], zoom, threshold, fp_weight, ignore_index)
    return main


def dual_grad(logits_nhwc, t_nhwc, ys, zoom, threshold, pl_weight, ce_weight, fp_weight, ignore_index=255):
    """Closed form of d dual_definition / d logits: each stream's pseudo-label gradient halved, the FP gradient of the
    perturbed rows whole, every one taken back through the upsample's adjoint."""
    n = ys[0].shape[0]
    parts = []
    for k in range(2):
        eff, wt, _ = effective(t_nhwc, ys[k], zoom, threshold, pl_weight, ce_weight, ignore_index)
        parts.append(pl_grad(logits_nhwc[k * n:(k + 1) * n], eff, wt, zoom) / 2)
    if logits_nhwc.shape[0] > 2 * n:
        parts.append(fp_grad(logits_nhwc[2 * n:], t_nhwc, ys[0], zoom, threshold, fp_weight, ignore_index))
    return torch.cat(parts, 0)


def logits(orc, x2, s=None):
    """(main [2N (+ N)], aux [2N]) 1/8-resolution NCHW logits of an Oracle in training mode: the backbone on the 2N
    views x2 (BatchNorm statistics over the 2N), the context module (PPM or PSA) and cls once on [f_1, f_2, f_1 * s]
    (s None: on [f_1, f_2]), aux on layer3."""
    f3, f4 = orc.backbone(x2)
    t = f4 if s is None else fork(f4, s)
    ctx = orc.ppm(t) if orc.arch == 'psp' else orc.psa(t)
    return orc.head(ctx, 'cls'), orc.head(f3, 'aux')


def forward(orc, x2, s, ys, t_nhwc, zoom, threshold, pl_weight, ce_weight, fp_weight, ignore_index=255):
    """(main, aux) of the step: dual_definition of the logits, and the mean over the streams of the aux head's plain
    cross-entropy on the labelled pixels of ys[k]."""
    main, aux = logits(orc, x2, s)
    loss = dual_definition(main.permute(0, 2, 3, 1), t_nhwc, ys, zoom, threshold, pl_weight, ce_weight, fp_weight,
                           ignore_index)
    if zoom != 1:
        aux = F.interpolate(aux, size=ys[0].shape[1:], mode='bilinear', align_corners=True)
    n = ys[0].shape[0]
    return loss, (F.cross_entropy(aux[:n], ys[0], ignore_index=ignore_index) +
                  F.cross_entropy(aux[n:], ys[1], ignore_index=ignore_index)) / 2
