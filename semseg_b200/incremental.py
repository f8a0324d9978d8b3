"""Class-incremental semantic segmentation: growing a trained network's classifier for the next step's classes.

Each step of class-incremental training (Pascal VOC 15-5 / 15-1, ADE20K 100-50 / 50-50, ...) adds classes to the network
of the previous step. `expand_classifier` grows the student's classifier with MiB's initialisation (Cermelli et al.,
CVPR 2020), and losses.IncrementalLoss trains it with MiB's unbiased cross-entropy and unbiased distillation from the
previous step's network:

    teacher = old.eval()
    student = expand_classifier(copy.deepcopy(old).train(), new_classes)
    student.criterion = losses.IncrementalLoss(teacher)

A network that has run graphed training steps holds its CUDA graphs, which do not deep-copy: build the student as a
fresh network of the old class count, load the old state_dict into it, then expand it.
"""
import math

import torch
from torch import nn

from . import functional as SF


def _grow(conv, new_classes):
    """A copy of the 1x1 classifier `conv` with `new_classes` more output channels, MiB-initialised: each new weight row
    is the background row, and the background bias and each new bias are b_0 - log(new_classes + 1)."""
    c_old = conv.out_channels
    w, b = conv.weight, conv.bias
    out = nn.Conv2d(conv.in_channels, c_old + new_classes, 1).to(device=w.device, dtype=w.dtype)
    out.train(conv.training)
    with torch.no_grad():
        out.weight[:c_old].copy_(w)
        out.weight[c_old:].copy_(w[0:1].expand(new_classes, -1, -1, -1))
        out.bias[:c_old].copy_(b)
        b0 = b[0] - math.log(new_classes + 1)
        out.bias[0] = b0
        out.bias[c_old:] = b0
    out.weight.requires_grad_(w.requires_grad)
    out.bias.requires_grad_(b.requires_grad)
    return out


def expand_classifier(model, new_classes):
    """Grow a semseg_b200 PSPNet or PSANet by `new_classes` classes, in place, and return it.

    cls[4] (and aux[4], when the network has one) becomes an nn.Conv2d with C_old + new_classes output channels: the old
    rows are kept bit for bit, each new row is a copy of the background row (class 0), and the background bias and each
    new bias become b_0 - log(new_classes + 1). The grown network then gives every old class the probability the old
    network gave it, and splits the old background probability evenly between the background and the new classes: its
    B-mass (background plus new classes) is the old background probability. The network's cached operand slabs are
    forgotten. The state_dict has the keys and shapes of a freshly built network with C_old + new_classes classes.

    Expand before wrapping the network in DistributedDataParallel or DataParallel, and build the optimizer's parameter
    groups afterwards: the classifier's parameters are new tensors. At most 256 classes in all."""
    from .psanet import PSANet
    from .pspnet import PSPNet
    if isinstance(model, (nn.DataParallel, nn.parallel.DistributedDataParallel)):
        raise TypeError("expand_classifier: expand the bare network before wrapping it in %s" % type(model).__name__)
    if not isinstance(model, (PSPNet, PSANet)):
        raise TypeError("expand_classifier: a semseg_b200 PSPNet or PSANet expected, got %s" % type(model).__name__)
    if isinstance(new_classes, bool) or not isinstance(new_classes, int):
        raise TypeError("new_classes must be an int, got %r" % (new_classes,))
    if new_classes < 1:
        raise ValueError("new_classes must be >= 1, got %d" % new_classes)
    c = model.cls[4].out_channels + new_classes
    if c > 256:
        raise ValueError("expand_classifier: %d classes in all; the native kernels take at most 256" % c)
    model.cls[4] = _grow(model.cls[4], new_classes)
    if hasattr(model, "aux"):
        model.aux[4] = _grow(model.aux[4], new_classes)
    SF.invalidate_packs(model)
    return model
