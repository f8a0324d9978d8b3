"""Test-time adaptation: TENT (Wang et al., ICLR 2021) for the PSPNet / PSANet of this package.

A trained network meets a shifted test domain (other weather, another city, another camera). TENT adapts it on the test
batches themselves: each batch runs through the network with batch-statistics BatchNorm, and the BatchNorm affine
parameters take an SGD step on the mean Shannon entropy of the prediction. The prediction comes from that same forward.
The step is the package's training step with losses.EntropyLoss on an all-unlabelled target: the fused upsample +
entropy tail, graphed after a few eager calls, with no weight gradient computed for the frozen convolutions.
"""
import math

import torch
from torch import nn

from . import losses
from .optim import FusedSGD

# the modules whose BatchNorm gamma / beta TENT trains: the backbone, the context module, the classifier
_ADAPTED = ("layer0", "layer1", "layer2", "layer3", "layer4", "ppm", "psa", "cls")


class Tent:
    """Tent(model, lr, momentum=0.9, steps=1, episodic=False): test-time entropy minimisation of `model`.

    `model` is a PSPNet or PSANet of this package, bare (not wrapped in DistributedDataParallel or nn.DataParallel), on a
    CUDA device, and carrying its aux head, as a network built in training mode has (tool/test.py builds it that way).
    Anything else raises. The constructor configures the model in place, and this is all it changes:

      * model.train(): every BatchNorm takes batch statistics;
      * requires_grad_(False) on every parameter, then True on the BatchNorm weight / bias of layer0 - layer4, the
        context module (ppm / psa) and cls; the aux head stays frozen;
      * the Dropout2d of cls and aux go to eval mode, so a prediction depends only on the batch and the weights;
      * model.criterion = losses.EntropyLoss(ignore_index=<the model's>, ent_weight=1.0, ce_weight=0.0).

    It builds an optim.FusedSGD over those BatchNorm parameters (lr, momentum, no weight decay) and keeps a snapshot of
    every parameter and buffer of the model for reset().

    tent(x): x fp32 [N, 3, H, W] on the model's device with (H - 1) % 8 == 0 and (W - 1) % 8 == 0, normalised as in
    training. Runs `steps` times forward, backward and optimizer step on x, with a cached all-ignore_index int64 target at
    the model's zoomed size, and returns the int64 argmax [N, Ho, Wo] of the last forward, taken before that step's
    update, as TENT does. tent.loss holds that forward's mean entropy as a device scalar (no host synchronisation). With
    episodic=True, reset() runs before every call. The call enables autograd itself, so it may sit inside torch.no_grad().

    tent.reset(): restores the snapshot bit for bit, parameters and buffers (BatchNorm running statistics included), and
    clears the momentum buffers.

    The BatchNorm running statistics keep updating by their momentum, as in any training forward; Tent's own predictions
    never read them (they use the batch statistics). The aux head's loss is the plain cross-entropy over the labelled
    pixels, 0 with a zero gradient on the all-unlabelled target; its backward still runs. Repeated calls with one input
    shape replay one captured step (graphs.train_step)."""

    def __init__(self, model, lr, momentum=0.9, steps=1, episodic=False):
        from .pspnet import PSPNet
        from .psanet import PSANet
        if isinstance(model, (nn.parallel.DistributedDataParallel, nn.DataParallel)):
            raise TypeError("Tent: pass the bare network, not a %s wrapper (Tent adapts one model on one device)" %
                            type(model).__name__)
        if not isinstance(model, (PSPNet, PSANet)):
            raise TypeError("Tent: model must be a semseg_b200 PSPNet or PSANet, got %s" % type(model).__name__)
        if getattr(model, "aux", None) is None:
            raise ValueError("Tent: the model has no aux head; build it in training mode (as tool/test.py does) and "
                             "load the trained weights into it")
        for name, v in (("lr", lr), ("momentum", momentum)):
            if isinstance(v, bool) or not isinstance(v, (int, float)):
                raise TypeError("Tent: %s must be a number, got %r" % (name, v))
            if not (math.isfinite(v) and v >= 0.0):
                raise ValueError("Tent: %s must be finite and >= 0, got %r" % (name, v))
        if isinstance(steps, bool) or not isinstance(steps, int):
            raise TypeError("Tent: steps must be an int, got %r" % (steps,))
        if steps < 1:
            raise ValueError("Tent: steps must be >= 1, got %r" % steps)
        if not all(t.is_cuda for t in model.parameters()):
            raise ValueError("Tent: the model must be on a CUDA device (no CPU fallback)")
        self.model, self.steps, self.episodic = model, steps, bool(episodic)

        model.train()
        model.requires_grad_(False)
        params = []
        for name in _ADAPTED:
            mod = getattr(model, name, None)
            if mod is None:
                continue
            for m in mod.modules():
                if isinstance(m, nn.modules.batchnorm._BatchNorm):
                    for p in (m.weight, m.bias):
                        if p is not None:
                            params.append(p.requires_grad_(True))
        model.cls[3].eval()
        model.aux[3].eval()
        model.criterion = losses.EntropyLoss(ignore_index=getattr(model.criterion, "ignore_index", 255),
                                             ent_weight=1.0, ce_weight=0.0)
        self.params = params
        self.optimizer = FusedSGD(params, lr=lr, momentum=momentum, weight_decay=0.0)
        self._state = list(model.parameters()) + list(model.buffers())
        self._snapshot = [t.detach().clone() for t in self._state]
        self._target = None
        self.loss = None

    def reset(self):
        """Restore every parameter and buffer of the model to the snapshot taken at construction, bit for bit, and
        clear the optimizer's momentum buffers."""
        with torch.no_grad():
            torch._foreach_copy_([t.detach() for t in self._state], self._snapshot)
        self.optimizer.state.clear()

    def _ignore_target(self, x):
        n, _, hi, wi = x.shape
        z = self.model.zoom_factor
        shape = (n, (hi - 1) // 8 * z + 1, (wi - 1) // 8 * z + 1)
        y = self._target
        if y is None or tuple(y.shape) != shape or y.device != x.device:
            y = self._target = torch.full(shape, self.model.criterion.ignore_index, dtype=torch.int64,
                                          device=x.device)
        return y

    def __call__(self, x):
        if not torch.is_tensor(x) or x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("Tent: x must be an fp32 [N, 3, H, W] tensor, got %s" %
                             ("%s %s" % (x.dtype, tuple(x.shape)) if torch.is_tensor(x) else type(x).__name__))
        if (x.shape[2] - 1) % 8 or (x.shape[3] - 1) % 8:
            raise ValueError("Tent: the input size needs (H - 1) % 8 == 0 and (W - 1) % 8 == 0, got %dx%d" %
                             (x.shape[2], x.shape[3]))
        dev = self.params[0].device
        if x.device != dev:
            raise ValueError("Tent: x is on %s, the model on %s" % (x.device, dev))
        if self.episodic:
            self.reset()
        y = self._ignore_target(x)
        with torch.enable_grad():
            for _ in range(self.steps):
                pred, main, aux = self.model(x, y)
                self.optimizer.zero_grad(set_to_none=True)
                torch.autograd.backward((main, aux))
                # a replayed step hands out the graph's static outputs: copies survive the next call
                pred, self.loss = pred.clone(), main.detach().clone()
                self.optimizer.step()
        return pred
