"""L-infinity PGD and SegPGD attacks on PSPNet / PSANet, on the fused upsample + cross-entropy tail and graphed.

PGD (Madry et al., ICLR 2018) and SegPGD (Gu et al., ECCV 2022) perturb the input within an eps-ball around the clean
image, in pixel units, by K steps of size alpha along the sign of the loss gradient. Each iteration runs

    1. the eval-mode differentiable forward to the 1/8-resolution logits (functional.network_mode(False,
       input_grad=True): frozen BatchNorm stages, bit-identical to the eval forward),
    2. the fused-tail loss: the plain cross-entropy (kind='pgd', the _UpsampleCE kernels) or the SegPGD loss
       (kind='segpgd': each valid pixel's nll weighted 1 - lambda_t where the prediction is right and lambda_t where
       it is wrong, lambda_t = (t - 1) / (2K) at iteration t = 1..K), so the [N, classes, H, W] logits never exist,
    3. its input gradient from the stem dgrad kernel, and
    4. the projected sign step (csrc/adversarial.cu), which also keeps every pixel inside [0, 255].

The network's parameters are constants throughout: no weight gradient is computed (even for parameters that require
one), no `.grad` is touched and no buffer changes. After graphs.WARMUP_CALLS eager calls with an unchanged key, the
whole attack (the weight re-pack, the random start and all K iterations) replays as one CUDA graph. The same function
runs the attack inside a training step for PGD adversarial training (losses.AdversarialLoss).
"""
import contextlib
import math
import os
import warnings

import torch
from torch import nn

from . import functional as SF
from . import graphs
from . import losses
from . import ops
from . import precision

# the trainer's normalisation in 0-255 pixel units (value_scale = 255, tool/train.py)
IMAGENET_MEAN = (0.485 * 255, 0.456 * 255, 0.406 * 255)
IMAGENET_STD = (0.229 * 255, 0.224 * 255, 0.225 * 255)
KINDS = ("pgd", "segpgd")


def _number(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise TypeError("%s must be a number, got %r" % (name, v))
    v = float(v)
    if not math.isfinite(v):
        raise ValueError("%s must be finite, got %r" % (name, v))
    return v


def _triple(name, v, positive):
    if isinstance(v, (str, bytes)) or not hasattr(v, "__len__") or len(v) != 3:
        raise TypeError("%s must hold three numbers (one per channel), got %r" % (name, v))
    out = tuple(_number("%s[%d]" % (name, k), e) for k, e in enumerate(v))
    if positive and not all(e > 0.0 for e in out):
        raise ValueError("%s must be positive, got %r" % (name, out))
    return out


def segpgd_lambdas(steps):
    """SegPGD's weight schedule: lambda_t = (t - 1) / (2 steps) at iteration t = 1..steps."""
    return [(t - 1) / (2.0 * steps) for t in range(1, steps + 1)]


@contextlib.contextmanager
def constant_parameters(model):
    """Every parameter of `model` replaced by a detached alias of its storage for the enclosed code: the network's
    autograd nodes see constants, so no weight gradient is computed and nothing reaches `.grad`, while the kernels read
    the same memory (an in-place edit is seen). Inside a captured training step the aliases are of the capture's
    parameter proxies."""
    slots = [(m, name, p) for m in model.modules() for name, p in m._parameters.items()
             if p is not None and p.requires_grad]
    for m, name, p in slots:
        m._parameters[name] = p.detach()
    try:
        yield
    finally:
        for m, name, p in slots:
            m._parameters[name] = p


def run(model, attack, x0, y):
    """The attack itself: -> (x_adv fp32 NCHW, per-iteration losses fp32 [steps]), both on the device, without a host
    synchronisation. `model` must have every module in eval mode and its operand slabs packed (functional.prepack); the
    caller checks its inputs. PGDAttack.attack and losses.AdversarialLoss (inside a training step) both call this."""
    box = attack._box
    x0 = x0.detach().contiguous()
    y = y.contiguous()
    zoom = model.zoom_factor
    if attack.random_start:
        x = ops.adv_start(x0, torch.rand(x0.shape, device=x0.device), box)
    else:
        x = x0.clone()
    lams = segpgd_lambdas(attack.steps) if attack.kind == "segpgd" else None
    per_step = []
    with constant_parameters(model), graphs.no_boundary(), torch.enable_grad(), \
            SF.network_mode(False, input_grad=True):
        for t in range(attack.steps):
            xg = x.detach().requires_grad_(True)
            logits = model._logits_nhwc(xg)[0]
            if lams is None:
                loss, _ = SF._UpsampleCE.apply(logits, y, attack.ignore_index, zoom)
            else:
                loss, _ = SF.upsample_segpgd(logits, y, attack.ignore_index, zoom, lams[t])
            (g,) = torch.autograd.grad(loss, xg)
            per_step.append(loss.detach())
            del logits, loss, xg
            ops.adv_step(x, g, x0, box, out=x)
    return x, torch.stack(per_step)


def check_model(model, name):
    """A bare PSPNet / PSANet of this package with native kernels: no DataParallel / DDP wrapper, no Fp8Eval."""
    from .fp8 import Fp8Eval
    from .pspnet import _SegNet
    if isinstance(model, Fp8Eval):
        raise TypeError("%s: Fp8Eval has no backward; attack the bf16 model it wraps" % name)
    if isinstance(model, (nn.DataParallel, nn.parallel.DistributedDataParallel)):
        raise TypeError("%s: pass the bare network (model.module), not its %s wrapper" % (name, type(model).__name__))
    if not isinstance(model, _SegNet):
        raise TypeError("%s: the model must be a semseg_b200 PSPNet or PSANet, got %s" % (name, type(model).__name__))


def check_inputs(model, x, y, kind, name):
    """x fp32 CUDA [N, 3, H, W] with (H-1) % 8 == 0 and (W-1) % 8 == 0; y int64 at the model's zoomed size, no wider
    than the `kind` attack's tail kernels stage."""
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
        raise TypeError("%s: the input must be a CUDA fp32 [N, 3, H, W] tensor, got %s" %
                        (name, (x.dtype, tuple(x.shape), str(x.device)) if torch.is_tensor(x) else type(x).__name__))
    if (x.shape[2] - 1) % 8 != 0 or (x.shape[3] - 1) % 8 != 0:
        raise ValueError("%s: the input size must be 8k+1 each way, got %dx%d" % (name, x.shape[2], x.shape[3]))
    if not (torch.is_tensor(y) and y.dtype == torch.int64 and y.device == x.device and y.dim() == 3):
        raise TypeError("%s: the target must be an int64 [N, H', W'] tensor on %s" % (name, x.device))
    # the SegPGD backward is the focal one: its width limit
    tail = _PLAIN_CE if kind == "pgd" else _FOCAL
    if y.shape[0] != x.shape[0] or not SF.fused_tail_supported(tail, None, y, model.zoom_factor, x.shape):
        z = model.zoom_factor
        raise ValueError("%s: the target must be [%d, %d, %d] (the model's zoom %d; SegPGD at most 2389 columns at "
                         "zoom 8), got %s" % (name, x.shape[0], z * ((x.shape[2] - 1) // 8) + 1,
                                              z * ((x.shape[3] - 1) // 8) + 1, z, tuple(y.shape)))


_PLAIN_CE = nn.CrossEntropyLoss()
_FOCAL = losses.FocalLoss(gamma=0.0)


class _Graph:
    __slots__ = ("calls", "failed", "graph", "pool", "x", "y", "out", "losses", "keep")

    def __init__(self):
        self.calls, self.failed, self.graph = 0, False, None


class PGDAttack:
    """L-infinity PGD (kind='pgd', cross-entropy) or SegPGD (kind='segpgd') on a PSPNet / PSANet of this package.

    eps (>= 0) and alpha (> 0) are in 0-255 pixel units like `mean` and `std`, the trainer's normalisation (default:
    ImageNet's, value_scale 255); the input is the normalised batch the network sees. `steps` >= 1 iterations, each
    x <- clip_box(clip_ball(x + alpha sign(grad))), from a uniform random start in the ball (random_start) or the clean
    image. FGSM is PGDAttack(eps, alpha=eps, steps=1, random_start=False). Pixels of `ignore_index` (and targets
    outside [0, classes)) do not count in the loss.

    `attack(model, x, y)` (or calling the object) returns the adversarial batch, fp32 NCHW, detached; `losses` is then
    the device fp32 [steps] tensor of the per-iteration losses. `model` is a bare PSPNet / PSANet on CUDA with every
    module in eval mode; `x` fp32 [N, 3, H, W] with (H-1) % 8 == 0 and (W-1) % 8 == 0; `y` int64 at the model's zoomed
    size. The model's parameters, buffers, `.grad` and modes are left as they are.

    Graphed: after graphs.WARMUP_CALLS eager calls with the same shapes, zoom, precision mode, parameter storage and
    options, the whole attack replays as one CUDA graph that re-packs the weights first (in-place weight edits are
    seen), draws fresh random starts from torch's generator and runs the K iterations. At most graphs.MAX_GRAPHS
    captures per model; SEMSEG_B200_GRAPH=0 disables capture, and a failed capture warns and stays eager."""

    def __init__(self, eps, alpha, steps, kind="pgd", random_start=True, mean=IMAGENET_MEAN, std=IMAGENET_STD,
                 ignore_index=255):
        self.eps = _number("eps", eps)
        if self.eps < 0.0:
            raise ValueError("eps must be >= 0, got %r" % eps)
        self.alpha = _number("alpha", alpha)
        if self.alpha <= 0.0:
            raise ValueError("alpha must be > 0, got %r" % alpha)
        if isinstance(steps, bool) or not isinstance(steps, int):
            raise TypeError("steps must be an int, got %r" % (steps,))
        if steps < 1:
            raise ValueError("steps must be >= 1, got %r" % steps)
        if not isinstance(kind, str):
            raise TypeError("kind must be one of %s, got %r" % (KINDS, kind))
        if kind not in KINDS:
            raise ValueError("kind must be one of %s, got %r" % (KINDS, kind))
        if not isinstance(random_start, bool):
            raise TypeError("random_start must be a bool, got %r" % (random_start,))
        if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
            raise TypeError("ignore_index must be an int, got %r" % (ignore_index,))
        self.steps, self.kind, self.random_start, self.ignore_index = steps, kind, random_start, ignore_index
        self.mean = _triple("mean", mean, False)
        self.std = _triple("std", std, True)
        self._box = ops.adv_box(self.eps, self.alpha, self.mean, self.std)
        self.losses = None

    def __repr__(self):
        return "PGDAttack(eps=%g, alpha=%g, steps=%d, kind=%r, random_start=%r, mean=%r, std=%r, ignore_index=%d)" % (
            self.eps, self.alpha, self.steps, self.kind, self.random_start, self.mean, self.std, self.ignore_index)

    def key(self):
        """The options a captured attack bakes in (launch arguments and the iteration count)."""
        return (self.eps, self.alpha, self.steps, self.kind, self.random_start, self.mean, self.std,
                self.ignore_index)

    def __call__(self, model, x, y):
        return self.attack(model, x, y)

    def attack(self, model, x, y):
        check_model(model, "PGDAttack")
        crit = model.criterion if isinstance(model.criterion, nn.Module) else None
        skip = set(id(m) for m in crit.modules()) if crit is not None else set()
        if any(m.training for m in model.modules() if id(m) not in skip):
            raise RuntimeError("PGDAttack: every module of the model must be in eval mode (call model.eval())")
        check_inputs(model, x, y, self.kind, "PGDAttack")
        dev = next(model.parameters()).device
        if dev != x.device:
            raise RuntimeError("PGDAttack: the model is on %s, the input on %s" % (dev, x.device))
        st = self._graph(model, x, y)
        if st is not None:
            st.x.copy_(x, non_blocking=True)
            st.y.copy_(y, non_blocking=True)
            st.graph.replay()
            x_adv, self.losses = st.out.clone(), st.losses.clone()
            return x_adv
        SF.prepack(model)
        x_adv, self.losses = run(model, self, x, y)
        return x_adv

    def _graph(self, model, x, y):
        """The captured attack for this call's key (None: run eagerly)."""
        if not graphs.enabled():
            return None
        store = model.__dict__.setdefault("_sb_adv_graphs", {})
        ptrs = tuple(p.data_ptr() for p in model.parameters())
        key = (tuple(x.shape), tuple(y.shape), x.device.index, model.zoom_factor, precision.get_mode(), len(ptrs),
               hash(ptrs), self.key())
        st = store.get(key)
        if st is None:
            st = store[key] = _Graph()
        if st.failed:
            return None
        if st.graph is None:
            st.calls += 1
            if st.calls <= graphs.WARMUP_CALLS:
                return None
            if sum(1 for v in store.values() if v.graph is not None) >= graphs.MAX_GRAPHS:
                st.failed = True
                return None
            try:
                self._capture(st, model, x, y)
            except Exception as e:      # noqa: BLE001 - stay on the eager path (same kernels), say so once
                st.failed, st.graph = True, None
                if os.environ.get("SEMSEG_B200_GRAPH_DEBUG"):
                    raise
                warnings.warn("semseg_b200: CUDA-graph capture of the attack failed (%s: %s); continuing eagerly" %
                              (type(e).__name__, str(e).splitlines()[0][:200] if str(e) else ""))
                torch.cuda.synchronize()
                return None
        return st

    def _capture(self, st, model, x, y):
        st.x = x.detach().clone(memory_format=torch.contiguous_format)
        st.y = y.clone(memory_format=torch.contiguous_format)
        torch.cuda.synchronize()
        st.pool = torch.cuda.graph_pool_handle()
        st.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(st.graph, pool=st.pool, capture_error_mode="thread_local"):
            SF.prepack(model, force=True)        # every replay re-packs the slabs: in-place weight edits are seen
            st.out, st.losses = run(model, self, st.x, st.y)
        # the graph addresses the whole-model plan's slabs: keep them alive with it
        st.keep = model.__dict__.get("_sb_pack_plan")
        torch.cuda.synchronize()
