"""FusedSGD: torch.optim.SGD's update (momentum, dampening, weight decay, nesterov — the optimizer of tool/train.py:140)
for every parameter tensor in ONE kernel launch (csrc/sgd.cu) instead of ~33 foreach launches (SURVEY.md §8 f4).

Drop-in for `torch.optim.SGD(params_list, lr=..., momentum=..., weight_decay=...)` at tool/train.py:140 (same constructor
arguments, same param_groups — the trainer's per-iteration `optimizer.param_groups[i]['lr'] = ...` keeps working, and
momentum, dampening, weight decay and nesterov are honoured per group — and the same state_dict layout: state[p] =
{'momentum_buffer': tensor} once p has taken a step with a gradient under a non-zero momentum, which starts the buffer
from that gradient, so checkpoints move between the two classes).
fp32 CUDA parameters only; the conv operand slabs are refreshed by the model's own one-launch re-pack at the next forward
(semseg_b200.functional.prepack), which notices the update through `bump_versions`.
"""
import ctypes

import torch

from . import _lib
from .ops import _stream


class FusedSGD(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False):
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov)
        super().__init__(params, defaults)
        if len(self.param_groups) > 16:
            raise ValueError("FusedSGD supports up to 16 parameter groups")
        self._table = None

    def _buffer(self, p):
        st = self.state.get(p)
        return st.get("momentum_buffer") if st else None

    def _build(self, plist, first, key, device):
        chunk = int(_lib.load().semseg_sgd_chunk_elems())
        items = (_lib.SgdItem * len(plist))()
        c0 = 0
        for k, (gi, p) in enumerate(plist):
            it = items[k]
            it.w, it.buf, it.n = p.data_ptr(), key[k][1], p.numel()
            it.group, it.chunk0, it.first = gi, c0, int(first[k])
            c0 += (p.numel() + chunk - 1) // chunk
        dev = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).to(device)
        dev_ptrs = torch.zeros((len(plist),), dtype=torch.int64, device=device)
        return dict(items=dev, n=len(plist), chunks=c0, dev_ptrs=dev_ptrs, last_ptrs=None, key=key)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        plist = [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"]]
        if not plist:
            return loss
        for _, p in plist:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise _lib.SemsegError("FusedSGD needs contiguous fp32 CUDA parameters (no CPU fallback)")
        h = _lib.SgdHyper()
        for gi, g in enumerate(self.param_groups):
            h.lr[gi], h.momentum[gi] = float(g["lr"]), float(g["momentum"])
            h.weight_decay[gi], h.dampening[gi] = float(g["weight_decay"]), float(g["dampening"])
            h.nesterov |= int(bool(g["nesterov"])) << gi
        ptrs, first, key = [], [], []
        for gi, p in plist:
            g = p.grad
            if g is not None and not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous()):
                g = p.grad = g.contiguous().float()
            ptrs.append(g.data_ptr() if g is not None else 0)
            b = self._buffer(p)
            # like torch.optim.SGD, a parameter gets its momentum buffer on its first step with a gradient under a
            # non-zero momentum (the kernel's fp32 value), and the buffer starts from that gradient
            first.append(b is None and g is not None and h.momentum[gi] != 0)
            if first[-1]:
                b = self.state[p]["momentum_buffer"] = torch.empty_like(p, memory_format=torch.preserve_format)
            key.append((p.data_ptr(), b.data_ptr() if b is not None else 0))
        t = self._table
        if t is None or t["key"] != key or any(first):
            t = self._table = self._build(plist, first, key, plist[0][1].device)
        if ptrs != t["last_ptrs"]:
            # Upload the gradient pointer table only when it changed, from a FRESH pinned buffer each time: the copy is
            # asynchronous, so a reused staging buffer could be overwritten by the next step's pointers before this
            # step's copy has run (torch's pinned-memory allocator keeps a freed block alive until its copy completed).
            t["dev_ptrs"].copy_(torch.tensor(ptrs, dtype=torch.int64).pin_memory(), non_blocking=True)
            t["last_ptrs"] = ptrs
        lib = _lib.load()
        _lib.check(lib.semseg_sgd_multi(ctypes.c_void_p(t["items"].data_ptr()), ctypes.c_void_p(t["dev_ptrs"].data_ptr()),
                                        t["n"], t["chunks"], ctypes.byref(h), _stream()), "semseg_sgd_multi")
        # the raw update does not touch the autograd version counters; the conv operand caches are keyed on them
        _bump_versions([p for _, p in plist if p.grad is not None])
        if any(first):
            self._table = None       # rebuild once with these first flags cleared
        return loss


def ema_table(pairs):
    """(device item table, items, chunks) of semseg_ema_multi for [(shadow, source)] pairs of non-empty contiguous CUDA
    tensors, fp32 (averaged) or int64 (copied)."""
    chunk = int(_lib.load().semseg_sgd_chunk_elems())
    items = (_lib.EmaItem * len(pairs))()
    c0 = 0
    for it, (e, w) in zip(items, pairs):
        it.shadow, it.source, it.n, it.chunk0 = e.data_ptr(), w.data_ptr(), e.numel(), c0
        it.kind = _lib.EMA_LERP_F32 if e.dtype == torch.float32 else _lib.EMA_COPY_I64
        c0 += (e.numel() + chunk - 1) // chunk
    return torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).to(pairs[0][0].device), len(pairs), c0


def _bump_versions(ts):
    """Tell the operand-slab caches (keyed on autograd version counters) that a raw kernel wrote `ts`."""
    bump = getattr(torch._C._autograd, "_unsafe_set_version_counter", None)
    if bump is not None:
        bump(ts, [t._version + 1 for t in ts])
    else:
        torch._foreach_add_(ts, 0)         # older torch: an in-place no-op bumps the counters


class ModelEMA:
    """An exponential moving average of a network's weights: the mean teacher of Mean Teacher / CutMix-Seg / UniMatch,
    and the copy many users evaluate and checkpoint.

    ModelEMA(model, decay=0.999): `model` is a PSPNet or PSANet of this package, bare or wrapped in
    DistributedDataParallel / nn.DataParallel (its `.module` is taken). `ema.module` is a deep copy of the network in
    eval mode, every parameter with requires_grad=False, sharing no tensor with the student, with a plain
    nn.CrossEntropyLoss(ignore_index) as its criterion (a losses.DistillationLoss that holds `ema.module` is never
    copied into it), and the student's conv caches and captured steps left behind. It is not a submodule of the student:
    hand it to losses.DistillationLoss / losses.PseudoLabelLoss as the teacher, evaluate it, or save it.

    ema.update(model): every floating-point parameter and buffer of the shadow (conv weights and biases, BatchNorm gamma,
    beta, running mean and variance) becomes e + (1 - decay) (w - e), in torch.lerp's form (bit-equal to
    torch._foreach_lerp_(shadow, source, 1 - decay)); integer buffers (num_batches_tracked) are copied. Tensors pair by
    named_parameters() / named_buffers() (the criterion's own buffers excepted); a name, shape or dtype mismatch raises.
    One kernel launch for the whole model (csrc/sgd.cu ema_multi_kernel) on the current stream; the shadow's version
    counters are bumped, so its next eager forward re-packs its operand slabs. Call it after optimizer.step(), on the
    same stream: the next step's teacher forward then reads the updated shadow, captured or not.

    Like an optimizer, it holds the tensors it paired: moving them (model.to(...), load_state_dict into new storage)
    is noticed and the pairing is rebuilt, but a Parameter object replaced by another one needs a new ModelEMA.

    `decay` is read at every call: a ramp such as Tarvainen's min(decay, 1 - 1/(t+1)) is `ema.decay = ...` before each
    update, as the trainer rewrites learning rates. fp32 / int64 CUDA tensors only: there is no CPU fallback.

    Under DistributedDataParallel each rank updates its own shadow from the same all-reduced parameters; with plain
    (non-Sync) BatchNorm the shadows' running statistics differ per rank, as the students' do."""

    def __init__(self, model, decay=0.999):
        import copy
        from torch import nn
        from .pspnet import PSPNet
        from .psanet import PSANet
        net = self._unwrap(model)
        if not isinstance(net, (PSPNet, PSANet)):
            raise TypeError("ModelEMA: model must be a semseg_b200 PSPNet or PSANet (or DDP / DataParallel of one), got %s"
                            % type(net).__name__)
        self.decay = decay
        self._check_decay()
        crit = getattr(net, "criterion", None)
        # the copy skips the student's criterion (a plain cross-entropy takes its place) and its per-module caches: conv
        # operand slabs, pack plans and captured graphs belong to the student's tensors
        memo = {}
        if crit is not None:
            memo[id(crit)] = nn.CrossEntropyLoss(ignore_index=getattr(crit, "ignore_index", 255))
        for m in net.modules():
            for k, v in m.__dict__.items():
                # caches are objects of their own; a shared constant (True, an empty tuple) must not enter the memo
                if k.startswith("_sb_") and not isinstance(v, (bool, int, float, str, type(None))) and v != ():
                    memo[id(v)] = None
        shadow = copy.deepcopy(net, memo)
        for m in shadow.modules():
            for k in [k for k in m.__dict__ if k.startswith("_sb_")]:
                del m.__dict__[k]
        shadow.eval()
        for p in shadow.parameters():
            p.requires_grad_(False)
        shadow._sb_ema_shadow = True     # graphs / losses: a teacher that changes every step (see losses._TeacherLoss)
        self.module = shadow
        self._table = None

    @staticmethod
    def _unwrap(model):
        from torch import nn
        if isinstance(model, (nn.parallel.DistributedDataParallel, nn.DataParallel)):
            return model.module
        return model

    def _check_decay(self):
        d = self.decay
        if isinstance(d, bool) or not isinstance(d, (int, float)):
            raise TypeError("ModelEMA: decay must be a number, got %r" % (d,))
        if not 0.0 <= float(d) <= 1.0:
            raise ValueError("ModelEMA: decay must lie in [0, 1], got %r" % (d,))

    @staticmethod
    def _pairs(shadow, net):
        """[(shadow tensor, source tensor)] by name: parameters, then buffers (the criterion's excepted)."""
        out = []
        for what in ("named_parameters", "named_buffers"):
            a = [(k, t) for k, t in getattr(shadow, what)() if not k.startswith("criterion.")]
            b = [(k, t) for k, t in getattr(net, what)() if not k.startswith("criterion.")]
            if [k for k, _ in a] != [k for k, _ in b]:
                raise ValueError("ModelEMA: the model's %s differ from the shadow's: %s" % (
                    what[6:], sorted(set(k for k, _ in a) ^ set(k for k, _ in b))[:8]))
            for (k, e), (_, w) in zip(a, b):
                if e.shape != w.shape or e.dtype != w.dtype:
                    raise ValueError("ModelEMA: %s is %s %s in the model and %s %s in the shadow" %
                                     (k, w.dtype, tuple(w.shape), e.dtype, tuple(e.shape)))
                if e.dtype not in (torch.float32, torch.int64):
                    raise TypeError("ModelEMA: %s is %s; fp32 and int64 tensors only" % (k, e.dtype))
                out.append((k, e, w))
        for k, e, w in out:
            if not (e.is_cuda and w.is_cuda and e.device == w.device and e.is_contiguous() and w.is_contiguous()):
                raise _lib.SemsegError("ModelEMA: %s must be contiguous and on one CUDA device in the model and the "
                                       "shadow (no CPU fallback)" % k)
        return [(e, w) for _, e, w in out]

    @torch.no_grad()
    def update(self, model):
        """shadow <- lerp(shadow, model, 1 - decay) over every floating-point tensor, integer buffers copied; one launch."""
        from . import ops
        self._check_decay()
        net = self._unwrap(model)
        # the pairing is validated when the table is built; later calls only check that the same model comes and that
        # none of the held tensors moved (walking both module trees every step would cost milliseconds of host time)
        t = self._table
        if t is None or t[0] is not net or t[1] != tuple(x.data_ptr() for x in t[3]):
            pairs = [(e, w) for e, w in self._pairs(self.module, net) if e.numel() > 0]
            held = [x for pair in pairs for x in pair]
            t = self._table = (net, tuple(x.data_ptr() for x in held), ema_table(pairs), held, [e for e, _ in pairs])
        ops.ema_multi(*t[2], float(self.decay))
        _bump_versions(t[4])

    def state_dict(self):
        """The shadow's state_dict plus the decay: a checkpoint of the EMA."""
        return {"module": self.module.state_dict(), "decay": self.decay}

    def load_state_dict(self, state):
        """Restore a state_dict() (in place: a captured step that reads the shadow keeps its addresses)."""
        self.module.load_state_dict(state["module"])
        self.decay = state["decay"]
        self._check_decay()
