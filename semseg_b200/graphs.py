"""CUDA-graph execution of a whole training step (forward + backward) behind the unchanged module API.

A PSPNet50 step is ~700 kernel launches (PSPNet101: ~1300) enqueued from Python; at the reference's own per-GPU batch
(2 images, tool/train.py:154) the GPU finishes a step several times faster than the host can enqueue it, and under
DistributedDataParallel every host hiccup turns into a cross-rank wait inside the SyncBatchNorm exchanges. After a few
eager steps with the same input shape, `model(x, y)` in training mode therefore captures

    forward  : module input -> (argmax, main_loss, aux_loss)              [one graph]
    backward : d(main_loss, aux_loss)/d(parameters, and the input when it needs a gradient) via torch.autograd.grad
                                                                            [one graph]

into two CUDA graphs (the same kernels, in the same order, on the same stream) and replays them from ONE autograd node
whose inputs are the module's parameters: `loss.backward()`, DDP's gradient hooks, `optimizer.step()` and checkpoints see
exactly what they saw before. Captured along with the kernels: the one-launch weight re-pack, the BatchNorm
running-statistics updates, the SyncBN peer exchanges (their slots are baked in, the sequence number is a device-resident
step counter incremented inside the graph — csrc/bn.cu st_ll / ld_ll) and dropout's Philox state.

Limits (same as torch.cuda.make_graphed_callables): a second training forward before the backward of the first one
overwrites the first one's saved activations — gradient accumulation over several forwards needs SEMSEG_B200_GRAPH=0.
The NCCL fallback of the SyncBN exchange and criteria the fused tail does not implement (functional.fused_tail_supported)
are not captured (such models simply stay eager). With a teacher criterion the teacher forward (a mean teacher's
re-pack included), the draws, the strong view, the mixing and the extra student streams are captured with the step.
Set SEMSEG_B200_GRAPH=0 to disable; any capture failure also falls back to the eager path (same kernels) with a warning.
"""
import contextlib
import os
import warnings

import torch
import torch.distributed as dist

from . import losses, precision

WARMUP_CALLS = 3          # eager calls with an unchanged key before capturing
MAX_GRAPHS = 4            # captured input shapes per model (each keeps a private activation pool); others stay eager
_capturing = False
_boundary = None          # activation noted by the model during capture: where the backward is cut in two
_no_boundary = 0          # > 0 inside passes that are not the step's own forward (an adversarial attack's)


def enabled():
    return os.environ.get("SEMSEG_B200_GRAPH", "1") != "0"


def capturing():
    """True while a step is being captured: per-step device work that the eager path skips when nothing changed (weight
    re-pack, step-counter increment) must be issued unconditionally so that it becomes part of the graph."""
    return _capturing


def note_boundary(t):
    """Called by the model's forward while a step is being captured: `t` (the activation entering the dilated stages)
    cuts the backward pass into two graphs — everything after it (heads, layer4, layer3: 97 % of the parameters) and
    everything before it (stem, layer1, layer2). The first graph's parameter gradients are handed to autograd (and to
    DDP's bucket hooks: their all-reduce starts) while the second graph still computes, which restores the
    communication / computation overlap a single backward graph would lose."""
    global _boundary
    if _capturing and not _no_boundary and t.requires_grad:
        _boundary = t
    return t


@contextlib.contextmanager
def no_boundary():
    """Network passes run inside a captured step that are not the step's own forward (the K passes of an adversarial
    attack, losses.AdversarialLoss): their activations need a gradient too, but the step's backward must not be cut
    at them."""
    global _no_boundary
    _no_boundary += 1
    try:
        yield
    finally:
        _no_boundary -= 1


class _Step:
    __slots__ = ("key", "calls", "failed", "fwd", "bwd", "bwd2", "x", "y", "pred", "main", "aux", "g_main", "g_aux",
                 "grads", "grads2", "t_mid", "d_mid", "n_tail", "params", "pool", "keep", "launches", "dx_slot", "crit",
                 "last")

    def __init__(self, key):
        self.key, self.calls, self.failed, self.fwd, self.dx_slot = key, 0, False, None, False


def _set_grad_outputs(st, g_main, g_aux):
    if g_main is None:
        st.g_main.zero_()
    else:
        st.g_main.copy_(g_main)
    if g_aux is None:
        st.g_aux.zero_()
    else:
        st.g_aux.copy_(g_aux)


def _fresh(gs):
    """Per-step copies of the graph's static gradient tensors, as views of ONE new flat buffer filled by a fused
    multi-tensor copy: autograd's AccumulateGrad adopts such a view as `param.grad` without cloning it (it would clone
    the static tensors themselves, one small kernel per parameter, because this module keeps references to them)."""
    idx = [i for i, g in enumerate(gs) if g is not None]
    if not idx:
        return tuple(gs)
    src = [gs[i] for i in idx]
    offs, total = [], 0
    for g in src:
        offs.append(total)
        total += (g.numel() + 3) & ~3                      # 16-byte aligned sub-buffers
    flat = torch.empty((total,), dtype=src[0].dtype, device=src[0].device)
    views = [flat[o:o + g.numel()].view(g.shape) for o, g in zip(offs, src)]
    torch._foreach_copy_(views, src)
    out = [None] * len(gs)
    for i, v in zip(idx, views):
        out[i] = v
    return tuple(out)


class _Replay(torch.autograd.Function):
    """One autograd node for the whole step: forward replays the forward graph, backward replays the backward graph and
    returns the parameter gradients (static tensors of the graph's memory pool)."""

    @staticmethod
    def forward(ctx, st, x, y, *params):
        _replay_forward(st, x, y)
        ctx.st = st
        pred, main, aux = st.pred.detach(), st.main.detach(), st.aux.detach()
        ctx.mark_non_differentiable(pred)
        return pred, main, aux

    @staticmethod
    def backward(ctx, _g_pred, g_main, g_aux):
        st = ctx.st
        _set_grad_outputs(st, g_main, g_aux)
        st.bwd.replay()
        return _with_dx(st, _fresh(st.grads))


def _replay_forward(st, x, y):
    """The forward graph replayed on `x`, `y`. A teacher criterion's last_mix(), last_strong(), last_fp() and
    last_relation() are then the replayed step's: the records its captured forward wrote, static tensors of that step
    (each captured input shape has its own), are put back."""
    st.x.copy_(x, non_blocking=True)
    st.y.copy_(y, non_blocking=True)
    st.fwd.replay()
    if st.last:
        st.crit._last.update(st.last)


def _with_dx(st, gs):
    """(None, dx, None) + parameter gradients from the gradients `gs` a backward graph produced, the input gradient last
    when the step was captured with an input that needs one."""
    if st.dx_slot:
        return (None, gs[-1], None) + gs[:-1]
    return (None, None, None) + gs


class _ReplayHead(torch.autograd.Function):
    """Two-segment form, first node: replays the whole forward graph, returns the boundary activation; its backward
    replays the SECOND backward graph (stem, layer1, layer2) from the boundary gradient the tail node left in place."""

    @staticmethod
    def forward(ctx, st, x, y, *params_head):
        _replay_forward(st, x, y)
        ctx.st = st
        return st.t_mid.detach()

    @staticmethod
    def backward(ctx, d_mid):
        st = ctx.st
        if d_mid.data_ptr() != st.d_mid.data_ptr():
            st.d_mid.copy_(d_mid)
        st.bwd2.replay()
        return _with_dx(st, _fresh(st.grads2))


class _ReplayTail(torch.autograd.Function):
    """Two-segment form, second node: hands out the static outputs; its backward replays the FIRST backward graph
    (heads, layer4, layer3) and returns the boundary gradient plus those parameters' gradients."""

    @staticmethod
    def forward(ctx, st, t_mid, *params_tail):
        ctx.st = st
        pred, main, aux = st.pred.detach(), st.main.detach(), st.aux.detach()
        ctx.mark_non_differentiable(pred)
        return pred, main, aux

    @staticmethod
    def backward(ctx, _g_pred, g_main, g_aux):
        st = ctx.st
        _set_grad_outputs(st, g_main, g_aux)
        st.bwd.replay()
        return (None, st.d_mid) + _fresh(st.grads)


def _sync_bn_ready(model):
    """(ok, exchange): multi-rank SyncBatchNorm is only captured with the NVLink peer exchange (no NCCL call inside)."""
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return True
    if not any(isinstance(m, torch.nn.SyncBatchNorm) for m in model.modules()):
        return True
    from . import p2p
    return p2p.get_exchange(dist.group.WORLD) is not None


def _capture(model, impl, st, x, y):
    global _capturing
    from . import _lib
    # Parameter proxies: the backward graph is captured with torch.autograd.grad w.r.t. FRESH leaves that alias the
    # parameters' storage. The real parameters' AccumulateGrad nodes may be kept alive from earlier eager iterations (by a
    # loss tensor, or by DistributedDataParallel, which stashes them at construction) and are bound to the stream they
    # were created on; letting the capture deliver gradients to them would make that (legacy) stream depend on the
    # capturing stream, which CUDA forbids (cudaErrorStreamCaptureImplicit).
    slots, seen = [], set()
    for mod in model.modules():
        for name, prm in mod._parameters.items():
            if prm is not None and prm.requires_grad and id(prm) not in seen:
                seen.add(id(prm))
                slots.append((mod, name, prm))
    st.params = [prm for _, _, prm in slots]
    st.x, st.y = torch.empty_like(x), torch.empty_like(y)
    st.x.copy_(x.detach())
    st.y.copy_(y)
    torch.cuda.synchronize()
    st.pool = torch.cuda.graph_pool_handle()
    st.fwd, st.bwd, st.bwd2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), None
    crit = getattr(model, "criterion", None)
    last = getattr(crit, "_last", {})
    # the records' identities only: holding the eager step's records would keep their tensors alive through the capture
    # (a forward writes each record as a new dict while the old one still exists, so the ids cannot repeat)
    before = {k: id(v) for k, v in last.items()}
    l0 = _lib.launch_count()
    global _boundary
    _capturing, _boundary = True, None
    proxies = []
    # an input that needs a gradient is captured as a leaf aliasing st.x; its gradient is the last one the backward
    # graph (the second one in the two-segment form) produces
    st.dx_slot = x.requires_grad
    x_in = st.x.detach().requires_grad_(True) if st.dx_slot else st.x
    x_leaf = [x_in] if st.dx_slot else []
    try:
        for mod, name, prm in slots:
            q = prm.detach().requires_grad_(True)      # same storage, new leaf
            mod._parameters[name] = q
            proxies.append(q)
        with torch.cuda.graph(st.fwd, pool=st.pool, capture_error_mode="thread_local"):
            with torch.enable_grad():
                st.pred, st.main, st.aux = impl(x_in, st.y)
        st.g_main, st.g_aux = torch.ones_like(st.main), torch.ones_like(st.aux)
        t_mid = _boundary
        head_ids = set()
        if t_mid is not None and os.environ.get("SEMSEG_B200_GRAPH_SEGMENTS", "2") != "1":
            for name in getattr(model, "_sb_head_modules", ()):
                # the proxies only: a frozen parameter has none and must not be counted into the head
                head_ids.update(id(q) for q in getattr(model, name).parameters() if q.requires_grad)
        if head_ids:
            # parameters reordered: head (before the boundary) first, tail after
            order = [k for k, q in enumerate(proxies) if id(q) in head_ids] + \
                    [k for k, q in enumerate(proxies) if id(q) not in head_ids]
            n_head = len(head_ids)
            st.params = [st.params[k] for k in order]
            prox_head = [proxies[k] for k in order[:n_head]]
            prox_tail = [proxies[k] for k in order[n_head:]]
            with torch.cuda.graph(st.bwd, pool=st.pool, capture_error_mode="thread_local"):
                gs = torch.autograd.grad((st.main, st.aux), [t_mid] + prox_tail, (st.g_main, st.g_aux), allow_unused=True)
            st.d_mid, st.grads = gs[0], gs[1:]
            st.bwd2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(st.bwd2, pool=st.pool, capture_error_mode="thread_local"):
                st.grads2 = torch.autograd.grad((t_mid,), prox_head + x_leaf, (st.d_mid,), allow_unused=True)
            st.t_mid, st.n_tail = t_mid.detach(), len(prox_tail)
        else:
            with torch.cuda.graph(st.bwd, pool=st.pool, capture_error_mode="thread_local"):
                st.grads = torch.autograd.grad((st.main, st.aux), proxies + x_leaf, (st.g_main, st.g_aux),
                                               allow_unused=True)
    finally:
        _capturing, _boundary = False, None
        for mod, name, prm in slots:
            mod._parameters[name] = prm
    st.launches = _lib.launch_count() - l0          # native kernels per replayed step (forward + backward graphs)
    # the last-step records the captured forward wrote: static tensors of the graph's pool, refreshed by every replay
    st.crit, st.last = crit, {k: v for k, v in last.items() if before.get(k) != id(v)}
    # drop the autograd graph built during capture; the static outputs live on in the graphs' private memory pool
    st.pred, st.main, st.aux = st.pred.detach(), st.main.detach(), st.aux.detach()
    del proxies, x_in, x_leaf
    # the graphs reference the persistent weight slabs: keep their owner alive as long as the graphs (a distillation
    # teacher's slabs are its convs' own packs, filled by the eager warm-up calls; the teacher is kept with them)
    st.keep = model.__dict__.get("_sb_pack_plan")
    teacher = getattr(crit, "teacher", None)      # a distillation or pseudo-label criterion's
    if teacher is not None:
        # a mean teacher's slabs are its whole-model plan's, re-packed inside the captured step
        st.keep = (st.keep, teacher, teacher.__dict__.get("_sb_pack_plan"),
                   [m.__dict__.get("_sb_conv_plan") for m in teacher.modules()])
    torch.cuda.synchronize()


def train_step(model, impl, x, y):
    """Run `impl(x, y)` (the module's eager training forward, returning (pred, main_loss, aux_loss)) through the captured
    graphs when possible; returns None when the caller should run the eager path itself."""
    if not (enabled() and x.is_cuda and y is not None and torch.is_grad_enabled()):
        return None
    if getattr(model, "_is_replica", False):
        return None                           # nn.DataParallel replica (tool/train.py:159): rebuilt every call, threads
    steps = model.__dict__.setdefault("_sb_graph_steps", {})
    # the graphs address the parameters' storage directly: a parameter that was re-allocated since the capture
    # (model.to(...), a swapped nn.Parameter) must not hit a stale graph, so the storage addresses are part of the key
    ptrs = tuple(p.data_ptr() for p in model.parameters() if p.requires_grad)
    # BatchNorm modes (batch statistics or frozen) decide which kernels the step runs: freezing or unfreezing a layer
    # after a capture must capture again, not replay the old step
    bn_modes = tuple(m.training for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm))
    # likewise the heads' Dropout2d modes: a dropout switched to eval mode (adapt.Tent) runs no mask kernel
    drop_modes = tuple(m.training for m in model.modules() if isinstance(m, torch.nn.Dropout2d))
    # an input that needs a gradient runs other kernels (the phase-form stem conv, its dgrad): a capture of its own
    # the criterion's options are launch arguments baked into the graphs: each criterion declares its own
    crit_key = losses.graph_key(getattr(model, "criterion", None))
    key = (tuple(x.shape), x.dtype, tuple(y.shape), y.dtype, x.device.index, precision.get_mode(), len(ptrs), hash(ptrs),
           dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1, bn_modes, drop_modes,
           x.requires_grad, crit_key)
    if x.requires_grad and x.dtype != torch.float32:
        return None                           # the captured input gradient is handed out in the parameters' fp32 buffer
    st = steps.get(key)
    if st is None:
        st = steps[key] = _Step(key)
    if st.failed:
        return None
    if st.fwd is None:
        st.calls += 1
        if st.calls <= WARMUP_CALLS:
            return None                       # eager warm-up (also creates the weight-pack plan, the peer exchange, ...)
        if not _sync_bn_ready(model) or sum(1 for v in steps.values() if v.fwd is not None) >= MAX_GRAPHS:
            st.failed = True                  # NCCL-path SyncBN, or too many input shapes already hold a memory pool
            return None
        try:
            _capture(model, impl, st, x, y)
        except Exception as e:      # noqa: BLE001 - stay on the eager path (same kernels), say so once
            st.failed, st.fwd = True, None
            if os.environ.get("SEMSEG_B200_GRAPH_DEBUG"):
                raise
            warnings.warn("semseg_b200: CUDA-graph capture of the training step failed (%s: %s); continuing eagerly" %
                          (type(e).__name__, str(e).splitlines()[0][:200] if str(e) else ""))
            torch.cuda.synchronize()
            return None
    if st.bwd2 is not None:
        n_head = len(st.params) - st.n_tail
        t_mid = _ReplayHead.apply(st, x, y, *st.params[:n_head])
        return _ReplayTail.apply(st, t_mid, *st.params[n_head:])
    return _Replay.apply(st, x, y, *st.params)


def launches_per_step(model):
    """Native kernel launches inside one replayed step of `model` (0 when no step has been captured)."""
    steps = model.__dict__.get("_sb_graph_steps", {})
    return max([getattr(s, "launches", 0) or 0 for s in steps.values() if s.fwd is not None] + [0])
