"""Autograd functions of the hot path, operating on NHWC bf16 activations.

Each Function is a thin scheduler of C-ABI kernel launches (semseg_b200/ops.py); the fp32 master weights
stay ordinary nn.Parameters (OIHW) so torch.optim.SGD, DistributedDataParallel and state_dict see exactly
what the reference's modules expose (tool/train.py:134-140,157).

conv + BatchNorm(train) + ReLU (+ residual) is three launches forward:
    conv_fprop (raw bf16 + per-tile partial statistics)  ->  bn_merge/finalize  ->  bn_apply
because training-mode BN needs the batch (and, under SyncBN, cross-rank) statistics of the complete conv
output before anything can be normalised (model/resnet.py:77-83). In eval mode the BN folds into the conv
epilogue and the whole thing is a single kernel.

Frozen BatchNorm — a BN layer in eval mode inside a network that trains (`model.train()`, then `.eval()` on the BN
layers) — normalises with its running statistics, leaves them untouched and still passes gradients: its forward is the
eval kernel (or conv + apply when gamma needs a gradient) and its backward one pass (ops.bn_bwd_frozen). `_bn_mode` is
the one place that decides which of the three forms a stage takes.
"""
import contextlib
import functools
import threading

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

from . import losses
from . import ops
from . import p2p
from . import precision
from .dist_utils import gather_rank_stats
from .ops import EPI_RAW, EPI_AFFINE, EPI_F32


# ------------------------------------------------------------------------------------------------ helpers
def packed(conv, need_dgrad=True, split=False):
    """bf16 operand slabs of conv.weight (hi + lo slabs when split; also the patch slab of a stem conv), re-packed only
    when the parameter changed (optimizer step / load). The cache key is (parameter version, storage pointer): in-place
    edits through `.data` do not bump the version — call `invalidate_packs(model)` after such an edit. A miss refreshes
    the conv's own one-conv plan, which is rebuilt only for a new storage, storage form or first need of dgrad slabs."""
    w = conv.weight
    key = (w._version, w.data_ptr(), need_dgrad, split)
    cache = conv.__dict__.get("_sb_pack")
    if cache is not None and cache[0] == key:
        return cache[1]
    if cache is not None and cache[0][:2] == key[:2] and cache[0][3] == split and cache[0][2]:
        return cache[1]                       # a pack with dgrad slabs also serves a forward-only request
    plan = conv.__dict__.get("_sb_conv_plan")
    if plan is None or not plan.valid_for([w], split) or (need_dgrad and plan.packs[0].wd is None):
        wc = w.detach()
        plan = ops.WeightPackPlan([wc if wc.is_contiguous() else wc.contiguous()], split, dgrad=need_dgrad,
                                  patches=[_is_patch_conv(conv)])
        conv.__dict__["_sb_conv_plan"] = plan
    plan.refresh()
    pw = plan.packs[0]
    conv.__dict__["_sb_pack"] = (key[:2] + (pw.wd is not None, split), pw)
    return pw


def invalidate_packs(model):
    """Forget every cached operand slab of `model` (needed after weights were modified through `.data`, which does not
    bump the version counter the cache is keyed on)."""
    for m in model.modules():
        m.__dict__.pop("_sb_pack", None)
    model.__dict__.pop("_sb_pack_plan", None)


def _is_patch_conv(conv):
    """The 3-channel stride-2 stem conv (model/resnet.py:106-108), which can run as a 1x1 conv over input patches."""
    return (conv.kernel_size == (3, 3) and conv.stride == (2, 2) and conv.dilation == (1, 1) and conv.padding == (1, 1)
            and conv.in_channels <= 3 and conv.groups == 1)


def prepack(model, force=False, dgrad=True):
    """Refresh the operand slabs of every native conv of `model` in one launch when its weights changed (call at the top
    of a training forward; force=True while the step is being captured into a CUDA graph, so that the re-pack is part
    of every replay). Convs keep working without it: `packed` re-packs each conv through its own one-conv plan.
    dgrad=False packs the forward slabs only (a network that runs forward only, such as a mean teacher)."""
    convs = [m for m in model.modules() if isinstance(m, nn.Conv2d) and m.weight.is_cuda and
             m.weight.dtype == torch.float32 and m.weight.is_contiguous() and m.kernel_size[0] == m.kernel_size[1] and
             m.kernel_size[0] * m.kernel_size[1] <= ops.MAX_TAPS]
    if not convs:
        return
    split = precision.split_enabled()
    keys = [(c.weight._version, c.weight.data_ptr(), dgrad, split) for c in convs]
    if not force and all(c.__dict__.get("_sb_pack", (None,))[0] == k for c, k in zip(convs, keys)):
        return                                            # nothing changed since the last pack
    plan = model.__dict__.get("_sb_pack_plan")
    weights = [c.weight.detach() for c in convs]
    if plan is None or not plan.valid_for(weights, split) or (dgrad and plan.packs[0].wd is None):
        plan = ops.WeightPackPlan(weights, split, dgrad=dgrad, patches=[_is_patch_conv(c) for c in convs])
        model.__dict__["_sb_pack_plan"] = plan
    plan.refresh()
    for c, k, pw in zip(convs, keys, plan.packs):
        c.__dict__["_sb_pack"] = (k, pw)


# Whether the network being run is in training mode, per thread (nn.DataParallel replicas run in threads,
# tool/train.py:159). Set by the forward of PSPNet / PSANet and of the modules that can be run on their own.
_net = threading.local()


@contextlib.contextmanager
def network_mode(training, input_grad=True):
    """Runs the enclosed forward as part of a network in training mode (True) or not (False) on this thread.
    `input_grad`: whether the network's input needs a gradient (see _bn_mode)."""
    prev = getattr(_net, "training", False), getattr(_net, "input_grad", True)
    _net.training, _net.input_grad = bool(training), bool(input_grad)
    try:
        yield
    finally:
        _net.training, _net.input_grad = prev


@contextlib.contextmanager
def fp8_plan(plan):
    """Runs the enclosed eval forward with `plan` (semseg_b200/fp8.py) consulted by every eval-mode conv + BatchNorm stage
    on this thread: it runs the stages it covers in FP8 (or, while calibrating, records their input range) and returns
    None for the others, which take the bf16 path."""
    prev = getattr(_net, "fp8", None)
    _net.fp8 = plan
    try:
        yield
    finally:
        _net.fp8 = prev


def network_forward(fn):
    """Decorator of a module's forward(x, ...): the module is the network being run, in its own training mode."""
    @functools.wraps(fn)
    def forward(self, *args, **kwargs):
        x = args[0] if args else kwargs.get("x")
        with network_mode(self.training, torch.is_tensor(x) and x.requires_grad):
            return fn(self, *args, **kwargs)
    return forward


def _needs_grad(ts):
    return any(t is not None and t.requires_grad for t in ts)


def _bn_mode(bn, acts, params=()):
    """How a conv + `bn` stage runs, given the tensors its gradients would flow to (None entries allowed): its activation
    inputs `acts` (x, the residual) and its parameters `params`:
      "batch"  : batch statistics (BN in training mode, or without running statistics), running statistics updated;
      "frozen" : running statistics, differentiable — BN in eval mode, autograd enabled, and either the network in
                 training mode with some input or parameter needing a gradient, or the network in eval mode, its input
                 needing a gradient and an activation input of the stage needing one (input gradients of an eval
                 network: saliency, adversarial attacks);
      "eval"   : the folded single kernel, detached (model.eval() on an input that needs no gradient — the reference's
                 validate(), where activations may still need a gradient through a parameter such as PSA's attention
                 conv — torch.no_grad(), or nothing needs a gradient)."""
    if bn.training or bn.running_mean is None:
        return "batch"
    if torch.is_grad_enabled():
        if getattr(_net, "training", False):
            if _needs_grad(acts) or _needs_grad(params):
                return "frozen"
        elif getattr(_net, "input_grad", True) and _needs_grad(acts):
            return "frozen"
    return "eval"


def _sync_group(bn):
    """Process group when `bn` is a SyncBatchNorm that must synchronise, else None."""
    if isinstance(bn, nn.SyncBatchNorm) and dist.is_available() and dist.is_initialized():
        pg = bn.process_group if bn.process_group is not None else dist.group.WORLD
        if dist.get_world_size(pg) > 1:
            return pg
    return None


def _bn_momentum(bn):
    # nn.BatchNorm semantics: momentum None = cumulative moving average
    if bn.momentum is None:
        return 1.0 / float(bn.num_batches_tracked.item() + 1)
    return bn.momentum


def _batch_stats(sp, bn, pg):
    """Per-CTA statistics partials of the conv output -> (mean_invstd, scale_shift) of the batch, over every rank of
    `pg` under SyncBN. Updates the running statistics and num_batches_tracked like nn.BatchNorm in training mode."""
    track = bn.track_running_stats and bn.running_mean is not None
    mom = _bn_momentum(bn) if track else 0.0
    rm, rv = (bn.running_mean, bn.running_var) if track else (None, None)
    px = p2p.get_exchange(pg) if pg is not None else None
    if pg is None or (px is not None and 3 * sp.shape[-1] <= p2p.SLOT_FLOATS):
        # merge the per-CTA partials and finalise in one launch; under SyncBN the statistics are exchanged over NVLink
        # peer memory inside that kernel (no NCCL call)
        mi, ss = ops.bn_finalize_partials(sp, bn.weight, bn.bias, bn.eps, mom, rm, rv, px=px)
    else:
        # SyncBN over NCCL: every rank's local (mean, M2, count), then one finalise
        mi, ss = ops.bn_finalize(gather_rank_stats(ops.bn_merge_partials(sp), pg), bn.weight, bn.bias, bn.eps, mom,
                                 rm, rv)
    if track and bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
    return mi, ss


def _bn_backward(pg, dy, y, raw, mi, gamma, relu, want_dres, ss=None):
    """Shared BN(+ReLU) backward: returns (d_raw, dres, dgamma, dbeta). The ReLU mask comes from the saved output `y`,
    or — when `y` is None and `ss` (scale/shift) is given, i.e. no residual — is recomputed from `raw` (saves one
    tensor read in each of the two passes)."""
    n, h, w, c = raw.shape[-4:]
    if not dy.is_contiguous():
        dy = dy.contiguous()
    px = p2p.get_exchange(pg) if pg is not None else None
    if pg is None or (px is not None and 2 * c <= p2p.SLOT_FLOATS):
        # under SyncBN the cross-rank sum is taken over NVLink peer memory inside the reduction kernel (no NCCL call)
        local, sums = ops.bn_bwd_reduce(dy, y if relu else None, raw, mi, relu, ss if y is None else None, px=px)
    else:
        local, sums = ops.bn_bwd_reduce(dy, y if relu else None, raw, mi, relu, ss if y is None else None)
        local = local.clone()                   # local sums feed dgamma/dbeta (DDP averages them)
        dist.all_reduce(sums, group=pg)
    dbeta, dgamma = local[0], local[1]
    # under SyncBN the per-channel sample count is the one the forward exchange measured (mi row 2): exact also when the
    # ranks hold different numbers of pixels, like torch.nn.SyncBatchNorm's gathered counts
    count = float(n * h * w) if pg is None else 0.0
    d_raw, dres, _ = ops.bn_bwd_apply(dy, y if relu else None, raw, mi, gamma, sums, count, relu, want_dres=want_dres,
                                      scale_shift=ss if y is None else None)
    return d_raw, dres, dgamma, dbeta


# ------------------------------------------------------------------------------------------------ conv+bn+act
class _ConvForm:
    """How the conv of one stage runs on the stride-1 tensor-core kernel, chosen once from (conv, x, input_needs_grad,
    BatchNorm mode). It owns the input transform, the taps and the weight slab, and the fprop / dgrad / wgrad of its form:
      "direct" : stride 1, any dilation.
      "phases" : stride 2 (stem conv1, layer2.0 conv2 / downsample — model/resnet.py:108,130-137) through a 2x2 phase
                 decomposition of the input (space_to_phases): tap (r, s) reads phase ((r+1)&1, (s+1)&1) shifted by
                 -1 or 0; dgrad is one small conv per phase, wgrad reads the phases.
      "patches": the 3-channel stride-2 stem conv on an input that needs no gradient: one 1x1 conv over 27-value input
                 patches (ops.im2col3x3s2) instead of 9 taps of a 3(->64)-channel K block. Eval mode always takes the
                 phase form: the patch form sums in another order, so its output bits differ.
    The stem conv's input gradient, whichever form ran forward, is one CUDA-core kernel over the patch slab
    (ops.stem_dgrad3x3s2), written as fp32 NCHW."""
    __slots__ = ("kind", "pw", "wf", "xin", "taps", "img_add", "out_nhw", "in_shape", "stem")

    def __init__(self, conv, x, input_needs_grad, mode):
        split = ops.is_split(x)
        self.pw = packed(conv, need_dgrad=mode != "eval", split=split)
        self.wf, self.img_add, self.out_nhw = self.pw.wf, None, None
        self.in_shape = tuple(x.shape[-4:])
        self.stem = _is_patch_conv(conv) and conv.out_channels == 64
        n, h, w, _ = self.in_shape
        k = conv.kernel_size[0]
        if conv.stride[0] == 1:
            self.kind, self.xin, self.taps = "direct", x, ops.conv_taps(k, conv.dilation[0])
        elif mode != "eval" and not input_needs_grad and _is_patch_conv(conv) and x.shape[-1] >= 4:
            self.kind, self.xin = "patches", ops.im2col3x3s2(x, conv.in_channels)
            self.taps, self.wf = ops.conv_taps(1, 1), self.pw.wp
        else:
            self.kind, self.xin = "phases", ops.space_to_phases(x)          # [4N, Hh, Wh, C]
            t2 = ops.conv_taps_s2(k, n)
            self.taps, self.img_add = [t[:3] for t in t2], [t[3] for t in t2]
            self.out_nhw = (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1)

    def fprop(self, **kw):
        """The conv on the transformed input; `kw` are ops.conv_fprop's epilogue / statistics / output options."""
        return ops.conv_fprop(self.xin, self.wf, self.pw.cout, self.taps, img_add=self.img_add, out_nhw=self.out_nhw,
                              **kw)

    def dgrad(self, d_raw, dx_add=None, nchw=False):
        """Input gradient from the conv output's gradient `d_raw`. `dx_add` (same shape as dx) is summed into dx — in
        the dgrad epilogue (AFFINE mode with a residual operand) for the direct form: this is how gradient fan-in is
        fused. nchw=True (stem conv only, no `dx_add`): the fp32 NCHW gradient of the module input, as the kernel
        writes it."""
        pw = self.pw
        n, h, w, c = self.in_shape
        if self.stem:
            dx = ops.stem_dgrad3x3s2(d_raw, pw.wp, pw.cin, h, w)
            if nchw:
                assert dx_add is None
                return dx
            dx = ops.f32_to_act(dx.permute(0, 2, 3, 1).contiguous(), ops.is_split(d_raw), pad_to=c)
            return dx if dx_add is None else ops.add_act(dx, dx_add)
        assert not nchw, "only the stem conv writes an NCHW input gradient"
        mirrored = [(-dh, -dw, wt) for dh, dw, wt in self.taps]       # taps of the transposed conv
        if self.kind == "direct":
            dx, _ = ops.conv_fprop(d_raw, pw.wd, pw.cin, mirrored, epi=EPI_RAW if dx_add is None else EPI_AFFINE,
                                   residual=dx_add)
            return dx
        if pw.cin % 64 != 0:
            raise NotImplementedError("semseg_b200: input gradient of a stride-2 conv needs Cin % 64 == 0")
        hh, wh = self.xin.shape[-3], self.xin.shape[-2]
        dxp = ops.empty_act((4 * n, hh, wh, pw.cin), ops.is_split(d_raw), d_raw.device)
        for q in range(4):
            sub = [t for t, a in zip(mirrored, self.img_add) if a == q * n]      # the taps that read phase q
            part = ops.act_batch_slice(dxp, q * n, (q + 1) * n)
            if sub:
                ops.conv_fprop(d_raw, pw.wd, pw.cin, sub, out=part, out_nhw=(n, hh, wh))
            else:
                part.zero_()
        dx = ops.phases_to_space(dxp, n, h, w)
        return dx if dx_add is None else ops.add_act(dx, dx_add)

    def wgrad(self, d_raw):
        """Weight gradient, fp32 OIHW like conv.weight."""
        pw = self.pw
        # the kernel reduces over every channel of the tensor it reads: 32 patch columns, or Cin padded to 8 (stem)
        dw = ops.conv_wgrad(self.xin, d_raw, self.xin.shape[-1], pw.cout, self.taps, img_add=self.img_add)
        if self.kind == "patches":          # [Cout, 32, 1, 1]: column (r*3+s)*Cin + c holds weight[:, c, r, s]
            return dw[:, :9 * pw.cin, 0, 0].reshape(pw.cout, 3, 3, pw.cin).permute(0, 3, 1, 2).contiguous()
        return dw[:, :pw.cin].contiguous() if dw.shape[1] != pw.cin else dw


class _CbaState:
    """What one conv+BN(+residual)(+ReLU) stage keeps for its backward pass."""
    __slots__ = ("form", "bn", "frozen", "relu", "has_res", "raw", "y", "mi", "ss", "pg")


def cba_forward(x, conv, bn, relu, residual, out=None, input_needs_grad=True, mode="batch"):
    """conv (1x1 / 3x3; stride 1 with any dilation, or stride 2; see _ConvForm) + BatchNorm in `mode` (see _bn_mode)
    + optional residual + ReLU. Returns (y, state for cba_backward).
      "batch" : three launches: conv (raw + per-CTA statistics) -> finalise (+ SyncBN exchange) -> apply.
      "frozen": running statistics — no statistics, no SyncBN exchange, running statistics and num_batches_tracked
                untouched. When gamma needs a gradient: conv (raw) -> apply with the folded scale / shift, and raw is
                kept for dgamma's x-hat; otherwise the eval kernel, and only x and y are kept.
      "eval"  : the eval kernel: conv + folded BN + residual + ReLU in one launch."""
    form = _ConvForm(conv, x, input_needs_grad, mode)
    raw = mi = pg = None
    if mode == "batch":
        raw, sp = form.fprop(stats=True)
        pg = _sync_group(bn)
        mi, ss = _batch_stats(sp, bn, pg)
    else:
        ss = ops.bn_fold_eval(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
        if mode == "frozen" and bn.weight is not None and bn.weight.requires_grad:
            raw, _ = form.fprop()
    if raw is not None:
        y = ops.bn_apply(raw, ss, residual=residual, relu=relu, out=out)
    else:
        y, _ = form.fprop(epi=EPI_AFFINE, relu=relu, scale=ss[0], shift=ss[1], residual=residual, out=out)
    st = _CbaState()
    # ReLU mask for backward: recomputed from raw when there is raw and no residual, else the saved output
    need_y = relu and (residual is not None or raw is None)
    st.form, st.bn, st.frozen, st.relu, st.has_res = form, bn, mode != "batch", relu, residual is not None
    st.raw, st.y, st.mi, st.pg = raw, (y if need_y else None), mi, pg
    st.ss = ss if (mode == "batch" and relu and not need_y) else None     # the frozen backward derives its own
    return y, st


def cba_backward(st, dy, need_dx=True, need_dw=True, need_dres=False, dx_add=None, dx_nchw=False):
    """Backward of cba_forward: returns (dx, dw, dgamma, dbeta, dres). `dx_add` (same shape as dx) is summed into
    dx; dx_nchw: the stem conv's dx as fp32 NCHW (see _ConvForm.dgrad)."""
    bn = st.bn
    want_dres = st.has_res and need_dres
    if st.frozen:
        want_g, want_b = st.raw is not None, bn.bias is not None and bn.bias.requires_grad
        if not (need_dx or need_dw or want_dres or want_g or want_b):
            return None, None, None, None, None
        # one pass: d_raw = dz*scale (+ dres = dz) and, when gamma / beta need them, the deterministic channel sums
        d_raw, dres, sums = ops.bn_bwd_frozen(dy if dy.is_contiguous() else dy.contiguous(), st.y, st.raw, bn.weight,
                                              bn.bias, bn.running_mean, bn.running_var, bn.eps, st.relu,
                                              want_dres=want_dres, want_sums=want_g or want_b)
        dgamma = sums[1] if want_g else None
        dbeta = sums[0] if want_b else None
    else:
        d_raw, dres, dgamma, dbeta = _bn_backward(st.pg, dy, st.y, st.raw, st.mi, bn.weight, st.relu, want_dres, st.ss)
    dx = st.form.dgrad(d_raw, dx_add, nchw=dx_nchw) if need_dx else None
    dw = st.form.wgrad(d_raw) if need_dw else None
    return dx, dw, dgamma, dbeta, dres


class _ConvBnAct(torch.autograd.Function):
    """Autograd wrapper of one cba_forward / cba_backward stage. `x` is an activation, or — for the stem conv — the
    module's fp32 NCHW input, converted here and given its gradient straight from the stem dgrad kernel."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, residual, conv, bn, relu, out, frozen):
        ctx.nchw = x.dtype != torch.bfloat16
        xa = ops.nchw_to_nhwc_bf16(x.contiguous().float(), split=precision.split_enabled()) if ctx.nchw else x
        y, st = cba_forward(xa, conv, bn, relu, residual, out, input_needs_grad=ctx.needs_input_grad[0],
                            mode="frozen" if frozen else "batch")
        ctx.st = st
        if out is not None:
            ctx.mark_dirty(out)
        return y

    @staticmethod
    def backward(ctx, dy):
        ni = ctx.needs_input_grad
        dx, dw, dgamma, dbeta, dres = cba_backward(ctx.st, dy, need_dx=ni[0], need_dw=ni[1], need_dres=ni[4],
                                                   dx_nchw=ctx.nchw)
        ctx.st = None
        return dx, dw, dgamma, dbeta, dres, None, None, None, None, None


class _BottleneckFn(torch.autograd.Function):
    """A whole Bottleneck (model/resnet.py:74-94) as one autograd node: conv1-bn1-relu, conv2-bn2-relu, conv3-bn3,
    (+ downsample conv-bn), residual add, relu. Besides saving three autograd nodes per block, the backward pass
    fuses the gradient fan-in (dx = dgrad(conv1) + d(residual branch)) into the dgrad epilogue instead of a separate
    elementwise add. `frozen` holds one flag per BatchNorm (bn1, bn2, bn3, downsample): frozen or batch statistics."""

    @staticmethod
    def forward(ctx, x, blk, frozen, *params):
        m1, m2, m3, md = ("frozen" if f else "batch" for f in frozen)
        y1, s1 = cba_forward(x, blk.conv1, blk.bn1, True, None, mode=m1)
        y2, s2 = cba_forward(y1, blk.conv2, blk.bn2, True, None, mode=m2)
        if blk.downsample is not None:
            res, sd = cba_forward(x, blk.downsample[0], blk.downsample[1], False, None, mode=md)
        else:
            res, sd = x, None
        y3, s3 = cba_forward(y2, blk.conv3, blk.bn3, True, res, mode=m3)
        ctx.states = (s1, s2, s3, sd)
        return y3

    @staticmethod
    def backward(ctx, dy):
        s1, s2, s3, sd = ctx.states
        ctx.states = None
        ni = ctx.needs_input_grad      # x, blk, frozen, then (conv weight, gamma, beta) per stage from index 3
        need_dx = ni[0]
        d2, dw3, dg3, db3, dres = cba_backward(s3, dy, need_dw=ni[9], need_dres=True)
        d1, dw2, dg2, db2, _ = cba_backward(s2, d2, need_dw=ni[6])
        grads_ds = ()
        if sd is not None:
            dxd, dwd, dgd, dbd, _ = cba_backward(sd, dres, need_dx=need_dx, need_dw=ni[12])
            dres_to_x = dxd
            grads_ds = (dwd, dgd, dbd)
        else:
            dres_to_x = dres
        dx, dw1, dg1, db1, _ = cba_backward(s1, d1, need_dx=need_dx, need_dw=ni[3],
                                            dx_add=dres_to_x if need_dx else None)
        return (dx, None, None, dw1, dg1, db1, dw2, dg2, db2, dw3, dg3, db3) + grads_ds


def bottleneck(x, blk):
    """Fused Bottleneck when every stage is covered by the native kernels and each BatchNorm uses batch statistics or is
    frozen (see _bn_mode), else stage by stage."""
    convs = [blk.conv1, blk.conv2, blk.conv3] + ([blk.downsample[0]] if blk.downsample is not None else [])
    bns = [blk.bn1, blk.bn2, blk.bn3] + ([blk.downsample[1]] if blk.downsample is not None else [])
    cins = [x.shape[-1], blk.conv1.out_channels, blk.conv2.out_channels, x.shape[-1]]
    params = [blk.conv1.weight, blk.bn1.weight, blk.bn1.bias, blk.conv2.weight, blk.bn2.weight, blk.bn2.bias,
              blk.conv3.weight, blk.bn3.weight, blk.bn3.bias]
    if blk.downsample is not None:
        params += [blk.downsample[0].weight, blk.downsample[1].weight, blk.downsample[1].bias]
    modes = [_bn_mode(b, (x,), params) for b in bns]   # one autograd node: any gradient runs through every stage
    fused = (torch.is_grad_enabled() and "eval" not in modes and
             all(_is_native_conv(c, ci) for c, ci in zip(convs, cins)) and
             (blk.downsample is None or len(blk.downsample) == 2))
    if fused:
        frozen = tuple(m == "frozen" for m in modes) + (False,) * (4 - len(modes))
        return _BottleneckFn.apply(x, blk, frozen, *params)
    y = conv_bn_act(x, blk.conv1, blk.bn1, relu=True)
    y = conv_bn_act(y, blk.conv2, blk.bn2, relu=True)
    residual = conv_bn_act(x, blk.downsample[0], blk.downsample[1], relu=False) if blk.downsample is not None else x
    return conv_bn_act(y, blk.conv3, blk.bn3, relu=True, residual=residual)


def _is_native_conv(conv, cin):
    """Convs the tensor-core kernel covers: 1x1 / 3x3 'same' convs, stride 1 (any dilation) or stride 2 (dilation 1)."""
    ok = (conv.kernel_size in ((1, 1), (3, 3)) and conv.groups == 1 and conv.bias is None and
          conv.padding == (conv.dilation[0] * (conv.kernel_size[0] // 2),) * 2 and
          conv.dilation[0] == conv.dilation[1] and cin % 8 == 0 and conv.out_channels % 64 == 0)
    if conv.stride == (1, 1):
        return ok
    return ok and conv.stride == (2, 2) and conv.dilation == (1, 1)


def _require_native(conv, cin):
    """There is exactly one backend: a convolution the sm_90a kernel does not cover is an error, never a library
    (cuDNN) fallback. Every convolution of PSPNet / PSANet (model/resnet.py, model/pspnet.py, model/psanet.py) is covered."""
    if not _is_native_conv(conv, cin):
        raise NotImplementedError(
            "semseg_b200: convolution %r on %d input channels is outside the tensor-core kernel's coverage (1x1 / 3x3 "
            "'same' convs without bias, stride 1 with any dilation or stride 2 undilated, Cin %% 8 == 0, Cout %% 64 == 0); "
            "there is no library fallback" % (conv, cin))


def conv_bn_act(x, conv, bn, relu=True, residual=None, out=None):
    """NHWC activation -> NHWC activation: conv -> BatchNorm -> (+residual) -> (ReLU), training, frozen or eval
    semantics of `bn` (see _bn_mode)."""
    mode = _bn_mode(bn, (x, residual), (conv.weight, bn.weight, bn.bias))
    _require_native(conv, x.shape[-1])
    if mode != "eval":
        return _ConvBnAct.apply(x, conv.weight, bn.weight, bn.bias, residual, conv, bn, relu, out, mode == "frozen")
    # Eval-mode BatchNorm: conv + folded BN + residual + ReLU are ONE kernel. It has no backward: the reference's
    # validate() (tool/train.py:353-359) calls model.eval()(input) without torch.no_grad() and never back-propagates,
    # so the result is returned detached (a later .backward() through it raises torch's usual "does not require grad").
    # A frozen BatchNorm takes this path only when nothing of the stage needs a gradient (see _bn_mode).
    plan = getattr(_net, "fp8", None)
    if plan is not None:
        y = plan.conv_bn_act(x, conv, bn, relu, residual, out)
        if y is not None:
            return y
    return cba_forward(x, conv, bn, relu, residual, out, mode="eval")[0]


def stem_conv_bn_act(x, conv, bn, relu=True):
    """The module's fp32 NCHW input -> first stem stage (3-channel stride-2 conv -> BatchNorm -> ReLU), NHWC activation.
    When `x` needs a gradient, the input conversion is part of the stage's autograd node and x.grad comes as fp32 NCHW
    straight from the stem dgrad kernel; otherwise this is conv_bn_act(to_nhwc_bf16(x)), the patch form in training."""
    if not (torch.is_grad_enabled() and x.requires_grad):
        return conv_bn_act(to_nhwc_bf16(x), conv, bn, relu=relu)
    mode = _bn_mode(bn, (x,), (conv.weight, bn.weight, bn.bias))
    _require_native(conv, ops.round_up(x.shape[1], 8))
    return _ConvBnAct.apply(x, conv.weight, bn.weight, bn.bias, None, conv, bn, relu, None, mode == "frozen")


# ------------------------------------------------------------------------------------------------ classifier
class _ConvBiasF32(torch.autograd.Function):
    """1x1 conv with bias producing fp32 NHWC logits (model/pspnet.py:69,77)."""

    @staticmethod
    def forward(ctx, x, weight, bias, conv):
        pw = packed(conv, split=ops.is_split(x))
        y, _ = ops.conv_fprop(x, pw.wf, pw.cout, ops.conv_taps(1, 1), epi=EPI_F32, shift=bias)
        ctx.save_for_backward(x)
        ctx.pw = pw
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        pw = ctx.pw
        n, h, w, c = dy.shape
        cp = pw.wd.shape[-1]  # Cout rounded up to 8 (zero padded operand)
        dyb = ops.f32_to_act(dy.contiguous(), ops.is_split(x))      # [N,h,w,cp], padding columns zero
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx, _ = ops.conv_fprop(dyb, pw.wd, pw.cin, ops.conv_taps(1, 1))
        if ctx.needs_input_grad[1]:
            dwp = ops.conv_wgrad(x, dyb, pw.cin, cp, ops.conv_taps(1, 1))
            dw = dwp[:c].contiguous()
        if ctx.needs_input_grad[2]:
            db = dy.sum(dim=(0, 1, 2))
        return dx, dw, db, None


def conv_bias_f32(x, conv, out=None):
    """1x1 conv + bias -> fp32 NHWC. `out` (inference only): a pixel-contiguous fp32 [N, H, W, cout] view to write
    into, e.g. one draw's slice of a larger buffer."""
    assert conv.kernel_size == (1, 1) and conv.stride == (1, 1) and x.shape[-1] % 8 == 0
    if torch.is_grad_enabled() and (x.requires_grad or conv.weight.requires_grad):
        assert out is None, "conv_bias_f32: out= is for the inference forward"
        return _ConvBiasF32.apply(x, conv.weight, conv.bias, conv)
    pw = packed(conv, need_dgrad=False, split=ops.is_split(x))
    y, _ = ops.conv_fprop(x, pw.wf, pw.cout, ops.conv_taps(1, 1), epi=EPI_F32, shift=conv.bias, out_f32=out)
    return y


# ------------------------------------------------------------------------------------------------ fused tail
class _UpsampleCE(torch.autograd.Function):
    """bilinear xZ upsample (align_corners; Z = zoom_factor in {1, 2, 4, 8}, none at 1) + CrossEntropyLoss(ignore_index,
    mean) + argmax in one kernel each way (model/pspnet.py:94-103) — the [N, classes, H, W] logits tensor is never
    materialised."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom):
        info, amax, lse = ops.upsample_ce_fwd(logits, target, ignore_index, zoom=zoom)
        ctx.save_for_backward(logits, target, lse, info)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, info = ctx.saved_tensors
        return ops.upsample_ce_bwd(logits, target, ctx.ignore_index, lse, info, grad_loss, zoom=ctx.zoom), None, None, None


class _UpsampleCEWeighted(torch.autograd.Function):
    """The fused tail with nn.CrossEntropyLoss(weight, label_smoothing): loss = sum of the valid pixels' smoothed,
    weighted losses / D, D = sum of their target weights; 0 with a zero gradient when D = 0. The class weights are
    read on the device at every launch (a CUDA-graph replay sees in-place edits) and get no gradient, as in torch."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, weight, label_smoothing):
        info, amax, lse = ops.upsample_ce_weighted_fwd(logits, target, ignore_index, weight, label_smoothing,
                                                       zoom=zoom)
        ctx.save_for_backward(logits, target, lse, info, weight)
        ctx.ignore_index, ctx.zoom, ctx.label_smoothing = ignore_index, zoom, label_smoothing
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, info, weight = ctx.saved_tensors
        dl = ops.upsample_ce_weighted_bwd(logits, target, ctx.ignore_index, weight, ctx.label_smoothing, lse, info,
                                          grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None


class _UpsampleCEOhem(torch.autograd.Function):
    """The fused tail with the OHEM cross-entropy of losses.OhemCrossEntropyLoss: the forward also keeps each pixel's
    p_t and the device threshold, and the backward trains exactly the pixels the forward kept. With class weights the
    loss is the mean of w_t * nll over the kept pixels (the selection stays unweighted)."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, thresh, min_kept, weight=None):
        info, amax, lse, pt, _nll, thr = ops.upsample_ce_ohem_fwd(logits, target, ignore_index, thresh, min_kept,
                                                                  zoom=zoom, weight=weight)
        ctx.save_for_backward(logits, target, lse, pt, thr, info, weight)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, pt, thr, info, weight = ctx.saved_tensors
        dl = ops.upsample_ce_ohem_bwd(logits, target, ctx.ignore_index, lse, pt, thr, info, grad_loss, zoom=ctx.zoom,
                                      weight=weight)
        return dl, None, None, None, None, None, None


class _UpsampleCEDice(torch.autograd.Function):
    """The fused tail with losses.DiceLoss: soft Dice over every pixel of the call, plus ce_weight * CE. The forward
    keeps the per-class gradient table it reduced on the device; the backward needs nothing else from the host."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, smooth, eps, ce_weight):
        info, amax, lse, table = ops.upsample_ce_dice_fwd(logits, target, ignore_index, smooth, eps, ce_weight,
                                                          zoom=zoom)
        ctx.save_for_backward(logits, target, lse, table)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, table = ctx.saved_tensors
        dl = ops.upsample_ce_dice_bwd(logits, target, ctx.ignore_index, lse, table, grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None, None


class _UpsampleCEFocal(torch.autograd.Function):
    """The fused tail with losses.FocalLoss: the mean over the valid pixels of w_t (1 - p_t)^gamma nll. The forward
    keeps each pixel's gradient modulator; the backward is the plain one scaled per pixel. The class weights are read
    on the device at every launch (a CUDA-graph replay sees in-place edits) and get no gradient."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, gamma, weight=None):
        info, amax, lse, mod = ops.upsample_ce_focal_fwd(logits, target, ignore_index, weight, gamma, zoom=zoom)
        ctx.save_for_backward(logits, target, lse, mod, info)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, mod, info = ctx.saved_tensors
        dl = ops.upsample_ce_focal_bwd(logits, target, ctx.ignore_index, lse, mod, info, grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None


class _UpsampleCERelaxed(torch.autograd.Function):
    """The fused tail with losses.BoundaryRelaxationLoss at border > 0: the omega-weighted mean of -log of each valid
    pixel's label-set mass. The forward keeps each pixel's label set and log2(R / (1 - R)); the backward needs nothing
    else from the host. The class weights are read on the device at every launch and get no gradient."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, border, weight=None):
        info, amax, lse, sets, lq = ops.upsample_ce_relax_fwd(logits, target, ignore_index, weight, border, zoom=zoom)
        ctx.save_for_backward(logits, lse, sets, lq, info)
        ctx.zoom = zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, lse, sets, lq, info = ctx.saved_tensors
        dl = ops.upsample_ce_relax_bwd(logits, lse, sets, lq, info, grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None


class _UpsampleSegPGD(torch.autograd.Function):
    """The fused tail with the SegPGD attack loss (adversarial.PGDAttack(kind='segpgd')): the mean over the valid pixels
    of w nll, w = 1 - lam where the argmax hits the target and lam elsewhere, the weights constants. The forward keeps
    each pixel's weight; the backward is the focal one with that modulator map."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, lam):
        info, amax, lse, mod = ops.upsample_segpgd_fwd(logits, target, ignore_index, lam, zoom=zoom)
        ctx.save_for_backward(logits, target, lse, mod, info)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, mod, info = ctx.saved_tensors
        dl = ops.upsample_ce_focal_bwd(logits, target, ctx.ignore_index, lse, mod, info, grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None


def upsample_segpgd(logits, target, ignore_index, zoom, lam):
    """-> (SegPGD loss scalar, argmax) of fp32 NHWC logits against the zoomed target (see _UpsampleSegPGD)."""
    return _UpsampleSegPGD.apply(logits, target.contiguous(), int(ignore_index), int(zoom), float(lam))


class _UpsampleCEEntropy(torch.autograd.Function):
    """The fused tail with losses.EntropyLoss: ce_weight * CE over the labelled pixels plus ent_weight * the mean
    softmax entropy over the unlabelled ones. The forward keeps each pixel's lse and expected logit; the backward
    weighs the two sets with the forward's counts on the device."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, ent_weight, ce_weight):
        info, amax, lse, mu = ops.upsample_ce_entropy_fwd(logits, target, ignore_index, zoom=zoom)
        ctx.save_for_backward(logits, target, lse, mu, info)
        ctx.cfg = (ignore_index, zoom, ent_weight, ce_weight)
        ctx.mark_non_differentiable(amax)
        return torch.add(info[0] * ce_weight, info[2], alpha=ent_weight), amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, mu, info = ctx.saved_tensors
        ignore_index, zoom, ent_weight, ce_weight = ctx.cfg
        dl = ops.upsample_ce_entropy_bwd(logits, target, ignore_index, ent_weight, ce_weight, lse, mu, info, grad_loss,
                                         zoom=zoom)
        return dl, None, None, None, None, None


def _crf_cfg(crit):
    return crit.radius, crit.sigma_xy, crit.sigma_rgb, crit.mean, crit.std


class _UpsampleCECRF(torch.autograd.Function):
    """The fused tail with losses.GatedCRFLoss: ce_weight * CE (the plain forward and backward, unchanged) plus
    crf_weight * the Gated CRF term on the grid of zoom `crf_zoom` (the tail's own at='output', 1 at 'logits'), with the
    image sampled at stride `istride`. The CRF forward keeps S per grid pixel; its backward adds into the CE gradient."""

    @staticmethod
    def forward(ctx, logits, target, image, ignore_index, zoom, crf_zoom, istride, crf_weight, ce_weight, cfg):
        info, amax, lse = ops.upsample_ce_fwd(logits, target, ignore_index, zoom=zoom)
        cinfo, s, crf_lse = ops.gated_crf_fwd(logits, lse if crf_zoom == zoom else None, image, crf_zoom, istride,
                                              *cfg)
        ctx.save_for_backward(logits, target, image, lse, info, crf_lse, s)
        ctx.cfg = (ignore_index, zoom, crf_zoom, istride, crf_weight, ce_weight, cfg)
        ctx.mark_non_differentiable(amax)
        return torch.add(info[0] * ce_weight, cinfo[0], alpha=crf_weight), amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, image, lse, info, crf_lse, s = ctx.saved_tensors
        ignore_index, zoom, crf_zoom, istride, crf_weight, ce_weight, cfg = ctx.cfg
        dl = ops.upsample_ce_bwd(logits, target, ignore_index, lse, info, grad_loss * ce_weight, zoom=zoom)
        ops.gated_crf_bwd(logits, crf_lse, image, s, crf_weight, grad_loss, dl, crf_zoom, istride, *cfg)
        return dl, None, None, None, None, None, None, None, None, None


class _GatedCRF(torch.autograd.Function):
    """The Gated CRF term alone (unweighted) on the grid of fp32 NHWC logits, the image at the same grid (zoom 1)."""

    @staticmethod
    def forward(ctx, logits, image, cfg):
        cinfo, s, lse = ops.gated_crf_fwd(logits, None, image, 1, 1, *cfg)
        ctx.save_for_backward(logits, image, lse, s)
        ctx.cfg = cfg
        return cinfo[0].clone()

    @staticmethod
    def backward(ctx, grad_loss):
        logits, image, lse, s = ctx.saved_tensors
        dl = torch.zeros_like(logits, memory_format=torch.contiguous_format)
        ops.gated_crf_bwd(logits, lse, image, s, 1.0, grad_loss, dl, 1, 1, *ctx.cfg)
        return dl, None, None


def gated_crf(logits, image, criterion):
    """The unweighted Gated CRF term of losses.GatedCRFLoss `criterion` on the grid of fp32 NHWC logits [N,H,W,C], the
    NCHW fp32 image [N,3,H,W] on the same grid (a constant: it gets no gradient)."""
    return _GatedCRF.apply(logits, image.detach().contiguous(), _crf_cfg(criterion))


def _abl_cfg(crit):
    return crit.max_n_ratio, crit.max_clip_dist, crit.label_smoothing


class _UpsampleCEABL(torch.autograd.Function):
    """The fused tail with losses.ActiveBoundaryLoss: ce_weight * CE (the plain forward and backward, unchanged) plus
    abl_weight * the ABL term on the tail's output grid. The ABL forward keeps its state (distance map, selection and
    w dl/dz per selected pixel); its backward adds into the CE gradient."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, abl_weight, ce_weight, cfg):
        info, amax, lse = ops.upsample_ce_fwd(logits, target, ignore_index, zoom=zoom)
        ainfo, state = ops.abl_fwd(logits, lse, target, ignore_index, zoom, *cfg)
        ctx.save_for_backward(logits, target, lse, info, ainfo, state)
        ctx.cfg = (ignore_index, zoom, abl_weight, ce_weight)
        ctx.mark_non_differentiable(amax)
        return torch.add(info[0] * ce_weight, ainfo[0], alpha=abl_weight), amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, info, ainfo, state = ctx.saved_tensors
        ignore_index, zoom, abl_weight, ce_weight = ctx.cfg
        dl = ops.upsample_ce_bwd(logits, target, ignore_index, lse, info, grad_loss * ce_weight, zoom=zoom)
        ops.abl_bwd(logits, lse, state, ainfo, abl_weight, grad_loss, dl, zoom)
        return dl, None, None, None, None, None, None


class _UpsampleCELovasz(torch.autograd.Function):
    """The fused tail with losses.LovaszSoftmaxLoss, plus ce_weight * CE. The forward keeps the per pixel-class
    Lovász gradient weights (gamma, 4 C bytes per output pixel) it scattered from the sorted segments; the sort's
    buffers are released when it returns."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, classes_all, per_image, ce_weight):
        info, amax, lse, gamma = ops.upsample_ce_lovasz_fwd(logits, target, ignore_index, classes_all, per_image,
                                                            ce_weight, zoom=zoom)
        ctx.save_for_backward(logits, target, lse, gamma)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, gamma = ctx.saved_tensors
        dl = ops.upsample_ce_lovasz_bwd(logits, target, ctx.ignore_index, lse, gamma, grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None, None


class _UpsampleCEKD(torch.autograd.Function):
    """The fused tail with losses.DistillationLoss: ce_weight * CE (the plain forward, at zoom `zoom`) plus
    kd_weight * T^2 * KL(teacher || student) (the distillation forward, at zoom `kd_zoom`: the model's zoom, or 1 on the
    1/8-resolution maps). The backward writes the CE gradient and the distillation kernels add theirs into the same
    buffer. The teacher map is a constant: it gets no gradient."""

    @staticmethod
    def forward(ctx, logits, teacher_logits, target, ignore_index, zoom, kd_zoom, temperature, kd_weight, ce_weight):
        info, amax, lse = ops.upsample_ce_fwd(logits, target, ignore_index, zoom=zoom)
        kl, lse_kd = ops.upsample_kd_fwd(logits, teacher_logits, temperature, zoom=kd_zoom)
        ctx.save_for_backward(logits, teacher_logits, target, lse, info, lse_kd)
        ctx.cfg = (ignore_index, zoom, kd_zoom, temperature, kd_weight, ce_weight)
        ctx.mark_non_differentiable(amax)
        return torch.add(info[0] * ce_weight, kl[0], alpha=kd_weight * temperature * temperature), amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, teacher_logits, target, lse, info, lse_kd = ctx.saved_tensors
        ignore_index, zoom, kd_zoom, temperature, kd_weight, ce_weight = ctx.cfg
        dl = ops.upsample_ce_bwd(logits, target, ignore_index, lse, info, grad_loss * ce_weight, zoom=zoom)
        ops.upsample_kd_bwd(logits, teacher_logits, temperature, kd_weight, lse_kd, grad_loss, dl, zoom=kd_zoom)
        return dl, None, None, None, None, None, None, None, None


class _UpsampleCEIncremental(torch.autograd.Function):
    """The fused tail with losses.IncrementalLoss: ce_weight * the unbiased CE (the kUnbiased forward, at zoom `zoom`)
    plus, with the previous step's logits `teacher_logits` (C_old classes) and kd_weight > 0, kd_weight * the unbiased
    distillation (at zoom `kd_zoom`: the model's zoom, or 1 on the 1/8-resolution maps). Without teacher logits it is
    the unbiased CE alone (the aux head's loss). The backward writes the CE gradient and the distillation kernels add
    theirs into the same buffer. The teacher map is a constant: it gets no gradient."""

    @staticmethod
    def forward(ctx, logits, teacher_logits, target, ignore_index, zoom, kd_zoom, c_old, alpha, kd_weight, ce_weight):
        info, amax, lse, lse_old = ops.upsample_ce_unbiased_fwd(logits, target, ignore_index, c_old, zoom=zoom)
        kd = teacher_logits is not None and kd_weight > 0.0
        ctx.mark_non_differentiable(amax)
        ctx.cfg = (ignore_index, zoom, kd_zoom, c_old, alpha, kd_weight, ce_weight, kd)
        if not kd:
            ctx.save_for_backward(logits, target, lse, lse_old, info)
            return (info[0] if ce_weight == 1.0 else info[0] * ce_weight), amax
        kd_info, lse_kd = ops.upsample_unkd_fwd(logits, teacher_logits, alpha, zoom=kd_zoom)
        ctx.save_for_backward(logits, target, lse, lse_old, info, teacher_logits, lse_kd)
        return torch.add(info[0] * ce_weight, kd_info[0], alpha=kd_weight), amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        ignore_index, zoom, kd_zoom, c_old, alpha, kd_weight, ce_weight, kd = ctx.cfg
        logits, target, lse, lse_old, info = ctx.saved_tensors[:5]
        g = grad_loss if ce_weight == 1.0 else grad_loss * ce_weight
        dl = ops.upsample_ce_unbiased_bwd(logits, target, ignore_index, c_old, lse, lse_old, info, g, zoom=zoom)
        if kd:
            teacher_logits, lse_kd = ctx.saved_tensors[5:]
            ops.upsample_unkd_bwd(logits, teacher_logits, alpha, kd_weight, lse_kd, grad_loss, dl, zoom=kd_zoom)
        return dl, None, None, None, None, None, None, None, None, None


class _UpsampleCEPL(torch.autograd.Function):
    """The fused tail with losses.PseudoLabelLoss: ce_weight * CE over the labelled pixels plus pl_weight * the
    confidence-masked pseudo-label CE over the unlabelled ones. The forward keeps each pixel's effective target and
    weight; the backward is the focal backward on them (w_p (p_c - [c = y_p]), the plain cols kernel with a count of 1).
    The teacher map is a constant: it gets no gradient."""

    @staticmethod
    def forward(ctx, logits, teacher_logits, target, ignore_index, zoom, threshold, pl_weight, ce_weight):
        info, amax, lse, eff, wt = ops.upsample_pl_fwd(logits, teacher_logits, target, ignore_index, threshold,
                                                       pl_weight, ce_weight, zoom=zoom)
        ctx.save_for_backward(logits, eff, lse, wt, info)
        ctx.zoom = zoom
        ctx.mark_non_differentiable(amax)
        return torch.add(info[0] * ce_weight, info[2], alpha=pl_weight), amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, eff, lse, wt, info = ctx.saved_tensors
        dl = ops.upsample_ce_focal_bwd(logits, eff, -1, lse, wt, info[4:], grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None, None, None


class _UpsampleCEPLMix(_UpsampleCEPL):
    """The fused tail with losses.MixPseudoLabelLoss: _UpsampleCEPL on the mixed target, each output pixel's teacher
    image n or its partner (n + 1) mod N as the input-grid mix mask says (ops.upsample_pl_fwd's mixed form). The
    backward is _UpsampleCEPL's, on the effective targets and weights."""

    @staticmethod
    def forward(ctx, logits, teacher_logits, target, ignore_index, zoom, threshold, pl_weight, ce_weight, mix_mask):
        info, amax, lse, eff, wt = ops.upsample_pl_fwd(logits, teacher_logits, target, ignore_index, threshold,
                                                       pl_weight, ce_weight, zoom=zoom, mix_mask=mix_mask)
        ctx.save_for_backward(logits, eff, lse, wt, info)
        ctx.zoom = zoom
        ctx.mark_non_differentiable(amax)
        return torch.add(info[0] * ce_weight, info[2], alpha=pl_weight), amax

    @staticmethod
    def backward(ctx, grad_loss, grad_amax):
        return _UpsampleCEPL.backward(ctx, grad_loss, grad_amax) + (None,)


class _UpsampleCERMI(torch.autograd.Function):
    """The fused tail with losses.RMILoss: RMI + BCE (+ CE) over the call. The forward keeps the pooled Y / Q maps and
    the per-(image, class) gradient table it computed on the device; the backward needs nothing else from the host."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, zoom, bce_weight, pos_alpha, ce_weight):
        info, amax, lse, pooled, table = ops.upsample_ce_rmi_fwd(logits, target, ignore_index, bce_weight, pos_alpha,
                                                                 ce_weight, zoom=zoom)
        ctx.save_for_backward(logits, target, lse, pooled, table)
        ctx.ignore_index, ctx.zoom = ignore_index, zoom
        ctx.mark_non_differentiable(amax)
        return info[0], amax

    @staticmethod
    def backward(ctx, grad_loss, _grad_amax):
        logits, target, lse, pooled, table = ctx.saved_tensors
        dl = ops.upsample_ce_rmi_bwd(logits, target, ctx.ignore_index, lse, pooled, table, grad_loss, zoom=ctx.zoom)
        return dl, None, None, None, None, None, None


class _RelationKD(torch.autograd.Function):
    """losses.DistillationLoss's relation term R of the student's and the teacher's cls[2] features (csrc/relation.cu):
    the forward forms both networks' nodes and the fused KL, the backward recomputes the similarity tiles from the saved
    log-sum-exps and routes the node gradient through the normalisation to each window's maximum. The teacher's
    features are a constant: they get no gradient."""

    @staticmethod
    def forward(ctx, f_s, f_t, temperature, pool):
        split = ops.is_split(f_s)
        xs, arg, inv = ops.relation_nodes(f_s, pool, split, student=True)
        xt = ops.relation_nodes(f_t, pool, split)[0]
        loss, lse = ops.relation_kl_fwd(xs, xt, temperature)
        ctx.save_for_backward(f_s, xs, xt, arg, inv, lse)
        ctx.cfg = (temperature, pool)
        return loss.view(())

    @staticmethod
    def backward(ctx, grad):
        f_s, xs, xt, arg, inv, lse = ctx.saved_tensors
        temperature, pool = ctx.cfg
        dn = ops.relation_kl_bwd(xs, xt, temperature, lse, grad)
        return ops.relation_nodes_bwd(f_s, pool, arg, inv, dn), None, None, None


def relation_kd(f_s, f_t, temperature, pool):
    """CIRKD's mini-batch pixel-to-pixel relation term (losses.DistillationLoss states it) of NHWC activations
    f_s, f_t [B,h,w,512] -> fp32 scalar, differentiable in f_s. There is no fallback: another width, a pool outside
    [1, 16] or mismatched shapes raise."""
    if tuple(f_s.shape[-4:]) != tuple(f_t.shape[-4:]):
        raise ValueError("relation_kd: the student's features %s and the teacher's %s differ in shape" %
                         (tuple(f_s.shape[-4:]), tuple(f_t.shape[-4:])))
    if f_s.shape[-1] != ops.RELATION_C:
        raise ValueError("relation_kd: the relation kernels take %d channels, got %d (no fallback)" %
                         (ops.RELATION_C, f_s.shape[-1]))
    return _RelationKD.apply(f_s, f_t.detach(), float(temperature), int(pool))


def _class_weight_supported(weight, target, classes):
    """Class weights the fused kernels read: None, or a contiguous 1-D fp32 tensor on the target's CUDA device (of
    length `classes` when that is known)."""
    if weight is None:
        return True
    return (torch.is_tensor(weight) and weight.dtype == torch.float32 and weight.dim() == 1 and weight.is_contiguous()
            and weight.is_cuda and weight.device == target.device and (classes is None or weight.numel() == classes))


# The Dice rows kernels stage 12 bytes per pixel of an interval's Z output rows in at most 224 KB of shared memory
# (csrc/tail.cu kDiceSmemMax): Wo <= 2389 at zoom 8.
_DICE_PIXEL_BYTES, _DICE_STAGE_BYTES = 12, 224 * 1024
# The RMI rows kernel stages 8 bytes per pixel in the same 224 KB (Wo <= 3584 at zoom 8); RMI needs a target of at least
# 12 x 12, three pooled cells each way.
_RMI_PIXEL_BYTES, _RMI_MIN_SIZE = 8, 12
# The plain backward rows kernel stages 8 bytes per pixel of an interval's Z output rows in 160 KB (Wo <= 2560 at zoom 8).
_CRF_CE_PIXEL_BYTES, _CRF_CE_STAGE_BYTES = 8, 160 * 1024


def fused_tail_supported(criterion, logits, target, zoom_factor, x_size=None):
    """The fused kernel implements exactly nn.CrossEntropyLoss(weight, ignore_index=k, reduction='mean',
    label_smoothing), losses.OhemCrossEntropyLoss and losses.FocalLoss (each with or without class weights) and
    losses.DiceLoss, at every zoom factor of the model (1, 2, 4, 8) with the target at the zoomed size zoom*(h'-1)+1 of
    the 1/8-resolution logits. The weighted / smoothed forms need the target on a CUDA device and class weights as a
    contiguous fp32 [classes] tensor on that device; any other weight, another reduction, and any subclass keep the
    ATen tail. DiceLoss, FocalLoss and losses.LovaszSoftmaxLoss also need the target no wider than their kernels stage
    (2389 columns at zoom 8), and the Lovász loss fewer than 2^31 target pixels. losses.DistillationLoss takes the plain
    form's conditions, and so does losses.AdversarialLoss (plain cross-entropy on the attacked batch; the attack checks
    its own tail's limits); losses.PseudoLabelLoss and losses.MixPseudoLabelLoss, whose backward is the focal one, and
    losses.EntropyLoss, whose rows kernel stages the same words, losses.IncrementalLoss, whose unbiased CE and
    distillation rows kernels stage as many bytes per pixel, and losses.BoundaryRelaxationLoss (at every border; its
    class weights as the weighted form's), the Dice width limit. losses.RMILoss needs a target of
    at least 12 x 12 and no wider than its rows kernel stages (3584 columns
    at zoom 8). losses.GatedCRFLoss and losses.ActiveBoundaryLoss need the target no wider than the plain backward
    stages (2560 columns at zoom 8); their classes (<= 256, checked here with the logits) and options are in the
    kernels' limits by construction.
    `logits` fp32 NHWC, or None with the NCHW input size `x_size` (decision before the network has run)."""
    if type(criterion) in (losses.DistillationLoss, losses.AdversarialLoss):
        ok = True
    elif type(criterion) is nn.CrossEntropyLoss:
        eps = getattr(criterion, 'label_smoothing', 0.0)
        plain = criterion.weight is None and eps == 0.0
        ok = (criterion.reduction == 'mean' and 0.0 <= eps <= 1.0 and
              (plain or (target is not None and target.is_cuda)))
    elif type(criterion) in (losses.DiceLoss, losses.FocalLoss, losses.PseudoLabelLoss, losses.MixPseudoLabelLoss,
                             losses.EntropyLoss):
        # the focal rows kernel (the pseudo-label backward too) and the entropy rows kernel stage the Dice words
        ok = (zoom_factor in (1, 2, 4, 8) and target is not None and target.dim() == 3 and
              _DICE_PIXEL_BYTES * zoom_factor * target.shape[2] <= _DICE_STAGE_BYTES)
    elif type(criterion) in (losses.GatedCRFLoss, losses.ActiveBoundaryLoss):
        # the cross-entropy part is the plain tail's, whose backward stages 8 bytes per pixel of Z rows in 160 KB; the
        # CRF and ABL kernels take any width (csrc/crf.cu, csrc/boundary.cu), and the criteria keep their options in
        # the kernels' limits
        ok = (zoom_factor in (1, 2, 4, 8) and target is not None and target.dim() == 3 and
              _CRF_CE_PIXEL_BYTES * zoom_factor * target.shape[2] <= _CRF_CE_STAGE_BYTES)
    elif type(criterion) is losses.BoundaryRelaxationLoss:
        # the relaxation rows kernel stages 12 bytes per pixel, the Dice words' size, at every border; border 0 runs
        # the (weighted) cross-entropy kernels, whose limit is wider, and keeps the same decision
        ok = (zoom_factor in (1, 2, 4, 8) and target is not None and target.dim() == 3 and
              _DICE_PIXEL_BYTES * zoom_factor * target.shape[2] <= _DICE_STAGE_BYTES)
    elif type(criterion) is losses.IncrementalLoss:
        # the unbiased CE and distillation rows kernels stage 12 bytes per pixel, the Dice words' size, in the same 224 KB
        ok = (zoom_factor in (1, 2, 4, 8) and target is not None and target.dim() == 3 and
              _DICE_PIXEL_BYTES * zoom_factor * target.shape[2] <= _DICE_STAGE_BYTES)
    elif type(criterion) is losses.RMILoss:
        ok = (zoom_factor in (1, 2, 4, 8) and target is not None and target.dim() == 3 and
              target.shape[1] >= _RMI_MIN_SIZE and target.shape[2] >= _RMI_MIN_SIZE and
              _RMI_PIXEL_BYTES * zoom_factor * target.shape[2] <= _DICE_STAGE_BYTES)
    elif type(criterion) is losses.LovaszSoftmaxLoss:
        # the Lovász rows kernel stages the Dice words; its sort payloads hold a pixel index in 31 bits
        ok = (zoom_factor in (1, 2, 4, 8) and target is not None and target.dim() == 3 and
              _DICE_PIXEL_BYTES * zoom_factor * target.shape[2] <= _DICE_STAGE_BYTES and
              target.numel() < 2 ** 31)
    else:
        ok = type(criterion) is losses.OhemCrossEntropyLoss
    if not (ok and zoom_factor in (1, 2, 4, 8)
            and target is not None and target.dtype == torch.int64 and target.dim() == 3):
        return False
    if not _class_weight_supported(getattr(criterion, "weight", None), target,
                                   None if logits is None else logits.shape[-1]):
        return False
    if logits is None:
        h, w = (x_size[2] - 1) // 8 + 1, (x_size[3] - 1) // 8 + 1      # the network's output stride is 8
    else:
        if logits.shape[-1] > 256:
            return False
        h, w = logits.shape[1], logits.shape[2]
    return target.shape[1] == zoom_factor * (h - 1) + 1 and target.shape[2] == zoom_factor * (w - 1) + 1


def upsample_ce(logits, target, ignore_index, zoom=8, criterion=None, teacher_logits=None, mix_mask=None,
                image=None, image_stride=None):
    """-> (mean CE loss scalar, argmax int64 [N,H,W]); H = zoom*(h-1)+1, W = zoom*(w-1)+1. With a
    losses.OhemCrossEntropyLoss `criterion`, the loss is its OHEM cross-entropy (its own ignore_index and class
    weights); with an nn.CrossEntropyLoss that has class weights or label smoothing, its weighted / smoothed mean;
    with a losses.DiceLoss, its Dice (+ CE) loss (its own ignore_index); with a losses.RMILoss, its RMI + BCE (+ CE)
    loss; with a losses.LovaszSoftmaxLoss, its
    Lovász-Softmax (+ CE) loss; with a losses.FocalLoss, its focal loss (its own ignore_index, gamma and class
    weights); with a losses.DistillationLoss and the teacher's fp32 NHWC logits `teacher_logits`
    (the student's shape), its distillation loss, and with a losses.PseudoLabelLoss and them its pseudo-label loss
    (without them: the plain mean CE, the loss of the aux head). With a losses.MixPseudoLabelLoss, the teacher's logits
    of the unmixed batch and the mix mask `mix_mask` (ops.mix_apply's), the mixed pseudo-label loss on the mixed target;
    without the mask it is a losses.PseudoLabelLoss. With a losses.EntropyLoss, its ce_weight * CE over the labelled
    pixels plus ent_weight * mean entropy over the unlabelled ones (its own ignore_index); the networks score their aux
    head with the plain form. With a losses.GatedCRFLoss and the network's fp32 NCHW input `image` (a constant),
    ce_weight * CE plus crf_weight * its Gated CRF term; `image_stride` is the image's pixel stride on the loss grid
    (default: 8 / zoom at at='output', 8 at at='logits'); without an image a positive crf_weight raises. With a
    losses.ActiveBoundaryLoss, ce_weight * CE plus abl_weight * its boundary term on the output grid. With a
    losses.IncrementalLoss and the previous step's fp32 NHWC logits `teacher_logits` ([N, h, w, C_old]), ce_weight *
    its unbiased CE plus kd_weight * its unbiased distillation; without them the unbiased CE alone (the aux head's
    loss). With a losses.BoundaryRelaxationLoss, its relaxed loss over each pixel's label set (its own ignore_index,
    border and class weights; border 0 is the (weighted) cross-entropy step). The default criterion runs the plain
    kernels."""
    if isinstance(criterion, losses.ActiveBoundaryLoss):
        if criterion.abl_weight == 0.0:
            # no ABL kernel: the plain step, bit for bit when ce_weight is 1
            loss, amax = _UpsampleCE.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom))
            return (loss if criterion.ce_weight == 1.0 else loss * criterion.ce_weight), amax
        return _UpsampleCEABL.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                    criterion.abl_weight, criterion.ce_weight, _abl_cfg(criterion))
    if isinstance(criterion, losses.GatedCRFLoss):
        if criterion.crf_weight == 0.0:
            # no CRF kernel: the plain step, bit for bit when ce_weight is 1
            loss, amax = _UpsampleCE.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom))
            return (loss if criterion.ce_weight == 1.0 else loss * criterion.ce_weight), amax
        if image is None:
            raise ValueError("GatedCRFLoss with crf_weight > 0 needs the image on the fused tail")
        out = criterion.at == 'output'
        istride = image_stride if image_stride is not None else (8 // int(zoom) if out else 8)
        return _UpsampleCECRF.apply(logits, target.contiguous(), image.detach().contiguous(), criterion.ignore_index,
                                    int(zoom), int(zoom) if out else 1, int(istride), criterion.crf_weight,
                                    criterion.ce_weight, _crf_cfg(criterion))
    if type(criterion) is losses.MixPseudoLabelLoss and teacher_logits is not None and mix_mask is not None:
        return _UpsampleCEPLMix.apply(logits, teacher_logits.detach(), target.contiguous(), criterion.ignore_index,
                                      int(zoom), criterion.threshold, criterion.pl_weight, criterion.ce_weight,
                                      mix_mask)
    if isinstance(criterion, losses.IncrementalLoss):
        kd_zoom = 1 if criterion.at == 'logits' else int(zoom)
        t = None if teacher_logits is None else teacher_logits.detach()
        ce_weight = 1.0 if t is None else criterion.ce_weight
        return _UpsampleCEIncremental.apply(logits, t, target.contiguous(), criterion.ignore_index, int(zoom), kd_zoom,
                                            criterion.c_old, criterion.alpha, criterion.kd_weight, ce_weight)
    if isinstance(criterion, losses.DistillationLoss) and teacher_logits is not None:
        kd_zoom = 1 if criterion.at == 'logits' else int(zoom)
        return _UpsampleCEKD.apply(logits, teacher_logits.detach(), target.contiguous(), criterion.ignore_index,
                                   int(zoom), kd_zoom, criterion.temperature, criterion.kd_weight, criterion.ce_weight)
    if isinstance(criterion, losses.PseudoLabelLoss) and teacher_logits is not None:
        return _UpsampleCEPL.apply(logits, teacher_logits.detach(), target.contiguous(), criterion.ignore_index,
                                   int(zoom), criterion.threshold, criterion.pl_weight, criterion.ce_weight)
    if isinstance(criterion, losses.EntropyLoss):
        return _UpsampleCEEntropy.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                        criterion.ent_weight, criterion.ce_weight)
    if isinstance(criterion, losses.LovaszSoftmaxLoss):
        return _UpsampleCELovasz.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                       criterion.classes == 'all', bool(criterion.per_image), criterion.ce_weight)
    if isinstance(criterion, losses.FocalLoss):
        if criterion.weight is None:
            return _UpsampleCEFocal.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                          criterion.gamma)
        return _UpsampleCEFocal.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom), criterion.gamma,
                                      criterion.weight)
    if isinstance(criterion, losses.BoundaryRelaxationLoss):
        w = criterion.weight
        if criterion.border == 0:
            # every set is the pixel's own label: the (weighted) cross-entropy step, bit for bit
            if w is None:
                return _UpsampleCE.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom))
            return _UpsampleCEWeighted.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom), w, 0.0)
        if w is None:
            return _UpsampleCERelaxed.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                            criterion.border)
        return _UpsampleCERelaxed.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                        criterion.border, w)
    if isinstance(criterion, losses.RMILoss):
        return _UpsampleCERMI.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom), criterion.bce_weight,
                                    criterion.pos_alpha, criterion.ce_weight)
    if isinstance(criterion, losses.DiceLoss):
        return _UpsampleCEDice.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom), criterion.smooth,
                                     criterion.eps, criterion.ce_weight)
    if isinstance(criterion, losses.OhemCrossEntropyLoss):
        if criterion.weight is None:
            return _UpsampleCEOhem.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom),
                                         criterion.thresh, criterion.min_kept)
        return _UpsampleCEOhem.apply(logits, target.contiguous(), criterion.ignore_index, int(zoom), criterion.thresh,
                                     criterion.min_kept, criterion.weight)
    if isinstance(criterion, nn.CrossEntropyLoss) and (criterion.weight is not None or
                                                       getattr(criterion, 'label_smoothing', 0.0) != 0.0):
        return _UpsampleCEWeighted.apply(logits, target.contiguous(), ignore_index, int(zoom), criterion.weight,
                                         float(criterion.label_smoothing))
    return _UpsampleCE.apply(logits, target.contiguous(), ignore_index, int(zoom))


def upsample_fp(logits, target, zoom, criterion, teacher_logits, mix_mask=None):
    """The feature-perturbation term of a losses.PseudoLabelLoss (or MixPseudoLabelLoss, with the mix mask) whose
    fp_weight > 0: fp_weight * its pseudo-label term on the perturbed stream's fp32 NHWC logits, with no labelled term.
    It is the pseudo-label tail of upsample_ce with ce_weight 0 and pl_weight = fp_weight -> (loss, argmax)."""
    args = (logits, teacher_logits.detach(), target.contiguous(), criterion.ignore_index, int(zoom), criterion.threshold,
            criterion.fp_weight, 0.0)
    if mix_mask is not None:
        return _UpsampleCEPLMix.apply(*args, mix_mask)
    return _UpsampleCEPL.apply(*args)


# ------------------------------------------------------------------------------------------------ pyramid pooling
class _PPMLink:
    """Carries the identity-branch gradient of x from the concat node to the pooling node of one PPM invocation.

    x feeds both AdaptiveAvgPool (all bins) and the concat (model/pspnet.py:20-26); autograd would add the two gradients
    with a strided ATen kernel (one of them is a channel slice of the 4096-wide concat gradient). The concat node always
    runs first in backward (the pooled branch reaches x only through it), so it parks its slice here and returns no
    gradient for x; the pooling node's kernel adds the slice while it writes dx."""
    __slots__ = ("dx_identity",)

    def __init__(self):
        self.dx_identity = None


class _PPMPool(torch.autograd.Function):
    """AdaptiveAvgPool2d of every bin in one launch (model/pspnet.py:14)."""

    @staticmethod
    def forward(ctx, x, bins, link):
        ctx.bins, ctx.shape, ctx.link = bins, tuple(x.shape[-4:]), link
        return tuple(ops.ppm_pool(x, bins))

    @staticmethod
    def backward(ctx, *dpooled):
        n, h, w, c = ctx.shape
        add = None
        if ctx.link is not None:
            add, ctx.link.dx_identity = ctx.link.dx_identity, None
        return ops.ppm_pool_bwd(list(dpooled), ctx.bins, n, h, w, c, add=add), None, None


class _PPMUpsampleConcat(torch.autograd.Function):
    """cat([x, bilinear(f_1), ..., bilinear(f_nb)], channel) written in place (model/pspnet.py:25-26)."""

    @staticmethod
    def forward(ctx, x, bins, link, *feats):
        ctx.bins, ctx.c, ctx.cr, ctx.link = bins, x.shape[-1], feats[0].shape[-1], link
        return ops.ppm_upsample_concat(x, list(feats), bins)

    @staticmethod
    def backward(ctx, dout):
        if not dout.is_contiguous():
            dout = dout.contiguous()
        dfeats = ops.ppm_upsample_bwd(dout, ctx.c, ctx.bins, ctx.cr)
        dx = dout[..., :ctx.c]
        if ctx.link is not None and ctx.needs_input_grad[0] and all(ctx.needs_input_grad[3:]):
            ctx.link.dx_identity = dx      # summed into dx by the pooling node's kernel (see _PPMLink)
            dx = None
        return (dx, None, None) + tuple(dfeats)


def ppm_pool(x, bins, link=None):
    return _PPMPool.apply(x, tuple(bins), link)


def ppm_upsample_concat(x, feats, bins, link=None):
    return _PPMUpsampleConcat.apply(x, tuple(bins), link, *feats)


def ppm_link():
    return _PPMLink()


# ------------------------------------------------------------------------------------------------ fused PSA attention
class _PSAAttend(torch.autograd.Function):
    """psa_mask (or the compact mode's dense view) -> softmax over the source positions (or none) -> aggregation bmm ->
    1/normalization_factor (model/psanet.py:76-91) as one kernel each way; nothing [HW x HW] is written to HBM (with
    softmax the backward recomputes the probabilities from the logits and the saved per-target (max, 1/sum); without it
    the probabilities are the logits, and neither the statistics nor the output are kept)."""

    @staticmethod
    def forward(ctx, attn, feat, psa_type, mask_h, mask_w, scale, compact, softmax):
        out, stats = ops.psa_attend(attn, feat, psa_type, mask_h, mask_w, scale, compact=compact, softmax=softmax)
        if softmax:
            ctx.save_for_backward(attn, feat, out, stats)
        else:
            ctx.save_for_backward(attn, feat)
        ctx.cfg = (psa_type, mask_h, mask_w, scale, compact, softmax)
        return out

    @staticmethod
    def backward(ctx, dout):
        psa_type, mask_h, mask_w, scale, compact, softmax = ctx.cfg
        attn, feat, out, stats = ctx.saved_tensors + (None, None) * (not softmax)
        if not dout.is_contiguous():
            dout = dout.contiguous()
        form = dict(compact=compact, softmax=softmax)
        dattn = dfeat = None
        if ctx.needs_input_grad[1]:
            dfeat, _ = ops.psa_attend(attn, dout, psa_type, mask_h, mask_w, scale, stats=stats, mode=1, **form)
        if ctx.needs_input_grad[0]:
            dattn = ops.psa_attend_bwd_attn(attn, stats, feat, out, dout, psa_type, mask_h, mask_w, scale, **form)
        return dattn, dfeat, None, None, None, None, None, None


def psa_attend(attn, feat, psa_type, mask_h, mask_w, scale, compact=False, softmax=True):
    """attn fp32 NHWC [N,h,w,mask_h*mask_w], feat NHWC activation [N,h,w,512] -> aggregated features [N,h,w,512].
    compact: the dense form of the reference's compact mode (mask_h*mask_w == h*w); softmax: its psa_softmax."""
    return _PSAAttend.apply(attn.contiguous(), feat, psa_type, mask_h, mask_w, scale, compact, softmax)


def psa_attend_supported(feat, mask_h, mask_w, compact=False):
    """Whether the fused kernels cover this geometry: 512 channels, at most 128 columns, and odd masks (window form) or a
    mask of exactly h*w entries (compact mode's dense form)."""
    if feat.shape[-1] != 512 or feat.shape[-2] > 128:
        return False
    if compact:
        return mask_h * mask_w == feat.shape[-3] * feat.shape[-2]
    return mask_h % 2 == 1 and mask_w % 2 == 1


# ------------------------------------------------------------------------------------------------ bilinear resize
class _ResizeBilinear(torch.autograd.Function):
    """F.interpolate(mode='bilinear', align_corners=True) on an NHWC activation (model/psanet.py:61,97), deterministic
    gather backward."""

    @staticmethod
    def forward(ctx, x, size):
        ctx.in_size = tuple(x.shape[-3:-1])
        return ops.resize_bilinear(x, size)

    @staticmethod
    def backward(ctx, dy):
        return ops.resize_bilinear_bwd(dy if dy.is_contiguous() else dy.contiguous(), ctx.in_size), None


def resize_bilinear(x, size):
    return _ResizeBilinear.apply(x, tuple(size))


# ------------------------------------------------------------------------------------------------ misc NHWC ops
class _NCHWToAct(torch.autograd.Function):
    """fp32 NCHW -> activation (differentiable): the gradient goes back as fp32 NCHW through the split-aware
    transpose, the padding channels dropped."""

    @staticmethod
    def forward(ctx, x, split):
        ctx.c = x.shape[1]
        return ops.nchw_to_nhwc_bf16(x.contiguous().float(), split=split)

    @staticmethod
    def backward(ctx, dy):
        return ops.nhwc_bf16_to_nchw((dy if dy.is_contiguous() else dy.contiguous())[..., :ctx.c]), None


def to_nhwc_bf16(x_nchw):
    """fp32 NCHW module input -> NHWC activation (channels padded to a multiple of 8 with zeros) in the storage form of
    the current precision mode (precision.py): plain bf16, or (hi, lo) bf16 planes for bf16x3. Differentiable when
    the input needs a gradient."""
    if torch.is_grad_enabled() and x_nchw.requires_grad:
        return _NCHWToAct.apply(x_nchw, precision.split_enabled())
    return ops.nchw_to_nhwc_bf16(x_nchw.contiguous().float(), split=precision.split_enabled())


class _ActToF32(torch.autograd.Function):
    """activation -> fp32 NHWC (differentiable)."""

    @staticmethod
    def forward(ctx, x):
        ctx.split = ops.is_split(x)
        return ops.act_to_f32(x)

    @staticmethod
    def backward(ctx, dy):
        return ops.f32_to_act(dy.contiguous(), ctx.split)


class _F32ToAct(torch.autograd.Function):
    """fp32 NHWC -> activation in the requested storage form (differentiable)."""

    @staticmethod
    def forward(ctx, x, split):
        return ops.f32_to_act(x.contiguous(), split)

    @staticmethod
    def backward(ctx, dy):
        return ops.act_to_f32(dy.contiguous()), None


def act_to_f32(x):
    return _ActToF32.apply(x)


def f32_to_act(x, split):
    return _F32ToAct.apply(x, split)


def to_nchw_f32(y):
    """NHWC activation -> fp32 NCHW (what the reference's modules return)."""
    if not (torch.is_grad_enabled() and y.requires_grad):
        return ops.nhwc_bf16_to_nchw(y)
    return act_to_f32(y).permute(0, 3, 1, 2)


class _Fork(torch.autograd.Function):
    """x -> k aliases of x whose gradients are summed by the split-aware add kernel (autograd's own accumulation would
    add the hi and lo planes of two split gradients separately, losing the error compensation)."""

    @staticmethod
    def forward(ctx, x, k):
        return tuple(x.view_as(x) for _ in range(k))

    @staticmethod
    def backward(ctx, *grads):
        acc = None
        for g in grads:
            if g is None:
                continue
            g = g if g.is_contiguous() else g.contiguous()
            acc = g if acc is None else ops.add_act(acc, g)
        return acc, None


def fork(x, k=2):
    """k handles on x for k consumers (gradient fan-in through one native add per extra branch)."""
    if not (torch.is_grad_enabled() and x.requires_grad):
        return (x,) * k
    return _Fork.apply(x, k)


class _ScaleNC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        ctx.save_for_backward(scale)
        return ops.scale_nc(x, scale)

    @staticmethod
    def backward(ctx, dy):
        (scale,) = ctx.saved_tensors
        return ops.scale_nc(dy if dy.is_contiguous() else dy.contiguous(), scale), None


class _FPFork(torch.autograd.Function):
    """x [M] -> cat(x, x[:N] * scale) [M + N] (UniMatch's feature-perturbation batch; M > N when the first N images are
    one stream of several) in one native launch. The backward is the fold kernel alone, d[:M] with scale * d[M:] added
    to its first N images, rounded once: autograd never sums the two parts (as in _Fork, a split-aware sum, here with the
    scale in the same fp32 expression). No gradient reaches the scale. M = N runs the plain fork and fold."""

    @staticmethod
    def forward(ctx, x, scale):
        ctx.save_for_backward(scale)
        ctx.prefix = x.shape[-4] != scale.shape[0]
        return ops.fp_fork_prefix(x, scale) if ctx.prefix else ops.fp_fork(x, scale)

    @staticmethod
    def backward(ctx, d):
        (scale,) = ctx.saved_tensors
        d = d if d.is_contiguous() else d.contiguous()
        return (ops.fp_fold_prefix(d, scale) if ctx.prefix else ops.fp_fold(d, scale)), None


def fp_fork(x, scale):
    """cat(x, x[:N] * scale[n, c]) along the batch of an M-image activation (scale fp32 [N, C], N <= M); differentiable
    in x."""
    return _FPFork.apply(x, scale)


def dropout2d_scale(n, c, p, device):
    """nn.Dropout2d's draw: fp32 [n, c], 0 or 1/(1-p) per (image, channel). dropout2d_nhwc and the Monte Carlo dropout
    draws of the sliding-window predictor both take it from here, so one seed gives both the same masks."""
    return torch.empty((n, c), device=device, dtype=torch.float32).bernoulli_(1.0 - p).mul_(1.0 / (1.0 - p))


def dropout2d_nhwc(x, p, training):
    """nn.Dropout2d on NHWC: one Bernoulli per (n, c), kept channels scaled by 1/(1-p) (model/pspnet.py:68,76)."""
    if not training or p == 0.0:
        return x
    return _ScaleNC.apply(x, dropout2d_scale(x.shape[-4], x.shape[-1], p, x.device))


class _MaxPool3x3s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y, code = ops.maxpool3x3s2_fwd(x, want_argcode=True)
        ctx.save_for_backward(code)
        ctx.in_shape = tuple(x.shape[-4:])
        return y

    @staticmethod
    def backward(ctx, dy):
        (code,) = ctx.saved_tensors
        return ops.maxpool3x3s2_bwd(code, dy, ctx.in_shape)


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def maxpool_nhwc(x, pool):
    if (_pair(pool.kernel_size) == (3, 3) and _pair(pool.stride) == (2, 2) and _pair(pool.padding) == (1, 1)
            and _pair(pool.dilation) == (1, 1) and not pool.ceil_mode and x.shape[-1] % 8 == 0):
        return _MaxPool3x3s2.apply(x)
    raise NotImplementedError("semseg_b200: only MaxPool2d(kernel_size=3, stride=2, padding=1) (model/resnet.py:115) is "
                              "implemented; there is no library fallback (got %r)" % (pool,))
