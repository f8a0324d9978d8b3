"""FP8 (e4m3) inference for this package's PSPNet / PSANet: post-training quantisation with static scales.

    q = Fp8Eval(model)            # eval-mode network on CUDA; the model itself is never modified
    for x in calib_batches:
        q.calibrate(x)            # bf16 eval forward; device amax of every FP8 conv input
    q.freeze()                    # e4m3 weight slabs, per-output-channel weight scales, folded epilogue scales
    logits = q(x)                 # what model(x) returns, computed with e4m3 tensor-core convolutions
    SlidingWindowPredictor(q, classes, crop, crop, mean, std)

Which stages run in FP8 (`fp8_stages`): every conv + BatchNorm stage with Cin % 128 == 0 in layer1..layer4, the PPM
branches, PSA's reduce / attention[0] / proj and cls[0]. The stem, layer1's 64-channel convs, PSA's mask-logit conv, the
classifier and every non-conv kernel keep their bf16 path.

Scales: activation qscale = 448 / amax (per tensor, amax = max |x| over the calibration batches, dequantised by
amax / 448); weights per output channel the same with amax_c. Every quantisation is q = sat_e4m3(v * qscale) in fp32,
rounded to nearest even and saturated to +-448 (never NaN). Dequantisation folds into the conv epilogue's BatchNorm scale:
scale[c] = bn_scale[c] * (s_w[c] * s_x).

Storage: a conv whose only consumer is an FP8 conv (bottleneck conv1 -> stride-1 conv2, conv2 -> conv3) writes e4m3
only, at the consumer's qscale; a block output writes bf16 (the residual stream) plus an e4m3 twin at the next block's
conv1 qscale; everything else writes bf16, and an FP8 conv quantises a bf16 input itself (one launch)."""
import numpy as np
import torch

from . import functional as SF
from . import ops
from . import precision

E4M3_MAX = 448.0


def _net_of(model):
    """The PSPNet / PSANet behind `model` (nn.DataParallel over one device unwrapped), validated for FP8 eval."""
    from .psanet import PSANet
    from .pspnet import PSPNet
    if isinstance(model, torch.nn.DataParallel):
        if len(model.device_ids) > 1:
            raise ValueError("Fp8Eval: nn.DataParallel over %d devices is not supported; wrap model.module"
                             % len(model.device_ids))
        model = model.module
    if type(model) not in (PSPNet, PSANet):
        raise TypeError("Fp8Eval: needs a semseg_b200 PSPNet or PSANet, got %s" % type(model).__name__)
    p = next(iter(model.parameters()))
    if not p.is_cuda:
        raise ValueError("Fp8Eval: the model is on %s; FP8 inference runs on CUDA only" % p.device)
    return model


def fp8_stages(model):
    """[(name, conv, bn)] of the conv + BatchNorm stages of a semseg_b200 PSPNet / PSANet that run in FP8, in forward
    order: Cin % 128 == 0 among the bottleneck convs and downsamples, the PPM branches, PSA's reduce / attention[0] /
    proj (and their _p twins) and cls[0]. Names are those of model.named_modules()."""
    out = []
    for lname in ("layer1", "layer2", "layer3", "layer4"):
        for i, blk in enumerate(getattr(model, lname)):
            pairs = [("conv1", blk.conv1, blk.bn1), ("conv2", blk.conv2, blk.bn2), ("conv3", blk.conv3, blk.bn3)]
            if blk.downsample is not None:
                pairs.append(("downsample.0", blk.downsample[0], blk.downsample[1]))
            out += [("%s.%d.%s" % (lname, i, n), c, b) for n, c, b in pairs]
    if getattr(model, "use_ppm", False):
        out += [("ppm.features.%d.1" % i, f[1], f[2]) for i, f in enumerate(model.ppm.features)]
    if getattr(model, "use_psa", False):
        for n in ("reduce", "attention", "reduce_p", "attention_p", "proj"):
            seq = getattr(model.psa, n, None)
            if seq is not None:
                out.append(("psa.%s.0" % n, seq[0], seq[1]))
    out.append(("cls.0", model.cls[0], model.cls[1]))
    return [(n, c, b) for n, c, b in out if c.in_channels % 128 == 0]


def _qscale(amax):
    """fp32 (qscale = 448 / amax, s = amax / 448); an all-zero tensor (amax 0) gets qscale 1."""
    a = np.float32(amax) if amax > 0 else np.float32(E4M3_MAX)
    return np.float32(E4M3_MAX) / a, a / np.float32(E4M3_MAX)


def _param_key(conv, bn):
    return tuple((t._version, t.data_ptr()) for t in (conv.weight, bn.weight, bn.bias, bn.running_mean,
                                                     bn.running_var) if t is not None)


class _Stage:
    __slots__ = ("name", "conv", "bn", "qscale", "wf", "scale", "shift", "bf16_out", "out_qscale", "key")


class _Calibrator:
    """fp8_plan of a calibration forward: records the input amax of every FP8 stage, runs nothing itself."""

    def __init__(self, index, bits, seen):
        self.index, self.bits, self.seen = index, bits, seen

    def conv_bn_act(self, x, conv, bn, relu, residual, out):
        k = self.index.get(conv)
        if k is not None:
            ops.fp8_amax(x, self.bits[k:k + 1])
            self.seen[k] += 1
        return None


class _Plan:
    """fp8_plan of the FP8 forward: runs every frozen stage on the e4m3 conv kernel."""

    def __init__(self, stages):
        self.stages = {st.conv: st for st in stages}
        self.twin = None        # (bf16 block output, qscale, its e4m3 copy) for the next block's conv1 / downsample

    def conv_bn_act(self, x, conv, bn, relu, residual, out):
        st = self.stages.get(conv)
        if st is None:
            if x.dtype == ops.E4M3:
                raise RuntimeError("Fp8Eval: an e4m3 activation reached the bf16 stage of %r" % (conv,))
            return None
        if out is not None:
            raise NotImplementedError("Fp8Eval: an FP8 stage writes its own output tensors (out= is not supported)")
        k = conv.kernel_size[0]
        img_add = out_nhw = None
        if conv.stride[0] == 2:     # the phase form (functional._ConvForm), quantised after the phase split
            n, h, w = x.shape[:3]
            t2 = ops.conv_taps_s2(k, n)
            taps, img_add = [t[:3] for t in t2], [t[3] for t in t2]
            out_nhw = (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1)
            if x.dtype == ops.E4M3:
                raise RuntimeError("Fp8Eval: the stride-2 stage %s needs a bf16 input" % st.name)
            x8 = ops.fp8_quantize(ops.space_to_phases(x), st.qscale)
        else:
            taps = ops.conv_taps(k, conv.dilation[0])
            if x.dtype == ops.E4M3:
                x8 = x                   # written by its producer at this stage's qscale
            elif self.twin is not None and self.twin[0] is x and self.twin[1] == st.qscale:
                x8 = self.twin[2]
            else:
                x8 = ops.fp8_quantize(x, st.qscale)
        y, y8 = ops.conv_fprop_e4m3(x8, st.wf, conv.out_channels, taps, scale=st.scale, shift=st.shift, relu=relu,
                                    residual=residual, bf16_out=st.bf16_out, y8_qscale=st.out_qscale,
                                    img_add=img_add, out_nhw=out_nhw)
        if y is None:
            return y8
        if y8 is not None:
            self.twin = (y, st.out_qscale, y8)
        return y


class Fp8Eval:
    """FP8 eval wrapper of a semseg_b200 PSPNet / PSANet (see the module docstring). `calibration`: a dict from
    `calibration()` of an earlier wrapper of the same architecture, which replaces calibrate(). One wrapper holds
    per-call state (the e4m3 twin of the last block output), so it must not be called from two threads at once."""

    def __init__(self, model, calibration=None):
        self.model = _net_of(model)
        self._check_eval()
        self._stages = fp8_stages(self.model)
        self._index = {c: k for k, (_, c, _) in enumerate(self._stages)}
        dev = self.model.cls[0].weight.device
        self._bits = torch.zeros((len(self._stages),), dtype=torch.int32, device=dev)
        self._seen = [0] * len(self._stages)
        self._plan = None
        if calibration is not None:
            names = [n for n, _, _ in self._stages]
            if sorted(calibration) != sorted(names):
                missing = sorted(set(names) - set(calibration))
                extra = sorted(set(calibration) - set(names))
                raise ValueError("Fp8Eval: the calibration does not match the model's FP8 stages (missing %s, "
                                 "unknown %s)" % (missing[:4], extra[:4]))
            vals = np.array([calibration[n] for n in names], dtype=np.float32)
            if not np.all(np.isfinite(vals)) or np.any(vals < 0):
                raise ValueError("Fp8Eval: calibration amax values must be finite and >= 0")
            self._bits.copy_(torch.from_numpy(vals.view(np.int32)))
            self._seen = [1] * len(self._stages)

    # ---- the nn.Module surface SlidingWindowPredictor and callers use
    @property
    def training(self):
        return self.model.training

    def parameters(self):
        return self.model.parameters()

    def _check_eval(self):
        if self.model.training:
            raise RuntimeError("Fp8Eval: the model is in training mode; FP8 is eval-only (call model.eval())")

    # ---- calibration
    def calibrate(self, x):
        """One bf16 eval forward of the fp32 NCHW batch `x`; folds max |input| of every FP8 stage into the running
        amax on the device (no host synchronisation). Invalidates an earlier freeze()."""
        self._check_eval()
        self._plan = None
        with torch.no_grad(), precision.mode("bf16"), SF.fp8_plan(_Calibrator(self._index, self._bits, self._seen)):
            self.model(x)

    def calibration(self):
        """{stage name: amax} (fp32 values as Python floats) of the calibration so far."""
        vals = self._bits.cpu().numpy().view(np.float32)
        return {n: float(v) for (n, _, _), v in zip(self._stages, vals)}

    def freeze(self):
        """Quantise the weights (e4m3 slabs, per-output-channel scales) and fold the dequantisation into the
        epilogue scales. Needs calibrate() (or a `calibration`) to have reached every FP8 stage."""
        self._check_eval()
        missed = [n for (n, _, _), s in zip(self._stages, self._seen) if s == 0]
        if missed:
            raise RuntimeError("Fp8Eval.freeze: calibrate() has not reached %d FP8 stages (%s ...)"
                               % (len(missed), ", ".join(missed[:3])))
        amax = self._bits.cpu().numpy().view(np.float32)
        bad = [n for (n, _, _), a in zip(self._stages, amax) if not np.isfinite(a)]
        if bad:
            raise RuntimeError("Fp8Eval.freeze: calibrate() saw non-finite activations at %d FP8 stages (%s ...); an "
                               "infinite scale would turn the logits into NaN" % (len(bad), ", ".join(bad[:3])))
        stages = []
        for (name, conv, bn), a in zip(self._stages, amax):
            st = _Stage()
            st.name, st.conv, st.bn = name, conv, bn
            st.qscale, s_x = _qscale(float(a))
            st.wf, s_w = ops.fp8_pack_weights(conv.weight)
            ss = ops.bn_fold_eval(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
            st.scale = (ss[0] * (s_w * float(s_x))).contiguous()
            st.shift = ss[1].contiguous()
            st.bf16_out, st.out_qscale = True, None
            st.key = _param_key(conv, bn)
            stages.append(st)
        by_conv = {st.conv: st for st in stages}
        blocks = [b for l in (self.model.layer1, self.model.layer2, self.model.layer3, self.model.layer4) for b in l]
        for i, blk in enumerate(blocks):
            s1, s2, s3 = by_conv.get(blk.conv1), by_conv.get(blk.conv2), by_conv.get(blk.conv3)
            if s1 is not None and s2 is not None and blk.conv2.stride == (1, 1):
                s1.bf16_out, s1.out_qscale = False, s2.qscale        # conv1 -> conv2 only
            if s2 is not None and s3 is not None:
                s2.bf16_out, s2.out_qscale = False, s3.qscale        # conv2 -> conv3 only
            nxt = by_conv.get(blocks[i + 1].conv1) if i + 1 < len(blocks) else None
            if s3 is not None and nxt is not None:
                s3.out_qscale = nxt.qscale                           # block output: bf16 + e4m3 twin
        self._plan = _Plan(stages)

    # ---- the FP8 forward
    def _enter(self, x):
        self._check_eval()
        if self._plan is None:
            raise RuntimeError("Fp8Eval: call freeze() after calibrate() before running the FP8 network")
        if torch.is_tensor(x) and x.requires_grad:
            raise RuntimeError("Fp8Eval: the FP8 forward has no backward; pass an input that does not require grad")
        for st in self._plan.stages.values():
            if _param_key(st.conv, st.bn) != st.key:
                raise RuntimeError("Fp8Eval: the weights or BatchNorm statistics of %s changed since freeze(); call "
                                   "freeze() again" % st.name)
        self._plan.twin = None

    def __call__(self, x):
        """Same contract as model.eval()(x): fp32 NCHW logits [N, classes, H, W]."""
        self._enter(x)
        try:
            with torch.no_grad(), precision.mode("bf16"), SF.fp8_plan(self._plan):
                return self.model(x)
        finally:
            self._plan.twin = None

    def _eval_logits_nhwc(self, x):
        """fp32 NHWC logits before the final upsample (the sliding-window engine's native finish)."""
        self._enter(x)
        try:
            with torch.no_grad(), precision.mode("bf16"), SF.fp8_plan(self._plan):
                return self.model._eval_logits_nhwc(x)
        finally:
            self._plan.twin = None
