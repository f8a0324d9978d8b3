"""GPU tier of FP8 (e4m3) inference: the quantise / amax / pack kernels bit for bit against tests/fp8_oracle.py, the e4m3
conv element by element against an fp64 conv of the dequantised operands, the networks against the fake-quant oracle,
and the sliding-window predictor on top."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from semseg_b200 import functional as SF
from semseg_b200 import ops
from semseg_b200 import precision
from semseg_b200.fp8 import Fp8Eval, fp8_stages
from tests import fp8_oracle as O
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _strict_fp32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("amax", [1.0, 3.3e-3, 2.5e4])
def test_quantize_every_bf16_pattern(amax):
    bits = torch.arange(65536, dtype=torch.int32).to(torch.int16)
    x = bits.view(torch.bfloat16).reshape(1, 64, 64, 16).cuda()
    qs, _ = O.qscale_of(amax)
    got = ops.fp8_quantize(x, qs)
    ref = O.quantize(x.cpu(), qs)
    g, r = got.cpu().view(torch.uint8), ref.view(torch.uint8)
    nan = ref.float().isnan()
    assert torch.equal(got.cpu().float().isnan(), nan)
    assert torch.equal(g[~nan], r[~nan])


def test_amax_exact_and_accumulating():
    g = torch.Generator(device="cuda").manual_seed(3)
    bits = torch.zeros(1, dtype=torch.int32, device="cuda")
    ref = 0.0
    for k in range(3):
        x = (torch.randn((2, 17, 23, 136), device="cuda", generator=g) * (10.0 ** k)).to(torch.bfloat16)
        ops.fp8_amax(x, bits)
        ref = max(ref, float(x.float().abs().amax()))
        assert bits.view(torch.float32).item() == ref
    view = torch.empty((1, 9, 9, 256), dtype=torch.bfloat16, device="cuda").fill_(1.0)[..., 64:192]   # a channel slice
    view[0, 4, 4, 7] = -1000.0
    b2 = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.fp8_amax(view, b2)
    assert b2.view(torch.float32).item() == 1000.0


@pytest.mark.parametrize("shape", [(64, 128, 1, 1), (512, 4096, 3, 3), (256, 256, 3, 3), (2048, 1024, 1, 1)])
def test_pack_matches_oracle(shape):
    w = torch.randn(shape, generator=torch.Generator().manual_seed(5)) * 0.05
    w[1] = 0.0
    wf, sw = ops.fp8_pack_weights(w.cuda())
    rwf, rsw = O.pack_weights(w)
    assert torch.equal(wf.cpu().view(torch.uint8), rwf.view(torch.uint8))
    assert torch.equal(sw.cpu(), rsw)


# (Cin, Cout, k, dilation, stride, N, H, W, residual, relu, outputs)
CONV_CASES = [
    (128, 64, 1, 1, 1, 1, 9, 13, False, True, "bf16"),
    (256, 128, 1, 1, 1, 2, 17, 11, True, True, "both"),
    (128, 128, 3, 1, 1, 3, 15, 19, False, True, "e4m3"),
    (256, 256, 3, 2, 1, 1, 21, 20, False, False, "both"),
    (512, 512, 3, 4, 1, 2, 12, 23, False, True, "bf16"),
    (1024, 256, 1, 1, 1, 1, 31, 29, False, True, "e4m3"),
    (2048, 512, 1, 1, 1, 2, 11, 9, True, True, "both"),
    (4096, 512, 3, 1, 1, 1, 13, 14, False, True, "bf16"),
    (128, 128, 3, 1, 2, 2, 25, 23, False, True, "bf16"),     # layer2.0 conv2 (phase form)
    (256, 512, 1, 1, 2, 1, 17, 30, False, False, "bf16"),    # layer2.0 downsample (phase form)
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "ci%d_co%d_k%d_d%d_s%d_n%d_%s" % (c[:6] + (c[10],)))
def test_e4m3_conv_elementwise(case):
    cin, cout, k, dil, stride, n, h, w, res, relu, outs = case
    g = torch.Generator().manual_seed(cin + cout + k + dil)
    x = torch.randn((n, h, w, cin), generator=g).abs().to(torch.bfloat16) * (1 + (cin % 3))
    wt = torch.randn((cout, cin, k, k), generator=g) / (cin * k * k) ** 0.5
    amax = float(x.float().abs().max())
    qs, sx = O.qscale_of(amax)
    bn_scale = torch.rand(cout, generator=g) + 0.5
    shift = torch.randn(cout, generator=g) * 0.1
    wf, sw = ops.fp8_pack_weights(wt.cuda())
    scale = (bn_scale.cuda() * (sw * float(sx))).contiguous()
    xc = x.cuda()
    if stride == 2:
        t2 = ops.conv_taps_s2(k, n)
        taps, img_add = [t[:3] for t in t2], [t[3] for t in t2]
        out_nhw = (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1)
        x8 = ops.fp8_quantize(ops.space_to_phases(xc), qs)
    else:
        taps, img_add, out_nhw = ops.conv_taps(k, dil), None, None
        x8 = ops.fp8_quantize(xc, qs)
    ho, wo = out_nhw[1:] if out_nhw else (h, w)
    resid = (torch.randn((n, ho, wo, cout), generator=g) * 0.5).to(torch.bfloat16) if res else None
    out_qs = O.qscale_of(4.0)[0]
    y, y8 = ops.conv_fprop_e4m3(x8, wf, cout, taps, scale=scale, shift=shift.cuda(), relu=relu,
                                residual=resid.cuda() if res else None, bf16_out=outs != "e4m3",
                                y8_qscale=out_qs if outs != "bf16" else None, img_add=img_add, out_nhw=out_nhw)
    # fp64 reference from the dequantised operands (the device's own quantised input)
    xq = O.quantize(x, qs).double() * float(sx)
    wq = O.dequant_weights(wt)
    pad = dil * (k // 2)
    acc = F.conv2d(xq.permute(0, 3, 1, 2), wq, stride=stride, padding=pad, dilation=dil).permute(0, 2, 3, 1)
    mag = F.conv2d(xq.abs().permute(0, 3, 1, 2), wq.abs(), stride=stride, padding=pad, dilation=dil).permute(0, 2, 3, 1)
    ref = acc * bn_scale.double() + shift.double()
    if res:
        ref = ref + resid.double()
    if relu:
        ref = ref.clamp_min(0)
    # accumulation error bound: the FP8 tensor core keeps about 13 bits within one 128-channel K block (DESIGN §4)
    bound = 2.0 ** -12 * mag * bn_scale.double()
    if y is not None:
        err = (y.cpu().double() - ref).abs()
        ratio = float(((err - 2.0 ** -8 * ref.abs()) / bound.clamp_min(1e-30)).max())
        print("conv %s: bf16 output excess over rounding = %.3f of the accumulation bound" % (case, ratio))
        assert bool((err <= 2.0 ** -8 * ref.abs() + bound).all())
    if y8 is not None:
        q_ref = O.e4m3(ref.float() * out_qs)
        # within one e4m3 step of the oracle's rounding of every value the error bound allows (near zero the bound
        # spans several subnormal steps), and equal where no rounding boundary lies within the bound
        lo, hi = O.e4m3((ref - bound).float() * out_qs), O.e4m3((ref + bound).float() * out_qs)
        got = O.e4m3_order(y8.cpu().view(torch.uint8))
        assert bool((got >= O.e4m3_order(lo.view(torch.uint8)) - 1).all())
        assert bool((got <= O.e4m3_order(hi.view(torch.uint8)) + 1).all())
        safe = lo.view(torch.uint8) == hi.view(torch.uint8)
        assert bool(safe.any())
        assert torch.equal(y8.cpu().view(torch.uint8)[safe], q_ref.view(torch.uint8)[safe])


NETS = [
    ("psp50", lambda: util.build_pspnet(50, classes=150), 473, "psp", dict(layers=50, classes=150)),
    ("psp101", lambda: util.build_pspnet(101, classes=19), 713, "psp", dict(layers=101, classes=19)),
    ("psa50", lambda: util.build_psanet(50, classes=21, mask=59), 465, "psa", None),
]


class _Recorder:
    """fp8_plan that runs the frozen plan and keeps every FP8 stage's input, residual and outputs."""

    def __init__(self, plan):
        self.plan, self.calls = plan, []

    def conv_bn_act(self, x, conv, bn, relu, residual, out):
        st = self.plan.stages.get(conv)
        tw = self.plan.twin          # the e4m3 twin the stage reads instead of a bf16 block output, if any
        xin = tw[2] if (st is not None and tw is not None and tw[0] is x and tw[1] == st.qscale) else x
        y = self.plan.conv_bn_act(x, conv, bn, relu, residual, out)
        if st is not None:
            y8 = y if y.dtype == ops.E4M3 else (self.plan.twin[2] if st.out_qscale is not None else None)
            self.calls.append((st, xin, residual, relu, None if y.dtype == ops.E4M3 else y, y8))
        return y


def _consumers(model, names):
    """{stage name: the FP8 stage that reads its e4m3 output} from the network's structure: bottleneck conv1 -> conv2
    (stride 1), conv2 -> conv3, conv3 -> the next block's conv1."""
    blocks = [("%s.%d" % (ln, i), b) for ln in ("layer1", "layer2", "layer3", "layer4")
              for i, b in enumerate(getattr(model, ln))]
    out = {}
    for i, (p, blk) in enumerate(blocks):
        if p + ".conv2" in names and blk.conv2.stride == (1, 1):
            out[p + ".conv1"] = p + ".conv2"
        out[p + ".conv2"] = p + ".conv3"
        if i + 1 < len(blocks):
            out[p + ".conv3"] = blocks[i + 1][0] + ".conv1"
    return {k: v for k, v in out.items() if k in names and v in names}


def _check_stage(st, x, residual, relu, y, y8, cal, consumer_qs):
    """One FP8 stage against fp64 from the device's own input: the input quantised (or read) at the stage's calibrated
    scale, the oracle's e4m3 weights, BatchNorm folded in fp64. Returns the largest error as a share of the bound."""
    conv, bn = st.conv, st.bn
    qs, sx = O.qscale_of(cal[st.name])
    xq = (x.float().double() if x.dtype == ops.E4M3 else O.quantize(x, qs).double()) * float(sx)
    wq = O.dequant_weights(conv.weight)
    k, dil, stride = conv.kernel_size[0], conv.dilation[0], conv.stride[0]
    args = dict(stride=stride, padding=dil * (k // 2), dilation=dil)
    acc = F.conv2d(xq.permute(0, 3, 1, 2), wq, **args).permute(0, 2, 3, 1)
    mag = F.conv2d(xq.abs().permute(0, 3, 1, 2), wq.abs(), **args).permute(0, 2, 3, 1)
    g = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    b = bn.bias.double() - bn.running_mean.double() * g
    ref = acc * g + b
    if residual is not None:
        ref = ref + residual.double()
    if relu:
        ref = ref.clamp_min(0)
    # accumulation bound (DESIGN §4) plus the fp32 folding of BatchNorm and dequantisation scales
    bound = 2.0 ** -12 * mag * g.abs() + 1e-6 * ((acc * g).abs() + b.abs())
    worst = 0.0
    if y is not None:
        err = (y.double() - ref).abs() - 2.0 ** -8 * ref.abs()
        worst = float((err / bound).max())
        assert bool((err <= bound).all()), (st.name, worst)
    if y8 is not None:
        cq = consumer_qs
        lo, hi = O.e4m3((ref - bound).float() * cq), O.e4m3((ref + bound).float() * cq)
        got = O.e4m3_order(y8.view(torch.uint8))
        assert bool((got >= O.e4m3_order(lo.view(torch.uint8)) - 1).all()), st.name
        assert bool((got <= O.e4m3_order(hi.view(torch.uint8)) + 1).all()), st.name
    return worst


@pytest.mark.parametrize("net", NETS, ids=lambda n: n[0])
def test_network_against_fake_quant_oracle(net):
    name, build, size, arch, okw = net
    from oracle.torch_oracle import Oracle  # noqa: F401
    model = build().cuda().eval()
    g = torch.Generator().manual_seed(7)
    x = torch.randn((1, 3, size, size), generator=g).cuda()
    with torch.no_grad():
        before = model(x)
    q = Fp8Eval(model)
    q.calibrate(x)
    q.freeze()
    got = q(x)
    again = q(x)
    assert torch.equal(got, again)                               # reruns are bit-identical
    with torch.no_grad():
        after = model(x)
    assert torch.equal(before, after)                            # the model itself is untouched
    cal = q.calibration()
    names = [n for n, _, _ in fp8_stages(model)]
    assert set(cal) == set(names)
    # stage by stage: every FP8 stage ran once, on the e4m3 kernel, at its calibrated scales, and wrote its e4m3 output
    # at the scale of the stage that reads it
    rec = _Recorder(q._plan)
    q._enter(x)
    with torch.no_grad(), precision.mode("bf16"), SF.fp8_plan(rec):
        assert torch.equal(q.model(x), got)
    assert sorted(st.name for st, *_ in rec.calls) == sorted(names)      # forward order: downsample after conv2
    cons = _consumers(model, set(names))
    worst = 0.0
    for st, xin, res, relu, y, y8 in rec.calls:
        assert (y8 is not None) == (st.name in cons), st.name
        cq = O.qscale_of(cal[cons[st.name]])[0] if st.name in cons else None
        worst = max(worst, _check_stage(st, xin, res, relu, y, y8, cal, cq))
    del rec
    print("%s: %d FP8 stages within their bound (largest error %.2f of it)" % (name, len(names), worst))
    q2 = Fp8Eval(model, calibration=cal)
    q2.freeze()
    assert torch.equal(q2(x), got)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    if arch == "psp":
        orc = O.FakeQuantOracle(sd, cal, arch="psp", **okw).eval()
    else:
        m = model.psa
        orc = O.FakeQuantOracle(sd, cal, arch="psa", layers=50, classes=21, psa_type=m.psa_type, compact=m.compact,
                                shrink_factor=m.shrink_factor, mask_h=m.mask_h, mask_w=m.mask_w,
                                normalization_factor=m.normalization_factor, psa_softmax=m.psa_softmax).eval()
    with torch.no_grad():
        ref = orc.forward(x)
        plain = Oracle(sd, **(okw or dict(arch="psa", layers=50, classes=21, psa_type=m.psa_type, compact=m.compact,
                                               shrink_factor=m.shrink_factor, mask_h=m.mask_h, mask_w=m.mask_w,
                                               normalization_factor=m.normalization_factor,
                                               psa_softmax=m.psa_softmax))).eval().forward(x)
    rel = float((got.double() - ref.double()).norm() / ref.double().norm())
    rel_bf16 = float((before.double() - plain.double()).norm() / plain.double().norm())
    rel_q = float((ref.double() - plain.double()).norm() / plain.double().norm())
    print("%s: FP8 vs fake-quant oracle rel-L2 %.3e (bf16 vs fp32 oracle %.3e; quantisation itself %.3e)"
          % (name, rel, rel_bf16, rel_q))
    # Every stage is within its per-conv bound of its own input (above). End to end, the device rounds its activations to
    # bf16 before quantising them, so some e4m3 roundings (steps of 2^-3 relative) land on the other side of a boundary
    # than the fp32 oracle's, and these untrained seeded networks amplify such differences as they amplify the bf16 gap
    # tenfold (DESIGN §4). The device must still be closer to the fake-quant oracle than the fp32 network is.
    assert rel < rel_q


class _Foreign(torch.nn.Module):
    """The FP8 network behind a module the engine does not recognise: forces the ATen finish."""

    def __init__(self, q):
        super().__init__()
        self.q = q
        self.anchor = torch.nn.Parameter(torch.zeros(1, device="cuda"))

    def forward(self, x):
        return self.q(x)


def test_predictor_native_finish_matches_aten_finish():
    from semseg_b200 import inference
    from semseg_b200.anomaly import AnomalyScorer
    from semseg_b200.densecrf import DenseCRF
    c = util.SW_CFG
    classes, crop = 7, 65
    model = util.build_pspnet(50, classes=classes).cuda().eval()
    image = util.sw_image(seed=11, h=100, w=150)
    scales, base = [0.75, 1.0, 1.25], 150
    q = Fp8Eval(model)
    for s in (1, 2):
        q.calibrate(torch.randn((2, 3, crop, crop), generator=torch.Generator().manual_seed(s)).cuda())
    q.freeze()
    aten = inference.SlidingWindowPredictor(_Foreign(q), classes, crop, crop, c["mean"], c["std"], max_batch=8)
    ref_scores, ref_amax = aten(image, base, scales)
    native = inference.SlidingWindowPredictor(q, classes, crop, crop, c["mean"], c["std"], max_batch=8)
    assert inference._native_net(q, classes, crop, crop, torch.device("cuda")) is q
    scores, amax = native(image, base, scales)
    assert native.forward_calls == aten.forward_calls
    assert np.abs(scores - ref_scores).max() <= 2e-6
    top2 = np.sort(ref_scores, axis=2)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 4e-6
    assert clear.mean() > 0.9 and np.array_equal(amax[clear], ref_amax[clear])
    ex_scores, _ = native(image, base, scales, exact=True)
    assert np.abs(ex_scores - ref_scores).max() <= 2e-6
    crf = inference.SlidingWindowPredictor(q, classes, crop, crop, c["mean"], c["std"], max_batch=8, crf=DenseCRF())
    cs, ca = crf(image, base, scales)
    aten_crf = inference.SlidingWindowPredictor(_Foreign(q), classes, crop, crop, c["mean"], c["std"], max_batch=8,
                                                crf=DenseCRF())
    rcs, rca = aten_crf(image, base, scales)
    assert cs.shape == scores.shape and np.abs(cs - rcs).max() <= 1e-4
    top2 = np.sort(rcs, axis=2)[..., -2:]
    sure = (top2[..., 1] - top2[..., 0]) > 2e-4
    assert sure.mean() > 0.9 and np.array_equal(ca[sure], rca[sure])
    an = inference.SlidingWindowPredictor(q, classes, crop, crop, c["mean"], c["std"], max_batch=8,
                                          anomaly=AnomalyScorer(kind="maxlogit"))
    out = an(image, base, scales)
    s0 = out[0] if isinstance(out[0], np.ndarray) else out[0].cpu().numpy()
    assert np.array_equal(s0, scores) and tuple(out[-1].shape) == (100, 150)
