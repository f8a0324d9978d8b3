"""GPU tier (-m gpu): the parity-precision operand mode "bf16x3" (semseg_b200/precision.py) against fp32 references.

north_star's bar — "logits match the reference PyTorch path on identical random-init weights and synthetic inputs to
1e-3 rel fp32 with bit-exact argmax masks" — is asserted here at the network level (PSPNet50 @ 473x473 and PSANet50 @
465x465, eval on the freshly constructed model: the regime BASELINE.md §4.6 / SURVEY.md §7 define as the parity regime),
and much tighter bounds at kernel and block level where nothing amplifies a rounding error:

  * conv fprop / dgrad / wgrad, BN, pooling, PPM kernels on split (hi, lo) activations vs torch fp32 (TF32 off): <= 5e-5
  * Bottleneck (d = 2, 4) and PPM blocks, train mode: forward <= 1e-4, every gradient <= 1e-3
  * networks: eval logits rel-L2 <= 1e-4 (north_star asks 1e-3), ZERO argmax flips at every pixel whose fp32 top-1/top-2
    margin exceeds twice the largest logit error; train-step losses to 1e-4.

What "bit-exact argmax" can mean on 447 458 pixels is measured by tools/probe_x3_floor.py: the fp32 oracle against ITSELF
with another cuDNN algorithm (channels_last) already differs in a few near-tie pixels — the reference is not bit-exact
against itself — and so does the fp32 oracle with every conv operand rounded to 16 mantissa bits and EXACT fp32
accumulation (the best any hi/lo bf16 scheme can do). The raw flip count is therefore asserted against a floor
(<= 64 of ~440k pixels, i.e. 1.5e-4 of the pixels), the margin-aware count against 0.

The reference arithmetic is fp32 (model/resnet.py:63-92, model/pspnet.py:80-105); the oracle is oracle/torch_oracle.py
(pinned to the reference's own outputs in tests/test_oracle_cpu.py) running fp32 on the GPU with TF32 disabled.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _strict_fp32_and_x3():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from semseg_b200 import precision
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    prev = precision.get_mode()
    precision.set_mode("bf16x3")
    yield
    precision.set_mode(prev)


def _split(x_nhwc_f32):
    from semseg_b200 import ops
    return ops.f32_to_act(x_nhwc_f32.contiguous(), True)


def _f32(act):
    from semseg_b200 import ops
    return ops.act_to_f32(act)


def test_split_storage_round_trip_and_layout_kernels():
    """hi + lo carries 16 mantissa bits: |v - (hi + lo)| <= 2^-17 |v|; the layout kernels agree with it."""
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((2, 13, 11, 24), device="cuda", generator=g) * 3
    a = _split(x)
    assert a.shape == (2, 2, 13, 11, 24) and a.dtype == torch.bfloat16
    back = _f32(a)
    assert float(((back - x).abs() / x.abs().clamp_min(1e-20)).max()) < 2.0 ** -16
    assert torch.equal(a[0].float(), x.to(torch.bfloat16).float())               # hi = bf16(v)
    xn = x.permute(0, 3, 1, 2).contiguous()
    b = ops.nchw_to_nhwc_bf16(xn, split=True)
    assert torch.equal(b, a)
    assert torch.equal(ops.nhwc_bf16_to_nchw(b), back.permute(0, 3, 1, 2))
    # channel padding 3 -> 8 is zero in both planes
    c = ops.nchw_to_nhwc_bf16(xn[:, :3].contiguous(), split=True)
    assert c.shape[-1] == 8 and float(c[..., 3:].float().abs().max()) == 0.0


CONV_CASES = [(2, 12, 12, 64, 256, 1, 1), (2, 60, 60, 256, 256, 3, 2), (1, 60, 60, 512, 512, 3, 4),
              (1, 30, 30, 512, 2048, 1, 1), (1, 59, 59, 64, 64, 3, 1), (2, 31, 29, 128, 192, 3, 1),
              (16, 1, 1, 2048, 512, 1, 1), (1, 90, 90, 256, 256, 3, 2)]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_x3_fprop_dgrad_wgrad_vs_torch_fp32(case):
    from semseg_b200 import ops
    n, h, w, cin, cout, k, dil = case
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((n, h, w, cin), device="cuda", generator=g)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) / (cin * k * k) ** 0.5
    dy = torch.randn((n, h, w, cout), device="cuda", generator=g)
    xs, dys = _split(x), _split(dy)
    pw = ops.pack_weights(wt, split=True)
    y, sp = ops.conv_fprop(xs, pw.wf, cout, ops.conv_taps(k, dil), stats=True)
    # reference on exactly the values the kernel sees (hi + lo of x; w is within 2^-17 of its split form)
    xf = _f32(xs).permute(0, 3, 1, 2).requires_grad_(True)
    wf = wt.clone().requires_grad_(True)
    ref = F.conv2d(xf, wf, padding=dil * (k // 2), dilation=dil)
    ref.backward(_f32(dys).permute(0, 3, 1, 2))
    assert util.rel_l2(_f32(y), ref.permute(0, 2, 3, 1)) < 3e-5
    st = ops.bn_merge_partials(sp)
    yf = _f32(y).reshape(-1, cout)
    assert torch.allclose(st[0], yf.mean(0), atol=5e-5)
    assert torch.allclose(st[1] / st[2], yf.var(0, unbiased=False), rtol=1e-3, atol=1e-7)
    dx, _ = ops.conv_fprop(dys, pw.wd, cin, ops.conv_taps(k, dil, transpose=True))
    assert util.rel_l2(_f32(dx), xf.grad.permute(0, 2, 3, 1)) < 3e-5
    dw = ops.conv_wgrad(xs, dys, cin, cout, ops.conv_taps(k, dil))
    assert util.rel_l2(dw, wf.grad) < 3e-5


def test_conv_x3_epilogues():
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    n, h, w, cin, cout = 2, 30, 30, 128, 256
    x = torch.randn((n, h, w, cin), device="cuda", generator=g)
    wt = torch.randn((cout, cin, 3, 3), device="cuda", generator=g) * 0.03
    res = torch.randn((n, h, w, cout), device="cuda", generator=g)
    scale = torch.rand((cout,), device="cuda", generator=g) + 0.5
    shift = torch.randn((cout,), device="cuda", generator=g)
    xs, rs = _split(x), _split(res)
    pw = ops.pack_weights(wt, split=True)
    conv = lambda a, ww: F.conv2d(a.permute(0, 3, 1, 2), ww, padding=ww.shape[-1] // 2).permute(0, 2, 3, 1)  # noqa: E731
    y, _ = ops.conv_fprop(xs, pw.wf, cout, ops.conv_taps(3, 1), epi=ops.EPI_AFFINE, relu=True, scale=scale,
                          shift=shift, residual=rs)
    ref = torch.relu(conv(_f32(xs), wt) * scale + shift + _f32(rs))
    assert util.rel_l2(_f32(y), ref) < 3e-5
    w2 = torch.randn((150, cin, 1, 1), device="cuda", generator=g) * 0.05
    b2 = torch.randn((150,), device="cuda", generator=g)
    y2, _ = ops.conv_fprop(xs, ops.pack_weights(w2, split=True).wf, 150, ops.conv_taps(1, 1), epi=ops.EPI_F32, shift=b2)
    assert util.rel_l2(y2, conv(_f32(xs), w2) + b2) < 3e-5
    # channel-slice output of a wider split buffer
    buf = torch.zeros((2, n, h, w, 512), device="cuda", dtype=torch.bfloat16)
    ops.conv_fprop(xs, pw.wf, cout, ops.conv_taps(3, 1), out=buf[..., 256:512])
    assert util.rel_l2(_f32(buf[..., 256:512]), conv(_f32(xs), wt)) < 3e-5
    assert bool((buf[..., :256] == 0).all())


def test_bn_and_elementwise_kernels_split_vs_torch():
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    n, h, w, c = 2, 30, 30, 256
    x = _split(torch.randn((n, h, w, c), device="cuda", generator=g) * 2 + 0.5)
    res = _split(torch.randn((n, h, w, c), device="cuda", generator=g))
    dy = _split(torch.randn((n, h, w, c), device="cuda", generator=g))
    gamma = torch.rand((c,), device="cuda", generator=g) + 0.5
    beta = torch.randn((c,), device="cuda", generator=g)
    xf = _f32(x).permute(0, 3, 1, 2).requires_grad_(True)
    rf = _f32(res).permute(0, 3, 1, 2).requires_grad_(True)
    gm, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    pre = F.batch_norm(xf, None, None, gm, bt, True, 0.1, 1e-5) + rf
    yr = torch.relu(pre)
    # statistics from the conv epilogue of an identity-free path are covered above; here: finalize from fp32 moments
    v = xf.detach().permute(0, 2, 3, 1).reshape(-1, c)
    stats = torch.stack([v.mean(0), v.var(0, unbiased=False) * v.shape[0], torch.full((c,), float(v.shape[0]),
                                                                                          device="cuda")])
    mi, ss = ops.bn_finalize(stats, gamma, beta, 1e-5, 0.1, None, None)
    y = ops.bn_apply(x, ss, residual=res, relu=True)
    assert util.rel_l2(_f32(y), yr.permute(0, 2, 3, 1)) < 2e-5
    yr.backward(_f32(dy).permute(0, 3, 1, 2))
    _, sums = ops.bn_bwd_reduce(dy, y, x, mi, True)
    dx, dres, dgb = ops.bn_bwd_apply(dy, y, x, mi, gamma, sums, float(n * h * w), True, want_dres=True)
    assert util.rel_l2(_f32(dx), xf.grad.permute(0, 2, 3, 1)) < 5e-5
    assert util.rel_l2(_f32(dres), rf.grad.permute(0, 2, 3, 1)) < 2e-5
    assert util.rel_l2(dgb[0], gm.grad) < 2e-5 and util.rel_l2(dgb[1], bt.grad) < 2e-5
    # add / per-(image, channel) scale
    s = ops.add_act(x, res)
    assert util.rel_l2(_f32(s), _f32(x) + _f32(res)) < 2e-5
    sc = torch.rand((n, c), device="cuda", generator=g)
    assert util.rel_l2(_f32(ops.scale_nc(x, sc)), _f32(x) * sc.view(n, 1, 1, c)) < 2e-5


def test_maxpool_and_stride2_split_vs_torch():
    from semseg_b200 import functional as SF
    g = torch.Generator(device="cuda").manual_seed(0)
    x = _split(torch.relu(torch.randn((2, 37, 37, 64), device="cuda", generator=g))).requires_grad_(True)
    y = SF.maxpool_nhwc(x, torch.nn.MaxPool2d(3, 2, 1))
    xr = _f32(x.detach()).permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.max_pool2d(xr, 3, 2, 1)
    assert torch.equal(_f32(y), yr.permute(0, 2, 3, 1))
    gy = _split(torch.randn(tuple(y.shape[-4:]), device="cuda", generator=g))
    y.backward(gy)
    yr.backward(_f32(gy).permute(0, 3, 1, 2))
    assert util.rel_l2(_f32(x.grad), xr.grad.permute(0, 2, 3, 1)) < 2e-5
    # stride-2 conv + BN + ReLU through the phase decomposition, and the 3-channel stem through the patch form
    for (n, h, w, cin, cout, k) in [(2, 31, 31, 128, 128, 3), (2, 31, 31, 256, 512, 1), (2, 65, 65, 3, 64, 3)]:
        torch.manual_seed(0)
        conv = torch.nn.Conv2d(cin, cout, k, stride=2, padding=k // 2, bias=False).cuda()
        bn = torch.nn.BatchNorm2d(cout).cuda()
        torch.nn.init.uniform_(bn.weight, 0.5, 1.5)
        torch.nn.init.normal_(bn.bias, 0, 0.2)
        xin = torch.randn((n, cin, h, w), device="cuda", generator=g)
        xi = SF.to_nhwc_bf16(xin)
        need_dx = cin % 64 == 0
        if need_dx:
            xi.requires_grad_(True)
        yy = SF.conv_bn_act(xi, conv, bn, relu=True)
        xr = _f32(xi.detach()).permute(0, 3, 1, 2)[:, :cin].contiguous().requires_grad_(True)
        wr = conv.weight.detach().clone().requires_grad_(True)
        gr, br = bn.weight.detach().clone().requires_grad_(True), bn.bias.detach().clone().requires_grad_(True)
        yr = torch.relu(F.batch_norm(F.conv2d(xr, wr, None, 2, k // 2), None, None, gr, br, True, 0.1, 1e-5))
        assert util.rel_l2(_f32(yy), yr.permute(0, 2, 3, 1)) < 1e-4, (cin, cout, k)
        gy = _split(torch.randn(tuple(yy.shape[-4:]), device="cuda", generator=g))
        yy.backward(gy)
        yr.backward(_f32(gy).permute(0, 3, 1, 2))
        assert util.rel_l2(conv.weight.grad, wr.grad) < 1e-3 and util.rel_l2(bn.weight.grad, gr.grad) < 1e-3
        assert util.rel_l2(bn.bias.grad, br.grad) < 1e-3
        if need_dx:
            assert util.rel_l2(_f32(xi.grad).permute(0, 3, 1, 2), xr.grad) < 1e-3


def _bn_train(x, g, b):
    return F.batch_norm(x, None, None, g, b, True, 0.1, 1e-5)


@pytest.mark.parametrize("dil,planes", [(2, 256), (4, 512)])
def test_bottleneck_block_x3_vs_oracle(dil, planes):
    """The named kernel path (1x1 -> dilated 3x3 -> 1x1 + BN/ReLU/residual, model/resnet.py:74-94) in train mode.

    Forward vs the fp32 oracle: <= 1e-4. Gradients: ReLU's derivative is discontinuous, so a forward difference of
    eps flips the mask of ~0.8*eps of the elements and each flip is an O(1) change of that element's gradient: against
    the PLAIN fp32 oracle the gradient error floor is ~sqrt(0.8*eps) (3e-3 at eps = 1e-5; the fp32 reference against
    itself with another summation order, eps ~ 1e-6, sits at ~1e-3). The gradient kernels are therefore checked to
    <= 1e-3 against the fp32 oracle evaluated WITH THE SAME ReLU MASKS (mask-matched oracle: y = a * [our y > 0], exact
    fp32 forward and backward otherwise), and to the flip floor (<= 1e-2) against the plain oracle."""
    from semseg_b200.resnet import Bottleneck
    from semseg_b200 import functional as SF
    from oracle.torch_oracle import Oracle
    torch.manual_seed(0)
    blk = Bottleneck(planes * 4, planes).cuda()
    blk.conv2.dilation, blk.conv2.padding = (dil, dil), (dil, dil)
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            torch.nn.init.uniform_(m.weight, 0.5, 1.5)
            torch.nn.init.normal_(m.bias, 0, 0.2)
    x = torch.randn((2, planes * 4, 30, 30), device="cuda")
    sd = {"layer1.0." + k: v.detach().clone() for k, v in blk.state_dict().items()}
    for k, v in sd.items():
        if v.dtype.is_floating_point and "running" not in k:
            v.requires_grad_(True)
    orc = Oracle(sd)
    xi = SF.to_nhwc_bf16(x).requires_grad_(True)
    xo = _f32(xi.detach()).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yo = orc.bottleneck(xo, "layer1.0", 1, dil, False)
    yi = blk.forward_nhwc(xi)
    assert util.rel_l2(_f32(yi).permute(0, 3, 1, 2), yo) < 1e-4
    go = _split(torch.randn((2, 30, 30, planes * 4), device="cuda"))
    gof = _f32(go).permute(0, 3, 1, 2)
    yo.backward(gof)
    yi.backward(go)
    # plain oracle: mask-flip floor
    assert util.rel_l2(_f32(xi.grad).permute(0, 3, 1, 2), xo.grad) < 1e-2
    for k, p in blk.named_parameters():
        assert util.rel_l2(p.grad, sd["layer1.0." + k].grad) < 1e-2, k
    # mask-matched oracle: the stage outputs of the same kernels give the masks (stage-by-stage == fused, bit for bit)
    with torch.no_grad():
        y1 = SF.conv_bn_act(xi.detach(), blk.conv1, blk.bn1, relu=True)
        y2 = SF.conv_bn_act(y1, blk.conv2, blk.bn2, relu=True)
    m1 = (_f32(y1) > 0).permute(0, 3, 1, 2).float()
    m2 = (_f32(y2) > 0).permute(0, 3, 1, 2).float()
    m3 = (_f32(yi.detach()) > 0).permute(0, 3, 1, 2).float()
    w = {k: v.detach().clone().requires_grad_(True) for k, v in blk.named_parameters()}
    xm = xo.detach().clone().requires_grad_(True)
    a1 = _bn_train(F.conv2d(xm, w["conv1.weight"]), w["bn1.weight"], w["bn1.bias"]) * m1
    a2 = _bn_train(F.conv2d(a1, w["conv2.weight"], padding=dil, dilation=dil), w["bn2.weight"], w["bn2.bias"]) * m2
    a3 = (_bn_train(F.conv2d(a2, w["conv3.weight"]), w["bn3.weight"], w["bn3.bias"]) + xm) * m3
    a3.backward(gof)
    e_dx = util.rel_l2(_f32(xi.grad).permute(0, 3, 1, 2), xm.grad)
    e_p = {k: util.rel_l2(p.grad, w[k].grad) for k, p in blk.named_parameters()}
    print("bottleneck d%d bf16x3 mask-matched: dx %.2e, worst param %.2e" % (dil, e_dx, max(e_p.values())))
    assert e_dx < 1e-3, e_dx
    assert all(v < 1e-3 for v in e_p.values()), e_p


def test_ppm_block_x3_vs_torch():
    """PPM (model/pspnet.py:8-26) in train mode with both gradient paths of x: forward <= 1e-4; gradients <= 1e-3 against
    the fp32 reference evaluated with the same ReLU masks (see the Bottleneck test), <= 1e-2 against the plain one."""
    import copy
    from semseg_b200.pspnet import PPM
    from semseg_b200 import functional as SF
    torch.manual_seed(3)
    n, h, w, c, cr, bins = 6, 24, 24, 128, 64, (1, 2, 3, 6)
    ppm = PPM(c, cr, bins).cuda().train()
    ref = copy.deepcopy(ppm)
    ref2 = copy.deepcopy(ppm)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = _split(torch.randn((n, h, w, c), device="cuda", generator=g)).requires_grad_(True)
    go = _split(torch.randn((n, h, w, c + len(bins) * cr), device="cuda", generator=g))
    out = ppm.forward_nhwc(x)
    out.backward(go)
    with torch.no_grad():   # branch outputs of the same kernels -> ReLU masks
        pooled = SF.ppm_pool(x.detach(), bins)
        masks = [(_f32(SF.conv_bn_act(p_, f[1], f[2], relu=True)) > 0).permute(0, 3, 1, 2).float()
                 for p_, f in zip(pooled, copy.deepcopy(ppm).features)]

    def reference(mod, use_masks):
        xr = _f32(x.detach()).permute(0, 3, 1, 2).requires_grad_(True)
        feats = [xr]
        for i, f in enumerate(mod.features):
            y = _bn_train(F.conv2d(F.adaptive_avg_pool2d(xr, f[0].output_size), f[1].weight), f[2].weight, f[2].bias)
            y = y * masks[i] if use_masks else torch.relu(y)
            feats.append(F.interpolate(y, (h, w), mode="bilinear", align_corners=True))
        o = torch.cat(feats, 1)
        o.backward(_f32(go).permute(0, 3, 1, 2))
        return o, xr.grad

    out_ref, dx_ref = reference(ref, False)
    assert util.rel_l2(_f32(out).permute(0, 3, 1, 2), out_ref) < 1e-4
    assert util.rel_l2(_f32(x.grad).permute(0, 3, 1, 2), dx_ref) < 1e-2
    _, dx_m = reference(ref2, True)
    e_dx = util.rel_l2(_f32(x.grad).permute(0, 3, 1, 2), dx_m)
    errs = {}
    for (k, p), (_, q) in zip(ppm.named_parameters(), ref2.named_parameters()):
        if "features.0" in k:
            continue     # bin 1: BatchNorm over n = 6 single-pixel samples, analytically ~zero gradients (noise / noise)
        errs[k] = util.rel_l2(p.grad, q.grad)
    print("ppm bf16x3 mask-matched: dx %.2e, worst param %.2e" % (e_dx, max(errs.values())))
    assert e_dx < 1e-3, e_dx
    assert all(v < 1e-3 for v in errs.values()), errs


def _eval_parity(arch, size, classes, n):
    build = util.build_pspnet if arch == "psp" else util.build_psanet
    mk = 2 * ((size - 1) // 16 + 1) - 1
    okw = {} if arch == "psp" else dict(mask_h=mk, mask_w=mk)
    bkw = {} if arch == "psp" else dict(mask=mk)
    model = build(50, classes, **bkw).cuda()
    orc, sd = util.oracle_from(model, arch, layers=50, classes=classes, **okw)
    x, y = util.synth(n, size, size, classes, device="cuda")
    model.eval()
    orc.eval()
    with torch.no_grad():
        lo = orc.forward(x)
        lm = model(x)
    e = util.rel_l2(lm, lo)
    am, ao = lm.argmax(1), lo.argmax(1)
    flips = int((am != ao).sum().item())
    # margin-aware count (SURVEY.md §7 c): flips at pixels whose oracle top-1 / top-2 gap exceeds twice the max error
    top2 = lo.topk(2, dim=1).values
    gap = top2[:, 0] - top2[:, 1]
    max_err = float((lm - lo).abs().max())
    hard = int(((am != ao) & (gap > 2 * max_err)).sum().item())
    return dict(model=model, orc=orc, sd=sd, x=x, y=y, rel_l2=e, flips=flips, hard_flips=hard, max_err=max_err,
                pixels=am.numel(), min_gap=float(gap.min()))


def _train_loss_parity(r, tol):
    model, orc, x, y = r["model"], r["orc"], r["x"], r["y"]
    model.train()
    orc.train()
    _, ml, al = model(x, y)
    (ml + 0.4 * al).backward()
    _, mlo, alo = orc.forward(x, y)
    assert abs(ml.item() - mlo.item()) < tol * abs(mlo.item()), (ml.item(), mlo.item())
    assert abs(al.item() - alo.item()) < tol * abs(alo.item()), (al.item(), alo.item())
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in model.parameters())


def test_pspnet50_473_eval_logits_1e3_and_exact_argmax():
    """north_star parity gate, BASELINE config-2 shape: PSPNet50 @ 473x473, 150 classes, fresh model, eval."""
    r = _eval_parity("psp", 473, 150, 2)
    print("PSPNet50@473 bf16x3: rel_l2 %.3e, max abs err %.3e, argmax flips %d / %d (margin-aware %d), min top-2 gap %.3e"
          % (r["rel_l2"], r["max_err"], r["flips"], r["pixels"], r["hard_flips"], r["min_gap"]))
    assert r["rel_l2"] <= 1e-4, r["rel_l2"]                   # north_star: 1e-3
    assert r["hard_flips"] == 0                               # no flip outside the fp32 near-tie pixels
    assert r["flips"] <= 64, (r["flips"], r["pixels"])        # near-tie floor of 16-bit operands (module docstring)
    _train_loss_parity(r, 1e-4)


def test_psanet50_465_eval_logits_1e3_and_exact_argmax():
    """north_star parity gate, BASELINE config-3 shape: PSANet50 @ 465x465 (59x59 maps, 59x59 mask), fresh model, eval."""
    r = _eval_parity("psa", 465, 150, 2)
    print("PSANet50@465 bf16x3: rel_l2 %.3e, max abs err %.3e, argmax flips %d / %d (margin-aware %d), min top-2 gap %.3e"
          % (r["rel_l2"], r["max_err"], r["flips"], r["pixels"], r["hard_flips"], r["min_gap"]))
    assert r["rel_l2"] <= 1e-4, r["rel_l2"]
    assert r["hard_flips"] == 0
    assert r["flips"] <= 64, (r["flips"], r["pixels"])
    _train_loss_parity(r, 1e-4)


def test_pspnet101_config4_shape_x3_eval_and_losses():
    """BASELINE config 4 per-GPU shard (PSPNet101, 713x713 -> 90x90 maps, 19 classes, 2 images): eval logits, losses and
    gradient norms against the fp32 oracle."""
    model = util.build_pspnet(101, 19).cuda()
    orc, sd = util.oracle_from(model, "psp", layers=101, classes=19)
    x, y = util.synth(2, 713, 713, 19, device="cuda")
    model.eval()
    orc.eval()
    with torch.no_grad():
        lo, lm = orc.forward(x), model(x)
    assert util.rel_l2(lm, lo) <= 2e-4
    top2 = lo.topk(2, dim=1).values
    flips = lm.argmax(1) != lo.argmax(1)
    hard = flips & ((top2[:, 0] - top2[:, 1]) > 2 * float((lm - lo).abs().max()))
    print("PSPNet101@713 bf16x3: rel_l2 %.3e, argmax flips %d / %d (margin-aware %d)" %
          (util.rel_l2(lm, lo), int(flips.sum()), flips.numel(), int(hard.sum())))
    assert int(hard.sum()) == 0 and int(flips.sum()) <= 128
    model.train()
    orc.train()
    _, ml, al = model(x, y)
    (ml + 0.4 * al).backward()
    _, mlo, alo = orc.forward(x, y)
    (mlo + 0.4 * alo).backward()
    assert abs(ml.item() - mlo.item()) < 1e-4 * mlo.item() and abs(al.item() - alo.item()) < 1e-4 * alo.item()
    # head gradients are upstream of nothing chaotic: element-wise; backbone: magnitudes (train-mode BN nets are chaotic)
    params = dict(model.named_parameters())
    for k in ("cls.4.weight", "cls.4.bias", "aux.4.weight", "aux.4.bias"):
        assert util.rel_l2(params[k].grad, sd[k].grad) < 2e-2, k
    for k, p in params.items():
        a, b = float(p.grad.double().norm()), float(sd[k].grad.double().norm())
        if b > 1e-6 and "ppm.features.0" not in k:
            assert 0.5 < a / b < 2.0, (k, a, b)
