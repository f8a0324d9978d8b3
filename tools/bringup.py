"""GPU bring-up diagnostics for the CUDA kernels (needs an H100).

Each check runs in its own subprocess under a timeout so that a trapped / failed kernel (sticky CUDA
error) does not take the remaining checks down. Prints error patterns, not just pass/fail, because a
round-trip to the GPU box is expensive.  Usage: python tools/bringup.py [check ...]
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _ref_conv(x_nhwc, w, dil):
    import torch
    import torch.nn.functional as F
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    xf = x_nhwc.float().permute(0, 3, 1, 2)
    wf = w.to(torch.bfloat16).float()
    k = w.shape[-1]
    y = F.conv2d(xf, wf, padding=dil * (k // 2), dilation=dil)
    return y.permute(0, 2, 3, 1).contiguous()


def _report(name, got, ref, tol):
    import torch
    got = got.float()
    err = (got - ref).abs()
    scale = ref.abs().max().item() + 1e-12
    mx = err.max().item()
    rel = mx / scale
    bad = torch.isnan(got).sum().item()
    ok = rel < tol and bad == 0
    print("%-46s max_abs_err %.4e  ref_max %.4e  rel %.3e  nan %d  %s" % (name, mx, scale, rel, bad,
                                                                           "OK" if ok else "FAIL"), flush=True)
    if not ok:
        # error pattern: by channel block of 8 and by pixel index mod 128
        e = err.reshape(-1, err.shape[-1])
        per_c = e.max(dim=0).values
        print("   worst channels:", torch.topk(per_c, min(8, per_c.numel())).indices.tolist())
        per_p = e.max(dim=1).values
        idx = torch.topk(per_p, min(8, per_p.numel())).indices.tolist()
        print("   worst pixels (flat):", idx)
        cb = per_c.reshape(-1, 8).max(dim=1).values
        print("   err by 8-channel block:", ["%.2e" % v for v in cb[:32].tolist()])
        print("   got[0,0,0,:8] ", got.reshape(-1, got.shape[-1])[0, :8].tolist())
        print("   ref[0,0,0,:8] ", ref.reshape(-1, ref.shape[-1])[0, :8].tolist())
    return ok


def check_psamask():
    import numpy as np
    import torch
    import oracle
    from semseg_b200 import ops
    ok = True
    rng = np.random.default_rng(0)
    for (N, H, W, mH, mW) in [(2, 4, 5, 7, 9), (1, 6, 7, 5, 3), (2, 5, 5, 9, 9), (2, 30, 30, 59, 59),
                              (1, 8, 8, 21, 21)]:
        for t in (0, 1):
            x = rng.standard_normal((N, mH * mW, H, W)).astype(np.float32)
            g = rng.standard_normal((N, H * W, H, W)).astype(np.float32)
            o = ops.psamask_fwd(torch.from_numpy(x).cuda(), t, mH, mW).cpu().numpy()
            d = ops.psamask_bwd(torch.from_numpy(g).cuda(), t, mH, mW).cpu().numpy()
            e1 = np.array_equal(o, oracle.psamask_fwd(x, t, mH, mW))
            e2 = np.array_equal(d, oracle.psamask_bwd(g, t, mH, mW))
            print("psamask", (N, H, W, mH, mW), "type", t, "fwd", e1, "bwd", e2, flush=True)
            ok &= e1 and e2
    return ok


def _conv_case(N, H, W, cin, cout, k, dil, seed=0):
    import torch
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((N, H, W, cin), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.0 / (cin * k * k) ** 0.5)
    pw = ops.pack_weights(w)
    y, sp = ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(k, dil), stats=True)
    torch.cuda.synchronize()
    ref = _ref_conv(x, w, dil)
    name = "fprop N%d %dx%d cin%d cout%d k%d d%d" % (N, H, W, cin, cout, k, dil)
    ok = _report(name, y, ref, 8e-3)
    # statistics of the stored bf16 tensor
    st = ops.bn_merge_partials(sp)
    yf = y.float().reshape(-1, cout)
    mean_ref = yf.mean(0)
    var_ref = yf.var(0, unbiased=False)
    cnt = st[2]
    me = (st[0] - mean_ref).abs().max().item()
    ve = ((st[1] / cnt) - var_ref).abs().max().item() / (var_ref.max().item() + 1e-12)
    cnt_ok = bool((cnt == yf.shape[0]).all().item())
    sok = me < 1e-4 and ve < 1e-4 and cnt_ok
    print("   stats: mean err %.3e  var rel err %.3e  count ok %s  %s" % (me, ve, cnt_ok, "OK" if sok else "FAIL"),
          flush=True)
    return ok and sok


def check_conv_small():
    ok = True
    ok &= _conv_case(1, 8, 16, 64, 64, 1, 1)      # one full 128-pixel tile, single k-block
    ok &= _conv_case(1, 8, 16, 128, 128, 1, 1)    # two k-blocks, BLOCK_N=128
    ok &= _conv_case(2, 12, 12, 64, 256, 1, 1)    # partial tiles, BLOCK_N=256
    ok &= _conv_case(1, 8, 16, 64, 64, 3, 1)      # taps + halo
    return ok


def check_conv_shapes():
    ok = True
    ok &= _conv_case(2, 60, 60, 256, 256, 3, 2)
    ok &= _conv_case(2, 60, 60, 512, 512, 3, 4)
    ok &= _conv_case(2, 60, 60, 1024, 256, 1, 1)
    ok &= _conv_case(2, 60, 60, 512, 2048, 1, 1)
    ok &= _conv_case(1, 119, 119, 64, 64, 3, 1)
    ok &= _conv_case(2, 59, 59, 256, 512, 3, 1)
    ok &= _conv_case(1, 90, 90, 256, 256, 3, 2)
    return ok


def check_conv_epilogues():
    import torch
    from semseg_b200 import ops
    ok = True
    g = torch.Generator(device="cuda").manual_seed(1)
    N, H, W, cin, cout = 2, 30, 30, 128, 256
    x = torch.randn((N, H, W, cin), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn((cout, cin, 3, 3), device="cuda", generator=g) * 0.03
    res = torch.randn((N, H, W, cout), device="cuda", generator=g).to(torch.bfloat16)
    scale = torch.rand((cout,), device="cuda", generator=g) + 0.5
    shift = torch.randn((cout,), device="cuda", generator=g)
    pw = ops.pack_weights(w)
    y, _ = ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(3, 1), epi=ops.EPI_AFFINE, relu=True, scale=scale,
                             shift=shift, residual=res)
    ref = torch.relu(_ref_conv(x, w, 1) * scale + shift + res.float())
    ok &= _report("affine+residual+relu epilogue", y, ref, 8e-3)
    # fp32 epilogue with bias and Cout = 150
    cout2 = 150
    w2 = torch.randn((cout2, cin, 1, 1), device="cuda", generator=g) * 0.05
    b2 = torch.randn((cout2,), device="cuda", generator=g)
    pw2 = ops.pack_weights(w2)
    y2, _ = ops.conv_fprop(x, pw2.wf, cout2, ops.conv_taps(1, 1), epi=ops.EPI_F32, shift=b2)
    ref2 = _ref_conv(x, w2, 1) + b2
    ok &= _report("fp32 epilogue, bias, Cout=150", y2, ref2, 2e-3)
    # output into a channel slice of a wider buffer
    buf = torch.zeros((N, H, W, 512), device="cuda", dtype=torch.bfloat16)
    ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(3, 1), out=buf[..., 256:512])
    ok &= _report("raw epilogue into channel slice", buf[..., 256:512], _ref_conv(x, w, 1), 8e-3)
    ok &= bool((buf[..., :256] == 0).all().item())
    return ok


def check_dgrad_wgrad():
    import torch
    import torch.nn.functional as F
    from semseg_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    ok = True
    g = torch.Generator(device="cuda").manual_seed(2)
    for (N, H, W, cin, cout, k, dil) in [(1, 8, 16, 64, 64, 1, 1), (2, 30, 30, 128, 256, 3, 2),
                                          (2, 60, 60, 256, 256, 3, 2), (2, 60, 60, 512, 128, 1, 1),
                                          (1, 30, 30, 64, 512, 3, 4)]:
        x = torch.randn((N, H, W, cin), device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn((cout, cin, k, k), device="cuda", generator=g) * 0.05)
        dy = torch.randn((N, H, W, cout), device="cuda", generator=g).to(torch.bfloat16)
        xf = x.float().permute(0, 3, 1, 2).requires_grad_(True)
        wf = w.to(torch.bfloat16).float().requires_grad_(True)
        yref = F.conv2d(xf, wf, padding=dil * (k // 2), dilation=dil)
        yref.backward(dy.float().permute(0, 3, 1, 2))
        dx_ref = xf.grad.permute(0, 2, 3, 1).contiguous()
        dw_ref = wf.grad
        pw = ops.pack_weights(w)
        dx, _ = ops.conv_fprop(dy, pw.wd, cin, ops.conv_taps(k, dil, transpose=True))
        tag = "N%d %dx%d cin%d cout%d k%d d%d" % (N, H, W, cin, cout, k, dil)
        ok &= _report("dgrad " + tag, dx, dx_ref, 8e-3)
        dw = ops.conv_wgrad(x, dy, cin, cout, ops.conv_taps(k, dil))
        ok &= _report("wgrad " + tag, dw.reshape(cout, -1), dw_ref.reshape(cout, -1), 2e-3)
    return ok


def check_bn():
    import torch
    from semseg_b200 import ops
    ok = True
    g = torch.Generator(device="cuda").manual_seed(3)
    N, H, W, C = 2, 30, 30, 256
    x = (torch.randn((N, H, W, C), device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)
    gamma = torch.rand((C,), device="cuda", generator=g) + 0.5
    beta = torch.randn((C,), device="cuda", generator=g)
    rm = torch.zeros(C, device="cuda")
    rv = torch.ones(C, device="cuda")
    v = x.float().reshape(-1, C)      # fp32 moments of x: (mean, M2, count)
    st = torch.stack([v.mean(0), v.var(0, unbiased=False) * v.shape[0], torch.full((C,), float(v.shape[0]),
                                                                                   device="cuda")])
    mi, ss = ops.bn_finalize(st, gamma, beta, 1e-5, 0.1, rm, rv)
    res = torch.randn((N, H, W, C), device="cuda", generator=g).to(torch.bfloat16)
    y = ops.bn_apply(x, ss, residual=res, relu=True)
    xf = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    gm = gamma.clone().requires_grad_(True)
    bt = beta.clone().requires_grad_(True)
    rm2 = torch.zeros(C, device="cuda")
    rv2 = torch.ones(C, device="cuda")
    rf = res.float().permute(0, 3, 1, 2).requires_grad_(True)
    yref = torch.relu(torch.nn.functional.batch_norm(xf, rm2, rv2, gm, bt, True, 0.1, 1e-5) + rf)
    ok &= _report("bn_apply fwd", y, yref.permute(0, 2, 3, 1), 1e-2)
    ok &= _report("running_mean", rm[None], rm2[None], 1e-4)
    ok &= _report("running_var", rv[None], rv2[None], 1e-4)
    dy = torch.randn((N, H, W, C), device="cuda", generator=g).to(torch.bfloat16)
    # reference backward uses the same relu mask as our bf16 output (mask from our y)
    mask = (y.float() > 0).permute(0, 3, 1, 2)
    pre = torch.nn.functional.batch_norm(xf, None, None, gm, bt, True, 0.1, 1e-5) + rf
    (pre * mask * dy.float().permute(0, 3, 1, 2)).sum().backward()
    _, sums = ops.bn_bwd_reduce(dy, y, x, mi, True)
    dx, dres, dgb = ops.bn_bwd_apply(dy, y, x, mi, gamma, sums, float(N * H * W), True, want_dres=True)
    ok &= _report("bn bwd dx", dx, xf.grad.permute(0, 2, 3, 1), 1e-2)
    ok &= _report("bn bwd dres", dres, rf.grad.permute(0, 2, 3, 1), 1e-2)
    ok &= _report("bn bwd dgamma", dgb[0][None], gm.grad[None], 1e-3)
    ok &= _report("bn bwd dbeta", dgb[1][None], bt.grad[None], 1e-3)
    return ok


def check_layout():
    import torch
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn((2, 3, 17, 23), device="cuda", generator=g)
    y = ops.nchw_to_nhwc_bf16(x)
    ok = _report("nchw->nhwc bf16 (C=3 padded to 8)", y[..., :3], x.permute(0, 2, 3, 1).to(torch.bfloat16).float(),
                 1e-6)
    ok &= bool((y[..., 3:] == 0).all().item())
    z = torch.randn((2, 9, 11, 150), device="cuda", generator=g)
    ok &= _report("nhwc f32 -> nchw", ops.nhwc_f32_to_nchw(z).permute(0, 2, 3, 1), z, 1e-7)
    return ok


def check_perf():
    import torch
    from semseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for (N, H, W, cin, cout, k, dil) in [(16, 60, 60, 512, 512, 3, 4), (16, 60, 60, 256, 256, 3, 2),
                                          (16, 60, 60, 4096, 512, 3, 1), (16, 60, 60, 1024, 256, 1, 1),
                                          (16, 60, 60, 512, 2048, 1, 1), (16, 119, 119, 64, 64, 3, 1)]:
        x = torch.randn((N, H, W, cin), device="cuda", generator=g).to(torch.bfloat16)
        w = torch.randn((cout, cin, k, k), device="cuda", generator=g) * 0.02
        dy = torch.randn((N, H, W, cout), device="cuda", generator=g).to(torch.bfloat16)
        pw = ops.pack_weights(w)
        flops = 2.0 * N * H * W * cin * cout * k * k
        def timeit(fn, iters=5):
            fn()
            ts = []
            for _ in range(iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            return sorted(ts)[len(ts) // 2]
        t_f = timeit(lambda: ops.conv_fprop(x, pw.wf, cout, ops.conv_taps(k, dil), stats=True))
        t_d = timeit(lambda: ops.conv_fprop(dy, pw.wd, cin, ops.conv_taps(k, dil, transpose=True)))
        t_w = timeit(lambda: ops.conv_wgrad(x, dy, cin, cout, ops.conv_taps(k, dil)))
        print("perf N%d %dx%d cin%d cout%d k%d d%d: fprop %.3f ms %.0f TF/s | dgrad %.3f ms %.0f TF/s | wgrad %.3f ms "
              "%.0f TF/s" % (N, H, W, cin, cout, k, dil, t_f, flops / t_f / 1e9, t_d, flops / t_d / 1e9, t_w,
                             flops / t_w / 1e9), flush=True)
    return True


CHECKS = {
    "psamask": check_psamask,
    "layout": check_layout,
    "bn": check_bn,
    "conv_small": check_conv_small,
    "conv_shapes": check_conv_shapes,
    "conv_epilogues": check_conv_epilogues,
    "dgrad_wgrad": check_dgrad_wgrad,
    "perf": check_perf,
}


def main():
    names = sys.argv[1:] or list(CHECKS)
    if len(names) == 1 and os.environ.get("BRINGUP_CHILD") == "1":
        ok = CHECKS[names[0]]()
        sys.exit(0 if ok else 1)
    summary = {}
    for n in names:
        print("=" * 30, n, flush=True)
        env = dict(os.environ, BRINGUP_CHILD="1")
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), n], env=env, timeout=300)
            summary[n] = "OK" if r.returncode == 0 else "FAIL(rc=%d)" % r.returncode
        except subprocess.TimeoutExpired:
            summary[n] = "TIMEOUT"
    print("=" * 30, "SUMMARY", summary, flush=True)
    sys.exit(0 if all(v == "OK" for v in summary.values()) else 1)


if __name__ == "__main__":
    main()
