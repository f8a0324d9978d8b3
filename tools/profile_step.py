"""Per-kernel breakdown of one training step (torch.profiler / CUPTI) + CPU enqueue time vs GPU time.
Usage (on the GPU box): python tools/profile_step.py [--batch 16] [--size 473] [--arch psp]"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--layers", type=int, default=50)
    ap.add_argument("--arch", default="psp")
    ap.add_argument("--out", default="profile_out/profile_step.txt")
    ap.add_argument("--ncu", action="store_true", help="run exactly one step between cudaProfilerStart/Stop")
    args = ap.parse_args()
    from model.pspnet import PSPNet
    from model.psanet import PSANet
    torch.manual_seed(0)
    if args.arch == "psp":
        model = PSPNet(layers=args.layers, classes=args.classes, zoom_factor=8, pretrained=False).cuda()
    else:
        mk = 2 * ((args.size - 1) // 16 + 1) - 1
        model = PSANet(layers=args.layers, classes=args.classes, zoom_factor=8, mask_h=mk, mask_w=mk,
                       pretrained=False).cuda()
    opt = bench.build_optimizer(model, args.arch)
    model.train()
    x, y = bench.synth_batch(args.batch, args.size, args.classes, 0)
    x, y = x.cuda(), y.cuda()

    def step():
        _, ml, al = model(x, y)
        loss = ml + 0.4 * al
        opt.zero_grad()
        loss.backward()
        opt.step()

    for _ in range(8):          # eager warm-up + (unless SEMSEG_B200_GRAPH=0) capture of the step graphs
        step()
    torch.cuda.synchronize()
    if args.ncu:
        torch.cuda.cudart().cudaProfilerStart()
        step()
        torch.cuda.synchronize()
        torch.cuda.cudart().cudaProfilerStop()
        return
    # CPU enqueue time vs GPU time
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        step()
    e1.record()
    t_cpu = (time.perf_counter() - t0) / 3
    torch.cuda.synchronize()
    t_gpu = e0.elapsed_time(e1) / 3
    lines = ["cpu enqueue %.1f ms/step, gpu %.1f ms/step" % (t_cpu * 1e3, t_gpu)]
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    agg = {}
    for e in ev:
        a = agg.setdefault(e.name, [0.0, 0])
        a[0] += e.device_time
        a[1] += 1
    tot = sum(v[0] for v in agg.values())
    lines.append("total kernel time %.2f ms over %d launches" % (tot / 1e3, sum(v[1] for v in agg.values())))
    for name, (t, c) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:45]:
        lines.append("%8.3f ms %5.1f%% x%-4d %s" % (t / 1e3, 100 * t / tot, c, name[:110]))
    # per-launch spread of the short, many-launch kernels (latency-bound candidates)
    per = {}
    for e in ev:
        per.setdefault(e.name, []).append(e.device_time)
    for name, ts in per.items():
        if len(ts) >= 16 and any(k in name for k in ("wgrad_reduce", "bn_finalize", "bn_bwd_reduce_final", "pack_w")):
            ts = sorted(ts)
            lines.append("  spread %-40s min %.1f  median %.1f  p90 %.1f  max %.1f us" %
                         (name.split("(")[0][-40:], ts[0], ts[len(ts) // 2], ts[int(len(ts) * 0.9)], ts[-1]))
    txt = "\n".join(lines)
    print(txt)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    open(args.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
