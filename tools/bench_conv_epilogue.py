"""Per-shape timing of the fprop/dgrad convolution kernel (`conv_igemm_kernel`) in each of its bf16 epilogues.

The shapes are those of bench.py's step (PSPNet50 473x473, 150 classes, 16 images by default): one eager training step
runs with `ops.conv_fprop` wrapped, which records every distinct geometry (input, packed weights, Cout, taps, phase
offsets, output grid) and whether the module's forward (`fprop`) or its input gradient (`dgrad`) launched it. Each
geometry is then run on fresh seeded bf16 tensors in three epilogues:
  * raw_stats : RAW + the batch-statistics rows (what a batch-statistics BN forward launches);
  * affine_res: AFFINE with scale, shift, residual and ReLU (eval-mode conv+BN+residual; the dgrad gradient fan-in is
                the same epilogue without scale and shift);
  * raw       : plain RAW (no statistics).
Every launch is timed with CUDA events, the 50 MB L2 flushed before each one, as bench.py's roofline does.

`--lib NAME=PATH` (repeatable) loads several builds of libsemseg_b200.so into the one process and times them
alternately, launch by launch, on the same tensors; the outputs (and statistics rows) of every build are compared with
the first one's by `torch.equal`. Prints one JSON line per (geometry, epilogue) with the median ms, TFLOP/s and output
GB/s of each build, then a summary line with the GPU, its power limit and the SM clock read in the same process, and
the per-epilogue totals of one step's launches (each geometry weighted by how often the step launched it)."""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["SEMSEG_B200_GRAPH"] = "0"      # the recording step must run the Python path

import torch  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import _lib, ops  # noqa: E402

EPILOGUES = ("raw_stats", "affine_res", "raw")


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, power, sm, sm_max = [s.strip() for s in q.stdout.strip().split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, subprocess.SubprocessError, ValueError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown", "sm_clock": "unknown"}


def record_shapes(batch, size, classes, layers):
    """{geometry: launches per step} of one eager training step of bench.py's PSPNet."""
    from model.pspnet import PSPNet
    seen = collections.Counter()
    orig = ops.conv_fprop

    def wrapped(x, w3d, cout, taps, **kw):
        caller = sys._getframe(1).f_code.co_name
        if kw.get("epi", ops.EPI_RAW) != ops.EPI_F32 and not ops.is_split(x):
            n, h, w, c = x.shape[-4:]
            key = (caller if caller in ("fprop", "dgrad") else "other", (n, h, w, c), tuple(w3d.shape), cout,
                   tuple(tuple(t) for t in taps), tuple(kw["img_add"]) if kw.get("img_add") else None,
                   tuple(kw["out_nhw"]) if kw.get("out_nhw") else None)
            seen[key] += 1
        return orig(x, w3d, cout, taps, **kw)

    torch.manual_seed(0)
    model = PSPNet(layers=layers, classes=classes, zoom_factor=8, pretrained=False).cuda().train()
    x, y = bench.synth_batch(batch, size, classes, 0)
    ops.conv_fprop = wrapped
    try:
        _, ml, al = model(x.cuda(), y.cuda())
        (ml + 0.4 * al).backward()
        torch.cuda.synchronize()
    finally:
        ops.conv_fprop = orig
    del model
    torch.cuda.empty_cache()
    return seen


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build of libsemseg_b200.so to time (repeatable; default: the package's own)")
    ap.add_argument("--reps", type=int, default=7, help="timed launches per build, geometry and epilogue")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--layers", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    libs = {}
    for spec in args.lib or ["this=" + _lib.LIB_PATH]:
        name, path = spec.split("=", 1)
        _lib._lib, _lib.LIB_PATH = None, os.path.abspath(path)
        libs[name] = _lib.load()
    names = list(libs)

    def use(name):
        _lib._lib = libs[name]

    use(names[0])
    shapes = record_shapes(args.batch, args.size, args.classes, args.layers)
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    totals = {e: {nm: 0.0 for nm in names} for e in EPILOGUES}
    all_equal = True
    for (role, xs, ws, cout, taps, img_add, out_nhw), count in sorted(shapes.items(), key=lambda kv: str(kv[0])):
        n, h, w = out_nhw if out_nhw else xs[:3]
        x = torch.randn(xs, device=dev, generator=g).to(torch.bfloat16)
        w3d = (torch.randn(ws, device=dev, generator=g) * 0.05).to(torch.bfloat16)
        scale = torch.rand(cout, device=dev, generator=g) + 0.5
        shift = torch.randn(cout, device=dev, generator=g) * 0.1
        res = torch.randn((n, h, w, cout), device=dev, generator=g).to(torch.bfloat16)
        flops = 2.0 * n * h * w * xs[3] * cout * len(taps)
        out_bytes = 2.0 * n * h * w * cout
        for epi in EPILOGUES:
            kw = dict(img_add=list(img_add) if img_add else None, out_nhw=out_nhw)
            if epi == "raw_stats":
                kw["stats"] = True
            elif epi == "affine_res":
                kw.update(epi=ops.EPI_AFFINE, scale=scale, shift=shift, residual=res, relu=True)
            outs, ts = {}, {nm: [] for nm in names}
            for nm in names:               # warm-up launch, kept for the bit comparison
                use(nm)
                outs[nm] = ops.conv_fprop(x, w3d, cout, list(taps), **kw)
            for _ in range(args.reps):
                for nm in names:
                    use(nm)
                    flush.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    ops.conv_fprop(x, w3d, cout, list(taps), **kw)
                    b.record()
                    torch.cuda.synchronize()
                    ts[nm].append(a.elapsed_time(b))
            ref_y, ref_sp = outs[names[0]]
            equal = all(torch.equal(y, ref_y) and (sp is None or torch.equal(sp, ref_sp)) for y, sp in outs.values())
            all_equal &= equal
            line = {"role": role, "x": list(xs), "cout": cout, "taps": len(taps), "phases": img_add is not None,
                    "launches_per_step": count, "epilogue": epi, "bits_equal": equal}
            for nm in names:
                ms = sorted(ts[nm])[len(ts[nm]) // 2]
                totals[epi][nm] += ms * count
                line[nm] = {"ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1),
                            "out_gbs": round(out_bytes / ms / 1e6, 1)}
            print(json.dumps(line), flush=True)
            del outs
    summary = dict(_gpu_info(), shapes=len(shapes), all_bits_equal=all_equal,
                   step_ms={e: {nm: round(v, 3) for nm, v in d.items()} for e, d in totals.items()})
    print(json.dumps(summary), flush=True)
    use(names[0])


if __name__ == "__main__":
    main()
