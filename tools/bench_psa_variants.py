"""Training-step throughput of PSANet's attention options: the fused kernels against the ATen composition.

PSANet50 at BASELINE's config-3 shape (465x465, 150 classes, 59x59 feature maps, 30x30 attention), one GPU, the default
`bf16` mode, bench.py's step (tool/train.py:267-276: model(input, target), loss = main + 0.4 aux, zero_grad, backward, SGD
with the reference's 8 parameter groups). For each of the four (compact, psa_softmax) combinations two arms run:
  * fused: csrc/psa_fused.cu, mask gather (compact: the dense form) -> softmax (or none) -> aggregation in one kernel;
  * aten : SEMSEG_B200_PSA_FUSED=0, psa_mask (compact: the dense view) -> softmax -> bmm in ATen.
The mask is sized as tool/train.py:63-70 sizes it: 30x30 compact, 59x59 windowed. Every arm is a copy of one seeded model
per combination, built, warmed up and (when graphs are on) captured under its own SEMSEG_B200_PSA_FUSED setting, because a
captured graph does not read the setting again. Arms alternate within a round and rounds repeat (`--rounds`), at 16 and at
2 images per step. After the warm-up `--steps` steps are timed with CUDA events. Prints one JSON line per round,
combination, batch size and arm, with the GPU name and power limit read in the same process. Not part of bench.py's
contract.
"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit"] = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = "unknown"
    return info


def time_arm(base, fused, x, y, steps, n_warm):
    """Build, warm up (and capture) a copy of `base` under its own SEMSEG_B200_PSA_FUSED setting; ms per step."""
    prev = os.environ.get("SEMSEG_B200_PSA_FUSED")
    os.environ["SEMSEG_B200_PSA_FUSED"] = "1" if fused else "0"
    try:
        model = copy.deepcopy(base).cuda().train()
        opt = bench.build_optimizer(model, "psa")

        def step():
            _, main_loss, aux_loss = model(x, y)
            loss = main_loss + 0.4 * aux_loss
            opt.zero_grad()
            loss.backward()
            opt.step()

        for _ in range(n_warm):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        kernels = graphs.launches_per_step(model)
        del model, opt
        torch.cuda.empty_cache()
        return e0.elapsed_time(e1) / steps, kernels
    finally:
        if prev is None:
            os.environ.pop("SEMSEG_B200_PSA_FUSED", None)
        else:
            os.environ["SEMSEG_B200_PSA_FUSED"] = prev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per arm, batch size and round")
    ap.add_argument("--warmup", type=int, default=3, help="eager steps per arm before the graph warm-up")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batches", default="16,2", help="images per step, comma separated")
    ap.add_argument("--size", type=int, default=465)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--layers", type=int, default=50)
    ap.add_argument("--psa-type", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_psa_variants measures on a GPU; there is no CPU arm"
    from model.psanet import PSANet

    info = _gpu_info()
    n_warm = max(3, args.warmup) + (graphs.WARMUP_CALLS + 1 if graphs.enabled() else 0)
    h = (args.size - 1) // 16 + 1
    combos = [(c, s) for c in (False, True) for s in (True, False)]
    bases = {}
    for compact, softmax in combos:
        mask = h if compact else 2 * h - 1
        torch.manual_seed(0)
        bases[compact, softmax] = (PSANet(layers=args.layers, classes=args.classes, zoom_factor=8, psa_type=args.psa_type,
                                          compact=compact, mask_h=mask, mask_w=mask, psa_softmax=softmax,
                                          pretrained=False), mask)
    data = {n: tuple(t.cuda() for t in bench.synth_batch(n, args.size, args.classes, 100))
            for n in (int(b) for b in args.batches.split(","))}
    for rnd in range(args.rounds):
        for (compact, softmax), (base, mask) in bases.items():
            for n, (x, y) in data.items():
                arms = ("fused", "aten") if rnd % 2 == 0 else ("aten", "fused")
                for arm in arms:
                    ms, kernels = time_arm(base, arm == "fused", x, y, args.steps, n_warm)
                    print(json.dumps(dict(info, round=rnd, compact=compact, psa_softmax=softmax, mask=mask, arm=arm,
                                          batch=n, img_per_s=n / (ms / 1e3), ms_per_step=ms,
                                          kernels_per_graphed_step=kernels,
                                          workload="PSANet%d psa_type %d %dx%d, %d classes, bf16, one GPU" % (
                                              args.layers, args.psa_type, args.size, args.size, args.classes))),
                          flush=True)


if __name__ == "__main__":
    main()
