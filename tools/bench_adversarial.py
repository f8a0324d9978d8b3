"""Cost of the attacks and of PGD adversarial training (semseg_b200/adversarial.py, losses.AdversarialLoss).

Attack: a 10-iteration PGD and SegPGD attack (eps 8, alpha 2, random start), graphed, timed per call and reported per
iteration, against the idiom users write today on this package (eval model, frozen parameters, x.requires_grad_(),
eager F.cross_entropy on the upsampled logits, backward, sign step) and against oracle.torch_oracle.Oracle with the
same seeded weights on cuDNN (fp32 NCHW, torch's default TF32 settings), for PSPNet50 473x473 and PSANet50 465x465,
150 classes, 16 images by default.
Training: bench.py's PSPNet50 step (main + 0.4 aux, SGD), graphed, with plain cross-entropy and with AdversarialLoss at
K = 1 and 3.
Arms run alternately within each group, `--rounds` times, timed with CUDA events; each arm's peak memory
(torch.cuda.max_memory_allocated over its timed calls) and the native kernels per graphed training step are reported.
Prints JSON lines with the GPU, its power limit and SM clock, read in the same process.
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
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
from semseg_b200 import graphs  # noqa: E402
from semseg_b200.adversarial import PGDAttack  # noqa: E402
from semseg_b200.losses import AdversarialLoss  # noqa: E402

STEPS = 10
EPS, ALPHA = 8.0, 2.0


def _gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in q.stdout.strip().split(",")]
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = (vals + ["unknown"] * 3)[:3]
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = info["sm_clock"] = "unknown"
    return info


def _nets(arch, classes):
    from semseg_b200.psanet import PSANet
    from semseg_b200.pspnet import PSPNet
    torch.manual_seed(0)
    if arch == "psp":
        return PSPNet(layers=50, classes=classes, zoom_factor=8, pretrained=False), 473, {}
    return PSANet(layers=50, classes=classes, zoom_factor=8, psa_type=2, mask_h=59, mask_w=59,
                  pretrained=False), 465, dict(psa_type=2, mask_h=59, mask_w=59)


def _timed(fn, calls):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls, torch.cuda.max_memory_allocated() / 2 ** 30


def _attack_arms(arch, args, dev):
    """name -> (callable, iterations per call)."""
    from oracle.torch_oracle import Oracle
    model, size, okw = _nets(arch, args.classes)
    model = model.to(dev).eval()
    x0, y = bench.synth_batch(args.batch, size, args.classes, 100)
    x0, y = x0.to(dev), y.to(dev)
    arms = {}
    for kind in ("pgd", "segpgd"):
        atk = PGDAttack(EPS, ALPHA, STEPS, kind=kind)
        arms["%s_%s10_graphed" % (arch, kind)] = (lambda atk=atk: atk(model, x0, y), STEPS)
    # the hand-written idiom: frozen copies of the parameters, eager, ATen cross-entropy on the upsampled logits
    frozen = copy.deepcopy(model)
    for p in frozen.parameters():
        p.requires_grad_(False)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    orc = Oracle(sd, arch=arch, layers=50, classes=args.classes, **okw).eval()
    state = {"eager_aten": x0.clone(), "cudnn": x0.clone()}
    fwd = {"eager_aten": frozen, "cudnn": orc.forward}
    step = ALPHA / 58.0

    def it(name):
        def run():
            x = state[name].requires_grad_(True)
            F.cross_entropy(fwd[name](x), y, ignore_index=255).backward()
            with torch.no_grad():
                state[name] = (x + step * x.grad.sign()).detach()
        return run
    for k in fwd:
        arms["%s_attack_iteration_%s" % (arch, k)] = (it(k), 1)
    return arms


def _train_arms(args, dev):
    torch.manual_seed(0)
    base, _, _ = _nets("psp", args.classes)
    base = base.to(dev).train()
    x, y = bench.synth_batch(args.batch, 473, args.classes, 100)
    x, y = x.to(dev), y.to(dev)
    arms = {}
    for k in (0, 1, 3):
        m = copy.deepcopy(base)
        if k:
            m.criterion = AdversarialLoss(PGDAttack(EPS, 2.5 * EPS / k, k))
        opt = bench.build_optimizer(m, "psp")

        def run(m=m, opt=opt):
            _, ml, al = m(x, y)
            opt.zero_grad()
            (ml + 0.4 * al).backward()
            opt.step()
        arms["psp_train_%s" % ("ce" if k == 0 else "adv_k%d" % k)] = (run, m)
    return arms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=2, help="timed calls per round and arm")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--groups", default="psp,psa,train")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_adversarial measures on a GPU"
    dev = torch.device("cuda", 0)
    for group in args.groups.split(","):
        if group == "train":
            train = _train_arms(args, dev)
            arms = {k: (v[0], 1) for k, v in train.items()}
        else:
            arms = _attack_arms(group, args, dev)
        for fn, _ in arms.values():                 # eager warm-up, then the graph capture
            for _ in range(graphs.WARMUP_CALLS + 2):
                fn()
        ms = {k: [] for k in arms}
        peak = {k: 0.0 for k in arms}
        for _ in range(args.rounds):
            for name, (fn, iters) in arms.items():
                t, mem = _timed(fn, args.calls)
                ms[name].append(round(t / iters, 2))
                peak[name] = max(peak[name], round(mem, 2))
        rec = dict(_gpu_info(), group=group, batch=args.batch, classes=args.classes, precision="bf16",
                   eps=EPS, alpha=ALPHA, calls_per_round=args.calls, peak_gib=peak)
        if group == "train":
            rec["ms_per_step"] = ms
            rec["kernels_per_graphed_step"] = {k: graphs.launches_per_step(v[1]) for k, v in train.items()}
            del train
        else:
            rec["ms_per_iteration"] = ms
        print(json.dumps(rec), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
