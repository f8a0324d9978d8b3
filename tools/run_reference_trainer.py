"""Drive the reference's UNMODIFIED tool/train.py over this repository's drop-in packages (SURVEY.md §8 a16 / b1).

    python tools/run_reference_trainer.py [--gpus 2] [--arch psp|psa] [--iters 20] [--size 473] [--out profile_out/trainer]

What it does (nothing of the reference is edited):
  1. copies baseline/_ref (the untouched reference tree, baseline/install_reference.py) to a scratch directory — the
     trainer writes checkpoints / event files relative to its cwd;
  2. writes a small synthetic list-file dataset (JPEG images + PNG label maps read by util/dataset.py:63-66 through
     cv2.imread) and ./initmodel/resnet50_v2.pth (model/resnet.py:199 loads it with strict=False);
  3. puts two shims on PYTHONPATH via sitecustomize: `collections.Iterable` (removed in Python 3.10, used by
     util/transform.py:79) and a no-op `tensorboardX.SummaryWriter` (tool/train.py:18) — neither touches arithmetic;
  4. runs   PYTHONPATH=<this repo>:<shims>:.  python tool/train.py --config=config/ade20k/ade20k_<arch>50.yaml KEY VAL ...
     from the scratch copy. `model.pspnet` / `model.psanet` / `lib.psa.functional` resolve to THIS repository (regular
     packages shadow the reference's namespace directories, SURVEY.md Appendix E); `util/`, `tool/`, `config/` are the
     reference's. The trainer spawns one process per GPU (mp.spawn), converts to SyncBatchNorm and wraps in
     DistributedDataParallel itself (tool/train.py:141-157); with `evaluate True` it also runs validate()
     (tool/train.py:343-397: model.eval()(input) WITHOUT torch.no_grad()).
The trainer's log is copied to <out>/train_log.txt and a summary line is printed.
"""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref")

SITECUSTOMIZE = '''
import collections, collections.abc, sys, types
if not hasattr(collections, "Iterable"):
    collections.Iterable = collections.abc.Iterable          # util/transform.py:79,118,171
if "tensorboardX" not in sys.modules:
    tb = types.ModuleType("tensorboardX")
    class SummaryWriter(object):                                # tool/train.py:18,147
        def __init__(self, *a, **k): pass
        def add_scalar(self, *a, **k): pass
        def close(self): pass
    tb.SummaryWriter = SummaryWriter
    sys.modules["tensorboardX"] = tb
'''


def make_dataset(root, n_train, n_val, classes, h=300, w=400, seed=0):
    import cv2
    import numpy as np
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    os.makedirs(os.path.join(root, "labels"), exist_ok=True)
    os.makedirs(os.path.join(root, "list"), exist_ok=True)
    lists = {"training": [], "validation": []}
    for k in range(n_train + n_val):
        img = (rng.random((h // 20 + 1, w // 20 + 1, 3)) * 255).astype(np.uint8)
        img = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)            # smooth colour blobs
        lab = rng.integers(0, classes, size=(h // 50 + 1, w // 50 + 1)).astype(np.uint8)
        lab = cv2.resize(lab, (w, h), interpolation=cv2.INTER_NEAREST)           # blocky class regions
        lab[rng.random((h, w)) < 0.03] = 255                                     # ignore label
        ip, lp = "images/%04d.jpg" % k, "labels/%04d.png" % k
        cv2.imwrite(os.path.join(root, ip), img)
        cv2.imwrite(os.path.join(root, lp), lab)
        lists["training" if k < n_train else "validation"].append("%s %s" % (ip, lp))
    for name, lines in lists.items():
        with open(os.path.join(root, "list", name + ".txt"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--arch", default="psp", choices=["psp", "psa"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--per-gpu", type=int, default=4)
    ap.add_argument("--size", type=int, default=473)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--out", default=os.path.join(ROOT, "profile_out", "trainer"))
    ap.add_argument("--keep", action="store_true")
    a = ap.parse_args()
    if not os.path.isdir(os.path.join(REF, "tool")):
        sys.path.insert(0, os.path.join(ROOT, "baseline"))
        import install_reference
        if install_reference.install() is None:
            print("baseline/_ref is absent and /root/reference does not exist: cannot run the reference trainer")
            return 2
    work = tempfile.mkdtemp(prefix="semseg_trainer_")
    ref = os.path.join(work, "ref")
    shutil.copytree(REF, ref)
    shims = os.path.join(work, "shims")
    os.makedirs(shims)
    with open(os.path.join(shims, "sitecustomize.py"), "w") as fh:
        fh.write(SITECUSTOMIZE)

    # synthetic dataset: iterations = epochs * floor(n_train / global_batch); 5 iterations per epoch
    gb = a.per_gpu * a.gpus
    per_epoch = 5
    epochs = max(1, (a.iters + per_epoch - 1) // per_epoch)
    data = os.path.join(work, "data")
    make_dataset(data, gb * per_epoch, gb, a.classes)

    # ./initmodel/resnet50_v2.pth: random-init backbone under a fixed seed (no network access for the real checkpoint)
    sys.path.insert(0, ROOT)
    import torch
    from semseg_b200 import resnet as our_resnet
    torch.manual_seed(0)
    os.makedirs(os.path.join(ref, "initmodel"))
    torch.save(our_resnet.resnet50(pretrained=False).state_dict(), os.path.join(ref, "initmodel", "resnet50_v2.pth"))

    cfg = "config/ade20k/ade20k_%s50.yaml" % ("pspnet" if a.arch == "psp" else "psanet")
    save = os.path.join(work, "exp")
    os.makedirs(save)
    opts = ["data_root", data, "train_list", os.path.join(data, "list", "training.txt"), "val_list",
            os.path.join(data, "list", "validation.txt"), "classes", str(a.classes), "train_gpu",
            "[" + ",".join(str(i) for i in range(a.gpus)) + "]", "batch_size", str(gb), "batch_size_val", str(gb),
            "epochs", str(epochs), "workers", "4", "print_freq", "1", "save_freq", str(epochs), "save_path", save,
            "train_h", str(a.size), "train_w", str(a.size), "evaluate", "True"]
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, shims, "."])
    cmd = [sys.executable, "tool/train.py", "--config=" + cfg] + opts
    print("cwd=%s\n$ PYTHONPATH=%s %s" % (ref, env["PYTHONPATH"], " ".join(cmd)), flush=True)
    r = subprocess.run(cmd, cwd=ref, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    os.makedirs(a.out, exist_ok=True)
    log = os.path.join(a.out, "train_log_%s_%dgpu.txt" % (a.arch, a.gpus))
    with open(log, "w") as fh:
        fh.write("$ cd <scratch copy of baseline/_ref> && PYTHONPATH=<repo>:<shims>:. python " + " ".join(cmd[1:]) + "\n")
        fh.write(r.stdout)
    iters = re.findall(r"Epoch: \[(\d+)/(\d+)\]\[(\d+)/(\d+)\].*?MainLoss ([0-9.]+) AuxLoss ([0-9.]+) Loss ([0-9.]+)", r.stdout)
    val = re.findall(r"Val result: mIoU/mAcc/allAcc ([0-9.]+)/([0-9.]+)/([0-9.]+)", r.stdout)
    ckpt = [f for f in os.listdir(save) if f.endswith(".pth")]
    which = subprocess.run([sys.executable, "-c", "import model.pspnet, lib.psa.functional as f; "
                            "print(model.pspnet.__file__, f.__file__)"], cwd=ref, env=env, capture_output=True, text=True)
    print("model package used by the trainer:", which.stdout.strip())
    ok = r.returncode == 0 and len(iters) >= a.iters and len(val) >= 1 and len(ckpt) >= 1
    if iters:
        print("iterations logged: %d; first loss %s, last loss %s" % (len(iters), iters[0][6], iters[-1][6]))
    print("validation passes: %d %s; checkpoints: %s" % (len(val), val[-1:] if val else "", ckpt))
    print("reference trainer over the drop-in packages: rc=%d -> %s (log: %s)" % (r.returncode, "OK" if ok else "FAIL",
                                                                               os.path.relpath(log, ROOT)))
    if not ok:
        print(r.stdout[-3000:])
    if not a.keep:
        shutil.rmtree(work, ignore_errors=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
